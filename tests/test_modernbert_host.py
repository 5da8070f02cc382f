"""CPU: ModernBERT retrievers — dispatch and the published shapes, every refusal with its message, layer types / windows / RoPE
frequencies bit for bit against transformers for both config spellings, the synthetic directories and the masked-LM checkpoint
layout, the tokenizer, and the batches built with it against the reference's builders."""
import os

import pytest
import torch


def _cfg(name="modernbert-tiny", **kw):
    from dalm_b200 import synthetic
    return dict(synthetic.modernbert_config(name), **kw)


def _hf_config(cfg):
    from transformers import ModernBertConfig
    return ModernBertConfig(**{k: v for k, v in cfg.items() if k not in ("architectures", "model_type")})


@pytest.mark.parametrize("name", ["modernbert-tiny", "modernbert-hd64", "ModernBERT-base", "gte-modernbert-base",
                                  "modernbert-embed-base", "ModernBERT-large"])
def test_dispatch(name):
    from dalm_b200.engine import params
    cfg = _cfg(name)
    assert params.model_kind(cfg) == "modernbert"
    assert (cfg["vocab_size"], cfg["pad_token_id"], cfg["norm_eps"], cfg["max_position_embeddings"]) == (50368, 50283, 1e-5, 8192)


def test_published_shapes():
    want = {"ModernBERT-base": (768, 1152, 22, 12), "gte-modernbert-base": (768, 1152, 22, 12),
            "modernbert-embed-base": (768, 1152, 22, 12), "ModernBERT-large": (1024, 2624, 28, 16)}
    for n, w in want.items():
        c = _cfg(n)
        assert (c["hidden_size"], c["intermediate_size"], c["num_hidden_layers"], c["num_attention_heads"]) == w, n
        assert (c["local_attention"], c["global_attn_every_n_layers"], c["global_rope_theta"], c["local_rope_theta"]) == \
            (128, 3, 160000.0, 10000.0)
    assert {n: _cfg(n)["hidden_size"] // _cfg(n)["num_attention_heads"] for n in ("modernbert-tiny", "modernbert-hd64")} == \
        {"modernbert-tiny": 32, "modernbert-hd64": 64}


@pytest.mark.parametrize("setting,value,match", [
    ("attention_dropout", 0.1, "attention_dropout=0.1"),
    ("mlp_dropout", 0.1, "mlp_dropout=0.1"),
    ("embedding_dropout", 0.1, "embedding_dropout=0.1"),
    ("hidden_activation", "gelu_new", "hidden_activation='gelu_new'"),
    ("hidden_activation", "silu", "hidden_activation='silu'"),
    ("norm_bias", True, "norm_bias=true"),
    ("mlp_bias", True, "mlp_bias=true"),
    ("attention_bias", True, "attention_bias=true"),
    ("rope_scaling", {"rope_type": "linear", "factor": 2.0}, "RoPE type 'linear'"),
    ("rope_parameters", {"full_attention": {"rope_type": "dynamic", "factor": 2.0, "rope_theta": 1e5}}, "RoPE type 'dynamic'"),
    ("num_attention_heads", 4, "head_dim 16"),
])
def test_refusals(setting, value, match):
    from dalm_b200.engine import params
    from dalm_b200.engine.modernbert import ModernBertEncoder
    cfg = _cfg(**{setting: value})
    with pytest.raises(NotImplementedError, match=match):
        params.model_kind(cfg)
    with pytest.raises(NotImplementedError, match=match):
        ModernBertEncoder(cfg, params.random_state_dict("modernbert", _cfg(), seed=0), device="cpu")


def test_modernbert_decoder_is_refused():
    from dalm_b200.engine import params
    with pytest.raises(NotImplementedError, match="model_type 'modernbert-decoder' is not built"):
        params.model_kind(dict(_cfg(), model_type="modernbert-decoder"))


def test_mode_refusals(monkeypatch, tmp_path):
    from dalm_b200.engine import params
    from dalm_b200.engine.modernbert import ModernBertEncoder
    from dalm_b200.models.rag_e2e_base_model import build_decoder, build_encoder
    from dalm_b200.training.utils.train_utils import load_adapter_dir
    cfg = _cfg()
    sd = params.random_state_dict("modernbert", cfg, seed=0)
    cpu = torch.device("cpu")
    with pytest.raises(NotImplementedError, match=r"query / key / value.*--no-use-peft"):
        build_encoder("", True, cpu, state_dict=sd, cfg=cfg)
    with pytest.raises(NotImplementedError, match="query / key / value"):
        ModernBertEncoder(cfg, sd, device="cpu", lora=True)
    with pytest.raises(NotImplementedError, match="use_bnb on a ModernBERT retriever.*needs LoRA"):
        build_encoder("", False, cpu, state_dict=sd, cfg=cfg, full=True, bnb=True)
    with pytest.raises(NotImplementedError, match="retriever_is_autoregressive=True: ModernBERT is a bidirectional encoder"):
        build_encoder("", False, cpu, state_dict=sd, cfg=cfg, autoregressive=True, full=True)
    with pytest.raises(NotImplementedError, match="generator of kind 'modernbert' is not a causal decoder"):
        build_decoder("", False, cpu, state_dict=sd, cfg=cfg)
    monkeypatch.setenv("DALM_B200_NF4_STORAGE", "1")
    with pytest.raises(NotImplementedError, match="DALM_B200_NF4_STORAGE=1: 4-bit storage is not built for ModernBERT"):
        build_encoder("", False, cpu, state_dict=sd, cfg=cfg, bnb=True)
    frozen = build_encoder("", False, cpu, state_dict=sd, cfg=cfg)          # eval-retriever / eval-rag: frozen bf16
    assert frozen.full is None and not frozen.trainable
    with pytest.raises(NotImplementedError, match="query / key / value"):
        load_adapter_dir(frozen, str(tmp_path))                                # attach_pre_trained_peft_layers(retriever)


def _spellings():
    """(our config, what the hub / transformers 5 writes) pairs covering both spellings of layer types and RoPE theta"""
    base = _cfg("modernbert-tiny")
    legacy = dict(base, num_hidden_layers=7, global_attn_every_n_layers=2, global_rope_theta=80000.0, local_rope_theta=5000.0)
    legacy_default = {k: v for k, v in base.items() if k not in ("global_attn_every_n_layers", "global_rope_theta",
                                                                  "local_rope_theta")}
    new = {k: v for k, v in base.items() if k not in ("global_attn_every_n_layers", "global_rope_theta", "local_rope_theta")}
    new.update(num_hidden_layers=5, layer_types=["full_attention", "sliding_attention", "full_attention", "full_attention",
                                                 "sliding_attention"],
               rope_parameters={"full_attention": {"rope_type": "default", "rope_theta": 123456.0},
                                "sliding_attention": {"rope_type": "default", "rope_theta": 7777.0}})
    mixed = dict(new, rope_parameters={"full_attention": {"rope_type": "default"}}, local_rope_theta=2500.0, local_attention=64)
    return {"legacy": legacy, "legacy-default": legacy_default, "transformers5": new, "mixed": mixed,
            "large": _cfg("ModernBERT-large")}


@pytest.mark.parametrize("which", ["legacy", "legacy-default", "transformers5", "mixed", "large"])
def test_layers_windows_and_frequencies_match_transformers(which):
    from transformers.models.modernbert.modeling_modernbert import ModernBertRotaryEmbedding

    from dalm_b200.engine import params
    cfg = _spellings()[which]
    hc = _hf_config(cfg)
    rot = ModernBertRotaryEmbedding(hc)
    got = params.modernbert_layers(cfg)
    assert len(got) == hc.num_hidden_layers and hc.layer_types[0] == "full_attention"
    for (w, f), lt in zip(got, hc.layer_types):
        assert w == (hc.sliding_window + 1 if lt == "sliding_attention" else 0)
        assert f.dtype == torch.float32 and torch.equal(f, getattr(rot, f"{lt}_inv_freq")), (which, lt)
    assert params.modernbert_layer_types(cfg) == list(hc.layer_types)
    # the same resolution from the config.json transformers itself writes
    saved = hc.to_dict()
    assert [w for w, _ in params.modernbert_layers(saved)] == [w for w, _ in got]
    assert all(torch.equal(a[1], b[1]) for a, b in zip(params.modernbert_layers(saved), got))


def test_random_state_dict_norms_are_not_one():
    from dalm_b200.engine import params
    sd = params.random_state_dict("modernbert", _cfg(), seed=0)
    assert "layers.0.attn_norm.weight" not in sd and "layers.1.attn_norm.weight" in sd
    for k in ("embeddings.norm.weight", "layers.1.attn_norm.weight", "layers.0.mlp_norm.weight", "final_norm.weight"):
        assert not torch.equal(sd[k], torch.ones_like(sd[k])) and (sd[k] - 1).abs().max() < 0.2, k
    assert sd["layers.0.mlp.Wi.weight"].shape == (2 * 96, 64) and sd["layers.0.attn.Wqkv.weight"].shape == (192, 64)


@pytest.mark.parametrize("name", ["modernbert-tiny", "modernbert-hd64"])
def test_synthetic_dirs_load_in_transformers(tmp_path, name):
    from transformers import AutoModel, AutoTokenizer, ModernBertModel

    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.modernbert import _hf_names
    d = synthetic.write_model_dir(str(tmp_path / name), "modernbert", name)
    m = ModernBertModel.from_pretrained(d)
    assert type(AutoModel.from_pretrained(d)).__name__ == "ModernBertModel"
    ours, theirs = params.load_state_dict(d), m.state_dict()
    assert set(ours) == set(theirs)
    for k, v in ours.items():
        assert torch.equal(theirs[k], v), k
    assert m.embeddings.tok_embeddings.padding_idx == 50283
    # a ModernBertForMaskedLM checkpoint (answerdotai/ModernBERT-*): `model.` prefix plus head.* / decoder.*
    mlm = {"model." + k: v for k, v in ours.items()}
    mlm.update({"head.dense.weight": torch.zeros(1), "head.norm.weight": torch.zeros(1), "decoder.bias": torch.zeros(1)})
    assert {k: v for k, v in _hf_names(mlm).items()} .keys() == ours.keys()
    assert AutoTokenizer.from_pretrained(d).pad_token_id == 50283


def test_masked_lm_layout_matches_transformers():
    from transformers import ModernBertForMaskedLM

    from dalm_b200.engine.modernbert import _hf_names
    hc = _hf_config(_cfg())
    mlm = ModernBertForMaskedLM(hc).state_dict()
    from transformers import ModernBertModel
    assert set(_hf_names(mlm)) == set(ModernBertModel(hc).state_dict())


def test_tokenizer_layout(tmp_path):
    from transformers import AutoTokenizer

    from dalm_b200 import synthetic
    tok = AutoTokenizer.from_pretrained(synthetic.build_modernbert_tokenizer(str(tmp_path / "tok")))
    assert len(tok) == 50368
    assert (tok.unk_token_id, tok.cls_token_id, tok.sep_token_id, tok.pad_token_id, tok.mask_token_id) == \
        (50280, 50281, 50282, 50283, 50284)
    assert tok.padding_side == "right" and "token_type_ids" not in tok.model_input_names
    enc = tok(["#query# kato mi ren", "#passage# sol"], padding="max_length", max_length=16)
    assert "token_type_ids" not in enc
    for ids, mask in zip(enc["input_ids"], enc["attention_mask"]):
        n = sum(mask)
        assert ids[0] == 50281 and ids[n - 1] == 50282 and all(i < 50280 for i in ids[1:n - 1])     # [CLS] ... [SEP]
        assert ids[n:] == [50283] * (16 - n)
    assert tok.decode(enc["input_ids"][0], skip_special_tokens=True).strip() == "#query# kato mi ren"


def _gen_tokenizer():
    from transformers import AutoTokenizer
    t = AutoTokenizer.from_pretrained(os.path.join(os.path.dirname(__file__), "golden", "tok_llama"))
    t.pad_token = t.eos_token
    t.add_eos_token = True
    return t


def test_batches_match_reference(tmp_path):
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference tree not available")
    from transformers import AutoTokenizer

    from dalm_b200 import synthetic
    from dalm_b200.training.utils.rag_e2e_dataloader_utils import preprocess_dataset as pre_e2e
    from dalm_b200.training.utils.retriever_only_dataloader_utils import preprocess_dataset as pre_ret
    ref = ref_import.load()
    tok = AutoTokenizer.from_pretrained(synthetic.build_modernbert_tokenizer(str(tmp_path / "tok")))
    norm = lambda v: [list(x) if isinstance(x, (list, tuple)) else (x.tolist() if hasattr(x, "tolist") else x) for x in v]
    rows = list(synthetic.synthetic_rows(12, seed=5))
    ex = {k: [r[k] for r in rows] for k in ("Abstract", "Question", "Answer")}
    kw = dict(query_column_name="Question", passage_column_name="Abstract", answer_column_name="Answer", query_max_len=50,
              passage_max_len=128, generator_max_len=256)
    got = pre_e2e(ex, retriever_tokenizer=tok, generator_tokenizer=_gen_tokenizer(), **kw)
    want = ref.preprocess_e2e(ex, retriever_tokenizer=tok, generator_tokenizer=_gen_tokenizer(), **kw)
    assert set(got) == set(want)
    for k in want:
        assert norm(got[k]) == norm(want[k]), k
    assert not any(k.endswith("token_type_ids") for k in got)
    assert all(x[0] == 50281 for x in got["retriever_query_input_ids"])
    kw = dict(query_column_name="Question", passage_column_name="Abstract", query_max_len=32, passage_max_len=200)
    ex = {k: ex[k] for k in ("Abstract", "Question")}
    got, want = pre_ret(ex, tokenizer=tok, **kw), ref.preprocess_retriever(ex, tokenizer=tok, **kw)
    assert set(got) == set(want)
    for k in want:
        assert norm(got[k]) == norm(want[k]), k
