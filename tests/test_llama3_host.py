"""CPU: Llama 3.x generators / autoregressive retrievers — the RoPE frequencies of every built type bit for bit against
transformers' rope init functions, the tables of the configs without scaling unchanged, the RoPE types that are refused, the
synthetic Llama 3 directories against transformers' LlamaForCausalLM, and the batches built with the Llama 3 tokenizer
against the reference's builders."""
import math
import os

import pytest
import torch


def _hf_inv_freq(cfg):
    """transformers' own frequencies for an HF config dict: (inv_freq, attention factor)"""
    from transformers import LlamaConfig
    from transformers.modeling_rope_utils import ROPE_INIT_FUNCTIONS
    c = LlamaConfig(**{k: v for k, v in cfg.items() if k not in ("architectures", "model_type")})
    rt = c.rope_parameters["rope_type"]
    if rt == "default":
        from transformers.models.llama.modeling_llama import LlamaRotaryEmbedding
        return LlamaRotaryEmbedding.compute_default_rope_parameters(c)
    return ROPE_INIT_FUNCTIONS[rt](c)


def _old_inv_freq(theta, hd):
    """the frequencies the decoders built before scaling was supported (kept here to pin that they do not move)"""
    return 1.0 / (float(theta) ** (torch.arange(0, hd, 2, dtype=torch.float32) / hd))


def _llama2(**kw):
    from dalm_b200 import synthetic
    return dict(synthetic.llama_config("llama-tiny", vocab_size=400), **kw)


def _to_rope_parameters(cfg):
    """transformers 5's spelling of the same config: `rope_parameters` carrying rope_theta, no top-level rope_theta"""
    out = {k: v for k, v in cfg.items() if k not in ("rope_scaling", "rope_theta")}
    out["rope_parameters"] = dict(cfg.get("rope_scaling") or {"rope_type": "default"}, rope_theta=cfg["rope_theta"])
    return out


def _published():
    from dalm_b200 import synthetic
    return {n: synthetic.llama3_config(n) for n in ("llama-3.1-8b", "llama-3.2-1b", "llama-3.2-3b", "llama-3.3-70b")}


@pytest.mark.parametrize("name", ["llama-3.1-8b", "llama-3.2-1b", "llama-3.2-3b", "llama-3.3-70b", "llama3-tiny", "llama3.2-tiny",
                                  "llama2-linear-2", "llama2-linear-4", "llama2-linear-legacy-type"])
@pytest.mark.parametrize("spelling", ["rope_scaling", "rope_parameters"])
def test_inv_freq_bitwise_equal_to_transformers(name, spelling):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    if name.startswith("llama2-linear"):
        key = "type" if "legacy" in name else "rope_type"
        cfg = _llama2(rope_scaling={key: "linear", "factor": 4.0 if name.endswith("4") else 2.0})
    else:
        cfg = synthetic.llama3_config(name, vocab_size=400)
    if spelling == "rope_parameters":
        cfg = _to_rope_parameters(cfg)
    hd = cfg.get("head_dim") or cfg["hidden_size"] // cfg["num_attention_heads"]
    ref, attention_factor = _hf_inv_freq(cfg)
    ours = params.rope_inv_freq(cfg, hd)
    assert attention_factor == 1.0                                   # the cos / sin tables need no post-scaling
    assert ours.dtype == torch.float32 and ours.shape == (hd // 2,)
    assert torch.equal(ours, ref), (ours - ref).abs().max()
    assert not torch.equal(ours, _old_inv_freq(params.rope_parameters(cfg)["rope_theta"], hd))   # the scaling does something
    assert params.model_kind(cfg) == "llama"


def test_llama31_8b_differs_from_default_in_35_frequencies():
    from dalm_b200.engine import params
    cfg = _published()["llama-3.1-8b"]
    assert cfg["rope_scaling"] == {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                   "original_max_position_embeddings": 8192}
    assert (params.rope_inv_freq(cfg, 128) != _old_inv_freq(500000.0, 128)).sum().item() == 35


@pytest.mark.parametrize("name,hd", [("llama3-tiny", 128), ("llama3.2-tiny", 64)])
def test_tiny_configs_hit_every_llama3_band(name, hd):
    """original_max_position_embeddings = 64 puts frequencies in all three bands at the tiny head_dims: kept, divided by
    factor, and blended (strictly between the two)"""
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    cfg = synthetic.llama3_config(name, vocab_size=400)
    rs = cfg["rope_scaling"]
    assert cfg["head_dim"] == hd and cfg["num_key_value_heads"] < cfg["num_attention_heads"]
    base = _old_inv_freq(cfg["rope_theta"], hd)
    got = params.rope_inv_freq(cfg, hd)
    wavelen = 2 * math.pi / base
    orig = rs["original_max_position_embeddings"]
    kept = wavelen < orig / rs["high_freq_factor"]
    divided = wavelen > orig / rs["low_freq_factor"]
    blended = ~kept & ~divided
    assert kept.any() and divided.any() and blended.any(), (kept.sum(), divided.sum(), blended.sum())
    assert torch.equal(got[kept], base[kept])
    assert torch.equal(got[divided], base[divided] / rs["factor"])
    b = blended
    assert ((got[b] < base[b]) & (got[b] > base[b] / rs["factor"])).all()


@pytest.mark.parametrize("kind,name", [("llama", "llama-tiny"), ("llama", "llama-hd128"), ("llama", "Llama-2-7b-hf"),
                                       ("qwen2", "qwen2-tiny"), ("qwen2", "qwen2.5-7b"), ("qwen3", "qwen3-tiny"),
                                       ("qwen3", "qwen3-8b"), ("falcon", "falcon-tiny"), ("falcon", "falcon-7b")])
def test_tables_without_scaling_unchanged(kind, name):
    """configs without RoPE scaling: the frequencies and the decoders' cos / sin tables are bit for bit the ones built before,
    and equal transformers' default"""
    from types import SimpleNamespace

    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.falcon import FalconDecoder
    from dalm_b200.engine.llama import LlamaDecoder
    cfg = getattr(synthetic, f"{kind}_config")(name)
    hd = cfg.get("head_dim") or cfg["hidden_size"] // cfg["num_attention_heads"]
    inv = params.rope_inv_freq(cfg, hd)
    old = _old_inv_freq(cfg["rope_theta"], hd)
    assert torch.equal(inv, old)
    if kind != "falcon":
        assert torch.equal(inv, _hf_inv_freq(cfg)[0])
    L = 300
    fr = torch.outer(torch.arange(L, dtype=torch.float32), old)
    for cls in (LlamaDecoder, FalconDecoder):
        fake = SimpleNamespace(inv_freq=inv, _rope_cache={}, dev=torch.device("cpu"))
        cos_t, sin_t = cls._rope(fake, L)
        assert torch.equal(cos_t, fr.cos()) and torch.equal(sin_t, fr.sin())
        assert cls._rope(fake, L)[0] is cos_t                             # cached per L


@pytest.mark.parametrize("rope", [
    {"rope_type": "dynamic", "factor": 2.0},
    {"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 8192},
    {"type": "yarn", "factor": 4.0, "original_max_position_embeddings": 8192},
    {"rope_type": "longrope", "short_factor": [1.0] * 32, "long_factor": [2.0] * 32, "original_max_position_embeddings": 4096},
    {"rope_type": "proportional", "partial_rotary_factor": 0.5},
    {"rope_type": "ntk-by-parts", "factor": 2.0},
])
@pytest.mark.parametrize("spelling", ["rope_scaling", "rope_parameters"])
def test_llama_refuses_unbuilt_rope_types(rope, spelling):
    from dalm_b200.engine import params
    cfg = _llama2(**{spelling: dict(rope, rope_theta=10000.0) if spelling == "rope_parameters" else rope})
    rt = rope.get("rope_type", rope.get("type"))
    with pytest.raises(NotImplementedError, match=rt):
        params.model_kind(cfg)
    with pytest.raises(NotImplementedError, match=rt):
        params.rope_inv_freq(cfg, 64)


@pytest.mark.parametrize("rope", [{"rope_type": "linear", "factor": 2.0}, {"type": "dynamic", "factor": 2.0},
                                  {"rope_type": "llama3", "factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                   "original_max_position_embeddings": 8192}])
def test_falcon_refuses_scaled_rope(rope):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.falcon import FalconDecoder
    cfg = dict(synthetic.falcon_config("falcon-tiny", 400), rope_scaling=rope)
    rt = rope.get("rope_type", rope.get("type"))
    with pytest.raises(NotImplementedError, match=rt):
        params.model_kind(cfg)
    with pytest.raises(NotImplementedError, match=rt):
        FalconDecoder(cfg, params.random_state_dict("falcon", cfg, seed=0), device="cpu")
    assert params.model_kind(synthetic.falcon_config("falcon-tiny", 400)) == "falcon"


def test_llama_decoder_refuses_before_building():
    from dalm_b200.engine.llama import LlamaDecoder
    with pytest.raises(NotImplementedError, match="yarn"):
        LlamaDecoder(_llama2(rope_scaling={"rope_type": "yarn", "factor": 4.0}), {}, device="cpu")


def test_published_shapes():
    from dalm_b200.engine import params
    want = {"llama-3.1-8b": (4096, 32, 8, 128, 14336, False, 8.0), "llama-3.2-1b": (2048, 16, 8, 64, 8192, True, 32.0),
            "llama-3.2-3b": (3072, 28, 8, 128, 8192, True, 32.0), "llama-3.3-70b": (8192, 80, 8, 128, 28672, False, 8.0)}
    for n, c in _published().items():
        got = (c["hidden_size"], c["num_hidden_layers"], c["num_key_value_heads"], c["head_dim"], c["intermediate_size"],
               c["tie_word_embeddings"], c["rope_scaling"]["factor"])
        assert got == want[n], n
        assert c["vocab_size"] == 128256 and c["rope_theta"] == 500000.0 and c["model_type"] == "llama"
        assert c["head_dim"] == c["hidden_size"] // c["num_attention_heads"]
        assert params.model_kind(c) == "llama"


def test_synthetic_llama3_dirs_load_in_transformers(tmp_path):
    """the synthetic directories load in LlamaForCausalLM with equal state dicts (tied and untied), and its rotary embedding
    holds our frequencies"""
    from transformers import LlamaForCausalLM

    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    for name, tied in (("llama3-tiny", False), ("llama3.2-tiny", True)):
        d = synthetic.write_model_dir(str(tmp_path / name), "llama", name, vocab_size=504,
                                      generation_config=synthetic.LLAMA3_GENERATION["instruct"])
        m = LlamaForCausalLM.from_pretrained(d)
        cfg = params.load_config(d)
        ours = params.load_state_dict(d)
        theirs = m.state_dict()
        assert set(ours) == set(theirs) - ({"lm_head.weight"} if tied else set())
        for k, v in ours.items():
            assert torch.equal(theirs[k], v), k
        assert (m.lm_head.weight.data_ptr() == m.model.embed_tokens.weight.data_ptr()) == tied
        assert m.config.rope_parameters["rope_type"] == "llama3"
        hf_inv = m.model.rotary_emb.inv_freq
        assert torch.equal(hf_inv, params.rope_inv_freq(cfg, cfg["head_dim"]))
        assert m.model.rotary_emb.attention_scaling == 1.0
        assert m.generation_config.eos_token_id == [1, 3, 2] and m.generation_config.do_sample


def test_llama3_tokenizer_layout(tmp_path):
    import json

    from transformers import AutoTokenizer

    from dalm_b200 import synthetic
    d = synthetic.build_llama3_tokenizer(str(tmp_path / "tok"), 504)
    with open(os.path.join(d, "tokenizer_config.json")) as f:
        tc = json.load(f)
    assert "add_bos_token" not in tc and "add_eos_token" not in tc and tc["tokenizer_class"] == "PreTrainedTokenizerFast"
    tok = AutoTokenizer.from_pretrained(d)
    assert len(tok) == 504
    assert tok.convert_tokens_to_ids(synthetic.LLAMA3_SPECIAL) == [0, 1, 2, 3]
    assert (tok.bos_token, tok.eos_token) == ("<|begin_of_text|>", "<|end_of_text|>")
    text = "#query# kato mi ren, 123 exsol"
    ids = tok(text)["input_ids"]
    assert ids[0] == 0 and 0 not in ids[1:] and 1 not in ids                 # BOS from the post-processor, no EOS
    assert tok.decode(ids, skip_special_tokens=True) == text
    assert tok.decode(ids[:1]) == "<|begin_of_text|>"


def _trainer_tokenizer(d):
    """a generator tokenizer set up as the trainer does it (reference train_rage2e.py:301-304), which is also how an
    autoregressive retriever's tokenizer is set up (rag_e2e_base_model.py:41-44 of the reference)"""
    from transformers import AutoTokenizer
    t = AutoTokenizer.from_pretrained(d)
    t.pad_token = t.eos_token
    t.add_eos_token = True
    return t


def test_generator_batches_match_reference_with_llama3_tokenizer(tmp_path):
    """the trainer's generator batches, built with a Llama 3 tokenizer set up as the trainer does it, equal the reference's
    preprocess_dataset output for the same rows, whatever add_eos_token does to this tokenizer's BOS / EOS"""
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference tree not available")
    from transformers import AutoTokenizer

    from dalm_b200 import synthetic
    from dalm_b200.training.utils.rag_e2e_dataloader_utils import preprocess_dataset
    ref = ref_import.load()
    gold = os.path.join(os.path.dirname(__file__), "golden")
    rt = AutoTokenizer.from_pretrained(os.path.join(gold, "tok_bert"))
    d = synthetic.build_llama3_tokenizer(str(tmp_path / "tok_llama3"), 504)
    rows = list(synthetic.synthetic_rows(12, seed=5))
    ex = {k: [r[k] for r in rows] for k in ("Abstract", "Question", "Answer")}
    kw = dict(query_column_name="Question", passage_column_name="Abstract", answer_column_name="Answer", query_max_len=50,
              passage_max_len=128, generator_max_len=256)
    got = preprocess_dataset(ex, retriever_tokenizer=rt, generator_tokenizer=_trainer_tokenizer(d), **kw)
    want = ref.preprocess_e2e(ex, retriever_tokenizer=rt, generator_tokenizer=_trainer_tokenizer(d), **kw)
    assert set(got) == set(want)
    norm = lambda v: [list(x) if isinstance(x, (list, tuple)) else (x.tolist() if hasattr(x, "tolist") else x) for x in v]
    for k in want:
        assert norm(got[k]) == norm(want[k]), k
    assert all(len(x) == 256 for x in got["generator_input_input_ids"])


def test_autoregressive_retriever_batches_match_reference_with_llama3_tokenizer(tmp_path):
    """an autoregressive Llama 3 retriever: the retriever-only trainer's batches equal the reference builder's, and the pooling
    mask is the reference's eos_mask, which selects the last column of every row"""
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference tree not available")
    from dalm_b200 import synthetic
    from dalm_b200.models.rag_e2e_base_model import pooling_mask
    from dalm_b200.training.utils.retriever_only_dataloader_utils import preprocess_dataset
    ref = ref_import.load()
    d = synthetic.build_llama3_tokenizer(str(tmp_path / "tok_llama3"), 504)
    rows = list(synthetic.synthetic_rows(10, seed=8))
    ex = {k: [r[k] for r in rows] for k in ("Abstract", "Question")}
    kw = dict(query_column_name="Question", passage_column_name="Abstract", query_max_len=32, passage_max_len=200)
    got = preprocess_dataset(ex, tokenizer=_trainer_tokenizer(d), **kw)
    want = ref.preprocess_retriever(ex, tokenizer=_trainer_tokenizer(d), **kw)
    assert set(got) == set(want)
    for k in want:
        assert [list(x) for x in got[k]] == [list(x) for x in want[k]], k
    for p in ("query_", "passage_"):
        mask = torch.tensor(got[p + "attention_mask"])
        pm = pooling_mask(mask, True)
        assert torch.equal(pm, ref.eos_mask(mask))
        assert torch.equal(pm.argmax(1), torch.full((mask.shape[0],), mask.shape[1] - 1))
