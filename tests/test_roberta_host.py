"""CPU: XLM-RoBERTa / RoBERTa retrievers — dispatch of both model types and the published shapes, every refusal, the length
check against the position table, the synthetic directories and tokenizers against transformers, and the batches built with
those tokenizers against the reference's builders."""
import os

import pytest
import torch


def _cfg(name="xlmr-tiny", **kw):
    from dalm_b200 import synthetic
    return dict(synthetic.roberta_config(name, vocab_size=300), **kw)


@pytest.mark.parametrize("name,mt", [("xlmr-tiny", "xlm-roberta"), ("xlmr-hd64", "xlm-roberta"), ("roberta-tiny", "roberta"),
                                     ("multilingual-e5-base", "xlm-roberta"), ("xlm-roberta-base", "xlm-roberta"),
                                     ("bge-m3", "xlm-roberta")])
def test_dispatch(name, mt):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    cfg = synthetic.roberta_config(name)
    assert cfg["model_type"] == mt and params.model_kind(cfg) == "roberta"
    assert cfg["pad_token_id"] == 1 and cfg["type_vocab_size"] == 1 and cfg["layer_norm_eps"] == 1e-5
    assert cfg["vocab_size"] == (50265 if mt == "roberta" else 250002)


def test_published_shapes():
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    want = {"multilingual-e5-base": (768, 12, 12, 3072, 514, 512), "xlm-roberta-base": (768, 12, 12, 3072, 514, 512),
            "bge-m3": (1024, 24, 16, 4096, 8194, 8192)}
    for n, w in want.items():
        c = synthetic.roberta_config(n)
        got = (c["hidden_size"], c["num_hidden_layers"], c["num_attention_heads"], c["intermediate_size"],
               c["max_position_embeddings"], params.roberta_max_len(c))
        assert got == w, n
    hd = {n: synthetic.roberta_config(n)["hidden_size"] // synthetic.roberta_config(n)["num_attention_heads"]
          for n in ("xlmr-tiny", "xlmr-hd64")}
    assert hd == {"xlmr-tiny": 32, "xlmr-hd64": 64}


def test_random_state_dict_uses_bert_names():
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    cfg = _cfg()
    r = params.random_state_dict("roberta", cfg, seed=0)
    b = params.random_state_dict("bert", dict(synthetic.bert_config("bge-tiny", 300), type_vocab_size=1,
                                              max_position_embeddings=514), seed=0)
    assert {k: v.shape for k, v in r.items()} == {k: v.shape for k, v in b.items()}
    assert r["embeddings.position_embeddings.weight"].shape == (514, 64)
    assert r["embeddings.token_type_embeddings.weight"].shape == (1, 64)


@pytest.mark.parametrize("setting,value,match", [
    ("position_embedding_type", "relative_key", "position_embedding_type='relative_key'"),
    ("position_embedding_type", "relative_key_query", "position_embedding_type='relative_key_query'"),
    ("hidden_act", "gelu_new", "hidden_act='gelu_new'"),
    ("hidden_act", "relu", "hidden_act='relu'"),
    ("is_decoder", True, "is_decoder"),
    ("add_cross_attention", True, "add_cross_attention"),
])
@pytest.mark.parametrize("name", ["xlmr-tiny", "roberta-tiny"])
def test_refusals(setting, value, match, name):
    from dalm_b200.engine import params
    from dalm_b200.engine.bert import BertEncoder
    cfg = _cfg(name, **{setting: value})
    with pytest.raises(NotImplementedError, match=match):
        params.model_kind(cfg)
    with pytest.raises(NotImplementedError, match=match):
        BertEncoder(cfg, params.random_state_dict("roberta", _cfg(name), seed=0), device="cpu")


def test_decoder_and_autoregressive_paths_refuse_roberta():
    from dalm_b200.engine import params
    from dalm_b200.models.rag_e2e_base_model import build_decoder, build_encoder
    cfg = _cfg()
    sd = params.random_state_dict("roberta", cfg, seed=0)
    with pytest.raises(NotImplementedError, match="generator of kind 'roberta' is not a causal decoder"):
        build_decoder("", False, torch.device("cpu"), state_dict=sd, cfg=cfg)
    with pytest.raises(NotImplementedError, match="autoregressive retrievers are built for Llama, Qwen2 and Qwen3 models only"):
        build_encoder("", False, torch.device("cpu"), state_dict=sd, cfg=cfg, autoregressive=True)


def test_encoder_refusal_names_both_families():
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.models.rag_e2e_base_model import build_encoder
    cfg = synthetic.falcon_config("falcon-tiny", 400)
    with pytest.raises(NotImplementedError, match=r"BERT \(bge-\*\) or \(XLM-\)RoBERTa"):
        build_encoder("", False, torch.device("cpu"), state_dict=params.random_state_dict("falcon", cfg), cfg=cfg)


@pytest.mark.parametrize("name,P,ok", [("xlmr-tiny", 514, 512), ("bge-m3-positions", 8194, 8192)])
def test_too_long_sequences_raise_before_any_launch(name, P, ok):
    """query_max_len / passage_max_len past the usable table: a ValueError naming the length and the limit, raised before any
    kernel launch (this runs on a CPU-built encoder, where a launch would fail differently)"""
    from dalm_b200.engine import params
    from dalm_b200.engine.bert import BertEncoder
    cfg = _cfg(max_position_embeddings=P)
    enc = BertEncoder(cfg, params.random_state_dict("roberta", cfg, seed=0), device="cpu")
    mk = lambda B, L: (torch.full((B, L), 5, dtype=torch.int64), torch.ones(B, L, dtype=torch.int64))
    for segs in ([mk(2, ok + 1)], [mk(4, 50), mk(4, ok + 8)], [mk(4, ok + 1), mk(4, 128)]):
        L = max(ids.shape[1] for ids, _ in segs)
        with pytest.raises(ValueError, match=rf"sequence length {L} exceeds the {ok} positions.*max_position_embeddings {P}"):
            enc.forward_segments(segs, save=False)


def test_nf4_storage_accepts_roberta(monkeypatch):
    from dalm_b200.models import rag_e2e_base_model as m
    monkeypatch.setenv("DALM_B200_NF4_STORAGE", "1")
    assert m._nf4_storage(True, False, "roberta")
    with pytest.raises(NotImplementedError, match="qwen2"):
        m._nf4_storage(True, False, "qwen2")


@pytest.mark.parametrize("name,cls", [("xlmr-tiny", "XLMRobertaModel"), ("xlmr-hd64", "XLMRobertaModel"),
                                      ("roberta-tiny", "RobertaModel")])
def test_synthetic_dirs_load_in_transformers(tmp_path, name, cls):
    import transformers
    from transformers import AutoModel, AutoTokenizer

    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    d = synthetic.write_model_dir(str(tmp_path / name), "roberta", name, vocab_size=1200)
    m = getattr(transformers, cls).from_pretrained(d)
    assert type(AutoModel.from_pretrained(d)).__name__ == cls
    ours, theirs = params.load_state_dict(d), m.state_dict()
    assert set(ours) == set(theirs)
    for k, v in ours.items():
        assert torch.equal(theirs[k], v), k
    assert m.embeddings.padding_idx == 1 and m.embeddings.position_embeddings.padding_idx == 1
    tok = AutoTokenizer.from_pretrained(d)
    assert len(tok) == 1200 and tok.model_max_length == 512


@pytest.mark.parametrize("builder,cls", [("build_xlmr_tokenizer", "XLMRobertaTokenizer"),
                                         ("build_roberta_tokenizer", "RobertaTokenizer")])
def test_tokenizer_layout(tmp_path, builder, cls):
    from transformers import AutoTokenizer

    from dalm_b200 import synthetic
    d = getattr(synthetic, builder)(str(tmp_path / "tok"), 1200)
    tok = AutoTokenizer.from_pretrained(d)
    assert type(tok).__name__ == cls
    assert (tok.bos_token_id, tok.pad_token_id, tok.eos_token_id, tok.unk_token_id, tok.mask_token_id) == (0, 1, 2, 3, 1199)
    enc = tok(["#query# kato mi ren", "#passage# sol"], padding="max_length", max_length=16)
    assert "token_type_ids" not in enc
    for ids, mask in zip(enc["input_ids"], enc["attention_mask"]):
        n = sum(mask)
        assert ids[0] == 0 and ids[n - 1] == 2 and 0 not in ids[1:n] and 2 not in ids[1:n - 1]     # <s> ... </s>
        assert ids[n:] == [1] * (16 - n)                                                              # right-padded with <pad> = 1
    assert tok.decode(enc["input_ids"][0], skip_special_tokens=True).strip() == "#query# kato mi ren"


def _gen_tokenizer():
    from transformers import AutoTokenizer
    t = AutoTokenizer.from_pretrained(os.path.join(os.path.dirname(__file__), "golden", "tok_llama"))
    t.pad_token = t.eos_token
    t.add_eos_token = True
    return t


def test_rag_e2e_batches_match_reference_with_xlmr_tokenizer(tmp_path):
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference tree not available")
    from transformers import AutoTokenizer

    from dalm_b200 import synthetic
    from dalm_b200.training.utils.rag_e2e_dataloader_utils import preprocess_dataset
    ref = ref_import.load()
    rt = AutoTokenizer.from_pretrained(synthetic.build_xlmr_tokenizer(str(tmp_path / "tok_xlmr"), 1200))
    rows = list(synthetic.synthetic_rows(12, seed=5))
    ex = {k: [r[k] for r in rows] for k in ("Abstract", "Question", "Answer")}
    kw = dict(query_column_name="Question", passage_column_name="Abstract", answer_column_name="Answer", query_max_len=50,
              passage_max_len=128, generator_max_len=256)
    got = preprocess_dataset(ex, retriever_tokenizer=rt, generator_tokenizer=_gen_tokenizer(), **kw)
    want = ref.preprocess_e2e(ex, retriever_tokenizer=rt, generator_tokenizer=_gen_tokenizer(), **kw)
    assert set(got) == set(want)
    norm = lambda v: [list(x) if isinstance(x, (list, tuple)) else (x.tolist() if hasattr(x, "tolist") else x) for x in v]
    for k in want:
        assert norm(got[k]) == norm(want[k]), k
    assert not any(k.endswith("token_type_ids") for k in got)
    assert all(x[0] == 0 for x in got["retriever_query_input_ids"])
    assert any(1 in x for x in got["retriever_query_input_ids"])                                 # padded with <pad> = 1


@pytest.mark.parametrize("builder", ["build_xlmr_tokenizer", "build_roberta_tokenizer"])
def test_retriever_only_batches_match_reference(tmp_path, builder):
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference tree not available")
    from transformers import AutoTokenizer

    from dalm_b200 import synthetic
    from dalm_b200.training.utils.retriever_only_dataloader_utils import preprocess_dataset
    ref = ref_import.load()
    tok = AutoTokenizer.from_pretrained(getattr(synthetic, builder)(str(tmp_path / "tok"), 1200))
    rows = list(synthetic.synthetic_rows(10, seed=8))
    ex = {k: [r[k] for r in rows] for k in ("Abstract", "Question")}
    kw = dict(query_column_name="Question", passage_column_name="Abstract", query_max_len=32, passage_max_len=200)
    got = preprocess_dataset(ex, tokenizer=tok, **kw)
    want = ref.preprocess_retriever(ex, tokenizer=tok, **kw)
    assert set(got) == set(want)
    for k in want:
        assert [list(x) for x in got[k]] == [list(x) for x in want[k]], k
