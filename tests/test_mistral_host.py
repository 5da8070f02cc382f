"""CPU: Mistral generators / autoregressive retrievers and sliding-window attention — model_type dispatch and the settings that
are refused, the per-layer windows against transformers' config classes, the synthetic Mistral directories (with and without
an lm_head) in transformers, the headless key mapping, and the batches built with the Mistral (Llama SentencePiece) tokenizer
against the reference's builders."""
import os

import pytest
import torch


def _mistral(name="mistral-tiny", **kw):
    from dalm_b200 import synthetic
    return dict(synthetic.mistral_config(name, vocab_size=400), **kw)


def _qwen(mt, n, **kw):
    from dalm_b200 import synthetic
    cfg = synthetic.qwen2_config("qwen2-tiny", 400) if mt == "qwen2" else synthetic.qwen3_config("qwen3-tiny", 400)
    cfg = {k: v for k, v in cfg.items() if k not in ("use_sliding_window", "sliding_window", "max_window_layers")}
    return dict(cfg, num_hidden_layers=n, **kw)


def _hf_windows(cfg):
    """the window of every layer as transformers' config class resolves it (None = full attention)"""
    from transformers import AutoConfig
    c = AutoConfig.for_model(cfg["model_type"], **{k: v for k, v in cfg.items() if k not in ("architectures", "model_type")})
    n = c.num_hidden_layers
    types = getattr(c, "layer_types", None) if cfg["model_type"] != "mistral" else None
    if types is None:
        types = ["sliding_attention"] * n
    return [c.sliding_window if (t == "sliding_attention" and c.sliding_window is not None) else 0 for t in types]


# ----------------------------------------------------------------------------------------------------------------
# dispatch and refusals
# ----------------------------------------------------------------------------------------------------------------
def test_model_kind_mistral():
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    for name in synthetic.MISTRAL_SHAPES:
        assert params.model_kind(synthetic.mistral_config(name)) == "mistral"
    assert params.attention_biases("mistral", _mistral(attention_bias=True)) == (False, False)
    params.check_llama_family(_mistral(mlp_bias=True))           # MistralMLP has no bias whatever the key says


def test_mistral_config_must_carry_its_shape():
    """a config that leaves the shape to MistralConfig's defaults is refused, naming the missing keys"""
    from dalm_b200.engine import params
    with pytest.raises(NotImplementedError, match="mistral: a config without hidden_size, intermediate_size"):
        params.model_kind({"model_type": "mistral"})
    cfg = _mistral()
    with pytest.raises(NotImplementedError, match="without vocab_size"):
        params.model_kind({k: v for k, v in cfg.items() if k != "vocab_size"})
    assert params.model_kind({k: v for k, v in cfg.items() if k != "sliding_window"}) == "mistral"   # window: 4096


@pytest.mark.parametrize("mt", ["qwen2", "qwen3"])
@pytest.mark.parametrize("kw", [dict(max_window_layers=4), dict(max_window_layers=6), dict(sliding_window=None),
                                dict(layer_types=["full_attention"] * 4)])
def test_qwen_sliding_window_without_sliding_layers_refused(mt, kw):
    """use_sliding_window=true that selects no windowed layer: transformers runs full attention, the Qwen documentation of
    max_window_layers reads the other way round; refused, naming the setting"""
    from dalm_b200.engine import params
    cfg = _qwen(mt, 4, use_sliding_window=True, **dict(dict(sliding_window=64), **kw))
    assert not any(params.sliding_windows(cfg))
    with pytest.raises(NotImplementedError, match="use_sliding_window=true selects no sliding-window layer"):
        params.model_kind(cfg)


@pytest.mark.parametrize("rope", [{"rope_type": "linear", "factor": 2.0}, {"rope_type": "llama3", "factor": 8.0},
                                  {"type": "dynamic", "factor": 2.0}, {"rope_type": "yarn", "factor": 4.0}])
def test_mistral_refuses_scaled_rope(rope):
    from dalm_b200.engine import params
    t = rope.get("rope_type", rope.get("type"))
    with pytest.raises(NotImplementedError, match=f"mistral: RoPE type '{t}'"):
        params.model_kind(_mistral(rope_scaling=rope))


def test_mistral_refusals_name_their_setting(monkeypatch):
    from dalm_b200.engine import params
    from dalm_b200.engine.llama import LlamaDecoder
    from dalm_b200.models import rag_e2e_base_model as rm
    with pytest.raises(NotImplementedError, match="head_dim 96"):
        LlamaDecoder(_mistral(head_dim=96), {}, device="cpu")
    monkeypatch.setenv("DALM_B200_NF4_STORAGE", "1")
    with pytest.raises(NotImplementedError, match="DALM_B200_NF4_STORAGE=1.*'mistral'"):
        rm._nf4_storage(True, False, "mistral")
    with pytest.raises(NotImplementedError, match="model_type 'mixtral'"):
        params.model_kind(dict(_mistral(), model_type="mixtral"))


def test_qwen_sliding_window_no_longer_refused():
    from dalm_b200.engine import params
    for mt in ("qwen2", "qwen3"):
        assert params.model_kind(_qwen(mt, 4, use_sliding_window=True, sliding_window=64, max_window_layers=2)) == mt


# ----------------------------------------------------------------------------------------------------------------
# per-layer windows against transformers
# ----------------------------------------------------------------------------------------------------------------
WINDOW_CASES = [
    ("mistral", dict()),                                          # key absent: MistralConfig's 4096
    ("mistral", dict(sliding_window=None)),
    ("mistral", dict(sliding_window=4096)),
    ("mistral", dict(sliding_window=48, layer_types=["full_attention", "sliding_attention"])),   # ignored by MistralConfig
    ("qwen2", dict()),
    ("qwen2", dict(use_sliding_window=False, sliding_window=64)),
    ("qwen2", dict(use_sliding_window=True, sliding_window=64, max_window_layers=0)),
    ("qwen2", dict(use_sliding_window=True, sliding_window=64, max_window_layers=1)),
    ("qwen2", dict(use_sliding_window=True, sliding_window=64, max_window_layers=4)),
    ("qwen2", dict(use_sliding_window=True, sliding_window=64)),  # max_window_layers absent: 28
    ("qwen2", dict(use_sliding_window=True, sliding_window=32, max_window_layers=3,
                   layer_types=["sliding_attention", "full_attention", "sliding_attention", "full_attention"])),
    ("qwen3", dict(use_sliding_window=True, sliding_window=64, max_window_layers=1)),
    ("qwen3", dict(use_sliding_window=False, sliding_window=64, max_window_layers=1)),
    ("qwen3", dict(use_sliding_window=True, sliding_window=16, max_window_layers=2,
                   layer_types=["full_attention", "sliding_attention", "sliding_attention", "sliding_attention"])),
]


@pytest.mark.parametrize("mt,kw", WINDOW_CASES)
def test_sliding_windows_match_transformers(mt, kw):
    from dalm_b200.engine import params
    if mt == "mistral":
        cfg = {k: v for k, v in _mistral().items() if k != "sliding_window"}
        cfg = dict(cfg, num_hidden_layers=2, **kw)
    else:
        cfg = _qwen(mt, 4, **kw)
    assert params.sliding_windows(cfg) == _hf_windows(cfg)


def test_llama_has_no_window():
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    assert params.sliding_windows(synthetic.llama_config("llama-tiny")) == [0, 0]


def test_published_shapes():
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    v01 = synthetic.mistral_config("Mistral-7B-v0.1")
    assert (v01["sliding_window"], v01["rope_theta"], v01["vocab_size"], v01["intermediate_size"]) == (4096, 1e4, 32000, 14336)
    v03 = synthetic.mistral_config("Mistral-7B-v0.3")
    assert (v03["sliding_window"], v03["rope_theta"], v03["vocab_size"]) == (None, 1e6, 32768)
    assert params.sliding_windows(v03) == [0] * 32
    e5 = synthetic.mistral_config("e5-mistral-7b-instruct")
    assert e5["architectures"] == ["MistralModel"] and params.sliding_windows(e5) == [4096] * 32
    nemo = synthetic.mistral_config("Mistral-Nemo-Base-2407")
    assert (nemo["hidden_size"], nemo["head_dim"], nemo["vocab_size"]) == (5120, 128, 131072)
    assert nemo["hidden_size"] // nemo["num_attention_heads"] != nemo["head_dim"]
    tiny = [synthetic.mistral_config(n) for n in ("mistral-tiny", "mistral-hd64", "mistral-nowin")]
    assert [c["head_dim"] for c in tiny] == [128, 64, 64]
    assert [c["sliding_window"] for c in tiny] == [48, 37, None]


# ----------------------------------------------------------------------------------------------------------------
# synthetic directories and the headless layout
# ----------------------------------------------------------------------------------------------------------------
def test_synthetic_mistral_dirs_load_in_transformers(tmp_path):
    from transformers import AutoConfig, AutoTokenizer, MistralForCausalLM, MistralModel

    from dalm_b200.engine import params
    for name, headless, cls in (("mistral-tiny", False, MistralForCausalLM), ("mistral-hd64", True, MistralModel),
                                ("mistral-nowin", False, MistralForCausalLM)):
        from dalm_b200 import synthetic
        d = synthetic.write_model_dir(str(tmp_path / name), "mistral", name, vocab_size=400, headless=headless)
        cfg = params.load_config(d)
        assert cfg["architectures"] == [cls.__name__]
        hc = AutoConfig.from_pretrained(d)
        assert hc.model_type == "mistral" and hc.sliding_window == cfg["sliding_window"]
        m, info = cls.from_pretrained(d, output_loading_info=True)
        assert not info["missing_keys"] and not info["unexpected_keys"], info
        sd = params.load_state_dict(d)
        assert any(k.startswith("model.") for k in sd) != headless and ("lm_head.weight" in sd) != headless
        hf = m.state_dict()
        for k, v in sd.items():
            assert torch.equal(hf[k], v), k
        tok = AutoTokenizer.from_pretrained(d)
        assert tok.convert_tokens_to_ids(["<unk>", "<s>", "</s>"]) == [0, 1, 2]


def test_headless_key_mapping_round_trips():
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.llama import _with_prefix
    cfg = _mistral("mistral-hd64")
    sd = params.random_state_dict("mistral", cfg, seed=1)
    hl = synthetic.headless_state_dict(sd)
    assert set(hl) == {k[len("model."):] for k in sd if k != "lm_head.weight"}
    assert all(not k.startswith(("model.", "lm_head")) for k in hl)
    back = _with_prefix(hl)
    assert set(back) == set(sd) - {"lm_head.weight"} and all(back[k] is hl[k[len("model."):]] for k in back)


# ----------------------------------------------------------------------------------------------------------------
# batches against the reference's builders
# ----------------------------------------------------------------------------------------------------------------
def _trainer_tokenizer(d):
    """a generator tokenizer set up as the trainer does it (reference train_rage2e.py:301-304), which is also how an
    autoregressive retriever's tokenizer is set up"""
    from transformers import AutoTokenizer
    t = AutoTokenizer.from_pretrained(d)
    t.pad_token = t.eos_token
    t.add_eos_token = True
    return t


def test_generator_batches_match_reference_with_mistral_tokenizer(tmp_path):
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference tree not available")
    from transformers import AutoTokenizer

    from dalm_b200 import synthetic
    from dalm_b200.training.utils.rag_e2e_dataloader_utils import preprocess_dataset
    ref = ref_import.load()
    gold = os.path.join(os.path.dirname(__file__), "golden")
    rt = AutoTokenizer.from_pretrained(os.path.join(gold, "tok_bert"))
    d = synthetic.write_model_dir(str(tmp_path / "mistral"), "mistral", "mistral-hd64", vocab_size=800, with_weights=False)
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


def test_autoregressive_retriever_batches_match_reference_with_mistral_tokenizer(tmp_path):
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference tree not available")
    from dalm_b200 import synthetic
    from dalm_b200.models.rag_e2e_base_model import pooling_mask
    from dalm_b200.training.utils.retriever_only_dataloader_utils import preprocess_dataset
    ref = ref_import.load()
    d = synthetic.write_model_dir(str(tmp_path / "e5"), "mistral", "mistral-tiny", vocab_size=800, with_weights=False,
                                  headless=True)
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
