"""CPU: Qwen2 generators / autoregressive retrievers — config dispatch and the settings that are refused, the synthetic Qwen2
directory against transformers' Qwen2ForCausalLM, random attention biases, the use_bnb treatment of biases, and the
generator batches built with a Qwen2 tokenizer against the reference's builder."""
import os

import pytest
import torch


def _qcfg(**kw):
    from dalm_b200 import synthetic
    return dict(synthetic.qwen2_config("qwen2-tiny", vocab_size=504), **kw)


def test_model_kind_maps_qwen2():
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    assert params.model_kind(_qcfg()) == "qwen2"
    assert params.model_kind(synthetic.qwen2_config("qwen2.5-7b")) == "qwen2"
    assert params.model_kind(synthetic.llama_config("llama-tiny")) == "llama"
    # transformers 5 writes its default RoPE parameters into every config it saves: not a refusal
    assert params.model_kind(_qcfg(rope_parameters={"rope_theta": 1e6, "rope_type": "default"})) == "qwen2"
    assert params.model_kind(_qcfg(rope_scaling=None)) == "qwen2"
    with pytest.raises(NotImplementedError, match="mistral"):
        params.model_kind({"model_type": "mistral"})


@pytest.mark.parametrize("extra,match", [
    (dict(use_sliding_window=True, sliding_window=4096), "sliding"),
    (dict(layer_types=["full_attention", "sliding_attention"]), "sliding"),
    (dict(rope_scaling={"type": "yarn", "factor": 4.0, "original_max_position_embeddings": 32768}), "yarn"),
    (dict(rope_scaling={"rope_type": "dynamic", "factor": 2.0}), "dynamic"),
    (dict(rope_parameters={"rope_theta": 1e6, "rope_type": "yarn", "factor": 4.0}), "yarn"),
    (dict(mlp_bias=True), "mlp_bias"),
])
def test_qwen2_refusals(extra, match):
    from dalm_b200.engine import params
    with pytest.raises(NotImplementedError, match=match):
        params.model_kind(_qcfg(**extra))


def test_llama_mlp_bias_refused():
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    with pytest.raises(NotImplementedError, match="mlp_bias"):
        params.model_kind(dict(synthetic.llama_config("llama-tiny"), mlp_bias=True))
    assert params.attention_biases("llama", dict(synthetic.llama_config("llama-tiny"), attention_bias=True)) == (True, True)
    assert params.attention_biases("llama", synthetic.llama_config("llama-tiny")) == (False, False)
    assert params.attention_biases("qwen2", _qcfg()) == (True, False)


def test_nf4_storage_refuses_qwen2(monkeypatch):
    from dalm_b200.models.rag_e2e_base_model import _nf4_storage
    monkeypatch.setenv("DALM_B200_NF4_STORAGE", "1")
    with pytest.raises(NotImplementedError, match="qwen2"):
        _nf4_storage(True, False, "qwen2")
    assert _nf4_storage(True, False, "llama") is True


def test_random_state_dict_biases():
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    cfg = synthetic.qwen2_config("qwen2-tiny", vocab_size=504)
    sd = params.random_state_dict("qwen2", cfg, seed=3, bias_std=0.5)
    nq, nkv = 14 * 64, 2 * 64
    for l in range(cfg["num_hidden_layers"]):
        p = f"model.layers.{l}.self_attn."
        assert sd[p + "q_proj.bias"].shape == (nq,) and sd[p + "k_proj.bias"].shape == (nkv,) and sd[p + "v_proj.bias"].shape == (nkv,)
        for n in "qkv":
            assert 0.4 < sd[p + f"{n}_proj.bias"].std().item() < 0.6
        assert p + "o_proj.bias" not in sd
    assert "lm_head.weight" not in sd                                     # tied
    assert "lm_head.weight" in params.random_state_dict("qwen2", synthetic.qwen2_config("qwen2-hd128", 504), seed=3)
    # a Llama config with attention_bias gets all four biases; a plain one none, and its draws are unchanged
    lcfg = synthetic.llama_config("llama-tiny", 400)
    plain = params.random_state_dict("llama", lcfg, seed=2)
    assert not [k for k in plain if k.endswith(".bias")]
    ab = params.random_state_dict("llama", dict(lcfg, attention_bias=True), seed=2)
    assert sorted(k.split(".")[-2] for k in ab if k.endswith(".bias") and ".0." in k) == ["k_proj", "o_proj", "q_proj", "v_proj"]
    assert all(ab[k].abs().sum() > 0 for k in ab if k.endswith(".bias"))


def test_synthetic_qwen2_dir_loads_in_transformers(tmp_path):
    from transformers import AutoTokenizer, Qwen2ForCausalLM

    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    for name, tied in (("qwen2-tiny", True), ("qwen2-hd128", False)):
        d = synthetic.write_model_dir(str(tmp_path / name), "qwen2", name, vocab_size=504, bias_std=0.5,
                                      generation_config=synthetic.QWEN2_GENERATION["base"])
        m = Qwen2ForCausalLM.from_pretrained(d)
        ours = params.load_state_dict(d)
        theirs = m.state_dict()
        want = set(theirs) - ({"lm_head.weight"} if tied else set())
        assert set(ours) == want
        for k, v in ours.items():
            assert torch.equal(theirs[k], v), k
        assert (m.lm_head.weight.data_ptr() == m.model.embed_tokens.weight.data_ptr()) == tied
        assert os.path.isfile(os.path.join(d, "generation_config.json"))
    tok = AutoTokenizer.from_pretrained(d)
    assert type(tok).__name__ == "Qwen2Tokenizer"
    assert tok.pad_token == tok.eos_token == "<|endoftext|>" and tok.bos_token is None
    assert tok.convert_tokens_to_ids(["<|im_start|>", "<|im_end|>"]) == [1, 2]
    text = "#query# kato mi ren"
    assert tok.decode(tok(text)["input_ids"]) == text


def test_bnb_biases_take_the_fp16_cast():
    """use_bnb: only nn.Linear weights go through the NF4 round trip; attention biases take the fp16 cast"""
    from dalm_b200.engine import params
    names = ["model.layers.0.self_attn.q_proj.bias", "model.layers.0.self_attn.k_proj.bias",
             "model.layers.0.self_attn.v_proj.bias", "model.layers.0.self_attn.o_proj.bias"]
    assert not any(params.is_bnb_linear_weight(n) for n in names)
    assert params.is_bnb_linear_weight("model.layers.0.self_attn.q_proj.weight")
    g = torch.Generator().manual_seed(0)
    sd = {n: torch.randn(96, generator=g) * 0.5 + 1e-4 for n in names}
    out = params.bnb_nf4_state_dict(sd, "cpu")
    for n in names:
        want = sd[n].to(torch.float16).to(torch.float32)
        assert torch.equal(out[n], want) and not torch.equal(out[n], sd[n])


def test_generator_batches_match_reference_with_qwen2_tokenizer(tmp_path):
    """the trainer's generator batches, built with a Qwen2 tokenizer set up as the trainer does it, equal the reference's
    preprocess_dataset output for the same rows (whatever add_eos_token does on this tokenizer)"""
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference tree not available")
    from transformers import AutoTokenizer

    from dalm_b200 import synthetic
    from dalm_b200.training.utils.rag_e2e_dataloader_utils import preprocess_dataset
    ref = ref_import.load()
    gold = os.path.join(os.path.dirname(__file__), "golden")
    rt = AutoTokenizer.from_pretrained(os.path.join(gold, "tok_bert"))
    d = synthetic.build_qwen2_tokenizer(str(tmp_path / "tok_qwen2"), 504)
    toks = []
    for _ in range(2):
        gt = AutoTokenizer.from_pretrained(d)
        gt.pad_token = gt.eos_token
        gt.add_eos_token = True
        toks.append(gt)
    rows = list(synthetic.synthetic_rows(12, seed=5))
    ex = {k: [r[k] for r in rows] for k in ("Abstract", "Question", "Answer")}
    kw = dict(query_column_name="Question", passage_column_name="Abstract", answer_column_name="Answer", query_max_len=50,
              passage_max_len=128, generator_max_len=256)
    got = preprocess_dataset(ex, retriever_tokenizer=rt, generator_tokenizer=toks[0], **kw)
    want = ref.preprocess_e2e(ex, retriever_tokenizer=rt, generator_tokenizer=toks[1], **kw)
    assert set(got) == set(want)
    norm = lambda v: [list(x) if isinstance(x, (list, tuple)) else (x.tolist() if hasattr(x, "tolist") else x) for x in v]
    for k in want:
        assert norm(got[k]) == norm(want[k]), k
    assert all(len(x) == 256 for x in got["generator_input_input_ids"])
