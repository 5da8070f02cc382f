"""CPU: Qwen3 generators / autoregressive retrievers — config dispatch and the settings that are refused, the synthetic Qwen3
directory against transformers' Qwen3ForCausalLM (tied and untied), random q / k norm weights, and the use_bnb treatment of
the q / k norm weights."""
import pytest
import torch


def _qcfg(name="qwen3-tiny", **kw):
    from dalm_b200 import synthetic
    return dict(synthetic.qwen3_config(name, vocab_size=504), **kw)


def test_model_kind_maps_qwen3():
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    for name in ("qwen3-tiny", "qwen3-hd128", "qwen3-0.6b", "qwen3-8b"):
        assert params.model_kind(synthetic.qwen3_config(name)) == "qwen3"
    assert params.model_kind(_qcfg(rope_parameters={"rope_theta": 1e6, "rope_type": "default"})) == "qwen3"
    assert params.model_kind(_qcfg(layer_types=["full_attention", "full_attention"])) == "qwen3"
    with pytest.raises(NotImplementedError, match="qwen3_moe"):
        params.model_kind(dict(_qcfg(), model_type="qwen3_moe"))


@pytest.mark.parametrize("extra,match", [
    (dict(use_sliding_window=True, sliding_window=4096), "sliding"),
    (dict(layer_types=["full_attention", "sliding_attention"]), "sliding"),
    (dict(rope_scaling={"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 32768}), "yarn"),
    (dict(rope_parameters={"rope_theta": 1e6, "rope_type": "linear", "factor": 2.0}), "linear"),
    (dict(mlp_bias=True), "mlp_bias"),
    (dict(head_dim=64), "head_dim"),
])
def test_qwen3_refusals(extra, match):
    from dalm_b200.engine import params
    with pytest.raises(NotImplementedError, match=match):
        params.model_kind(_qcfg(**extra))


def test_qwen3_attention_bias_and_nf4_storage(monkeypatch):
    from dalm_b200.engine import params
    from dalm_b200.models.rag_e2e_base_model import _nf4_storage
    assert params.attention_biases("qwen3", _qcfg()) == (False, False)
    assert params.attention_biases("qwen3", _qcfg(attention_bias=True)) == (True, True)
    sd = params.random_state_dict("qwen3", _qcfg(attention_bias=True), seed=1)
    assert sorted(k.split(".")[-2] for k in sd if k.endswith(".bias") and ".0." in k) == ["k_proj", "o_proj", "q_proj", "v_proj"]
    monkeypatch.setenv("DALM_B200_NF4_STORAGE", "1")
    with pytest.raises(NotImplementedError, match="qwen3"):
        _nf4_storage(True, False, "qwen3")


def test_random_state_dict_qk_norms():
    from dalm_b200.engine import params
    cfg = _qcfg()
    sd = params.random_state_dict("qwen3", cfg, seed=3, qk_norm_std=0.5)
    for l in range(cfg["num_hidden_layers"]):
        p = f"model.layers.{l}.self_attn."
        assert sd[p + "q_proj.weight"].shape == (4 * 128, 384) and sd[p + "o_proj.weight"].shape == (384, 4 * 128)
        assert sd[p + "k_proj.weight"].shape == (128, 384)
        for n in ("q_norm", "k_norm"):
            w = sd[p + f"{n}.weight"]
            assert w.shape == (128,) and 0.85 < w.mean().item() < 1.15 and 0.4 < w.std().item() < 0.6
        assert not torch.equal(sd[p + "q_norm.weight"], sd[p + "k_norm.weight"])
        assert not [k for k in sd if k.startswith(p) and k.endswith(".bias")]
    assert "lm_head.weight" not in sd                                    # qwen3-tiny is tied
    d = params.random_state_dict("qwen3", cfg, seed=3)                   # default spread: initializer_range
    assert 0.01 < d["model.layers.0.self_attn.q_norm.weight"].std().item() < 0.03
    # the Qwen2 / Llama draws are untouched by the new branch
    from dalm_b200 import synthetic
    a = params.random_state_dict("qwen2", synthetic.qwen2_config("qwen2-tiny", 504), seed=3, qk_norm_std=0.5)
    b = params.random_state_dict("qwen2", synthetic.qwen2_config("qwen2-tiny", 504), seed=3)
    assert set(a) == set(b) and all(torch.equal(a[k], b[k]) for k in a)


def test_synthetic_qwen3_dir_loads_in_transformers(tmp_path):
    from transformers import AutoTokenizer, Qwen3ForCausalLM

    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    for name, tied in (("qwen3-tiny", True), ("qwen3-hd128", False)):
        d = synthetic.write_model_dir(str(tmp_path / name), "qwen3", name, vocab_size=504, qk_norm_std=0.5,
                                      generation_config=synthetic.QWEN3_GENERATION["base"])
        m = Qwen3ForCausalLM.from_pretrained(d)
        ours = params.load_state_dict(d)
        theirs = m.state_dict()
        want = set(theirs) - ({"lm_head.weight"} if tied else set())
        assert set(ours) == want
        for k, v in ours.items():
            assert torch.equal(theirs[k], v), k
        assert (m.lm_head.weight.data_ptr() == m.model.embed_tokens.weight.data_ptr()) == tied
        assert m.config.head_dim == 128 and m.model.layers[0].self_attn.q_norm.weight.std() > 0.3
    tok = AutoTokenizer.from_pretrained(d)
    assert type(tok).__name__ == "Qwen2Tokenizer" and tok.pad_token == tok.eos_token == "<|endoftext|>"


def test_published_shapes():
    from dalm_b200 import synthetic
    c = synthetic.qwen3_config("qwen3-0.6b")
    assert (c["hidden_size"], c["num_attention_heads"] * c["head_dim"], c["tie_word_embeddings"]) == (1024, 2048, True)
    c = synthetic.qwen3_config("qwen3-8b")
    qkv = (c["num_attention_heads"] + 2 * c["num_key_value_heads"]) * 128
    assert (qkv, c["hidden_size"], c["tie_word_embeddings"]) == (6144, 4096, False)
    # qwen3-tiny takes the row-kernel path (q|k width not a multiple of 256), qwen3-hd128 the fused epilogue
    for name, fused in (("qwen3-tiny", False), ("qwen3-hd128", True)):
        c = synthetic.qwen3_config(name)
        assert (((c["num_attention_heads"] + c["num_key_value_heads"]) * 128) % 256 == 0) == fused
        assert c["num_attention_heads"] * 128 != c["hidden_size"]


def test_bnb_qk_norms_take_the_fp16_cast():
    """use_bnb: q_norm / k_norm weights are norms, not nn.Linear weights: the fp16 cast, never the NF4 round trip"""
    from dalm_b200.engine import params
    names = ["model.layers.0.self_attn.q_norm.weight", "model.layers.3.self_attn.k_norm.weight"]
    assert not any(params.is_bnb_linear_weight(n) for n in names)
    g = torch.Generator().manual_seed(0)
    sd = {n: 1 + torch.randn(128, generator=g) * 0.5 + 1e-4 for n in names}
    out = params.bnb_nf4_state_dict(sd, "cpu")
    for n in names:
        want = sd[n].to(torch.float16).to(torch.float32)
        assert torch.equal(out[n], want) and not torch.equal(out[n], sd[n])
