"""CPU: Qwen3-MoE configs (model kind, refusals with their reasons, which layers are sparse), the random-init hub layout, and
the synthetic directory as transformers' Qwen3MoeForCausalLM loads it."""
import os

import pytest
import torch

from dalm_b200 import synthetic
from dalm_b200.engine import params


def _mcfg(name="qwen3-moe-tiny", **kw):
    return dict(synthetic.qwen3_moe_config(name, vocab_size=400), **kw)


def test_model_kind_maps_qwen3_moe():
    for name in synthetic.QWEN3_MOE_SHAPES:
        assert params.model_kind(synthetic.qwen3_moe_config(name)) == "qwen3_moe"
    assert params.model_kind(_mcfg(rope_parameters={"rope_theta": 1e6, "rope_type": "default"})) == "qwen3_moe"
    assert params.model_kind(_mcfg(num_experts=0)) == "qwen3_moe"                  # no sparse layer: a dense Qwen3


@pytest.mark.parametrize("extra,match", [
    (dict(head_dim=64), "qwen3_moe: head_dim=64"),
    (dict(rope_scaling={"rope_type": "yarn", "factor": 4.0}), "qwen3_moe: RoPE type 'yarn'"),
    (dict(moe_intermediate_size=192), "moe_intermediate_size=192 .*multiple of 128"),
    (dict(num_experts=260), "num_experts=260 .*multiple of 8 up to 256"),
    (dict(num_experts=12), "num_experts=12 .*multiple of 8"),
    (dict(num_experts_per_tok=17, num_experts=64), "num_experts_per_tok=17 .*min\\(num_experts, 16\\)"),
    (dict(num_experts_per_tok=0), "num_experts_per_tok=0"),
    (dict(mlp_bias=True), "mlp_bias=true"),
])
def test_qwen3_moe_refusals(extra, match):
    with pytest.raises(NotImplementedError, match=match):
        params.model_kind(_mcfg(**extra))


@pytest.mark.parametrize("key", params.QWEN3_MOE_KEYS)
def test_qwen3_moe_needs_its_shape_keys(key):
    cfg = _mcfg()
    del cfg[key]
    with pytest.raises(NotImplementedError, match=f"qwen3_moe: a config without {key}"):
        params.model_kind(cfg)


def test_dense_layers_need_intermediate_size():
    cfg = _mcfg()
    del cfg["intermediate_size"]
    with pytest.raises(NotImplementedError, match="qwen3_moe: dense MLP layers .* need intermediate_size"):
        params.model_kind(cfg)
    assert params.model_kind(dict(cfg, mlp_only_layers=[])) == "qwen3_moe"           # every layer sparse: not needed


@pytest.mark.parametrize("step,only,n", [(1, [], 4), (2, [], 4), (3, [], 7), (1, [0, 3], 5), (2, [1], 6), (4, [3], 4)])
def test_moe_layers_match_transformers(step, only, n):
    """the sparse layers are the ones Qwen3MoeDecoderLayer gives a Qwen3MoeSparseMoeBlock"""
    from transformers import Qwen3MoeConfig
    from transformers.models.qwen3_moe.modeling_qwen3_moe import Qwen3MoeDecoderLayer, Qwen3MoeSparseMoeBlock
    cfg = _mcfg(num_hidden_layers=n, decoder_sparse_step=step, mlp_only_layers=only)
    hf = Qwen3MoeConfig(**{k: v for k, v in cfg.items() if k not in ("architectures", "model_type")})
    want = [isinstance(Qwen3MoeDecoderLayer(hf, i).mlp, Qwen3MoeSparseMoeBlock) for i in range(n)]
    assert params.moe_layers(cfg) == want


def test_sliding_windows_qwen3_moe():
    """Qwen3MoeConfig: sliding_window on every layer with use_sliding_window (default 4096), none without"""
    assert params.sliding_windows(_mcfg()) == [0, 0, 0]
    assert params.sliding_windows(_mcfg(use_sliding_window=True, sliding_window=64)) == [64, 64, 64]
    cfg = _mcfg(use_sliding_window=True)
    del cfg["sliding_window"]
    assert params.sliding_windows(cfg) == [4096] * 3


def test_random_state_dict_hub_layout():
    cfg = _mcfg()
    sd = params.random_state_dict("qwen3_moe", cfg, seed=3, router_std=0.7)
    H, E, I = cfg["hidden_size"], cfg["num_experts"], cfg["moe_intermediate_size"]
    assert sd["model.layers.0.mlp.gate.weight"].shape == (E, H)
    assert sd["model.layers.0.mlp.experts.7.gate_proj.weight"].shape == (I, H)
    assert sd["model.layers.2.mlp.experts.0.down_proj.weight"].shape == (H, I)
    assert "model.layers.1.mlp.gate_proj.weight" in sd and "model.layers.1.mlp.gate.weight" not in sd   # the dense layer
    assert 0.6 < sd["model.layers.0.mlp.gate.weight"].std().item() < 0.8
    assert "model.layers.0.self_attn.q_norm.weight" in sd


def _fused(sd, cfg):
    """transformers 5's layout of the experts: gate_up_proj [E, 2I, H] (gate rows, then up rows), down_proj [E, H, I]"""
    out = {k: v for k, v in sd.items() if ".mlp.experts." not in k}
    for l, sparse in enumerate(params.moe_layers(cfg)):
        if sparse:
            p = f"model.layers.{l}.mlp.experts."
            E = cfg["num_experts"]
            out[p + "gate_up_proj"] = torch.stack([torch.cat([sd[p + f"{e}.gate_proj.weight"], sd[p + f"{e}.up_proj.weight"]])
                                                   for e in range(E)])
            out[p + "down_proj"] = torch.stack([sd[p + f"{e}.down_proj.weight"] for e in range(E)])
    return out


@pytest.mark.parametrize("name", ["qwen3-moe-tiny", "qwen3-moe-hd128"])
def test_synthetic_directory_loads_in_transformers(tmp_path, name):
    """write_model_dir(kind="qwen3_moe"): transformers' Qwen3MoeForCausalLM loads the hub layout, and its parameters are
    exactly the fused layout (gate_up_proj / down_proj) made from it, which the engine also loads; the Qwen2 tokenizer
    round-trips"""
    from safetensors.torch import load_file
    from transformers import AutoTokenizer, Qwen3MoeForCausalLM
    d = synthetic.write_model_dir(str(tmp_path / "m"), "qwen3_moe", name, vocab_size=400, router_std=0.5)
    cfg = params.load_config(d)
    sd = load_file(os.path.join(d, "model.safetensors"))
    m = Qwen3MoeForCausalLM.from_pretrained(d, dtype=torch.float32)
    got = m.state_dict()
    want = _fused(sd, cfg)
    assert set(got) == set(want) | ({"lm_head.weight"} if cfg["tie_word_embeddings"] else set())
    for k, v in want.items():
        assert torch.equal(got[k], v), k
    tok = AutoTokenizer.from_pretrained(d)
    assert tok.decode(tok("ka to mi")["input_ids"]) == "ka to mi"


@pytest.fixture(scope="module")
def moe_dir(tmp_path_factory):
    return synthetic.write_model_dir(str(tmp_path_factory.mktemp("moe") / "m"), "qwen3_moe", "qwen3-moe-tiny", vocab_size=400,
                                     with_weights=False)


@pytest.mark.parametrize("kw,match", [
    (dict(full=True), "full fine-tuning of a qwen3_moe generator is not built: grouped expert weight gradients .*550 GB"),
    (dict(bnb=True), "use_bnb on a qwen3_moe generator is not built: the 4-bit treatment of the fused 3-D expert weights"),
])
def test_build_decoder_refusals(moe_dir, kw, match):
    from dalm_b200.models.rag_e2e_base_model import build_decoder
    with pytest.raises(NotImplementedError, match=match):
        build_decoder(moe_dir, lora=False, device=torch.device("cpu"), **kw)


def test_nf4_storage_refused(moe_dir, monkeypatch):
    from dalm_b200.models.rag_e2e_base_model import build_decoder
    monkeypatch.setenv("DALM_B200_NF4_STORAGE", "1")
    with pytest.raises(NotImplementedError, match="qwen3_moe"):
        build_decoder(moe_dir, lora=True, device=torch.device("cpu"), bnb=True)


def test_autoregressive_retriever_refused(moe_dir):
    from dalm_b200.models.rag_e2e_base_model import build_encoder
    with pytest.raises(NotImplementedError, match="autoregressive retrievers are built for Llama, Qwen2 and Qwen3 models only"):
        build_encoder(moe_dir, lora=True, device=torch.device("cpu"), autoregressive=True)
