"""CPU: OLMo 2 / OLMo 3 / OLMoE configs (model kind, refusals with their reasons, sliding windows, YaRN frequencies and attention
factor against transformers), the random-init layout, and the synthetic directories as transformers' Olmo2ForCausalLM /
Olmo3ForCausalLM / OlmoeForCausalLM load them."""
import os

import pytest
import torch

from dalm_b200 import synthetic
from dalm_b200.engine import params

KIND = {"olmo2-tiny": "olmo2", "olmo2-hd128-gqa": "olmo2", "olmo3-tiny": "olmo3", "olmoe-tiny": "olmoe"}


def _cfg(name="olmo2-tiny", **kw):
    return dict(synthetic.olmo_config(name, vocab_size=400), **kw)


def test_model_kind_maps_olmo():
    for name in synthetic.OLMO_SHAPES:
        cfg = synthetic.olmo_config(name)
        assert params.model_kind(cfg) == cfg["model_type"]
    assert params.model_kind(_cfg(rope_scaling=None, rope_parameters={"rope_theta": 5e5, "rope_type": "default"})) == "olmo2"


@pytest.mark.parametrize("name,extra,match", [
    ("olmoe-tiny", dict(clip_qkv=8.0), "olmoe: clip_qkv=8.0 is not built"),
    ("olmo2-tiny", dict(clip_qkv=4.0), "olmo2: clip_qkv=4.0 is not built"),
    ("olmo2-tiny", dict(hidden_act="gelu"), "olmo2: hidden_act='gelu' is not built; only 'silu'"),
    ("olmo3-tiny", dict(head_dim=32), "olmo3: head_dim=32 is not built"),
    ("olmo2-tiny", dict(num_attention_heads=8), "olmo2: head_dim=32 is not built"),
    ("olmo2-tiny", dict(rope_scaling={"rope_type": "linear", "factor": 2.0}), "olmo2: RoPE type 'linear'"),
    ("olmo3-tiny", dict(rope_scaling={"rope_type": "dynamic", "factor": 2.0}), "olmo3: RoPE type 'dynamic'"),
    ("olmoe-tiny", dict(rope_scaling={"rope_type": "llama3", "factor": 8.0}), "olmoe: RoPE type 'llama3'"),
    ("olmoe-tiny", dict(intermediate_size=192), "olmoe: intermediate_size=192 .*multiple of 128"),
    ("olmoe-tiny", dict(num_experts=12), "olmoe: num_experts=12 .*multiple of 8"),
    ("olmoe-tiny", dict(num_experts=264), "olmoe: num_experts=264 .*up to 256"),
    ("olmoe-tiny", dict(num_experts_per_tok=9), "olmoe: num_experts_per_tok=9 .*min\\(num_experts, 16\\)"),
    ("olmo2-tiny", dict(attention_bias=True), "olmo2: attention_bias=true"),
    ("olmo2-tiny", dict(hidden_size=16384, num_attention_heads=128, num_key_value_heads=8),
     "olmo2: 128 q \\+ 8 k heads of 128 are not built"),
])
def test_olmo_refusals(name, extra, match):
    with pytest.raises(NotImplementedError, match=match):
        params.model_kind(_cfg(name, **extra))


@pytest.mark.parametrize("key", ["num_experts", "num_experts_per_tok"])
def test_olmoe_needs_its_moe_keys(key):
    cfg = _cfg("olmoe-tiny")
    del cfg[key]
    with pytest.raises(NotImplementedError, match=f"olmoe: a config without {key}"):
        params.model_kind(cfg)


def test_olmo2_needs_its_shape_keys():
    cfg = _cfg()
    del cfg["intermediate_size"]
    with pytest.raises(NotImplementedError, match="olmo2: a config without intermediate_size"):
        params.model_kind(cfg)


@pytest.mark.parametrize("mt", ["llama", "qwen2", "qwen3", "mistral"])
def test_yarn_still_refused_for_other_families(mt):
    cfg = {"llama": synthetic.llama_config("llama-tiny", 400), "qwen2": synthetic.qwen2_config("qwen2-tiny", 400),
           "qwen3": synthetic.qwen3_config("qwen3-tiny", 400), "mistral": synthetic.mistral_config("mistral-tiny", 400)}[mt]
    cfg = dict(cfg, rope_scaling={"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 2048})
    with pytest.raises(NotImplementedError, match=f"{mt}: RoPE type 'yarn'"):
        params.model_kind(cfg)


YARN_CASES = [
    dict(rope_type="yarn", factor=4.0, original_max_position_embeddings=128),
    dict(rope_type="yarn", factor=8.0, original_max_position_embeddings=8192, attention_factor=1.2079441541679836,
         beta_fast=32, beta_slow=1),
    dict(rope_type="yarn", factor=8.0, original_max_position_embeddings=4096, truncate=False),
    dict(rope_type="yarn", factor=16.0, original_max_position_embeddings=2048, beta_fast=16, beta_slow=2, mscale=0.707,
         mscale_all_dim=1.0),
    dict(rope_type="yarn", factor=2.0, original_max_position_embeddings=1024, attention_factor=0.9, truncate=False),
]


@pytest.mark.parametrize("case", range(len(YARN_CASES)))
@pytest.mark.parametrize("name", ["olmo3-tiny", "olmo2-hd128-gqa"])
def test_yarn_matches_transformers(name, case):
    """inverse frequencies bit-equal to transformers' yarn init function, and the same attention factor"""
    from transformers import AutoConfig
    from transformers.modeling_rope_utils import ROPE_INIT_FUNCTIONS
    cfg = _cfg(name, rope_scaling=dict(YARN_CASES[case]), max_position_embeddings=65536, rope_theta=500000.0)
    hf = AutoConfig.for_model(**{k: v for k, v in cfg.items() if k != "architectures"})
    want_freq, want_factor = ROPE_INIT_FUNCTIONS["yarn"](hf, "cpu")
    hd = cfg["hidden_size"] // cfg["num_attention_heads"]
    got = params.rope_inv_freq(cfg, hd)
    assert got.dtype == torch.float32 and torch.equal(got, want_freq)
    assert params.rope_attention_factor(cfg, hd) == want_factor


def test_default_rope_has_unit_attention_factor():
    assert params.rope_attention_factor(_cfg(), 64) == 1.0


def test_sliding_windows_olmo3():
    """Olmo3Config: sliding_window on the layers layer_types marks sliding; without the list every fourth layer is full"""
    from transformers import Olmo3Config
    cfg = _cfg("olmo3-tiny")
    assert params.sliding_windows(cfg) == [16, 16, 16, 0]
    for n in (4, 6, 9):
        c = dict(cfg, num_hidden_layers=n)
        del c["layer_types"]
        hf = Olmo3Config(**{k: v for k, v in c.items() if k not in ("architectures", "model_type")})
        assert params.sliding_windows(c) == [16 if t == "sliding_attention" else 0 for t in hf.layer_types]
    types = ["full_attention", "sliding_attention", "sliding_attention", "full_attention"]
    assert params.sliding_windows(dict(cfg, layer_types=types)) == [0, 16, 16, 0]
    assert params.sliding_windows(dict(cfg, sliding_window=None)) == [0, 0, 0, 0]
    with pytest.raises(ValueError, match="layer_types lists 2 layers"):
        params.sliding_windows(dict(cfg, layer_types=types[:2]))
    assert params.sliding_windows(_cfg()) == [0, 0] and params.sliding_windows(_cfg("olmoe-tiny")) == [0, 0, 0]


def test_olmoe_every_layer_sparse():
    from transformers import OlmoeConfig
    from transformers.models.olmoe.modeling_olmoe import OlmoeDecoderLayer, OlmoeSparseMoeBlock
    cfg = _cfg("olmoe-tiny")
    hf = OlmoeConfig(**{k: v for k, v in cfg.items() if k not in ("architectures", "model_type")})
    assert params.moe_layers(cfg) == [isinstance(OlmoeDecoderLayer(hf, i).mlp, OlmoeSparseMoeBlock) for i in range(3)]


def _fused(sd, cfg):
    out = {k: v for k, v in sd.items() if ".mlp.experts." not in k}
    for l in range(cfg["num_hidden_layers"]):
        p = f"model.layers.{l}.mlp.experts."
        E = cfg["num_experts"]
        out[p + "gate_up_proj"] = torch.stack([torch.cat([sd[p + f"{e}.gate_proj.weight"], sd[p + f"{e}.up_proj.weight"]])
                                               for e in range(E)])
        out[p + "down_proj"] = torch.stack([sd[p + f"{e}.down_proj.weight"] for e in range(E)])
    return out


@pytest.mark.parametrize("name", list(KIND))
def test_synthetic_directory_loads_in_transformers(tmp_path, name):
    """write_model_dir: transformers' Olmo2 / Olmo3 / OlmoeForCausalLM load every tensor unchanged (OLMoE's experts in its
    fused layout), q_norm / k_norm span the whole projection widths, and the tokenizer round-trips"""
    from safetensors.torch import load_file
    from transformers import AutoModelForCausalLM, AutoTokenizer
    kind = KIND[name]
    d = synthetic.write_model_dir(str(tmp_path / "m"), kind, name, vocab_size=400, qk_norm_std=0.1)
    cfg = params.load_config(d)
    sd = load_file(os.path.join(d, "model.safetensors"))
    m = AutoModelForCausalLM.from_pretrained(d, dtype=torch.float32)
    assert type(m).__name__ == synthetic.OLMO_ARCH[kind]
    got = m.state_dict()
    want = _fused(sd, cfg) if kind == "olmoe" else sd
    assert set(got) == set(want)
    for k, v in want.items():
        assert torch.equal(got[k], v), k
    hd = cfg["hidden_size"] // cfg["num_attention_heads"]
    assert sd["model.layers.0.self_attn.q_norm.weight"].shape == (cfg["num_attention_heads"] * hd,)
    assert sd["model.layers.0.self_attn.k_norm.weight"].shape == (cfg["num_key_value_heads"] * hd,)
    assert ("model.layers.0.input_layernorm.weight" in sd) == (kind == "olmoe")
    assert ("model.layers.0.post_feedforward_layernorm.weight" in sd) == (kind != "olmoe")
    tok = AutoTokenizer.from_pretrained(d)
    assert tok.decode(tok("ka to mi")["input_ids"]) == "ka to mi"
    if kind == "olmo3":                                          # transformers reads the same windows and YaRN factor
        assert [w if t == "sliding_attention" else 0 for t, w in
                zip(m.config.layer_types, [m.config.sliding_window] * 4)] == params.sliding_windows(cfg)
        assert m.model.rotary_emb.attention_scaling == params.rope_attention_factor(cfg, hd)


@pytest.fixture(scope="module")
def olmo_dirs(tmp_path_factory):
    root = tmp_path_factory.mktemp("olmo")
    return {n: synthetic.write_model_dir(str(root / n), KIND[n], n, vocab_size=400, with_weights=False)
            for n in ("olmo2-tiny", "olmoe-tiny")}


@pytest.mark.parametrize("kw,match", [
    (dict(full=True), "full fine-tuning of a olmoe generator is not built: grouped expert weight gradients .*125 GB"),
    (dict(bnb=True), "use_bnb on a olmoe generator is not built"),
])
def test_build_decoder_refuses_olmoe_modes(olmo_dirs, kw, match):
    from dalm_b200.models.rag_e2e_base_model import build_decoder
    with pytest.raises(NotImplementedError, match=match):
        build_decoder(olmo_dirs["olmoe-tiny"], lora=False, device=torch.device("cpu"), **kw)


@pytest.mark.parametrize("name", ["olmo2-tiny", "olmoe-tiny"])
def test_nf4_storage_refused(olmo_dirs, monkeypatch, name):
    from dalm_b200.models.rag_e2e_base_model import build_decoder
    monkeypatch.setenv("DALM_B200_NF4_STORAGE", "1")
    kind = KIND[name]                                # olmoe: use_bnb itself is refused first
    with pytest.raises(NotImplementedError, match=f"(4-bit storage is built for .* not '{kind}'|use_bnb on a {kind} generator)"):
        build_decoder(olmo_dirs[name], lora=True, device=torch.device("cpu"), bnb=True)


def test_olmoe_autoregressive_retriever_refused(olmo_dirs):
    from dalm_b200.models.rag_e2e_base_model import build_encoder
    with pytest.raises(NotImplementedError, match="autoregressive retrievers are built for .* OLMo 2 and OLMo 3"):
        build_encoder(olmo_dirs["olmoe-tiny"], lora=True, device=torch.device("cpu"), autoregressive=True)
