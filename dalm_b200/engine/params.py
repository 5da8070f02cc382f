"""HF-named parameter dictionaries: seeded random init (no checkpoints are reachable offline) and directory loading."""
from __future__ import annotations

import json
import math
import os
from typing import Dict, List, Optional

import torch


def _normal(gen: torch.Generator, shape, std: float, dtype, device) -> torch.Tensor:
    # CPU generator: reproducible across devices (tests, fixtures). A CUDA generator (bench-scale 7B models) draws on
    # the device directly.
    if gen.device.type == "cuda":
        return torch.empty(shape, dtype=torch.float32, device=gen.device).normal_(0.0, std, generator=gen).to(dtype)
    t = torch.empty(shape, dtype=torch.float32)
    t.normal_(mean=0.0, std=std, generator=gen)
    return t.to(device=device, dtype=dtype)


def random_state_dict(kind: str, cfg: Dict, seed: int = 0, dtype=torch.float32, device="cpu",
                      bias_std: Optional[float] = None, qk_norm_std: Optional[float] = None,
                      router_std: Optional[float] = None) -> Dict[str, torch.Tensor]:
    """HF parameter names for BertModel / XLMRobertaModel / RobertaModel / ModernBertModel (no prefix) / LlamaForCausalLM / Qwen2ForCausalLM /
    Qwen3ForCausalLM / MistralForCausalLM / FalconForCausalLM, init N(0, initializer_range), LN = (1, 0). Decoder attention biases (Qwen2's q/k/v, Llama's and Qwen3's
    `attention_bias`) are drawn from N(0, bias_std) (default: initializer_range) rather than HF's zeros, so that a dropped bias
    changes the outputs. Qwen3's q_norm / k_norm weights are 1 + N(0, qk_norm_std) (default: initializer_range), so that a
    dropped or swapped norm shows; so are every LayerNorm weight of ModernBERT. Qwen3MoeForCausalLM's sparse layers are
    written in the hub layout (`mlp.gate.weight` [E, H], `mlp.experts.{e}.{gate,up,down}_proj.weight`), the router weights
    drawn from N(0, router_std) (default: initializer_range): a larger std spreads the router probabilities, so that the
    top-k choice is far from ties."""
    on_device = torch.device(device).type == "cuda" and cfg.get("_device_rng", False)
    gen = torch.Generator(device=device) if on_device else torch.Generator()
    gen.manual_seed(seed)
    std = float(cfg.get("initializer_range", 0.02))
    H = cfg["hidden_size"]
    sd: Dict[str, torch.Tensor] = {}
    ones = lambda n: torch.ones(n, dtype=dtype, device=device)
    zeros = lambda n: torch.zeros(n, dtype=dtype, device=device)
    if kind in ("bert", "roberta"):                              # RoBERTa / XLM-R keep BertModel's parameter names and shapes
        F, V = cfg["intermediate_size"], cfg["vocab_size"]
        sd["embeddings.word_embeddings.weight"] = _normal(gen, (V, H), std, dtype, device)
        sd["embeddings.position_embeddings.weight"] = _normal(gen, (cfg["max_position_embeddings"], H), std, dtype, device)
        sd["embeddings.token_type_embeddings.weight"] = _normal(gen, (cfg["type_vocab_size"], H), std, dtype, device)
        sd["embeddings.LayerNorm.weight"] = ones(H)
        sd["embeddings.LayerNorm.bias"] = zeros(H)
        for l in range(cfg["num_hidden_layers"]):
            p = f"encoder.layer.{l}."
            for n in ("query", "key", "value"):
                sd[p + f"attention.self.{n}.weight"] = _normal(gen, (H, H), std, dtype, device)
                sd[p + f"attention.self.{n}.bias"] = _normal(gen, (H,), std, dtype, device)
            sd[p + "attention.output.dense.weight"] = _normal(gen, (H, H), std, dtype, device)
            sd[p + "attention.output.dense.bias"] = _normal(gen, (H,), std, dtype, device)
            sd[p + "attention.output.LayerNorm.weight"] = ones(H) + _normal(gen, (H,), std, dtype, device)
            sd[p + "attention.output.LayerNorm.bias"] = _normal(gen, (H,), std, dtype, device)
            sd[p + "intermediate.dense.weight"] = _normal(gen, (F, H), std, dtype, device)
            sd[p + "intermediate.dense.bias"] = _normal(gen, (F,), std, dtype, device)
            sd[p + "output.dense.weight"] = _normal(gen, (H, F), std, dtype, device)
            sd[p + "output.dense.bias"] = _normal(gen, (H,), std, dtype, device)
            sd[p + "output.LayerNorm.weight"] = ones(H) + _normal(gen, (H,), std, dtype, device)
            sd[p + "output.LayerNorm.bias"] = _normal(gen, (H,), std, dtype, device)
        sd["pooler.dense.weight"] = _normal(gen, (H, H), std, dtype, device)   # loaded by AutoModel, unused by the path
        sd["pooler.dense.bias"] = zeros(H)
    elif kind in ("llama", "qwen2", "qwen3", "mistral", "qwen3_moe"):
        F, V = cfg.get("intermediate_size"), cfg["vocab_size"]
        sparse = moe_layers(cfg) if kind == "qwen3_moe" else [False] * cfg["num_hidden_layers"]
        nh, nkv = cfg["num_attention_heads"], cfg.get("num_key_value_heads", cfg["num_attention_heads"])
        hd = cfg.get("head_dim") or H // nh
        qkv_bias, o_bias = attention_biases(kind, cfg)
        bstd = std if bias_std is None else float(bias_std)
        sd["model.embed_tokens.weight"] = _normal(gen, (V, H), std, dtype, device)
        for l in range(cfg["num_hidden_layers"]):
            p = f"model.layers.{l}."
            sd[p + "self_attn.q_proj.weight"] = _normal(gen, (nh * hd, H), std, dtype, device)
            sd[p + "self_attn.k_proj.weight"] = _normal(gen, (nkv * hd, H), std, dtype, device)
            sd[p + "self_attn.v_proj.weight"] = _normal(gen, (nkv * hd, H), std, dtype, device)
            sd[p + "self_attn.o_proj.weight"] = _normal(gen, (H, nh * hd), std, dtype, device)
            if qkv_bias:
                sd[p + "self_attn.q_proj.bias"] = _normal(gen, (nh * hd,), bstd, dtype, device)
                sd[p + "self_attn.k_proj.bias"] = _normal(gen, (nkv * hd,), bstd, dtype, device)
                sd[p + "self_attn.v_proj.bias"] = _normal(gen, (nkv * hd,), bstd, dtype, device)
            if o_bias:
                sd[p + "self_attn.o_proj.bias"] = _normal(gen, (H,), bstd, dtype, device)
            if kind in ("qwen3", "qwen3_moe"):
                nstd = std if qk_norm_std is None else float(qk_norm_std)
                sd[p + "self_attn.q_norm.weight"] = ones(hd) + _normal(gen, (hd,), nstd, dtype, device)
                sd[p + "self_attn.k_norm.weight"] = ones(hd) + _normal(gen, (hd,), nstd, dtype, device)
            if sparse[l]:
                E, I = cfg["num_experts"], cfg["moe_intermediate_size"]
                sd[p + "mlp.gate.weight"] = _normal(gen, (E, H), std if router_std is None else float(router_std), dtype, device)
                for e in range(E):
                    sd[p + f"mlp.experts.{e}.gate_proj.weight"] = _normal(gen, (I, H), std, dtype, device)
                    sd[p + f"mlp.experts.{e}.up_proj.weight"] = _normal(gen, (I, H), std, dtype, device)
                    sd[p + f"mlp.experts.{e}.down_proj.weight"] = _normal(gen, (H, I), std, dtype, device)
            else:
                sd[p + "mlp.gate_proj.weight"] = _normal(gen, (F, H), std, dtype, device)
                sd[p + "mlp.up_proj.weight"] = _normal(gen, (F, H), std, dtype, device)
                sd[p + "mlp.down_proj.weight"] = _normal(gen, (H, F), std, dtype, device)
            sd[p + "input_layernorm.weight"] = ones(H) + _normal(gen, (H,), std, dtype, device)
            sd[p + "post_attention_layernorm.weight"] = ones(H) + _normal(gen, (H,), std, dtype, device)
        sd["model.norm.weight"] = ones(H) + _normal(gen, (H,), std, dtype, device)
        if not cfg.get("tie_word_embeddings", False):             # tied checkpoints store no lm_head (Qwen2 0.5B-3B)
            sd["lm_head.weight"] = _normal(gen, (V, H), std, dtype, device)
    elif kind == "modernbert":                                   # ModernBertModel names (no prefix); no biases anywhere
        F, V = cfg["intermediate_size"], cfg["vocab_size"]
        sd["embeddings.tok_embeddings.weight"] = _normal(gen, (V, H), std, dtype, device)
        sd["embeddings.norm.weight"] = ones(H) + _normal(gen, (H,), std, dtype, device)
        for l in range(cfg["num_hidden_layers"]):
            p = f"layers.{l}."
            if l > 0:                                              # layer 0's attn_norm is nn.Identity
                sd[p + "attn_norm.weight"] = ones(H) + _normal(gen, (H,), std, dtype, device)
            sd[p + "attn.Wqkv.weight"] = _normal(gen, (3 * H, H), std, dtype, device)
            sd[p + "attn.Wo.weight"] = _normal(gen, (H, H), std, dtype, device)
            sd[p + "mlp_norm.weight"] = ones(H) + _normal(gen, (H,), std, dtype, device)
            sd[p + "mlp.Wi.weight"] = _normal(gen, (2 * F, H), std, dtype, device)
            sd[p + "mlp.Wo.weight"] = _normal(gen, (H, F), std, dtype, device)
        sd["final_norm.weight"] = ones(H) + _normal(gen, (H,), std, dtype, device)
    elif kind == "falcon":
        V = cfg["vocab_size"]
        nh = cfg["num_attention_heads"]
        hd = H // nh
        F = cfg.get("ffn_hidden_size") or 4 * H
        sd["transformer.word_embeddings.weight"] = _normal(gen, (V, H), std, dtype, device)
        for l in range(cfg["num_hidden_layers"]):
            p = f"transformer.h.{l}."
            sd[p + "input_layernorm.weight"] = ones(H) + _normal(gen, (H,), std, dtype, device)
            sd[p + "input_layernorm.bias"] = _normal(gen, (H,), std, dtype, device)
            sd[p + "self_attention.query_key_value.weight"] = _normal(gen, ((nh + 2) * hd, H), std, dtype, device)
            sd[p + "self_attention.dense.weight"] = _normal(gen, (H, H), std, dtype, device)
            sd[p + "mlp.dense_h_to_4h.weight"] = _normal(gen, (F, H), std, dtype, device)
            sd[p + "mlp.dense_4h_to_h.weight"] = _normal(gen, (H, F), std, dtype, device)
        sd["transformer.ln_f.weight"] = ones(H) + _normal(gen, (H,), std, dtype, device)
        sd["transformer.ln_f.bias"] = _normal(gen, (H,), std, dtype, device)
        # lm_head is tied to the word embeddings (tie_word_embeddings=True): not stored separately
    else:
        raise ValueError(f"unknown model kind {kind!r}")
    return sd


def load_config(path: str) -> Dict:
    with open(os.path.join(path, "config.json")) as f:
        return json.load(f)


RANDOM_INIT_MARKER = "dalm_b200_random_init.json"


def load_state_dict(path: str) -> Dict[str, torch.Tensor]:
    """Reads *.safetensors (single or sharded) or pytorch_model.bin from an HF-layout directory. A directory written by
    `synthetic.write_model_dir(..., with_weights=False)` carries a marker instead of weights ({"seed": n}): the public
    architecture is then random-initialised on the fly (on the GPU when there is one) - the offline stand-in for a hub
    checkpoint that BASELINE.json's configs prescribe ("random-init"), without writing 27 GB of Llama-2-7B to disk."""
    from safetensors.torch import load_file

    marker = os.path.join(path, RANDOM_INIT_MARKER)
    if os.path.exists(marker):
        with open(marker) as f:
            seed = int(json.load(f).get("seed", 0))
        cfg = load_config(path)
        on_gpu = torch.cuda.is_available()
        dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", torch.cuda.current_device()))) if on_gpu else torch.device("cpu")
        return random_state_dict(model_kind(cfg), dict(cfg, _device_rng=on_gpu), seed=seed,
                                 dtype=torch.bfloat16 if on_gpu else torch.float32, device=dev)
    files = sorted(f for f in os.listdir(path) if f.endswith(".safetensors") and not f.startswith("adapter"))
    sd: Dict[str, torch.Tensor] = {}
    if files:
        for f in files:
            sd.update(load_file(os.path.join(path, f)))
        return sd
    binf = os.path.join(path, "pytorch_model.bin")
    if os.path.exists(binf):
        return torch.load(binf, map_location="cpu", weights_only=True)
    raise FileNotFoundError(f"no weights (model.safetensors / pytorch_model.bin) under {path}")


def model_kind(cfg: Dict) -> str:
    """the engine family of an HF config; raises for model types, and for variants of the built ones, that are not built"""
    mt = cfg.get("model_type", "")
    if mt == "bert":
        return "bert"
    if mt in ("roberta", "xlm-roberta"):
        check_roberta(cfg)
        return "roberta"
    if mt in ("llama", "qwen2", "qwen3", "mistral", "qwen3_moe"):
        check_llama_family(cfg)
        return mt
    if mt == "modernbert":
        check_modernbert(cfg)
        return "modernbert"
    if mt == "falcon":
        check_rope_type(cfg)
        return "falcon"
    raise NotImplementedError(
        f"model_type {mt!r} is not built in dalm_b200 (supported: bert, roberta, xlm-roberta and modernbert encoders; llama, "
        "qwen2, qwen3, qwen3_moe, mistral and falcon decoders)")


def _rope_type(cfg: Dict) -> str:
    for key in ("rope_scaling", "rope_parameters"):
        rp = cfg.get(key)
        if isinstance(rp, dict):
            t = rp.get("rope_type", rp.get("type"))
            if t not in (None, "default"):
                return str(t)
    return "default"


def rope_parameters(cfg: Dict) -> Dict:
    """the RoPE settings of an HF config as transformers reads them: the hub spelling `rope_scaling` when it is set, else
    transformers 5's `rope_parameters`; `rope_type` (or the legacy `type`, default 'default') and `rope_theta` (the dict's own,
    else the top-level key, else 10000) always present"""
    rp = cfg.get("rope_scaling") or cfg.get("rope_parameters") or {}
    rp = dict(rp) if isinstance(rp, dict) else {}
    rp["rope_type"] = rp.get("rope_type", rp.get("type")) or "default"
    rp.setdefault("rope_theta", cfg.get("rope_theta", 10000.0))
    return rp


# RoPE types whose frequencies are a fixed table: a position-indexed cos / sin table represents them exactly. `dynamic` changes
# the frequencies with the sequence length, `yarn` / `longrope` also scale the attention, `proportional` rotates part of a head.
BUILT_ROPE_TYPES = {"llama": ("default", "linear", "llama3")}


def check_rope_type(cfg: Dict) -> str:
    """the config's RoPE type; raises NotImplementedError, naming it, when the model family does not build it"""
    mt = cfg.get("model_type", "")
    rt = rope_parameters(cfg)["rope_type"]
    built = BUILT_ROPE_TYPES.get(mt, ("default",))
    if rt not in built:
        raise NotImplementedError(f"{mt}: RoPE type {rt!r} (rope_scaling / rope_parameters) is not built; built: "
                                  + ", ".join(repr(t) for t in built))
    return rt


def rope_inv_freq(cfg: Dict, head_dim: int) -> torch.Tensor:
    """fp32 [head_dim / 2] inverse frequencies of the config's RoPE, bit for bit what transformers' rope init functions
    (modeling_rope_utils: default, `linear`, `llama3`) compute on the CPU: the same fp32 operations in the same order. All
    three have attention factor 1, so cos / sin tables built from these frequencies are the whole of the position encoding."""
    rt = check_rope_type(cfg)
    rp = rope_parameters(cfg)
    base = rp["rope_theta"]
    inv_freq = 1.0 / (base ** (torch.arange(0, head_dim, 2, dtype=torch.int64).to(dtype=torch.float) / head_dim))
    if rt == "linear":
        inv_freq /= rp["factor"]
    elif rt == "llama3":
        factor, low, high = rp["factor"], rp["low_freq_factor"], rp["high_freq_factor"]
        old_len = rp.get("original_max_position_embeddings") or cfg.get("original_max_position_embeddings") \
            or cfg["max_position_embeddings"]
        low_freq_wavelen, high_freq_wavelen = old_len / low, old_len / high
        wavelen = 2 * math.pi / inv_freq
        # wavelengths above old_len / low are divided by factor, those below old_len / high kept, the band between blended
        scaled = torch.where(wavelen > low_freq_wavelen, inv_freq / factor, inv_freq)
        smooth = (old_len / wavelen - low) / (high - low)
        smoothed = (1 - smooth) * scaled / factor + smooth * scaled
        medium = ~(wavelen < high_freq_wavelen) * ~(wavelen > low_freq_wavelen)
        inv_freq = torch.where(medium, smoothed, scaled)
    return inv_freq


def check_llama_family(cfg: Dict) -> None:
    """refuses the settings of a llama / qwen2 / qwen3 / mistral config that LlamaDecoder would otherwise silently compute wrong"""
    mt = cfg.get("model_type", "")
    if mt == "mistral":
        missing = [k for k in MISTRAL_SHAPE_KEYS if k not in cfg]
        if missing:
            raise NotImplementedError(f"mistral: a config without {', '.join(missing)} is not built (transformers would fill "
                                      "in MistralConfig's defaults, the 7B shape; the shape is read from config.json only)")
    if mt in ("llama", "mistral"):
        check_rope_type(cfg)
    if mt != "mistral" and cfg.get("mlp_bias", False):        # MistralMLP has no bias whatever the key says
        raise NotImplementedError(f"{mt}: mlp_bias=true is not built (the fused SwiGLU MLP has no bias)")
    if mt == "qwen3_moe":
        check_qwen3_moe(cfg)
    if mt in ("qwen3", "qwen3_moe"):
        hd = cfg.get("head_dim") or cfg["hidden_size"] // cfg["num_attention_heads"]
        if hd != 128:
            raise NotImplementedError(f"{mt}: head_dim={hd} is not built (the q/k norm kernels take head_dim 128)")
    if mt == "qwen3_moe":
        rt = _rope_type(cfg)
        if rt != "default":
            raise NotImplementedError(f"{mt}: RoPE type {rt!r} (rope_scaling / rope_parameters) is not built; only 'default'")
    if mt in ("qwen2", "qwen3"):
        if not cfg.get("use_sliding_window", False) and "sliding_attention" in (cfg.get("layer_types") or ()):
            # transformers then sets sliding_window to None but still builds sliding-window masks for those layers
            raise NotImplementedError(f"{mt}: layer_types marks sliding_attention layers while use_sliding_window is false")
        if cfg.get("use_sliding_window", False) and not any(sliding_windows(cfg)):
            # transformers then runs full attention on every layer, while the Qwen documentation of max_window_layers reads
            # the other way round (the first max_window_layers layers windowed): the config does not say which it means
            raise NotImplementedError(
                f"{mt}: use_sliding_window=true selects no sliding-window layer (sliding_window="
                f"{cfg.get('sliding_window', 4096)}, max_window_layers={cfg.get('max_window_layers', 28)} of "
                f"{cfg.get('num_hidden_layers')} layers, layer_types={cfg.get('layer_types')}); set use_sliding_window=false "
                "or list the sliding_attention layers in layer_types")
        rt = _rope_type(cfg)
        if rt != "default":
            raise NotImplementedError(f"{mt}: RoPE type {rt!r} (rope_scaling / rope_parameters) is not built; only 'default'")


# Qwen3-MoE: the keys without which transformers would fill in Qwen3MoeConfig's 30B-A3B defaults (the shape is read from
# config.json only), and the bounds of the routing kernels (csrc/moe.cu) and of the gate GEMM (N = E, then K = E: % 8)
QWEN3_MOE_KEYS = ("num_experts", "num_experts_per_tok", "moe_intermediate_size")
MOE_MAX_EXPERTS, MOE_MAX_TOPK = 256, 16


def check_qwen3_moe(cfg: Dict) -> None:
    """refuses a qwen3_moe config the routed MLP would otherwise compute wrong or cannot run"""
    missing = [k for k in QWEN3_MOE_KEYS if k not in cfg]
    if missing:
        raise NotImplementedError(f"qwen3_moe: a config without {', '.join(missing)} is not built (transformers would fill in "
                                  "Qwen3MoeConfig's defaults, the 30B-A3B shape; the shape is read from config.json only)")
    E, k, I = int(cfg["num_experts"]), int(cfg["num_experts_per_tok"]), int(cfg["moe_intermediate_size"])
    if E > 0:
        if E % 8 or E > MOE_MAX_EXPERTS:
            raise NotImplementedError(f"qwen3_moe: num_experts={E} is not built (the router kernels take a multiple of 8 up to "
                                      f"{MOE_MAX_EXPERTS})")
        if not 1 <= k <= min(E, MOE_MAX_TOPK):
            raise NotImplementedError(f"qwen3_moe: num_experts_per_tok={k} is not built (the router takes 1 to "
                                      f"min(num_experts, {MOE_MAX_TOPK}))")
        if I <= 0 or I % 128:
            raise NotImplementedError(f"qwen3_moe: moe_intermediate_size={I} is not built (the grouped SwiGLU GEMM takes a "
                                      "multiple of 128: 128-feature gate / up blocks)")
        if cfg["hidden_size"] % 64:
            raise NotImplementedError(f"qwen3_moe: hidden_size={cfg['hidden_size']} is not built (the experts' down-projection "
                                      "dgrad takes a multiple of 64)")
    if not all(moe_layers(cfg)) and "intermediate_size" not in cfg:
        raise NotImplementedError("qwen3_moe: dense MLP layers (mlp_only_layers / decoder_sparse_step) need intermediate_size "
                                  "in config.json")


def moe_layers(cfg: Dict) -> List[bool]:
    """which layers of a qwen3_moe config run the routed MLP, as Qwen3MoeDecoderLayer decides: not in `mlp_only_layers`,
    num_experts > 0 and (i + 1) % decoder_sparse_step == 0; the others run the dense SwiGLU MLP of `intermediate_size`"""
    n = int(cfg["num_hidden_layers"])
    only = set(cfg.get("mlp_only_layers") or ())
    step = int(cfg.get("decoder_sparse_step", 1))
    return [i not in only and int(cfg.get("num_experts", 0)) > 0 and (i + 1) % step == 0 for i in range(n)]


MISTRAL_DEFAULT_WINDOW = 4096                                    # MistralConfig's sliding_window when the key is absent
MISTRAL_SHAPE_KEYS = ("hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads", "vocab_size")


def sliding_windows(cfg: Dict) -> List[int]:
    """the key window of every layer (0 = full causal attention), resolved as transformers' config classes resolve it:
    - mistral: `sliding_window` for every layer; an absent key means 4096, null means none. MistralConfig ignores
      `layer_types` (alternating layers are Ministral, another model type), and so does this.
    - qwen2 / qwen3: `sliding_window` only with `use_sliding_window`, on the layers `layer_types` marks "sliding_attention",
      or when that list is absent on layers i >= `max_window_layers` (default 28).
    - qwen3_moe: `sliding_window` (default 4096) on every layer when `use_sliding_window`, as Qwen3MoeConfig and its
      attention read it (no `max_window_layers` or `layer_types`).
    - llama: none.
    A layer with window w lets query i see key j iff i - w < j <= i, in the indices of the padded row."""
    mt, n = cfg.get("model_type", ""), int(cfg["num_hidden_layers"])
    if mt == "mistral":
        w = cfg.get("sliding_window", MISTRAL_DEFAULT_WINDOW)
        return [int(w) if w else 0] * n
    if mt == "qwen3_moe":
        w = cfg.get("sliding_window", 4096) if cfg.get("use_sliding_window", False) else 0
        return [int(w) if w else 0] * n
    if mt in ("qwen2", "qwen3"):
        w = cfg.get("sliding_window", 4096)
        if not cfg.get("use_sliding_window", False) or not w:
            return [0] * n
        types = cfg.get("layer_types")
        if types is None:
            first = int(cfg.get("max_window_layers", 28))
            types = ["sliding_attention" if i >= first else "full_attention" for i in range(n)]
        if len(types) != n:
            raise ValueError(f"{mt}: layer_types lists {len(types)} layers, num_hidden_layers is {n}")
        return [int(w) if t == "sliding_attention" else 0 for t in types]
    return [0] * n


def check_roberta(cfg: Dict) -> None:
    """refuses the settings of a roberta / xlm-roberta config that BertEncoder would otherwise silently compute wrong"""
    mt = cfg.get("model_type", "")
    pet = cfg.get("position_embedding_type", "absolute")
    if pet != "absolute":
        raise NotImplementedError(f"{mt}: position_embedding_type={pet!r} is not built; only 'absolute'")
    act = cfg.get("hidden_act", "gelu")
    if act != "gelu":
        raise NotImplementedError(f"{mt}: hidden_act={act!r} is not built; only 'gelu' (erf)")
    if cfg.get("is_decoder", False):
        raise NotImplementedError(f"{mt}: is_decoder=true (causal self-attention) is not built")
    if cfg.get("add_cross_attention", False):
        raise NotImplementedError(f"{mt}: add_cross_attention=true is not built")


MODERNBERT_THETA = {"full_attention": ("global_rope_theta", 160000.0), "sliding_attention": ("local_rope_theta", 10000.0)}


def modernbert_rope_parameters(cfg: Dict) -> Dict[str, Dict]:
    """{"full_attention": {...}, "sliding_attention": {...}} as ModernBertConfig resolves them: `rope_parameters` when given,
    `rope_scaling` merged into both, and a missing rope_theta taken from the hub spelling `global_rope_theta` /
    `local_rope_theta` (defaults 160000 / 10000)"""
    rp = cfg.get("rope_parameters")
    rp = {k: dict(v) if isinstance(v, dict) else v for k, v in rp.items()} if isinstance(rp, dict) else {}
    rs = cfg.get("rope_scaling")
    out = {}
    for lt, (key, theta) in MODERNBERT_THETA.items():
        d = rp.get(lt) or {"rope_type": "default"}
        if rs is not None:
            d.update(rs)
        d.setdefault("rope_theta", cfg.get(key, theta))
        d["rope_type"] = d.get("rope_type", d.get("type")) or "default"
        out[lt] = d
    return out


def modernbert_layer_types(cfg: Dict) -> List[str]:
    """`layer_types`, or else layer i is full attention iff i % global_attn_every_n_layers == 0 (default 3)"""
    n = int(cfg["num_hidden_layers"])
    types = cfg.get("layer_types")
    if types is None:
        every = int(cfg.get("global_attn_every_n_layers", 3))
        types = ["sliding_attention" if i % every else "full_attention" for i in range(n)]
    if len(types) != n:
        raise ValueError(f"modernbert: layer_types lists {len(types)} layers, num_hidden_layers is {n}")
    return list(types)


def modernbert_layers(cfg: Dict) -> List[tuple]:
    """(window, inv_freq) of every layer. window: 0 for a global layer; for a local one local_attention // 2 + 1, so that query
    i sees key j iff |i - j| < window, i.e. |i - j| <= local_attention // 2 (transformers' sliding-window mask). inv_freq: fp32
    [head_dim / 2], bit for bit ModernBertRotaryEmbedding's buffer of the layer's type."""
    hd = cfg["hidden_size"] // cfg["num_attention_heads"]
    rope = modernbert_rope_parameters(cfg)
    freqs = {lt: rope_inv_freq({"model_type": "modernbert", "rope_parameters": dict(rp)}, hd) for lt, rp in rope.items()}
    win = int(cfg.get("local_attention", 128)) // 2 + 1
    return [(win if t == "sliding_attention" else 0, freqs[t]) for t in modernbert_layer_types(cfg)]


def check_modernbert(cfg: Dict) -> None:
    """refuses the settings of a modernbert config that ModernBertEncoder would otherwise silently compute wrong. Every
    published ModernBERT retriever has zero dropout, no biases and the erf GELU."""
    for k in ("attention_dropout", "mlp_dropout", "embedding_dropout"):
        if float(cfg.get(k) or 0.0) != 0.0:
            raise NotImplementedError(f"modernbert: {k}={cfg[k]} is not built (dropout is not built for ModernBERT)")
    act = cfg.get("hidden_activation", "gelu")
    if act != "gelu":
        raise NotImplementedError(f"modernbert: hidden_activation={act!r} is not built; only 'gelu' (erf)")
    for k in ("norm_bias", "mlp_bias", "attention_bias"):
        if cfg.get(k, False):
            raise NotImplementedError(f"modernbert: {k}=true is not built (biases are not built for ModernBERT)")
    for lt, rp in modernbert_rope_parameters(cfg).items():
        if rp["rope_type"] != "default":
            raise NotImplementedError(f"modernbert: RoPE type {rp['rope_type']!r} ({lt}) is not built; only 'default'")
    hd = cfg["hidden_size"] // cfg["num_attention_heads"]
    if hd not in (32, 64, 128):
        raise NotImplementedError(f"modernbert: head_dim {hd} is not built (the attention kernels take 32 / 64 / 128)")
    modernbert_layer_types(cfg)


def roberta_max_len(cfg: Dict) -> int:
    """the longest sequence a roberta / xlm-roberta position table serves: positions run from pad_token_id + 1, so
    max_position_embeddings - pad_token_id - 1 (512 for the 514-row tables, 8192 for bge-m3's 8194)"""
    return int(cfg["max_position_embeddings"]) - int(cfg.get("pad_token_id", 1)) - 1


def attention_biases(kind: str, cfg: Dict):
    """(q/k/v projections carry a bias, o_proj carries a bias) for a llama-family config: Qwen2 has q/k/v biases only, Llama
    and Qwen3 have all four when `attention_bias` is set, Mistral has none (MistralAttention ignores the key)"""
    if kind == "qwen2":
        return True, False
    if kind == "mistral":
        return False, False
    # qwen3_moe: Qwen3MoeAttention, Qwen3's attention (`attention_bias` on all four projections)
    ab = bool(cfg.get("attention_bias", False))
    return ab, ab


def is_bnb_linear_weight(name: str) -> bool:
    """the tensors `load_in_4bit` replaces: every nn.Linear weight except the LM head (transformers keeps `lm_head` and tied
    output embeddings out of the conversion); embeddings and norms are not Linear"""
    return (name.endswith(".weight") and "embed" not in name and "LayerNorm" not in name and "layernorm" not in name
            and "norm.weight" not in name and "ln_f" not in name and not name.startswith("lm_head"))


def bnb_nf4_state_dict(sd: Dict[str, torch.Tensor], device) -> Dict[str, torch.Tensor]:
    """`use_bnb` (reference rag_e2e_base_model.py:136-142): fp32 tensors on `device` holding exactly the values the
    reference's 4-bit model computes with — nn.Linear weights through the NF4 quantise/dequantise round trip (csrc/nf4.cu),
    everything else through the fp16 cast transformers applies when a bitsandbytes config is given without torch_dtype."""
    from .. import ops

    out = {}
    for k, v in sd.items():
        t = v.to(device=device, dtype=torch.float32).contiguous().clone()
        if t.dim() == 2 and is_bnb_linear_weight(k):
            ops.nf4_roundtrip_(t)
        else:
            t = t.to(torch.float16).to(torch.float32)            # dtype casts only
        out[k] = t
    return out
