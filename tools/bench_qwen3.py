"""Qwen3-8B-shaped measurements on one GPU, printed as one JSON line:
  * the card's name and power limit (part of every number below);
  * `gemm_rope` at the 8B q|k|v shape (M = 18 x 256 rows, N = 6144, K = 4096) without and with the per-head q/k RMSNorm in the
    epilogue (the norm launch also writes the pre-norm q|k columns and rstd the backward reads), alternated, CUDA events;
  * the norm-RoPE backward kernel (with the norm weights' gradients) against `rope_(backward=True)` on the same q|k columns;
  * greedy decode tokens/s (prompt 256, 256 new tokens, no EOS) at B = 8 (decode_gemm path) and B = 64 (wgmma path), next to
    transformers' `generate` on the same random bf16 weights on the same GPU.
    python tools/bench_qwen3.py [--skip-hf]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from dalm_b200 import ops, synthetic  # noqa: E402
from dalm_b200.engine import params  # noqa: E402
from dalm_b200.engine.llama import LlamaDecoder  # noqa: E402
from tools.bench_qwen2 import card, decode_rates, time_pair  # noqa: E402

bf16, f32 = torch.bfloat16, torch.float32


def kernel_norm_cost(dev, cfg):
    H, hd = cfg["hidden_size"], cfg["head_dim"]
    nq, nkv = cfg["num_attention_heads"], cfg["num_key_value_heads"]
    N, rc = (nq + 2 * nkv) * hd, (nq + nkv) * hd
    g = torch.Generator(device=dev).manual_seed(0)
    w = (torch.randn(N, H, device=dev, generator=g) * 0.02).to(bf16)
    L, M = 256, 18 * 256
    a = torch.randn(M, H, device=dev, generator=g).to(bf16)
    inv = 1.0 / (cfg["rope_theta"] ** (torch.arange(0, 128, 2, dtype=f32, device=dev) / 128))
    fr = torch.outer(torch.arange(L, dtype=f32, device=dev), inv)
    cos_t, sin_t = fr.cos().contiguous(), fr.sin().contiguous()
    qn = 1 + 0.1 * torch.randn(128, device=dev, generator=g)
    kn = 1 + 0.1 * torch.randn(128, device=dev, generator=g)
    out = torch.empty(M, N, dtype=bf16, device=dev)
    pre = torch.empty(M, rc, dtype=bf16, device=dev)
    rstd = torch.empty(M, nq + nkv, dtype=f32, device=dev)
    norm = dict(q_norm=qn, k_norm=kn, nq_heads=nq, eps=cfg["rms_norm_eps"], pre_out=pre, rstd_out=rstd)
    t0, t1 = time_pair(lambda: ops.gemm_rope(a, w, cos_t, sin_t, L, rc, out=out),
                       lambda: ops.gemm_rope(a, w, cos_t, sin_t, L, rc, out=out, **norm))
    ops.gemm_rope(a, w, cos_t, sin_t, L, rc, out=out, **norm)
    d = torch.randn(M, N, device=dev, generator=g).to(bf16)
    dwq, dwk = torch.zeros(128, device=dev), torch.zeros(128, device=dev)
    # both kernels work in place; re-running them on their own output keeps the values finite (rotations, rstd-scaled maps)
    b0, b1 = time_pair(lambda: ops.rope_(d, 0, nq + nkv, hd, cos_t, sin_t, L, backward=True),
                       lambda: ops.qk_norm_rope_bwd_(d, nq + nkv, nq, qn, kn, cos_t, sin_t, L, pre, rstd, dw_q=dwq, dw_k=dwk))
    return {"gemm_rope_shape_MxNxK": [M, N, H], "gemm_rope_us": {"rope": t0, "qk_norm_rope": t1},
            "bwd_rows_x_qk_cols": [M, rc], "bwd_us": {"rope_backward": b0, "qk_norm_rope_bwd": b1}}


def hf_model(cfg, sd, dev):
    from transformers import Qwen3Config, Qwen3ForCausalLM
    from transformers.initialization import no_init_weights
    keep = {k: v for k, v in cfg.items() if k not in ("architectures", "model_type")}
    with no_init_weights(), torch.device(dev):
        m = Qwen3ForCausalLM(Qwen3Config(**keep)).to(bf16)
    m.load_state_dict(sd, strict=False)
    return m.eval()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-hf", action="store_true", help="leave out transformers' generate")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_qwen3: needs a CUDA device")
    dev = torch.device("cuda:0")
    cfg = synthetic.qwen3_config("qwen3-8b")
    res = {"what": "Qwen3-8B shape", **card(), "torch": torch.__version__}
    res["qk_norm_cost"] = kernel_norm_cost(dev, cfg)
    sd = params.random_state_dict("qwen3", dict(cfg, _device_rng=True), seed=0, dtype=bf16, device=dev)
    dec = LlamaDecoder(cfg, sd, device=dev)
    hf = None if args.skip_hf else hf_model(cfg, sd, dev)
    del sd
    torch.cuda.empty_cache()
    res["greedy_decode"] = [decode_rates(dec, hf, cfg, dev, B) for B in (8, 64)]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
