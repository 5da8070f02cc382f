"""A/B of two builds of libdalm_b200.so in one GPU session: the parent commit's library against the working tree's.

    python tools/ab_gemm_epilogue.py --build-parent REV        # CPU, once: build REV's library into build/ab_parent/
    python tools/ab_gemm_epilogue.py hash                      # outputs of both libraries, hashed and compared
    python tools/ab_gemm_epilogue.py gemm [--rounds 3]         # GEMM times, the arms alternating
    python tools/ab_gemm_epilogue.py bench [--rounds 3]        # bench.py cfg-3 (rounds x per arm) and cfg-2 (once per arm)

bench.py runs as `--gpus 1 --steps 10 --warmup 3` without its CPU-oracle and HF-eager baselines, which time other code.

Every arm runs in a subprocess of its own with dalm_b200._lib.LIB_PATH pointed at its library. For bench.py, which loads the
in-tree library, the arm's library is copied into dalm_b200/csrc/ before each run and the working tree's copy is put back at
the end. Results are JSON lines; per case the median and the spread (max - min) of each arm.
"""
import argparse, hashlib, json, os, shutil, statistics, subprocess, sys, tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PARENT_LIB = os.path.join(ROOT, "build", "ab_parent", "libdalm_b200.so")
TREE_LIB = os.path.join(ROOT, "dalm_b200", "csrc", "libdalm_b200.so")


def build_parent(rev):
    """REV's dalm_b200/csrc + include, built in a scratch directory; the library goes to build/ab_parent/"""
    with tempfile.TemporaryDirectory() as tmp:
        arch = subprocess.run(["git", "-C", ROOT, "archive", rev, "dalm_b200/csrc", "include"], check=True, capture_output=True).stdout
        subprocess.run(["tar", "-x", "-C", tmp], input=arch, check=True)
        subprocess.run([sys.executable, os.path.join(tmp, "dalm_b200", "csrc", "build.py"), "--force"], check=True, cwd=tmp)
        os.makedirs(os.path.dirname(PARENT_LIB), exist_ok=True)
        shutil.copy(os.path.join(tmp, "dalm_b200", "csrc", "libdalm_b200.so"), PARENT_LIB)
    print(PARENT_LIB)


# ------------------------------------------------------------------------------------------------------------------------
# workers (one library per process)
# ------------------------------------------------------------------------------------------------------------------------
def _setup(lib):
    sys.path.insert(0, ROOT)
    from dalm_b200 import _lib
    _lib.LIB_PATH = lib
    import torch
    from dalm_b200 import ops
    return torch, ops


def _hash_cases(torch, ops):
    """(name, fn) -> fn() returns the output tensors. Random (not integer) operands: any change in summation or rounding
    order changes bits."""
    dev = torch.device("cuda:0")
    bf16, f32 = torch.bfloat16, torch.float32
    g = torch.Generator(device=dev)

    def rnd(*shape, dt=bf16, scale=1.0):
        return (torch.randn(*shape, generator=g, device=dev) * scale).to(dt)

    variants = [
        dict(out=f32), dict(out=bf16, alpha=0.5, bias=True), dict(out=f32, alpha=0.25, bias=True, resid=f32),
        dict(out=bf16, bias=True, resid=bf16), dict(out=f32, bias=True, act=1), dict(out=bf16, alpha=2.0, act=1),
        dict(out=f32, bias=True, resid=f32, drop=0.1), dict(out=bf16, bias=True, act=2), dict(out=bf16, resid=f32),
        dict(out=bf16, bias=True, drop=0.1),
    ]
    stages = {64: 8, 128: 6, 256: 4}

    def plain(layout, bn, M, N, K, var, max_ctas, seed):
        def fn():
            g.manual_seed(seed)
            ash, bsh = {0: ((M, K), (N, K)), 1: ((M, K), (K, N)), 2: ((K, M), (K, N))}[layout]
            a, b = rnd(*ash, scale=0.5), rnd(*bsh, scale=0.5)
            bias = rnd(N, dt=f32) if var.get("bias") else None
            resid = rnd(M, N, dt=var["resid"]) if var.get("resid") else (rnd(M, N, scale=2.0) if var.get("act") == 2 else None)
            drop = ops.Drop(var["drop"], seed=77 + seed, stream=5) if var.get("drop") else None
            out = ops.gemm(a, b, out_dtype=var["out"], alpha=var.get("alpha", 1.0), bias=bias, act=var.get("act", 0),
                           resid=resid, block_n=bn, max_ctas=max_ctas, drop=drop, layout=layout)
            return [out]
        return fn

    cases = []
    i = 0
    for layout in (0, 1, 2):
        for bn in (64, 128, 256) + ((2128, 2256) if layout == 0 else ()):
            tn = bn % 1000
            for var in variants:
                M = 264 if layout == 2 else (513 if bn > 1000 else 257)
                K = 64 * (stages[tn] + 1) - (3 if layout == 2 else 0)
                for max_ctas in (0, 2):
                    cases.append((f"edge L{layout} bn{bn} M{M} N{2 * tn + 8} K{K} ctas{max_ctas} {var}",
                                  plain(layout, bn, M, 2 * tn + 8, K, var, max_ctas, i)))
                    i += 1
    M = 4608
    for layout, bn, N, K, var in [(0, 0, 4096, 4096, dict(out=bf16)), (1, 0, 4096, 4096, dict(out=bf16)),
                                  (2, 0, 4096, 4096, dict(out=f32)), (0, 0, 4096, 4096, dict(out=f32, resid=f32)),
                                  (0, 0, 11008, 4096, dict(out=bf16)), (0, 2256, 4096, 4096, dict(out=bf16)),
                                  (0, 2128, 4096, 4096, dict(out=f32, resid=f32)), (0, 0, 4096, 4096, dict(out=bf16, bias=True, act=2))]:
        cases.append((f"step L{layout} bn{bn} M{M} N{N} K{K} {var}", plain(layout, bn, M, N, K, var, 0, i))); i += 1
    for N, K, var in [(1024, 1024, dict(out=f32, bias=True, resid=f32, drop=0.1)), (4096, 1024, dict(out=bf16, bias=True, act=1)),
                      (1024, 4096, dict(out=f32, bias=True, resid=f32, drop=0.1)), (3072, 1048, dict(out=bf16, bias=True))]:
        cases.append((f"bert M3204 N{N} K{K} {var}", plain(0, 0, 3204, N, K, var, 0, i))); i += 1

    def swiglu(M, N, K, seed):
        def fn():
            g.manual_seed(seed)
            return list(ops.gemm_swiglu(rnd(M, K, scale=0.5), rnd(N, K, scale=0.5)))
        return fn

    def gelu(M, N, K, seed):
        def fn():
            g.manual_seed(seed)
            return list(ops.gemm_gelu(rnd(M, K, scale=0.5), rnd(N, K, scale=0.5), bias=rnd(N, dt=f32)))
        return fn

    def rope(M, N, K, rope_cols, with_bias, seed, norm=False):
        def fn():
            g.manual_seed(seed)
            L = 256
            cos_t, sin_t = rnd(L, 64, dt=f32), rnd(L, 64, dt=f32)
            a, w = rnd(M, K, scale=0.5), rnd(N, K, scale=0.5)
            bias = rnd(N, dt=f32) if with_bias else None
            if not norm:
                return [ops.gemm_rope(a, w, cos_t, sin_t, L, rope_cols, bias=bias)]
            nh = rope_cols // 128
            pre = torch.empty(M, rope_cols, dtype=bf16, device=dev)
            rstd = torch.empty(M, nh, dtype=f32, device=dev)
            out = ops.gemm_rope(a, w, cos_t, sin_t, L, rope_cols, bias=bias, q_norm=1 + rnd(128, dt=f32, scale=0.5),
                                k_norm=1 + rnd(128, dt=f32, scale=0.5), nq_heads=nh * 3 // 4, eps=1e-6, pre_out=pre, rstd_out=rstd)
            return [out, pre, rstd]
        return fn

    for M, N, K in [(257, 512, 320), (4608, 22016, 4096)]:
        cases.append((f"swiglu M{M} N{N} K{K}", swiglu(M, N, K, i))); i += 1
    for M, N, K in [(257, 136, 512), (257, 264, 384), (257, 520, 320), (3204, 4096, 1024), (4608, 4096, 4096)]:
        cases.append((f"gelu_pair M{M} N{N} K{K}", gelu(M, N, K, i))); i += 1
    for M, N, K, rc in [(257, 520, 320, 512), (4608, 12288, 4112, 8192)]:
        for b in (False, True):
            cases.append((f"rope M{M} N{N} K{K} bias {b}", rope(M, N, K, rc, b, i))); i += 1
    norm_cases = [(f"norm_rope M{M} N{N} K{K} bias {b}", rope(M, N, K, rc, b, i + j, norm=True))
                  for j, (M, N, K, rc, b) in enumerate([(257, 520, 320, 512, True), (4608, 6144, 2048, 4096, False)])]
    return cases, norm_cases


def worker_hash(lib, dump_dir):
    torch, ops = _setup(lib)
    cases, norm_cases = _hash_cases(torch, ops)
    res = {}
    for name, fn in cases:
        outs = fn()
        torch.cuda.synchronize()
        h = hashlib.sha256()
        for o in outs:
            h.update(o.contiguous().view(torch.uint8).cpu().numpy().tobytes())
        res[name] = h.hexdigest()
    for j, (name, fn) in enumerate(norm_cases):
        torch.save([o.cpu() for o in fn()], os.path.join(dump_dir, f"norm{j}.pt"))
        res[name] = f"norm{j}.pt"
    print(json.dumps(res))


def _timeit(torch, fn, window):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record(); fn(); e.record(); torch.cuda.synchronize()
    iters = max(10, int(window / max(s.elapsed_time(e) * 1e-3, 1e-6)) + 1)
    s.record()
    for _ in range(iters): fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e-3 / iters


def worker_gemm(lib, window):
    torch, ops = _setup(lib)
    dev = torch.device("cuda:0")
    bf16, f32 = torch.bfloat16, torch.float32
    M = 4608
    # (name, M, N, K, kind): the cfg-3 generator GEMMs at their real epilogues, then bge-large's at M = 3204
    shapes = [("qkv fwd (rope)", M, 12288, 4112, "rope"), ("o_proj fwd (f32+resid)", M, 4096, 4096, "f32+resid"),
              ("gate/up fwd (swiglu)", M, 22016, 4096, "swiglu"), ("down fwd (f32+resid)", M, 4096, 11008, "f32+resid"),
              ("dgrad down", M, 11008, 4096, "bf16"), ("dgrad gate/up", M, 4096, 22016, "bf16"), ("dgrad o", M, 4096, 4096, "bf16"),
              ("dgrad qkv", M, 4096, 12304, "bf16"), ("lm_head", M, 32000, 4096, "bf16"), ("lm_head dgrad", M, 4096, 32000, "bf16"),
              ("bert qkv", 3204, 3072, 1048, "bias"), ("bert out-proj (drop+f32 resid)", 3204, 1024, 1024, "drop"),
              ("bert ffn in K1024 (gelu)", 3204, 4096, 1024, "gelu"), ("bert ffn in K4096 (gelu pair)", 3204, 4096, 4096, "gelu2"),
              ("bert ffn out K4096 (drop+f32 resid)", 3204, 1024, 4096, "drop")]
    res = {}
    for name, m, n, k, kind in shapes:
        nbuf = max(2, int(-(-4 * 50e6 // (2 * (m + n) * k))) + 1)
        As = [(torch.randn(m, k, device=dev) * 0.1).to(bf16) for _ in range(nbuf)]
        Bs = [(torch.randn(n, k, device=dev) * 0.1).to(bf16) for _ in range(nbuf)]
        bias = torch.randn(n, device=dev)
        if kind == "rope":
            out, L = torch.empty(m, n, dtype=bf16, device=dev), 256
            cs, sn = torch.randn(L, 64, device=dev), torch.randn(L, 64, device=dev)
            call = lambda a, b: ops.gemm_rope(a, b, cs, sn, L, 8192, out=out)
        elif kind in ("f32+resid", "drop"):
            out, r = torch.empty(m, n, dtype=f32, device=dev), torch.randn(m, n, device=dev)
            drop = ops.Drop(0.1, seed=3, stream=1) if kind == "drop" else None
            call = lambda a, b: ops.gemm(a, b, out=out, resid=r, bias=bias if drop else None, drop=drop)
        elif kind == "swiglu":
            gu, act = torch.empty(m, n, dtype=bf16, device=dev), torch.empty(m, n // 2, dtype=bf16, device=dev)
            call = lambda a, b: ops.gemm_swiglu(a, b, gu, act)
        elif kind == "gelu2":
            pre, act = torch.empty(m, n, dtype=bf16, device=dev), torch.empty(m, n, dtype=bf16, device=dev)
            call = lambda a, b: ops.gemm_gelu(a, b, bias=bias, pre=pre, act=act)
        else:
            out = torch.empty(m, n, dtype=bf16, device=dev)
            call = lambda a, b: ops.gemm(a, b, out=out, bias=bias if kind in ("bias", "gelu") else None, act=1 if kind == "gelu" else 0)
        i = [0]

        def fn():
            j = i[0] % nbuf; i[0] += 1
            call(As[j], Bs[j])
        res[name] = {"us": _timeit(torch, fn, window) * 1e6, "tflops": 2.0 * m * n * k}
        del As, Bs
        torch.cuda.empty_cache()
    print(json.dumps(res))


# ------------------------------------------------------------------------------------------------------------------------
# driver
# ------------------------------------------------------------------------------------------------------------------------
def _run_worker(mode, lib, *extra):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", mode, "--lib", lib, *extra],
                       capture_output=True, text=True, cwd=ROOT)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise SystemExit(f"{mode} worker failed for {lib}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def _stats(xs):
    return {"median": statistics.median(xs), "spread": max(xs) - min(xs), "n": len(xs), "all": xs}


def gpu_info():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()


def do_hash(arms):
    import torch
    with tempfile.TemporaryDirectory() as tmp:
        got = {}
        for arm, lib in arms.items():
            os.makedirs(os.path.join(tmp, arm))
            got[arm] = _run_worker("hash", lib, "--dump", os.path.join(tmp, arm))
        p, n = got["parent"], got["new"]
        same = [k for k in p if not k.startswith("norm_rope") and p[k] == n[k]]
        diff = [k for k in p if not k.startswith("norm_rope") and p[k] != n[k]]
        print(json.dumps({"hash_cases": len(same) + len(diff), "identical": len(same), "different": diff}), flush=True)
        for k in p:
            if k.startswith("norm_rope"):
                a = torch.load(os.path.join(tmp, "parent", p[k]))
                b = torch.load(os.path.join(tmp, "new", n[k]))
                row = {"case": k}
                for name, x, y in zip(("out", "pre", "rstd"), a, b):
                    d = (x.double() - y.double()).abs()
                    row[name] = {"max_abs_diff": d.max().item(), "differing": int((x != y).sum()), "of": x.numel(),
                                 "max_rel_diff": (d / y.double().abs().clamp_min(1e-30)).max().item()}
                print(json.dumps(row), flush=True)


def do_gemm(arms, rounds, window):
    times = {arm: {} for arm in arms}
    for r in range(rounds):
        for arm, lib in (arms.items() if r % 2 == 0 else reversed(list(arms.items()))):
            for name, v in _run_worker("gemm", lib, "--window", str(window)).items():
                times[arm].setdefault(name, []).append(v["us"])
                flops = v["tflops"]
                times[arm].setdefault("_flop", {})[name] = flops
    for name in times["parent"]:
        if name == "_flop":
            continue
        row = {"gemm": name}
        for arm in arms:
            row[arm] = {k: round(v, 2) if isinstance(v, float) else v for k, v in _stats(times[arm][name]).items() if k != "all"}
            row[arm]["tflops"] = round(times[arm]["_flop"][name] / (row[arm]["median"] * 1e-6) / 1e12, 1)
        row["speedup"] = round(row["parent"]["median"] / row["new"]["median"], 4)
        print(json.dumps(row), flush=True)


def do_bench(arms, rounds, configs):
    keep = TREE_LIB + ".ab_keep"
    shutil.copy(TREE_LIB, keep)
    res = {}
    try:
        plan = [(cfg, r) for cfg in configs for r in range(rounds if cfg == "cfg-3" else 1)]
        for cfg, r in plan:
            for arm, lib in (arms.items() if r % 2 == 0 else reversed(list(arms.items()))):
                shutil.copy(keep if arm == "new" else lib, TREE_LIB)
                cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", "10", "--warmup", "3", "--config", cfg,
                       "--cpu-baseline", "0", "--gpu-eager-baseline", "0"]
                out = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
                line = [l for l in out.stdout.splitlines() if l.startswith("{")]
                if out.returncode != 0 or not line:
                    sys.stderr.write(out.stdout[-3000:] + out.stderr[-3000:])
                    raise SystemExit(f"bench.py failed for {arm} {cfg}")
                j = json.loads(line[-1])
                print(json.dumps({"arm": arm, "config": cfg, "result": j}), flush=True)
                res.setdefault((cfg, arm), []).append(j)
    finally:
        shutil.move(keep, TREE_LIB)
    for (cfg, arm), js in res.items():
        sps = [j.get("samples_per_s", j.get("value")) for j in js]
        print(json.dumps({"config": cfg, "arm": arm, "samples_per_s": _stats(sps)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("mode", nargs="?", choices=["hash", "gemm", "bench"])
    ap.add_argument("--build-parent", metavar="REV")
    ap.add_argument("--parent-lib", default=PARENT_LIB)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window", type=float, default=0.4, help="seconds of timed launches per GEMM per round")
    ap.add_argument("--configs", default="cfg-3,cfg-2", help="bench: cfg-3 runs --rounds times per arm, the others once")
    ap.add_argument("--worker", choices=["hash", "gemm"])
    ap.add_argument("--lib")
    ap.add_argument("--dump")
    args = ap.parse_args()
    if args.build_parent:
        return build_parent(args.build_parent)
    if args.worker == "hash":
        return worker_hash(args.lib, args.dump)
    if args.worker == "gemm":
        return worker_gemm(args.lib, args.window)
    arms = {"parent": os.path.abspath(args.parent_lib), "new": TREE_LIB}
    for lib in arms.values():
        if not os.path.exists(lib):
            raise SystemExit(f"{lib} is missing (--build-parent REV / python -m dalm_b200.csrc.build)")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    {"hash": lambda: do_hash(arms), "gemm": lambda: do_gemm(arms, args.rounds, args.window),
     "bench": lambda: do_bench(arms, args.rounds, args.configs.split(","))}[args.mode]()


if __name__ == "__main__":
    main()
