"""-m gpu: sampling (`sample_step` and `generate(do_sample=True)`) against oracle/sampling.py, which tests/test_sampling_host.py
pins to the installed transformers' warpers.

Kernel level: the warped scores (test hook scores_out) against HF's warper stack and the oracle on bf16 logits up to
V = 128256; the inverse-CDF choice with injected uniforms; the bookkeeping against greedy_step; the Philox draws against the
oracle distribution (chi-square with a fixed seed, so the test is deterministic). Model level: reproducibility under
torch.manual_seed, CUDA-graph replay == eager launches, greedy's output layout and stop rule, and the first sampled token's
distribution against the oracle applied to the engine's own prefill logits. Then `dalm eval-rag` on a generator whose
generation_config asks for sampling, as Llama-2-7b-hf's does.
"""
import numpy as np
import pytest
import torch

from oracle import sampling as osmp

pytestmark = pytest.mark.gpu
bf16, f32, i64 = torch.bfloat16, torch.float32, torch.int64
LLAMA2_7B_GEN = {"bos_token_id": 1, "do_sample": True, "eos_token_id": 2, "max_length": 4096, "pad_token_id": 0,
                 "temperature": 0.6, "top_p": 0.9, "transformers_version": "4.31.0.dev0"}


def _state(B, T, dev):
    return dict(unfinished=torch.ones(B, dtype=torch.int32, device=dev), tokens=torch.full((B, T), -1, dtype=i64, device=dev),
                mask=torch.zeros(B, T, dtype=i64, device=dev), next_ids=torch.zeros(B, dtype=i64, device=dev),
                pos=torch.zeros(B, dtype=i64, device=dev), alive=torch.zeros(T, dtype=torch.int32, device=dev))


def _sample(logits, V, col=0, T=2, state=None, eos=None, pad=0, **kw):
    from dalm_b200 import ops
    st = state or _state(logits.shape[0], T, logits.device)
    ops.sample_step_(logits, V, eos, pad, st["unfinished"], st["tokens"], st["mask"], col, st["next_ids"], st["pos"],
                     st["alive"], **kw)
    return st


def _bf16_rows(V, T, top_k, top_p, seed, n=3):
    g = torch.Generator().manual_seed(seed)
    scale = 2.0 if V <= 1000 else 6.0
    rows = []
    for _ in range(n):
        for _ in range(500):
            row = (torch.randn(V, generator=g) * scale).to(bf16)
            if osmp.clear_of_cut(row.float()[None], T, top_k, top_p, ties_ok=True):
                rows.append(row)
                break
        else:
            raise AssertionError("no row clear of the top-p cut")
    return torch.stack(rows)


@pytest.mark.parametrize("V", [7, 1000, 32000, 128256])
@pytest.mark.parametrize("top_p", [1.0, 0.9, 0.5, 1e-6])
def test_filter_parity(cuda_dev, V, top_p):
    """removed sets identical to the oracle's and kept scores bit-identical; against HF the same, except which tokens of a
    tie group straddling the top-p cut go (HF's unstable sort decides; the count is the same)"""
    for T in (0.6, 1.0, 1.7):
        for k in (0, 1, 50, V + 5):
            rows = _bf16_rows(V, T, k, top_p, seed=V + int(T * 10) + 7 * k)
            pad = 8
            logits = torch.full((rows.shape[0], V + pad), 100.0, dtype=bf16)
            logits[:, :V] = rows                                                 # padded vocabulary columns must never count
            logits = logits.to(cuda_dev)
            scores = torch.full((rows.shape[0], V + pad), 7.0, dtype=f32, device=cuda_dev)
            _sample(logits, V, temperature=T, top_k=k, top_p=top_p, seed=1, scores_out=scores)
            got = scores[:, :V].cpu()
            assert (scores[:, V:] == 7.0).all()
            ora = torch.from_numpy(osmp.warp(rows.float(), T, k, top_p)).float()
            assert torch.equal(torch.isinf(got), torch.isinf(ora)), (T, k)
            fin = torch.isfinite(ora)
            assert torch.equal(got[fin].view(torch.int32), ora[fin].view(torch.int32)), (T, k)
            hf = osmp.hf_warp(rows.float(), T, k, top_p)
            for r in range(rows.shape[0]):
                differ = torch.isinf(got[r]) != torch.isinf(hf[r])
                if differ.any():
                    tie = osmp.straddling_value(rows[r].float(), T, k, top_p)
                    x = torch.from_numpy(osmp.warp(rows[r].float(), T, k, 1.0)).float()
                    assert tie is not None and (x[differ] == tie).all(), (T, k, r)
                    assert torch.isfinite(got[r]).sum() == torch.isfinite(hf[r]).sum()
                both = torch.isfinite(got[r]) & torch.isfinite(hf[r])
                assert torch.equal(got[r][both].view(torch.int32), hf[r][both].view(torch.int32))


def test_tie_group_straddling_the_cut(cuda_dev):
    """a tie group split by the top-p cut loses its lowest indices first: the (x, index) rule"""
    found = 0
    for seed in range(200):
        rows = _bf16_rows(1000, 1.0, 0, 0.9, seed=1000 + seed, n=1)
        if osmp.straddling_value(rows[0].float(), 1.0, 0, 0.9) is None:
            continue
        scores = torch.empty(1, 1000, dtype=f32, device=cuda_dev)
        _sample(rows.to(cuda_dev), 1000, top_p=0.9, scores_out=scores)
        ora = torch.from_numpy(osmp.warp(rows.float(), 1.0, 0, 0.9)).float()
        assert torch.equal(torch.isinf(scores.cpu()), torch.isinf(ora))
        found += 1
        if found == 5:
            break
    assert found == 5


def test_inverse_cdf_choice(cuda_dev):
    g = torch.Generator().manual_seed(3)
    V, T, k, p = 1000, 0.7, 50, 0.9
    row = _bf16_rows(V, T, k, p, seed=11, n=1)[0]
    w = osmp.warp(row.float(), T, k, p)
    c, Z = osmp.prefix_mass(w)
    kept = np.nonzero(np.isfinite(w))[0]
    us = [0.0, 1 - 2 ** -24] + torch.rand(20, generator=g).double().tolist()
    for j in kept[:-1][:: max(1, len(kept) // 8)]:
        us += [c[j] / Z - 2e-6, c[j] / Z + 2e-6]                                  # each side of a boundary, 2e-6 * Z away
    us = [u for u in us if 0.0 <= u < 1.0]
    B = len(us)
    logits = row[None].expand(B, V).contiguous().to(cuda_dev)
    u = torch.tensor(us, dtype=torch.float64, device=cuda_dev)
    st = _sample(logits, V, temperature=T, top_k=k, top_p=p, seed=5, u=u)
    want = [osmp.choose(w, x) for x in us]
    assert st["tokens"][:, 0].tolist() == want
    # 10^5 Philox draws never pick a removed token
    many = row[None].expand(100_000, V).contiguous().to(cuda_dev)
    st = _sample(many, V, temperature=T, top_k=k, top_p=p, seed=9)
    drawn = torch.unique(st["tokens"][:, 0]).cpu().numpy()
    assert np.isin(drawn, kept).all() and len(drawn) > 1


@pytest.mark.parametrize("device_col", [False, True])
def test_bookkeeping_matches_greedy_step(cuda_dev, device_col):
    """top_k = 1 on logits without a tied maximum: sample_step writes exactly what greedy_step writes, in host-column and
    device-column mode, with finished rows, EOS, padded vocabulary columns and replays past the end"""
    from dalm_b200 import ops
    g = torch.Generator().manual_seed(0)
    B, V, Vp, T = 6, 1000, 1008, 4
    logits = torch.randn(B, Vp, generator=g).to(bf16).to(cuda_dev)
    logits[:, V:] = 100.0
    logits[0, 77] = 70.0; logits[1, 999] = 60.0; logits[2, 5] = 60.0; logits[4, 0] = 60.0; logits[5, 333] = 60.0
    eos = torch.tensor([5, 9], device=cuda_dev)
    mk = lambda: dict(_state(B, T, cuda_dev), unfinished=torch.tensor([1, 1, 1, 0, 1, 1], dtype=torch.int32, device=cuda_dev),
                      pos=torch.arange(B, dtype=i64, device=cuda_dev) * 3)
    a, b = mk(), mk()
    ca = torch.zeros(B, dtype=torch.int32, device=cuda_dev) if device_col else None
    cb = ca.clone() if device_col else None
    for step in range(T + 1 if device_col else T - 1):
        col_a = ca if device_col else step + 1
        col_b = cb if device_col else step + 1
        ops.greedy_step_(logits, V, eos, 77, a["unfinished"], a["tokens"], a["mask"], col_a, a["next_ids"], a["pos"], a["alive"])
        ops.sample_step_(logits, V, eos, 77, b["unfinished"], b["tokens"], b["mask"], col_b, b["next_ids"], b["pos"], b["alive"],
                         temperature=0.9, top_k=1, top_p=0.8, seed=step)
        for key in a:
            assert torch.equal(a[key], b[key]), (step, key)
        if device_col:
            assert torch.equal(ca, cb)
    assert a["unfinished"].tolist() == [1, 1, 0, 0, 1, 1] and (a["tokens"][3, 1:] == 77).all()


def test_draw_statistics(cuda_dev):
    from scipy.stats import chisquare
    g = torch.Generator().manual_seed(4)
    V, T, k, p, N = 64, 0.8, 20, 0.9, 8192
    row = (torch.randn(V, generator=g) * 1.5).to(bf16)
    logits = row[None].expand(N, V).contiguous().to(cuda_dev)
    toks = lambda seed, col=0: _sample(logits, V, col=col, temperature=T, top_k=k, top_p=p, seed=seed)["tokens"][:, col].cpu()
    a = toks(12345)
    prob = osmp.probs(osmp.warp(row.float(), T, k, p))
    kept = prob > 0
    counts = np.bincount(a.numpy(), minlength=V)
    assert counts[~kept].sum() == 0
    exp = prob[kept] * N
    obs = counts[kept]
    big = exp >= 5                                                               # pool the rare tokens into one cell
    f_obs = np.append(obs[big], obs[~big].sum())
    f_exp = np.append(exp[big], exp[~big].sum())
    if f_exp[-1] == 0:
        f_obs, f_exp = f_obs[:-1], f_exp[:-1]
    assert chisquare(f_obs, f_exp).pvalue > 1e-6
    assert torch.equal(toks(12345), a)                                           # same seed, same column: same tokens
    assert not torch.equal(toks(54321), a)                                       # another seed: other tokens
    assert not torch.equal(toks(12345, col=1), a)                                # another column: other draws


# ----------------------------------------------------------------------------------------------------------------
# whole decoders
# ----------------------------------------------------------------------------------------------------------------
def _decoder(kind, dev):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    V = 512
    if kind == "llama":
        from dalm_b200.engine.llama import LlamaDecoder
        cfg = synthetic.llama_config("llama-tiny", vocab_size=V)
        sd = params.random_state_dict("llama", cfg, seed=2)
        return LlamaDecoder(cfg, {k: (v.to(bf16).float() if v.dim() == 2 else v) for k, v in sd.items()}, device=dev), V
    from dalm_b200.engine.falcon import FalconDecoder
    cfg = synthetic.falcon_config("falcon-mini", vocab_size=V)
    sd = params.random_state_dict("falcon", cfg, seed=3)
    return FalconDecoder(cfg, {k: (v.to(bf16).float() if v.dim() == 2 else v) for k, v in sd.items()}, device=dev), V


def _prompt(B, L0, V, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, V, (B, L0), generator=g)
    mask = torch.ones(B, L0, dtype=i64)
    mask[1, :3] = 0
    mask[2, L0 - 3:] = 0
    return ids, mask


@pytest.mark.parametrize("kind", ["llama", "falcon"])
def test_generate_sampling(cuda_dev, monkeypatch, kind):
    from dalm_b200.engine import decoding
    dec, V = _decoder(kind, cuda_dev)
    ids, mask = _prompt(4, 12, V, seed=1)
    L0, T = 12, 34
    kw = dict(do_sample=True, temperature=0.7, top_k=20, top_p=0.9, max_length=T, early_stopping=True)

    def gen(seed, graph, **extra):
        monkeypatch.setenv("DALM_B200_DECODE_GRAPH", graph)
        torch.manual_seed(seed)
        return dec.generate(input_ids=ids.to(cuda_dev), attention_mask=mask.to(cuda_dev), **dict(kw, **extra)).cpu()

    free = gen(7, "0", eos_token_id=[], pad_token_id=0)
    assert free.shape == (4, T) and torch.equal(free[:, :L0], ids)
    assert torch.equal(gen(7, "0", eos_token_id=[], pad_token_id=0), free)          # reproducible under manual_seed
    assert not torch.equal(gen(8, "0", eos_token_id=[], pad_token_id=0), free)
    replayed = gen(7, "1", eos_token_id=[], pad_token_id=0)
    assert decoding.LAST_RUN["graph_replays"] >= 4 and torch.equal(replayed, free)   # graph replay == eager launches
    # EOS ids from the free run: the same draws up to each row's EOS, pad after it, stop right after the last row's EOS
    eos = sorted({int(free[0, 14]), int(free[1, 20]), int(free[2, 17]), int(free[3, 23])})
    for graph in ("0", "1"):
        out = gen(7, graph, eos_token_id=eos, pad_token_id=eos[0])
        ends = []
        for r in range(4):
            hit = [c for c in range(L0, T) if int(free[r, c]) in eos]
            end = hit[0] if hit else T - 1
            ends.append(end)
            assert torch.equal(out[r, :end + 1], free[r, :end + 1])
            assert (out[r, end + 1:] == eos[0]).all()
        assert out.shape[1] == min(T, max(ends) + 1)


@pytest.mark.parametrize("kind", ["llama", "falcon"])
def test_first_token_distribution(cuda_dev, monkeypatch, kind):
    """4096 copies of one prompt, one new token each: the counts fit the oracle distribution of the engine's own prefill
    logits (summed over the rows, in case rows round differently)"""
    from scipy.stats import chisquare

    from dalm_b200 import ops
    dec, V = _decoder(kind, cuda_dev)
    ids = torch.randint(3, V, (1, 10), generator=torch.Generator().manual_seed(5))
    mask = torch.ones_like(ids)
    N, T, k, p = 4096, 0.7, 20, 0.9
    rec = []
    real = ops.sample_step_

    def recording(logits, V_, *a, **kw):
        rec.append(logits[:, :V_].float().cpu())
        return real(logits, V_, *a, **kw)

    monkeypatch.setattr(ops, "sample_step_", recording)
    torch.manual_seed(0)
    out = dec.generate(input_ids=ids.expand(N, -1).to(cuda_dev), attention_mask=mask.expand(N, -1).to(cuda_dev), max_new_tokens=1,
                       do_sample=True, temperature=T, top_k=k, top_p=p, eos_token_id=[], pad_token_id=0).cpu()
    assert out.shape == (N, 11) and len(rec) == 1
    first = out[:, 10].numpy()
    uniq, inv = torch.unique(rec[0], dim=0, return_inverse=True)
    prob = np.zeros(V)
    for i in range(uniq.shape[0]):
        prob += osmp.probs(osmp.warp(uniq[i].to(bf16).float(), T, k, p)) * int((inv == i).sum())
    counts = np.bincount(first, minlength=V)
    assert counts[prob == 0].sum() == 0
    kept = prob > 0
    big = prob[kept] >= 5
    f_obs = np.append(counts[kept][big], counts[kept][~big].sum())
    f_exp = np.append(prob[kept][big], prob[kept][~big].sum())
    if f_exp[-1] == 0:
        f_obs, f_exp = f_obs[:-1], f_exp[:-1]
    assert chisquare(f_obs, f_exp).pvalue > 1e-6


def test_evaluate_rag_samples_with_llama2_generation_config(cuda_dev, tmp_path, capsys, caplog):
    import csv as _csv
    import json
    import logging
    import os

    from dalm_b200 import synthetic
    from dalm_b200.eval.eval_rag import evaluate_rag
    words = synthetic.word_list()
    path = str(tmp_path / "short.csv")
    with open(path, "w", newline="") as f:
        w = _csv.DictWriter(f, fieldnames=["Abstract", "Question", "Answer"])
        w.writeheader()
        for i in range(6):
            w.writerow({"Abstract": " ".join(words[20 + 6 * i:26 + 6 * i]), "Question": " ".join(words[200 + 4 * i:204 + 4 * i]),
                        "Answer": " ".join(words[400 + i:402 + i])})
    rdir = synthetic.write_model_dir(str(tmp_path / "bge-tiny"), "bert", "bge-tiny", vocab_size=1200)
    gdir = synthetic.write_model_dir(str(tmp_path / "llama-tiny"), "llama", "llama-tiny", vocab_size=1200)
    with open(os.path.join(gdir, "generation_config.json"), "w") as f:
        json.dump(LLAMA2_7B_GEN, f)
    caplog.set_level(logging.INFO, logger="dalm_b200.eval.eval_rag")
    torch.manual_seed(0)
    res = evaluate_rag(path, rdir, gdir, None, None, "Abstract", "Question", "Answer", embed_dim=64, max_length=96,
                       test_batch_size=4, query_batch_size=4, top_k=3, evaluate_generator=True)
    out = capsys.readouterr().out
    assert res.total_examples == 6 and "Exact match:" in out
    assert "sampling (temperature 0.6, top-k 50, top-p 0.9)" in caplog.text
