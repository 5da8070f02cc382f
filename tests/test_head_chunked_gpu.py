"""-m gpu: the chunked lm_head + CE head (dalm_b200/engine/head.py) against the materialised-logits path it replaces and
against the fp64 closed form of reference train_utils.py:113-138 (oracle/losses.py)."""
import pytest
import torch

from model_helpers import llama_rag_models, r16_2d, rag_batch, rel

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32


def _case(B, L, V, seed, left_pad=True):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, V, (B, L), generator=g)
    mask = torch.ones(B, L, dtype=torch.int64)
    if left_pad:
        mask[0, :3] = 0
    mask[-1, L - 4:] = 0
    return ids, mask


@pytest.mark.parametrize("V,ld", [(1000, 1000), (997, 1000), (32000, 32000)])
def test_ce_rows_chunks_equal_the_whole_pass(cuda_dev, V, ld):
    """ce_marginal_rows over ragged row ranges == one ce_marginal launch, bit for bit (same kernel, other row origin)"""
    from dalm_b200 import ops
    dev = cuda_dev
    B, L = 3, 21
    ids, mask = _case(B, L, V, 5)
    g = torch.Generator().manual_seed(6)
    full = torch.zeros(B, L, ld)
    full[:, :, :V] = torch.randn(B, L, V, generator=g) * 3
    lg = full.to(dev, bf16)
    idd, md = ids.to(dev), mask.to(dev)
    qlen = torch.full((B,), 4, dtype=torch.int64, device=dev)
    _, nsum = ops.marginal_counts(md, qlen)
    ref_lp, ref_dl = ops.ce_marginal(lg[:, :, :V], idd, md, nsum, need_grad=True, inplace=False, grad_out=0.5)
    tok_lp = torch.full((B, L), 7.0, dtype=f32, device=dev)
    flat = lg.reshape(B * L, ld).clone()
    for r0, n in ((0, 10), (10, 1), (11, 31), (42, B * L - 42)):
        chunk = flat[r0:r0 + n].clone()                       # a scratch that holds just this chunk
        ops.ce_marginal_rows_(chunk, idd, md, nsum, tok_lp, r0, V, need_grad=True, grad_out=0.5)
        flat[r0:r0 + n] = chunk
    assert torch.equal(tok_lp, ref_lp)
    assert torch.equal(flat.view(B, L, ld)[:, :, :V], ref_dl[:, :, :V])
    assert float(flat.view(B, L, ld)[:, :, V:].abs().sum()) == 0.0    # pad columns stay zero for the head's dgrad
    fwd_only = torch.empty(B, L, dtype=f32, device=dev)
    c = lg.reshape(B * L, ld)[5:30].clone()
    c0 = c.clone()
    ops.ce_marginal_rows_(c, idd, md, nsum, fwd_only, 5, V, need_grad=False)
    assert torch.equal(fwd_only.view(-1)[5:30], ref_lp.view(-1)[5:30]) and torch.equal(c, c0)     # forward only: logits untouched


def test_ce_rows_rejects_rows_outside_the_batch(cuda_dev):
    from dalm_b200 import _lib, ops
    dev = cuda_dev
    ids, mask = _case(2, 8, 64, 1)
    nsum = torch.ones(1, device=dev)
    tok = torch.empty(2, 8, device=dev)
    with pytest.raises(_lib.DalmB200Error):
        ops.ce_marginal_rows_(torch.zeros(9, 64, dtype=bf16, device=dev), ids.to(dev), mask.to(dev), nsum, tok, 8, 64)


@pytest.mark.parametrize("M_rows,V,H,budget_rows", [((3, 100), 1000, 256, 128), ((2, 256), 32000, 512, 256), ((5, 77), 520, 128, 128)])
def test_chunked_head_matches_materialised_logits(cuda_dev, M_rows, V, H, budget_rows):
    """tok_lp, d(hf) and the head's weight gradient: chunked sweep vs [B,L,V] logits -> ce_marginal -> dgrad / wgrad, plus the
    fp64 closed form on the same bf16 operands"""
    from dalm_b200 import ops
    from dalm_b200.engine.head import chunked_head_loss
    dev = cuda_dev
    B, L = M_rows
    M = B * L
    Vp = (V + 7) // 8 * 8
    g = torch.Generator().manual_seed(17)
    hf = (torch.randn(M, H, generator=g) * 0.7).to(bf16)
    W = torch.zeros(Vp, H)
    W[:V] = torch.randn(V, H, generator=g) * 0.08
    W = W.to(bf16)
    ids, mask = _case(B, L, V, 3)
    hfd, Wd, idd, md = hf.to(dev), W.to(dev), ids.to(dev), mask.to(dev)
    WT = Wd.t().contiguous()
    _, nsum = ops.marginal_counts(md, torch.full((B,), 2, dtype=torch.int64, device=dev))
    # materialised path
    logits = ops.gemm(hfd, Wd).view(B, L, Vp)[:, :, :V]
    ref_lp, dl = ops.ce_marginal(logits, idd, md, nsum, need_grad=True, inplace=True, grad_out=1.0)
    dl2 = torch.as_strided(dl, (M, Vp), (Vp, 1), dl.storage_offset())
    ref_dhf = ops.gemm(dl2, WT)
    ref_dW = torch.zeros(Vp, H, dtype=f32, device=dev)
    ops.wgrad_(dl2, hfd, ref_dW, False)
    budget = budget_rows * Vp * 2
    # frozen head (resident transpose) and trainable head (MN-major dgrad + chunk-accumulated wgrad)
    lp1, dhf1 = chunked_head_loss(hfd, Wd, WT, V, idd, md, nsum, True, 1.0, None, budget)
    dW = torch.full((Vp, H), 3.0, dtype=f32, device=dev)                        # stale values: the first chunk must overwrite
    lp2, dhf2 = chunked_head_loss(hfd, Wd, None, V, idd, md, nsum, True, 1.0,
                                  lambda d, x, first: ops.wgrad_(d, x, dW, not first), budget)
    lp3, none = chunked_head_loss(hfd, Wd, WT, V, idd, md, nsum, False, 1.0, None, budget)
    assert none is None
    for lp in (lp1, lp2, lp3):
        assert (lp - ref_lp).abs().max().item() < 1e-5
    assert rel(dhf1, ref_dhf) < 2e-3 and rel(dhf2, ref_dhf) < 2e-3
    assert rel(dW, ref_dW) < 2e-3
    # fp64 closed form: lp[b,t] = log_softmax(hf W^T)[ids[b,t+1]], d hf = sum_v dlogits W
    x, w = hf.double(), W[:V].double()
    lg = (x @ w.t()).view(B, L, V)
    lsm = torch.log_softmax(lg, -1)
    want = torch.zeros(B, L, dtype=torch.float64)
    want[:, :-1] = lsm[:, :-1].gather(-1, ids[:, 1:].unsqueeze(-1)).squeeze(-1) * mask[:, 1:]
    got = lp1.double().cpu().clone()
    got[:, :-1] *= mask[:, 1:]
    assert (got - want).abs().max().item() < 3e-2               # bf16 logits: |x| <~ 10 -> half-ulp 0.03
    N = mask[:, 1:].sum().item()
    coef = torch.zeros(B, L, 1, dtype=torch.float64)
    coef[:, :-1, 0] = mask[:, 1:] / N
    onehot = torch.zeros(B, L, V, dtype=torch.float64)
    onehot[:, :-1].scatter_(-1, ids[:, 1:].unsqueeze(-1), 1.0)
    dlg = coef * (lsm.exp() - onehot)
    assert rel(dhf1, (dlg.view(M, V) @ w)) < 3e-2
    assert rel(dW[:V], dlg.view(M, V).t() @ x) < 3e-2


def test_fused_step_chunked_head_equals_materialised(cuda_dev):
    """the whole fused RAG step with the chunked head == the same step through [B,L,V] logits (PEFT and full fine-tuning)"""
    from dalm_b200.engine import head
    from dalm_b200.training.utils import train_utils as tu
    model, enc, dec, _, _ = llama_rag_models(cuda_dev, 500, r16_2d)
    batch = rag_batch(5, 12, 24, 40, 600, 500, seed=23)
    old_budget, old_flag = head.L2_BUDGET, tu._CHUNKED_HEAD
    try:
        res = {}
        for chunked in (False, True):
            tu._CHUNKED_HEAD = chunked
            head.L2_BUDGET = 128 * 504 * 2                      # 128-row chunks: 200 rows -> two chunks, the second ragged
            enc.lora.zero_grad(); dec.lora.zero_grad()
            out = tu.fused_rag_step(model, batch, 100.0)
            res[chunked] = (out["losses"].clone(), enc.lora.grad.clone(), dec.lora.grad.clone())
        assert (res[True][0] - res[False][0]).abs().max().item() < 1e-5
        assert rel(res[True][1], res[False][1]) < 1e-4 and rel(res[True][2], res[False][2]) < 2e-3
    finally:
        head.L2_BUDGET, tu._CHUNKED_HEAD = old_budget, old_flag
