"""-m gpu: ModernBERT retrievers — the bidirectional sliding window in the training attention kernels and the GeGLU row kernels
against fp64, and the encoder against transformers' ModernBertModel (eager attention, fp32, the same bf16-rounded weights).

Kernels: query i sees key j iff |i - j| < window (ModernBERT's local layers pass local_attention // 2 + 1), combined with the
key-padding mask. Rows are checked against fp64 with the bounds of test_mistral_gpu on poisoned inputs and guarded outputs; a
query that sees no key (a padded query far from every valid key) gives output 0, lse +inf and no gradient anywhere.

Models: padded query rows of local layers can see no key; transformers then gives finite values that differ between its own
attention paths. Those rows are never pooled, so only valid rows are compared, and every row must be finite. The q / k blocks of
Wqkv are drawn 8x wider than initializer_range, and the v block and Wo 4x, so that attention is peaked and its output weighs in
the residual stream: the same encoder with full attention and the global theta on every layer then misses by more than 10x the
tolerance (the control; at initializer_range it misses by less than the tolerance).
"""
import math

import pytest
import torch

from exact_helpers import Guarded, _attn_bwd64, _attn_fns, _attn_ref64, _expect_close, _poisoned, _row_mask, dev, ops  # noqa: F401
from model_helpers import attach_lora, draw_lora_B, lora_grad_error, r16, rel

pytestmark = pytest.mark.gpu
bf16, f32, f64, i64 = torch.bfloat16, torch.float32, torch.float64, torch.int64
PAD = 50283
QK_SCALE, V_SCALE = 8.0, 4.0
TOL = 1.5e-2                    # relative error of the last hidden state on valid rows (bf16 GEMM operands, fp32 residual)


# ----------------------------------------------------------------------------------------------------------------
# 1. attention kernels against fp64
# ----------------------------------------------------------------------------------------------------------------
KINDS = [("wg", 64), ("wg", 128), ("mma", 32), ("mma", 64), ("mma", 128)]
LENGTHS = (65, 200, 257, 1000)
PATTERNS = ("right64", "left64", "holes", "empty")


def _visible_bidir(mask, L, window):
    """[B, 1, Lq, Lk] visibility: key-padding mask and, when window > 0, |i - j| < window"""
    i = torch.arange(L, device=mask.device)
    band = torch.ones(L, L, dtype=torch.bool, device=mask.device)
    if window > 0:
        band = (i[None, :] - i[:, None]).abs() < window
    return mask.bool()[:, None, None, :] & band


def _params():
    out, n = [], 0
    for kind, D in KINDS:
        for L in LENGTHS:
            for w in (1, 17, 65, L):
                out.append((kind, D, L, w, PATTERNS[n % 4]))
                n += 1
    return out


def _run(ops, dev, kind, D, B, L, H, mask, window, seed):
    g = torch.Generator().manual_seed(seed)
    q, k, v, d_out = (_poisoned(torch.randn(B * L, H * D, generator=g).to(bf16).to(dev)) for _ in range(4))
    fwd, bwd = _attn_fns(ops, kind)
    out = Guarded(B * L, H * D, bf16, dev)
    _, lse = fwd(q, k, v, mask, B, L, H, H, D, False, out=out.view, window=window, bidirectional=True)
    dq, dk, dv = (Guarded(B * L, H * D, bf16, dev) for _ in range(3))
    bwd(q, k, v, mask, out.view, lse, d_out, B, L, H, H, D, False, dq=dq.view, dk=dk.view, dv=dv.view, window=window,
        bidirectional=True)
    return (q, k, v, d_out), out, lse, dq, dk, dv


@pytest.mark.parametrize("kind,D,L,window,pattern", _params())
def test_bidirectional_window_rows_vs_fp64(ops, dev, kind, D, L, window, pattern):
    """forward, dQ, dK and dV with a bidirectional window, every row against fp64: windows of one key, shorter than a tile,
    across tile edges and the whole row; right and left padding (>= 64 pad tokens: padded queries whose window holds no valid
    key), interior holes and a sample with every key masked"""
    B, H = 3, 2
    mask = _row_mask(B, L, pattern, torch.Generator().manual_seed(L * 131 + D + window)).to(dev)
    sc = 1.0 / math.sqrt(D)
    (q, k, v, d_out), out, lse, dq, dk, dv = _run(ops, dev, kind, D, B, L, H, mask, window, seed=L + 7 * window + D)
    what = f"{kind} attention D {D} L {L} bidirectional window {window} {pattern}"
    vis = _visible_bidir(mask, L, window)
    qd, kd, vd = (t.double() for t in (q, k, v))
    ref, lse_ref = _attn_ref64(qd, kd, vd, vis, B, L, H, H, D, sc)
    for name, t in (("out", out.view), ("dq", dq.view), ("dk", dk.view), ("dv", dv.view)):
        assert torch.isfinite(t).all(), f"{what}: non-finite {name}"
    valid = vis.expand(B, H, L, L).any(-1)                                       # [B, H, L]: the query sees some key
    no_query = (~valid).permute(0, 2, 1).reshape(B * L, H)
    assert (out.view.view(B * L, H, D)[no_query] == 0).all(), f"{what}: rows without a visible key need output 0"
    assert (torch.isinf(lse[~valid]) & (lse[~valid] > 0)).all(), f"{what}: rows without a visible key need lse = +inf"
    vmax = v.double().abs().view(B, L, H, D).amax((1, 3))
    tol = (vmax[:, None, :, None] / 128).expand(B, L, H, D).reshape(B * L, H * D)
    _expect_close(out.view, ref, tol, what + " out", 64)
    lerr = (lse.double() - lse_ref).abs()[valid]
    assert lerr.max() < 1e-4, f"{what}: lse off by {lerr.max().item():.3e}"
    want = _attn_bwd64(qd, kd, vd, d_out.double(), out.view.double(), vis, B, L, H, H, D, sc)
    masked_key = (mask == 0).reshape(B * L, 1).expand(B * L, H)                 # key j is always visible to query j
    floor = None
    for name, got, w, zero in (("dv", dv.view, want[2], masked_key), ("dq", dq.view, want[0], no_query),
                               ("dk", dk.view, want[1], masked_key)):
        gr, wr = got.double().view(B * L, H, D), w.view(B * L, H, D)
        err, nrm = (gr - wr).norm(dim=-1), wr.norm(dim=-1)
        med = nrm[~zero].median()
        if floor is None:
            floor = 1e-4 * med
        bad = err > 0.04 * nrm + 0.01 * med + floor
        if bad.any():
            r, h = bad.nonzero()[0].tolist()
            pytest.fail(f"{what}: {name} {int(bad.sum())} bad rows; first token {r} (sample {r // L}, position {r % L}) head {h}: "
                        f"error {err[r, h].item():.3e} vs row norm {nrm[r, h].item():.3e}")
        assert (gr[zero] == 0).all(), f"{what}: {name} nonzero where every contribution is masked"
    for name, gd in (("out", out), ("dq", dq), ("dk", dk), ("dv", dv)):
        gd.check(f"{what} {name}")


@pytest.mark.parametrize("kind,D", KINDS)
@pytest.mark.parametrize("L", [65, 200, 257])
def test_wide_window_is_bit_identical_to_none(ops, dev, kind, D, L):
    """a bidirectional window >= L masks nothing and skips no tile: out, lse, dq, dk, dv bit-equal to window = 0"""
    mask = _row_mask(3, L, "holes", torch.Generator().manual_seed(L)).to(dev)
    base = _run(ops, dev, kind, D, 3, L, 2, mask, 0, seed=L)
    for w in (L, L + 5, 1 << 30):
        got = _run(ops, dev, kind, D, 3, L, 2, mask, w, seed=L)
        for i, name in ((1, "out"), (2, "lse"), (3, "dq"), (4, "dk"), (5, "dv")):
            a, b = (got[i], base[i]) if i == 2 else (got[i].view, base[i].view)
            assert torch.equal(a, b), f"{kind} D {D} L {L} window {w}: {name} differs from window 0"


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("L,window", [(200, 65), (257, 17), (1000, 65), (130, 64)])
def test_bidirectional_wg_agrees_with_mma(ops, dev, D, L, window):
    mask = _row_mask(3, L, "right64", torch.Generator().manual_seed(3)).to(dev)
    a = _run(ops, dev, "wg", D, 3, L, 2, mask, window, seed=5)
    b = _run(ops, dev, "mma", D, 3, L, 2, mask, window, seed=5)
    assert rel(a[1].view.float(), b[1].view.float()) < 1e-2
    fin = torch.isfinite(b[2])
    assert torch.equal(fin, torch.isfinite(a[2])) and (a[2][fin] - b[2][fin]).abs().max() < 1e-4
    for i in (3, 4, 5):
        assert rel(a[i].view.float(), b[i].view.float()) < 2e-2


def test_bidirectional_window_argument_checks(ops, dev):
    """a window without causal runs only when asked for with bidirectional=True, which excludes causal; a negative window and
    probability dropout with a window stay refused"""
    from dalm_b200 import _lib
    B, L, H, D = 1, 64, 2, 64
    x = torch.zeros(B * L, H * D, dtype=bf16, device=dev)
    for fwd in (ops.attention_fwd, ops.attention_tc_fwd):
        with pytest.raises(_lib.DalmB200Error, match="window 8 without causal is a bidirectional window"):
            fwd(x, x, x, None, B, L, H, H, D, False, window=8)
        with pytest.raises(_lib.DalmB200Error, match="exclusive"):
            fwd(x, x, x, None, B, L, H, H, D, True, window=8, bidirectional=True)
        with pytest.raises(_lib.DalmB200Error, match="window"):
            fwd(x, x, x, None, B, L, H, H, D, False, window=-1, bidirectional=True)
        with pytest.raises(_lib.DalmB200Error, match="dropout"):
            fwd(x, x, x, None, B, L, H, H, D, False, window=8, bidirectional=True, drop=ops.Drop(0.1, 1, 1, None))
        out, lse = fwd(x, x, x, None, B, L, H, H, D, False, window=8, bidirectional=True)
        assert torch.isfinite(lse).all() and torch.isfinite(out).all()
    o, lse = ops.attention_tc_fwd(x, x, x, None, B, L, H, H, D, False, window=8, bidirectional=True)
    with pytest.raises(_lib.DalmB200Error, match="window 8 without causal is a bidirectional window"):
        ops.attention_tc_bwd(x, x, x, None, o, lse, x, B, L, H, H, D, False, window=8)


# ----------------------------------------------------------------------------------------------------------------
# 2. GeGLU
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,F,pad", [(7, 96, 0), (300, 1152, 40), (129, 2624, 8)])
def test_geglu_fwd_bwd_vs_fp64(cuda_dev, M, F, pad):
    """act = gelu_erf(input) * gate from a [input | gate] buffer with a row stride wider than 2F; the backward in place writes
    [d input | d gate] and leaves the stride's tail alone"""
    from dalm_b200 import ops
    g = torch.Generator().manual_seed(M + F)
    base = _poisoned(torch.empty(M, 2 * F + pad, dtype=bf16).normal_(0, 1.5, generator=g).to(cuda_dev))
    x = base[:, :2 * F]
    x0 = x.double().clone()
    act = Guarded(M, F, bf16, cuda_dev)
    ops.geglu_fwd(x, F, act=act.view)
    inp, gate = x0[:, :F], x0[:, F:]
    gelu = 0.5 * inp * (1 + torch.erf(inp / math.sqrt(2)))
    want = gelu * gate
    assert (act.view.double() - want).abs().max() <= 2 ** -7 * want.abs().max() * 1.01 + 1e-6
    assert ((act.view.double() - want).abs() <= want.abs() * 2 ** -7 + 1e-3).all()
    act.check(f"geglu_fwd M {M} F {F}")
    d = torch.empty(M, F, dtype=bf16).normal_(0, 1, generator=g).to(cuda_dev)
    tail = base[:, 2 * F:].clone()
    ops.geglu_bwd_(x, d, F)
    dd = d.double()
    pdf = torch.exp(-0.5 * inp * inp) / math.sqrt(2 * math.pi)
    want_in, want_gate = dd * gate * (0.5 * (1 + torch.erf(inp / math.sqrt(2))) + inp * pdf), dd * gelu
    for name, got, w in (("d input", x[:, :F], want_in), ("d gate", x[:, F:], want_gate)):
        assert ((got.double() - w).abs() <= w.abs() * 2 ** -7 + 1e-3 * w.abs().max()).all(), name
    assert torch.equal(base[:, 2 * F:], tail)


# ----------------------------------------------------------------------------------------------------------------
# 3. encoder against transformers
# ----------------------------------------------------------------------------------------------------------------
def _state(cfg, seed):
    from dalm_b200.engine import params
    sd = params.random_state_dict("modernbert", cfg, seed=seed)
    H = cfg["hidden_size"]
    for k in sd:
        if k.endswith("attn.Wqkv.weight"):
            sd[k][:2 * H] *= QK_SCALE
            sd[k][2 * H:] *= V_SCALE
        if k.endswith("attn.Wo.weight"):
            sd[k] *= V_SCALE
    return r16(sd)


def _padded(B, L, seed, pad="right"):
    """[CLS] w .. w [SEP] rows with [PAD] where the mask is 0; lengths cycle through L, L // 3 + 1, L - 5"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.full((B, L), PAD, dtype=i64)
    mask = torch.zeros(B, L, dtype=i64)
    for b in range(B):
        n = (L, L // 3 + 1, L - 5)[b % 3]
        s = L - n if pad == "left" else 0
        ids[b, s:s + n] = torch.randint(5, 50000, (n,), generator=g)
        ids[b, s], ids[b, s + n - 1] = 50281, 50282
        mask[b, s:s + n] = 1
    return ids, mask


def _encoder(cuda_dev, name, seed, full=False, cfg_extra=None):
    from dalm_b200 import synthetic
    from dalm_b200.engine.modernbert import ModernBertEncoder
    cfg = dict(synthetic.modernbert_config(name), **(cfg_extra or {}))
    sd = _state(cfg, seed)
    return cfg, sd, ModernBertEncoder(cfg, sd, device=cuda_dev, full=full)


@pytest.mark.parametrize("name,B,L,pad", [("modernbert-tiny", 3, 70, "right"), ("modernbert-tiny", 3, 70, "left"),
                                          ("modernbert-hd64", 3, 150, "right"), ("modernbert-hd64", 3, 150, "left"),
                                          ("modernbert-hd64", 1, 8192, "right")])
def test_encoder_forward_matches_transformers(cuda_dev, name, B, L, pad):
    from oracle import models as om
    cfg, sd, enc = _encoder(cuda_dev, name, seed=7)
    ids, mask = _padded(B, L, seed=L, pad=pad)
    hid, _ = enc.forward_hidden(ids.to(cuda_dev), mask.to(cuda_dev), save=False)
    assert torch.isfinite(hid).all()
    with torch.no_grad():
        ref = om.build_modernbert(cfg, sd).to(cuda_dev)(ids.to(cuda_dev), mask.to(cuda_dev))[0]
    valid = mask.bool().to(cuda_dev)
    err = rel(hid[valid], ref[valid])
    assert err < TOL, err
    if L > 1000:
        return
    # control: every layer global (full attention, theta 160000) misses by more than 10x the tolerance
    _, _, ctl = _encoder(cuda_dev, name, seed=7, cfg_extra={"layer_types": ["full_attention"] * cfg["num_hidden_layers"]})
    assert ctl.windows == [0] * cfg["num_hidden_layers"]
    hc, _ = ctl.forward_hidden(ids.to(cuda_dev), mask.to(cuda_dev), save=False)
    assert rel(hc[valid], ref[valid]) > 10 * TOL


def test_full_finetune_every_gradient_pad_row_and_round_trip(cuda_dev, tmp_path):
    """a retriever-only step with Adam: the loss and every parameter's gradient against HF autograd; the [PAD] row of
    tok_embeddings gets no gradient and does not move; hf_state_dict reloads in ModernBertModel.from_pretrained and embeds
    the same"""
    from transformers import ModernBertModel

    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    from dalm_b200.optim import FusedAdam
    from dalm_b200.training.utils.train_utils import fused_retriever_step, save_full_dir
    from oracle import models as om
    cfg, sd, enc = _encoder(cuda_dev, "modernbert-tiny", seed=9, full=True)
    se = AutoModelForSentenceEmbedding("", use_bnb=False, get_peft=False, _model=enc, _load_tokenizer=False)
    q, qm = _padded(6, 20, seed=1, pad="right")
    p, pm = _padded(6, 48, seed=2, pad="left")
    rb = {"query_input_ids": q, "query_attention_mask": qm, "passage_input_ids": p, "passage_attention_mask": pm}
    want = om.retriever_step(om.build_modernbert(cfg, sd), rb)
    opt = FusedAdam(se.parameters(), lr=1e-3)
    opt.zero_grad()
    out = fused_retriever_step(se, rb, 100.0)
    assert abs(out["loss"].item() - want["loss"].item()) / abs(want["loss"].item()) < 2e-2
    worst, n = ("", 0.0), 0
    for key, name in enc._names.items():
        rg = want["grads"]["retriever." + name]
        worst = max(worst, (name, rel(enc.full.g(key), rg)), key=lambda t: t[1])
        n += 1
    assert n == len(sd) and worst[1] < 6e-2, worst
    gt = enc.full.g("tok")
    assert torch.count_nonzero(gt[PAD]) == 0 and gt[50281].abs().max() > 0
    w_pad = enc.full.w32("tok")[PAD].clone()
    opt.step()
    assert torch.equal(enc.full.w32("tok")[PAD], w_pad)
    d = str(tmp_path / "saved")
    save_full_dir(enc, d)
    m = ModernBertModel.from_pretrained(d).float().eval().to(cuda_dev)
    ours = enc.hf_state_dict()
    assert set(ours) == set(m.state_dict())
    for k, v in ours.items():
        assert torch.equal(m.state_dict()[k].cpu(), v), k
    from oracle import pooling
    with torch.no_grad():
        e_ref = se(p, pm)
        e_hf = pooling.normalize(pooling.mean_pooling(m(p.to(cuda_dev), pm.to(cuda_dev))[0].cpu(), pm))
    assert rel(e_ref, e_hf) < TOL


# ----------------------------------------------------------------------------------------------------------------
# 4. steps
# ----------------------------------------------------------------------------------------------------------------
def test_retriever_only_step_under_cuda_graph_equals_eager(cuda_dev):
    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    from dalm_b200.training.utils.train_utils import GraphedStep, fused_retriever_step
    cfg, sd, enc = _encoder(cuda_dev, "modernbert-hd64", seed=31, full=True)
    se = AutoModelForSentenceEmbedding("", use_bnb=False, get_peft=False, _model=enc, _load_tokenizer=False)
    mk = lambda s, pad: dict(zip(("query_input_ids", "query_attention_mask"), _padded(6, 24, s, pad)),
                             **dict(zip(("passage_input_ids", "passage_attention_mask"), _padded(6, 80, s + 1, pad))))
    b1, b2 = mk(41, "right"), mk(43, "left")
    eager = []
    for b in (b1, b2):
        enc.zero_grad_buffers()
        out = fused_retriever_step(se, b, 100.0)
        eager.append((out["loss"].item(), enc.full.grad.clone()))
    graphed = GraphedStep(fused_retriever_step, se, b1, 100.0, zero_grads=enc.zero_grad_buffers)
    for b, (loss, grad) in zip((b1, b2), eager):
        enc.zero_grad_buffers()
        got = graphed(b)["loss"].item()
        assert abs(got - loss) <= 1e-6 * abs(loss), (got, loss)
        assert rel(enc.full.grad, grad) < 1e-5


def test_fused_rag_step_modernbert_retriever_llama_generator(cuda_dev):
    """a fully fine-tuned ModernBERT retriever and a LoRA Llama generator against the HF / PEFT composition"""
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.llama import LlamaDecoder
    from dalm_b200.models.rag_e2e_base_model import AutoModelForRagE2E, Mode
    from dalm_b200.training.utils.train_utils import fused_rag_step
    from oracle import models as om
    cfg, sd, enc = _encoder(cuda_dev, "modernbert-tiny", seed=11, full=True)
    lcfg = synthetic.llama_config("llama-tiny", 500)
    lsd = r16(params.random_state_dict("llama", lcfg, seed=12))
    dec = LlamaDecoder(lcfg, lsd, device=cuda_dev, lora=True)
    g = torch.Generator().manual_seed(13)
    draw_lora_B(dec, g)
    model = AutoModelForRagE2E("", "", get_peft=Mode.GENERATOR, _retriever=enc, _generator=dec, _load_tokenizers=False)
    bert, llama = om.build_modernbert(cfg, sd), om.build_llama(lcfg, lsd)
    attach_lora(llama, dec)
    q, qm = _padded(5, 20, seed=21, pad="right")
    p, pm = _padded(5, 40, seed=22, pad="left")
    Lg = 40
    batch = {"retriever_query_input_ids": q, "retriever_query_attention_mask": qm, "retriever_passage_input_ids": p,
             "retriever_passage_attention_mask": pm, "generator_input_input_ids": torch.randint(3, 500, (5, Lg), generator=g),
             "generator_input_attention_mask": torch.ones(5, Lg, dtype=i64),
             "query_passage_input_len": torch.randint(1, Lg + 3, (5,), generator=g)}
    batch["generator_input_attention_mask"][0, :5] = 0
    ref = om.rag_step(bert, llama, batch)
    enc.zero_grad_buffers(); dec.lora.zero_grad()
    got = fused_rag_step(model, batch, 100.0)["losses"].cpu()
    assert abs(got[2].item() - ref["loss"].item()) / abs(ref["loss"].item()) < 1e-3
    assert abs(got[0].item() - ref["Lc"].item()) / abs(ref["Lc"].item()) < 2e-2
    worst = max(rel(enc.full.g(key), ref["grads"]["retriever." + name]) for key, name in enc._names.items())
    assert worst < 6e-2, worst
    worst = lora_grad_error(dec, ref["grads"], "generator.")
    assert worst < 6e-2, worst


# ----------------------------------------------------------------------------------------------------------------
# 5. trainers and evaluations end to end
# ----------------------------------------------------------------------------------------------------------------
def test_train_and_evaluate_with_modernbert_directory(cuda_dev, tmp_path):
    import os

    from safetensors.torch import load_file
    from transformers import ModernBertModel

    from dalm_b200 import synthetic
    from dalm_b200.eval.eval_rag import evaluate_rag
    from dalm_b200.eval.eval_retriever_only import evaluate_retriever
    from dalm_b200.models.rag_e2e_base_model import Mode
    from dalm_b200.training.rag_e2e.train_rage2e import train_e2e
    from dalm_b200.training.retriever_only.train_retriever_only import train_retriever
    csv = synthetic.write_csv(str(tmp_path / "toy.csv"), 12, seed=5)
    rdir = synthetic.write_model_dir(str(tmp_path / "modernbert-tiny"), "modernbert", "modernbert-tiny")
    gdir = synthetic.write_model_dir(str(tmp_path / "llama-tiny"), "llama", "llama-tiny", vocab_size=900)
    out = str(tmp_path / "out_ret")
    train_retriever(rdir, csv, per_device_train_batch_size=2, query_max_len=16, passage_max_len=48, num_train_epochs=1,
                    output_dir=out, use_peft=False, use_bnb=False, with_tracking=False)
    saved = os.path.join(out, "retriever")
    sd, sd0 = load_file(os.path.join(saved, "model.safetensors")), load_file(os.path.join(rdir, "model.safetensors"))
    assert set(sd) == set(sd0) and sum((sd[k] - sd0[k]).abs().max() > 0 for k in sd0) > 20
    assert torch.equal(sd["embeddings.tok_embeddings.weight"][PAD], sd0["embeddings.tok_embeddings.weight"][PAD])
    ModernBertModel.from_pretrained(saved)
    res = evaluate_retriever(csv, saved, None, "Abstract", "Question", embed_dim=64, max_length=48, test_batch_size=8, top_k=5)
    assert res.total_examples == 12 and 0.0 <= res.recall <= 1.0
    out2 = str(tmp_path / "out_e2e")
    train_e2e(csv, rdir, gdir, per_device_train_batch_size=2, query_max_len=16, passage_max_len=48, generator_max_len=64,
              num_train_epochs=1, output_dir=out2, use_peft=Mode.GENERATOR, with_tracking=False, num_warmup_steps=1)
    assert os.path.exists(os.path.join(out2, "retriever", "model.safetensors"))
    assert os.path.exists(os.path.join(out2, "generator", "adapter_model.bin"))
    res = evaluate_rag(csv, os.path.join(out2, "retriever"), gdir, None, os.path.join(out2, "generator"), "Abstract",
                       "Question", "Answer", embed_dim=64, max_length=64, test_batch_size=4, query_batch_size=4, top_k=3,
                       evaluate_generator=False)
    assert res.total_examples == 12 and 0.0 <= res.recall <= 1.0
