"""-m gpu: XLM-RoBERTa / RoBERTa retrievers against transformers' XLMRobertaModel / RobertaModel (eager attention) at the
tolerances the BERT encoder tests use: the roberta_embed kernel and the padding-aware scatter exactly, the encoder forward and
LoRA backward (with a control that BERT's column positions miss), full fine-tuning of every parameter including the
padding_idx rows, dropout with replayed masks, the fused RAG step, CUDA-graph capture, use_bnb storage, and the trainers and
evaluations end to end on a synthetic XLM-R directory."""
import json
import os

import pytest
import torch

from exact_helpers import _dense_poisoned, _expect_equal, _poisoned
from model_helpers import attach_lora, check_rag_lora_grads, compare_full_grads, draw_lora_B, hf_grads, lora_grad_error, r16, rel

pytestmark = pytest.mark.gpu
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
PAD = 1                                   # pad_token_id of every published XLM-R / RoBERTa checkpoint


def _encoder(dev, name="xlmr-tiny", V=700, seed=1, lora_B=True, **kw):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.bert import BertEncoder
    cfg = synthetic.roberta_config(name, V)
    cfg.update(kw.pop("cfg", {}))
    sd = r16(params.random_state_dict("roberta", cfg, seed=seed))
    enc = BertEncoder(cfg, sd, device=dev, **kw)
    if enc.lora is not None and lora_B:
        draw_lora_B(enc, torch.Generator().manual_seed(seed + 4))
    return cfg, sd, enc


def _padded(B, L, V, seed, pad="right"):
    """<s> w .. w </s> rows with <pad> = 1 where the mask is 0, as the XLM-R tokenizer writes them. Row lengths cycle through
    L - 6, L (no padding), L // 2 + 1"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(4, V, (B, L), generator=g)
    mask = torch.ones(B, L, dtype=torch.int64)
    for b in range(B):
        n = (L - 6, L, L // 2 + 1)[b % 3]
        s = L - n if pad == "left" else 0
        ids[b, :] = PAD
        ids[b, s:s + n] = torch.randint(4, V, (n,), generator=g)
        ids[b, s], ids[b, s + n - 1] = 0, 2
        mask[b, :] = 0
        mask[b, s:s + n] = 1
    return ids, mask


def _hf_positions(ids, pad=PAD):
    from transformers.models.xlm_roberta.modeling_xlm_roberta import XLMRobertaEmbeddings
    return XLMRobertaEmbeddings.create_position_ids_from_input_ids(ids, pad)


class _DenseGuarded:
    """a dense [n] output (the layout the embedding kernels write) between two 4096-element sentinel bands"""
    G = 4096

    def __init__(self, n, dtype, dev):
        itype, self.bits = {f32: (torch.int32, 0x7FA5A5A5), torch.int64: (torch.int64, -0x5A5A5A5A)}[dtype]
        self.buf = torch.full((n + 2 * self.G,), self.bits, dtype=itype, device=dev)
        self.n, self.itype = n, itype
        self.view = self.buf.view(dtype)[self.G:self.G + n]

    def check(self, what):
        b = self.buf
        bad = int((b[:self.G] != self.bits).sum() + (b[self.G + self.n:] != self.bits).sum())
        assert bad == 0, f"{what}: {bad} guard elements overwritten"


# ----------------------------------------------------------------------------------------------------------------
# kernels
# ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,L,P,case", [(5, 40, 514, "mixed"), (2, 8192, 8194, "long"), (3, 40, 24, "clamped")])
def test_roberta_embed_positions_and_sum(cuda_dev, B, L, P, case):
    """positions bit-equal to HF's create_position_ids_from_input_ids (right, left and no padding, pad ids inside a row,
    out-of-range word ids read as row 0; positions past a short table clamped); integer tables make the fp32 sum exact, so z
    is compared bit for bit with the fp64 sum; NaN-poisoned tables and guarded outputs"""
    from dalm_b200 import ops
    dev, H, V = cuda_dev, 264, 300
    if case == "long":
        ids, _ = _padded(B, L, V, seed=3, pad="left")
        ids[1] = _padded(1, L, V, seed=4, pad="right")[0][0]
        ids[1, 4000:] = PAD
    else:
        ids = torch.cat([_padded(3, L, V, seed=5, pad=p)[0] for p in ("right", "left")])[:B]
        ids[-1, 7] = PAD                                                  # a pad id inside a row is a pad position for HF too
        ids[-1, 9:13] = torch.tensor([-1, V, 2 ** 40, V - 1])
    g = torch.Generator(device=dev).manual_seed(21)
    word = torch.randint(-100, 101, (V, H), generator=g, device=dev).to(bf16)
    pos = torch.randint(-100, 101, (P, H), generator=g, device=dev).to(bf16)
    typ = torch.randint(-100, 101, (H,), generator=g, device=dev).to(bf16)
    want_pos = _hf_positions(ids).clamp(0, P - 1).to(dev)
    zg, pg = _DenseGuarded(B * L * H, f32, dev), _DenseGuarded(B * L, torch.int64, dev)
    z, p = ops.roberta_embed(ids.to(dev), _dense_poisoned(word), _dense_poisoned(pos), _poisoned(typ), PAD,
                             out=zg.view.view(B * L, H), pos_ids=pg.view)
    zg.check("roberta_embed z"); pg.check("roberta_embed pos_ids")
    assert torch.equal(p.view(B, L), want_pos)
    if case == "clamped":
        assert (_hf_positions(ids) >= P).any()
    else:
        assert torch.equal(p.view(B, L).cpu(), _hf_positions(ids))
    idc = ids.to(dev).view(-1)
    row = torch.where((idc >= 0) & (idc < V), idc, torch.zeros_like(idc))
    _expect_equal(z, word.double()[row] + pos.double()[p] + typ.double(), "roberta_embed")
    # non-integer tables: the same fp32 additions in bert_embed's order, (word + pos) + type
    wr, pr, tr = (torch.randn(s, generator=g, device=dev).to(bf16) for s in ((V, H), (P, H), (H,)))
    z2, _ = ops.roberta_embed(ids.to(dev), wr, pr, tr, PAD)
    assert torch.equal(z2, (wr.float()[row] + pr.float()[p]) + tr.float())


def test_scatter_with_positions_and_padding_idx(cuda_dev):
    """integer gradients (exact whatever the atomic order): with pos_ids / pad_id the scatter is index_add_ over the tokens
    whose id is not pad (word table) and the positions that are not pad (position table); row pad of either table is left
    as it was. pos_ids=None, pad_id=-1 gives the bits of the call without them."""
    from dalm_b200 import ops
    dev, B, L, V, H, P = cuda_dev, 6, 24, 200, 132, 40
    ids = torch.cat([_padded(3, L, V, seed=7, pad=p)[0] for p in ("right", "left")]).to(dev)
    ids[0, 5], ids[1, 3:6] = PAD, torch.tensor([-1, V, 0], device=dev)
    M = B * L
    g = torch.Generator(device=dev).manual_seed(22)
    zero = torch.zeros(V, H, dtype=bf16, device=dev)
    _, pos_ids = ops.roberta_embed(ids, zero, torch.zeros(P, H, dtype=bf16, device=dev), zero[0], PAD)
    d = torch.randint(-8, 9, (M, H), generator=g, device=dev).float()
    w0 = torch.randint(-4, 5, (V, H), generator=g, device=dev).float()
    p0 = torch.randint(-4, 5, (P, H), generator=g, device=dev).float()
    dw, dp = w0.clone(), p0.clone()
    flat = ids.view(-1).contiguous()
    ops.embed_scatter_add_(_dense_poisoned(d), flat, dw, dp, L, pos_ids=pos_ids, pad_id=PAD)
    row = torch.where((flat >= 0) & (flat < V), flat, torch.zeros_like(flat))
    kw, kp = flat != PAD, pos_ids != PAD
    assert (~kw).sum() > 10 and (~kp).sum() == (~kw).sum()
    _expect_equal(dw, w0.double().index_add(0, row[kw], d[kw].double()), "scatter dword (padding_idx)")
    _expect_equal(dp, p0.double().index_add(0, pos_ids[kp], d[kp].double()), "scatter dpos (pos_ids, padding_idx)")
    assert torch.equal(dw[PAD], w0[PAD]) and torch.equal(dp[PAD], p0[PAD])
    a_w, a_p, b_w, b_p = w0.clone(), p0[:L].clone(), w0.clone(), p0[:L].clone()
    ops.embed_scatter_add_(d, flat, a_w, a_p, L)
    ops.embed_scatter_add_(d, flat, b_w, b_p, L, pos_ids=None, pad_id=-1)
    assert torch.equal(a_w, b_w) and torch.equal(a_p, b_p)
    _expect_equal(b_w, w0.double().index_add(0, row, d.double()), "scatter dword (no padding_idx)")
    _expect_equal(b_p, p0[:L].double().index_add(0, torch.arange(M, device=dev) % L, d.double()), "scatter dpos (m % L)")


# ----------------------------------------------------------------------------------------------------------------
# encoder
# ----------------------------------------------------------------------------------------------------------------
def _fwd_bwd_check(dev, name, B, L, pad, cfg_extra=None):
    from dalm_b200 import ops
    from oracle import models as om, pooling
    V = 700
    cfg, sd, enc = _encoder(dev, name, V, lora=True, cfg=cfg_extra or {})
    ref = om.build_roberta(cfg, sd)
    attach_lora(ref, enc)
    ids, mask = _padded(B, L, V, seed=B * L, pad=pad)
    hid, ctx = enc.forward_hidden(ids.to(dev), mask.to(dev))
    ref_hid = ref(ids, mask)[0]
    valid = mask.bool()
    e = rel(hid.cpu()[valid], ref_hid[valid])
    assert e < 1e-2, e                                    # bf16 GEMM operands through N layers (test_engine_gpu's budget)
    with torch.no_grad():                                 # control: BERT's column positions (m % L) are far off
        col = ref(ids, mask, position_ids=torch.arange(L).expand(B, L))[0]
    assert rel(hid.cpu()[valid], col[valid]) > 10 * 1e-2
    emb, norm = ops.pool_norm_fwd(hid, mask.to(dev), True)
    ref_emb = pooling.normalize(pooling.mean_pooling(ref_hid, mask))
    assert rel(emb, ref_emb) < 5e-3
    d_emb = torch.randn(B, cfg["hidden_size"], generator=torch.Generator().manual_seed(9))
    ref_emb.backward(d_emb)
    enc.lora.zero_grad()
    enc.backward_hidden(ctx, ops.pool_norm_bwd(emb, norm, d_emb.to(dev), mask.to(dev), L, True))
    worst = lora_grad_error(enc, hf_grads(ref))
    assert worst < 5e-2, worst                            # bf16 activations / gradients (test_engine_gpu's budget)


@pytest.mark.parametrize("name,B,L,pad", [("xlmr-tiny", 3, 20, "right"), ("xlmr-tiny", 3, 20, "left"), ("xlmr-hd64", 2, 50, "right"),
                                          ("xlmr-hd64", 3, 40, "left"), ("roberta-tiny", 3, 24, "right")])
def test_encoder_fwd_bwd_lora(cuda_dev, name, B, L, pad):
    _fwd_bwd_check(cuda_dev, name, B, L, pad)


def test_encoder_fwd_bwd_lora_long_passages(cuda_dev):
    """Lp 2048 on a 2050-row position table: the whole usable length"""
    _fwd_bwd_check(cuda_dev, "xlmr-hd64", 2, 2048, "right", cfg_extra=dict(max_position_embeddings=2050))


def _rbatch(B, Lq, Lp, V, seed):
    q, qm = _padded(B, Lq, V, seed, pad="right")
    p, pm = _padded(B, Lp, V, seed + 1, pad="left")
    return {"query_input_ids": q, "query_attention_mask": qm, "passage_input_ids": p, "passage_attention_mask": pm}


def test_full_finetune_every_gradient_padding_rows_and_round_trip(cuda_dev, tmp_path):
    from transformers import XLMRobertaModel

    from dalm_b200.engine.bert import BertEncoder
    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    from dalm_b200.optim import FusedAdam
    from dalm_b200.training.utils.train_utils import fused_retriever_step, save_full_dir
    from oracle import models as om
    cfg, sd, enc = _encoder(cuda_dev, "xlmr-tiny", 600, full=True)
    se = AutoModelForSentenceEmbedding("", use_bnb=False, get_peft=False, _model=enc, _load_tokenizer=False)
    ref = om.build_roberta(cfg, sd)
    rb = _rbatch(6, 12, 24, 600, seed=51)
    want = om.retriever_step(ref, rb)
    opt = FusedAdam(se.parameters(), lr=1e-3)
    opt.zero_grad()
    out = fused_retriever_step(se, rb, 100.0)
    assert abs(out["loss"].item() - want["loss"].item()) / abs(want["loss"].item()) < 2e-2
    assert compare_full_grads(enc, want["grads"], "retriever.") > 30
    gw, gp = enc.full.g("word"), enc.full.g("pos")
    assert torch.count_nonzero(gw[PAD]) == 0 and torch.count_nonzero(gp[PAD]) == 0
    assert torch.count_nonzero(want["grads"]["retriever.embeddings.word_embeddings.weight"][PAD]) == 0
    assert gp[PAD + 1].abs().max() > 0 and gw[0].abs().max() > 0           # <s> and position 2 do receive gradient
    w_pad, p_pad = enc.full.w32("word")[PAD].clone(), enc.full.w32("pos")[PAD].clone()
    w0 = enc.full.w32("word")[0].clone()
    opt.step()
    assert torch.equal(enc.full.w32("word")[PAD], w_pad) and torch.equal(enc.full.w32("pos")[PAD], p_pad)
    assert not torch.equal(enc.full.w32("word")[0], w0)
    d = str(tmp_path / "saved")
    save_full_dir(enc, d)
    m = XLMRobertaModel.from_pretrained(d)
    theirs, ours = m.state_dict(), enc.hf_state_dict()
    for k, v in ours.items():
        assert torch.equal(theirs[k], v), k
    assert {k for k in theirs if "position_ids" not in k and "token_type_ids" not in k} == set(ours)
    no_pool = BertEncoder(cfg, {k: v for k, v in sd.items() if not k.startswith("pooler.")}, device=cuda_dev, full=True)
    assert not any(k.startswith("pooler.") for k in no_pool.hf_state_dict())        # bge-m3 ships no pooler


def test_encoder_train_mode_matches_hf_with_replayed_masks(cuda_dev, monkeypatch):
    """dropout on (hidden, attention probabilities, LoRA input) vs HF XLMRobertaModel with torch's dropout patched to replay
    our masks in call order, as test_dropout_gpu does for BERT"""
    from dalm_b200 import ops
    from oracle import models as om, pooling
    cfg, sd, enc = _encoder(cuda_dev, "xlmr-tiny", 800, seed=3, lora=True)
    enc.train()
    B, L, H, nh = 3, 20, cfg["hidden_size"], cfg["num_attention_heads"]
    ids, mask = _padded(B, L, 800, seed=4, pad="left")
    hid, ctx = enc.forward_hidden(ids.to(cuda_dev), mask.to(cuda_dev))
    call = ctx.call
    sc = lambda p, layer, site, shape: ops.dropout_scale(int(torch.tensor(shape).prod()), ops.Drop(p, enc.drop_seed, (call << 24) | (layer << 8) | site, enc.drop_offset), cuda_dev).view(shape).cpu()
    Lp = (L + 7) // 8 * 8
    queue = [sc(enc.p_hidden, 255, 0, (B, L, H))]
    for l in range(enc.nl):
        lm = sc(enc.p_lora, l, 3, (B, L, H))
        queue += [lm, lm, lm, sc(enc.p_attn, l, 8, (B, nh, L, Lp))[..., :L], sc(enc.p_hidden, l, 1, (B, L, H)), sc(enc.p_hidden, l, 2, (B, L, H))]
    ref = om.build_roberta(cfg, sd)
    attach_lora(ref, enc, dropout=0.05)
    ref.train()
    used = []

    def replay(x, p=0.5, training=True, inplace=False):
        if not training or p == 0.0:
            return x
        m = queue[len(used)]
        assert tuple(m.shape) == tuple(x.shape), (len(used), m.shape, x.shape)
        used.append(p)
        return x * m.to(x.dtype)
    monkeypatch.setattr(torch.nn.functional, "dropout", replay)
    monkeypatch.setattr(torch, "dropout", lambda x, p, train: replay(x, p, train))
    ref_hid = ref(ids, mask)[0]
    assert len(used) == len(queue)
    valid = mask.bool()
    assert rel(hid.cpu()[valid], ref_hid[valid]) < 1.2e-2
    emb, norm = ops.pool_norm_fwd(hid, mask.to(cuda_dev), True)
    ref_emb = pooling.normalize(pooling.mean_pooling(ref_hid, mask))
    d_emb = torch.randn(B, H, generator=torch.Generator().manual_seed(6))
    ref_emb.backward(d_emb)
    enc.lora.zero_grad()
    enc.backward_hidden(ctx, ops.pool_norm_bwd(emb, norm, d_emb.to(cuda_dev), mask.to(cuda_dev), L, True))
    worst = lora_grad_error(enc, hf_grads(ref))
    assert worst < 6e-2, worst


# ----------------------------------------------------------------------------------------------------------------
# steps
# ----------------------------------------------------------------------------------------------------------------
def test_fused_rag_step_xlmr_retriever_llama_generator(cuda_dev):
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.llama import LlamaDecoder
    from dalm_b200.models.rag_e2e_base_model import AutoModelForRagE2E, Mode
    from dalm_b200.training.utils.train_utils import fused_rag_step
    from oracle import models as om
    cfg, sd, enc = _encoder(cuda_dev, "xlmr-tiny", 600, seed=11, lora=True)
    lcfg = synthetic.llama_config("llama-tiny", 500)
    lsd = r16(params.random_state_dict("llama", lcfg, seed=12))
    dec = LlamaDecoder(lcfg, lsd, device=cuda_dev, lora=True)
    g = torch.Generator().manual_seed(13)
    draw_lora_B(dec, g)
    model = AutoModelForRagE2E("", "", get_peft=Mode.BOTH, _retriever=enc, _generator=dec, _load_tokenizers=False)
    bert, llama = om.build_roberta(cfg, sd), om.build_llama(lcfg, lsd)
    attach_lora(bert, enc)
    attach_lora(llama, dec)
    rb = _rbatch(5, 12, 24, 600, seed=21)
    Lg = 40
    batch = {"retriever_query_input_ids": rb["query_input_ids"], "retriever_query_attention_mask": rb["query_attention_mask"],
             "retriever_passage_input_ids": rb["passage_input_ids"], "retriever_passage_attention_mask": rb["passage_attention_mask"],
             "generator_input_input_ids": torch.randint(3, 500, (5, Lg), generator=g),
             "generator_input_attention_mask": torch.ones(5, Lg, dtype=torch.int64),
             "query_passage_input_len": torch.randint(1, Lg + 3, (5,), generator=g)}
    batch["generator_input_attention_mask"][0, :5] = 0
    ref = om.rag_step(bert, llama, batch)
    enc.lora.zero_grad(); dec.lora.zero_grad()
    got = fused_rag_step(model, batch, 100.0)["losses"].cpu()
    assert abs(got[2].item() - ref["loss"].item()) / abs(ref["loss"].item()) < 1e-3
    assert abs(got[0].item() - ref["Lc"].item()) / abs(ref["Lc"].item()) < 2e-2
    check_rag_lora_grads(enc, dec, ref)


def test_retriever_only_step_under_cuda_graph_equals_eager(cuda_dev):
    """the positions are computed on the device from the graph's static id buffer: a replay with other ids (other padding)
    gives the eager step's loss and LoRA gradients"""
    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    from dalm_b200.training.utils.train_utils import GraphedStep, fused_retriever_step
    from oracle import models as om
    cfg, sd, enc = _encoder(cuda_dev, "xlmr-hd64", 600, seed=31, lora=True)
    se = AutoModelForSentenceEmbedding("", use_bnb=False, get_peft=True, _model=enc, _load_tokenizer=False)
    b1, b2 = _rbatch(6, 16, 40, 600, seed=41), _rbatch(6, 16, 40, 600, seed=43)
    b2 = {k: v.flip(1) for k, v in b2.items()}                            # left-padded queries, right-padded passages
    eager = []
    for b in (b1, b2):
        enc.lora.zero_grad()
        out = fused_retriever_step(se, b, 100.0)
        eager.append((out["loss"].item(), enc.lora.grad.clone()))
    ref = om.build_roberta(cfg, sd)
    attach_lora(ref, enc)
    want = om.retriever_step(ref, b2)
    assert abs(eager[1][0] - want["loss"].item()) / abs(want["loss"].item()) < 2e-2
    graphed = GraphedStep(fused_retriever_step, se, b1, 100.0, zero_grads=enc.lora.zero_grad)
    for b, (loss, grad) in zip((b1, b2), eager):
        enc.lora.zero_grad()
        got = graphed(b)["loss"].item()
        assert abs(got - loss) <= 1e-6 * abs(loss), (got, loss)
        assert rel(enc.lora.grad, grad) < 1e-5


def test_use_bnb_storage_equals_resident(cuda_dev, tmp_path, monkeypatch):
    """`use_bnb` through the drop-in wrapper on a synthetic XLM-R directory: DALM_B200_NF4_STORAGE=1 embeds exactly like the
    dequantised-resident default and trains with the same loss and LoRA gradients"""
    from dalm_b200 import synthetic
    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    from dalm_b200.training.utils.train_utils import fused_retriever_step
    rdir = synthetic.write_model_dir(str(tmp_path / "xlmr-tiny"), "roberta", "xlmr-tiny", vocab_size=1200)
    ids, mask = _padded(4, 24, 1200, seed=5, pad="right")
    m_res = AutoModelForSentenceEmbedding(rdir, use_bnb=True, get_peft=True)
    monkeypatch.setenv("DALM_B200_NF4_STORAGE", "1")
    m_st = AutoModelForSentenceEmbedding(rdir, use_bnb=True, get_peft=True)
    assert m_st.model.nf4 is not None and m_res.model.nf4 is None and m_st.model.roberta
    with torch.no_grad():
        assert torch.equal(m_res(ids, mask), m_st(ids, mask))
    batch = {"query_input_ids": ids, "query_attention_mask": mask, "passage_input_ids": ids.flip(1), "passage_attention_mask": mask.flip(1)}
    for m in (m_res, m_st):
        m.model.lora.flat.copy_(m_res.model.lora.flat); m.model.repack_lora(); m.model.lora.zero_grad()
    l_res = fused_retriever_step(m_res, batch, 100.0)["loss"].item()
    l_st = fused_retriever_step(m_st, batch, 100.0)["loss"].item()
    assert abs(l_res - l_st) < 1e-5 * max(1.0, abs(l_res))
    assert rel(m_st.model.lora.grad, m_res.model.lora.grad) < 2e-2 and m_st.model.lora.grad.abs().max().item() > 0


# ----------------------------------------------------------------------------------------------------------------
# trainers and evaluations end to end
# ----------------------------------------------------------------------------------------------------------------
def test_train_and_evaluate_with_xlmr_directory(cuda_dev, tmp_path):
    from safetensors.torch import load_file
    from transformers import XLMRobertaModel

    from dalm_b200 import synthetic
    from dalm_b200.eval.eval_rag import evaluate_rag
    from dalm_b200.eval.eval_retriever_only import evaluate_retriever
    from dalm_b200.models.rag_e2e_base_model import Mode
    from dalm_b200.training.rag_e2e.train_rage2e import train_e2e
    from dalm_b200.training.retriever_only.train_retriever_only import train_retriever
    csv = synthetic.write_csv(str(tmp_path / "toy.csv"), 12, seed=5)
    rdir = synthetic.write_model_dir(str(tmp_path / "xlmr-tiny"), "roberta", "xlmr-tiny", vocab_size=1200)
    gdir = synthetic.write_model_dir(str(tmp_path / "llama-tiny"), "llama", "llama-tiny", vocab_size=900)
    # retriever only, LoRA, with a step checkpoint and a resume from it
    out = str(tmp_path / "out_ret")
    train_retriever(rdir, csv, per_device_train_batch_size=2, query_max_len=16, passage_max_len=32, num_train_epochs=1,
                    output_dir=out, use_peft=True, use_bnb=False, with_tracking=False, checkpointing_steps="3")
    ac = json.load(open(os.path.join(out, "retriever", "adapter_config.json")))
    assert sorted(ac["target_modules"]) == ["key", "query", "value"] and ac["base_model_name_or_path"] == rdir
    train_retriever(rdir, csv, per_device_train_batch_size=2, query_max_len=16, passage_max_len=32, num_train_epochs=1,
                    output_dir=out, use_peft=True, use_bnb=False, with_tracking=False,
                    resume_from_checkpoint=os.path.join(out, "step_3"))
    res = evaluate_retriever(csv, rdir, os.path.join(out, "retriever"), "Abstract", "Question", embed_dim=64, max_length=32,
                             test_batch_size=8, top_k=5)
    assert res.total_examples == 12 and 0.0 <= res.recall <= 1.0
    # retriever only, fully fine-tuned: the saved directory loads into XLMRobertaModel with moved weights
    out_f = str(tmp_path / "out_full")
    train_retriever(rdir, csv, per_device_train_batch_size=2, query_max_len=16, passage_max_len=32, num_train_epochs=1,
                    output_dir=out_f, use_peft=False, use_bnb=False, with_tracking=False)
    sd, sd0 = load_file(os.path.join(out_f, "retriever", "model.safetensors")), load_file(os.path.join(rdir, "model.safetensors"))
    assert sum((sd[k] - sd0[k]).abs().max() > 0 for k in sd0 if not k.startswith("pooler")) > 30
    assert torch.equal(sd["embeddings.word_embeddings.weight"][PAD], sd0["embeddings.word_embeddings.weight"][PAD])
    XLMRobertaModel.from_pretrained(os.path.join(out_f, "retriever"))
    # RAG end to end, LoRA on both, with resume, then eval-rag
    out2 = str(tmp_path / "out_e2e")
    kw = dict(per_device_train_batch_size=2, query_max_len=16, passage_max_len=32, generator_max_len=64, num_train_epochs=1,
              output_dir=out2, use_peft=Mode.BOTH, with_tracking=False)
    train_e2e(csv, rdir, gdir, checkpointing_steps="3", num_warmup_steps=1, **kw)
    for sub in ("retriever", "generator"):
        assert os.path.exists(os.path.join(out2, sub, "adapter_model.bin"))
    train_e2e(csv, rdir, gdir, resume_from_checkpoint=os.path.join(out2, "step_3"), **kw)
    res = evaluate_rag(csv, rdir, gdir, os.path.join(out2, "retriever"), os.path.join(out2, "generator"), "Abstract", "Question",
                       "Answer", embed_dim=64, max_length=64, test_batch_size=4, query_batch_size=4, top_k=3,
                       evaluate_generator=False)
    assert res.total_examples == 12 and 0.0 <= res.recall <= 1.0
