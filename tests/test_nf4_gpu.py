"""-m gpu: `use_bnb` — the NF4 quantise/dequantise round trip (csrc/nf4.cu) bit-exact against the oracle restatement of
bitsandbytes' algorithm (oracle/nf4.py, "parity unpinned": bitsandbytes is absent offline), and the wrappers loading through it."""
import numpy as np
import pytest
import torch

from model_helpers import draw_lora_B, rag_batch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("shape,scale,seed", [((64,), 1.0, 0), ((5, 40), 0.02, 1), ((384, 384), 0.02, 2), ((1000, 129), 3.0, 3),
                                              ((7,), 1e-3, 4)])
def test_nf4_roundtrip_bit_exact_vs_oracle(cuda_dev, shape, scale, seed):
    from dalm_b200 import ops
    from oracle import nf4
    w = (np.random.default_rng(seed).standard_normal(shape) * scale).astype(np.float32)
    if w.size > 200:
        w.reshape(-1)[64:128] = 0.0                                               # an all-zero block
        w.reshape(-1)[130] = w.reshape(-1)[128:192].__abs__().max() * 2            # a block dominated by one outlier
    want, codes, absmax = nf4.roundtrip(w)
    t = torch.from_numpy(w.copy()).to(cuda_dev)
    got, gc, ga = ops.nf4_roundtrip_(t, want_codes=True)
    assert np.array_equal(gc.cpu().numpy(), codes)                                 # integer codes: bit-exact
    assert np.array_equal(ga.cpu().numpy(), absmax)
    assert np.array_equal(got.cpu().numpy(), want)                                 # dequantised fp16 values: bit-exact
    again = ops.nf4_roundtrip_(got.clone())
    assert torch.equal(again, got)                                                 # size-independent property: idempotent
    err = np.abs(want - w.astype(np.float16).astype(np.float32)).reshape(-1)
    bound = np.repeat(absmax, 64)[: w.size] * 0.153 + 1e-6                         # half the widest gap between NF4 levels (0.3038)
    assert (err <= bound).all()


def test_nf4_boundaries_and_levels(cuda_dev):
    from dalm_b200 import ops
    from oracle import nf4
    levels = nf4.NF4.astype(np.float32)
    mids = (np.float32(0.5) * (levels[:-1] + levels[1:])).astype(np.float32)
    # a block whose absmax is exactly 1: levels map to themselves, midpoints go DOWN (`>` in bitsandbytes' decision tree)
    blk = np.zeros(64, np.float32); blk[:16] = levels; blk[16:31] = mids; blk[31] = np.nextafter(mids[3], np.float32(1))
    t = torch.from_numpy(blk.copy()).to(cuda_dev)
    _, codes, absmax = ops.nf4_roundtrip_(t, want_codes=True)
    _, ocodes, _ = nf4.roundtrip(blk)
    c = codes.cpu().numpy()
    assert np.array_equal(c, ocodes) and absmax.item() == 1.0
    assert c[:16].tolist() == list(range(16))


def test_wrappers_load_through_nf4(cuda_dev, tmp_path):
    """use_bnb=True (the reference's retriever-only default): embeddings equal the oracle HF model loaded with the oracle's NF4
    values, and differ from the un-quantised model; use_bnb without PEFT on the same sub-model is refused"""
    from safetensors.torch import load_file
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.models.rag_e2e_base_model import AutoModelForRagE2E, Mode, inference_only
    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    from oracle import models as om, nf4
    import json, os
    rdir = synthetic.write_model_dir(str(tmp_path / "bge-tiny"), "bert", "bge-tiny", vocab_size=1200)
    gdir = synthetic.write_model_dir(str(tmp_path / "llama-tiny"), "llama", "llama-tiny", vocab_size=904)
    m_q = AutoModelForSentenceEmbedding(rdir, use_bnb=True, get_peft=True)
    m_f = AutoModelForSentenceEmbedding(rdir, use_bnb=False, get_peft=True)
    sd = load_file(os.path.join(rdir, "model.safetensors"))
    qsd = {}
    for k, v in sd.items():
        if v.dim() == 2 and params.is_bnb_linear_weight(k):
            qsd[k] = torch.from_numpy(nf4.roundtrip(v.float().numpy())[0])
        else:
            qsd[k] = v.half().float()
    n_quant = sum(v.dim() == 2 and params.is_bnb_linear_weight(k) for k, v in sd.items())
    assert n_quant == 2 * 6 + 1                                                    # 6 Linear per layer x 2 layers + pooler
    bert = om.build_bert(json.load(open(os.path.join(rdir, "config.json"))), qsd)
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(5, 1200, (4, 24), generator=g); mask = torch.ones_like(ids); mask[1, 15:] = 0
    want = om.retrieval_forward(bert, ids, mask).detach()
    with torch.no_grad():
        got_q, got_f = m_q(ids, mask).cpu(), m_f(ids, mask).cpu()
    rel = lambda a, b: ((a - b).norm() / b.norm()).item()
    assert rel(got_q, want) < 2e-2                                                 # bf16 forward vs fp32 oracle on the SAME NF4 values
    assert rel(got_f, want) > 2 * rel(got_q, want)                                 # and the quantisation is really applied
    with pytest.raises(NotImplementedError):
        AutoModelForSentenceEmbedding(rdir, use_bnb=True, get_peft=False)          # 4-bit base + no adapters: nothing trainable
    rag = AutoModelForRagE2E(rdir, gdir, get_peft=Mode.BOTH, use_bnb=Mode.GENERATOR)
    gsd = load_file(os.path.join(gdir, "model.safetensors"))
    w0 = gsd["model.layers.0.mlp.down_proj.weight"].float()
    assert torch.equal(rag.generator_model.layers[0]["Wd"].cpu().float(), torch.from_numpy(nf4.roundtrip(w0.numpy())[0]).bfloat16().float())
    assert torch.equal(rag.generator_model.lm_head.cpu().float()[:904], gsd["lm_head.weight"].half().float().bfloat16().float())   # head: fp16 cast only


@pytest.mark.parametrize("rows,cols,tail", [(48, 64, 0), (384, 384, 24), (1000, 1024, 16), (130, 4544, 0)])
def test_nf4_packed_storage_bit_exact_vs_oracle(cuda_dev, rows, cols, tail):
    """4-bit STORAGE: packed codes (first element in the high nibble, bitsandbytes' layout) and absmax bit-exact against the
    oracle; the per-use expansion gives bf16(fp16(code * absmax)) = exactly what the dequantised-resident mode keeps; the LoRA
    tail block is copied behind each row"""
    from dalm_b200 import ops
    from oracle import nf4
    w = (np.random.default_rng(rows + cols).standard_normal((rows, cols)) * 0.02).astype(np.float32)
    w[1, :64] = 0.0
    want, codes, absmax = nf4.roundtrip(w)
    t = torch.from_numpy(w.copy()).to(cuda_dev)
    packed, am = ops.nf4_quantize(t)
    assert np.array_equal(packed.cpu().numpy(), (codes[0::2] << 4) | codes[1::2])
    assert np.array_equal(am.cpu().numpy(), absmax)
    ld = cols + (64 if tail else 0)
    out = torch.full((rows, ld), 7.0, dtype=torch.bfloat16, device=cuda_dev)
    tl = torch.randn(rows, tail, device=cuda_dev).to(torch.bfloat16) if tail else None
    ops.nf4_dequant_(packed, am, rows, cols, out, tl)
    assert torch.equal(out[:, :cols].cpu(), torch.from_numpy(want).bfloat16())
    resident = ops.nf4_roundtrip_(t.clone()).to(torch.bfloat16)                   # the default mode's values
    assert torch.equal(out[:, :cols], resident)
    if tail:
        assert torch.equal(out[:, cols:cols + tail], tl) and float((out[:, cols + tail:] - 7.0).abs().max()) == 0.0


def test_nf4_storage_mode_equals_resident_mode(cuda_dev, monkeypatch):
    """DALM_B200_NF4_STORAGE=1 (weights kept as packed codes, expanded per use, dgrad against W[out,in] read MN-major) trains
    exactly like the dequantised-resident default: same loss, same LoRA gradients (BERT encoder + Llama decoder, fused step)"""
    from dalm_b200 import synthetic
    from dalm_b200.engine import params
    from dalm_b200.engine.bert import BertEncoder
    from dalm_b200.engine.llama import LlamaDecoder
    from dalm_b200.models.rag_e2e_base_model import AutoModelForRagE2E, Mode
    from dalm_b200.training.utils.train_utils import fused_rag_step
    dev = cuda_dev
    bcfg, lcfg = synthetic.bert_config("bge-tiny", 600), synthetic.llama_config("llama-mini", 500)
    bsd = params.random_state_dict("bert", bcfg, seed=11)
    lsd = params.random_state_dict("llama", lcfg, seed=12)
    batch = rag_batch(4, 12, 24, 40, 600, 500, seed=21)
    res = []
    for storage in (False, True):
        if storage:
            enc = BertEncoder(bcfg, bsd, device=dev, lora=True, nf4_storage=True)
            dec = LlamaDecoder(lcfg, lsd, device=dev, lora=True, nf4_storage=True)
            assert enc.nf4.nbytes() > 0 and "WoT" not in enc.layers[0] and "WdT" not in dec.layers[0]
        else:
            enc = BertEncoder(bcfg, params.bnb_nf4_state_dict(bsd, dev), device=dev, lora=True)
            dec = LlamaDecoder(lcfg, params.bnb_nf4_state_dict(lsd, dev), device=dev, lora=True)
        g = torch.Generator().manual_seed(13)
        draw_lora_B(enc, g); draw_lora_B(dec, g)
        model = AutoModelForRagE2E("", "", get_peft=Mode.BOTH, _retriever=enc, _generator=dec, _load_tokenizers=False)
        enc.lora.zero_grad(); dec.lora.zero_grad()
        out = fused_rag_step(model, batch, 100.0)
        res.append((out["losses"].clone(), enc.lora.grad.clone(), dec.lora.grad.clone()))
        if storage:                                                                # the expanded weight == the resident one
            assert torch.equal(dec.layers[0]["Wd"], dec_res_Wd) and torch.equal(enc.layers[1]["Wi"], enc_res_Wi)
        else:
            dec_res_Wd, enc_res_Wi = dec.layers[0]["Wd"].clone(), enc.layers[1]["Wi"].clone()
    rel = lambda a, b: ((a - b).norm() / (b.norm() + 1e-30)).item()
    assert (res[0][0] - res[1][0]).abs().max().item() < 2e-3 * res[0][0].abs().max().item()
    assert rel(res[1][1], res[0][1]) < 2e-2 and rel(res[1][2], res[0][2]) < 2e-2   # same math, other GEMM layouts / rounding points


def test_wrappers_in_nf4_storage_mode(cuda_dev, tmp_path, monkeypatch):
    """DALM_B200_NF4_STORAGE=1 through the drop-in wrappers: `use_bnb=True` keeps the encoder's Linear weights packed, embeddings
    are identical to the dequantised-resident default (same GEMM operands), adapters attach and train"""
    from dalm_b200 import synthetic
    from dalm_b200.models.retriever_only_base_model import AutoModelForSentenceEmbedding
    from dalm_b200.training.utils.train_utils import fused_retriever_step
    rdir = synthetic.write_model_dir(str(tmp_path / "bge-tiny"), "bert", "bge-tiny", vocab_size=1200)
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(5, 1200, (4, 24), generator=g); mask = torch.ones_like(ids); mask[1, 15:] = 0
    m_res = AutoModelForSentenceEmbedding(rdir, use_bnb=True, get_peft=True)
    monkeypatch.setenv("DALM_B200_NF4_STORAGE", "1")
    m_st = AutoModelForSentenceEmbedding(rdir, use_bnb=True, get_peft=True)
    assert m_st.model.nf4 is not None and m_res.model.nf4 is None and "WoT" not in m_st.model.layers[0]
    with torch.no_grad():
        e_res, e_st = m_res(ids, mask), m_st(ids, mask)
    assert torch.equal(e_res, e_st)
    batch = {"query_input_ids": ids, "query_attention_mask": mask, "passage_input_ids": ids.flip(1), "passage_attention_mask": mask.flip(1)}
    for m in (m_res, m_st):                                    # same adapters -> same loss and the same LoRA gradients
        m.model.lora.flat.copy_(m_res.model.lora.flat); m.model.repack_lora(); m.model.lora.zero_grad()
    l_res = fused_retriever_step(m_res, batch, 100.0)["loss"].item()
    l_st = fused_retriever_step(m_st, batch, 100.0)["loss"].item()
    assert abs(l_res - l_st) < 1e-5 * max(1.0, abs(l_res))
    rel = ((m_st.model.lora.grad - m_res.model.lora.grad).norm() / (m_res.model.lora.grad.norm() + 1e-30)).item()
    assert rel < 2e-2 and m_st.model.lora.grad.abs().max().item() > 0
