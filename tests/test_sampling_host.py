"""CPU: sampling in `generate` (do_sample=True).

* oracle/sampling.py (the fp64 restatement the GPU kernel is checked against) equals the installed transformers' own
  TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper element for element: the same tokens removed, kept scores
  bit-identical. Rows are redrawn until no cumulative share HF computes lies within 1e-5 of 1 - top_p and no tie group
  straddles the top-p cut: that is the only place where summation order (fp32 in HF, fp64 here) or HF's unstable sort can
  flip a token.
* the generation-config resolver equals HF's `_prepare_generation_config` for a checkpoint without a generation config,
  with Llama-2-7b-hf's published one and with Falcon-7B's, each with and without call overrides.
* beam search and sampling processors that are not built raise; the dispatcher sends greedy calls on exactly as before.
"""
import json
import os
import warnings

import numpy as np
import pytest
import torch

from dalm_b200 import synthetic
from dalm_b200.engine import decoding, params
from oracle import sampling as osmp

bf16 = torch.bfloat16

# generation_config.json as published on the Hugging Face hub
LLAMA2_7B_GEN = {"bos_token_id": 1, "do_sample": True, "eos_token_id": 2, "max_length": 4096, "pad_token_id": 0,
                 "temperature": 0.6, "top_p": 0.9, "transformers_version": "4.31.0.dev0"}
FALCON_7B_GEN = {"_from_model_config": True, "bos_token_id": 11, "eos_token_id": 11, "transformers_version": "4.27.4"}


def draw_rows(V, T, top_k, top_p, seed, n=4):
    """n fp32 rows [n, V] clear of the top-p cut; the second half has a tie group at the k-th largest value (unless the
    settings make every such group straddle the cut, as top_k=1 with top_p < 1 does: then a row without one)"""
    g = torch.Generator().manual_seed(seed)
    scale = 2.0 if V <= 1000 else 6.0                                        # wide enough that the cut token's share > 2e-5
    rows = []
    for r in range(n):
        for attempt in range(500):
            row = torch.randn(V, generator=g) * scale
            if r >= n // 2 and V > 3 and attempt < 100:
                k = min(max(top_k, 1), V)
                kth = torch.sort(row.float(), descending=True).values[k - 1]
                idx = torch.randperm(V, generator=g)[:3]
                row[idx] = kth                                           # >= 4 tokens tied at the k-th value
            if osmp.clear_of_cut(row.float()[None], T, top_k, top_p):
                rows.append(row)
                break
        else:
            raise AssertionError("no row clear of the top-p cut")
    return torch.stack(rows)


@pytest.mark.parametrize("V", [7, 1000, 32000])
@pytest.mark.parametrize("T", [0.6, 1.0, 1.7])
@pytest.mark.parametrize("top_k", [0, 1, 50, "V+5"])
@pytest.mark.parametrize("top_p", [1.0, 0.9, 0.5, 1e-6])
def test_oracle_matches_hf_warpers(V, T, top_k, top_p):
    k = V + 5 if top_k == "V+5" else top_k
    rows = draw_rows(V, T, k, top_p, seed=V * 7 + int(T * 10) + k)
    want = osmp.hf_warp(rows.float(), T, k, top_p)
    got = torch.from_numpy(osmp.warp(rows.float(), T, k, top_p)).float()
    assert torch.equal(torch.isinf(got), torch.isinf(want))
    fin = torch.isfinite(want)
    assert torch.equal(got[fin].view(torch.int32), want[fin].view(torch.int32))       # kept scores bit for bit
    assert fin.any(-1).all()


def test_oracle_choice_and_ties():
    """inverse CDF in index order; a tie group straddling the top-p cut loses its lowest indices first"""
    row = np.log(np.array([1.0, 2.0, 2.0, 2.0, 3.0]))
    w = osmp.warp(torch.tensor(row, dtype=torch.float32), 1.0, 0, 1.0)
    c, Z = osmp.prefix_mass(w)
    assert osmp.choose(w, 0.0) == 0 and osmp.choose(w, (c[0] - 1e-9) / Z) == 0 and osmp.choose(w, (c[0] + 1e-9) / Z) == 1
    assert osmp.choose(w, 1 - 2 ** -24) == 4
    # shares 0.1, 0.2, 0.2, 0.2, 0.3: 1 - top_p = 0.35 removes index 0 (0.1) and index 1 (0.3); index 2 (0.5) stays
    w = osmp.warp(torch.tensor(row, dtype=torch.float32), 1.0, 0, 0.65)
    assert np.isinf(w[:2]).all() and np.isfinite(w[2:]).all()


# ----------------------------------------------------------------------------------------------------------------
# generation config
# ----------------------------------------------------------------------------------------------------------------
def _saved_llama(tmp_path, gen):
    from oracle import models as om
    cfg = synthetic.llama_config("llama-tiny", 400)
    model = om.build_llama(cfg, params.random_state_dict("llama", cfg, seed=2))
    d = str(tmp_path)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model.save_pretrained(d)
    gpath = os.path.join(d, "generation_config.json")
    if os.path.exists(gpath):
        os.remove(gpath)
    if gen is not None:
        with open(gpath, "w") as f:
            json.dump(gen, f)
    return d


@pytest.mark.parametrize("which", ["none", "llama2", "falcon"])
@pytest.mark.parametrize("overrides", [{}, {"do_sample": False}, {"top_k": 0}, {"temperature": 1.3}])
def test_resolver_matches_prepare_generation_config(tmp_path, which, overrides):
    from transformers import LlamaForCausalLM
    gen = {"none": None, "llama2": LLAMA2_7B_GEN, "falcon": FALCON_7B_GEN}[which]
    d = _saved_llama(tmp_path, gen)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model = LlamaForCausalLM.from_pretrained(d)
        call = dict(max_length=96, early_stopping=True, **overrides)     # the reference's eval-rag call, plus overrides
        hf, _ = model._prepare_generation_config(None, **call)
    ours = decoding.resolve_generation_config(params.load_config(d), decoding.load_generation_config(d), call)
    eos = lambda e: [] if e is None else (list(e) if isinstance(e, (list, tuple)) else [int(e)])
    for f in ("do_sample", "temperature", "top_k", "top_p", "pad_token_id", "max_length"):
        assert ours[f] == getattr(hf, f), (f, ours[f], getattr(hf, f))
    assert eos(ours["eos_token_id"]) == eos(hf.eos_token_id)
    assert (decoding.load_generation_config(d) is None) == (gen is None)


class _Dec:
    def __init__(self, gen=None):
        self.cfg = synthetic.llama_config("llama-tiny", 400)
        self.generation_config = gen


def test_unbuilt_settings_raise():
    ids = torch.zeros(1, 3, dtype=torch.int64)
    with pytest.raises(NotImplementedError, match="num_beams"):
        decoding.generate(_Dec(), ids, num_beams=2)
    with pytest.raises(NotImplementedError, match="num_beams"):
        decoding.generate(_Dec(LLAMA2_7B_GEN), ids, num_beams=2)
    with pytest.raises(NotImplementedError, match="typical_p"):
        decoding.generate(_Dec(), ids, do_sample=True, typical_p=0.9)
    with pytest.raises(NotImplementedError, match="repetition_penalty"):
        decoding.generate(_Dec(LLAMA2_7B_GEN), ids, repetition_penalty=1.2)     # the file asks for sampling
    with pytest.raises(NotImplementedError, match="min_p"):
        decoding.generate(_Dec(dict(LLAMA2_7B_GEN, min_p=0.1)), ids)
    with pytest.raises(NotImplementedError, match="greedy search only"):
        decoding.greedy_generate(_Dec(), ids, do_sample=True)
    for bad in (dict(temperature=0.0), dict(top_p=0.0), dict(top_k=-1)):
        with pytest.raises(ValueError):
            decoding.sample_generate(_Dec(), ids, **bad)


def test_dispatch(monkeypatch):
    """greedy calls without a generation config reach greedy_generate with the caller's kwargs untouched (unknown flags
    included); a sampling config reaches sample_generate with its warper settings, special tokens and max_length"""
    seen = []
    monkeypatch.setattr(decoding, "greedy_generate", lambda dec, ids, mask, **kw: seen.append(("greedy", kw)))
    monkeypatch.setattr(decoding, "sample_generate", lambda dec, ids, mask, **kw: seen.append(("sample", kw)))
    ids = torch.zeros(2, 3, dtype=torch.int64)
    kw = dict(max_length=40, early_stopping=True, eos_token_id=[], pad_token_id=None, token_type_ids=None)
    decoding.generate(_Dec(), ids, **kw)
    assert seen[-1] == ("greedy", kw)
    decoding.generate(_Dec(), ids, max_new_tokens=3, do_sample=False, num_beams=1)
    assert seen[-1] == ("greedy", dict(max_new_tokens=3))
    decoding.generate(_Dec(LLAMA2_7B_GEN), ids, max_length=96, early_stopping=True)
    assert seen[-1] == ("sample", dict(max_length=96, early_stopping=True, eos_token_id=2, pad_token_id=0, temperature=0.6,
                                       top_k=50, top_p=0.9))
    decoding.generate(_Dec(LLAMA2_7B_GEN), ids, max_length=96, do_sample=False)
    assert seen[-1] == ("greedy", dict(max_length=96, eos_token_id=2, pad_token_id=0))
    decoding.generate(_Dec(), ids, do_sample=True, top_k=20, temperature=0.7)
    assert seen[-1][0] == "sample" and seen[-1][1]["top_k"] == 20 and seen[-1][1]["top_p"] == 1.0
    assert decoding.decoding_mode(_Dec(LLAMA2_7B_GEN), max_length=96) == "sampling (temperature 0.6, top-k 50, top-p 0.9)"
    assert decoding.decoding_mode(_Dec(), max_length=96).startswith("greedy")
