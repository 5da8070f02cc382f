"""CPU: the parts of bench.py's contract that do not need a GPU — rank-strided batches (accelerate order, the N>1 arm),
the reference arm's JSON line (same metric / unit / workload as the GPU arm, rank 0 only)."""
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_rank_strided_batches(tmp_path, monkeypatch):
    import bench
    monkeypatch.setattr(torch.distributed, "barrier", lambda *a, **k: None)
    cache = str(tmp_path)
    single = bench.make_batches(4, 0, 1, cache)                       # global batches 0..3 of the shared order
    r0 = bench.make_batches(2, 0, 2, cache)
    r1 = bench.make_batches(2, 1, 2, cache)
    assert {"retriever_query_input_ids", "retriever_passage_input_ids", "generator_input_input_ids",
            "generator_input_attention_mask", "query_passage_input_len"} <= set(single[0])
    for b in range(2):
        for k in single[0]:
            assert torch.equal(r0[b][k], single[2 * b][k]) and torch.equal(r1[b][k], single[2 * b + 1][k])      # rank r: batches r, r+W, ...
    x = single[0]
    assert x["generator_input_input_ids"].shape == (bench.BS, bench.LG) and x["generator_input_input_ids"].dtype == torch.int64
    assert x["retriever_query_input_ids"].shape == (bench.BS, bench.LQ) and x["retriever_passage_input_ids"].shape == (bench.BS, bench.LP)
    assert int(x["generator_input_attention_mask"].min()) == 1        # the "full" synthetic set: every sequence hits truncation


def test_reference_arm_line(monkeypatch, capsys, tmp_path):
    """the reference arm reports what it RAN: `steps` / `warmup` are the executed counts (the CLI's are kept beside them),
    nothing is extrapolated (VERDICT r1 weak 5)"""
    import bench
    calls = {}

    def fake_run(batch, rows, warmup, steps, budget_s):
        calls.update(rows=rows, warmup=warmup, steps=steps, budget_s=budget_s)
        return {"value": 0.25, "cores": 8, "steps_run": 2, "warmup_run": 1, "s_per_step": 8.0, "rows": rows, "sample": "stubbed sample"}
    monkeypatch.setattr(bench, "cpu_reference_run", fake_run)
    monkeypatch.setattr(sys, "argv", ["bench.py", "--impl", "reference", "--gpus", "2", "--steps", "3", "--warmup", "1"])
    monkeypatch.setenv("RANK", "1"); monkeypatch.setenv("WORLD_SIZE", "2")
    bench.main()                                                      # other ranks exit without work and without output
    assert capsys.readouterr().out.strip() == ""
    monkeypatch.setenv("RANK", "0")
    bench.main()
    out = [l for l in capsys.readouterr().out.splitlines() if l.strip()]
    assert len(out) == 1                                              # ONE JSON line
    line = json.loads(out[0])
    assert calls["steps"] == 3 and calls["warmup"] == 1 and calls["rows"] == 2
    assert line["impl"] == "reference" and line["metric"] == bench.METRIC and line["unit"] == "samples/s"
    assert line["higher_is_better"] is True and line["n_gpus"] == 2
    assert line["steps"] == 2 and line["warmup"] == 1 and line["steps_requested"] == 3       # executed, not echoed
    assert line["extrapolated"] is False and line["ms_per_step"] == 8000.0 and line["rows_per_step"] == 2
    assert line["value"] == 0.25 and line["cpu_baseline"] == {"value": 0.25, "unit": "samples/s", "cores": 8, "kind": "port", "sample": "stubbed sample"}
    assert line["e2e"] == {"value": 0.25, "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    args = bench.parse()
    assert line["config"]["workload"] == bench.workload_name(args)   # the same workload name as the GPU arm prints
