"""Where the time of restaging bench.py's configs[1] table from host memory goes (the `e2e_raw` step: five 100 M-row
columns from pinned memory through sdbg_stage_column, then the GROUP BY through the host API).

Reports, after warm-up:
  calls     host wall time of every call of the step (stage k, a, b, v, w, groupby), mean over --steps;
  h2d_ref   one 800 MB pinned -> device copy through torch, for the PCIe rate of this machine;
  device    per kernel / copy name: device time per step, from torch.profiler with CUDA activities (a separate pass);
  api       the CUDA runtime calls the profiler saw on the host (allocations, frees, synchronisations), time per step;
and the GPU name and power limit read in the same run.

    python tools/stage_bench.py [--rows 100000000] [--steps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (COLS, K, A, B, V, W_: the benchmark's own table)
import serenedb_b200 as sdb  # noqa: E402


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    rows, span = args.rows, 100000
    ctx = sdb.Context(0)
    src = sdb.Segment(ctx, rows)
    host = {}
    for f, (stream, kind, dt) in bench.COLS.items():
        src.synth_column(f, stream, kind, 0, rows)
        host[f] = torch.empty(rows, dtype=torch.int64 if dt == np.int64 else torch.float64, pin_memory=True)
        src.column_to_host(f, host[f].data_ptr(), rows)
    src.close()
    ctx.sync()
    preds = [sdb.pred(bench.A, "LT", 500000), sdb.pred(bench.B, "GE", 0.25)]
    eseg = sdb.Segment(ctx, rows)
    escan = sdb.IResearchScan([eseg])
    names = ["stage_%d" % f for f in bench.COLS] + ["groupby"]

    def step(wall=None):
        for f, (_, _, dt) in bench.COLS.items():
            t0 = time.perf_counter()
            eseg.stage_column(f, (host[f].data_ptr(), dt, rows))
            if wall is not None:
                wall["stage_%d" % f] += time.perf_counter() - t0
        t0 = time.perf_counter()
        res = escan.groupby(preds, bench.K, sum_int_field=bench.V, avg_f64_field=bench.W_, cap=span, n_groups_hint=span)
        if wall is not None:
            wall["groupby"] += time.perf_counter() - t0
        return res

    for _ in range(2):
        step()
    ctx.sync()
    wall = {n: 0.0 for n in names}
    t0 = time.perf_counter()
    for _ in range(args.steps):
        step(wall)
    total = (time.perf_counter() - t0) / args.steps * 1e3
    calls = {n: round(v / args.steps * 1e3, 3) for n, v in wall.items()}

    d = torch.empty(rows, dtype=torch.int64, device="cuda")
    d.copy_(host[bench.K], non_blocking=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(3):
        d.copy_(host[bench.K], non_blocking=True)
    torch.cuda.synchronize()
    h2d_ms = (time.perf_counter() - t0) / 3 * 1e3
    del d

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
            step()
        ctx.sync()
    device, api = {}, {}
    for e in prof.key_averages():
        dev_us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if e.key.startswith("cuda"):
            api[e.key] = {"calls_per_step": e.count / 2, "ms_per_step": round(e.cpu_time_total / 2 / 1e3, 3)}
        elif dev_us and not e.key.startswith("aten"):
            device[e.key[:60]] = round(dev_us / 2 / 1e3, 3)
            api[e.key] = {"calls_per_step": e.count / 2, "ms_per_step": round(e.cpu_time_total / 2 / 1e3, 3)}
    print(json.dumps({"gpu": gpu_info(), "rows": rows, "steps": args.steps, "step_ms": round(total, 3), "calls": calls,
                      "h2d_ref_ms": round(h2d_ms, 3), "device": dict(sorted(device.items(), key=lambda x: -x[1])[:20]),
                      "api": dict(sorted(api.items(), key=lambda x: -x[1]["ms_per_step"])[:15])}))


if __name__ == "__main__":
    main()
