"""The headline GROUP BY (bench.py configs[1]: a < 500000 AND b >= 0.25 -> GROUP BY k SUM(v), AVG(w), COUNT(*)) over the
same 100 M-row table held three ways, timed in one process:
  staged  the columns as sdbg_synth_column leaves them (int64 k, a, v bit-packed when that is smaller, b, w raw);
  raw64   the same values as borrowed raw device columns (sdbg_stage_column_device): int64 k, a, v = 40 B/row;
  raw32   k, a, v as borrowed int32 columns: 28 B/row.
Each is timed as shipped and with SDBG_GROUPBY_DEBUG=7 (no RED atomics: wrong results, the bandwidth floor of its
bytes). Reports ms per step (CUDA events on the library's stream, after warm-up), the GROUP BY kernel's own time, the
bytes the kernel really reads per step (packed words + FOR headers + raw columns + the 3.2 MB group table) and that
over kernel time against the HBM peak, and the GPU name and power limit read in the same run. Exits non-zero unless the
three layouts give the same groups.

    python tools/packed_bench.py [--rows 100000000] [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

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
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    rows, span = args.rows, 100000
    assert rows % 2 == 0, "borrowed device columns need an even row count"
    ctx = sdb.Context(0)
    dev = torch.device("cuda", 0)
    preds = [sdb.pred(bench.A, "LT", 500000), sdb.pred(bench.B, "GE", 0.25)]
    d_i64 = torch.zeros(4 * span, dtype=torch.int64, device=dev)
    d_f64 = torch.zeros(span, dtype=torch.float64, device=dev)

    staged = sdb.Segment(ctx, rows)
    for f, (stream, kind, _) in bench.COLS.items():
        staged.synth_column(f, stream, kind, 0, rows)
    host = {}
    for f, (_, _, dt) in bench.COLS.items():
        host[f] = torch.empty(rows, dtype=torch.int64 if dt == np.int64 else torch.float64)
        staged.column_to_host(f, host[f].data_ptr(), rows)
    keep = []
    segs = {"staged": staged}
    for name, idt in (("raw64", torch.int64), ("raw32", torch.int32)):
        seg = sdb.Segment(ctx, rows)
        for f, (_, _, dt) in bench.COLS.items():
            t = host[f].to(dev).to(idt if dt == np.int64 else torch.float64).contiguous()
            keep.append(t)
            seg.stage_column_device(f, t.data_ptr(), np.int32 if t.dtype == torch.int32 else dt, rows)
        segs[name] = seg

    # bytes the kernel reads per step: integer columns as the staged layout holds them (packed words + headers, computed
    # with the host writer of the same format), the doubles raw, plus the group table
    int_bytes = {}
    for f, (_, _, dt) in bench.COLS.items():
        if dt == np.int64:
            hd, wd, _ = sdb.pack_for(host[f].numpy())
            int_bytes[f] = min(hd.nbytes + wd.nbytes, rows * 8)
    dbl = sum(rows * 8 for f, (_, _, dt) in bench.COLS.items() if dt != np.int64)
    read_bytes = {"staged": sum(int_bytes.values()) + dbl + span * 32, "raw64": rows * 40 + span * 32,
                  "raw32": rows * 28 + span * 32}
    peak, peak_src = bench.peaks()

    results, groups = {}, {}
    for debug in (0, 7):
        os.environ["SDBG_GROUPBY_DEBUG"] = str(debug)
        for name, seg in segs.items():
            scan = sdb.IResearchScan([seg])

            def step():
                scan.groupby_partial(preds, bench.K, 0, span, bench.V, bench.W_, d_i64.data_ptr(), d_f64.data_ptr())
            for _ in range(args.warmup):
                step()
            ctx.sync()
            ctx.profile(True)
            ctx.timer_start()
            for _ in range(args.steps):
                step()
            ms = ctx.timer_stop() / args.steps
            k_ms, k_n = ctx.profile_read("groupby")
            ctx.profile(False)
            k_ms /= max(k_n, 1)
            key = "%s%s" % (name, "_nored" if debug else "")
            results[key] = {"ms_per_step": round(ms, 4), "kernel_ms": round(k_ms, 4), "bytes_read": read_bytes[name],
                            "gbs": round(read_bytes[name] / (k_ms * 1e-3) / 1e9, 1),
                            "frac_of_peak": round(read_bytes[name] / (k_ms * 1e-3) / 1e9 / peak, 3),
                            "mrows_s": round(rows / (ms * 1e-3) / 1e6, 1)}
            if not debug:
                groups[name] = scan.groupby_finalize(0, span, d_i64.data_ptr(), d_f64.data_ptr(), span).copy()
    os.environ.pop("SDBG_GROUPBY_DEBUG", None)
    same = all(np.array_equal(groups[n][f], groups["raw64"][f]) for n in groups for f in ("key", "count", "sum_lo", "sum_hi"))
    same = same and all(np.allclose(groups[n]["sum_f64"], groups["raw64"]["sum_f64"], rtol=1e-12) for n in groups)
    print(json.dumps({"gpu": gpu_info(), "rows": rows, "steps": args.steps, "peak_gbs": peak, "peak_source": peak_src,
                      "int_column_bytes": {str(f): b for f, b in int_bytes.items()}, "results": results, "same_groups": same}))
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
