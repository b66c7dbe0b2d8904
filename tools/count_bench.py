"""Count mode against the exact top-k way of counting, on bench.py's own corpora. Two workloads:
  1. the 10 M-doc synthetic corpus with the 4096 two-term disjunctions of bench.make_queries (BASELINE.json configs[2]);
  2. the configs[3] shape: a 5-term conjunction (p = .5/.4/.3/.25/.2) with n BETWEEN 250000 AND 749999, batch of 64.
For each it reports ms per step (CUDA events on the library's stream, L2 flushed before every step, after warm-up) of
  (a) sdbg_match_count_batch;
  (b) sdbg_bm25_topk_batch at pruning level 0 with k = 1 -- the cheapest exact count through the top-k;
  (c) the shipped top-k (pruning level 2, top-1000), for context;
exits non-zero unless (a) equals (b)'s total_matches for every query, and prints the GPU name and power limit read in
the same run.

    python tools/count_bench.py [--steps 10] [--warmup 2] [--docs 10000000] [--queries 4096]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (make_queries, N_TERMS, TOPK: the benchmark's own workload)
import serenedb_b200 as sdb  # noqa: E402
from serenedb_b200 import _native as N  # noqa: E402
from serenedb_b200.engine import _ptr, _seg_array  # noqa: E402


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def timed(ctx, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(steps):
        ctx.flush_l2()
        ctx.timer_start()
        fn()
        ms.append(ctx.timer_stop())
    return round(float(np.mean(ms)), 3), round(float(np.std(ms)), 3)


def workload(ctx, reader, queries, kind, filt, steps, warmup):
    segs, nq = _seg_array(reader.segments), len(queries)
    flat = np.ascontiguousarray([t for q in queries for t in q], dtype=np.uint32)
    off = np.zeros(nq + 1, np.uint32)
    off[1:] = np.cumsum([len(q) for q in queries])
    counts = np.zeros(nq, np.uint64)
    fp = C.byref(filt) if filt is not None else None

    def count():   # arguments marshalled once, like PreparedBatch
        N.check(N.lib().sdbg_match_count_batch(segs, len(reader.segments), kind, _ptr(flat), _ptr(off), nq, None, None, fp,
                                               _ptr(counts)), ctx._h)

    scorer = sdb.BM25(1.2, 0.75)
    exact = sdb.PreparedBatch(reader, queries, kind, scorer, 1, filt=filt)
    shipped = sdb.PreparedBatch(reader, queries, kind, scorer, bench.TOPK, filt=filt)
    ctx.set_wand(2)
    a = timed(ctx, count, steps, warmup)
    ctx.set_wand(0)
    b = timed(ctx, exact.run_host, steps, warmup)
    totals = exact.run_host()[2].copy()
    ctx.set_wand(2)
    c = timed(ctx, shipped.run_host, steps, warmup)
    count()
    return dict(a_count_ms=a[0], a_std=a[1], b_topk1_level0_ms=b[0], b_std=b[1], c_topk1000_level2_ms=c[0], c_std=c[1],
                matches=int(counts.sum()), equal=bool(np.array_equal(counts, totals)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=4096)
    args = ap.parse_args()
    threads = min(os.cpu_count() or 1, 64)

    ctx = sdb.Context(0)
    seg = sdb.Segment(ctx, args.docs)
    dc, sum_dl = seg.synth_corpus(0, 0, bench.N_TERMS, threads=threads)
    reader = sdb.IndexReader([seg], args.docs, sum_dl, dc)
    w1 = workload(ctx, reader, bench.make_queries(args.queries), sdb.OR, None, args.steps, args.warmup)
    w1["workload"] = "%d docs, %d two-term OR queries (bench.make_queries)" % (args.docs, args.queries)
    seg.close()

    seg4 = sdb.Segment(ctx, args.docs)
    dc4, sum_dl4 = seg4.synth_corpus(0, 1000000, 5, threads=threads)   # bench.py configs[3]: generator terms 1000000..1000004
    seg4.synth_column(9, 2, 6, 1, args.docs)
    reader4 = sdb.IndexReader([seg4], args.docs, sum_dl4, dc4)
    w2 = workload(ctx, reader4, [[0, 1, 2, 3, 4]] * 64, sdb.AND, sdb.pred(9, "BETWEEN", 250000, 749999), args.steps, args.warmup)
    w2["workload"] = "%d docs, 5-term AND (p = .5/.4/.3/.25/.2) + n BETWEEN 250000 AND 749999, batch of 64" % args.docs

    print(json.dumps({"gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup, "or_batch": w1, "and_filter_batch": w2}))
    if not (w1["equal"] and w2["equal"]):
        sys.exit(1)


if __name__ == "__main__":
    main()
