"""Cost of excluded terms on the benchmark's BM25 batch (BASELINE.json configs[2]): the 10 M-doc synthetic corpus and the
4096 two-term disjunctions, top-1000, built with bench.py's own generators. Every query additionally excludes one of the
256 terms (fixed seed, never one of its own). Reports ms per step for
  (a) the batch without exclusions, through sdbg_bm25_topk_batch (pruning level 2, the shipped default);
  (b) the batch with exclusions at pruning level 0;
  (c) the batch with exclusions at pruning level 2;
checks that (b) and (c) return identical hits, and prints the GPU name and power limit read in the same run.

    python tools/excl_bench.py [--steps 10] [--warmup 2] [--docs 10000000] [--queries 4096]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (make_queries, N_TERMS, TOPK: the benchmark's own workload)
import serenedb_b200 as sdb  # noqa: E402


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=4096)
    args = ap.parse_args()

    ctx = sdb.Context(0)
    seg = sdb.Segment(ctx, args.docs)
    dc, sum_dl = seg.synth_corpus(0, 0, bench.N_TERMS, threads=min(os.cpu_count() or 1, 64))
    reader = sdb.IndexReader([seg], args.docs, sum_dl, dc)
    queries = bench.make_queries(args.queries)
    rng = np.random.default_rng(20261015)
    excludes = []
    for q in queries:
        t = int(rng.integers(0, bench.N_TERMS))
        while t in q:
            t = int(rng.integers(0, bench.N_TERMS))
        excludes.append([t])
    scorer = sdb.BM25(1.2, 0.75)
    plain = sdb.PreparedBatch(reader, queries, sdb.OR, scorer, bench.TOPK)
    excl = sdb.PreparedBatch(reader, queries, sdb.OR, scorer, bench.TOPK, exclude=excludes)

    def timed(batch, level):
        ctx.set_wand(level)
        for _ in range(args.warmup):
            batch.run_host()
        ms = []
        for _ in range(args.steps):
            ctx.flush_l2()
            ctx.timer_start()
            batch.run_host()
            ms.append(ctx.timer_stop())
        hits, n_out, total = (x.copy() for x in batch.run_host())
        return float(np.mean(ms)), float(np.std(ms)), hits, n_out, total

    a = timed(plain, 2)
    b = timed(excl, 0)
    c = timed(excl, 2)
    same = bool(np.array_equal(b[3], c[3]) and all(np.array_equal(b[2][q, :b[3][q]], c[2][q, :c[3][q]]) for q in range(len(queries))))
    ctx.set_wand(2)
    print(json.dumps({
        "gpu": gpu_info(),
        "workload": "%d docs, %d two-term OR queries, top-%d; (b), (c): one excluded term per query" % (args.docs, len(queries), bench.TOPK),
        "a_plain_level2_ms": round(a[0], 3), "a_std": round(a[1], 3),
        "b_excl_level0_ms": round(b[0], 3), "b_std": round(b[1], 3),
        "c_excl_level2_ms": round(c[0], 3), "c_std": round(c[1], 3),
        "b_equals_c_hits": same,
        "matches_b_total": int(b[4].sum()), "matches_c_total_lower_bound": int(c[4].sum()),
        "steps": args.steps,
    }))
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
