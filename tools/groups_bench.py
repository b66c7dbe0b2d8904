"""Cost of conjunctions of OR groups on the benchmark's BM25 corpus (BASELINE.json configs[2]): the 10 M-doc synthetic
corpus built with bench.py's own generator, and 4096 queries `a & (b | c)`, top-1000: a and b are the two terms of each of
bench.py's two-term queries, c one more of the 256 terms (fixed seed, never a or b). Reports ms per step (mean and std
over the timed steps, L2 flushed before each) for
  (a) the grouped query at pruning level 0;
  (b) the grouped query at pruning level 2 (the shipped default);
  (c) the flat OR `a | b | c` at level 2 and (d) the AND `a & b` at level 2, as brackets;
  (e) the grouped count (sdbg_match_count_batch_groups);
checks that (a) and (b) return identical hits and that (e) equals the level-0 totals of (a), and prints the GPU name and
power limit read in the same run.

    python tools/groups_bench.py [--steps 10] [--warmup 2] [--docs 10000000] [--queries 4096]
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
from serenedb_b200 import _native as N  # noqa: E402
from serenedb_b200.engine import HIT_DTYPE, _groups, _ptr, _seg_array  # noqa: E402


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def make_group_queries(n):
    """bench.make_queries' pairs (a, b) with a third term c: `a & (b | c)`, the flat `a | b | c` and `a & b`."""
    rng = np.random.default_rng(20261015)
    grouped, flat_or, flat_and = [], [], []
    for q in bench.make_queries(n):
        a, b = int(q[0]), int(q[1])
        c = int(rng.integers(0, bench.N_TERMS))
        while c in (a, b):
            c = int(rng.integers(0, bench.N_TERMS))
        grouped.append([[a], [b, c]])
        flat_or.append([a, b, c])
        flat_and.append([a, b])
    return grouped, flat_or, flat_and


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
    grouped, flat_or, flat_and = make_group_queries(args.queries)
    scorer = sdb.BM25(1.2, 0.75)
    k = bench.TOPK

    def timed(fn, level):
        ctx.set_wand(level)
        for _ in range(args.warmup):
            fn()
        ms = []
        for _ in range(args.steps):
            ctx.flush_l2()
            ctx.timer_start()
            fn()
            ms.append(ctx.timer_stop())
        out = fn()
        return float(np.mean(ms)), float(np.std(ms)), tuple(x.copy() for x in out)

    # descriptors marshalled once, as PreparedBatch does for the flat forms: the timed region is the library call
    nq = len(grouped)
    ids, group_off, qgo = _groups(grouped)
    terms = (N.BM25Term * len(ids))(*[reader.stats(scorer, t) for t in ids])
    flat_ids = np.ascontiguousarray(ids, np.uint32)
    segs = _seg_array(reader.segments)
    hits, n_out, total = np.zeros((nq, k), HIT_DTYPE), np.zeros(nq, np.uint32), np.zeros(nq, np.uint64)
    counts = np.zeros(nq, np.uint64)

    def run_groups():
        N.check(N.lib().sdbg_bm25_topk_batch_groups(segs, 1, terms, _ptr(group_off), _ptr(qgo), nq, None, None, scorer.k, scorer.b,
                                                    None, k, sdb.FLT_MIN, _ptr(hits), _ptr(n_out), _ptr(total)), ctx._h)
        return hits, n_out, total

    def run_count():
        N.check(N.lib().sdbg_match_count_batch_groups(segs, 1, _ptr(flat_ids), _ptr(group_off), _ptr(qgo), nq, None, None, None,
                                                      _ptr(counts)), ctx._h)
        return (counts,)

    p_or = sdb.PreparedBatch(reader, flat_or, sdb.OR, scorer, k)
    p_and = sdb.PreparedBatch(reader, flat_and, sdb.AND, scorer, k)
    a = timed(run_groups, 0)
    b = timed(run_groups, 2)
    c = timed(p_or.run_host, 2)
    d = timed(p_and.run_host, 2)
    e = timed(run_count, 2)
    (ha, na, ta), (hb, nb, _) = a[2], b[2]
    same = bool(np.array_equal(na, nb) and all(np.array_equal(ha[q, :na[q]], hb[q, :nb[q]]) for q in range(len(grouped))))
    counts_ok = bool(np.array_equal(e[2][0], ta))
    ctx.set_wand(2)
    print(json.dumps({
        "gpu": gpu_info(),
        "workload": "%d docs, %d queries a & (b | c), top-%d" % (args.docs, len(grouped), k),
        "a_groups_level0_ms": round(a[0], 3), "a_std": round(a[1], 3),
        "b_groups_level2_ms": round(b[0], 3), "b_std": round(b[1], 3),
        "c_flat_or_abc_level2_ms": round(c[0], 3), "c_std": round(c[1], 3),
        "d_and_ab_level2_ms": round(d[0], 3), "d_std": round(d[1], 3),
        "e_groups_count_ms": round(e[0], 3), "e_std": round(e[1], 3),
        "a_equals_b_hits": same, "count_equals_level0_totals": counts_ok,
        "matches": int(ta.sum()), "steps": args.steps,
    }))
    if not (same and counts_ok):
        sys.exit(1)


if __name__ == "__main__":
    main()
