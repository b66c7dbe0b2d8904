"""Cost of OR groups with a minimum match count on the benchmark's BM25 corpus (BASELINE.json configs[2]): the 10 M-doc
synthetic corpus built with bench.py's own generator, and 4096 queries, top-1000: a and b are the two terms of each of
bench.py's two-term queries, c (and, for (e), d, e, f) further terms of the 256 (fixed seed, all distinct). Reports ms per
step (mean and std over the timed steps, L2 flushed before each) for
  (a) `2 of (a | b | c)` at pruning level 0;
  (b) the same at pruning level 2 (the shipped default);
  (c) the flat OR `a | b | c` at level 2, as a bracket;
  (d) the count of (a) (sdbg_match_count_batch_groups_min);
  (e) `3 of (a | b | c | d | e | f)` (the legacy window kernel) at levels 0 and 2;
checks that (a) and (b) return identical hits, as do the two levels of (e), and that (d) equals the level-0 totals of (a),
and prints the GPU name and power limit read in the same run. --only b times (b) alone.

    python tools/minmatch_bench.py [--steps 10] [--warmup 2] [--docs 10000000] [--queries 4096] [--only b]
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


def make_min_queries(n):
    """bench.make_queries' pairs extended to six distinct terms: the `2 of (a | b | c)` groups, the `3 of 6` groups and
    the flat `a | b | c`."""
    rng = np.random.default_rng(20261016)
    three, six, flat_or = [], [], []
    for q in bench.make_queries(n):
        ids = [int(q[0]), int(q[1])]
        while len(ids) < 6:
            t = int(rng.integers(0, bench.N_TERMS))
            if t not in ids:
                ids.append(t)
        three.append([ids[:3]])
        six.append([ids])
        flat_or.append(ids[:3])
    return three, six, flat_or


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=4096)
    ap.add_argument("--only", choices=["b"], default=None)
    args = ap.parse_args()

    ctx = sdb.Context(0)
    seg = sdb.Segment(ctx, args.docs)
    dc, sum_dl = seg.synth_corpus(0, 0, bench.N_TERMS, threads=min(os.cpu_count() or 1, 64))
    reader = sdb.IndexReader([seg], args.docs, sum_dl, dc)
    three, six, flat_or = make_min_queries(args.queries)
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
    nq = len(three)
    segs = _seg_array(reader.segments)

    def prepared(queries, m):
        ids, group_off, qgo = _groups(queries)
        terms = (N.BM25Term * len(ids))(*[reader.stats(scorer, t) for t in ids])
        gmin = np.full(len(queries), m, np.uint32)
        return ids, group_off, qgo, terms, gmin

    hits, n_out, total = np.zeros((nq, k), HIT_DTYPE), np.zeros(nq, np.uint32), np.zeros(nq, np.uint64)
    counts = np.zeros(nq, np.uint64)

    def topk(p):
        _, group_off, qgo, terms, gmin = p
        def run():
            N.check(N.lib().sdbg_bm25_topk_batch_groups_min(segs, 1, terms, _ptr(group_off), _ptr(qgo), _ptr(gmin), nq, None, None,
                                                            scorer.k, scorer.b, None, k, sdb.FLT_MIN, _ptr(hits), _ptr(n_out),
                                                            _ptr(total)), ctx._h)
            return hits, n_out, total
        return run

    p3, p6 = prepared(three, 2), prepared(six, 3)
    flat3 = np.ascontiguousarray(p3[0], np.uint32)

    def run_count():
        N.check(N.lib().sdbg_match_count_batch_groups_min(segs, 1, _ptr(flat3), _ptr(p3[1]), _ptr(p3[2]), _ptr(p3[4]), nq, None, None,
                                                          None, _ptr(counts)), ctx._h)
        return (counts,)

    if args.only == "b":
        b = timed(topk(p3), 2)
        print(json.dumps({"gpu": gpu_info(), "b_2of3_level2_ms": round(b[0], 3), "b_std": round(b[1], 3),
                          "matches": int(b[2][2].sum()), "steps": args.steps}))
        return
    a = timed(topk(p3), 0)
    b = timed(topk(p3), 2)
    c = timed(sdb.PreparedBatch(reader, flat_or, sdb.OR, scorer, k).run_host, 2)
    d = timed(run_count, 2)
    e0 = timed(topk(p6), 0)
    e2 = timed(topk(p6), 2)
    same = lambda x, y: bool(np.array_equal(x[1], y[1]) and all(np.array_equal(x[0][q, :x[1][q]], y[0][q, :y[1][q]]) for q in range(nq)))
    ab_same, e_same = same(a[2], b[2]), same(e0[2], e2[2])
    counts_ok = bool(np.array_equal(d[2][0], a[2][2]))
    ctx.set_wand(2)
    print(json.dumps({
        "gpu": gpu_info(),
        "workload": "%d docs, %d queries, top-%d" % (args.docs, nq, k),
        "a_2of3_level0_ms": round(a[0], 3), "a_std": round(a[1], 3),
        "b_2of3_level2_ms": round(b[0], 3), "b_std": round(b[1], 3),
        "c_flat_or_abc_level2_ms": round(c[0], 3), "c_std": round(c[1], 3),
        "d_2of3_count_ms": round(d[0], 3), "d_std": round(d[1], 3),
        "e_3of6_level0_ms": round(e0[0], 3), "e0_std": round(e0[1], 3),
        "e_3of6_level2_ms": round(e2[0], 3), "e2_std": round(e2[1], 3),
        "a_equals_b_hits": ab_same, "e_levels_equal_hits": e_same, "count_equals_level0_totals": counts_ok,
        "matches_2of3": int(a[2][2].sum()), "matches_3of6": int(e0[2][2].sum()), "steps": args.steps,
    }))
    if not (ab_same and e_same and counts_ok):
        sys.exit(1)


if __name__ == "__main__":
    main()
