"""Sorted scan and facet counts of group queries (sdbg_match_topk_by_column_batch_groups_min /
sdbg_match_facet_counts_batch_groups_min) on bench.py's 10 M-doc corpus, 4096 queries of two forms:
  `2 of (a | b | c)` (minmatch_bench.make_min_queries) and `a & (b | c)` (groups_bench.make_group_queries).
For each form:
  sort_uniform_asc        ORDER BY a uniform int64 column (synth_column kind 1) ASC, top-1000, at pruning levels 0 and 2;
  sort_clustered_desc     ORDER BY the clustered ts = row / 100 (kind 7) DESC ("newest first"), top-1000, levels 0 and 2;
  facet_2001 / facet_16   GROUP BY the 2001-key column (kind 3) / facet_bench's 16-key column;
each next to the grouped count of the same batch (sdbg_match_count_batch_groups_min: the floor, no column read) and the
flat `a | b | c` sort / facet of the same column (sdbg_match_topk_by_column_batch / sdbg_match_facet_counts_batch).
Times are ms per step (CUDA events on the library's stream, L2 flushed before every step, after warm-up; mean and std).
Also reported: windows judged / skipped by the zonemap (sdbg_scan_stats) per sorted run. Exits non-zero unless
n_out == min(k, count) and sum(counts) + nulls == count for every query. Prints the GPU name and power limit read in the
same run.

    python tools/groups_column_bench.py [--steps 10] [--warmup 2] [--docs 10000000] [--queries 4096]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  (N_TERMS, TOPK: the benchmark's own workload)
import serenedb_b200 as sdb  # noqa: E402
from serenedb_b200 import _native as N  # noqa: E402
from serenedb_b200.engine import SORT_HIT_DTYPE, _groups, _ptr, _seg_array  # noqa: E402
from count_bench import gpu_info, timed  # noqa: E402
from groups_bench import make_group_queries  # noqa: E402
from minmatch_bench import make_min_queries  # noqa: E402

# facet key field -> (key_min, key_span); the columns are those of sort_bench / facet_bench
COLUMNS = {3: (-1000, 2001), 4: (0, 16)}


def scan_stats(ctx):
    t, s = C.c_uint64(), C.c_uint64()
    N.check(N.lib().sdbg_scan_stats(ctx._h, C.byref(t), C.byref(s)))
    return t.value, s.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=4096)
    args = ap.parse_args()
    k = bench.TOPK

    ctx = sdb.Context(0)
    seg = sdb.Segment(ctx, args.docs)
    dc, sum_dl = seg.synth_corpus(0, 0, bench.N_TERMS, threads=min(os.cpu_count() or 1, 64))
    seg.synth_column(1, 11, 1, 1, args.docs)                                                  # uniform (sort_bench)
    seg.synth_column(2, 12, 7, 1, args.docs)                                                  # ts = row / 100
    seg.synth_column(3, 13, 3, 1, args.docs)                                                  # 2001 keys (facet_bench)
    seg.stage_column(4, np.random.default_rng(16).integers(0, 16, args.docs).astype(np.int64))   # 16 keys
    reader = sdb.IndexReader([seg], args.docs, sum_dl, dc)
    segs = _seg_array(reader.segments)
    three, _, flat3 = make_min_queries(args.queries)
    grouped, flat_or, _ = make_group_queries(args.queries)
    forms = {"two_of_three": (three, [[2]] * len(three), flat3), "a_and_b_or_c": (grouped, None, flat_or)}

    out = {"gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup,
           "workload": "%d docs, %d queries per form, top-%d" % (args.docs, args.queries, k)}
    ok = True
    for name, (queries, mins, flat) in forms.items():
        nq = len(queries)
        ids, group_off, qgo = _groups(queries)
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        gmin = np.ascontiguousarray([v for m in mins for v in m], dtype=np.uint32) if mins else None
        fl = np.ascontiguousarray([t for q in flat for t in q], dtype=np.uint32)
        off = np.zeros(nq + 1, np.uint32)
        off[1:] = np.cumsum([len(q) for q in flat])
        hits = np.zeros(nq * k, SORT_HIT_DTYPE)
        n_out = np.zeros(nq, np.uint32)
        counts = np.zeros(nq, np.uint64)
        fcounts = np.zeros(nq * 2001, np.uint64)
        nulls = np.zeros(nq, np.uint64)
        gp = _ptr(gmin) if gmin is not None else None

        def count():   # arguments marshalled once, like PreparedBatch
            N.check(N.lib().sdbg_match_count_batch_groups_min(segs, 1, _ptr(ids), _ptr(group_off), _ptr(qgo), gp, nq, None,
                                                              None, None, _ptr(counts)), ctx._h)

        def sort(field, desc, grp=True):
            if grp:
                return lambda: N.check(N.lib().sdbg_match_topk_by_column_batch_groups_min(
                    segs, 1, _ptr(ids), _ptr(group_off), _ptr(qgo), gp, nq, None, None, None, field, int(desc), 0, k,
                    _ptr(hits), _ptr(n_out)), ctx._h)
            return lambda: N.check(N.lib().sdbg_match_topk_by_column_batch(segs, 1, sdb.OR, _ptr(fl), _ptr(off), nq, None,
                                                                           None, None, field, int(desc), 0, k, _ptr(hits),
                                                                           _ptr(n_out)), ctx._h)

        def facet(field, grp=True):
            key_min, span = COLUMNS[field]
            if grp:
                return lambda: N.check(N.lib().sdbg_match_facet_counts_batch_groups_min(
                    segs, 1, _ptr(ids), _ptr(group_off), _ptr(qgo), gp, nq, None, None, None, field, key_min, span,
                    _ptr(fcounts), _ptr(nulls)), ctx._h)
            return lambda: N.check(N.lib().sdbg_match_facet_counts_batch(segs, 1, sdb.OR, _ptr(fl), _ptr(off), nq, None, None,
                                                                         None, field, key_min, span, _ptr(fcounts),
                                                                         _ptr(nulls)), ctx._h)

        ctx.set_wand(0)
        count()
        c = counts.copy()
        w = {"count_groups_ms": timed(ctx, count, args.steps, args.warmup)}
        for run, field, desc in (("sort_uniform_asc", 1, False), ("sort_clustered_desc", 2, True)):
            r = {}
            for level in (0, 2):
                ctx.set_wand(level)
                r["groups_level%d_ms" % level] = timed(ctx, sort(field, desc), args.steps, args.warmup)
                sort(field, desc)()
                r["groups_level%d_windows_judged_skipped" % level] = scan_stats(ctx)
                ok &= bool(np.array_equal(n_out, np.minimum(c, k)))
                r["flat_or_level%d_ms" % level] = timed(ctx, sort(field, desc, False), args.steps, args.warmup)
                sort(field, desc, False)()
                r["flat_or_level%d_windows_judged_skipped" % level] = scan_stats(ctx)
            w[run] = r
        ctx.set_wand(0)
        for run, field in (("facet_2001", 3), ("facet_16", 4)):
            span = COLUMNS[field][1]
            w[run] = {"groups_ms": timed(ctx, facet(field), args.steps, args.warmup)}
            facet(field)()
            ok &= bool(np.array_equal(fcounts[:nq * span].reshape(nq, span).sum(axis=1) + nulls, c))
            w[run]["flat_or_ms"] = timed(ctx, facet(field, False), args.steps, args.warmup)
        out[name] = w
    ctx.set_wand(2)
    out["invariants_hold"] = ok
    print(json.dumps(out))
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
