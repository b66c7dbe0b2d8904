"""Per-call latency of the synchronous count, facet, aggregate, sorted-scan and BM25 top-k entries: the host clock around each call
(every call ends with its one stream synchronisation), median over --calls calls after warm-up. The batch benchmarks time
4096 queries per step, which hides per-call costs (plan staging, the copy back, the single-term shortcut); this times
the small batches where those costs show:
  shortcut   sdbg_match_count_batch of one single-term query, answered from docs_count without a launch;
  nq = 1 / 64 two-term ORs (bench.make_queries) for count, facet (2001 keys), aggregate (ungrouped, bit-packed int64)
             and the sorted scan (k = 100);
  mixed      a 64-query group batch of all three shapes (one group, single-term groups, true groups) for count, facet,
             the sorted scan and the top-k;
  topk       sdbg_bm25_topk_batch (BM25, k = 100) of nq = 1 / 64 two-term ORs, and sdbg_topk_merge_gathered of 4096 x 1000
             keys (one rank's sdbg_bm25_topk_batch_device output) to host hits.
Prints one JSON line with microseconds per call and the GPU name and power limit read in the same run.

    python tools/pass_latency.py [--calls 200] [--docs 10000000]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
import serenedb_b200 as sdb  # noqa: E402
from serenedb_b200 import _native as N  # noqa: E402
from serenedb_b200.engine import FLT_MIN, PreparedBatch, _ptr, _query_args, _seg_array, merge_gathered  # noqa: E402
from count_bench import gpu_info  # noqa: E402

K = 100


def median_us(fn, calls):
    for _ in range(10):
        fn()
    t = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return round(float(np.median(t)) * 1e6, 1)


def flat_batch(queries):
    terms = np.ascontiguousarray([t for q in queries for t in q], dtype=np.uint32)
    off = np.zeros(len(queries) + 1, np.uint32)
    off[1:] = np.cumsum([len(q) for q in queries])
    return terms, off


def group_batch(queries):   # queries: lists of groups
    groups = [g for q in queries for g in q]
    terms = np.ascontiguousarray([t for g in groups for t in g], dtype=np.uint32)
    goff = np.zeros(len(groups) + 1, np.uint32)
    goff[1:] = np.cumsum([len(g) for g in groups])
    qoff = np.zeros(len(queries) + 1, np.uint32)
    qoff[1:] = np.cumsum([len(q) for q in queries])
    return terms, goff, qoff


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--docs", type=int, default=10_000_000)
    args = ap.parse_args()
    threads = min(os.cpu_count() or 1, 64)
    ctx = sdb.Context(0)
    seg = sdb.Segment(ctx, args.docs)
    dc, sum_dl = seg.synth_corpus(0, 0, bench.N_TERMS, threads=threads)
    seg.synth_column(1, 13, 3, 1, args.docs)   # 2001 keys in [-1000, 1000], bit-packed int64
    reader = sdb.IndexReader([seg], args.docs, sum_dl, dc)
    segs = _seg_array(reader.segments)
    lib = N.lib()
    out = {"gpu": gpu_info(), "calls": args.calls, "docs": args.docs, "us_per_call": {}}
    res = out["us_per_call"]

    def entries(tag, nq, terms, off, groups=None):
        counts = np.zeros(nq, np.uint64)
        fc, fn = np.zeros(nq * 2001, np.uint64), np.zeros(nq, np.uint64)
        agg = np.zeros(nq * 56, np.uint8)   # sizeof(sdbg_match_agg)
        nagg = np.zeros(nq * 56, np.uint8)
        hits, n_out = np.zeros(nq * K * 24, np.uint8), np.zeros(nq, np.uint32)
        if groups is None:
            q = (segs, 1, sdb.OR, _ptr(terms), _ptr(off), nq, None, None, None)
            calls = {"count": lambda: lib.sdbg_match_count_batch(*q, _ptr(counts)),
                     "facet": lambda: lib.sdbg_match_facet_counts_batch(*q, 1, -1000, 2001, _ptr(fc), _ptr(fn)),
                     "aggregate": lambda: lib.sdbg_match_aggregate_batch(*q, 2**64 - 1, 0, 1, 1, _ptr(agg), _ptr(nagg)),
                     "sort": lambda: lib.sdbg_match_topk_by_column_batch(*q, 1, 1, 0, K, _ptr(hits), _ptr(n_out))}
        else:
            goff, qoff = groups
            q = (segs, 1, _ptr(terms), _ptr(goff), _ptr(qoff), None, nq, None, None, None)
            calls = {"count": lambda: lib.sdbg_match_count_batch_groups_min(*q, _ptr(counts)),
                     "facet": lambda: lib.sdbg_match_facet_counts_batch_groups_min(*q, 1, -1000, 2001, _ptr(fc), _ptr(fn)),
                     "sort": lambda: lib.sdbg_match_topk_by_column_batch_groups_min(*q, 1, 1, 0, K, _ptr(hits), _ptr(n_out))}
        for name, fn_ in calls.items():
            run = (lambda f: lambda: N.check(f(), ctx._h))(fn_)
            res["%s_%s" % (tag, name)] = median_us(run, args.calls)

    terms, off = flat_batch([[7]])
    before = ctx.launches
    res["shortcut_count"] = median_us(lambda: N.check(lib.sdbg_match_count_batch(segs, 1, sdb.OR, _ptr(terms), _ptr(off), 1, None,
                                                                                 None, None, _ptr(np.zeros(1, np.uint64))), ctx._h),
                                      args.calls)
    out["shortcut_launches"] = ctx.launches - before
    queries = bench.make_queries(64)
    for nq in (1, 64):
        terms, off = flat_batch(queries[:nq])
        entries("or_nq%d" % nq, nq, terms, off)
    mixed = []
    for i, (a, b) in enumerate(queries):
        c = next(t for t in range(bench.N_TERMS) if t not in (a, b))
        mixed.append([[a, b]] if i % 3 == 0 else [[a], [b]] if i % 3 == 1 else [[a, b], [c]])
    terms, goff, qoff = group_batch(mixed)
    entries("mixed_nq64", len(mixed), terms, None, (goff, qoff))

    scorer = sdb.BM25()
    for nq in (1, 64):
        res["topk_or_nq%d" % nq] = median_us(PreparedBatch(reader, queries[:nq], sdb.OR, scorer, K).run_host, args.calls)
    gargs = _query_args(mixed, None, groups=True, stats=lambda t: reader.stats(scorer, t))
    hits, n_out, total = np.zeros(len(mixed) * K * 12, np.uint8), np.zeros(len(mixed), np.uint32), np.zeros(len(mixed), np.uint64)
    res["topk_mixed_nq64"] = median_us(lambda: N.check(lib.sdbg_bm25_topk_batch_groups_min(
        segs, 1, *gargs, scorer.k, scorer.b, None, K, FLT_MIN, _ptr(hits), _ptr(n_out), _ptr(total)), ctx._h), args.calls)
    import torch
    nq, k = 4096, 1000
    d_keys = torch.zeros(nq * k, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    PreparedBatch(reader, bench.make_queries(nq), sdb.OR, scorer, k).run_device(0, d_keys.data_ptr())
    res["topk_merge_4096x1000_to_host"] = median_us(lambda: merge_gathered(ctx, d_keys.data_ptr(), 1, nq, k),
                                                    max(args.calls // 10, 5))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
