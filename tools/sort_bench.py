"""Sorted scan (`WHERE body @@ '...' ORDER BY col LIMIT 1000`, sdbg_match_topk_by_column_batch) on bench.py's 10 M-doc
corpus with its 4096 two-term disjunctions (bench.make_queries), top-1000, in two workloads:
  (a) ORDER BY a uniform int64 column (synth_column kind 1) ASC;
  (b) ORDER BY the clustered ts = row / 100 (kind 7) DESC ("newest first").
Each is timed at pruning level 0 and 2, next to
  (c) sdbg_match_count_batch of the same batch: the bitmap work without the column gather;
  (d) the route callers had before, per query on the first 64 queries: sdbg_bm25_scan (StreamScoredDocs) of every match,
      sdbg_gather_column of the sort column and a host sort.
Times are ms per step (CUDA events on the library's stream, L2 flushed before every step, after warm-up; (d) is host
wall time around synchronous calls). Also reported: windows judged / skipped by the zonemap (sdbg_scan_stats), and the
32-byte sectors of the sort column holding the 64 sampled queries' matches, so times can be read against bytes. Exits
non-zero unless the sampled hits equal (d)'s and n_out equals min(k, count) for every query. Prints the GPU name and
power limit read in the same run.

    python tools/sort_bench.py [--steps 10] [--warmup 2] [--docs 10000000] [--queries 4096]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402  (make_queries, N_TERMS, TOPK: the benchmark's own workload)
import serenedb_b200 as sdb  # noqa: E402
from serenedb_b200 import _native as N  # noqa: E402
from serenedb_b200.engine import SORT_HIT_DTYPE, _ptr, _seg_array  # noqa: E402
from count_bench import gpu_info, timed  # noqa: E402

SAMPLE = 64


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
    threads = min(os.cpu_count() or 1, 64)
    k = bench.TOPK

    ctx = sdb.Context(0)
    seg = sdb.Segment(ctx, args.docs)
    dc, sum_dl = seg.synth_corpus(0, 0, bench.N_TERMS, threads=threads)
    seg.synth_column(1, 11, 1, 1, args.docs)   # uniform
    seg.synth_column(2, 12, 7, 1, args.docs)   # ts = row / 100
    reader = sdb.IndexReader([seg], args.docs, sum_dl, dc)
    queries = bench.make_queries(args.queries)
    segs, nq = _seg_array(reader.segments), len(queries)
    flat = np.ascontiguousarray([t for q in queries for t in q], dtype=np.uint32)
    off = np.zeros(nq + 1, np.uint32)
    off[1:] = np.cumsum([len(q) for q in queries])
    hits = np.zeros(nq * k, SORT_HIT_DTYPE)
    n_out = np.zeros(nq, np.uint32)
    counts = np.zeros(nq, np.uint64)

    def sorted_scan(field, desc):
        def run():   # arguments marshalled once, like PreparedBatch
            N.check(N.lib().sdbg_match_topk_by_column_batch(segs, 1, sdb.OR, _ptr(flat), _ptr(off), nq, None, None, None, field,
                                                            int(desc), 0, k, _ptr(hits), _ptr(n_out)), ctx._h)
        return run

    def count():
        N.check(N.lib().sdbg_match_count_batch(segs, 1, sdb.OR, _ptr(flat), _ptr(off), nq, None, None, None, _ptr(counts)),
                ctx._h)

    count()
    c = timed(ctx, count, args.steps, args.warmup)
    ok = True
    out = {"gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup,
           "workload": "%d docs, %d two-term OR queries (bench.make_queries), top-%d" % (args.docs, nq, k),
           "c_count_ms": c[0], "c_std": c[1]}
    # the sort column's 32-byte sectors holding the sampled queries' matches (row = doc - 1, 8-byte values)
    sample_docs = [sdb.StreamScoredDocs(reader, 0, queries[q], sdb.OR, sdb.BM25())[0] for q in range(SAMPLE)]
    out["sample_sectors"] = int(sum(len(np.unique((d.astype(np.int64) - 1) * 8 // 32)) for d in sample_docs))
    out["sample_matches"] = int(sum(len(d) for d in sample_docs))
    for name, field, desc in (("a_uniform_asc", 1, False), ("b_clustered_ts_desc", 2, True)):
        w = {}
        for level in (0, 2):
            ctx.set_wand(level)
            t = timed(ctx, sorted_scan(field, desc), args.steps, args.warmup)
            sorted_scan(field, desc)()
            judged, skipped = scan_stats(ctx)
            w["level%d_ms" % level], w["level%d_std" % level] = t
            w["level%d_windows_judged" % level], w["level%d_windows_skipped" % level] = judged, skipped
            ok &= bool(np.array_equal(n_out, np.minimum(counts, k)))
            # (d) per query: stream every match, gather the column, sort on the host
            t0 = time.perf_counter()
            for q in range(SAMPLE):
                docs, _ = sdb.StreamScoredDocs(reader, 0, queries[q], sdb.OR, sdb.BM25())
                vals, _ = seg.gather(field, docs, np.int64)
                o = np.lexsort((docs, -vals if desc else vals))[:k]
                h = hits[q * k:q * k + int(n_out[q])]
                ok &= bool(np.array_equal(h["doc"], docs[o]) and np.array_equal(h["value"], vals[o]))
            w["d_host_route_ms_per_query"] = round((time.perf_counter() - t0) * 1000 / SAMPLE, 3)
        out[name] = w
    ctx.set_wand(2)
    out["equal"] = ok
    print(json.dumps(out))
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
