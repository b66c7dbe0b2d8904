"""Aggregates over the matches (`SELECT [col,] count(*), count(v), sum(v), avg(v), min(v), max(v) ... WHERE body @@ '...'
[GROUP BY col]`, sdbg_match_aggregate_batch) on bench.py's 10 M-doc corpus with its 4096 two-term disjunctions
(bench.make_queries):
  (a) ungrouped, v = the bit-packed int64 column h % 2001 - 1000 (synth_column kind 3);
  (b) ungrouped, v = a float64 column (synth_column kind 4);
  (c) the float64 column GROUP BY the 2001-key column;
  (d) the float64 column GROUP BY a 16-key int64 column staged from a fixed seed (hot cells);
next to
  (e) the facet pass of the same batch on the 2001 and the 16 keys (sdbg_match_facet_counts_batch);
  (f) sdbg_match_count_batch: the bitmap work alone, the floor;
  (g) the host route per query on the first 64 queries: sdbg_bm25_scan (StreamScoredDocs) of every match,
      sdbg_gather_column of the value column and NumPy's sum / min / max.
Times are ms per step (CUDA events on the library's stream, L2 flushed before every step, after warm-up; (g) is host
wall time around synchronous calls). Exits non-zero unless every query's counts equal the count and the facet counts, and
the sampled queries' integer sums, minima and maxima equal (g)'s. Prints the GPU name and power limit read in the same
run.

    python tools/agg_bench.py [--steps 10] [--warmup 2] [--docs 10000000] [--queries 4096]
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

import bench  # noqa: E402  (make_queries, N_TERMS: the benchmark's own workload)
import serenedb_b200 as sdb  # noqa: E402
from serenedb_b200 import _native as N  # noqa: E402
from serenedb_b200.engine import MATCH_AGG_DTYPE, _ptr, _seg_array  # noqa: E402
from count_bench import gpu_info, timed  # noqa: E402

SAMPLE = 64


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
    seg.synth_column(1, 13, 3, 1, args.docs)                                                  # 2001 keys, bit-packed
    seg.stage_column(2, np.random.default_rng(16).integers(0, 16, args.docs).astype(np.int64))   # 16 keys
    seg.synth_column(3, 14, 4, 1, args.docs)                                                  # float64
    reader = sdb.IndexReader([seg], args.docs, sum_dl, dc)
    queries = bench.make_queries(args.queries)
    segs, nq = _seg_array(reader.segments), len(queries)
    flat = np.ascontiguousarray([t for q in queries for t in q], dtype=np.uint32)
    off = np.zeros(nq + 1, np.uint32)
    off[1:] = np.cumsum([len(q) for q in queries])
    counts = np.zeros(nq, np.uint64)

    def count():
        N.check(N.lib().sdbg_match_count_batch(segs, 1, sdb.OR, _ptr(flat), _ptr(off), nq, None, None, None, _ptr(counts)),
                ctx._h)

    def facet(field, key_min, span, out, nulls):
        def run():   # arguments marshalled once, like PreparedBatch
            N.check(N.lib().sdbg_match_facet_counts_batch(segs, 1, sdb.OR, _ptr(flat), _ptr(off), nq, None, None, None, field,
                                                          key_min, span, _ptr(out), _ptr(nulls)), ctx._h)
        return run

    def agg(key_field, key_min, span, value_field, out, nulls):
        def run():
            N.check(N.lib().sdbg_match_aggregate_batch(segs, 1, sdb.OR, _ptr(flat), _ptr(off), nq, None, None, None, key_field,
                                                       key_min, span, value_field, _ptr(out), _ptr(nulls)), ctx._h)
        return run

    count()
    c = timed(ctx, count, args.steps, args.warmup)
    ok = True
    out = {"gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup,
           "workload": "%d docs, %d two-term OR queries (bench.make_queries)" % (args.docs, nq),
           "f_count_ms": c[0], "f_std": c[1]}
    facet_counts = {}
    for name, field, key_min, span in (("e_facet_2001_keys", 1, -1000, 2001), ("e_facet_16_keys", 2, 0, 16)):
        fc = np.zeros((nq, span), np.uint64)
        fn = np.zeros(nq, np.uint64)
        run = facet(field, key_min, span, fc, fn)
        t = timed(ctx, run, args.steps, args.warmup)
        run()
        facet_counts[field] = fc.copy()
        out[name] = {"ms": t[0], "std": t[1]}
    results = {}
    for name, kf, key_min, span, vf in (("a_ungrouped_int64_packed", N.UINT64_MAX, 0, 1, 1),
                                        ("b_ungrouped_float64", N.UINT64_MAX, 0, 1, 3),
                                        ("c_float64_by_2001_keys", 1, -1000, 2001, 3),
                                        ("d_float64_by_16_keys", 2, 0, 16, 3)):
        cells = np.zeros((nq, span), MATCH_AGG_DTYPE)
        nulls = np.zeros(nq, MATCH_AGG_DTYPE)
        run = agg(kf, key_min, span, vf, cells, nulls)
        t = timed(ctx, run, args.steps, args.warmup)
        cells[:] = 0
        run()
        results[name] = cells.copy()
        ok &= bool(np.array_equal(cells["count"].sum(axis=1), counts) and not nulls["count"].any())
        if kf != N.UINT64_MAX:
            ok &= bool(np.array_equal(cells["count"], facet_counts[kf]))
        out[name] = {"ms": t[0], "std": t[1]}
    # (g) per query: stream every match, gather the value column, aggregate on the host
    for name, vf, dtype in (("g_host_route_int64_ms_per_query", 1, np.int64), ("g_host_route_float64_ms_per_query", 3, np.float64)):
        t0 = time.perf_counter()
        host = []
        for q in range(SAMPLE):
            docs, _ = sdb.StreamScoredDocs(reader, 0, queries[q], sdb.OR, sdb.BM25())
            vals, valid = seg.gather(vf, docs, dtype)
            v = vals[valid]
            host.append((len(docs), int(v.astype(object).sum()) if dtype == np.int64 else float(v.sum()), v.min(), v.max()))
        out[name] = round((time.perf_counter() - t0) * 1000 / SAMPLE, 3)
        cells = results["a_ungrouped_int64_packed" if dtype == np.int64 else "b_ungrouped_float64"][:, 0]
        for q, (n, s, mn, mx) in enumerate(host):
            if dtype == np.int64:
                gs = (int(cells["sum_hi"][q]) << 64) | (int(cells["sum_lo"][q]) & 0xFFFFFFFFFFFFFFFF)
                ok &= bool(cells["count"][q] == n and gs == s and cells["min"][q] == mn and cells["max"][q] == mx)
            else:
                ok &= bool(cells["count"][q] == n and abs(cells["sum_f64"][q] - s) <= 1e-9 * max(1.0, abs(s)) * n and
                           cells["min"][q:q + 1].view(np.float64)[0] == mn and cells["max"][q:q + 1].view(np.float64)[0] == mx)
    out["equal"] = ok
    print(json.dumps(out))
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
