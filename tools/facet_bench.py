"""Facet counts (`SELECT col, count(*) ... WHERE body @@ '...' GROUP BY col`, sdbg_match_facet_counts_batch) on bench.py's
10 M-doc corpus with its 4096 two-term disjunctions (bench.make_queries), in two workloads:
  (a) GROUP BY v = h % 2001 - 1000 (synth_column kind 3: 2001 keys, bit-packed);
  (b) GROUP BY a 16-key int64 column staged from a fixed seed: every match lands in one of 16 bins, the hot-bin case of
      the shared-memory histogram;
next to
  (c) sdbg_match_count_batch of the same batch: the bitmap work without the key reads and bin atomics;
  (d) the route callers had before, per query on the first 64 queries: sdbg_bm25_scan (StreamScoredDocs) of every match,
      sdbg_gather_column of the key column and np.bincount on the host.
Times are ms per step (CUDA events on the library's stream, L2 flushed before every step, after warm-up; (d) is host
wall time around synchronous calls). Exits non-zero unless, for every query, sum(counts) + nulls equals the count and
the sampled queries' counts equal (d)'s. Prints the GPU name and power limit read in the same run.

    python tools/facet_bench.py [--steps 10] [--warmup 2] [--docs 10000000] [--queries 4096]
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
from serenedb_b200.engine import _ptr, _seg_array  # noqa: E402
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
    seg.synth_column(1, 13, 3, 1, args.docs)                                                  # v: 2001 keys
    seg.stage_column(2, np.random.default_rng(16).integers(0, 16, args.docs).astype(np.int64))   # 16 keys
    reader = sdb.IndexReader([seg], args.docs, sum_dl, dc)
    queries = bench.make_queries(args.queries)
    segs, nq = _seg_array(reader.segments), len(queries)
    flat = np.ascontiguousarray([t for q in queries for t in q], dtype=np.uint32)
    off = np.zeros(nq + 1, np.uint32)
    off[1:] = np.cumsum([len(q) for q in queries])
    counts = np.zeros(nq, np.uint64)

    def facet(field, key_min, span, out, nulls):
        def run():   # arguments marshalled once, like PreparedBatch
            N.check(N.lib().sdbg_match_facet_counts_batch(segs, 1, sdb.OR, _ptr(flat), _ptr(off), nq, None, None, None, field,
                                                          key_min, span, _ptr(out), _ptr(nulls)), ctx._h)
        return run

    def count():
        N.check(N.lib().sdbg_match_count_batch(segs, 1, sdb.OR, _ptr(flat), _ptr(off), nq, None, None, None, _ptr(counts)),
                ctx._h)

    count()
    c = timed(ctx, count, args.steps, args.warmup)
    ok = True
    out = {"gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup,
           "workload": "%d docs, %d two-term OR queries (bench.make_queries)" % (args.docs, nq),
           "c_count_ms": c[0], "c_std": c[1]}
    sample_docs = [sdb.StreamScoredDocs(reader, 0, queries[q], sdb.OR, sdb.BM25())[0] for q in range(SAMPLE)]
    for name, field, key_min, span in (("a_2001_keys", 1, -1000, 2001), ("b_16_keys", 2, 0, 16)):
        fc = np.zeros((nq, span), np.uint64)
        fn = np.zeros(nq, np.uint64)
        run = facet(field, key_min, span, fc, fn)
        t = timed(ctx, run, args.steps, args.warmup)
        fc[:] = 0
        run()
        w = {"ms": t[0], "std": t[1]}
        ok &= bool(np.array_equal(fc.sum(axis=1) + fn, counts))
        # (d) per query: stream every match, gather the key column, count on the host
        t0 = time.perf_counter()
        for q in range(SAMPLE):
            docs, _ = sdb.StreamScoredDocs(reader, 0, queries[q], sdb.OR, sdb.BM25())
            vals, valid = seg.gather(field, docs, np.int64)
            host = np.bincount(vals[valid] - key_min, minlength=span)
            ok &= bool(np.array_equal(host, fc[q]) and np.array_equal(docs, sample_docs[q]) and valid.all())
        w["d_host_route_ms_per_query"] = round((time.perf_counter() - t0) * 1000 / SAMPLE, 3)
        out[name] = w
    out["equal"] = ok
    print(json.dumps(out))
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
