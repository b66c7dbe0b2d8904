"""The count, facet, aggregate and sorted-scan passes across GPUs (sdbg_dist_match_*_batch_groups_min) on one H100: bench.py's 10 M-doc
corpus cut by doc range into R shards (R in 1, 2, 8; each shard its own segment, as each rank would hold it) with its
4096 two-term disjunctions (bench.make_queries, run as one-group queries). Reports, in ms per step (CUDA events on the
library's stream, L2 flushed before every step, after warm-up):
  (a) the local entries over the unsharded corpus: count, facet counts on 2001 keys, aggregates of a float64 column
      ungrouped / by 16 keys / by 2001 keys;
  (b) per R, the device-form passes of every shard (what each rank runs before its collective): the slowest shard and the
      sum over shards; the dist entries at R = 1 without a communicator (the all-reduce a no-op, the all-gather a copy);
  (c) the aggregate merge kernel alone at R = 8 (torch.profiler, CUDA activities), with the gathered bytes it reads and
      the rate that implies, and the whole merge call (kernel, copy back, conversion);
  (d) the sorted scan (ORDER BY the float64 column DESC LIMIT 1000): the local entry, the device forms per shard, and at
      R = 8 the sorted merge kernel alone and the whole merge call, with the gathered bytes.
The NCCL collectives and the scaling across GPUs are not measured here: one GPU. Exits non-zero unless the merged counts
equal the unsharded ones and the merged sorted hits' values equal the unsharded scan's. Prints the GPU name and power
limit read in the same run.

    python tools/dist_match_bench.py [--steps 10] [--warmup 2] [--docs 10000000] [--queries 4096]
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

import bench  # noqa: E402  (make_queries, N_TERMS: the benchmark's own workload)
import serenedb_b200 as sdb  # noqa: E402
from serenedb_b200 import _native as N  # noqa: E402
from serenedb_b200.engine import MATCH_AGG_DTYPE, SORT_HIT_DTYPE, _ptr, _query_args, _seg_array  # noqa: E402
from count_bench import gpu_info, timed  # noqa: E402

AGGS = (("ungrouped", N.UINT64_MAX, 0, 1), ("16_keys", 2, 0, 16), ("2001_keys", 1, -1000, 2001))


def shard(ctx, doc0, n, threads):
    seg = sdb.Segment(ctx, n)
    dc, sum_dl = seg.synth_corpus(doc0, 0, bench.N_TERMS, threads=threads)
    seg.synth_column(1, 13, 3, doc0 + 1, n)                                                         # 2001 keys
    seg.stage_column(2, np.random.default_rng(16).integers(0, 16, doc0 + n)[doc0:].astype(np.int64))   # 16 keys
    seg.synth_column(3, 14, 4, doc0 + 1, n)                                                         # float64
    return seg, np.asarray(dc, np.uint64), sum_dl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=4096)
    args = ap.parse_args()
    threads = min(os.cpu_count() or 1, 64)
    import torch

    ctx = sdb.Context(0)
    whole, dc, sum_dl = shard(ctx, 0, args.docs, threads)
    queries = [[q] for q in bench.make_queries(args.queries)]
    nq = len(queries)
    qa = _query_args(queries, None, None, groups=True)
    out = {"gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup,
           "workload": "%d docs, %d two-term OR queries (bench.make_queries) as one-group queries" % (args.docs, nq),
           "collectives": "not measured (one GPU)"}
    ok = True

    def t(fn):
        m, s = timed(ctx, fn, args.steps, args.warmup)
        return {"ms": round(m, 3), "std": round(s, 3)}

    def segs_of(segs):
        return _seg_array(segs), len(segs)

    def count(segs, dist=False):
        sa, ns = segs_of(segs)
        res = np.zeros(nq, np.uint64)
        fn = N.lib().sdbg_dist_match_count_batch_groups_min if dist else N.lib().sdbg_match_count_batch_groups_min
        return lambda: N.check(fn(sa, ns, *qa, None, _ptr(res)), ctx._h), res

    def facet(segs, dist=False):
        sa, ns = segs_of(segs)
        res, nulls = np.zeros((nq, 2001), np.uint64), np.zeros(nq, np.uint64)
        fn = N.lib().sdbg_dist_match_facet_counts_batch_groups_min if dist else N.lib().sdbg_match_facet_counts_batch_groups_min
        return lambda: N.check(fn(sa, ns, *qa, None, 1, -1000, 2001, _ptr(res), _ptr(nulls)), ctx._h), res

    def agg(segs, kf, key_min, span, dist=False):
        sa, ns = segs_of(segs)
        res, nulls = np.zeros((nq, span), MATCH_AGG_DTYPE), np.zeros(nq, MATCH_AGG_DTYPE)
        fn = N.lib().sdbg_dist_match_aggregate_batch_groups_min if dist else N.lib().sdbg_match_aggregate_batch_groups_min
        return lambda: N.check(fn(sa, ns, *qa, None, kf, key_min, span, 3, _ptr(res), _ptr(nulls)), ctx._h), res

    def agg_device(segs, kf, key_min, span, d_ptr):
        sa, ns = segs_of(segs)
        return lambda: N.check(N.lib().sdbg_match_aggregate_batch_groups_min_device(sa, ns, *qa, None, kf, key_min, span, 3,
                                                                                     C.c_void_p(d_ptr)), ctx._h)

    def sort(segs, k=1000):
        sa, ns = segs_of(segs)
        hits, n = np.zeros(nq * k, SORT_HIT_DTYPE), np.zeros(nq, np.uint32)
        return lambda: N.check(N.lib().sdbg_match_topk_by_column_batch_groups_min(sa, ns, *qa, None, 3, 1, 0, k, _ptr(hits),
                                                                                   _ptr(n)), ctx._h), hits

    def sort_device(segs, rank, d_ptr, k=1000):
        sa, ns = segs_of(segs)
        return lambda: N.check(N.lib().sdbg_match_topk_by_column_batch_groups_min_device(sa, ns, *qa, None, 3, 1, 0, k, rank,
                                                                                          C.c_void_p(d_ptr)), ctx._h)

    def kernel_ms(fn, name):
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                fn()
            torch.cuda.synchronize()
        us = [e.device_time for e in prof.events() if name in e.name]
        return float(np.mean(us)) / 1000 if us else float("nan")

    # (a) local entries, unsharded
    run, counts = count([whole])
    out["a_local_count"] = t(run)
    run()
    run, fc = facet([whole])
    out["a_local_facet_2001_keys"] = t(run)
    for name, kf, key_min, span in AGGS:
        out["a_local_agg_" + name] = t(agg([whole], kf, key_min, span)[0])
    run, sort_hits = sort([whole])
    out["d_local_sort_k1000"] = t(run)
    run()
    # dist entries at R = 1 (no communicator)
    run, dcounts = count([whole], dist=True)
    out["b1_dist_count"] = t(run)
    run()
    ok &= bool(np.array_equal(dcounts, counts))
    run, dfc = facet([whole], dist=True)
    out["b1_dist_facet_2001_keys"] = t(run)
    run()
    ok &= bool(np.array_equal(dfc, fc))
    for name, kf, key_min, span in AGGS:
        out["b1_dist_agg_" + name] = t(agg([whole], kf, key_min, span, dist=True)[0])
    whole.close()

    for R in (2, 8):
        cuts = [i * args.docs // R for i in range(R + 1)]
        shards = [shard(ctx, a, b - a, threads)[0] for a, b in zip(cuts[:-1], cuts[1:])]
        res = {}
        total = np.zeros(nq, np.uint64)
        per = []
        for s in shards:
            run, c = count([s], dist=True)
            per.append(t(run)["ms"])
            run()
            total += c
        ok &= bool(np.array_equal(total, counts))
        res["count_device_form"] = {"max_shard_ms": max(per), "sum_ms": round(sum(per), 3)}
        for name, kf, key_min, span in AGGS:
            words = sdb.match_aggregate_device_bytes(nq, span) // 8
            buf = torch.zeros((R, words), dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            per = [t(agg_device([s], kf, key_min, span, buf[r].data_ptr()))["ms"] for r, s in enumerate(shards)]
            res["agg_device_form_" + name] = {"max_shard_ms": max(per), "sum_ms": round(sum(per), 3)}
            if R == 8:
                o, nl = np.zeros((nq, span), MATCH_AGG_DTYPE), np.zeros(nq, MATCH_AGG_DTYPE)
                merge = lambda: N.check(N.lib().sdbg_match_aggregate_merge_gathered(ctx._h, C.c_void_p(buf.data_ptr()), R, nq,
                                                                                    span, _ptr(o), _ptr(nl)), ctx._h)
                res["merge_call_" + name] = t(merge)
                ok &= bool(np.array_equal(o["count"].sum(axis=1) + nl["count"], counts))
                gathered = R * words * 8
                k_ms = kernel_ms(merge, "agg_merge_gathered_kernel")
                res["merge_kernel_" + name] = {"ms": round(k_ms, 4), "gathered_bytes": gathered,
                                               "GB_per_s": round(gathered / (k_ms * 1e6), 1)}
            del buf
        words = sdb.topk_by_column_device_bytes(nq, 1000) // 8
        buf = torch.zeros((R, words), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        per = [t(sort_device([s], r, buf[r].data_ptr()))["ms"] for r, s in enumerate(shards)]
        res["sort_device_form_k1000"] = {"max_shard_ms": max(per), "sum_ms": round(sum(per), 3)}
        if R == 8:
            hits, n = np.zeros(nq * 1000, SORT_HIT_DTYPE), np.zeros(nq, np.uint32)
            merge = lambda: N.check(N.lib().sdbg_match_topk_by_column_merge_gathered(ctx._h, C.c_void_p(buf.data_ptr()), R, nq,
                                                                                     1000, _ptr(hits), _ptr(n)), ctx._h)
            res["sort_merge_call_k1000"] = t(merge)
            ok &= bool(np.array_equal(hits["value"], sort_hits["value"]))
            res["sort_merge_kernel_k1000"] = {"ms": round(kernel_ms(merge, "sort_merge_gathered_kernel"), 4),
                                              "gathered_bytes": R * words * 8}
        del buf
        out["b%d" % R] = res
        for s in shards:
            s.close()
    out["equal"] = ok
    print(json.dumps(out))
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
