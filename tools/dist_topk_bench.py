"""The BM25 top-k of group queries across GPUs (sdbg_bm25_topk_batch_groups_min_device, sdbg_bm25_topk_merge_gathered) on
one H100: bench.py's 10 M-doc corpus (BASELINE.json configs[2]) cut by doc range into 8 shards, each its own segment as
each rank would hold it, with corpus-wide term statistics. Two batches of 4096 queries at k = 1000: the two-term ORs of
bench.make_queries (one group each) and `a & (b | c)` groups (the same pairs as b | c, with a third term a). Reports, in
ms per step (CUDA events on the library's stream, L2 flushed before every step, after warm-up):
  (a) the local entry over the unsharded corpus, one 10 M-doc segment (sdbg_bm25_topk_batch_groups_min);
  (b) the device form on each shard: the slowest shard and the sum over shards;
  (c) at R = 8, the new merge kernels alone (re-key, select, map back; torch.profiler, CUDA activities) against the flat
      path's merge (sdbg_topk_merge_gathered: its repack copies and the same select kernel) on the same OR queries, whose
      keys come from sdbg_bm25_topk_batch_device; and each whole merge call with its copy back to host hits.
The NCCL all-gather and the scaling across GPUs are not measured here: one GPU. Exits non-zero unless the merged hits of
both batches equal the local entry's hits over the 8 shard segments on one GPU (seg = the shard, as the merge reports the
rank) and, for the ORs, the flat path's merged hits. Prints the GPU name and power
limit read in the same run.

    python tools/dist_topk_bench.py [--steps 10] [--warmup 2] [--docs 10000000] [--queries 4096]
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
from serenedb_b200.engine import FLT_MIN, HIT_DTYPE, PreparedBatch, _ptr, _query_args, _seg_array  # noqa: E402
from count_bench import gpu_info, timed  # noqa: E402

K, R = 1000, 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=4096)
    args = ap.parse_args()
    threads = min(os.cpu_count() or 1, 64)
    import torch
    from torch.profiler import ProfilerActivity, profile

    ctx = sdb.Context(0)
    scorer = sdb.BM25()
    pairs = bench.make_queries(args.queries)
    rng = np.random.default_rng(5)
    batches = {"or2": [[list(p)] for p in pairs], "a_and_b_or_c": []}
    for p in pairs:
        a = int(rng.integers(0, bench.N_TERMS))
        while a in p:
            a = int(rng.integers(0, bench.N_TERMS))
        batches["a_and_b_or_c"].append([[a], list(p)])
    nq = args.queries
    out = {"gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup, "k": K, "ranks": R,
           "workload": "%d docs (BASELINE configs[2]) in %d doc-range shards, %d queries per batch" % (args.docs, R, nq),
           "collectives": "not measured (one GPU)"}
    ok = True

    def t(fn):
        m, s = timed(ctx, fn, args.steps, args.warmup)
        return {"ms": m, "std": s}

    def kernel_ms(fn, names):
        """Mean device time per call of the profiler events whose name contains one of `names`."""
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                fn()
            torch.cuda.synchronize()
        res = {}
        for name in names:
            us = [e.device_time for e in prof.events() if name in e.name]
            res[name] = round(float(np.sum(us)) / args.steps / 1000, 4) if us else None
        return res

    # the corpus, whole and as shards; the term statistics are the whole corpus's on every shard
    cuts = [i * args.docs // R for i in range(R + 1)]
    shards, dcs, sdl = [], np.zeros(bench.N_TERMS, np.uint64), 0
    for a, b in zip(cuts[:-1], cuts[1:]):
        s = sdb.Segment(ctx, b - a)
        dc, sum_dl = s.synth_corpus(a, 0, bench.N_TERMS, threads=threads)
        shards.append(s)
        dcs += np.asarray(dc, np.uint64)
        sdl += sum_dl
    readers = [sdb.IndexReader([s], args.docs, sdl, dcs) for s in shards]
    union = sdb.IndexReader(shards, args.docs, sdl, dcs)
    whole = sdb.Segment(ctx, args.docs)
    whole.synth_corpus(0, 0, bench.N_TERMS, threads=threads)
    one = sdb.IndexReader([whole], args.docs, sdl, dcs)

    def local(reader, qs):
        qa = _query_args(qs, None, None, groups=True, stats=lambda t: reader.stats(scorer, t))
        hits, n_out, total = np.zeros((nq, K), HIT_DTYPE), np.zeros(nq, np.uint32), np.zeros(nq, np.uint64)
        sa = _seg_array(reader.segments)
        return lambda: N.check(N.lib().sdbg_bm25_topk_batch_groups_min(sa, len(reader.segments), *qa, scorer.k, scorer.b, None, K, FLT_MIN,
                                                                       _ptr(hits), _ptr(n_out), _ptr(total)), ctx._h), hits, n_out

    def device(reader, qs, d_ptr):
        qa = _query_args(qs, None, None, groups=True, stats=lambda t: reader.stats(scorer, t))
        sa = _seg_array(reader.segments)
        return lambda: N.check(N.lib().sdbg_bm25_topk_batch_groups_min_device(sa, 1, *qa, scorer.k, scorer.b, None, K, FLT_MIN,
                                                                              C.c_void_p(d_ptr)), ctx._h)

    words = sdb.topk_groups_device_bytes(nq, K) // 8
    buf = torch.zeros((R, words), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    for name, qs in batches.items():
        res = {}
        res["a_local_unsharded"] = t(local(one, qs)[0])
        # the reference hits: the local entry over the same 8 segments (a sum of three or more term scores is added in
        # each segment's own docs_count order of the terms, so another segmentation can differ in the last bit)
        run, want, wn = local(union, qs)
        run()
        per = []
        for r, reader in enumerate(readers):
            fn = device(reader, qs, buf[r].data_ptr())
            per.append(t(fn)["ms"])
            fn()
        res["b_device_form"] = {"max_shard_ms": max(per), "sum_ms": round(sum(per), 3)}
        hits, n_out, total = np.zeros((nq, K), HIT_DTYPE), np.zeros(nq, np.uint32), np.zeros(nq, np.uint64)
        merge = lambda: N.check(N.lib().sdbg_bm25_topk_merge_gathered(ctx._h, C.c_void_p(buf.data_ptr()), R, nq, K, _ptr(hits),
                                                                      _ptr(n_out), _ptr(total)), ctx._h)
        res["c_merge_call"] = t(merge)
        res["c_merge_kernels"] = kernel_ms(merge, ("topk_rekey_gathered_kernel", "topk_merge_kernel", "topk_hits_gathered_kernel"))
        res["gathered_bytes"] = R * words * 8
        merge()
        same = np.array_equal(n_out, wn)
        for q in range(nq):
            h, w = hits[q, :n_out[q]], want[q, :wn[q]]
            same &= bool(np.array_equal(h["score"].view(np.uint32), w["score"].view(np.uint32)))
            same &= bool(np.array_equal(h["seg"], w["seg"]) and np.array_equal(h["doc"], w["doc"]))
        res["equal_local"] = bool(same)
        ok &= bool(same)
        if name == "or2":   # the flat path on the same queries: sdbg_bm25_topk_batch_device keys, sdbg_topk_merge_gathered
            keys = torch.zeros((R, nq, K), dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            flat = [list(p) for p in pairs]
            for r, reader in enumerate(readers):
                PreparedBatch(reader, flat, sdb.OR, scorer, K).run_device(r, keys[r].data_ptr())
            fh, fn_out = np.zeros((nq, K), HIT_DTYPE), np.zeros(nq, np.uint32)
            fmerge = lambda: N.check(N.lib().sdbg_topk_merge_gathered(ctx._h, C.c_void_p(keys.data_ptr()), R, nq, K, _ptr(fh),
                                                                      _ptr(fn_out)), ctx._h)
            res["c_flat_merge_call"] = t(fmerge)
            res["c_flat_merge_kernels"] = kernel_ms(lambda: N.check(N.lib().sdbg_topk_merge_gathered(
                ctx._h, C.c_void_p(keys.data_ptr()), R, nq, K, None, None), ctx._h), ("Memcpy DtoD", "topk_merge_kernel"))
            fmerge()
            same = np.array_equal(fn_out, n_out) and all(np.array_equal(fh[q, :n_out[q]], hits[q, :n_out[q]]) for q in range(nq))
            res["equal_flat_merge"] = bool(same)
            ok &= bool(same)
            del keys
        out[name] = res
    out["equal"] = ok
    print(json.dumps(out))
    for s in shards + [whole]:
        s.close()
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
