"""The match scan (Stream mode, sdbg_match_scan_batch_groups_min) on bench.py's 10 M-doc corpus. Workloads:
  (a) the 4096 two-term disjunctions of bench.make_queries at LIMIT 1000, unscored and scored, next to the shipped
      top-1000 by score (pruning level 2) of the same batch;
  (b) every match of the first 64 of those queries, scored, through the new entry and through StreamScoredDocs
      (sdbg_bm25_scan, one call pair per query);
  (c) 4096 `a & (b | c)` and 4096 `2 of (a | b | c)` queries (terms from make_queries' pairs) at LIMIT 1000, and a full
      drain of the first 64 of each.
Each is ms per call (CUDA events on the library's stream, L2 flushed before every call, after warm-up), with the matches
returned. Exits non-zero unless (b)'s docs and scores equal StreamScoredDocs'. Prints the GPU name and power limit read
in the same run.

    python tools/match_scan_bench.py [--steps 5] [--warmup 1] [--docs 10000000]
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
from serenedb_b200.engine import HIT_DTYPE, _ptr, _query_args, _seg_array  # noqa: E402


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def timed(ctx, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(steps):
        ctx.flush_l2()
        ctx.timer_start()
        fn()
        ms.append(ctx.timer_stop())
    return round(float(np.mean(ms)), 3), round(float(np.std(ms)), 3)


def prepared_scan(ctx, reader, queries, mins, scorer, limit):
    """The entry's arguments marshalled once (like PreparedBatch): returns (call, n_out, total)."""
    nq = len(queries)
    args = _query_args(queries, None, mins, groups=True, stats=lambda t: reader.stats(scorer or sdb.BM25(), t))
    hits = np.zeros((nq, limit), HIT_DTYPE)
    n_out, total = np.zeros(nq, np.uint32), np.zeros(nq, np.uint64)
    segs = _seg_array(reader.segments)
    k1, b = (scorer.k, scorer.b) if scorer else (0.0, 0.0)

    def call():
        N.check(N.lib().sdbg_match_scan_batch_groups_min(segs, len(reader.segments), *args, k1, b, None, None, limit,
                                                         int(scorer is not None), _ptr(hits), _ptr(n_out), _ptr(total)), ctx._h)
    return call, hits, n_out, total


def scan_row(ctx, reader, queries, mins, scorer, limit, steps, warmup):
    call, _, n_out, total = prepared_scan(ctx, reader, queries, mins, scorer, limit)
    ms, std = timed(ctx, call, steps, warmup)
    return dict(ms=ms, std=std, queries=len(queries), limit=limit, rows=int(n_out.sum()), matches=int(total.sum()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--docs", type=int, default=10_000_000)
    args = ap.parse_args()
    ctx = sdb.Context(0)
    ctx.set_wand(2)
    seg = sdb.Segment(ctx, args.docs)
    dc, sum_dl = seg.synth_corpus(0, 0, bench.N_TERMS, threads=min(os.cpu_count() or 1, 64))
    reader = sdb.IndexReader([seg], args.docs, sum_dl, dc)
    scorer = sdb.BM25()
    pairs = bench.make_queries(4096)
    ors = [[q] for q in pairs]
    out = {"gpu": gpu_info(), "docs": args.docs, "steps": args.steps, "warmup": args.warmup}

    # (a) LIMIT 1000 of 4096 two-term ORs, next to the shipped top-1000 by score
    out["a_or_limit1000_unscored"] = scan_row(ctx, reader, ors, None, None, 1000, args.steps, args.warmup)
    out["a_or_limit1000_scored"] = scan_row(ctx, reader, ors, None, scorer, 1000, args.steps, args.warmup)
    top = sdb.PreparedBatch(reader, pairs, sdb.OR, scorer, bench.TOPK)
    ms, std = timed(ctx, top.run_host, args.steps, args.warmup)
    out["a_or_top1000_by_score_level2"] = dict(ms=ms, std=std, queries=len(pairs), k=bench.TOPK)

    # (b) every match of the first 64, scored: one batch against StreamScoredDocs per query
    first = ors[:64]
    full = int(sdb.ExecuteCountGroupsBatch(reader, first).max())
    out["b_or64_drain_scored"] = scan_row(ctx, reader, first, None, scorer, full, args.steps, args.warmup)
    ms, std = timed(ctx, lambda: [sdb.StreamScoredDocs(reader, 0, q, sdb.OR, scorer) for q in pairs[:64]], args.steps, args.warmup)
    out["b_or64_stream_scored_docs"] = dict(ms=ms, std=std, queries=64)
    got = sdb.ExecuteMatchScanGroupsBatch(reader, first, scorer, limit=full)
    equal = all(np.array_equal(g[0][1], s[0]) and np.array_equal(g[0][2].view(np.uint32), s[1].view(np.uint32))
                for g, s in zip(got, (sdb.StreamScoredDocs(reader, 0, q, sdb.OR, scorer) for q in pairs[:64])))
    out["b_equal"] = bool(equal)

    # (c) `a & (b | c)` and `2 of (a | b | c)` at LIMIT 1000, and a full drain of 64 of each
    triples = [[pairs[i][0], pairs[i][1], pairs[(i + 1) % len(pairs)][0]] for i in range(len(pairs))]
    triples = [t for t in triples if len(set(t)) == 3]
    shapes = {"and_of_or": ([[t[0]], [t[1], t[2]]] for t in triples), "2_of_3": ([t] for t in triples)}
    for name, qs in shapes.items():
        qs = list(qs)
        mins = [[2]] * len(qs) if name == "2_of_3" else None
        for scored in (None, scorer):
            tag = "scored" if scored else "unscored"
            out["c_%s_limit1000_%s" % (name, tag)] = scan_row(ctx, reader, qs, mins, scored, 1000, args.steps, args.warmup)
        m64 = mins[:64] if mins else None
        full = int(sdb.ExecuteCountGroupsBatch(reader, qs[:64], min_match=m64).max())
        out["c_%s_drain64_scored" % name] = scan_row(ctx, reader, qs[:64], m64, scorer, full, args.steps, args.warmup)
    print(json.dumps(out))
    if not equal:
        sys.exit(1)


if __name__ == "__main__":
    main()
