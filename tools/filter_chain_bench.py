"""Filter chains (sdbg.h SDBG_OP_AND_NEXT) on the BASELINE.json configs[3] corpus: 10 M docs, the 5-term conjunction
(p = .5/.4/.3/.25/.2) top-1000 as a batch, and a batch of two-term disjunctions of the same terms counted and faceted
(key: a random int32 column in 0..63). Filters:
  (a) n BETWEEN 250000 AND 749999 alone (bench.py configs[3]'s filter; n is random per doc);
  (b) chains of 2 and 4 predicates on random columns;
  (c) a doc-ordered column (value = doc - 1, like an insertion timestamp) below 1 %, 10 % and 50 % of the docs, chained
      with (a)'s predicate.
For each it reports ms per batch (CUDA events on the library's stream, L2 flushed before every step, after warm-up), the
matches, and the share of 2048-doc zones the chain judges dead or pass: computed here from the columns' per-zone
min / max with the rule zone_verdict_kernel applies, for integer columns. The card's name and power limit are read in the
same run.

    python tools/filter_chain_bench.py [--steps 5] [--warmup 1] [--docs 10000000] [--queries 4096]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import serenedb_b200 as sdb  # noqa: E402

ZONE = 2048
N_COL, R1, R2, R3, TS, KEY = 9, 20, 21, 22, 23, 24


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


def zone_shares(cols, chain, n_docs):
    """Shares of zones where some predicate holds for no row (dead) and where every one holds for every row (pass)."""
    nz = (n_docs + ZONE - 1) // ZONE
    dead = np.zeros(nz, bool)
    every = np.ones(nz, bool)
    for field, op, *b in chain:
        v = cols[field][:n_docs]
        pad = np.concatenate([v, np.full(nz * ZONE - n_docs, v[-1])]).reshape(nz, ZONE)
        mn, mx = pad.min(axis=1).astype(object), pad.max(axis=1).astype(object)
        lo, hi = -(1 << 63), (1 << 63) - 1
        if op == "LT":
            hi = b[0] - 1
        elif op == "GE":
            lo = b[0]
        else:   # BETWEEN
            lo, hi = b
        dead |= np.array([x > hi or y < lo for x, y in zip(mn, mx)])
        every &= np.array([x >= lo and y <= hi for x, y in zip(mn, mx)])
    return round(float(dead.mean()), 4), round(float((every & ~dead).mean()), 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=4096)
    args = ap.parse_args()
    n = args.docs
    threads = min(os.cpu_count() or 1, 64)

    ctx = sdb.Context(0)
    seg = sdb.Segment(ctx, n)
    dc, sum_dl = seg.synth_corpus(0, 1000000, 5, threads=threads)   # bench.py configs[3]: generator terms 1000000..1000004
    seg.synth_column(N_COL, 2, 6, 1, n)                            # n = h % 1e6 for docs 1..N (int32)
    rng = np.random.default_rng(7)
    nv = np.zeros(n, np.int32)
    seg.column_to_host(N_COL, nv.ctypes.data, n)
    cols = {N_COL: nv.astype(np.int64)}
    for f in (R1, R2, R3):
        cols[f] = rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
    cols[TS] = np.arange(n, dtype=np.int64)
    for f in (R1, R2, R3, TS):
        seg.stage_column(f, cols[f])
    seg.stage_column(KEY, rng.integers(0, 64, n, dtype=np.int64).astype(np.int32))
    reader = sdb.IndexReader([seg], n, sum_dl, dc)
    scorer = sdb.BM25(1.2, 0.75)
    conj = [[0, 1, 2, 3, 4]] * args.queries
    pairs = [[0, 1], [1, 2], [2, 3], [3, 4], [0, 4], [1, 3]]
    disj = [pairs[i % len(pairs)] for i in range(args.queries)]

    nb = [(N_COL, "BETWEEN", 250000, 749999)]
    chains = {"none": [], "a_single": nb,
              "b_chain2": nb + [(R1, "GE", 0)],
              "b_chain4": nb + [(R1, "GE", 0), (R2, "LT", 1 << 61), (R3, "BETWEEN", -(1 << 61), 1 << 62)]}
    for pct in (1, 10, 50):
        chains["c_ordered_%dpct" % pct] = [(TS, "LT", n * pct // 100)] + nb
    ctx.set_wand(2)
    out = {}
    for name, chain in chains.items():
        filt = [sdb.pred(f, op, *b) for f, op, *b in chain] or None
        topk = sdb.PreparedBatch(reader, conj, sdb.AND, scorer, 1000, filt=filt)
        row = {}
        row["topk_ms"], row["topk_std"] = timed(ctx, topk.run_host, args.steps, args.warmup)
        row["topk_matches"] = int(topk.run_host()[2].sum())
        row["count_ms"], row["count_std"] = timed(ctx, lambda: sdb.ExecuteCountBatch(reader, disj, sdb.OR, filt=filt),
                                                  args.steps, args.warmup)
        row["count_matches"] = int(sdb.ExecuteCountBatch(reader, disj, sdb.OR, filt=filt).sum())
        row["facet_ms"], row["facet_std"] = timed(
            ctx, lambda: sdb.ExecuteFacetCountsBatch(reader, disj, sdb.OR, KEY, key_min=0, key_span=64, filt=filt),
            args.steps, args.warmup)
        if chain:
            row["zones_dead"], row["zones_pass"] = zone_shares(cols, chain, n)
        out[name] = row
        print(name, json.dumps(row), file=sys.stderr, flush=True)
    print(json.dumps({"gpu": gpu_info(), "docs": n, "queries": args.queries, "steps": args.steps, "warmup": args.warmup,
                      "results": out}))


if __name__ == "__main__":
    main()
