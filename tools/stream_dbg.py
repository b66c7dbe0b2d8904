"""Debug helper: OR / AND queries on a small corpus through the legacy kernel (SDBG_STREAM=0, pruning off = the exact
reference) and through the stream kernel at every pruning level; hits must be identical, totals identical without
pruning and a lower bound with it."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np
import serenedb_b200 as sdb

ctx = sdb.Context(0)
n = int(os.environ.get("PROBE_DOCS", 2_000_000))
g = sdb.Segment(ctx, n)
dc, sum_dl = g.synth_corpus(0, 0, 96, threads=16)
g.synth_column(9, 2, 6, 1, n)
reader = sdb.IndexReader([g], n, sum_dl, dc)
scorer = sdb.BM25()
filt = sdb.pred(9, "BETWEEN", 250000, 749999)
cases = [("OR", [[81, 1], [0, 1], [5, 59], [1, 36], [0], [0, 1, 2], [3, 40, 70, 90], [60, 61], [95], [2, 80, 90]], None, 100),
         ("OR", [[81, 1], [5, 59], [0, 2, 50]], filt, 100),
         ("AND", [[0, 1, 2, 3, 4], [5, 59], [1, 36, 80], [0, 95]], None, 100),
         ("AND", [[0, 1, 2, 3, 4], [5, 9]], filt, 1000)]
bad = 0
for kind, queries, f, k in cases:
    ref = None
    for env, wand in (({"SDBG_STREAM": "0"}, 0), ({"SDBG_STREAM": "1"}, 0), ({"SDBG_STREAM": "1"}, 1), ({"SDBG_STREAM": "1"}, 2)):
        os.environ.update(env)
        ctx.set_wand(wand)
        batch = sdb.PreparedBatch(reader, queries, sdb.AND if kind == "AND" else sdb.OR, scorer, k, filt=f)
        h, nout, tot = batch.run_host()
        if ref is None:
            ref = (h.copy(), nout.copy(), tot.copy())
        ok = all(nout[i] == ref[1][i] and np.array_equal(h[i][: nout[i]]["doc"], ref[0][i][: ref[1][i]]["doc"]) and
                 np.array_equal(h[i][: nout[i]]["score"], ref[0][i][: ref[1][i]]["score"]) for i in range(len(queries)))
        tok = np.array_equal(tot, ref[2]) if wand == 0 else bool(np.all(tot <= ref[2]))
        bad += (not ok) + (not tok)
        print(kind, "filt" if f else "-", env, "wand", wand, "hits ok", ok, "totals ok", tok, "seen %.0f%%" % (100.0 * tot.sum() / max(ref[2].sum(), 1)), flush=True)
        if not ok:
            print("   bad queries:", [queries[i] for i in range(len(queries)) if not (nout[i] == ref[1][i] and np.array_equal(h[i][: nout[i]]["doc"], ref[0][i][: ref[1][i]]["doc"]) and np.array_equal(h[i][: nout[i]]["score"], ref[0][i][: ref[1][i]]["score"]))])
print("FAILURES", bad)
