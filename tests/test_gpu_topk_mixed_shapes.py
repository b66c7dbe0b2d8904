"""A group top-k batch whose queries take all three shapes (one group, single-term groups, true groups with and without a
minimum match count), some with excluded terms, over two segments: every query's hits, n_out and total_matches equal
those of the same queries run as batches of one shape, bit for bit, at pruning levels 0 and 2. The batch is large enough
(n_queries * k >= 131072) for the key -> hit conversion to run on several host threads, and every array of the result
(keys, totals, counts) goes through the per-shape rows and back to query order."""
import numpy as np
import pytest

import orc
import serenedb_b200 as sdb
from gpu_util import ctx, to_gpu

pytestmark = pytest.mark.gpu

K = 2048
NQ = 96
N_TERMS = 12


def _shape(q, m):
    """0: one group, 1: single-term groups, 2: true groups (the library's split, after normalising full minimums)."""
    if any(1 < v < len(g) for g, v in zip(q, m)):
        return 2
    groups = sum(len(g) if v == len(g) else 1 for g, v in zip(q, m))
    return 0 if groups == 1 else 1 if groups == sum(len(g) for g in q) else 2


def test_mixed_shapes_equal_single_shape_batches():
    parts = [orc.synth_segment(n, list(range(N_TERMS)), doc0=d0) for n, d0 in ((120_000, 0), (90_000, 120_000))]
    reader = sdb.IndexReader([to_gpu(o) for o, _, _ in parts], sum(o.n_docs for o, _, _ in parts),
                             int(sum(dl.sum() for _, dl, _ in parts)),
                             [sum(len(lists[t][0]) for _, _, lists in parts) for t in range(N_TERMS)])
    rng = np.random.default_rng(11)
    qs, mins, xs = [], [], []
    for i in range(NQ):
        a, b, c, d = (int(t) for t in rng.choice(N_TERMS, size=4, replace=False))
        q, m = [([[a, b]], [1]), ([[a], [b]], [1, 1]), ([[a, b], [c]], [1, 1]), ([[a, b, c]], [2])][i % 4]
        qs.append(q)
        mins.append(m)
        xs.append([d] if i % 5 == 0 else [])
    shapes = np.array([_shape(q, m) for q, m in zip(qs, mins)])
    assert set(shapes.tolist()) == {0, 1, 2} and NQ * K >= 131072
    scorer = sdb.BM25()
    try:
        for lvl in (0, 2):
            ctx().set_wand(lvl)
            hits, n_out, total = sdb.ExecuteTopKGroupsBatch(reader, qs, scorer, K, exclude=xs, min_match=mins)
            assert n_out.max() > 0
            for sh in range(3):
                idx = np.flatnonzero(shapes == sh)
                h1, n1, t1 = sdb.ExecuteTopKGroupsBatch(reader, [qs[i] for i in idx], scorer, K, exclude=[xs[i] for i in idx],
                                                         min_match=[mins[i] for i in idx])
                assert np.array_equal(n_out[idx], n1), (lvl, sh)
                assert np.array_equal(total[idx], t1), (lvl, sh)
                for j, q in enumerate(idx):
                    assert hits[q, :n_out[q]].tobytes() == h1[j, :n1[j]].tobytes(), (lvl, sh, q)
    finally:
        ctx().set_wand(0)
