"""The NumPy statement of clause conjunctions (tests/phrase_and_reference.py) pinned to hand-written answers, and its two
identities: a query of one positive clause is the phrase statement (phrase_reference.py), and a query of one-slot
positive clauses of distinct terms is the flat AND (terms summed by ascending docs_count, ties in query order). Runs
without a GPU."""
import numpy as np

import phrase_and_reference as par
import phrase_reference as pr

f32 = np.float32
C0 = (f32(2.0), f32(1.5), f32(0.25))     # (c0, norm_const, norm_length) of a BM25 form
C1 = (f32(0.7), f32(1.2), f32(0.5))


def P(terms, rel=None):
    return (list(terms), rel, False)


def N(terms, rel=None):
    return (list(terms), rel, True)


def test_phrase_with_a_term():
    docs = [[0, 1, 2], [0, 2, 1], [1, 0], [2, 0, 1]]
    ds, fs = par.match(docs, [P([0, 1]), P([2])])
    assert ds.tolist() == [1, 4] and fs == [[1, 1], [1, 1]]


def test_two_phrases_sharing_a_term():
    docs = [[0, 1, 2], [0, 1, 3, 1, 2], [0, 1, 3], [2, 1, 2], [0, 1, 2, 0, 1, 2]]
    ds, fs = par.match(docs, [P([0, 1]), P([1, 2])])
    assert ds.tolist() == [1, 2, 5] and fs == [[1, 1], [1, 1], [2, 2]]


def test_phrase_and_its_own_term():
    docs = [[0, 1], [0, 2, 1], [1, 0], [0, 1, 0]]
    clauses = [P([0, 1]), P([0])]
    ds, fs = par.match(docs, clauses)
    assert ds.tolist() == [1, 4] and fs == [[1, 1], [1, 2]]
    # docs_count: term 0 in 4 docs, term 1 in 3: "0 1" costs 3, "0" costs 4, so "0 1" is added first
    assert par.cost_order(docs, clauses) == [0, 1]
    norms = np.array([len(d) for d in docs], np.uint32)
    got = par.scores(docs, clauses, ds, fs, norms, [C0, C1])
    want = [f32(f32(f32(0) + pr.score(1, 2, *C0)) + pr.score(1, 2, *C1)),
            f32(f32(f32(0) + pr.score(1, 3, *C0)) + pr.score(2, 3, *C1))]
    assert got.view(np.uint32).tolist() == np.array(want, np.float32).view(np.uint32).tolist()


def test_negated_phrase_overlapping_a_positive_one():
    docs = [[0, 1, 2], [0, 1, 3], [1, 2, 0, 1], [2, 1, 0, 1], [1, 2]]
    ds, _ = par.match(docs, [P([0, 1]), N([1, 2])])
    assert ds.tolist() == [2, 4]
    # a one-slot negated clause is an excluded term
    ds2, _ = par.match(docs, [P([0, 1]), N([3])])
    assert ds2.tolist() == par.match(docs, [P([0, 1])], excl=[3])[0].tolist() == [1, 3, 4]
    # a negated clause whose term the segment does not hold excludes nothing
    assert par.match(docs, [P([0, 1]), N([7, 1])])[0].tolist() == [1, 2, 3, 4]


def test_tie_in_clause_cost_keeps_query_order():
    docs = [[0, 1, 2, 3], [2, 3, 0, 1], [0, 1], [2, 3]]
    a, b = P([0, 1]), P([2, 3])       # both cost 3
    assert par.cost_order(docs, [a, b]) == [0, 1]
    assert par.cost_order(docs, [b, a]) == [0, 1]
    ds, fs = par.match(docs, [a, b])
    norms = np.array([len(d) for d in docs], np.uint32)
    s_ab = par.scores(docs, [a, b], ds, fs, norms, [C0, C1])
    assert s_ab[0] == f32(f32(f32(0) + pr.score(1, 4, *C0)) + pr.score(1, 4, *C1))
    s_ba = par.scores(docs, [b, a], ds, [f[::-1] for f in fs], norms, [C1, C0])
    assert s_ba[0] == f32(f32(f32(0) + pr.score(1, 4, *C1)) + pr.score(1, 4, *C0))
    # a cheaper clause goes first whatever its place in the query
    docs2 = docs + [[0, 1]]
    assert par.cost_order(docs2, [b, a]) == [0, 1]
    assert par.cost_order(docs2 + [[2, 3]] * 2, [a, b]) == [0, 1]
    assert par.cost_order([[0, 1]] * 3 + [[2, 3]], [a, b]) == [1, 0]


def test_tie_among_three_clauses_decides_the_score_bits():
    """With three positive clauses the order of the last two changes the fp32 sum: the cheapest clause first, then the
    tied pair in query order."""
    docs = [[0, 1, 2, 3], [0, 1, 2, 3], [2, 3, 0, 1, 4], [0, 1, 2, 3, 4, 4]]
    a, b, c = P([4]), P([0, 1]), P([2, 3])           # costs 2, 4, 4
    assert par.cost_order(docs, [b, c, a]) == [2, 0, 1]
    assert par.cost_order(docs, [c, b, a]) == [2, 0, 1]
    ka, kb, kc = (f32(0.1), f32(1.5), f32(0.25)), (f32(3.3), f32(1.2), f32(0.5)), (f32(0.7), f32(0.9), f32(0.3))
    ds, fs = par.match(docs, [b, c, a])
    assert ds.tolist() == [3, 4]
    norms = np.array([len(d) for d in docs], np.uint32)
    got_bc = par.scores(docs, [b, c, a], ds, fs, norms, [kb, kc, ka])
    got_cb = par.scores(docs, [c, b, a], ds, [[g[1], g[0], g[2]] for g in fs], norms, [kc, kb, ka])
    for i, (d, f) in enumerate(zip(ds, fs)):
        x, y, z = pr.score(f[2], norms[d - 1], *ka), pr.score(f[0], norms[d - 1], *kb), pr.score(f[1], norms[d - 1], *kc)
        bc = f32(f32(f32(f32(0) + x) + y) + z)
        cb = f32(f32(f32(f32(0) + x) + z) + y)
        assert bc != cb                   # these constants make the two tie orders differ in the last bit
        assert got_bc[i].view(np.uint32) == bc.view(np.uint32) and got_cb[i].view(np.uint32) == cb.view(np.uint32)


def _corpus(seed, n=300, vocab=8):
    rng = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, vocab + 1)
    p /= p.sum()
    return [rng.choice(vocab, size=int(rng.integers(1, 25)), p=p).tolist() for _ in range(n)], rng


def test_identity_one_positive_clause_is_the_phrase():
    segs = [_corpus(s)[0] for s in (1, 2)]
    norms = [np.array([len(d) for d in docs], np.uint32) for docs in segs]
    for phrase, rel in ([0, 1], None), ([1, 0, 1], None), ([0, 2], [0, 2]), ([3], None):
        clauses = [P(phrase, rel)]
        got = par.matches(segs, clauses, excl=[5])
        want = [pr.match(d, phrase, rel, [5]) for d in segs]
        for (gd, gf), (wd, wf) in zip(got, want):
            assert gd.tolist() == wd.tolist() and [f[0] for f in gf] == wf.tolist()
        h, t = par.topk(segs, clauses, got, norms, [C0], 25)
        h2, t2 = pr.topk(want, norms, C0, 25)
        assert t == t2 and h.tobytes() == h2.tobytes()


def _flat_and(segs, terms, norms, consts, k):
    """The flat AND top-k: tf per term, scores summed from 0 by ascending docs_count in the doc's segment, stable."""
    rows = []
    for si, docs in enumerate(segs):
        dc = [sum(1 for s in docs if t in s) for t in terms]
        order = sorted(range(len(terms)), key=lambda i: dc[i])
        for i, seq in enumerate(docs):
            if all(t in seq for t in terms):
                s = f32(0)
                for j in order:
                    s = f32(s + pr.score(seq.count(terms[j]), norms[si][i], *consts[j]))
                rows.append((s, i + 1, si))
    rows.sort(key=lambda r: (-r[0], r[2], r[1]))
    return rows[:k], len(rows)


def test_identity_one_slot_clauses_are_the_flat_and():
    segs = [_corpus(s)[0] for s in (3, 4, 5)]
    norms = [np.array([len(d) for d in docs], np.uint32) for docs in segs]
    consts = [C0, C1, (f32(1.1), f32(0.9), f32(0.3))]
    for terms in ([0, 1], [2, 0], [1, 3, 0], [4]):
        clauses = [P([t]) for t in terms]
        h, total = par.topk(segs, clauses, par.matches(segs, clauses), norms, consts[:len(terms)], 40)
        rows, total2 = _flat_and(segs, terms, norms, consts[:len(terms)], 40)
        assert total == total2
        assert [(float(r["score"]), int(r["doc"]), int(r["seg"])) for r in h] == [(float(s), d, si) for s, d, si in rows]
        assert h["score"].view(np.uint32).tolist() == np.array([r[0] for r in rows], np.float32).view(np.uint32).tolist()


def test_column_passes_and_scan_follow_the_matches():
    segs = [_corpus(s)[0] for s in (6, 7)]
    norms = [np.array([len(d) for d in docs], np.uint32) for docs in segs]
    clauses = [P([0, 1]), P([2]), N([1, 2])]
    m = par.matches(segs, clauses)
    cols = [{1: (np.arange(len(d), dtype=np.int64) % 7, None)} for d in segs]
    counts, nulls = par.facet_counts(m, [c[1] for c in cols], 0, 7)
    assert int(counts.sum()) + int(nulls) == par.count(m) > 0
    (ss, dd, sc), total = par.scan(segs, clauses, m, norms, [C0, C1, None], offset=1, limit=5)
    assert total == par.count(m) and len(dd) == min(5, total - 1)
    allp, _ = par.scan(segs, clauses, m, norms, [C0, C1, None])
    assert dd.tolist() == allp[1][1:6].tolist() and sc.tolist() == allp[2][1:6].tolist()


def test_engine_refuses_rel_pos_of_the_wrong_length():
    """A clause's (or phrase's) rel_pos of another length than its terms is refused before the library is called."""
    import pytest
    from serenedb_b200 import engine as E

    with pytest.raises(ValueError):
        E._clause(([0, 1, 2], [0, 1]))
    with pytest.raises(ValueError):
        E._phrase_args([[0, 1]], [[0]], None)
    assert E._clause(([0, 1], [0, 2])) == ([0, 1], [0, 2]) and E._clause([3]) == ([3], None)
