"""The NumPy statement of conjunctions of OR groups of phrases (tests/phrase_groups_reference.py) pinned to hand-written
answers, and its three identities: groups of one alternative are the clause conjunction (phrase_and_reference.py);
one-slot alternatives of distinct terms are the OR groups (groups_reference.py, min_match_reference.py with every minimum
1), scored as the flat OR of their terms; one group of one-slot alternatives is the flat OR. Runs without a GPU."""
import numpy as np
import pytest

import groups_reference as gr
import min_match_reference as mmr
import phrase_and_reference as par
import phrase_groups_reference as pgr
import phrase_reference as pr

f32 = np.float32
C0 = (f32(2.0), f32(1.5), f32(0.25))     # (c0, norm_const, norm_length) of a BM25 form
C1 = (f32(0.7), f32(1.2), f32(0.5))
C2 = (f32(1.1), f32(0.9), f32(0.3))


def G(*alts, neg=False):
    """A group of alternatives, each a list of terms or (terms, rel_pos)."""
    return ([(list(a[0]), a[1]) if isinstance(a, tuple) else (list(a), None) for a in alts], neg)


def _bits(x):
    return np.asarray(x, np.float32).view(np.uint32).tolist()


NEW, YORK, NYC, PIZZA = 0, 1, 2, 3


def test_new_york_or_nyc_and_pizza():
    docs = [[NEW, YORK, PIZZA], [NYC, PIZZA], [YORK, NEW, PIZZA], [NEW, YORK], [PIZZA, NYC, NEW, YORK, PIZZA], [PIZZA]]
    q = [G([NEW, YORK], [NYC]), G([PIZZA])]
    ds, fs = pgr.match(docs, q)
    assert ds.tolist() == [1, 2, 5]
    assert fs == [[1, 0, 1], [0, 1, 1], [1, 1, 2]]


def test_doc_matching_both_alternatives_scores_both():
    docs = [[NEW, YORK, NYC], [NYC], [NEW, YORK], [NYC, NYC, PIZZA]]
    q = [G([NEW, YORK], [NYC])]
    ds, fs = pgr.match(docs, q)
    assert ds.tolist() == [1, 2, 3, 4]
    # docs_count: "new york" 2 (min of new 2, york 2), nyc 3: the phrase is added first
    assert pgr.cost_order(docs, q) == [0, 1]
    norms = np.array([len(d) for d in docs], np.uint32)
    got = pgr.scores(docs, q, ds, fs, norms, [C0, C1])
    want = [f32(f32(f32(0) + pr.score(1, 3, *C0)) + pr.score(1, 3, *C1)),   # both alternatives
            f32(f32(0) + pr.score(1, 1, *C1)),                               # frequency 0 adds nothing, not bm25(0)
            f32(f32(0) + pr.score(1, 2, *C0)),
            f32(f32(0) + pr.score(2, 3, *C1))]
    assert _bits(got) == _bits(want)


def test_duplicate_alternative_scores_twice():
    docs = [[NEW, YORK], [NYC]]
    q = [G([NEW, YORK], [NEW, YORK])]
    ds, fs = pgr.match(docs, q)
    assert ds.tolist() == [1] and fs == [[1, 1]]
    got = pgr.scores(docs, q, ds, fs, None, [C0, C0])
    assert _bits(got) == _bits([f32(f32(f32(0) + pr.score(1, 1, *C0)) + pr.score(1, 1, *C0))])


def test_alternative_missing_in_a_segment_and_empty_group():
    """Segment 0 holds no NYC: that alternative matches nothing there, the phrase still does. Segment 1 holds neither
    term of ("new york" | nyc): the group, so the query, matches nothing there."""
    seg0 = [[NEW, YORK, PIZZA], [PIZZA], [YORK, PIZZA]]
    seg1 = [[PIZZA], [NEW, PIZZA], [PIZZA, PIZZA]]
    q = [G([NEW, YORK], [NYC]), G([PIZZA])]
    m = pgr.matches([seg0, seg1], q)
    assert m[0][0].tolist() == [1] and m[1][0].tolist() == []
    assert pgr.count(m) == 1


def test_negated_group_excludes_every_alternative():
    docs = [[0, 1], [2], [0, 2, 1], [3], [1, 0, 3], [0, 3, 1]]
    q = [G([3], [0], [1]), G([0, 1], [2], neg=True)]       # (3 | 0 | 1) & !("0 1" | 2)
    ds, _ = pgr.match(docs, q)
    assert ds.tolist() == [4, 5, 6]
    # !(A | B) is !A & !B: the clause conjunction with two negated clauses
    ands = par.match(docs, [([3], None, False), ([0, 1], None, True), ([2], None, True)])[0]
    assert pgr.match(docs, [G([3]), G([0, 1], [2], neg=True)])[0].tolist() == ands.tolist() == [4, 5, 6]
    # a negated alternative whose term the segment does not hold excludes nothing
    assert pgr.match(docs, [G([3], [0], [1]), G([7, 1], [9], neg=True)])[0].tolist() == [1, 3, 4, 5, 6]


def test_cost_tie_keeps_query_order_flattened():
    docs = [[0, 1, 2, 3], [2, 3, 0, 1], [0, 1], [2, 3]]
    a, b = ([0, 1], None), ([2, 3], None)       # both cost 3
    q_ab, q_ba = [G(a, b)], [G(b, a)]
    assert pgr.cost_order(docs, q_ab) == [0, 1] and pgr.cost_order(docs, q_ba) == [0, 1]
    # across groups: the flattened order of the alternatives decides a tie
    assert pgr.cost_order(docs, [G(b), G(a, [0])]) == [0, 1, 2]
    ds, fs = pgr.match(docs, q_ab)
    norms = np.array([len(d) for d in docs], np.uint32)
    s_ab = pgr.scores(docs, q_ab, ds, fs, norms, [C0, C1])
    assert s_ab[0] == f32(f32(f32(0) + pr.score(1, 4, *C0)) + pr.score(1, 4, *C1))
    s_ba = pgr.scores(docs, q_ba, ds, [f[::-1] for f in fs], norms, [C1, C0])
    assert s_ba[0] == f32(f32(f32(0) + pr.score(1, 4, *C1)) + pr.score(1, 4, *C0))


def _corpus(seed, n=300, vocab=8):
    rng = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, vocab + 1)
    p /= p.sum()
    return [rng.choice(vocab, size=int(rng.integers(1, 25)), p=p).tolist() for _ in range(n)]


def test_identity_groups_of_one_alternative_are_the_clause_conjunction():
    segs = [_corpus(s) for s in (1, 2)]
    norms = [np.array([len(d) for d in docs], np.uint32) for docs in segs]
    for clauses in ([([0, 1], None, False), ([2], None, False)], [([1, 0, 1], None, False), ([3, 4], None, True)],
                    [([0, 2], [0, 2], False), ([0], None, False), ([5], None, True)]):
        groups = [([(t, r)], n) for t, r, n in clauses]
        consts = [None if n else c for (_, _, n), c in zip(clauses, (C0, C1, C2))]
        got, want = pgr.matches(segs, groups, excl=[6]), par.matches(segs, clauses, excl=[6])
        for (gd, gf), (wd, wf) in zip(got, want):
            assert gd.tolist() == wd.tolist() and gf == wf
        h, t = pgr.topk(segs, groups, got, norms, consts, 30)
        h2, t2 = par.topk(segs, clauses, want, norms, consts, 30)
        assert t == t2 and h.tobytes() == h2.tobytes()


def _lists(docs, vocab=8):
    return [np.array([i + 1 for i, s in enumerate(docs) if t in s], np.uint32) for t in range(vocab)]


def _flat_or(segs, terms, matched, norms, consts, k):
    """The OR-groups top-k as the groups entries score it: the flat OR of the terms, each present term's bm25(tf, norm)
    summed from 0 by ascending docs_count in the doc's segment (stable), over the docs the groups match."""
    rows = []
    for si, (docs, ds) in enumerate(zip(segs, matched)):
        dc = [sum(1 for s in docs if t in s) for t in terms]
        order = sorted(range(len(terms)), key=lambda i: dc[i])
        for d in ds.tolist():
            seq, s = docs[d - 1], f32(0)
            for j in order:
                if terms[j] in seq:
                    s = f32(s + pr.score(seq.count(terms[j]), norms[si][d - 1], *consts[j]))
            rows.append((s, d, si))
    rows.sort(key=lambda r: (-r[0], r[2], r[1]))
    return rows[:k], len(rows)


@pytest.mark.parametrize("groups_terms", [[[0, 1], [2]], [[3], [1, 4, 0]], [[5, 2], [0, 6], [1]], [[0, 1, 2, 3]]])
def test_identity_one_slot_alternatives_are_the_or_groups(groups_terms):
    """Distinct one-slot alternatives: the OR-group statements (every minimum 1) match the same docs, and the score is the
    flat OR of the terms; one group of them (the last case) is the flat OR."""
    segs = [_corpus(s) for s in (3, 4, 5)]
    norms = [np.array([len(d) for d in docs], np.uint32) for docs in segs]
    terms = [t for g in groups_terms for t in g]
    consts = [(f32(0.5 + 0.3 * i), f32(1.0 + 0.1 * i), f32(0.2 + 0.05 * i)) for i in range(len(terms))]
    groups = [([([t], None) for t in g], False) for g in groups_terms]
    got = pgr.matches(segs, groups, excl=[7])
    for docs, (gd, _) in zip(segs, got):
        L = _lists(docs)
        assert gd.tolist() == gr.match_docs(L, groups_terms, [7]).tolist()
        assert gd.tolist() == mmr.match_docs(L, groups_terms, [7], mins=[1] * len(groups_terms)).tolist()
    h, total = pgr.topk(segs, groups, got, norms, consts, 40)
    rows, total2 = _flat_or(segs, terms, [ds for ds, _ in got], norms, consts, 40)
    assert total == total2
    assert [(int(r["doc"]), int(r["seg"])) for r in h] == [(d, si) for _, d, si in rows]
    assert _bits(h["score"]) == _bits([r[0] for r in rows])


def test_engine_refuses_malformed_groups():
    from serenedb_b200 import engine as E

    for bad in ([[]], [[[]]], [5], []):
        with pytest.raises(ValueError):
            E._phrase_groups([bad], None)
    with pytest.raises(ValueError):
        E._phrase_groups([[[[0, 1]]]], [None, None])
    with pytest.raises(ValueError):
        E._phrase_groups([[[([0, 1], [0])]]], None)
    g = E._phrase_groups([[[[0, 1], [2]], [[3]]]], [[[4, 5]]])
    assert g == [[([([0, 1], None), ([2], None)], False), ([([3], None)], False), ([([4, 5], None)], True)]]
