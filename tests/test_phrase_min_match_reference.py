"""The NumPy statement of minimum match counts over OR groups of phrases (tests/phrase_min_match_reference.py) pinned to
hand-written answers, and its three identities: every minimum 1 is the OR-group statement (phrase_groups_reference.py);
a minimum equal to the group's size is the clause conjunction of its alternatives (phrase_and_reference.py); one-slot
alternatives of distinct terms are the term OR groups with minimums (min_match_reference.py). Runs without a GPU."""
import numpy as np
import pytest

import min_match_reference as mmr
import phrase_and_reference as par
import phrase_groups_reference as pgr
import phrase_min_match_reference as pmr
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


NEW, YORK, CITY, NYC, BIG, APPLE, PIZZA = range(7)


def test_two_of_new_york_nyc_big_apple():
    docs = [[NEW, YORK, NYC], [NYC, BIG, APPLE], [NEW, YORK], [NYC, PIZZA], [YORK, NEW, NYC], [BIG, APPLE, NEW, YORK, NYC]]
    q = [G([NEW, YORK], [NYC], [BIG, APPLE])]
    ds, fs = pmr.match(docs, q, mins=[2])
    assert ds.tolist() == [1, 2, 6]
    assert fs == [[1, 1, 0], [0, 1, 1], [1, 1, 1]]
    assert pmr.match(docs, q, mins=[3])[0].tolist() == [6]
    # with pizza: an AND of the minimum group and a term
    assert pmr.match(docs, [q[0], G([PIZZA])], mins=[1, 1])[0].tolist() == [4]
    assert pmr.match(docs, [q[0], G([PIZZA])], mins=[2, 1])[0].tolist() == []


def test_duplicate_alternatives_each_count():
    """2 of (a | a | b): a doc holding a alone has two alternatives that occur; it matches, scored twice on a."""
    docs = [[NYC], [PIZZA], [NYC, PIZZA], [BIG]]
    q = [G([NYC], [NYC], [PIZZA])]
    ds, fs = pmr.match(docs, q, mins=[2])
    assert ds.tolist() == [1, 3]
    assert fs == [[1, 1, 0], [1, 1, 1]]
    got = pmr.scores(docs, q, ds, fs, None, [C0, C0, C1])
    want = [f32(f32(f32(0) + pr.score(1, 1, *C0)) + pr.score(1, 1, *C0)),
            f32(f32(f32(f32(0) + pr.score(1, 1, *C0)) + pr.score(1, 1, *C0)) + pr.score(1, 1, *C1))]
    assert _bits(got) == _bits(want)
    # 3 of it needs b too
    assert pmr.match(docs, q, mins=[3])[0].tolist() == [3]


def test_phrases_sharing_their_proxy_term():
    """2 of ("new york" | "york city" | nyc): "new york city" holds both phrases and matches without nyc."""
    docs = [[NEW, YORK, CITY], [NEW, YORK], [YORK, CITY, NYC], [NYC, YORK], [CITY, YORK, NEW]]
    q = [G([NEW, YORK], [YORK, CITY], [NYC])]
    ds, fs = pmr.match(docs, q, mins=[2])
    assert ds.tolist() == [1, 3]
    assert fs == [[1, 1, 0], [0, 1, 1]]


def test_repeated_term_inside_a_phrase():
    """"new new" counts its anchors only where the repeat holds; 2 of ("new new" | york)."""
    docs = [[NEW, NEW, YORK], [NEW, YORK, NEW], [NEW, NEW, NEW], [YORK]]
    q = [G([NEW, NEW], [YORK])]
    ds, fs = pmr.match(docs, q, mins=[2])
    assert ds.tolist() == [1]
    assert fs == [[1, 1]]
    assert pmr.match(docs, q, mins=[1])[1] == [[1, 1], [0, 1], [2, 0], [0, 1]]


def test_doc_with_more_than_m_alternatives_is_scored_on_all():
    docs = [[NEW, YORK, NYC, BIG, APPLE], [NYC, BIG, APPLE], [NYC]]
    q = [G([NEW, YORK], [NYC], [BIG, APPLE])]
    ds, fs = pmr.match(docs, q, mins=[2])
    assert ds.tolist() == [1, 2]
    norms = np.array([len(d) for d in docs], np.uint32)
    # docs_count: "new york" 1, nyc 3, "big apple" 2: cost order new york, big apple, nyc
    assert pmr.cost_order(docs, q) == [0, 2, 1]
    got = pmr.scores(docs, q, ds, fs, norms, [C0, C1, C2])
    want = [f32(f32(f32(f32(0) + pr.score(1, 5, *C0)) + pr.score(1, 5, *C2)) + pr.score(1, 5, *C1)),
            f32(f32(f32(0) + pr.score(1, 3, *C2)) + pr.score(1, 3, *C1))]
    assert _bits(got) == _bits(want)


def test_segment_lacking_a_term_cannot_reach_m():
    """Segment 1 holds no nyc: 2 of (pizza | nyc | "big apple") needs both of the others there."""
    seg0 = [[PIZZA, NYC], [BIG, APPLE], [PIZZA, BIG, APPLE]]
    seg1 = [[PIZZA], [PIZZA, BIG, APPLE], [BIG, APPLE]]
    q = [G([PIZZA], [NYC], [BIG, APPLE])]
    m = pmr.matches([seg0, seg1], q, mins=[2])
    assert m[0][0].tolist() == [1, 3] and m[1][0].tolist() == [2]
    assert pmr.count(m) == 3
    # 3 of it: no doc in either segment
    assert pmr.count(pmr.matches([seg0, seg1], q, mins=[3])) == 0


def test_minimum_group_next_to_a_negated_phrase():
    docs = [[NEW, YORK, NYC], [NYC, PIZZA, NEW, YORK], [NYC, BIG, APPLE]]
    q = [G([NEW, YORK], [NYC], [BIG, APPLE]), G([NYC, PIZZA], neg=True)]
    assert pmr.match(docs, q, mins=[2, 1])[0].tolist() == [1, 3]


def test_statement_refuses_out_of_range_minimums():
    q = [G([NEW], [NYC]), G([PIZZA], neg=True)]
    for mins in ([0, 1], [3, 1], [1, 2]):
        with pytest.raises(AssertionError):
            pmr.match([[NEW]], q, mins=mins)


def _corpus(seed, n=300, vocab=8):
    rng = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, vocab + 1)
    p /= p.sum()
    return [rng.choice(vocab, size=int(rng.integers(1, 25)), p=p).tolist() for _ in range(n)]


QUERIES = [
    [G([0, 1], [2], [3, 4]), G([5])],
    [G([1, 0], [0, 1], [2]), G([3], [4, 5], neg=True)],
    [G([0], [1], [2], [3]), G([4, 5], [6])],
]


@pytest.mark.parametrize("q", QUERIES)
def test_identity_every_minimum_one_is_the_or_groups(q):
    segs = [_corpus(s) for s in (1, 2)]
    norms = [np.array([len(d) for d in docs], np.uint32) for docs in segs]
    consts = [None if n else (f32(0.5 + 0.2 * j), f32(1.1), f32(0.3)) for j, (_, _, n) in enumerate(pgr.flat(q))]
    for mins in (None, [1] * len(q)):
        got, want = pmr.matches(segs, q, excl=[7], mins=mins), pgr.matches(segs, q, excl=[7])
        for (gd, gf), (wd, wf) in zip(got, want):
            assert gd.tolist() == wd.tolist() and gf == wf
        h, t = pmr.topk(segs, q, got, norms, consts, 30)
        h2, t2 = pgr.topk(segs, q, want, norms, consts, 30)
        assert t == t2 and h.tobytes() == h2.tobytes()


def test_identity_minimum_equal_to_size_is_the_clause_conjunction():
    segs = [_corpus(s) for s in (3, 4)]
    norms = [np.array([len(d) for d in docs], np.uint32) for docs in segs]
    q = [G([0, 1], [2], [3]), G([4], [5, 6], neg=True)]
    clauses = [([0, 1], None, False), ([2], None, False), ([3], None, False), ([4], None, True), ([5, 6], None, True)]
    consts = [C0, C1, C2, None, None]
    got, want = pmr.matches(segs, q, mins=[3, 1]), par.matches(segs, clauses)
    for (gd, gf), (wd, wf) in zip(got, want):
        assert gd.tolist() == wd.tolist() and gf == wf
    h, t = pmr.topk(segs, q, got, norms, consts, 40)
    h2, t2 = par.topk(segs, clauses, want, norms, consts, 40)
    assert t == t2 and h.tobytes() == h2.tobytes()


def _lists(docs, vocab=8):
    return [np.array([i + 1 for i, s in enumerate(docs) if t in s], np.uint32) for t in range(vocab)]


@pytest.mark.parametrize("groups_terms,mins", [([[0, 1, 2], [3]], [2, 1]), ([[3, 1, 4, 0], [5, 2]], [3, 2]),
                                               ([[0, 1, 2, 3, 4, 5]], [4]), ([[0, 6], [1, 2, 3]], [1, 2])])
def test_identity_one_slot_alternatives_are_the_min_match_groups(groups_terms, mins):
    segs = [_corpus(s) for s in (5, 6, 7)]
    groups = [([([t], None) for t in g], False) for g in groups_terms]
    got = pmr.matches(segs, groups, excl=[7], mins=mins)
    for docs, (gd, _) in zip(segs, got):
        assert gd.tolist() == mmr.match_docs(_lists(docs), groups_terms, [7], mins=mins).tolist()


def test_engine_min_match_argument():
    from serenedb_b200 import engine as E

    queries = [[[[0, 1], [2], [3]], [[4]]], [[[5], [6]]]]
    groups = E._phrase_groups(queries, [[[7, 8]], None])
    got = E._phrase_group_min([[2, 1], [1]], queries, groups)
    assert got.dtype == np.uint32 and got.tolist() == [2, 1, 1, 1]    # the negated group of exclude_phrases takes 1
    assert E._phrase_group_min(None, queries, groups) is None
    for bad in ([[2, 1]], [[2], [1]], [[2, 1], [1, 1]], [[2, -1], [1]]):
        with pytest.raises(ValueError):
            E._phrase_group_min(bad, queries, groups)
