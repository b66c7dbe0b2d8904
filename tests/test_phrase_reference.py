"""The NumPy statement of phrase queries (tests/phrase_reference.py) against hand-written answers, and a one-slot phrase
against the count reference's single-term result. No GPU needed."""
import numpy as np

import count_reference as cr
import phrase_reference as pr

A, B_, C_, D = 0, 1, 2, 3


def test_overlapping_matches_count():
    assert pr.phrase_freq([A, A, A], [A, A]) == 2
    assert pr.phrase_freq([A, A, A, A], [A, A, A]) == 2


def test_repeated_term():
    # "to be or not to be"
    seq = [0, 1, 2, 3, 0, 1]
    assert pr.phrase_freq(seq, [0, 1, 2, 3, 0, 1]) == 1
    assert pr.phrase_freq(seq, [0, 1]) == 2
    assert pr.phrase_freq(seq + [9], [0, 1, 2, 3, 0, 1]) == 1
    assert pr.phrase_freq([0, 1, 2, 3, 1, 0], [0, 1, 2, 3, 0, 1]) == 0


def test_gaps_through_rel_pos():
    seq = [A, D, B_, C_, A, B_]
    assert pr.phrase_freq(seq, [A, B_], [0, 2]) == 1          # "a _ b"
    assert pr.phrase_freq(seq, [A, B_]) == 1                   # the adjacent pair at the end
    assert pr.phrase_freq(seq, [A, C_], [0, 3]) == 1
    assert pr.phrase_freq(seq, [A, C_], [0, 2]) == 0


def test_first_and_last_positions():
    assert pr.phrase_freq([A, B_, C_, C_], [A, B_]) == 1
    assert pr.phrase_freq([C_, C_, A, B_], [A, B_]) == 1
    assert pr.phrase_freq([A, B_], [A, B_]) == 1
    assert pr.phrase_freq([A], [A, B_]) == 0                   # the phrase runs past the doc's end


def test_not_adjacent_or_reversed():
    assert pr.phrase_freq([A, C_, B_], [A, B_]) == 0
    assert pr.phrase_freq([B_, A], [A, B_]) == 0
    assert pr.phrase_freq([B_, C_, A], [A, B_]) == 0


def test_match_exclusions_and_deleted():
    docs = [[A, B_], [A, B_, C_], [C_, A, B_, A, B_], [B_, A], [A, B_, D]]
    d, f = pr.match(docs, [A, B_])
    assert d.tolist() == [1, 2, 3, 5] and f.tolist() == [1, 1, 2, 1]
    d, _ = pr.match(docs, [A, B_], excl=[C_])
    assert d.tolist() == [1, 5]
    d, _ = pr.match(docs, [A, B_], excl=[C_], deleted=[5])
    assert d.tolist() == [1]
    d, _ = pr.match(docs, [A, B_], mask=np.array([False, True, True, True, True]))
    assert d.tolist() == [2, 3, 5]
    assert pr.count([docs, [[A, B_]]], [A, B_], excl=[D]) == 4


def test_postings_and_staging_layout():
    docs = [[A, B_, A], [B_], [A]]
    post = pr.postings(docs, 2)
    assert post[A][0].tolist() == [1, 3] and post[A][1].tolist() == [2, 1] and post[A][2].tolist() == [0, 2, 0]
    pos, off = pr.staged_positions(post)
    assert off.tolist() == [0, 3, 5] and pos.tolist() == [0, 2, 0, 1, 0]


def test_one_slot_is_the_term():
    rng = np.random.default_rng(3)
    docs = [rng.integers(0, 6, rng.integers(1, 12)).tolist() for _ in range(400)]
    post = pr.postings(docs, 6)
    lists = [d for d, _, _ in post]
    deleted = [5, 17, 200]
    for t in range(6):
        d, f = pr.match(docs, [t], deleted=deleted)
        assert d.tolist() == cr.match_docs(lists, "AND", [t], deleted=deleted).tolist()
        keep = np.isin(post[t][0], d)
        assert f.tolist() == post[t][1][keep].tolist()


def test_scores_every_form():
    class S:
        idf, norm_const, norm_length, boost = np.float32(1.5), np.float32(0.3), np.float32(0.009), 1.0
    c = pr.consts(S, 1.2, 0.75)
    assert c[0] == np.float32(np.float32(np.float32(1.0) * np.float32(2.2)) * np.float32(1.5))
    s1, s2 = pr.score(1, 100, *c), pr.score(2, 100, *c)
    assert 0 < s1 < s2 < c[0]
    assert pr.score(2, 100, *pr.consts(S, 0.0, 0.75)) == 0
    bm15 = pr.consts(S, 1.2, 0.0)
    assert pr.score(2, 100, *bm15) == pr.score(2, 7, *bm15)     # no norms
    tf = pr.consts(S, -1, 1.0)
    assert pr.score(4, 16, *tf) == np.float32(np.float32(2 * 1.5) / np.float32(4))


def test_phrase_stats_sum_the_idfs_in_slot_order():
    """IndexReader.phrase_stats against a hand-computed float32 sum of the slots' idfs (a repeated term once per slot),
    with the first slot's norm constants and the given boost applied once."""
    import serenedb_b200 as sdb

    reader = sdb.IndexReader([], 10_000, 123_456, [7, 4000, 250, 9000])
    for scorer in (sdb.BM25(), sdb.BM25(1.5, 0.0), sdb.TFIDF(True)):
        idf = [np.float32(reader.stats(scorer, t).idf) for t in range(4)]
        for slots, boost in (([0, 1], 1.0), ([2, 0, 2, 3], 1.0), ([1, 1, 1], 2.5), ([3], 1.0)):
            want = np.float32(0)
            for t in slots:
                want = np.float32(want + idf[t])
            got = reader.phrase_stats(scorer, slots, boost)
            assert np.float32(got.idf) == want, (slots, float(got.idf), float(want))
            first = reader.stats(scorer, slots[0])
            assert (np.float32(got.norm_const), np.float32(got.norm_length)) == (np.float32(first.norm_const),
                                                                                 np.float32(first.norm_length))
            assert got.boost == boost
    # a repeated term is not summed once: "a a" doubles the idf of "a"
    assert np.float32(reader.phrase_stats(sdb.BM25(), [1, 1]).idf) == np.float32(2 * np.float32(reader.stats(sdb.BM25(), 1).idf))
