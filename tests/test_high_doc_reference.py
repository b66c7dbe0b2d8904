"""CPU guards of the doc-id-domain corpus (tests/high_doc_reference.py) and the doc-count limits that need no device:
the corpus reaches every encoding and landmark it is meant to, the NumPy restatement of the synthetic column matches
the generator up to 2^32 - 2, the remap keeps every list's order, and the host entries refuse doc counts outside
1 .. 2^32 - 2 instead of truncating them."""
import ctypes as C

import numpy as np
import pytest

import high_doc_reference as hd
import orc
import serenedb_b200 as sdb
from gpu_util import metas_of
from serenedb_b200 import _native

DE_VALUES, DE_SAME32, DE_BITSET, DE_SVB, DE_DELTA_SVB, DE_BITPACK31 = 0, 3, 4, 5, 7, 8 + 31 - 2


@pytest.fixture(scope="module")
def corpus():
    c = hd.TopCorpus()
    o = c.oracle_segment()
    return c, o, sdb.stage_parse_host(o.doc_bytes(), metas_of(o), has_wand=True)


def test_every_encoding_reaches_the_top(corpus):
    c, o, st = corpus
    enc = {name: hd.encodings(st, t) for name, t in c.names.items()}
    e, last = enc["raw_block"]
    assert e[0] == DE_VALUES and last[0] == 2 ** 31 + 300 and e[1] == DE_DELTA_SVB
    e, last = enc["bits31_across"]
    assert e[1] == DE_BITPACK31 and last[1] > 2 ** 31
    e, last = enc["same32_top"]
    assert e[1] == DE_SAME32 and last[1] == hd.TOP
    e, last = enc["same32_pair"]
    assert e == [DE_SAME32] and last[0] == hd.TOP
    e, last = enc["bitset_top"]
    assert e == [DE_VALUES, DE_BITSET] and last[1] == hd.TOP
    e, last = enc["dsvb_high"]
    assert e[1] == DE_DELTA_SVB and last[1] > 2 ** 31 + 2 ** 24
    e, last = enc["raw_tail_high"]
    assert e == [DE_VALUES] and last[0] == 2 ** 32 - 3
    e, last = enc["svb_high"]
    assert e == [DE_SVB] and last[0] == 2 ** 31 + 5
    e, last = enc["svb_top"]
    assert e[1] == DE_SVB and last[1] == hd.TOP
    for name, doc in (("single_2^31", 2 ** 31), ("single_top", hd.TOP)):
        t = c.names[name]
        assert o.term_meta(t).docs_count == 1 and int(o.term_meta(t).e_skip_start) + 1 == doc
        assert hd.encodings(st, t)[1].tolist() == [doc]
    # the staged block table and the oracle's decoder give back every list as written
    for t, (name, d, f) in enumerate(c.lists):
        od, of = o.decode_term(t)
        assert np.array_equal(od, d) and np.array_equal(of, f), name
        b0, b1 = st["term_blk_begin"][t], st["term_blk_begin"][t + 1]
        assert st["last_doc"][b1 - 1] == d[-1] and np.all(np.diff(st["last_doc"][b0:b1].astype(np.int64)) > 0), name


def test_landmarks_are_list_and_deleted_docs(corpus):
    c, _, _ = corpus
    every = np.unique(np.concatenate([d for _, d, _ in c.lists]))
    for x in hd.LANDMARKS:
        assert x in every and x in c.deleted and x in c.lists[c.names["landmarks"]][1], x
    assert every[-1] == hd.TOP and (every > 2 ** 31).sum() > 1000
    # deleted docs in every part of the range: the count kernel must mask past its first words
    assert (c.deleted < 32).sum() < len(c.deleted) // 2 and (c.deleted > 2 ** 32 - hd.WINDOW).any()


def test_remap_is_monotone(corpus):
    c, _, _ = corpus
    assert np.all(np.diff(c.U.astype(np.int64)) > 0)
    for _, d, _ in c.lists:
        s = c.small(d)
        assert np.all(np.diff(s.astype(np.int64)) > 0) and np.array_equal(c.big(s), d)


def test_synth_column_restatement_matches_generator():
    rows = np.array([0, 1, 2 ** 31 - 2, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 4096, 2 ** 32 - 3], np.uint64)
    rows = np.concatenate([rows, np.random.default_rng(0).integers(0, 2 ** 32 - 2, 200).astype(np.uint64)])
    for r in rows:   # the device's kind 6 is int32(h % 1000000): the oracle's kind 1 gives the same values as int64
        assert hd.full_values([int(r) + 1])[0] == orc.synth_column(hd.FULL_STREAM, 1, int(r), 1)[0], r
        assert hd.synth_hash(9, [int(r)])[0] == orc.lib().orc_synth_hash(9, int(r))
    want = orc.synth_column(hd.SHORT_STREAM, 0, 0, 4096)   # kind 0 is h % 100000: the same hashes
    got = hd.synth_hash(hd.SHORT_STREAM, np.arange(4096, dtype=np.uint64)) % np.uint64(100000)
    assert np.array_equal(got.astype(np.int64), want)


@pytest.mark.parametrize("n", [0, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 5, -1])
def test_engine_rejects_doc_counts_outside_the_id_range(n):
    with pytest.raises(ValueError):
        sdb.PostingsWriter(n)
    with pytest.raises(ValueError):   # checked before the context is touched
        sdb.Segment(None, n)


def test_writer_takes_the_largest_segment():
    w = sdb.PostingsWriter(hd.TOP, has_wand=True)
    w.add_term(np.array([2 ** 31, hd.TOP], np.uint32), np.array([1, 2], np.uint32))
    doc, metas = w.finish()
    o = orc.Segment(hd.TOP, has_wand=True)
    o.add_term(np.array([2 ** 31, hd.TOP], np.uint32), np.array([1, 2], np.uint32))
    assert np.array_equal(doc, o.doc_bytes()) and metas["docs_count"].tolist() == [2]
    h = C.c_void_p()
    assert _native.ERR[_native.lib().sdbg_writer_create(2 ** 32 - 1, 1, 0.75, None, C.byref(h))] == "EINVAL"
    assert not h.value


def test_split_corpus_reaches_the_top_ordinals():
    s = hd.SplitCorpus()
    a, b = s.segs
    assert a.n_docs + b.n_docs == hd.TOP and a.n_docs > 2 ** 31 and b.base == a.n_docs
    for c in (a, b):
        every = np.unique(np.concatenate([d for _, d, _ in c.lists]))
        assert every[-1] == c.n_docs and c.deleted[-1] == c.n_docs
        o = c.oracle_segment()
        st = sdb.stage_parse_host(o.doc_bytes(), metas_of(o), has_wand=c.has_wand)
        for t, (name, d, f) in enumerate(c.lists):
            od, of = o.decode_term(t)
            assert np.array_equal(od, d) and np.array_equal(of, f), name
            assert st["last_doc"][st["term_blk_begin"][t + 1] - 1] == d[-1], name
    assert int(b.base) + int(b.n_docs) == hd.TOP               # the last key ordinal is 2^32 - 2
    assert (np.unique(np.concatenate([d for _, d, _ in a.lists])) > 2 ** 31).sum() > 100   # norm rows past 2^31
    assert np.array_equal(b.values([1, 7]), hd.full_values([a.n_docs + 1, a.n_docs + 7]))


def test_split_norms_are_periodic():
    d = np.array([1, 2, 250, 251, 2 ** 31 - 1, 2 ** 31, hd.SPLIT_A - 251], np.uint64)
    n = hd.split_norm(d)
    assert np.array_equal(n, hd.split_norm(d + np.uint64(251))) and n.min() >= 1 and n.max() <= 251
    assert hd.split_norm_sum() == int(hd.split_norm(np.arange(1, hd.SPLIT_A % 251 + 1)).sum()) + \
        hd.SPLIT_A // 251 * int(hd.split_norm(np.arange(1, 252)).sum())
