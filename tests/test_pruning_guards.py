"""CPU guards for the GPU pruning and posting-shape tests: the shape corpora really reach every block encoding they are
meant to reach (an encoder change must not quietly empty the matrix), and the block-max bound rule of fill_qterm holds
where the stored pair alone does not."""
import numpy as np
import pytest

from gpu_util import metas_of
from serenedb_b200.engine import stage_parse_host
from shape_corpora import (B, K1, NORM_WIDTHS, SHAPE_SPAN, bm25_f32, bound_consts, shape_segment, stored_pair,
                           writer_avg_dl)

# block descriptor encodings (posting_format.hpp)
DE_VALUES, DE_SAME08, DE_SAME16, DE_SAME32, DE_BITSET, DE_SVB, DE_DSVB, DE_BITPACK02 = 0, 1, 2, 3, 4, 5, 7, 8
E_VALUES, E_SAME08, E_SAME16, E_SAME32, E_SVB, E_BITPACK01 = 0, 1, 2, 3, 4, 5


def _blocks(width):
    oseg, _, lists = shape_segment(width)
    st = stage_parse_host(oseg.doc_bytes(), metas_of(oseg))
    p = st["packed"].astype(np.int64)
    blk = dict(doc=p & 63, freq=(p >> 6) & 63, len=((p >> 12) & 127) + 1, words=p >> 25)
    names = np.empty(len(p), object)
    tb = st["term_blk_begin"]
    for t, (name, _, _) in enumerate(lists):
        names[tb[t]:tb[t + 1]] = name
    blk["name"] = names
    return blk


def _payload(enc, n, words, doc):
    """Bytes of one block's doc or freq payload, from its encoding (posting_format.hpp doc/freq_payload_bytes)."""
    if doc:
        sizes = {DE_VALUES: 4 * n, DE_SAME08: 1, DE_SAME16: 2, DE_SAME32: 4, DE_BITSET: 8 * words}
        return sizes.get(enc, 16 * (enc - 6) if enc >= DE_BITPACK02 else None)
    sizes = {E_VALUES: 4 * n, E_SAME08: 1, E_SAME16: 2, E_SAME32: 4}
    return sizes.get(enc, 16 * (enc - 4) if enc >= E_BITPACK01 else None)


@pytest.fixture(scope="module")
def staged():
    return {w: _blocks(w) for w in NORM_WIDTHS}


def test_shape_corpora_reach_every_encoding(staged):
    doc = set().union(*(set(b["doc"].tolist()) for b in staged.values()))
    freq = set().union(*(set(b["freq"].tolist()) for b in staged.values()))
    assert {DE_BITPACK02 + w - 2 for w in range(2, 32)} <= doc                      # doc widths 2..31
    assert {DE_VALUES, DE_SAME08, DE_SAME16, DE_SAME32, DE_BITSET, DE_SVB, DE_DSVB} <= doc
    assert {E_BITPACK01 + w - 1 for w in range(2, 32)} <= freq                      # freq widths 2..31
    assert {E_VALUES, E_SAME08, E_SAME16, E_SAME32, E_SVB} <= freq
    for w, b in staged.items():
        if w is None:
            continue
        # every width that fits the 2^24-doc span is there in a full block, for every norm width
        full = b["len"] == 128
        assert {DE_BITPACK02 + x - 2 for x in range(2, 25)} <= set(b["doc"][full].tolist()), w
        assert {E_BITPACK01 + x - 1 for x in range(2, 32)} <= set(b["freq"][full].tolist()), w
        assert {DE_SAME32, DE_BITSET, DE_SVB, DE_DSVB} <= set(b["doc"].tolist()), w
    # raw doc tails (ids and gaps >= 2^24) and the widest full blocks live in the segment without norms
    nb = staged[None]
    assert DE_VALUES in set(nb["doc"][nb["len"] < 128].tolist())
    assert {DE_BITPACK02 + x - 2 for x in range(25, 32)} <= set(nb["doc"][nb["len"] == 128].tolist())
    assert SHAPE_SPAN[None] > 2 ** 30


def test_shape_corpora_bitsets_and_wide_blocks(staged):
    b = staged[2]
    words = b["words"][b["doc"] == DE_BITSET]
    full_words = b["words"][(b["doc"] == DE_BITSET) & (b["len"] == 128)]
    # one-word tails up to the widest full-block bitset the encoder picks over bit-packing
    assert words.min() == 1 and full_words.min() <= 3 and full_words.max() >= 20, sorted(set(words.tolist()))
    for w, b in staged.items():
        sizes = [_payload(int(d), int(n), int(wd), True) + _payload(int(f), int(n), 0, False)
                 for d, f, n, wd in zip(b["doc"], b["freq"], b["len"], b["words"])
                 if _payload(int(d), int(n), int(wd), True) is not None and _payload(int(f), int(n), 0, False) is not None]
        assert max(sizes) > 512, w                                                    # beyond the prefetch slot


# ---------------------------------------------------------------- the bound rule (fill_qterm / bound_consts)
def test_block_max_bound_rule_property():
    """Random blocks (up to 128 postings, 1 <= tf <= dl <= 300) and random segment / query averages: the stored pair scored
    with the query's constants falls below the block's real best in some blocks; scored with the bound constants, never.
    float32 with the kernel's operation order and its 1.000001 margin."""
    rng = np.random.default_rng(12)
    k1, b = np.float32(K1), np.float32(B)
    nc = k1 - k1 * b
    old_bad = new_bad = 0
    for _ in range(3000):
        n = int(rng.integers(2, 129))
        dl = rng.integers(1, 301, n).astype(np.uint32)
        tf = np.minimum(rng.geometric(0.3, n), dl).astype(np.uint32)
        a_s = np.float32(rng.uniform(1.0, 300.0))
        a_q = np.float32(a_s * rng.choice([rng.uniform(0.8, 1.25), rng.uniform(0.02, 50.0)]))
        nl = (k1 * b) / a_q
        c0 = np.float32(rng.uniform(0.1, 10.0))
        f, nrm = stored_pair(tf, dl, a_s)
        best = bm25_f32(tf, dl, c0, nc, nl).max()
        old = bm25_f32(f, nrm, c0, nc, nl)
        bnc, bnl = bound_consts(nc, nl, k1, b, a_s)
        new = bm25_f32(f, nrm, c0, bnc, bnl)
        old_bad += bool(old * np.float32(1.000001) < best)
        new_bad += bool(new * np.float32(1.000001) < best)
    assert old_bad > 0
    assert new_bad == 0


def test_bound_consts_equal_query_constants_at_equal_averages():
    """A single segment (segment average == corpus average): the bound constants are the query's, bit for bit, so
    single-segment pruning is unchanged."""
    for avg in (np.float32(2.0), np.float32(137.25), np.float32(1e4 / 3)):
        k1, b = np.float32(K1), np.float32(B)
        nc, nl = k1 - k1 * b, (k1 * b) / avg
        bnc, bnl = bound_consts(nc, nl, k1, b, avg)
        assert bnc.view(np.uint32) == nc.view(np.uint32) and bnl.view(np.uint32) == nl.view(np.uint32)


def test_writer_avg_matches_norm_reader_definition():
    norms = np.array([0, 3, 5, 0, 9], np.uint32)
    assert writer_avg_dl(norms) == np.float32(17 / 3)
    assert writer_avg_dl(np.zeros(4, np.uint32)) == 0
