"""Corpus and references for the doc-id domain's top: doc ids at and above 2^31, up to the last valid id 2^32 - 2
(doc_limits::eof() = 2^32 - 1 is never a doc).

The corpus is a set of sparse lists placed at landmarks, with no norm column (every doc has norm 1), so nothing is
allocated per doc on the host. Every block encoding the writer can give a doc id up there appears at least once; the
CPU guard in test_high_doc_reference.py checks that on the staged block table.

The oracle has never been run at these ids, and it walks docs with the same uint32 loops as the product. So results
are checked against two independent statements instead:
- A monotone remap. The sorted set U of every doc that matters (list docs, deleted docs) is mapped onto 1..|U|, and
  the segment is rebuilt small with the same lists, freqs, norms (all 1), deleted docs and column values at the
  mapped docs. Scores depend only on freq, norm and the IndexReader statistics, which both segments get explicitly;
  ties go by (segment, doc), whose order a monotone map keeps. So the small segment's oracle result, mapped back
  through U, must equal the GPU's bit for bit.
- The NumPy references (count_reference, sort_reference, facet_reference) on the lists themselves, with per-row
  inputs given for the matched rows only.

TEST INFRASTRUCTURE: imported by tests only."""
import numpy as np

import orc
from shape_corpora import companion

TOP = 2 ** 32 - 2            # the last valid doc id, and the doc count of the `top` segment
EOF = 2 ** 32 - 1            # doc_limits::eof()
WINDOW = 65536               # the count / sorted-scan window (bm25_count.cuh)
ZONE = 2048                  # zonemap rows
SHORT_ROWS = 1 << 20         # rows of the short column: docs past it are NULL there

# doc ids every path must get right
LANDMARKS = sorted({
    2 ** 31 - 1, 2 ** 31, 2 ** 31 + 1,
    # the last full windows' boundaries (window w holds docs w * 65536 .. w * 65536 + 65535)
    2 ** 32 - 2 * WINDOW - 1, 2 ** 32 - 2 * WINDOW, 2 ** 32 - 2 * WINDOW + 1,
    2 ** 32 - WINDOW - 1, 2 ** 32 - WINDOW, 2 ** 32 - WINDOW + 1,
    # the last zones' boundaries (zone z holds rows 2048 z .. 2048 z + 2047, row = doc - 1)
    2 ** 32 - 2 * ZONE, 2 ** 32 - 2 * ZONE + 1, 2 ** 32 - ZONE, 2 ** 32 - ZONE + 1,
    # inside the last, partial window
    2 ** 32 - 1000, 2 ** 32 - 3, TOP,
})

FULL_FIELD, SHORT_FIELD = 21, 22
FULL_STREAM, SHORT_STREAM = 77, 78
FULL_KIND = 6                # synth_column kind 6: int32 h % 1000000


# ---------------------------------------------------------------- the synthetic column generator, restated
_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def synth_hash(stream, index):
    """splitmix64 finaliser over seed ^ (stream << 48) ^ index (SURVEY §8d) on a uint64 array; NumPy's uint64 arithmetic
    wraps modulo 2^64 like the C code."""
    idx = np.asarray(index, np.uint64)
    with np.errstate(over="ignore"):
        z = (np.uint64(0x5EDB2026) ^ np.uint64((int(stream) << 48) & 0xFFFFFFFFFFFFFFFF) ^ idx) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def full_values(docs):
    """The full-length int32 column (synth_column kind 6 from row 0) at the given docs (row = doc - 1)."""
    rows = np.asarray(docs, np.uint64) - np.uint64(1)
    return (synth_hash(FULL_STREAM, rows) % np.uint64(1000000)).astype(np.int32)


def short_column():
    """The short int32 column: SHORT_ROWS rows, so every doc past SHORT_ROWS is NULL in it."""
    return (synth_hash(SHORT_STREAM, np.arange(SHORT_ROWS, dtype=np.uint64)) % np.uint64(5000)).astype(np.int32)


# ---------------------------------------------------------------- corpus
def _f(rng, n, hi=4):
    return rng.integers(1, hi, n).astype(np.uint32)


def shape_terms(rng):
    """[(name, docs, freqs)]: one list per encoding that reaches the top of the id range, then the long lists."""
    out = []
    head = np.arange(1, 128, dtype=np.uint32)
    # a full block stored as raw values: one gap >= 2^31 makes bit-packing 32 bits wide; then a delta-StreamVByte tail
    d = np.concatenate([head, [2 ** 31 + 300], [2 ** 31 + 301, 2 ** 31 + 305, 2 ** 31 + 900]]).astype(np.uint32)
    out.append(("raw_block", d, _f(rng, len(d))))
    # bit-packed width-31 gaps in a block that crosses 2^31
    blk = np.concatenate([2 ** 31 - 200 + 3 * np.arange(64), 2 ** 31 + 2 ** 30 + 7 + 3 * np.arange(64)])
    d = np.concatenate([np.arange(1, 129), blk]).astype(np.uint32)
    out.append(("bits31_across", d, _f(rng, len(d))))
    # all-same gaps >= 2^31 ending at 2^32 - 2: a one-doc tail after a full block (Same32, gap 2^32 - 130)
    d = np.concatenate([np.arange(1, 129), [TOP]]).astype(np.uint32)
    out.append(("same32_top", d, _f(rng, len(d))))
    # all-same gaps of 2^31 - 1: the two-doc list 2^31 - 1, 2^32 - 2
    out.append(("same32_pair", np.array([2 ** 31 - 1, TOP], np.uint32), _f(rng, 2)))
    # a full block at the top stored raw (its first gap is ~2^32), then a bitset block whose last doc is 2^32 - 2
    cand = np.arange(TOP - 269, TOP + 1, dtype=np.uint32)
    keep = np.sort(rng.choice(len(cand) - 1, 255, replace=False))
    d = np.concatenate([cand[keep], [TOP]]).astype(np.uint32)
    out.append(("bitset_top", d, _f(rng, len(d))))
    # a full bit-packed block above 2^31, then a delta-StreamVByte tail with a 4-byte gap
    d = (2 ** 31 + 1 + np.cumsum(rng.integers(1, 8, 128))).astype(np.uint64)
    tail = d[-1] + np.cumsum([3, 300, 70000, 2 ** 24 + 5, 7, 1])
    d = np.concatenate([d, tail]).astype(np.uint32)
    out.append(("dsvb_high", d, _f(rng, len(d))))
    # a tail of 4-byte ids above 2^31 with 4-byte gaps: raw values (StreamVByte would be larger)
    d = np.array([2 ** 31 + 2 ** 28, 2 ** 31 + 2 ** 29 + 1, 2 ** 32 - 2 ** 20, 2 ** 32 - 3], np.uint32)
    out.append(("raw_tail_high", d, _f(rng, len(d))))
    # absolute StreamVByte tails with a 4-byte value above 2^31: absolute and delta coding tie at 10 bytes (raw: 16), and
    # the writer keeps the absolute form on a tie; alone, and after a full block
    out.append(("svb_high", np.array([1, 2, 3, 2 ** 31 + 5], np.uint32), _f(rng, 4)))
    d = np.concatenate([np.arange(1, 129), [130, 131, TOP]]).astype(np.uint32)
    out.append(("svb_top", d, _f(rng, len(d))))
    # single-doc terms, inline in the term meta
    out.append(("single_2^31", np.array([2 ** 31], np.uint32), np.array([3], np.uint32)))
    out.append(("single_top", np.array([TOP], np.uint32), np.array([2], np.uint32)))
    # every landmark in one list, with a few low docs (and rows of the short column)
    d = np.unique(np.concatenate([[1, 2, 1000, SHORT_ROWS - 1, SHORT_ROWS, SHORT_ROWS + 1], LANDMARKS])).astype(np.uint32)
    out.append(("landmarks", d, _f(rng, len(d), 6)))
    # long lists: uniform over the whole range, dense near 2^31 and in the last windows, low docs for the short column
    for name, n in (("spread_a", 6000), ("spread_b", 3000)):
        parts = [rng.integers(1, TOP + 1, n), rng.integers(2 ** 31 - 40000, 2 ** 31 + 40000, n // 3),
                 rng.integers(TOP - 3 * WINDOW, TOP + 1, n // 2), rng.integers(1, SHORT_ROWS + 5000, n // 6), LANDMARKS]
        d = np.unique(np.concatenate(parts)).astype(np.uint32)
        out.append((name, d, _f(rng, len(d), 8)))
    return out


class SegCorpus:
    """One segment's lists [(name, docs, freqs)] by term id, its deleted docs and the remap set U (every list doc and
    deleted doc). `base`: ordinals of the earlier segments of its call; the full-length column continues the rows of
    those segments, so its value at doc d is full_values(base + d). `norm`: doc ids -> norms (None: no norm column)."""

    def __init__(self, n_docs, lists, deleted, base=0, norm=None, has_wand=True):
        self.n_docs, self.lists, self.base, self.norm, self.has_wand = n_docs, lists, base, norm, has_wand
        for name, d, _ in lists:
            assert np.all(np.diff(d.astype(np.int64)) > 0) and d[0] >= 1 and d[-1] <= n_docs, name
        self.names = {name: t for t, (name, _, _) in enumerate(lists)}
        self.shapes = [t for t, (name, _, _) in enumerate(lists) if not name.endswith("+lead")]
        self.deleted = np.asarray(deleted, np.uint32)
        every = np.concatenate([d for _, d, _ in lists])
        self.U = np.unique(np.concatenate([every, self.deleted])).astype(np.uint32)
        self.docs_with_term = [len(d) for _, d, _ in lists]

    def oracle_segment(self):
        """The segment as the oracle's writer encodes it (the .doc stream staged on the GPU); no norms, so the writer
        needs no per-doc array."""
        o = orc.Segment(self.n_docs, has_wand=self.has_wand)
        for _, d, f in self.lists:
            o.add_term(d, f)
        return o

    # ---- the remap
    def small(self, docs):
        """High doc ids (members of U) -> their ids 1..|U| in the small segment."""
        docs = np.asarray(docs, np.uint32)
        i = np.searchsorted(self.U, docs)
        assert np.all(self.U[np.minimum(i, len(self.U) - 1)] == docs), "doc outside the remap set"
        return (i + 1).astype(np.uint32)

    def big(self, small_docs):
        return self.U[np.asarray(small_docs, np.int64) - 1]

    def _n_short(self):
        return int(np.searchsorted(self.U, SHORT_ROWS, side="right")) if self.base == 0 else 0

    def small_segment(self, with_mask=False):
        """The remapped segment in the oracle: same lists and freqs, the norms and column values of the mapped docs."""
        o = orc.Segment(len(self.U), has_wand=True)
        if self.norm is not None:
            o.set_norms(self.norm(self.U))
        for _, d, f in self.lists:
            o.add_term(self.small(d), f)
        o.add_column(FULL_FIELD, self.small_columns(FULL_FIELD)[0])
        if self._n_short():                               # mapped docs that have a short-column row
            o.add_column(SHORT_FIELD, self.small_columns(SHORT_FIELD)[0])
        if with_mask:
            o.set_docs_mask(self.small(self.deleted))
        return o

    def small_columns(self, field):
        """(values per small row, None) of a column in the remapped segment, for the NumPy references."""
        if field == FULL_FIELD:
            return full_values(np.uint64(self.base) + self.U.astype(np.uint64)), None
        return short_column()[self.U[:self._n_short()].astype(np.int64) - 1], None

    def values(self, docs):
        """The full-length column at the given docs of this segment."""
        return full_values(np.uint64(self.base) + np.asarray(docs, np.uint64))


def with_companions(terms, rng, n):
    """Each list but the long `spread` ones followed by its AND companion (shape_corpora.companion)."""
    out = []
    for name, d, f in terms:
        out.append((name, d, f))
        if not name.startswith("spread"):
            cd, cf = companion(d, rng, n)
            out.append((name + "+lead", cd, cf))
    return out


def deleted_docs(lists, landmarks, n, rng):
    """Every landmark, the docs on both sides of it, and a tenth of the list docs."""
    every = np.unique(np.concatenate([d for _, d, _ in lists]))
    near = np.concatenate([[x - 1, x, x + 1] for x in landmarks]).astype(np.int64)
    near = near[(near >= 1) & (near <= n)]
    return np.unique(np.concatenate([near, every[rng.random(len(every)) < 0.1]])).astype(np.uint32)


class TopCorpus(SegCorpus):
    """The `top` segment: exactly 2^32 - 2 docs, every encoding at the landmarks."""

    def __init__(self, seed=31):
        rng = np.random.default_rng(seed)
        lists = with_companions(shape_terms(rng), rng, TOP)
        super().__init__(TOP, lists, deleted_docs(lists, LANDMARKS, TOP, rng))


# ---------------------------------------------------------------- split: two segments of 2^32 - 2 docs in all
SPLIT_A = 2 ** 31 + 2 ** 20          # with a 1-byte norm column: norm rows past 2^31
SPLIT_B = TOP - SPLIT_A              # its ordinals are SPLIT_A + 1 .. 2^32 - 2
_NORM_PERIOD = 251


def split_norm(docs):
    """Norm of a doc of segment A: 1 .. 251, periodic in the doc id so that the 2 GB column is a tiled pattern."""
    return (1 + (np.asarray(docs, np.uint64) - np.uint64(1)) * np.uint64(37) % np.uint64(_NORM_PERIOD)).astype(np.uint32)


def split_norm_bytes():
    """Segment A's 1-byte norm column (row = doc - 1), SPLIT_A bytes."""
    pattern = split_norm(np.arange(1, _NORM_PERIOD + 1)).astype(np.uint8)
    return np.tile(pattern, SPLIT_A // _NORM_PERIOD + 1)[:SPLIT_A]


def split_norm_sum():
    pattern = split_norm(np.arange(1, _NORM_PERIOD + 1)).astype(np.int64)
    q, r = divmod(SPLIT_A, _NORM_PERIOD)
    return int(q * pattern.sum() + pattern[:r].sum())


def split_terms(n, landmarks, rng):
    """The same term names in each split segment: landmark docs, long lists, a single doc at n, a dense bitset block
    ending at n and a tail near n."""
    lm = np.asarray(sorted(landmarks), np.uint32)
    dense = np.arange(n - 299, n + 1, dtype=np.uint32)
    dense = np.concatenate([np.sort(rng.choice(dense[:-1], 255, replace=False)), [n]]).astype(np.uint32)
    out = [("landmarks", lm, _f(rng, len(lm), 6)),
           ("single_top", np.array([n], np.uint32), np.array([2], np.uint32)),
           ("dense_top", dense, _f(rng, len(dense))),
           ("tail_top", np.array([n - 2 ** 20, n - 70000, n - 5, n], np.uint32), _f(rng, 4))]
    for name, m in (("spread_a", 5000), ("spread_b", 2500)):
        parts = [rng.integers(1, n + 1, m), rng.integers(n - 3 * WINDOW, n + 1, m // 2), rng.integers(1, 200000, m // 6), lm]
        d = np.unique(np.concatenate(parts)).astype(np.uint32)
        out.append((name, d, _f(rng, len(d), 8)))
    return out


def split_landmarks():
    a = {1, 2, 2 ** 31 - 1, 2 ** 31, 2 ** 31 + 1, SPLIT_A - WINDOW, SPLIT_A - WINDOW + 1, SPLIT_A - 1, SPLIT_A}
    b = {1, 2, SPLIT_B // 2, SPLIT_B - WINDOW, SPLIT_B - WINDOW + 1, SPLIT_B - 2048, SPLIT_B - 1, SPLIT_B}
    return sorted(a), sorted(b)


class SplitCorpus:
    """Two segments whose doc counts sum to exactly 2^32 - 2: A (2^31 + 2^20 docs, 1-byte norms, written without
    block-max data so that the writer needs no norms) and B, whose keys carry ordinal_base = SPLIT_A, up to 2^32 - 2."""

    def __init__(self, seed=41):
        rng = np.random.default_rng(seed)
        la, lb = split_landmarks()
        segs = []
        for n, lm, base, norm, wand in ((SPLIT_A, la, 0, split_norm, False), (SPLIT_B, lb, SPLIT_A, None, True)):
            lists = with_companions(split_terms(n, lm, rng), rng, n)
            segs.append(SegCorpus(n, lists, deleted_docs(lists, lm, n, rng), base=base, norm=norm, has_wand=wand))
        self.segs = segs
        self.names = segs[0].names
        assert segs[1].names == self.names
        self.shapes = segs[0].shapes
        self.docs_with_term = [a + b for a, b in zip(segs[0].docs_with_term, segs[1].docs_with_term)]
        self.total_term_freq = split_norm_sum() + SPLIT_B


def map_hits(corpora, hits):
    """Oracle hits on the small segments -> the same hits at the high doc ids (corpora: SegCorpus per segment, or one)."""
    corpora = corpora if isinstance(corpora, (list, tuple)) else [corpora]
    out = hits.copy()
    for si, c in enumerate(corpora):
        m = out["seg"] == si
        if m.any():
            out["doc"][m] = c.big(out["doc"][m])
    return out


def encodings(stage, t):
    """Doc encodings (posting_format.hpp kDe*) of term t's blocks in a staged block table (engine.stage_parse_host)."""
    b0, b1 = int(stage["term_blk_begin"][t]), int(stage["term_blk_begin"][t + 1])
    return [int(p) & 63 for p in stage["packed"][b0:b1]], stage["last_doc"][b0:b1]
