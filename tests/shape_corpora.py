"""Corpora for the pruning and posting-shape tests, built from explicit Python lists so that every doc id, freq and
field length is known without decoding. Shared by the GPU tests and by the CPU guards that check the corpora still
reach the encodings and block-max situations they are meant to reach."""
import numpy as np

import orc

K1, B = 1.2, 0.75


# ---------------------------------------------------------------- BM25 restated
def bm25_f32(freq, norm, c0, nc, nl):
    """bm25() of bm25_kernels.cuh in NumPy float32, same operation order: c1 = nc + nl*norm; c0 - c0*c1/(c1 + freq)."""
    f32 = np.float32
    freq, norm = np.asarray(freq).astype(f32), np.asarray(norm).astype(f32)
    c1 = f32(nc) + f32(nl) * norm
    return (f32(c0) - (f32(c0) * c1) / (c1 + freq)).astype(f32)


def stored_pair(freqs, norms, avg_dl, b=B):
    """The block-max pair PostingWriter::feed keeps for one block: the first (freq, norm) with the largest
    freq / ((1-b)*avg_dl + b*norm), compared by cross-multiplication in float32 like the writer."""
    f32 = np.float32
    x = (f32(1) - f32(b)) * f32(avg_dl)
    best = (1, 0xFFFFFFFF)
    for f, n in zip(freqs, norms):
        mine = f32(f) * (x + f32(b) * f32(best[1]))
        theirs = f32(best[0]) * (x + f32(b) * f32(n))
        if mine > theirs:
            best = (int(f), int(n))
    return best


def bound_consts(nc, nl, k1, b, seg_avg_dl):
    """The bound-only constants of fill_qterm (sdbg_abi.cu): nl_b = min(nl, nl_s), nc_b = nc * min(1, nl / nl_s)."""
    f32 = np.float32
    if not seg_avg_dl > 0:
        return f32(nc), f32(nl)
    nl_s = (f32(k1) * f32(b)) / f32(seg_avg_dl)
    if f32(nl) < nl_s:
        return f32(nc) * (f32(nl) / nl_s), f32(nl)
    return f32(nc), nl_s


def writer_avg_dl(norms):
    """NormReader::GetAvg as the writer computes it: float(sum / non-zero count)."""
    norms = np.asarray(norms, np.uint64)
    nz = int(np.count_nonzero(norms))
    return np.float32(float(norms.sum()) / nz) if nz else np.float32(0)


def bm25_f64(tf, dl, docs_with_field, total_term_freq, docs_with_term, k1=K1, b=B):
    """BM25 from first principles in float64: idf of BM25::collect (bm25.cpp:279-310), then the textbook form."""
    idf = np.log1p((docs_with_field - docs_with_term + 0.5) / (docs_with_term + 0.5))
    avg = total_term_freq / docs_with_field
    tf = np.asarray(tf, np.float64)
    return idf * (k1 + 1) * tf / (tf + k1 * (1 - b + b * np.asarray(dl, np.float64) / avg))


class Corpus:
    """Segments given as (norms, [(docs, freqs), ...]) with the same term ids in every segment."""

    def __init__(self, segs):
        self.norms = [n for n, _ in segs]
        self.lists = [l for _, l in segs]
        self.n_terms = len(self.lists[0])
        self.osegs = []
        for norms, lists in segs:
            o = orc.Segment(len(norms), has_wand=True)
            o.set_norms(norms)
            for d, f in lists:
                o.add_term(np.asarray(d, np.uint32), np.asarray(f, np.uint32))
            self.osegs.append(o)
        self.docs_with_field = sum(len(n) for n in self.norms)
        self.total_term_freq = sum(int(np.asarray(n, np.uint64).sum()) for n in self.norms)
        self.docs_with_term = [sum(len(l[t][0]) for l in self.lists) for t in range(self.n_terms)]


# ---------------------------------------------------------------- A: segments whose average lengths differ
def adversarial_segments():
    """Segment A holds short docs (avgdl ~2) and segment B long ones (dl 100..300), so the corpus-wide avgdl is ~185.
    Term 0 covers all of A: 7 blocks of (tf 2, dl 2) and then, closing every 1024-doc stretch, one block of fillers
    (tf 1, dl 2) with a (tf 1, dl 1) and a (tf 10, dl 20). Under A's own average the writer keeps (1, 1) for that block;
    at the corpus average (10, 20) scores higher, so a bound taken from the stored pair with the query's constants would
    skip the block. Terms 1..5 are in ~97% of all docs (tiny idf: they add little to a score).
    Returns (norms_A, lists_A, norms_B, lists_B, positions of the (1, 1) and (10, 20) docs in A)."""
    rng = np.random.default_rng(2024)
    nA, nB = 8192, 100_000
    dlA = np.full(nA, 2, np.uint32)
    f0 = np.full(nA, 2, np.uint32)
    pair_docs, best_docs = [], []
    for w in range(8):
        b0 = w * 1024 + 7 * 128                     # docs b0+1 .. b0+128: the 8th block of the stretch
        f0[b0:b0 + 128] = 1
        dlA[b0 + 5], f0[b0 + 5] = 1, 1
        dlA[b0 + 90], f0[b0 + 90] = 20, 10
        pair_docs.append(b0 + 6)
        best_docs.append(b0 + 91)
    dlA[np.arange(nA) % 1024 == 3] = 3               # a few length-3 docs, tf 2 <= dl still holds
    dlB = rng.integers(100, 301, size=nB).astype(np.uint32)
    listsA = [(np.arange(1, nA + 1, dtype=np.uint32), f0)]
    listsB = [(np.sort(rng.choice(np.arange(1, nB + 1), size=100, replace=False)).astype(np.uint32), np.ones(100, np.uint32))]
    for _ in range(5):
        for n, lists in ((nA, listsA), (nB, listsB)):
            d = np.flatnonzero(rng.random(n) < 0.97).astype(np.uint32) + 1
            lists.append((d, np.ones(len(d), np.uint32)))
    return dlA, listsA, dlB, listsB, pair_docs, best_docs


def natural_segments(seed=11):
    """Three segments with their own length distributions (short 1..12, long 300..3000 with 2-byte norms, medium ~20..90)
    and 10 terms whose freqs grow with the doc length (tf = 1 + Binomial(dl - 1, q)), as in real text."""
    rng = np.random.default_rng(seed)
    p = [0.4, 0.2, 0.1, 0.05, 0.02, 0.01, 0.005, 0.3, 0.15, 0.003]
    q = [0.002, 0.01, 0.02, 0.005, 0.03, 0.01, 0.05, 0.004, 0.015, 0.02]
    segs = []
    for n, dl in ((50_000, lambda n: np.minimum(1 + rng.geometric(0.35, n), 12)),
                  (30_000, lambda n: rng.integers(300, 3001, n)),
                  (60_000, lambda n: 20 + rng.poisson(40, n))):
        norms = dl(n).astype(np.uint32)
        lists = []
        for t in range(len(p)):
            d = np.flatnonzero(rng.random(n) < p[t]).astype(np.uint32) + 1
            f = (1 + rng.binomial(norms[d - 1] - 1, q[t])).astype(np.uint32)
            lists.append((d, f))
        segs.append((norms, lists))
    return segs


def uniform_segments(n=120_000, parts=3, seed=5):
    """One corpus (shared length distribution) both whole and cut by doc range into `parts` segments."""
    rng = np.random.default_rng(seed)
    norms = (8 + rng.poisson(60, n)).astype(np.uint32)
    p = [0.3, 0.1, 0.03, 0.01, 0.2, 0.005]
    lists = []
    for t in range(len(p)):
        d = np.flatnonzero(rng.random(n) < p[t]).astype(np.uint32) + 1
        lists.append((d, (1 + rng.binomial(norms[d - 1] - 1, 0.01)).astype(np.uint32)))
    cuts = [i * n // parts for i in range(parts + 1)]
    segs = []
    for a, b in zip(cuts[:-1], cuts[1:]):
        sub = []
        for d, f in lists:
            m = (d > a) & (d <= b)
            sub.append(((d[m] - a).astype(np.uint32), f[m]))
        segs.append((norms[a:b].copy(), sub))
    return (norms, lists), segs, cuts


# ---------------------------------------------------------------- C: posting shapes
def _from_gaps(gaps, start=0):
    return (start + np.cumsum(np.asarray(gaps, np.uint64))).astype(np.uint32)


def shape_terms(span, rng):
    """Posting lists that reach every block encoding of the format within doc ids 1..span. Returns [(name, docs, freqs)]."""
    out = []
    small_f = lambda n: rng.integers(1, 4, n).astype(np.uint32)
    # doc bit-packing, widths 2..: two full blocks (the first one at the target width) and a 37-doc tail
    for w in range(2, 32):
        # up to 12 bits every gap is that wide (narrow gaps would make a bitset smaller); beyond, one gap per list is
        gaps = rng.integers(2 ** (w - 1), 2 ** w, 293) if w <= 12 else rng.integers(1, 8, 293)
        if w > 12:
            gaps[rng.integers(1, 128)] = 2 ** (w - 1) + rng.integers(0, 64)
        if int(gaps.sum()) >= span:
            break
        d = _from_gaps(gaps)
        out.append((f"doc_bits{w}", d, small_f(len(d))))
    # bitsets: dense full blocks (2..17 words) and tails down to one word
    for dens in (0.95, 0.6, 0.35, 0.2, 0.12):
        m = int(384 / dens)
        d = np.sort(rng.choice(np.arange(1, m + 1), 384, replace=False)).astype(np.uint32)
        out.append((f"bitset_{dens}", d, small_f(len(d))))
    d = np.concatenate([np.arange(1, 129), 128 + np.sort(rng.choice(np.arange(1, 64), 40, replace=False))]).astype(np.uint32)
    out.append(("bitset_tail1", d, small_f(len(d))))
    # the widest full-block bitset: one 11-bit gap makes bit-packing cost 176 bytes, a 20-word bitset 161. (A bitset is
    # only chosen while it is smaller than the bit-packed block, so full blocks never get near the 64-word limit.)
    d = np.concatenate([np.arange(1, 128), [1270], 1270 + np.arange(1, 30)]).astype(np.uint32)
    out.append(("bitset_wide", d, small_f(len(d))))
    # all-same gaps: 8 / 16 / 32 bit, full blocks and tails
    out.append(("same8", np.arange(3, 3 + 3 * 300, 3, dtype=np.uint32), small_f(300)))
    out.append(("same16", np.arange(300, 300 * 301, 300, dtype=np.uint32), small_f(300)))
    n32 = min(200, (span - 1) // 70000)
    out.append(("same32", np.arange(70000, 70000 * (n32 + 1), 70000, dtype=np.uint32), small_f(n32)))
    # StreamVByte tails: absolute values of 1, 2 and 3 bytes (gaps as wide, so delta coding is no smaller)
    out.append(("svb1", np.sort(rng.choice(np.arange(1, 256), 10, replace=False)).astype(np.uint32), small_f(10)))
    out.append(("svb2", _from_gaps(rng.integers(300, 5000, 10)), small_f(10)))
    out.append(("svb3", _from_gaps(rng.integers(70000, 1_000_000, 10)), small_f(10)))
    # delta StreamVByte tail after a full block: gaps of 1, 2, 3 (and 4 where the span allows) bytes
    tail_gaps = [3, 300, 70000, 5, 200, 90000, 1, 40000]
    if span > 2 ** 26:
        tail_gaps += [2 ** 24 + 5, 7]
    d = _from_gaps(np.concatenate([rng.integers(1, 8, 128), tail_gaps]), start=1000)
    out.append(("dsvb_mixed", d, small_f(len(d))))
    # freq bit-packing, widths 2..31 (width 1 would need a zero freq), all-same freqs, raw and StreamVByte freq tails
    for w in range(2, 32):
        f = rng.integers(1, 2 ** (w - 1) + 1, 293).astype(np.uint32)
        f[rng.integers(0, 128)] = 2 ** (w - 1) + rng.integers(0, 2 ** (w - 1))
        out.append((f"freq_bits{w}", _from_gaps(rng.integers(1, 30, 293)), f))
    for name, v in (("freq_same8", 5), ("freq_same16", 300), ("freq_same32", 70000)):
        out.append((name, _from_gaps(rng.integers(1, 30, 256)), np.full(256, v, np.uint32)))
    f = np.concatenate([small_f(128), rng.integers(2 ** 24, 2 ** 25, 10)]).astype(np.uint32)
    out.append(("freq_raw_tail", _from_gaps(rng.integers(1, 30, 138)), f))
    f = np.concatenate([small_f(128), [1, 300, 70000, 2 ** 24 + 3, 2, 5, 1000]]).astype(np.uint32)
    out.append(("freq_svb_tail", _from_gaps(rng.integers(1, 30, 135)), f))
    # blocks whose doc + freq payload exceeds the 512-byte prefetch slot (doc width 20, freq width 16 and wider)
    for dw, fw in ((20, 16), (23, 31)):
        if 3 * 2 ** (dw - 1) + 3000 < span:
            gaps = rng.integers(1, 8, 3 * 128 + 9)
            for blk in range(3):
                gaps[blk * 128 + 17] = 2 ** (dw - 1) + blk
            f = rng.integers(1, 50, len(gaps)).astype(np.uint32)
            for blk in range(3):
                f[blk * 128 + 40] = 2 ** (fw - 1) + blk
            out.append((f"wide_d{dw}_f{fw}", _from_gaps(gaps), f))
    # single-doc terms (inline in the term meta)
    for name, doc in (("single_first", 1), ("single_mid", span // 2), ("single_last", span)):
        out.append((name, np.array([doc], np.uint32), np.array([2], np.uint32)))
    return out


def raw_tail_terms(rng):
    """Doc tails that StreamVByte cannot shrink (ids and gaps >= 2^24): stored as raw values. Needs a ~2^26-doc span."""
    big = [2 ** 24 + 7, 2 ** 25 + 100, 2 ** 25 + 2 ** 24 + 5000, 2 ** 26 + 3]
    head = np.arange(1, 129, dtype=np.uint32)
    return [("doc_raw_tail", np.array(big, np.uint32), rng.integers(1, 4, 4).astype(np.uint32)),
            ("block_then_raw_tail", np.concatenate([head, np.array(big, np.uint32)]), rng.integers(1, 4, 132).astype(np.uint32))]


def companion(docs, rng, span):
    """A list about a fifth as long that shares some of `docs` and adds a few misses: the lead of an AND (or of a lead-mode
    disjunction) that probes `docs`."""
    take = docs[rng.random(len(docs)) < 0.15]
    miss = rng.integers(1, span + 1, max(1, len(docs) // 16)).astype(np.uint32)
    d = np.unique(np.concatenate([take, miss, docs[:1]])).astype(np.uint32)
    return d, np.ones(len(d), np.uint32)


# Norm columns of the shape segments: width 1 / 2 / 4 bytes (None: no norm column, every doc scores with norm 1).
NORM_WIDTHS = (None, 1, 2, 4)
SHAPE_SPAN = {None: 2 ** 30 + 2 ** 16, 1: 2 ** 24, 2: 2 ** 24, 4: 2 ** 24}


def shape_norms(width, n, rng):
    if width is None:
        return None
    hi = {1: 256, 2: 65536, 4: 400_000}[width]
    v = rng.integers(1, hi, n, dtype=np.uint32)
    v[0] = hi - 1                                   # the widest value fixes the column's width
    return v


def shape_segment(width, seed=0):
    """(orc.Segment, norms or None, [(name, docs, freqs)]) for one norm width; each shape term is followed by its
    AND companion. The segment without norms spans 2^30 docs and holds only the shapes that need doc ids past 2^24
    (the widest bit-packings, raw and 4-byte tails); the others hold every shape that fits 2^24 docs."""
    rng = np.random.default_rng(100 + (width or 0) + seed)
    span = SHAPE_SPAN[width]
    terms = shape_terms(span, rng)
    if width is None:
        terms = [t for t in terms if t[1][-1] > SHAPE_SPAN[1]] + raw_tail_terms(rng)
    norms = shape_norms(width, span, rng)
    oseg = orc.Segment(span, has_wand=True)
    if norms is not None:
        oseg.set_norms(norms)
    lists = []
    for name, d, f in terms:
        assert d[-1] <= span and np.all(np.diff(d.astype(np.int64)) > 0), name
        lists.append((name, d, f))
        cd, cf = companion(d, rng, span)
        lists.append((name + "+lead", cd, cf))
    for _, d, f in lists:
        oseg.add_term(d, f)
    return oseg, norms, lists
