"""Host-side mirror of the reference's interfaces for the hot path, over the C ABI (include/sdbg.h).

Names follow the reference: `BM25` (irs/search/bm25.hpp:58), `ExecuteTopK`
(irs/search/doc_collector.hpp:88-136), `ScoreDoc` hits (irs/index/iterators.hpp:93-101), the
`iresearch_scan` column scan with pushed `TableFilterSet` predicates
(server/connector/duckdb_table_function.cpp:1178-1219). Everything that touches postings or rows runs
in libsdbg.so on the GPU; this module only marshals arguments.
"""
import ctypes as C
import operator

import numpy as np

from . import _native as N

FLT_MIN = float(np.finfo(np.float32).tiny)  # doc_collector.hpp:102 initial score_threshold
HIT_DTYPE = np.dtype([("score", "<f4"), ("doc", "<u4"), ("seg", "<u4")])
GROUP_DTYPE = np.dtype([("key", "<i8"), ("count", "<u8"), ("sum_lo", "<i8"), ("sum_hi", "<i8"),
                        ("sum_f64", "<f8"), ("cnt_f64", "<u8")])
TERM_META_DTYPE = np.dtype([("docs_count", "<u4"), ("freq", "<u4"), ("doc_start", "<u8"),
                            ("e_skip_start", "<u8")])
OPS = dict(LT=0, LE=1, GT=2, GE=3, EQ=4, NE=5, BETWEEN=6, IS_NULL=7, IS_NOT_NULL=8)
TYPES = {np.dtype("int64"): 0, np.dtype("float64"): 1, np.dtype("int32"): 2}
OR, AND = 0, 1
NO_FIELD = N.UINT64_MAX


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


_INT64_MIN, _INT64_MAX = -(1 << 63), (1 << 63) - 1
MAX_DOC_ID = (1 << 32) - 2   # doc ids are 1 .. 2^32 - 2; 2^32 - 1 is doc_limits::eof()


def _check_docs_count(n):
    """A segment's doc count as an int in 1 .. MAX_DOC_ID; ctypes would silently truncate a larger one to 32 bits."""
    n = int(n)
    if not 1 <= n <= MAX_DOC_ID:
        raise ValueError(f"a segment holds 1 .. 2^32 - 2 docs, not {n}")
    return n


def _as_double(v):
    """An integer as the nearest double (+-inf beyond the double range)."""
    try:
        return float(v)
    except OverflowError:
        return float("inf") if v > 0 else float("-inf")


def pred(field, op, lo=0, hi=0):
    """One pushed column predicate (duckdb TableFilter), `column op lo` (BETWEEN: lo <= column <= hi), with SQL's meaning
    whatever the constants' types; NULL never passes. A float constant (Python float or any NumPy floating scalar) goes to
    libsdbg as a double, an integer constant (int, NumPy integer) inside int64 as an integer, and the library resolves
    both against the column's type (sdbg.h, sdbg_col_pred_resolve):
    - double column: IEEE comparison with the constant as a double (an integer is rounded to the nearest double). NaN
      compares false, so `<> NaN` holds for every non-NULL row; -0.0 == +0.0.
    - integer column: the exact comparison of the integer with the constant. v < 2.5 is v <= 2, v >= 2.5 is v >= 3;
      v < 1e300 and v > -inf hold for every row; NaN holds for no row, except `<> NaN`, which holds for every non-NULL
      row. `= 2.5` is resolved as no row and `<> 2.5` as every non-NULL row.
    An integer constant outside int64 goes as the nearest double (+-inf beyond the double range): on an integer column
    that keeps the exact answer (every row or none), on a double column it is the rounding above. The exception is an
    integer within 1024 below INT64_MIN, whose nearest double is -2^63 = INT64_MIN itself (ValueError: pass it as a
    float). BETWEEN with one float and one integer bound sends both as doubles, so such an integer bound must be a double
    exactly (ValueError)."""
    p = N.ColPred()
    p.field = int(field)
    p.op = OPS[op] if isinstance(op, str) else int(op)
    bounds = (lo, hi) if p.op == OPS["BETWEEN"] else (lo, 0)
    ints = [None if isinstance(x, (float, np.floating)) else operator.index(x) for x in bounds]
    if all(v is not None and _INT64_MIN <= v <= _INT64_MAX for v in ints):
        p.is_float = 0
        p.lo_i, p.hi_i = ints
        return p
    doubles = []
    for x, v in zip(bounds, ints):
        if v is None:
            doubles.append(float(x))
        elif _INT64_MIN <= v <= _INT64_MAX:
            if int(float(v)) != v:
                raise ValueError("integer bound %d next to a float bound is not a double: pass both bounds as integers or "
                                 "as floats" % v)
            doubles.append(float(v))
        else:
            d = _as_double(v)
            if v < _INT64_MIN and d == float(_INT64_MIN):
                raise ValueError("integer constant %d below INT64_MIN rounds to the double -2^63, which is INT64_MIN: "
                                 "no double stands for it on both column types" % v)
            doubles.append(d)
    p.is_float = 1
    p.lo_f, p.hi_f = doubles
    return p


def resolve_pred(p, dtype):
    """The predicate the kernels evaluate for pred() `p` on a column of `dtype` (int64 / float64 / int32):
    sdbg_col_pred_resolve, a host-only call. On an integer column lo_i / hi_i hold the integer form, on a double column
    lo_f / hi_f the double form."""
    out = N.ColPred()
    N.check(N.lib().sdbg_col_pred_resolve(C.byref(p), TYPES[np.dtype(dtype)], C.byref(out)))
    return out


def _pred_array(preds):
    arr = (N.ColPred * max(len(preds), 1))()
    for i, p in enumerate(preds):
        arr[i] = p
    return arr


class Context:
    """One GPU + one stream (one per worker, like one DocIterator per worker in the reference)."""

    def __init__(self, device=0):
        self._h = C.c_void_p()
        N.check(N.lib().sdbg_init(int(device), C.byref(self._h)))
        self.device = int(device)

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            N.lib().sdbg_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sync(self):
        N.check(N.lib().sdbg_sync(self._h), self._h)

    def timer_start(self):
        N.check(N.lib().sdbg_timer_start(self._h), self._h)

    def timer_stop(self):
        ms = C.c_float()
        N.check(N.lib().sdbg_timer_stop(self._h, C.byref(ms)), self._h)
        return ms.value

    def flush_l2(self):
        N.check(N.lib().sdbg_flush_l2(self._h), self._h)

    def set_wand(self, enabled=True):
        """Block-max pruning on/off (WandContext of irs::ExecuteTopK). Off => exact total_matches."""
        N.check(N.lib().sdbg_set_wand(self._h, int(enabled)), self._h)

    def profile(self, on=True):
        N.check(N.lib().sdbg_profile_enable(self._h, 1 if on else 0), self._h)

    def scan_stats(self):
        """(2048-row blocks judged by the zonemap pass of the last GROUP BY scan, blocks proven dead = never read)."""
        a, b = C.c_uint64(), C.c_uint64()
        N.check(N.lib().sdbg_scan_stats(self._h, C.byref(a), C.byref(b)), self._h)
        return a.value, b.value

    # ---- collectives (NCCL behind the C ABI; the host only has to ship the 128-byte id to every rank) ----
    @staticmethod
    def dist_unique_id():
        buf = (C.c_uint8 * 128)()
        N.check(N.lib().sdbg_dist_unique_id(buf))
        return bytes(buf)

    def dist_init(self, id128, rank, world):
        buf = (C.c_uint8 * 128).from_buffer_copy(bytes(id128))
        N.check(N.lib().sdbg_dist_init(self._h, buf, int(rank), int(world)), self._h)

    def dist_allreduce_i64(self, d_ptr, n):
        N.check(N.lib().sdbg_dist_allreduce_i64(self._h, C.c_void_p(int(d_ptr)), int(n)), self._h)

    def dist_allgather(self, d_send, d_recv, bytes_per_rank):
        N.check(N.lib().sdbg_dist_allgather(self._h, C.c_void_p(int(d_send)), C.c_void_p(int(d_recv)), int(bytes_per_rank)), self._h)

    def dist_groupby_merge(self, d_i64, d_f64, span, abs_bound):
        """Dense GROUP BY partials of all ranks -> global partials on every rank: one ncclAllReduce on this context's stream."""
        N.check(N.lib().sdbg_dist_groupby_merge(self._h, C.c_void_p(int(d_i64)), C.c_void_p(int(d_f64)), int(span), float(abs_bound)), self._h)

    def profile_read(self, kernel):
        """kernel: 'groupby' | 'topk' | 'merge' | 'count_sum' -> (total_ms, launches) since profile(True)."""
        kid = dict(groupby=0, topk=1, merge=2, count_sum=3)[kernel]
        ms, n = C.c_double(), C.c_uint64()
        N.check(N.lib().sdbg_profile_read(self._h, kid, C.byref(ms), C.byref(n)), self._h)
        return ms.value, n.value

    @property
    def launches(self):
        return int(N.lib().sdbg_launch_count(self._h))


class PostingsWriter:
    """Host mirror of irs PostingsWriterImpl (formats/posting/writer.hpp): builds a ".doc" stream."""

    def __init__(self, segment_docs, norms=None, has_wand=True, wand_b=0.75):
        self._h = C.c_void_p()
        _check_docs_count(segment_docs)
        self._norms = None if norms is None else np.ascontiguousarray(norms, dtype=np.uint32)
        N.check(N.lib().sdbg_writer_create(int(segment_docs), 1 if has_wand else 0, float(wand_b),
                                           _ptr(self._norms), C.byref(self._h)))

    def add_term(self, docs, freqs):
        docs = np.ascontiguousarray(docs, dtype=np.uint32)
        freqs = np.ascontiguousarray(freqs, dtype=np.uint32)
        N.check(N.lib().sdbg_writer_add_term(self._h, _ptr(docs), _ptr(freqs), len(docs)))

    def finish(self):
        """-> (doc_bytes uint8[n], term metas structured array)."""
        p, n, t, nt = C.c_void_p(), C.c_size_t(), C.c_void_p(), C.c_size_t()
        N.check(N.lib().sdbg_writer_finish(self._h, C.byref(p), C.byref(n), C.byref(t), C.byref(nt)))
        doc = np.zeros(n.value, np.uint8)
        if n.value:
            C.memmove(doc.ctypes.data, p.value, n.value)
        metas = np.zeros(nt.value, TERM_META_DTYPE)
        if nt.value:
            C.memmove(metas.ctypes.data, t.value, nt.value * TERM_META_DTYPE.itemsize)
        return doc, metas

    def __del__(self):
        if getattr(self, "_h", None) and self._h.value:
            N.lib().sdbg_writer_destroy(self._h)
            self._h = C.c_void_p()


def stage_parse_host(doc_bytes, metas, has_wand=True):
    """Host-only probe of the staging parser: the block table the kernels would read."""
    doc_bytes = np.ascontiguousarray(doc_bytes, dtype=np.uint8)
    metas = np.ascontiguousarray(metas, dtype=TERM_META_DTYPE)
    cap = int(sum((int(m) + 127) // 128 for m in metas["docs_count"])) + 1
    nblk = C.c_uint32()
    tbb = np.zeros(len(metas) + 1, np.uint32)
    last = np.zeros(cap, np.uint32)
    prev = np.zeros(cap, np.uint32)
    packed = np.zeros(cap, np.uint32)
    mf = np.zeros(cap, np.uint32)
    mn = np.zeros(cap, np.uint32)
    arena = C.c_uint64()
    N.check(N.lib().sdbg_debug_stage_host(_ptr(doc_bytes), len(doc_bytes), _ptr(metas), len(metas),
                                          1 if has_wand else 0, cap, C.byref(nblk), _ptr(tbb), _ptr(last),
                                          _ptr(prev), _ptr(packed), _ptr(mf), _ptr(mn), C.byref(arena)))
    n = nblk.value
    return dict(term_blk_begin=tbb, last_doc=last[:n], prev_last=prev[:n], packed=packed[:n],
                max_freq=mf[:n], max_norm=mn[:n], arena_bytes=arena.value)


class Segment:
    """One index segment resident in HBM: postings, norms, table columns."""

    def __init__(self, ctx, n_docs):
        self.ctx = ctx
        self.n_docs = _check_docs_count(n_docs)
        self._h = C.c_void_p()
        N.check(N.lib().sdbg_segment_create(ctx._h, self.n_docs, C.byref(self._h)), ctx._h)
        self.term_docs = None  # docs_count per term (filled by staging)
        self._keep = []        # host buffers that must outlive async copies
        self.col_types = {}    # field -> sdbg_type of the staged column

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            N.lib().sdbg_segment_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- staging ----
    def stage_postings(self, doc_bytes, metas, has_wand=True, wand_b=0.75):
        doc_bytes = np.ascontiguousarray(doc_bytes, dtype=np.uint8)
        metas = np.ascontiguousarray(metas, dtype=TERM_META_DTYPE)
        N.check(N.lib().sdbg_stage_postings(self._h, _ptr(doc_bytes), len(doc_bytes), _ptr(metas), len(metas),
                                            1 if has_wand else 0), self.ctx._h)
        N.check(N.lib().sdbg_segment_set_wand_b(self._h, float(wand_b)), self.ctx._h)   # pruning only for scorers with this b
        self.term_docs = metas["docs_count"].astype(np.uint64)

    def stage_norms(self, norm_bytes, byte_width):
        norm_bytes = np.ascontiguousarray(norm_bytes, dtype=np.uint8)
        rg = N.NormRg(byte_width, self.n_docs, 0)
        N.check(N.lib().sdbg_stage_norms(self._h, _ptr(norm_bytes), len(norm_bytes), C.byref(rg), 1), self.ctx._h)

    def set_wand_avg_dl(self, avg_dl):
        """Average field length the block-max pairs were chosen with, when the writer did not use the staged norms'
        own average (stage_norms sets that one). Call after stage_norms."""
        N.check(N.lib().sdbg_segment_set_wand_avg_dl(self._h, float(avg_dl)), self.ctx._h)

    def stage_column(self, field, values, validity=None):
        """values: numpy array (int64/float64/int32) or a (host_ptr, dtype, rows) triple of pinned memory."""
        if isinstance(values, tuple):
            ptr, dtype, rows = values
            t = TYPES[np.dtype(dtype)]
            vp = C.c_void_p(int(ptr))
        else:
            values = np.ascontiguousarray(values)
            t, rows, vp = TYPES[values.dtype], len(values), _ptr(values)
            self._keep.append(values)
        vv = None
        if validity is not None:
            validity = np.ascontiguousarray(validity, dtype=np.uint64)
            self._keep.append(validity)
            vv = _ptr(validity)
        N.check(N.lib().sdbg_stage_column(self._h, int(field), t, vp, vv, int(rows)), self.ctx._h)
        self.col_types[int(field)] = t

    def stage_column_for(self, field, packed):
        """Stage an int64 column from its frame-of-reference bit-packed form (pack_for): only the packed bytes cross PCIe,
        the values are unpacked on the GPU."""
        headers, words, rows = packed
        self._keep.append(packed)
        N.check(N.lib().sdbg_stage_column_for(self._h, int(field), _ptr(headers), _ptr(words), len(words), int(rows)), self.ctx._h)
        self.col_types[int(field)] = 0

    def stage_docs_mask(self, deleted_docs):
        """DocumentMask of the segment: doc ids that queries must neither score nor count (None / empty clears)."""
        d = np.ascontiguousarray(deleted_docs if deleted_docs is not None else [], dtype=np.uint32)
        N.check(N.lib().sdbg_stage_docs_mask(self._h, _ptr(d) if len(d) else None, len(d)), self.ctx._h)

    def stage_column_device(self, field, device_ptr, dtype, rows):
        N.check(N.lib().sdbg_stage_column_device(self._h, int(field), TYPES[np.dtype(dtype)],
                                                 C.c_void_p(int(device_ptr)), int(rows)), self.ctx._h)
        self.col_types[int(field)] = TYPES[np.dtype(dtype)]

    def column_device_ptr(self, field):
        p, r = C.c_void_p(), C.c_uint64()
        N.check(N.lib().sdbg_column_device_ptr(self._h, int(field), C.byref(p), C.byref(r)), self.ctx._h)
        return p.value, r.value

    def gather(self, field, docs, dtype):
        """Column values of the given hit docs (late materialisation, HitBatcher::MaterializeColumn): (values, valid)."""
        docs = np.ascontiguousarray(docs, dtype=np.uint32)
        out = np.zeros(len(docs), dtype)
        valid = np.zeros(len(docs), np.uint8)
        N.check(N.lib().sdbg_gather_column(self._h, int(field), _ptr(docs) if len(docs) else None, len(docs),
                                           _ptr(out) if len(docs) else None, _ptr(valid) if len(docs) else None), self.ctx._h)
        return out, valid.astype(bool)

    def column_to_host(self, field, host_ptr, rows):
        N.check(N.lib().sdbg_column_to_host(self._h, int(field), C.c_void_p(int(host_ptr)), int(rows)), self.ctx._h)

    def column_packed(self, field, rows):
        """The staged column's bit-packed storage as (headers, words) in pack_for's format, or None when it is held raw."""
        n = C.c_uint64(0)
        rc = N.lib().sdbg_column_for_to_host(self._h, int(field), None, None, 0, C.byref(n))
        if rc != -6 and rc != 0:   # -6: SDBG_ECAPACITY, *n = the words needed
            N.check(rc, self.ctx._h)
        if n.value == 0:
            return None
        headers = np.zeros((int(rows) + 2047) // 2048, FOR_BLOCK_DTYPE)
        words = np.zeros(n.value, np.uint64)
        N.check(N.lib().sdbg_column_for_to_host(self._h, int(field), _ptr(headers), _ptr(words), n.value, C.byref(n)), self.ctx._h)
        return headers, words

    def synth_corpus(self, doc0, t0, nt, threads=8, p_floor=0.0):
        """SURVEY §8d corpus shard: returns (docs_count per term, sum of doc lengths). p_floor > 0 gives every term at
        least that inclusion probability (a flat tail: an index far larger than L2)."""
        dc = np.zeros(nt, np.uint32)
        sdl = C.c_uint64()
        N.check(N.lib().sdbg_synth_corpus_ex(self._h, int(doc0), self.n_docs, int(t0), int(nt), int(threads), float(p_floor),
                                             _ptr(dc), C.byref(sdl)), self.ctx._h)
        self.term_docs = dc.astype(np.uint64)
        return dc, sdl.value

    def synth_column(self, field, stream, kind, row0, rows):
        N.check(N.lib().sdbg_synth_column(self._h, int(field), int(stream), int(kind), int(row0), int(rows)),
                self.ctx._h)
        self.col_types[int(field)] = 1 if kind in (2, 4) else 2 if kind == 6 else 0

    def posting_stats(self):
        a, b, c, d = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_uint64()
        N.check(N.lib().sdbg_segment_posting_stats(self._h, C.byref(a), C.byref(b), C.byref(c), C.byref(d)))
        return dict(payload_bytes=a.value, table_bytes=b.value, n_blocks=c.value, n_postings=d.value)

    def term_bytes(self, n_terms):
        out = np.zeros(int(n_terms), np.uint64)
        N.check(N.lib().sdbg_segment_term_bytes(self._h, _ptr(out), int(n_terms)), self.ctx._h)
        return out

    def column_minmax(self, field):
        mn, mx = C.c_int64(), C.c_int64()
        N.check(N.lib().sdbg_column_minmax_i64(self._h, int(field), C.byref(mn), C.byref(mx)), self.ctx._h)
        return mn.value, mx.value

    # ---- probes ----
    def decode_score_term(self, term, c0, norm_const, norm_length):
        n = int(self.term_docs[term])
        docs = np.zeros(max(n, 1), np.uint32)
        freqs = np.zeros(max(n, 1), np.uint32)
        scores = np.zeros(max(n, 1), np.float32)
        N.check(N.lib().sdbg_decode_score_term(self._h, int(term), float(c0), float(norm_const), float(norm_length),
                                               _ptr(docs), _ptr(freqs), _ptr(scores)), self.ctx._h)
        return docs[:n], freqs[:n], scores[:n]

    def filter_bitmap(self, preds, rows=None):
        rows = self.n_docs if rows is None else rows
        mask = np.zeros((rows + 63) // 64, np.uint64)
        N.check(N.lib().sdbg_filter_bitmap(self._h, _pred_array(preds), len(preds), _ptr(mask)), self.ctx._h)
        return mask


def _seg_array(segs):
    arr = (C.c_void_p * len(segs))()
    for i, s in enumerate(segs):
        arr[i] = s._h
    return arr


class BM25:
    """irs::BM25 (search/bm25.hpp:58): k, b and the statistics -> BM25Stats step (bm25.cpp:279-310)."""

    def __init__(self, k=1.2, b=0.75):
        self.k, self.b = float(k), float(b)

    def collect(self, docs_with_field, total_term_freq, docs_with_term, term=0, boost=1.0):
        t = N.BM25Term()
        N.check(N.lib().sdbg_bm25_collect(int(docs_with_field), int(total_term_freq), int(docs_with_term),
                                          self.k, self.b, C.byref(t)))
        t.term = int(term)
        t.boost = float(boost)
        return t

    def num(self, term):
        """c0 = boost*(k+1)*idf in fp32 (bm25.cpp:224)."""
        return np.float32(np.float32(np.float32(term.boost) * np.float32(self.k + np.float32(1))) * np.float32(term.idf))


class TFIDF:
    """irs::TFIDF (search/tfidf.cpp): sqrt(freq) * boost * idf, divided by sqrt(doc length) when `normalize`; idf from
    TFIDF::collect (:149-150). Runs through the same scan entry points: k = -1 is the ABI's reserved selector for it
    (sdbg_tfidf_topk_batch forwards exactly that), b != 0 means normalised. Always exhaustive."""

    def __init__(self, normalize=False):
        self.normalize = bool(normalize)
        self.k, self.b = -1.0, (1.0 if normalize else 0.0)

    def collect(self, docs_with_field, total_term_freq, docs_with_term, term=0, boost=1.0):
        t = N.BM25Term()
        N.check(N.lib().sdbg_tfidf_collect(int(docs_with_field), int(docs_with_term), C.byref(t)))
        t.term = int(term)
        t.boost = float(boost)
        return t

    def num(self, term):
        return np.float32(np.float32(term.boost) * np.float32(term.idf))


class IndexReader:
    """The segments of one snapshot on one GPU plus corpus-wide field statistics
    (FieldCollector / TermCollector sums over all segments, search/collectors.cpp:30-52)."""

    def __init__(self, segments, docs_with_field, total_term_freq, docs_with_term):
        self.segments = list(segments)
        self.docs_with_field = int(docs_with_field)
        self.total_term_freq = int(total_term_freq)
        self.docs_with_term = np.asarray(docs_with_term, dtype=np.uint64)  # per term id, global

    def stats(self, scorer, term, boost=1.0):
        return scorer.collect(self.docs_with_field, self.total_term_freq, int(self.docs_with_term[term]), term, boost)


def _exclusions(exclude, nq):
    """Per-query excluded term ids -> (flat ids u32, offsets u32 [nq + 1]), or None when no query excludes anything."""
    if exclude is None:
        return None
    if len(exclude) != nq:
        raise ValueError("exclude needs one list (or None) per query")
    lists = [list(x) if x is not None else [] for x in exclude]
    if not any(lists):
        return None
    off = np.zeros(nq + 1, np.uint32)
    off[1:] = np.cumsum([len(x) for x in lists])
    return np.ascontiguousarray([t for x in lists for t in x], dtype=np.uint32), off


def _query_args(queries, exclude, min_match=None, groups=False, stats=None):
    """The query arguments of a batch entry: (terms, term_off, nq, excl_terms, excl_off) of a flat entry or, with `groups`,
    (terms, group_off, query_group_off, group_min, nq, excl_terms, excl_off) of a group entry. terms: the term ids as u32
    (NULL when there are none), or with `stats` (term id -> sdbg_bm25_term) the scored entries' array. excl_terms and
    excl_off are NULL when no query excludes anything."""
    nq = len(queries)
    if groups:
        ids, group_off, query_group_off = _groups(queries)
        offsets = (_ptr(group_off), _ptr(query_group_off), _ptr(_group_min(min_match, queries)))
    else:
        ids = [t for q in queries for t in q]
        off = np.zeros(nq + 1, np.uint32)
        off[1:] = np.cumsum([len(q) for q in queries])
        offsets = (_ptr(off),)
    if stats is None:
        flat = np.ascontiguousarray(ids, dtype=np.uint32)
        terms = _ptr(flat) if len(flat) else None
    else:
        terms = (N.BM25Term * max(len(ids), 1))(*[stats(t) for t in ids])
    x = _exclusions(exclude, nq) or (None, None)
    return (terms,) + offsets + (nq, _ptr(x[0]), _ptr(x[1]))


def _one(x):
    """A single query's per-query argument (its terms, groups, exclusions or group minimums) as a batch of one."""
    return None if x is None else [list(x)]


def _ref(filt):
    return C.byref(filt) if filt is not None else None


def ExecuteTopKBatch(reader, queries, kind, scorer, k, filt=None, threshold=FLT_MIN, exclude=None):
    """Batch of ExecuteTopK calls (doc_collector.hpp:88-136). queries: list of term-id lists. exclude: None, or one list of
    excluded term ids (or None) per query -- `a & b & !c` (sdbg_bm25_topk_batch_excl).
    Returns (hits [Q, k] structured, n_out [Q], total_matches [Q])."""
    terms, off, nq, excl_terms, excl_off = _query_args(queries, exclude, stats=lambda t: reader.stats(scorer, t))
    hits = np.zeros((nq, k), HIT_DTYPE)
    n_out = np.zeros(nq, np.uint32)
    total = np.zeros(nq, np.uint64)
    head = (_seg_array(reader.segments), len(reader.segments), int(kind), terms, off, nq)
    tail = (scorer.k, scorer.b, _ref(filt), int(k), float(threshold), _ptr(hits), _ptr(n_out), _ptr(total))
    if excl_off is None:
        rc = N.lib().sdbg_bm25_topk_batch(*head, *tail)
    else:
        rc = N.lib().sdbg_bm25_topk_batch_excl(*head, excl_terms, excl_off, *tail)
    N.check(rc, reader.segments[0].ctx._h)
    return hits, n_out, total


def ExecuteCountBatch(reader, queries, kind, filt=None, exclude=None):
    """Count mode of the search scan (`SELECT count(*) ... WHERE body @@ '...'`, sdbg_match_count_batch): per query, the
    number of docs over all segments that match its term ids (OR / AND), are not deleted, pass `filt` and hold none of its
    `exclude` term ids. Nothing is scored, so no statistics are needed; exact at every pruning level. Returns uint64[Q]."""
    counts = np.zeros(len(queries), np.uint64)
    N.check(N.lib().sdbg_match_count_batch(_seg_array(reader.segments), len(reader.segments), int(kind),
                                           *_query_args(queries, exclude), _ref(filt), _ptr(counts)),
            reader.segments[0].ctx._h)
    return counts


def ExecuteCount(reader, query_terms, kind, filt=None, exclude=None):
    """ExecuteCountBatch for one query: its match count as an int."""
    return int(ExecuteCountBatch(reader, _one(query_terms), kind, filt, exclude=_one(exclude))[0])


SORT_HIT_DTYPE = np.dtype([("value", "<i8"), ("doc", "<u4"), ("seg", "<u4"), ("is_null", "u1"), ("pad", "V7")])
_SORT_VALUE_DTYPE = {0: np.int64, 1: np.float64, 2: np.int32}


def ExecuteTopKByColumnBatch(reader, queries, kind, sort_field, k, descending=False, nulls_first=False, filt=None,
                             exclude=None):
    """Sorted scan (`WHERE body @@ '...' ORDER BY col [DESC] [NULLS FIRST] LIMIT k`, sdbg_match_topk_by_column_batch): per
    query, the first k of the docs ExecuteCountBatch counts, ordered by column `sort_field` (int64 / int32 / float64,
    staged in every segment); ties, NULLs included, by (segment, doc). Returns a dict of per-query arrays: docs, segs,
    values (typed by the column; 0 for NULL), nulls (bool) and n_out (uint32[Q])."""
    vt = _sort_value_type(reader, sort_field)
    nq = len(queries)
    hits = np.zeros(max(nq, 1) * max(int(k), 1), SORT_HIT_DTYPE)
    n_out = np.zeros(max(nq, 1), np.uint32)
    N.check(N.lib().sdbg_match_topk_by_column_batch(_seg_array(reader.segments), len(reader.segments), int(kind),
                                                    *_query_args(queries, exclude), _ref(filt), int(sort_field),
                                                    int(bool(descending)), int(bool(nulls_first)), int(k), _ptr(hits),
                                                    _ptr(n_out)), reader.segments[0].ctx._h)
    return _sort_result(hits, n_out, nq, k, vt)


def _sort_value_type(reader, sort_field):
    col_type = reader.segments[0].col_types.get(int(sort_field))
    if col_type is None:   # the values come back as raw bits: their type must be known, not guessed
        raise ValueError("sort column %d was not staged through this Segment" % int(sort_field))
    return _SORT_VALUE_DTYPE[col_type]


def _sort_result(hits, n_out, nq, k, vt):
    """Sorted-scan hits [nq * k] -> the per-query dict the sorted-scan functions return."""
    out = dict(docs=[], segs=[], values=[], nulls=[], n_out=n_out[:nq])
    for q in range(nq):
        h = hits[q * k:q * k + int(n_out[q])]
        raw = h["value"].copy()
        out["values"].append(raw.view(np.float64) if vt is np.float64 else raw.astype(vt))
        out["docs"].append(h["doc"].copy())
        out["segs"].append(h["seg"].copy())
        out["nulls"].append(h["is_null"].astype(bool))
    return out


def _sort_row(r):
    """The first query of a sorted-scan result: dict of docs, segs, values, nulls."""
    return {key: r[key][0] for key in ("docs", "segs", "values", "nulls")}


def ExecuteTopKByColumn(reader, query_terms, kind, sort_field, k, descending=False, nulls_first=False, filt=None,
                        exclude=None):
    """ExecuteTopKByColumnBatch for one query: dict of docs, segs, values, nulls (arrays of n_out entries)."""
    return _sort_row(ExecuteTopKByColumnBatch(reader, _one(query_terms), kind, sort_field, k, descending, nulls_first, filt,
                                              exclude=_one(exclude)))


def ExecuteFacetCountsBatch(reader, queries, kind, key_field, key_min=None, key_span=None, filt=None, exclude=None):
    """Facet counts (`SELECT col, count(*) ... WHERE body @@ '...' GROUP BY col`, sdbg_match_facet_counts_batch): per
    query, how the docs ExecuteCountBatch counts split over the values of column `key_field` (int64 / int32, staged in
    every segment). The key range [key_min, key_min + key_span) defaults to the segments' column_minmax (an all-NULL column
    gives one bin). Returns dict(key_min, counts uint64[Q, key_span], nulls uint64[Q]): counts[q, v - key_min] = matches
    whose key is v, nulls[q] = matches whose key is NULL."""
    key_min, key_span = _facet_key_range(reader, key_field, key_min, key_span)
    nq = len(queries)
    counts = np.zeros((max(nq, 1), max(int(key_span), 1)), np.uint64)
    nulls = np.zeros(max(nq, 1), np.uint64)
    N.check(N.lib().sdbg_match_facet_counts_batch(_seg_array(reader.segments), len(reader.segments), int(kind),
                                                  *_query_args(queries, exclude), _ref(filt), int(key_field), int(key_min),
                                                  int(key_span), _ptr(counts), _ptr(nulls)), reader.segments[0].ctx._h)
    return dict(key_min=int(key_min), counts=counts[:nq], nulls=nulls[:nq])


def _facet_key_range(reader, key_field, key_min, key_span):
    """(key_min, key_span), each defaulting to the segments' column_minmax (an all-NULL column gives one bin)."""
    col_type = reader.segments[0].col_types.get(int(key_field))
    if col_type is None:   # the kernel reads raw values: their type must be known, not guessed
        raise ValueError("key column %d was not staged through this Segment" % int(key_field))
    if col_type not in (0, 2):
        raise ValueError("facet counts need an int64 or int32 key column")
    if key_min is None or key_span is None:
        mm = [s.column_minmax(key_field) for s in reader.segments]
        lo, hi = min(m[0] for m in mm), max(m[1] for m in mm)
        if lo > hi:   # every key NULL
            lo = hi = 0
        key_min = lo if key_min is None else key_min
        key_span = hi - key_min + 1 if key_span is None else key_span
    return key_min, key_span


def _facet_row(r):
    """The first query of a facet-counts result: {key: count} for the keys with matches, plus {None: n} when n > 0 matches
    have a NULL key."""
    row = r["counts"][0]
    out = {r["key_min"] + int(i): int(row[i]) for i in np.nonzero(row)[0]}
    if r["nulls"][0]:
        out[None] = int(r["nulls"][0])
    return out


def ExecuteFacetCounts(reader, query_terms, kind, key_field, key_min=None, key_span=None, filt=None, exclude=None):
    """ExecuteFacetCountsBatch for one query: {key: count} for the keys with matches, plus {None: n} when n > 0 matches
    have a NULL key."""
    return _facet_row(ExecuteFacetCountsBatch(reader, _one(query_terms), kind, key_field, key_min, key_span, filt,
                                              exclude=_one(exclude)))


MATCH_AGG_DTYPE = np.dtype([("count", "<u8"), ("count_value", "<u8"), ("sum_lo", "<i8"), ("sum_hi", "<i8"),
                            ("sum_f64", "<f8"), ("min", "<i8"), ("max", "<i8")])


def _agg_args(reader, value_field, key_field, key_min, key_span):
    """(value type code, key field, key_min, key_span) of an aggregate call; key_field None: one group, (0, 1)."""
    vt = reader.segments[0].col_types.get(int(value_field))
    if vt is None:   # the values come back as raw bits: their type must be known, not guessed
        raise ValueError("value column %d was not staged through this Segment" % int(value_field))
    if key_field is None:
        return vt, N.UINT64_MAX, 0, 1
    key_min, key_span = _facet_key_range(reader, key_field, key_min, key_span)
    return vt, int(key_field), key_min, key_span


def _agg_fields(a, vt):
    """Structured sdbg_match_agg cells -> dict of count, count_value, sum (Python ints in an object array for integer
    columns, float64 for float64 ones), avg (float64, NaN without values), min and max (typed by the column; 0 without
    values)."""
    cv = a["count_value"]
    if vt == 1:
        s = a["sum_f64"].copy()
        mn, mx = a["min"].view(np.float64).copy(), a["max"].view(np.float64).copy()
    else:
        s = np.empty(a.shape, dtype=object)
        for i in np.ndindex(a.shape):
            s[i] = (int(a["sum_hi"][i]) << 64) | (int(a["sum_lo"][i]) & 0xFFFFFFFFFFFFFFFF)
        mn, mx = a["min"].copy(), a["max"].copy()
    avg = np.full(a.shape, np.nan)
    for i in zip(*np.nonzero(cv)):
        avg[i] = s[i] / int(cv[i])
    return dict(count=a["count"].copy(), count_value=cv.copy(), sum=s, avg=avg, min=mn, max=mx)


def _agg_result(out, null_out, nq, key_min, vt):
    """The dict the aggregate functions return: key_min, the per-key fields [Q, key_span] and the NULL key's [Q]."""
    r = _agg_fields(out[:nq], vt)
    r["key_min"] = int(key_min)
    r["null"] = _agg_fields(null_out[:nq], vt)
    return r


def ExecuteMatchAggregatesBatch(reader, queries, kind, value_field, key_field=None, key_min=None, key_span=None, filt=None,
                                exclude=None):
    """Aggregates over a full-text query's matches (`SELECT col, count(*), count(v), sum(v), avg(v), min(v), max(v) ...
    WHERE body @@ '...' GROUP BY col`, sdbg_match_aggregate_batch): per query, over the docs ExecuteCountBatch counts,
    grouped by `key_field` as ExecuteFacetCountsBatch groups them (key range defaults likewise), or ungrouped (key_field
    None: one group, key_span 1). `value_field` is an int64 / int32 / float64 column. Returns dict(key_min, count,
    count_value, sum, avg, min, max, each [Q, key_span], null: the same fields [Q] for the NULL key). sum is exact (Python
    ints) for integer columns; avg is NaN and sum / min / max are 0 where a group has no non-NULL value."""
    vt, kf, key_min, key_span = _agg_args(reader, value_field, key_field, key_min, key_span)
    nq = len(queries)
    out = np.zeros((max(nq, 1), max(int(key_span), 1)), MATCH_AGG_DTYPE)
    null_out = np.zeros(max(nq, 1), MATCH_AGG_DTYPE)
    N.check(N.lib().sdbg_match_aggregate_batch(_seg_array(reader.segments), len(reader.segments), int(kind),
                                               *_query_args(queries, exclude), _ref(filt), kf, int(key_min), int(key_span),
                                               int(value_field), _ptr(out), _ptr(null_out)), reader.segments[0].ctx._h)
    return _agg_result(out, null_out, nq, key_min, vt)


def _agg_row(r, grouped):
    """The first query of an aggregate result: ungrouped its fields as a dict; grouped {key: fields} for the keys with
    matches, plus {None: fields} when matches have a NULL key."""
    names = ("count", "count_value", "sum", "avg", "min", "max")
    if not grouped:
        return {f: r[f][0][0] for f in names}
    out = {r["key_min"] + int(i): {f: r[f][0][i] for f in names} for i in np.nonzero(r["count"][0])[0]}
    if r["null"]["count"][0]:
        out[None] = {f: r["null"][f][0] for f in names}
    return out


def ExecuteMatchAggregates(reader, query_terms, kind, value_field, key_field=None, key_min=None, key_span=None, filt=None,
                           exclude=None):
    """ExecuteMatchAggregatesBatch for one query: ungrouped a dict of count, count_value, sum, avg, min, max; grouped
    {key: that dict} for the keys with matches, plus {None: ...} for the NULL key's matches."""
    return _agg_row(ExecuteMatchAggregatesBatch(reader, _one(query_terms), kind, value_field, key_field, key_min, key_span,
                                                filt, exclude=_one(exclude)), key_field is not None)


def _groups(queries):
    """Queries as lists of OR groups -> (flat term ids, group_off u32, query_group_off u32)."""
    groups = [list(g) for q in queries for g in q]
    query_group_off = np.zeros(len(queries) + 1, np.uint32)
    query_group_off[1:] = np.cumsum([len(q) for q in queries])
    group_off = np.zeros(len(groups) + 1, np.uint32)
    group_off[1:] = np.cumsum([len(g) for g in groups])
    return [t for g in groups for t in g], group_off, query_group_off


def _group_min(min_match, queries):
    """Per query one minimum per group -> group_min u32 indexed like group_off (None: every group needs 1 term)."""
    if min_match is None:
        return None
    if len(min_match) != len(queries) or any(len(m) != len(q) for m, q in zip(min_match, queries)):
        raise ValueError("min_match needs one value per group of each query")
    return np.ascontiguousarray([int(v) for m in min_match for v in m], dtype=np.uint32)


def _one_groups(groups):
    """A single query of OR groups as a batch of one."""
    return [[list(g) for g in groups]]


def ExecuteTopKGroupsBatch(reader, queries, scorer, k, filt=None, threshold=FLT_MIN, exclude=None, min_match=None):
    """Top-k of conjunctions of OR groups (`a & (b | c) & !d`, sdbg_bm25_topk_batch_groups_min). queries: per query a list of
    1..16 groups, each a non-empty list of term ids (1..16 distinct ids per query in all). A hit's score is the score the
    flat OR of the query's terms gives that doc. exclude: as in ExecuteTopKBatch. min_match: per query one minimum per
    group (`2 of (a | b | c)`: a doc needs that many of the group's terms), 1..the group's size; None: 1 everywhere.
    Returns (hits [Q, k], n_out [Q], total_matches [Q])."""
    args = _query_args(queries, exclude, min_match, groups=True, stats=lambda t: reader.stats(scorer, t))
    nq = len(queries)
    hits = np.zeros((nq, k), HIT_DTYPE)
    n_out = np.zeros(nq, np.uint32)
    total = np.zeros(nq, np.uint64)
    N.check(N.lib().sdbg_bm25_topk_batch_groups_min(_seg_array(reader.segments), len(reader.segments), *args, scorer.k,
                                                    scorer.b, _ref(filt), int(k), float(threshold), _ptr(hits), _ptr(n_out),
                                                    _ptr(total)), reader.segments[0].ctx._h)
    return hits, n_out, total


def ExecuteTopKGroups(reader, groups, scorer, k, filt=None, threshold=FLT_MIN, exclude=None, min_match=None):
    """ExecuteTopKGroupsBatch for one query (a list of OR groups; min_match: one minimum per group): (hits, total_matches)."""
    hits, n_out, total = ExecuteTopKGroupsBatch(reader, _one_groups(groups), scorer, k, filt, threshold, exclude=_one(exclude),
                                                min_match=_one(min_match))
    return hits[0, :n_out[0]].copy(), int(total[0])


def ExecuteCountGroupsBatch(reader, queries, filt=None, exclude=None, min_match=None):
    """Count mode for conjunctions of OR groups (sdbg_match_count_batch_groups_min): per query, the number of docs over all
    segments in which every group has a term (min_match: per query one minimum per group, as in ExecuteTopKGroupsBatch),
    that are not deleted, pass `filt` and hold none of its `exclude` term ids. Exact at every pruning level. Returns
    uint64[Q]."""
    counts = np.zeros(len(queries), np.uint64)
    N.check(N.lib().sdbg_match_count_batch_groups_min(_seg_array(reader.segments), len(reader.segments),
                                                      *_query_args(queries, exclude, min_match, groups=True), _ref(filt),
                                                      _ptr(counts)), reader.segments[0].ctx._h)
    return counts


def ExecuteCountGroups(reader, groups, filt=None, exclude=None, min_match=None):
    """ExecuteCountGroupsBatch for one query: its match count as an int."""
    return int(ExecuteCountGroupsBatch(reader, _one_groups(groups), filt, exclude=_one(exclude), min_match=_one(min_match))[0])


def ExecuteTopKByColumnGroupsBatch(reader, queries, sort_field, k, descending=False, nulls_first=False, filt=None,
                                   exclude=None, min_match=None):
    """Sorted scan of conjunctions of OR groups (`WHERE body @@ 'a & (b | c)' ORDER BY col LIMIT k`,
    sdbg_match_topk_by_column_batch_groups_min): per query, the first k of the docs ExecuteCountGroupsBatch counts, in the
    order of ExecuteTopKByColumnBatch. queries / exclude / min_match as in ExecuteCountGroupsBatch. Returns the dict
    ExecuteTopKByColumnBatch returns."""
    vt = _sort_value_type(reader, sort_field)
    nq = len(queries)
    hits = np.zeros(max(nq, 1) * max(int(k), 1), SORT_HIT_DTYPE)
    n_out = np.zeros(max(nq, 1), np.uint32)
    N.check(N.lib().sdbg_match_topk_by_column_batch_groups_min(
        _seg_array(reader.segments), len(reader.segments), *_query_args(queries, exclude, min_match, groups=True),
        _ref(filt), int(sort_field), int(bool(descending)), int(bool(nulls_first)), int(k), _ptr(hits), _ptr(n_out)),
        reader.segments[0].ctx._h)
    return _sort_result(hits, n_out, nq, k, vt)


def ExecuteTopKByColumnGroups(reader, groups, sort_field, k, descending=False, nulls_first=False, filt=None, exclude=None,
                              min_match=None):
    """ExecuteTopKByColumnGroupsBatch for one query (a list of OR groups): dict of docs, segs, values, nulls."""
    return _sort_row(ExecuteTopKByColumnGroupsBatch(reader, _one_groups(groups), sort_field, k, descending, nulls_first, filt,
                                                    exclude=_one(exclude), min_match=_one(min_match)))


def ExecuteFacetCountsGroupsBatch(reader, queries, key_field, key_min=None, key_span=None, filt=None, exclude=None,
                                  min_match=None):
    """Facet counts of conjunctions of OR groups (`WHERE body @@ 'a & (b | c)' GROUP BY col`,
    sdbg_match_facet_counts_batch_groups_min): per query, how the docs ExecuteCountGroupsBatch counts split over the values
    of column `key_field`. queries / exclude / min_match as in ExecuteCountGroupsBatch; the key range as in
    ExecuteFacetCountsBatch. Returns the dict ExecuteFacetCountsBatch returns."""
    key_min, key_span = _facet_key_range(reader, key_field, key_min, key_span)
    nq = len(queries)
    counts = np.zeros((max(nq, 1), max(int(key_span), 1)), np.uint64)
    nulls = np.zeros(max(nq, 1), np.uint64)
    N.check(N.lib().sdbg_match_facet_counts_batch_groups_min(
        _seg_array(reader.segments), len(reader.segments), *_query_args(queries, exclude, min_match, groups=True),
        _ref(filt), int(key_field), int(key_min), int(key_span), _ptr(counts), _ptr(nulls)), reader.segments[0].ctx._h)
    return dict(key_min=int(key_min), counts=counts[:nq], nulls=nulls[:nq])


def ExecuteFacetCountsGroups(reader, groups, key_field, key_min=None, key_span=None, filt=None, exclude=None,
                             min_match=None):
    """ExecuteFacetCountsGroupsBatch for one query: {key: count} plus {None: n} for NULL keys, as ExecuteFacetCounts."""
    return _facet_row(ExecuteFacetCountsGroupsBatch(reader, _one_groups(groups), key_field, key_min, key_span, filt,
                                                    exclude=_one(exclude), min_match=_one(min_match)))


def ExecuteMatchAggregatesGroupsBatch(reader, queries, value_field, key_field=None, key_min=None, key_span=None, filt=None,
                                      exclude=None, min_match=None):
    """Aggregates over the matches of conjunctions of OR groups (sdbg_match_aggregate_batch_groups_min): per query, over
    the docs ExecuteCountGroupsBatch counts. queries / exclude / min_match as in ExecuteCountGroupsBatch; the grouping and
    the result as in ExecuteMatchAggregatesBatch."""
    vt, kf, key_min, key_span = _agg_args(reader, value_field, key_field, key_min, key_span)
    nq = len(queries)
    out = np.zeros((max(nq, 1), max(int(key_span), 1)), MATCH_AGG_DTYPE)
    null_out = np.zeros(max(nq, 1), MATCH_AGG_DTYPE)
    N.check(N.lib().sdbg_match_aggregate_batch_groups_min(
        _seg_array(reader.segments), len(reader.segments), *_query_args(queries, exclude, min_match, groups=True),
        _ref(filt), kf, int(key_min), int(key_span), int(value_field), _ptr(out), _ptr(null_out)), reader.segments[0].ctx._h)
    return _agg_result(out, null_out, nq, key_min, vt)


def ExecuteMatchAggregatesGroups(reader, groups, value_field, key_field=None, key_min=None, key_span=None, filt=None,
                                 exclude=None, min_match=None):
    """ExecuteMatchAggregatesGroupsBatch for one query (a list of OR groups), in the form ExecuteMatchAggregates returns."""
    return _agg_row(ExecuteMatchAggregatesGroupsBatch(reader, _one_groups(groups), value_field, key_field, key_min, key_span,
                                                      filt, exclude=_one(exclude), min_match=_one(min_match)),
                    key_field is not None)


def ExecuteDistCountGroupsBatch(reader, queries, filt=None, exclude=None, min_match=None):
    """ExecuteCountGroupsBatch over the segments of every rank (sdbg_dist_match_count_batch_groups_min): this rank's counts
    are all-reduced on the device. Every rank makes the call with the same queries; a flat OR is one group per query, a
    flat AND single-term groups. Returns uint64[Q], the same on every rank."""
    counts = np.zeros(len(queries), np.uint64)
    N.check(N.lib().sdbg_dist_match_count_batch_groups_min(_seg_array(reader.segments), len(reader.segments),
                                                           *_query_args(queries, exclude, min_match, groups=True), _ref(filt),
                                                           _ptr(counts)), reader.segments[0].ctx._h)
    return counts


def _dist_key_range(key_min, key_span):
    if key_min is None or key_span is None:   # a per-rank column range would differ between ranks
        raise ValueError("the dist entries need key_min and key_span: the same range on every rank")
    return int(key_min), int(key_span)


# The dist wrappers check nothing that depends on this rank's segments before the library call: a missing or mistyped
# column is reported by the call after the collective, on every rank. The column type the results are decoded with is
# read after the call has succeeded, when every rank's segments are known to hold the column with one type.
def _value_type(reader, field):
    vt = reader.segments[0].col_types.get(int(field))
    if vt is None:   # the values come back as raw bits: their type must be known, not guessed
        raise ValueError("column %d was not staged through this Segment" % int(field))
    return vt


def ExecuteDistFacetCountsGroupsBatch(reader, queries, key_field, key_min, key_span, filt=None, exclude=None, min_match=None):
    """ExecuteFacetCountsGroupsBatch over the segments of every rank (sdbg_dist_match_facet_counts_batch_groups_min): the
    counts are all-reduced on the device. key_min / key_span are required and must be the same on every rank. Returns the
    dict ExecuteFacetCountsBatch returns."""
    key_min, key_span = _dist_key_range(key_min, key_span)
    nq = len(queries)
    counts = np.zeros((max(nq, 1), max(key_span, 1)), np.uint64)
    nulls = np.zeros(max(nq, 1), np.uint64)
    N.check(N.lib().sdbg_dist_match_facet_counts_batch_groups_min(
        _seg_array(reader.segments), len(reader.segments), *_query_args(queries, exclude, min_match, groups=True),
        _ref(filt), int(key_field), key_min, key_span, _ptr(counts), _ptr(nulls)), reader.segments[0].ctx._h)
    return dict(key_min=key_min, counts=counts[:nq], nulls=nulls[:nq])


def _dist_agg_key(key_field, key_min, key_span):
    """(key field, key_min, key_span) of a dist aggregate call; key_field None: one group, (0, 1)."""
    if key_field is None:
        return N.UINT64_MAX, 0, 1
    return (int(key_field),) + _dist_key_range(key_min, key_span)


def ExecuteDistMatchAggregatesGroupsBatch(reader, queries, value_field, key_field=None, key_min=None, key_span=None, filt=None,
                                          exclude=None, min_match=None):
    """ExecuteMatchAggregatesGroupsBatch over the segments of every rank (sdbg_dist_match_aggregate_batch_groups_min): each
    rank's cells are all-gathered and merged on the device. Grouped, key_min / key_span are required and must be the same
    on every rank. Returns the dict ExecuteMatchAggregatesBatch returns, the same on every rank."""
    kf, key_min, key_span = _dist_agg_key(key_field, key_min, key_span)
    nq = len(queries)
    out = np.zeros((max(nq, 1), max(key_span, 1)), MATCH_AGG_DTYPE)
    null_out = np.zeros(max(nq, 1), MATCH_AGG_DTYPE)
    N.check(N.lib().sdbg_dist_match_aggregate_batch_groups_min(
        _seg_array(reader.segments), len(reader.segments), *_query_args(queries, exclude, min_match, groups=True),
        _ref(filt), kf, key_min, key_span, int(value_field), _ptr(out), _ptr(null_out)), reader.segments[0].ctx._h)
    return _agg_result(out, null_out, nq, key_min, _value_type(reader, value_field))


def match_aggregate_device_bytes(nq, key_span=1):
    """Bytes of one rank's buffer of MatchAggregatesDevice: a 64-byte header and nq * (key_span + 1) cells of 48 bytes."""
    return 64 + int(nq) * (int(key_span) + 1) * 48


def MatchAggregatesDevice(reader, queries, value_field, d_cells_ptr, key_field=None, key_min=None, key_span=None, filt=None,
                          exclude=None, min_match=None):
    """This rank's aggregate cells left in HBM at d_cells_ptr (match_aggregate_device_bytes), for an all-gather and
    merge_aggregates_gathered (sdbg_match_aggregate_batch_groups_min_device). Nothing waits."""
    kf, key_min, key_span = _dist_agg_key(key_field, key_min, key_span)
    N.check(N.lib().sdbg_match_aggregate_batch_groups_min_device(
        _seg_array(reader.segments), len(reader.segments), *_query_args(queries, exclude, min_match, groups=True),
        _ref(filt), kf, key_min, key_span, int(value_field), C.c_void_p(int(d_cells_ptr))), reader.segments[0].ctx._h)


def merge_aggregates_gathered(ctx, d_all_ptr, n_ranks, nq, value_type, key_min=0, key_span=1):
    """The aggregates of n_ranks ranks' MatchAggregatesDevice buffers, back to back in HBM
    (sdbg_match_aggregate_merge_gathered). value_type: the value column's type code. Returns the dict
    ExecuteMatchAggregatesBatch returns."""
    out = np.zeros((max(int(nq), 1), max(int(key_span), 1)), MATCH_AGG_DTYPE)
    null_out = np.zeros(max(int(nq), 1), MATCH_AGG_DTYPE)
    N.check(N.lib().sdbg_match_aggregate_merge_gathered(ctx._h, C.c_void_p(int(d_all_ptr)), int(n_ranks), int(nq), int(key_span),
                                                        _ptr(out), _ptr(null_out)), ctx._h)
    return _agg_result(out, null_out, int(nq), key_min, value_type)


def ExecuteDistTopKByColumnGroupsBatch(reader, queries, sort_field, k, descending=False, nulls_first=False, filt=None,
                                       exclude=None, min_match=None):
    """ExecuteTopKByColumnGroupsBatch over the segments of every rank (sdbg_dist_match_topk_by_column_batch_groups_min):
    each rank's k best rows are all-gathered and merged on the device. Returns the dict ExecuteTopKByColumnBatch returns,
    with segs = the rank and docs = the ordinal within the rank + 1; the same on every rank."""
    nq = len(queries)
    hits = np.zeros(max(nq, 1) * max(int(k), 1), SORT_HIT_DTYPE)
    n_out = np.zeros(max(nq, 1), np.uint32)
    N.check(N.lib().sdbg_dist_match_topk_by_column_batch_groups_min(
        _seg_array(reader.segments), len(reader.segments), *_query_args(queries, exclude, min_match, groups=True),
        _ref(filt), int(sort_field), int(bool(descending)), int(bool(nulls_first)), int(k), _ptr(hits), _ptr(n_out)),
        reader.segments[0].ctx._h)
    return _sort_result(hits, n_out, nq, k, _SORT_VALUE_DTYPE[_value_type(reader, sort_field)])


def topk_by_column_device_bytes(nq, k):
    """Bytes of one rank's buffer of TopKByColumnDevice: a 64-byte header, nq row counts and nq * k rows of 24 bytes."""
    return 64 + int(nq) * (8 + 24 * int(k))


def TopKByColumnDevice(reader, queries, sort_field, k, rank, d_rows_ptr, descending=False, nulls_first=False, filt=None,
                       exclude=None, min_match=None):
    """This rank's k best rows per query left in HBM at d_rows_ptr (topk_by_column_device_bytes), for an all-gather and
    merge_topk_by_column_gathered (sdbg_match_topk_by_column_batch_groups_min_device)."""
    N.check(N.lib().sdbg_match_topk_by_column_batch_groups_min_device(
        _seg_array(reader.segments), len(reader.segments), *_query_args(queries, exclude, min_match, groups=True),
        _ref(filt), int(sort_field), int(bool(descending)), int(bool(nulls_first)), int(k), int(rank),
        C.c_void_p(int(d_rows_ptr))), reader.segments[0].ctx._h)


def merge_topk_by_column_gathered(ctx, d_all_ptr, n_ranks, nq, k, value_type):
    """The sorted hits of n_ranks ranks' TopKByColumnDevice buffers, back to back in HBM
    (sdbg_match_topk_by_column_merge_gathered). value_type: the sort column's type code. Returns the dict
    ExecuteTopKByColumnBatch returns, with segs = the rank and docs = the ordinal within the rank + 1."""
    hits = np.zeros(max(int(nq), 1) * max(int(k), 1), SORT_HIT_DTYPE)
    n_out = np.zeros(max(int(nq), 1), np.uint32)
    N.check(N.lib().sdbg_match_topk_by_column_merge_gathered(ctx._h, C.c_void_p(int(d_all_ptr)), int(n_ranks), int(nq), int(k),
                                                             _ptr(hits), _ptr(n_out)), ctx._h)
    return _sort_result(hits, n_out, int(nq), int(k), _SORT_VALUE_DTYPE[value_type])


FOR_BLOCK_DTYPE =np.dtype([("base", "<i8"), ("bits", "<u4"), ("off8", "<u4")])


def pack_for(values, out_words=None):
    """Host-side writer of the bit-packed column format (sdbg_pack_for): returns (headers, words, rows). `out_words` may be a
    preallocated (e.g. pinned) uint64 array."""
    values = np.ascontiguousarray(values, dtype=np.int64)
    rows = len(values)
    headers = np.zeros((rows + 2047) // 2048, FOR_BLOCK_DTYPE)
    n = C.c_uint64(0)
    words = out_words if out_words is not None else np.zeros(rows + 1, np.uint64)      # never larger than the raw column + slack
    rc = N.lib().sdbg_pack_for(_ptr(values), rows, _ptr(headers), _ptr(words), len(words), C.byref(n))
    N.check(rc)
    return headers, words[:n.value], rows


def StreamScoredDocs(reader, seg_idx, query, kind, scorer, filt=None, doc_min=1, doc_max=None, exclude=None):
    """The search scan's streaming mode (duckdb_search_full_scan.cpp:2370 RunStreamingScan over
    DocIterator::EmitScoredDocs): every match of `query` in docs [doc_min, doc_max) of segment `seg_idx` with its score,
    ascending by doc id; `exclude` = term ids whose docs are left out (sdbg_bm25_scan_excl). Returns (docs u32, scores f32)."""
    seg = reader.segments[seg_idx]
    x = np.ascontiguousarray(list(exclude) if exclude else [], dtype=np.uint32)
    terms = (N.BM25Term * len(query))(*[reader.stats(scorer, t) for t in query])
    fp = C.byref(filt) if filt is not None else None
    hi = int(doc_max) if doc_max is not None else 0xFFFFFFFF
    n = C.c_uint64(0)
    cap = 0
    docs = scores = None
    for _ in range(2):   # count-only call first, then one with exactly the room needed
        dp, sp = _ptr(docs) if docs is not None else None, _ptr(scores) if scores is not None else None
        if len(x):
            rc = N.lib().sdbg_bm25_scan_excl(seg._h, int(kind), terms, len(query), _ptr(x), len(x), scorer.k, scorer.b, fp,
                                             int(doc_min), hi, dp, sp, cap, C.byref(n))
        else:
            rc = N.lib().sdbg_bm25_scan(seg._h, int(kind), terms, len(query), scorer.k, scorer.b, fp, int(doc_min), hi,
                                        dp, sp, cap, C.byref(n))
        if rc == -6 and n.value > cap:
            cap = n.value
            docs, scores = np.zeros(cap, np.uint32), np.zeros(cap, np.float32)
            continue
        N.check(rc, seg.ctx._h)
        break
    if docs is None:
        return np.zeros(0, np.uint32), np.zeros(0, np.float32)
    return docs[:n.value], scores[:n.value]


def _flatten_queries(reader, queries, scorer):
    flat = [reader.stats(scorer, t) for q in queries for t in q]
    terms = (N.BM25Term * max(len(flat), 1))()
    for i, t in enumerate(flat):
        terms[i] = t
    off = np.zeros(len(queries) + 1, np.uint32)
    off[1:] = np.cumsum([len(q) for q in queries])
    return terms, off


class PreparedBatch:
    """Query descriptors marshalled once (terms + statistics), reusable across steps."""

    def __init__(self, reader, queries, kind, scorer, k, filt=None, threshold=FLT_MIN, exclude=None):
        self.reader, self.kind, self.scorer, self.k, self.filt, self.threshold = reader, int(kind), scorer, int(k), filt, float(threshold)
        self.nq = len(queries)
        self.terms, self.off = _flatten_queries(reader, queries, scorer)
        self.excl = _exclusions(exclude, self.nq)   # None: no query excludes anything
        self.hits = np.zeros((self.nq, self.k), HIT_DTYPE)
        self.n_out = np.zeros(self.nq, np.uint32)
        self.total = np.zeros(self.nq, np.uint64)

    def run_host(self):
        """Full API call: host descriptors in, host hits out."""
        r = self.reader
        fp = C.byref(self.filt) if self.filt is not None else None
        if self.excl is None:
            N.check(N.lib().sdbg_bm25_topk_batch(_seg_array(r.segments), len(r.segments), self.kind, self.terms,
                                                 _ptr(self.off), self.nq, self.scorer.k, self.scorer.b, fp, self.k, self.threshold,
                                                 _ptr(self.hits), _ptr(self.n_out), _ptr(self.total)), r.segments[0].ctx._h)
        else:
            N.check(N.lib().sdbg_bm25_topk_batch_excl(_seg_array(r.segments), len(r.segments), self.kind, self.terms,
                                                      _ptr(self.off), self.nq, _ptr(self.excl[0]), _ptr(self.excl[1]), self.scorer.k,
                                                      self.scorer.b, fp, self.k, self.threshold, _ptr(self.hits), _ptr(self.n_out),
                                                      _ptr(self.total)), r.segments[0].ctx._h)
        return self.hits, self.n_out, self.total

    def _no_exclusions(self, what):
        if self.excl is not None:
            raise NotImplementedError(what + " has no exclusion form: use run_host")

    def run_dist(self, to_host=True):
        """Distributed top-k (sdbg_dist_bm25_topk_batch): local scan, one all-gather, local selection -- all enqueued by
        the library on its stream. to_host=False leaves the merged keys in HBM and returns without waiting."""
        self._no_exclusions("run_dist")
        r = self.reader
        fp = C.byref(self.filt) if self.filt is not None else None
        if to_host:
            hits = np.zeros((self.nq, self.k), HIT_DTYPE)
            n_out = np.zeros(self.nq, np.uint32)
            hp, npp = _ptr(hits), _ptr(n_out)
        else:
            hits = n_out = None
            hp = npp = None
        N.check(N.lib().sdbg_dist_bm25_topk_batch(_seg_array(r.segments), len(r.segments), self.kind, self.terms, _ptr(self.off), self.nq,
                                                  self.scorer.k, self.scorer.b, fp, self.k, self.threshold, hp, npp), r.segments[0].ctx._h)
        return hits, n_out

    def run_device(self, rank, d_keys_ptr, d_totals_ptr=None):
        """Results stay in HBM as sortable keys (for the multi-GPU gather + merge)."""
        self._no_exclusions("run_device")
        r = self.reader
        fp = C.byref(self.filt) if self.filt is not None else None
        N.check(N.lib().sdbg_bm25_topk_batch_device(_seg_array(r.segments), len(r.segments), self.kind, self.terms,
                                                    _ptr(self.off), self.nq, self.scorer.k, self.scorer.b, fp, self.k, self.threshold,
                                                    int(rank), C.c_void_p(int(d_keys_ptr)),
                                                    C.c_void_p(int(d_totals_ptr)) if d_totals_ptr else None),
                r.segments[0].ctx._h)


def merge_gathered(ctx, d_keys_all_ptr, n_ranks, nq, k, to_host=True):
    """Global top-k from the keys every rank contributed ([rank][query][k] u64 in HBM)."""
    if not to_host:
        N.check(N.lib().sdbg_topk_merge_gathered(ctx._h, C.c_void_p(int(d_keys_all_ptr)), int(n_ranks), int(nq), int(k),
                                                 None, None), ctx._h)
        return None, None
    hits = np.zeros((nq, k), HIT_DTYPE)
    n_out = np.zeros(nq, np.uint32)
    N.check(N.lib().sdbg_topk_merge_gathered(ctx._h, C.c_void_p(int(d_keys_all_ptr)), int(n_ranks), int(nq), int(k),
                                             _ptr(hits), _ptr(n_out)), ctx._h)
    return hits, n_out


def ExecuteTopK(reader, query_terms, kind, scorer, k, filt=None, threshold=FLT_MIN, exclude=None):
    """irs::ExecuteTopK for one query: hits sorted by (score desc, seg asc, doc asc), total matches. exclude: term ids whose
    docs are left out (`a & b & !c`)."""
    hits, n_out, total = ExecuteTopKBatch(reader, _one(query_terms), kind, scorer, k, filt, threshold, exclude=_one(exclude))
    return hits[0, :n_out[0]].copy(), int(total[0])


class IResearchScan:
    """The ColScan / count shapes of the `iresearch_scan` table function
    (server/connector/duckdb_search_full_scan.hpp:56-77) with the aggregate above it pushed into the scan."""

    def __init__(self, segments):
        self.segments = list(segments)
        self.ctx = self.segments[0].ctx

    def count_sum(self, preds, sum_field=None):
        cnt = C.c_uint64()
        s128 = (C.c_int64 * 2)()
        sf = C.c_double()
        N.check(N.lib().sdbg_filter_count_sum(_seg_array(self.segments), len(self.segments), _pred_array(preds),
                                              len(preds), NO_FIELD if sum_field is None else int(sum_field),
                                              C.byref(cnt), s128, C.byref(sf)), self.ctx._h)
        si = (int(s128[1]) << 64) | (int(s128[0]) & 0xFFFFFFFFFFFFFFFF)
        return cnt.value, si, sf.value

    def prepare_count_sum(self, preds, sum_field=None):
        """The same call with its arguments marshalled once (a point query is ~10 us on the device side; building the
        ctypes arrays per call costs about as much). Returns a callable -> (count, sum_int, sum_f64)."""
        segs, n_segs, pa, n_preds = _seg_array(self.segments), len(self.segments), _pred_array(preds), len(preds)
        field = NO_FIELD if sum_field is None else int(sum_field)
        cnt, s128, sf = C.c_uint64(), (C.c_int64 * 2)(), C.c_double()
        pc, psf = C.byref(cnt), C.byref(sf)
        fn, h = N.lib().sdbg_filter_count_sum, self.ctx._h

        def run():
            rc = fn(segs, n_segs, pa, n_preds, field, pc, s128, psf)
            if rc:
                N.check(rc, h)
            return cnt.value, (int(s128[1]) << 64) | (int(s128[0]) & 0xFFFFFFFFFFFFFFFF), sf.value
        return run

    def groupby(self, preds, key_field, sum_int_field=None, avg_f64_field=None, cap=None, n_groups_hint=0):
        cap = int(cap if cap is not None else max(n_groups_hint, 1 << 20))
        out = np.zeros(cap, GROUP_DTYPE)
        n = C.c_uint64()
        N.check(N.lib().sdbg_filter_groupby(_seg_array(self.segments), len(self.segments), _pred_array(preds),
                                            len(preds), int(key_field), int(n_groups_hint),
                                            NO_FIELD if sum_int_field is None else int(sum_int_field),
                                            NO_FIELD if avg_f64_field is None else int(avg_f64_field),
                                            _ptr(out), cap, C.byref(n)), self.ctx._h)
        return out[:n.value]

    def groupby_partial(self, preds, key_field, key_min, key_span, sum_int_field, avg_f64_field, d_i64_ptr, d_f64_ptr):
        N.check(N.lib().sdbg_filter_groupby_partial(_seg_array(self.segments), len(self.segments), _pred_array(preds),
                                                    len(preds), int(key_field), int(key_min), int(key_span),
                                                    NO_FIELD if sum_int_field is None else int(sum_int_field),
                                                    NO_FIELD if avg_f64_field is None else int(avg_f64_field),
                                                    C.c_void_p(int(d_i64_ptr)), C.c_void_p(int(d_f64_ptr))), self.ctx._h)

    def groupby_finalize(self, key_min, key_span, d_i64_ptr, d_f64_ptr, cap, out=None):
        if out is None:
            out = np.empty(int(cap), GROUP_DTYPE)
        n = C.c_uint64()
        N.check(N.lib().sdbg_groupby_finalize(self.ctx._h, int(key_min), int(key_span), C.c_void_p(int(d_i64_ptr)),
                                              C.c_void_p(int(d_f64_ptr)), _ptr(out), int(cap), C.byref(n)), self.ctx._h)
        return out[:n.value]


def sum_i128(rows):
    """Python ints of the 128-bit SUM(int) column of a group result."""
    return [(int(h) << 64) | (int(l) & 0xFFFFFFFFFFFFFFFF) for l, h in zip(rows["sum_lo"], rows["sum_hi"])]
