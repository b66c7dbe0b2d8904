"""ctypes binding of libsdbg.so -- the only way Python reaches the kernels. Loading fails loudly:
there is no Python/CPU stand-in for any entry point."""
import ctypes as C
import os

from . import build as _build

_lib = None

OK = 0
ERR = {-1: "EINVAL", -2: "ENODEVICE", -3: "ECUDA", -4: "EFORMAT", -5: "ENOTFOUND", -6: "ECAPACITY",
       -7: "EUNSUPPORTED"}
UINT64_MAX = 0xFFFFFFFFFFFFFFFF


class TermMeta(C.Structure):
    _fields_ = [("docs_count", C.c_uint32), ("freq", C.c_uint32), ("doc_start", C.c_uint64),
                ("e_skip_start", C.c_uint64)]


class NormRg(C.Structure):
    _fields_ = [("byte_size", C.c_uint8), ("row_count", C.c_uint32), ("file_offset", C.c_uint64)]


class ColPred(C.Structure):
    _fields_ = [("field", C.c_uint64), ("op", C.c_int32), ("is_float", C.c_int32), ("lo_i", C.c_int64),
                ("hi_i", C.c_int64), ("lo_f", C.c_double), ("hi_f", C.c_double)]


class BM25Term(C.Structure):
    _fields_ = [("idf", C.c_float), ("norm_const", C.c_float), ("norm_length", C.c_float),
                ("boost", C.c_float), ("term", C.c_uint32)]


class Hit(C.Structure):
    _fields_ = [("score", C.c_float), ("doc", C.c_uint32), ("seg", C.c_uint32)]


class GroupRow(C.Structure):
    _fields_ = [("key", C.c_int64), ("count", C.c_uint64), ("sum_i128", C.c_int64 * 2),
                ("sum_f64", C.c_double), ("cnt_f64", C.c_uint64)]


class MatchAgg(C.Structure):
    _fields_ = [("count", C.c_uint64), ("count_value", C.c_uint64), ("sum_i128", C.c_int64 * 2), ("sum_f64", C.c_double),
                ("min", C.c_int64), ("max", C.c_int64)]


# every symbol include/sdbg.h declares: name -> (restype, argtypes)
_vp, _sz = C.c_void_p, C.c_size_t
_u32p, _u64p, _f32p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_float)
SIGNATURES = {
    "sdbg_init": (C.c_int, [C.c_int, C.POINTER(_vp)]),
    "sdbg_destroy": (None, [_vp]),
    "sdbg_last_error": (C.c_char_p, [_vp]),
    "sdbg_version": (C.c_char_p, []),
    "sdbg_timer_start": (C.c_int, [_vp]),
    "sdbg_timer_stop": (C.c_int, [_vp, _f32p]),
    "sdbg_sync": (C.c_int, [_vp]),
    "sdbg_launch_count": (C.c_uint64, [_vp]),
    "sdbg_flush_l2": (C.c_int, [_vp]),
    "sdbg_set_wand": (C.c_int, [_vp, C.c_int]),
    "sdbg_profile_enable": (C.c_int, [_vp, C.c_int]),
    "sdbg_profile_read": (C.c_int, [_vp, C.c_int, C.POINTER(C.c_double), _u64p]),
    "sdbg_segment_create": (C.c_int, [_vp, C.c_uint32, C.POINTER(_vp)]),
    "sdbg_segment_destroy": (None, [_vp]),
    "sdbg_stage_postings": (C.c_int, [_vp, _vp, _sz, _vp, _sz, C.c_int]),
    "sdbg_stage_norms": (C.c_int, [_vp, _vp, _sz, _vp, _sz]),
    "sdbg_stage_column": (C.c_int, [_vp, C.c_uint64, C.c_int, _vp, _vp, C.c_uint64]),
    "sdbg_stage_column_device": (C.c_int, [_vp, C.c_uint64, C.c_int, _vp, C.c_uint64]),
    "sdbg_column_device_ptr": (C.c_int, [_vp, C.c_uint64, C.POINTER(_vp), _u64p]),
    "sdbg_column_to_host": (C.c_int, [_vp, C.c_uint64, _vp, C.c_uint64]),
    "sdbg_pack_for": (C.c_int, [_vp, C.c_uint64, _vp, _vp, C.c_uint64, _u64p]),
    "sdbg_stage_column_for": (C.c_int, [_vp, C.c_uint64, _vp, _vp, C.c_uint64, C.c_uint64]),
    "sdbg_column_for_to_host": (C.c_int, [_vp, C.c_uint64, _vp, _vp, C.c_uint64, _u64p]),
    "sdbg_gather_column": (C.c_int, [_vp, C.c_uint64, _vp, _sz, _vp, _vp]),
    "sdbg_segment_posting_stats": (C.c_int, [_vp, _u64p, _u64p, _u64p, _u64p]),
    "sdbg_segment_term_bytes": (C.c_int, [_vp, _vp, _sz]),
    "sdbg_bm25_collect": (C.c_int, [C.c_uint64, C.c_uint64, C.c_uint64, C.c_float, C.c_float, C.POINTER(BM25Term)]),
    "sdbg_stage_docs_mask": (C.c_int, [_vp, _vp, _sz]),
    "sdbg_segment_set_wand_b": (C.c_int, [_vp, C.c_float]),
    "sdbg_segment_set_wand_avg_dl": (C.c_int, [_vp, C.c_float]),
    "sdbg_segment_context": (_vp, [_vp]),
    "sdbg_tfidf_collect": (C.c_int, [C.c_uint64, C.c_uint64, _vp]),
    "sdbg_tfidf_topk_batch": (C.c_int, [_vp, _sz, C.c_int, _vp, _vp, _sz, C.c_int, _vp, C.c_uint32, C.c_float, _vp, _vp, _vp]),
    "sdbg_scan_stats": (C.c_int, [_vp, _u64p, _u64p]),
    "sdbg_dist_unique_id": (C.c_int, [_vp]),
    "sdbg_dist_init": (C.c_int, [_vp, _vp, C.c_int, C.c_int]),
    "sdbg_dist_destroy": (C.c_int, [_vp]),
    "sdbg_dist_allreduce_i64": (C.c_int, [_vp, _vp, _sz]),
    "sdbg_dist_allgather": (C.c_int, [_vp, _vp, _vp, _sz]),
    "sdbg_dist_groupby_merge": (C.c_int, [_vp, _vp, _vp, C.c_uint64, C.c_double]),
    "sdbg_dist_bm25_topk_batch": (C.c_int, [_vp, _sz, C.c_int, _vp, _vp, _sz, C.c_float, C.c_float, _vp, C.c_uint32, C.c_float, _vp, _vp]),
    "sdbg_bm25_topk": (C.c_int, [_vp, _sz, C.c_int, _vp, _sz, C.c_float, C.c_float, _vp, C.c_uint32, C.c_float, _vp, _u32p,
                                 _u64p, _f32p]),
    "sdbg_bm25_topk_batch": (C.c_int, [_vp, _sz, C.c_int, _vp, _vp, _sz, C.c_float, C.c_float, _vp, C.c_uint32, C.c_float,
                                       _vp, _vp, _vp]),
    "sdbg_bm25_topk_batch_device": (C.c_int, [_vp, _sz, C.c_int, _vp, _vp, _sz, C.c_float, C.c_float, _vp, C.c_uint32,
                                              C.c_float, C.c_uint32, _vp, _vp]),
    "sdbg_bm25_scan": (C.c_int, [_vp, C.c_int, _vp, _sz, C.c_float, C.c_float, _vp, C.c_uint32, C.c_uint32, _vp, _vp, C.c_uint64,
                                 _u64p]),
    "sdbg_bm25_topk_batch_excl": (C.c_int, [_vp, _sz, C.c_int, _vp, _vp, _sz, _vp, _vp, C.c_float, C.c_float, _vp, C.c_uint32,
                                            C.c_float, _vp, _vp, _vp]),
    "sdbg_bm25_scan_excl": (C.c_int, [_vp, C.c_int, _vp, _sz, _vp, _sz, C.c_float, C.c_float, _vp, C.c_uint32, C.c_uint32, _vp,
                                      _vp, C.c_uint64, _u64p]),
    "sdbg_match_count_batch": (C.c_int, [_vp, _sz, C.c_int, _vp, _vp, _sz, _vp, _vp, _vp, _vp]),
    "sdbg_match_topk_by_column_batch": (C.c_int, [_vp, _sz, C.c_int, _vp, _vp, _sz, _vp, _vp, _vp, C.c_uint64, C.c_int, C.c_int,
                                                  C.c_uint32, _vp, _vp]),
    "sdbg_match_facet_counts_batch": (C.c_int, [_vp, _sz, C.c_int, _vp, _vp, _sz, _vp, _vp, _vp, C.c_uint64, C.c_int64,
                                                C.c_uint32, _vp, _vp]),
    "sdbg_bm25_topk_batch_groups": (C.c_int, [_vp, _sz, _vp, _vp, _vp, _sz, _vp, _vp, C.c_float, C.c_float, _vp, C.c_uint32,
                                              C.c_float, _vp, _vp, _vp]),
    "sdbg_match_count_batch_groups": (C.c_int, [_vp, _sz, _vp, _vp, _vp, _sz, _vp, _vp, _vp, _vp]),
    "sdbg_bm25_topk_batch_groups_min": (C.c_int, [_vp, _sz, _vp, _vp, _vp, _vp, _sz, _vp, _vp, C.c_float, C.c_float, _vp,
                                                  C.c_uint32, C.c_float, _vp, _vp, _vp]),
    "sdbg_match_count_batch_groups_min": (C.c_int, [_vp, _sz, _vp, _vp, _vp, _vp, _sz, _vp, _vp, _vp, _vp]),
    "sdbg_match_topk_by_column_batch_groups_min": (C.c_int, [_vp, _sz, _vp, _vp, _vp, _vp, _sz, _vp, _vp, _vp, C.c_uint64,
                                                             C.c_int, C.c_int, C.c_uint32, _vp, _vp]),
    "sdbg_match_facet_counts_batch_groups_min": (C.c_int, [_vp, _sz, _vp, _vp, _vp, _vp, _sz, _vp, _vp, _vp, C.c_uint64,
                                                           C.c_int64, C.c_uint32, _vp, _vp]),
    "sdbg_match_aggregate_batch": (C.c_int, [_vp, _sz, C.c_int, _vp, _vp, _sz, _vp, _vp, _vp, C.c_uint64, C.c_int64,
                                             C.c_uint32, C.c_uint64, _vp, _vp]),
    "sdbg_match_aggregate_batch_groups_min": (C.c_int, [_vp, _sz, _vp, _vp, _vp, _vp, _sz, _vp, _vp, _vp, C.c_uint64,
                                                        C.c_int64, C.c_uint32, C.c_uint64, _vp, _vp]),
    "sdbg_dist_match_count_batch_groups_min": (C.c_int, [_vp, _sz, _vp, _vp, _vp, _vp, _sz, _vp, _vp, _vp, _vp]),
    "sdbg_dist_match_facet_counts_batch_groups_min": (C.c_int, [_vp, _sz, _vp, _vp, _vp, _vp, _sz, _vp, _vp, _vp, C.c_uint64,
                                                                C.c_int64, C.c_uint32, _vp, _vp]),
    "sdbg_match_aggregate_batch_groups_min_device": (C.c_int, [_vp, _sz, _vp, _vp, _vp, _vp, _sz, _vp, _vp, _vp, C.c_uint64,
                                                               C.c_int64, C.c_uint32, C.c_uint64, _vp]),
    "sdbg_match_aggregate_merge_gathered": (C.c_int, [_vp, _vp, C.c_uint32, _sz, C.c_uint32, _vp, _vp]),
    "sdbg_dist_match_aggregate_batch_groups_min": (C.c_int, [_vp, _sz, _vp, _vp, _vp, _vp, _sz, _vp, _vp, _vp, C.c_uint64,
                                                             C.c_int64, C.c_uint32, C.c_uint64, _vp, _vp]),
    "sdbg_match_topk_by_column_batch_groups_min_device": (C.c_int, [_vp, _sz, _vp, _vp, _vp, _vp, _sz, _vp, _vp, _vp,
                                                                    C.c_uint64, C.c_int, C.c_int, C.c_uint32, C.c_uint32, _vp]),
    "sdbg_match_topk_by_column_merge_gathered": (C.c_int, [_vp, _vp, C.c_uint32, _sz, C.c_uint32, _vp, _vp]),
    "sdbg_dist_match_topk_by_column_batch_groups_min": (C.c_int, [_vp, _sz, _vp, _vp, _vp, _vp, _sz, _vp, _vp, _vp, C.c_uint64,
                                                                  C.c_int, C.c_int, C.c_uint32, _vp, _vp]),
    "sdbg_topk_merge_gathered": (C.c_int, [_vp, _vp, C.c_uint32, _sz, C.c_uint32, _vp, _vp]),
    "sdbg_decode_score_term": (C.c_int, [_vp, C.c_uint32, C.c_float, C.c_float, C.c_float, _vp, _vp, _vp]),
    "sdbg_col_pred_resolve": (C.c_int, [C.POINTER(ColPred), C.c_int, C.POINTER(ColPred)]),
    "sdbg_filter_bitmap": (C.c_int, [_vp, _vp, _sz, _vp]),
    "sdbg_filter_count_sum": (C.c_int, [_vp, _sz, _vp, _sz, C.c_uint64, _u64p, _vp, C.POINTER(C.c_double)]),
    "sdbg_filter_groupby": (C.c_int, [_vp, _sz, _vp, _sz, C.c_uint64, C.c_uint32, C.c_uint64, C.c_uint64, _vp,
                                      C.c_uint64, _u64p]),
    "sdbg_filter_groupby_partial": (C.c_int, [_vp, _sz, _vp, _sz, C.c_uint64, C.c_int64, C.c_uint64, C.c_uint64,
                                              C.c_uint64, _vp, _vp]),
    "sdbg_groupby_finalize": (C.c_int, [_vp, C.c_int64, C.c_uint64, _vp, _vp, _vp, C.c_uint64, _u64p]),
    "sdbg_column_minmax_i64": (C.c_int, [_vp, C.c_uint64, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "sdbg_writer_create": (C.c_int, [C.c_uint32, C.c_int, C.c_float, _vp, C.POINTER(_vp)]),
    "sdbg_writer_destroy": (None, [_vp]),
    "sdbg_writer_add_term": (C.c_int, [_vp, _vp, _vp, C.c_uint32]),
    "sdbg_writer_finish": (C.c_int, [_vp, C.POINTER(_vp), C.POINTER(_sz), C.POINTER(_vp), C.POINTER(_sz)]),
    "sdbg_synth_corpus": (C.c_int, [_vp, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, _vp, _u64p]),
    "sdbg_synth_corpus_ex": (C.c_int, [_vp, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_double, _vp, _u64p]),
    "sdbg_synth_column": (C.c_int, [_vp, C.c_uint64, C.c_uint64, C.c_int, C.c_uint64, C.c_uint64]),
    "sdbg_synth_hash": (C.c_uint64, [C.c_uint64, C.c_uint64]),
    "sdbg_debug_stage_host": (C.c_int, [_vp, _sz, _vp, _sz, C.c_int, C.c_uint32, _u32p, _vp, _vp, _vp, _vp, _vp,
                                        _vp, _u64p]),
}


def lib():
    """The loaded library. Builds it first when sources are newer (needs nvcc)."""
    global _lib
    if _lib is None:
        path = _build.build()
        if not os.path.exists(path):
            raise RuntimeError("libsdbg.so is missing: the CUDA extension must be built (serenedb_b200.build)")
        L = C.CDLL(path)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError here == ABI symbol missing: fail loudly
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


class SdbgError(RuntimeError):
    pass


def check(rc, ctx=None):
    if rc == OK:
        return
    msg = ERR.get(rc, str(rc))
    if ctx is not None:
        detail = lib().sdbg_last_error(ctx)
        if detail:
            msg += ": " + detail.decode(errors="replace")
    raise SdbgError(msg)
