/* include/sdbg.h -- C ABI of libsdbg.so: the H100 (sm_90a) implementation of SereneDB's
 * query-time hot path. Plain pointers and sizes only; no C++/torch types cross this boundary.
 *
 * What each entry point replaces in the reference (paths relative to /root/reference, "irs/" =
 * libs/iresearch/include/iresearch/):
 *
 *   sdbg_stage_postings   the per-segment open of the ".doc" stream + term metas that
 *                         PostingsReaderBase::prepare / ::decode perform
 *                         (irs/formats/posting/reader.hpp:100-226) -- index-load time.
 *   sdbg_stage_norms      NormColumnReader (irs/formats/column/norm_column_reader.hpp:43-108).
 *   sdbg_stage_column     ColumnReader open of a `.col` column (irs/formats/column/column_reader.hpp:90-256).
 *   sdbg_bm25_topk        the body of DocIterator::Collect for the WAND iterators built in
 *                         PostingsReaderImpl::WandIterator (irs/formats/posting/reader.hpp:457-501),
 *                         driven by irs::ExecuteTopK (irs/search/doc_collector.hpp:88-136) and by
 *                         CollectSegmentTopK (server/connector/duckdb_search_full_scan.cpp:1868-1921);
 *                         with `filt` it is TableFilterDocIterator::Collect
 *                         (irs/index/table_filter_iterator.cpp:450-475).
 *   sdbg_filter_bitmap    ColFilterChain::FilterWindow (irs/index/table_filter_iterator.cpp:147-264).
 *   sdbg_filter_count_sum RunCountScan / UNGROUPED_AGGREGATE over iresearch_scan
 *                         (server/connector/duckdb_search_full_scan.cpp:2201-2239).
 *   sdbg_filter_groupby   RunColScan + FullScanner::Scan feeding DuckDB's HASH_GROUP_BY
 *                         (duckdb_search_full_scan.cpp:2405-2433, server/connector/full_scanner.cpp:81-147).
 *
 * Conventions: every function returns 0 on success and a negative SDBG_E* code otherwise; it never
 * throws. The caller owns all host buffers. Handles are opaque. A context owns one CUDA device and
 * one stream; calls on one context are serialised by the caller (one context per worker thread,
 * like one DocIterator per (segment, query, worker) in the reference). There is NO CPU fallback:
 * without a CUDA device sdbg_init fails with SDBG_ENODEVICE.
 */
#ifndef SDBG_H_
#define SDBG_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SDBG_OK 0
#define SDBG_EINVAL (-1)    /* bad argument */
#define SDBG_ENODEVICE (-2) /* no CUDA device / wrong architecture */
#define SDBG_ECUDA (-3)     /* CUDA runtime error (see sdbg_last_error) */
#define SDBG_EFORMAT (-4)   /* corrupt posting stream */
#define SDBG_ENOTFOUND (-5) /* unknown field */
#define SDBG_ECAPACITY (-6) /* output buffer too small */
#define SDBG_EUNSUPPORTED (-7)

typedef struct sdbg_ctx sdbg_ctx;
typedef struct sdbg_segment sdbg_segment;

/* ---- lifecycle ---- */
int sdbg_init(int device, sdbg_ctx** out);
void sdbg_destroy(sdbg_ctx*);
const char* sdbg_last_error(const sdbg_ctx*);
const char* sdbg_version(void);
/* Device-side timing on the context's stream (CUDA events), so callers never guess the stream. */
int sdbg_timer_start(sdbg_ctx*);
int sdbg_timer_stop(sdbg_ctx*, float* ms);
int sdbg_sync(sdbg_ctx*);
/* Number of kernels this context has launched since creation (bench's gpu_launches claim). */
uint64_t sdbg_launch_count(const sdbg_ctx*);
/* Block-max (WAND / MaxScore) pruning, the `WandContext` of irs::ExecuteTopK (doc_collector.hpp:88). On by
 * default when the segment carries block-max data; results (hits) are identical either way, but with
 * pruning total_matches is a lower bound (wand_scoring_test.cpp:382-384). Level 1: blocks / windows whose
 * block-max bound cannot beat the threshold are dropped while planning (single-term queries:
 * SingleWandIterator's skip). Level 2 (default) adds MaxScore's essential / non-essential split for
 * disjunctions (max_score_iterator.hpp:406-508): once the threshold exceeds the global bound of the
 * largest list, that list is no longer scanned but probed per surviving candidate -- used for queries whose
 * largest list is bitset-encoded (a probe is then a bit test + popcount rank, no block decode). 0 = off. */
int sdbg_set_wand(sdbg_ctx*, int level);
/* Per-kernel device timing for roofline reports: when enabled, a CUDA event pair is recorded on the
 * context's stream around each hot kernel launch. kernel_id: 0 filter_groupby, 1 bm25_topk,
 * 2 topk_merge, 3 filter_count_sum. read() synchronises and returns the summed duration and the
 * number of launches since enable(1); enable() resets the counters. */
int sdbg_profile_enable(sdbg_ctx*, int on);
int sdbg_profile_read(sdbg_ctx*, int kernel_id, double* total_ms, uint64_t* launches);
/* Writes `bytes` of device memory (> L2) to evict cached inputs between timed iterations. */
int sdbg_flush_l2(sdbg_ctx*);

/* ---- staging (index-load time): host bytes are copied to HBM; the caller may free them ---- */
typedef struct {
  uint32_t docs_count;   /* TermMetaImpl::docs_count */
  uint32_t freq;         /* total term frequency */
  uint64_t doc_start;    /* offset of the term's stream in the .doc bytes handed in */
  uint64_t e_skip_start; /* e_single_doc when docs_count == 1 (same union as reader.hpp:213-217) */
} sdbg_term_meta;

/* Doc ids are 1 .. 2^32 - 2: doc_limits::eof() = 2^32 - 1 is never a doc. docs_count > 2^32 - 2: SDBG_EINVAL.
 * The top-k and sorted entries take at most 2^32 - 2 docs summed over a call's segments (more:
 * SDBG_EUNSUPPORTED, nothing queued); the count and facet entries have no per-call limit. */
int sdbg_segment_create(sdbg_ctx*, uint32_t docs_count, sdbg_segment** out);
void sdbg_segment_destroy(sdbg_segment*);
/* doc_file: the ".doc" stream (posting blocks + skip data, format "1_5simd"); has_wand != 0 when
 * the field was indexed with block-max data (optimize_top_k) in the (freq, norm) pair layout
 * (WandType::MinNorm / DivNorm, wand_writer.hpp:302-381). The pairs only bound the scores of the scorer
 * they were written for: as in the reference (the field's wand scorers are matched with Scorer::equals),
 * the caller enables pruning (sdbg_set_wand) only for queries of that scorer; pass 0 for a field whose wand
 * payload has another layout (BM15's freq-only entries). Builds the per-block offset table and copies
 * 16-byte-aligned block payloads to HBM. */
int sdbg_stage_postings(sdbg_segment*, const uint8_t* doc_file, size_t n, const sdbg_term_meta* terms,
                        size_t n_terms, int has_wand);
/* The segment's DocumentMask (index_meta.hpp:39-43: the set of deleted doc ids). Masked docs are neither
 * scored, collected nor counted by the BM25 calls, like SegmentReaderImpl::mask wrapping the query iterator
 * (segment_reader_impl.cpp:95-157,318-326; duckdb_search_full_scan.cpp:1898). n == 0 clears the mask. */
int sdbg_stage_docs_mask(sdbg_segment*, const uint32_t* deleted_docs, size_t n);
/* Term positions of the segment's field, for phrase queries (sdbg_phrase_*_batch): term t's positions are
 * positions[term_pos_off[t] .. term_pos_off[t+1]) (term_pos_off has n_terms + 1 entries), in posting order, posting i of
 * the term contributing exactly its freq_i positions, strictly ascending within the posting: the values the reference's
 * position iterator yields (PosAttr::value()), decoded once at load time. Call after sdbg_stage_postings; restaging the
 * postings drops the positions, restaging the positions replaces them. HBM layout (DESIGN.md §3): 8 B per posting block,
 * 4 B per posting and 4 B per position. Errors: NULL segment or term_pos_off, postings not staged, n_terms different from
 * the staged term count, a decreasing term_pos_off, or NULL positions with a non-empty range: SDBG_EINVAL; a term whose
 * position count differs from the sum of its postings' frequencies, or positions not strictly ascending within a
 * posting: SDBG_EFORMAT (the segment keeps the positions it had). Synchronous. */
int sdbg_stage_positions(sdbg_segment*, const uint32_t* positions, const uint64_t* term_pos_off, size_t n_terms);
/* The b of the BM25 scorer the segment's block-max (wand) entries were written for (wand_writer.hpp:142-175; default
   0.75). Block-max pruning is used only for queries whose scorer has the same b -- the check Scorer::equals makes in
   PostingsReaderImpl::WandIterator (formats/posting/reader.hpp:457-501); any other scorer is evaluated exhaustively. */
int sdbg_segment_set_wand_b(sdbg_segment*, float wand_b);
/* The average field length the segment's block-max entries were chosen with (the writer's NormReader::GetAvg,
   norm_reader_impl.hpp:83-88). sdbg_stage_norms sets it from the staged norms (sum / non-zero count), so only a writer
   that used another average needs this; call it after sdbg_stage_norms. 0 = no norms. Queries score the entries as upper
   bounds under their own (corpus-wide) average length, so pruning stays exact when the two averages differ. */
int sdbg_segment_set_wand_avg_dl(sdbg_segment*, float avg_dl);
/* Zonemap effect of the last GROUP BY or sorted scan. GROUP BY: 2048-row blocks judged / proven dead from their min-max
 * (never read). Sorted scan (sdbg_match_topk_by_column_batch(_groups_min)): 65 536-doc windows judged / skipped before
 * any list was decoded, over the whole call. */
int sdbg_scan_stats(sdbg_ctx*, uint64_t* blocks_total, uint64_t* blocks_skipped);
/* The context a segment was created in (for sdbg_last_error after a failed call that only has segments at hand). */
sdbg_ctx* sdbg_segment_context(const sdbg_segment*);
typedef struct { uint8_t byte_size; uint32_t row_count; uint64_t file_offset; } sdbg_norm_rg; /* norm_writer.hpp:41-48 */
/* Row groups of fixed-width (1/2/4 B) little-endian field lengths; row = doc - 1. */
int sdbg_stage_norms(sdbg_segment*, const uint8_t* bytes, size_t n, const sdbg_norm_rg* rgs, size_t n_rg);
typedef enum { SDBG_I64 = 0, SDBG_F64 = 1, SDBG_I32 = 2 } sdbg_type;
/* validity may be NULL (NOT NULL column); otherwise bit r of validity[r/64] set => row r is valid. */
int sdbg_stage_column(sdbg_segment*, uint64_t field, sdbg_type t, const void* values,
                      const uint64_t* validity, uint64_t rows);
/* Same, but `d_values` already lives in device memory (borrowed, not copied, not freed). The library caches statistics
   of the values (min / max, zonemap): once the owner's writes to the buffer are complete, it calls this
   again with the same buffer before the next query, which drops them. The values must be complete when this is called. */
int sdbg_stage_column_device(sdbg_segment*, uint64_t field, sdbg_type t, const void* d_values, uint64_t rows);
/* Device address of a staged column's raw values, for callers that write them in place. The call means "about to
   write": it drops the cached statistics of the values (min / max, zonemap), and a bit-packed column
   drops its packed form, so the raw values at this address are the column until it is restaged. Writes go on after the
   context's queued work (sdbg_sync) and must be complete before the next call that reads the column; a caller that writes
   again later calls this again first. */
int sdbg_column_device_ptr(sdbg_segment*, uint64_t field, void** d_values, uint64_t* rows);
/* Copies the first `rows` values of a staged column back to host memory (tests / bench set-up). */
int sdbg_column_to_host(sdbg_segment*, uint64_t field, void* host_dst, uint64_t rows);
/* Bytes of HBM held by the segment's postings (payload + tables) and how many blocks were staged. */
int sdbg_segment_posting_stats(const sdbg_segment*, uint64_t* payload_bytes, uint64_t* table_bytes,
                               uint64_t* n_blocks, uint64_t* n_postings);

/* Encoded bytes (block headers + payloads, as in the .doc stream) of the first n_terms terms. */
int sdbg_segment_term_bytes(const sdbg_segment*, uint64_t* bytes_out, size_t n_terms);

/* ---- predicates (pushed TableFilterSet entries; NULL never passes) ----
 * `column op lo` (BETWEEN: lo <= column AND column <= hi, so lo > hi selects nothing). is_float selects which pair holds
 * the constants: lo_f / hi_f when is_float != 0, lo_i / hi_i otherwise; the other pair is ignored. Every entry point
 * resolves the constants against the filtered column's type (sdbg_col_pred_resolve) before any kernel sees them:
 *   - double column: IEEE comparison with the constant as a double (an integer constant is rounded to the nearest
 *     double, as a SQL cast of the constant to the column type does). NaN compares false, so `<> NaN` holds for every
 *     non-NULL row; -0.0 equals +0.0.
 *   - integer column (int64 raw or bit-packed, int32): the exact comparison of the integer with the constant. A double
 *     constant becomes the tightest integer bounds (v < 2.5 is v <= 2, v >= 2.5 is v >= 3); bounds beyond int64 hold
 *     for every row or none (v < 1e300, v > -inf: every row; v = 1e30: none); NaN holds for none, except `<> NaN`,
 *     which holds for every non-NULL row; `= 2.5` holds for none and `<> 2.5` for every non-NULL row. */
enum { SDBG_OP_LT = 0, SDBG_OP_LE, SDBG_OP_GT, SDBG_OP_GE, SDBG_OP_EQ, SDBG_OP_NE, SDBG_OP_BETWEEN,
       SDBG_OP_IS_NULL, SDBG_OP_IS_NOT_NULL };
/* Filter chains (`WHERE body @@ '...' AND a < x AND b = y`). Every full-text entry's `filt` -- the top-k, scan, count,
 * sorted, facet and aggregate entries, their *_device forms and the sdbg_dist_* entries -- points at a chain: when
 * filt[i].op has SDBG_OP_AND_NEXT set, filt[i] is ANDed with filt[i + 1], and the chain ends at the first entry without
 * the bit. A chain holds at most 4 predicates: the bit on the 4th gives SDBG_EUNSUPPORTED before anything is queued, and
 * a 5th entry is never read. A chain of one is the single predicate; filt == NULL is no filter. Each predicate follows
 * the rules above against its own column (int64 raw or bit-packed, int32 or double; NOT NULL or nullable); predicates
 * may repeat a column. Every column needs at least as many rows as the segment has docs (else SDBG_EINVAL; a column
 * that is not staged: SDBG_ENOTFOUND). Before any posting list is read, the chain is judged per 2048-row zone from the
 * zonemaps of its NOT NULL columns (DESIGN.md §4.13): zones where it holds for no row are skipped and zones where it
 * holds for every row are not read; results do not depend on it. The first call that judges a NOT NULL column's zones
 * (and the first after its values change: restaging, sdbg_column_device_ptr) waits once for the context's stream, to
 * copy the column's zonemap to the host; this holds for every entry taking `filt`, the *_device and sdbg_dist_* forms
 * included. sdbg_col_pred_resolve and the columnar entries
 * (preds, n_preds) take no chain: the bit there is an op outside SDBG_OP_* (SDBG_EINVAL). */
#define SDBG_OP_AND_NEXT 0x100
typedef struct {
  uint64_t field;
  int32_t op;
  int32_t is_float;
  int64_t lo_i, hi_i;
  double lo_f, hi_f;
} sdbg_col_pred;
/* The predicate the kernels evaluate for `in` on a column of type `type` (sdbg_type), under the rules above: on a double
 * column is_float = 1 with lo_f / hi_f; on an integer column is_float = 0 with lo_i / hi_i, a double constant turned into
 * BETWEEN [lo_i, hi_i] (lo_i > hi_i: no row) or, for `<>` an integral constant inside int64, `<>` that integer. Host-only
 * (no device needed). Errors: NULL pointers, an op outside SDBG_OP_*, an unknown type: SDBG_EINVAL. */
int sdbg_col_pred_resolve(const sdbg_col_pred* in, int type, sdbg_col_pred* out);

/* ---- BM25 top-k (boundary B2, irs::DocIterator::Collect) ---- */
/* `filt` of every entry below (top-k, scan, count, sorted, facet, aggregate; *_device and sdbg_dist_* forms): NULL or a
 * filter chain, see SDBG_OP_AND_NEXT above. */
enum { SDBG_QUERY_OR = 0, SDBG_QUERY_AND = 1 };
typedef struct { float idf, norm_const, norm_length, boost; uint32_t term; } sdbg_bm25_term; /* BM25Stats (bm25.hpp:49-56) + boost */
typedef struct { float score; uint32_t doc; uint32_t seg; } sdbg_hit;                          /* irs::ScoreDoc (iterators.hpp:93-101) */

/* BM25::collect mirror (irs/search/bm25.cpp:279-310): corpus-wide statistics -> BM25Stats. idf is
 * computed in double and narrowed, avg_dl divides two floats, norm_const = k - k*b. boost is set to 1. */
int sdbg_bm25_collect(uint64_t docs_with_field, uint64_t total_term_freq, uint64_t docs_with_term, float k,
                      float b, sdbg_bm25_term* out);

/* (k1, b) are the scorer's parameters (BM25::k(), BM25::b()): like BM25::PrepareScorer (bm25.cpp:312-365) they
 * select the scoring form -- k1 == 0: BM1 (every score 0 without a filter boost, :112-126), b == 0: BM15
 * (c0 - c0 / (1 + freq / k1), no norms, :70-87), otherwise BM25 (:90-107). Block-max pruning is applied only to
 * the BM25 form: the staged (freq, norm) pairs were chosen for it (wand_type() differs per form, bm25.cpp:407-418).
 * One query over the segments of this GPU. Accepts docs with score > threshold_in (seed it with
 * FLT_MIN like doc_collector.hpp:102, or with the cross-worker threshold). out has room for k hits,
 * returned sorted by (score desc, seg asc, doc asc); *threshold_out = k-th score if k hits exist. */
int sdbg_bm25_topk(sdbg_segment* const* segs, size_t n_segs, int kind, const sdbg_bm25_term* terms,
                   size_t n_terms, float k1, float b, const sdbg_col_pred* filt, uint32_t k, float threshold_in,
                   sdbg_hit* out, uint32_t* n_out, uint64_t* total_matches, float* threshold_out);
/* A batch of independent queries in one launch set (the benchmark-game / many-workers shape).
 * Query q uses terms[term_off[q] .. term_off[q+1]); out holds n_queries*k hits, n_out/total per query.
 * Memory: the results take n_queries * (8k + 12) B of HBM and as much pinned host memory for the copy back; the
 * query descriptors are staged from pageable memory. Synchronous on the context's stream. */
/* k1 = -1 is reserved: it selects the TFIDF scorer (b != 0: normalised) -- sdbg_tfidf_topk_batch is the named entry. */
int sdbg_bm25_topk_batch(sdbg_segment* const* segs, size_t n_segs, int kind, const sdbg_bm25_term* terms,
                         const uint32_t* term_off, size_t n_queries, float k1, float b, const sdbg_col_pred* filt,
                         uint32_t k, float threshold_in, sdbg_hit* out, uint32_t* n_out,
                         uint64_t* total_matches);
/* TFIDF (irs::TFIDF, search/tfidf.cpp): statistics (:149-150; only .idf and .boost of the term are used) and the same
 * batched scan scored with sqrt(freq) * boost * idf [/ sqrt(doc length) when normalize] (:59-80). Always exhaustive. */
int sdbg_tfidf_collect(uint64_t docs_with_field, uint64_t docs_with_term, sdbg_bm25_term* out);
int sdbg_tfidf_topk_batch(sdbg_segment* const* segs, size_t n_segs, int kind, const sdbg_bm25_term* terms,
                          const uint32_t* term_off, size_t n_queries, int normalize, const sdbg_col_pred* filt, uint32_t k,
                          float threshold_in, sdbg_hit* out, uint32_t* n_out, uint64_t* total_matches);
/* Streaming mode of the search scan (server/connector/duckdb_search_full_scan.cpp:2370-2403 RunStreamingScan, which
 * drains DocIterator::EmitScoredDocs, iterators.hpp:202-204): EVERY match of one query in docs [doc_min, doc_max) of
 * one segment with its BM25 score, ascending by doc id. Disjunctions of 1..4 terms, conjunctions of 1..16, hybrid
 * filter and deleted-doc mask honoured. *n_out = number of matches; SDBG_ECAPACITY when cap is too small (*n_out then
 * says how much room is needed; cap = 0 with NULL outputs is the count-only form). */
int sdbg_bm25_scan(sdbg_segment*, int kind, const sdbg_bm25_term* terms, size_t n_terms, float k1, float b,
                   const sdbg_col_pred* filt, uint32_t doc_min, uint32_t doc_max, uint32_t* out_docs, float* out_scores,
                   uint64_t cap, uint64_t* n_out);
/* Excluded terms (`a & b & !c`, `(a | b) & !c`: the exclusion iterator the reference builds for an And with Not children,
 * irs/search/exclusion.hpp). A query is its positive part (the OR / AND of terms above) minus every doc that occurs in
 * any list of its excluded terms; the deleted-docs mask and the hybrid filter apply as before. Scores come from the
 * positive terms only, bit for bit as without exclusions: excluded terms carry only their term id. An excluded id the
 * segment does not hold (>= its term count, or no postings) excludes nothing there; an excluded term that is also a
 * positive one empties an AND and leaves an OR the docs of its other terms. A query with no positive term is not
 * supported. total_matches follows sdbg_bm25_topk: exact with pruning off, a lower bound with it.
 * sdbg_bm25_topk_batch_excl: terms / term_off as sdbg_bm25_topk_batch; query q excludes
 * excl_terms[excl_off[q] .. excl_off[q+1]) (0..16 term ids; excl_off has n_queries + 1 entries). k1 = -1 selects TFIDF as
 * there. An empty set everywhere gives exactly sdbg_bm25_topk_batch's result. More than 16 excluded terms in a query:
 * SDBG_EUNSUPPORTED; a decreasing excl_off, or NULL excl_terms with a non-empty range: SDBG_EINVAL.
 * sdbg_bm25_scan_excl: sdbg_bm25_scan minus the docs of excl_terms[0 .. n_excl).
 * The top-k of queries with exclusions across GPUs: sdbg_dist_bm25_topk_batch_groups_min (a flat query is a degenerate
 * groups query); sdbg_bm25_topk_batch_device and sdbg_dist_bm25_topk_batch take flat queries without exclusions only. */
int sdbg_bm25_topk_batch_excl(sdbg_segment* const* segs, size_t n_segs, int kind, const sdbg_bm25_term* terms,
                              const uint32_t* term_off, size_t n_queries, const uint32_t* excl_terms, const uint32_t* excl_off,
                              float k1, float b, const sdbg_col_pred* filt, uint32_t k, float threshold_in,
                              sdbg_hit* out, uint32_t* n_out, uint64_t* total_matches);
int sdbg_bm25_scan_excl(sdbg_segment*, int kind, const sdbg_bm25_term* terms, size_t n_terms,
                        const uint32_t* excl_terms, size_t n_excl, float k1, float b, const sdbg_col_pred* filt,
                        uint32_t doc_min, uint32_t doc_max, uint32_t* out_docs, float* out_scores, uint64_t cap, uint64_t* n_out);
/* Count mode of the search scan (SELECT count(*) ... WHERE body @@ '...' [AND <pushed column filter>]): counts[q] = number
 * of docs, summed over the segments, that match query q's positive part (OR / AND of terms[term_off[q] .. term_off[q+1]),
 * 1..16 term ids), are not deleted, pass the hybrid filter (NULL never passes, as in the top-k), and occur in none of
 * excl_terms[excl_off[q] .. excl_off[q+1]) (0..16 ids; excl_off NULL = no exclusions). Nothing is scored: no scorer
 * parameters. Exact at every pruning level: equal to total_matches of sdbg_bm25_topk_batch(_excl) at pruning level 0, for
 * any scorer (an excluded id a segment does not hold excludes nothing there). Errors and their codes are those of
 * sdbg_bm25_topk_batch_excl; NULL counts: SDBG_EINVAL. Synchronous on the context's stream: counts is in host memory on
 * return. A single-term query over a segment without filter, deleted docs or an excluded list holding blocks there is
 * answered from the term's docs_count, without a launch. */
int sdbg_match_count_batch(sdbg_segment* const* segs, size_t n_segs, int kind, const uint32_t* terms,
                           const uint32_t* term_off, size_t n_queries, const uint32_t* excl_terms,
                           const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t* counts);
/* Sorted scan (SELECT ... WHERE body @@ '...' [AND <pushed filter>] ORDER BY col [DESC] [NULLS FIRST|LAST] LIMIT k): per
 * query, the k first of the docs sdbg_match_count_batch counts for it, ordered by column `sort_field` (staged in every
 * segment with one type: int64 raw or bit-packed, int32 or float64; NOT NULL or nullable; row = doc - 1, and a doc past
 * the column's rows is NULL). Values ascend (descending = 0) or descend; NULLs all come first (nulls_first = 1) or last;
 * ties, NULLs included, go by (segment index asc, doc asc). float64: -0.0 equals +0.0, every NaN equals every NaN and
 * sorts above +inf. out[q * k .. q * k + n_out[q]) holds n_out[q] = min(k, matches) hits in that order: the stored value
 * bit for bit (int32 sign-extended, float64 as its bits; 0 for NULL), doc, segment index and a NULL flag. Identical at
 * every pruning level; levels 1 and 2 skip matches, and (NOT NULL sort columns) whole 65 536-doc windows, that the
 * zonemap shows cannot beat the k-th value found so far (sdbg_scan_stats: windows judged / skipped).
 * Errors: those of sdbg_match_count_batch; k == 0, NULL out or n_out, or a sort column whose type differs between
 * segments: SDBG_EINVAL; a segment without the sort column: SDBG_ENOTFOUND; k > 4096: SDBG_EUNSUPPORTED (each CTA keeps
 * 2 * next_pow2(k) 16-byte candidate keys in shared memory). Synchronous on the context's stream.
 * Device scratch: k keys of 16 B per work item before the per-query merge, where a work item is a range of 65 536-doc
 * windows of one query in one segment (at least one per query and segment holding a match, at most 2 x SMs), plus
 * n_queries * k * 24 B of hits: 4096 queries x 1 segment x 1 item at k = 1000 take 66 MB; k = 4096 over 20 segments
 * with one item each takes 5.4 GB. The hits come back through as much pinned host memory. A mixed-shape batch of the
 * groups entry below holds its per-shape rows in HBM (the same bytes again) before they go to query order. Split larger
 * batches. */
typedef struct { int64_t value; uint32_t doc; uint32_t seg; uint8_t is_null; } sdbg_sort_hit;
int sdbg_match_topk_by_column_batch(sdbg_segment* const* segs, size_t n_segs, int kind, const uint32_t* terms,
                                    const uint32_t* term_off, size_t n_queries, const uint32_t* excl_terms,
                                    const uint32_t* excl_off /* NULL: none */, const sdbg_col_pred* filt,
                                    uint64_t sort_field, int descending, int nulls_first, uint32_t k,
                                    sdbg_sort_hit* out /* n_queries * k */, uint32_t* n_out);
/* Facet counts (SELECT col, count(*) ... WHERE body @@ '...' [AND <pushed filter>] GROUP BY col): per query, how the docs
 * sdbg_match_count_batch counts for it split over the values of column `key_field` (staged in every segment with one
 * type: int64 raw or bit-packed, or int32; NOT NULL or nullable; may be the filter's column; row = doc - 1, and a doc past
 * the column's rows has a NULL key). counts[q * key_span + (v - key_min)] = query q's matches whose key is v, summed over
 * the segments; null_counts[q] = its matches whose key is NULL (one group, as in SQL). So sum(counts[q, :]) +
 * null_counts[q] equals sdbg_match_count_batch's count. Identical at every pruning level: nothing is pruned.
 * The caller gives the key range, so the dense layout can be all-reduced across GPUs as it is and a fixed domain (enum ids)
 * needs no statistics pass; sdbg_column_minmax_i64 gives a column's range (NULLs skipped).
 * Errors, all found before anything is queued: those of sdbg_match_count_batch; NULL counts or null_counts, key_span == 0,
 * key_min + key_span - 1 past INT64_MAX, or a key type that differs between segments: SDBG_EINVAL; a segment without the
 * key column: SDBG_ENOTFOUND; a float64 key column, or key_span > 32768 (each CTA keeps key_span u32 bins in shared
 * memory): SDBG_EUNSUPPORTED. Found after the scan: a counted doc whose key lies outside [key_min, key_min + key_span):
 * SDBG_EINVAL, and the outputs are unspecified. Synchronous on the context's stream.
 * Device scratch: n_queries * key_span * 8 B + n_queries * 8 B (4096 queries x 2001 keys: 66 MB), and as much pinned
 * host memory for the copy back; a mixed-shape batch of the groups entry below holds its per-shape rows in HBM (the same
 * bytes again) before they go to query order. Split larger batches. */
int sdbg_match_facet_counts_batch(sdbg_segment* const* segs, size_t n_segs, int kind, const uint32_t* terms,
                                  const uint32_t* term_off, size_t n_queries, const uint32_t* excl_terms,
                                  const uint32_t* excl_off /* NULL: none */, const sdbg_col_pred* filt,
                                  uint64_t key_field, int64_t key_min, uint32_t key_span,
                                  uint64_t* counts /* n_queries * key_span */, uint64_t* null_counts /* n_queries */);
/* Conjunctions of OR groups (`a & (b | c) & !d`: an And whose children are terms, Ors of terms and Nots of terms, as
 * synonym expansion and query rewriting produce). Query q is the AND of the groups [query_group_off[q],
 * query_group_off[q+1]) (1..16), group g the OR of terms[group_off[g] .. group_off[g+1]) (non-empty); its positive terms
 * number 1..16 in all and are distinct. It excludes excl_terms[excl_off[q] .. excl_off[q+1]) as sdbg_bm25_topk_batch_excl
 * does (excl_off NULL: none). A doc matches when every group has a term whose list holds it, no excluded list holds it,
 * it is not deleted and it passes the hybrid filter (NULL never passes). A group whose lists are all empty in a segment
 * matches nothing there.
 * Scores: a hit's score is bit for bit the score the flat OR of the query's positive terms gives that doc (same scorer and
 * statistics): the sum of its matching terms' scores in ascending docs_count order. BM25, BM15 (b = 0), BM1 (k1 = 0) and
 * TFIDF (k1 = -1) as in the other batch entries; block-max pruning only for BM25 with the index-time b. total_matches is
 * exact with pruning off and a lower bound with it; counts are exact at every pruning level and equal the level-0 totals.
 * Degenerate queries take the existing paths and give exactly their results: a query of one group runs as
 * sdbg_bm25_topk_batch_excl / sdbg_match_count_batch with kind OR, a query whose groups are all single terms as kind AND.
 * Errors, all found before anything is queued (whatever the shapes of a batch's queries): an empty group, a decreasing
 * offset array, a positive term id twice in a query, or NULL arrays with non-empty ranges: SDBG_EINVAL; more than 16
 * groups, positive terms or excluded terms in a query: SDBG_EUNSUPPORTED; otherwise the errors of
 * sdbg_bm25_topk_batch_excl / sdbg_match_count_batch.
 * The sorted scan and facet counts of group queries: sdbg_match_topk_by_column_batch_groups_min /
 * sdbg_match_facet_counts_batch_groups_min below.
 * Memory: as sdbg_bm25_topk_batch; a batch whose queries take several of the shapes above also holds its per-shape rows
 * in HBM (n_queries * (8k + 12) B) before they go to query order on the device.
 * The top-k of group queries across GPUs: sdbg_dist_bm25_topk_batch_groups_min below.
 * The streaming scan of group queries, batched over segments: sdbg_match_scan_batch_groups_min below.
 * Not supported yet: deeper nesting (an OR of ANDs), more than 16 positive terms. Phrases: sdbg_phrase_*_batch below. */
int sdbg_bm25_topk_batch_groups(sdbg_segment* const* segs, size_t n_segs, const sdbg_bm25_term* terms,
                                const uint32_t* group_off, const uint32_t* query_group_off, size_t n_queries,
                                const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                float k1, float b, const sdbg_col_pred* filt, uint32_t k, float threshold_in,
                                sdbg_hit* out, uint32_t* n_out, uint64_t* total_matches);
int sdbg_match_count_batch_groups(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                  const uint32_t* group_off, const uint32_t* query_group_off, size_t n_queries,
                                  const uint32_t* excl_terms, const uint32_t* excl_off, const sdbg_col_pred* filt,
                                  uint64_t* counts);
/* OR groups with a minimum match count (`2 of (a | b | c) & d`: an Or with min_match_count, as minimum_should_match and
 * relaxed natural-language queries produce). The groups entries' parameters plus group_min: group g (indexed like
 * group_off) needs group_min[g] of its s_g terms, 1 <= group_min[g] <= s_g; a doc satisfies the group when at least
 * group_min[g] of its posting lists hold it. group_min NULL: every group needs 1, exactly sdbg_*_batch_groups.
 * A term a segment does not hold is an empty list there and still counts in s_g, so a group with fewer than group_min[g]
 * non-empty lists in a segment matches nothing there. Scores, totals and counts as for the groups entries.
 * Normalisation: a group with group_min[g] == s_g is its terms as single-term groups; a query whose groups then all need
 * 1 term is an ordinary groups query and gives exactly its results.
 * Errors: group_min[g] == 0 or > s_g: SDBG_EINVAL; otherwise those of the groups entries. */
int sdbg_bm25_topk_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const sdbg_bm25_term* terms,
                                    const uint32_t* group_off, const uint32_t* query_group_off,
                                    const uint32_t* group_min /* NULL: all 1 */, size_t n_queries,
                                    const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                    float k1, float b, const sdbg_col_pred* filt, uint32_t k, float threshold_in,
                                    sdbg_hit* out, uint32_t* n_out, uint64_t* total_matches);
int sdbg_match_count_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                      const uint32_t* group_off, const uint32_t* query_group_off,
                                      const uint32_t* group_min /* NULL: all 1 */, size_t n_queries,
                                      const uint32_t* excl_terms, const uint32_t* excl_off, const sdbg_col_pred* filt,
                                      uint64_t* counts);
/* Sorted scan and facet counts of group queries (`WHERE body @@ 'a & (b | c)' ORDER BY col LIMIT k`, `... GROUP BY col`):
 * the query parameters of sdbg_match_count_batch_groups_min, then the output parameters of
 * sdbg_match_topk_by_column_batch / sdbg_match_facet_counts_batch. Per query, the docs sdbg_match_count_batch_groups_min
 * counts, sorted or counted per key under exactly the rules of those entries (column types, NULLs, ties, n_out =
 * min(k, matches), the dense counts layout, sum(counts[q, :]) + null_counts[q] == the count); identical at every pruning
 * level. Degenerate queries normalise as in the groups entries and give exactly the flat entries' results. After a sorted
 * call, sdbg_scan_stats reports the windows of the whole call. Errors: those of sdbg_match_count_batch_groups_min and of
 * the flat entry, all found before anything is queued, except the facet pass's out-of-range key, found after the scan. */
int sdbg_match_topk_by_column_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                               const uint32_t* group_off, const uint32_t* query_group_off,
                                               const uint32_t* group_min /* NULL: all 1 */, size_t n_queries,
                                               const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                               const sdbg_col_pred* filt, uint64_t sort_field, int descending, int nulls_first,
                                               uint32_t k, sdbg_sort_hit* out /* n_queries * k */, uint32_t* n_out);
int sdbg_match_facet_counts_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                             const uint32_t* group_off, const uint32_t* query_group_off,
                                             const uint32_t* group_min /* NULL: all 1 */, size_t n_queries,
                                             const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                             const sdbg_col_pred* filt, uint64_t key_field, int64_t key_min, uint32_t key_span,
                                             uint64_t* counts /* n_queries * key_span */, uint64_t* null_counts /* n_queries */);
/* Aggregates over the matches (SELECT col, count(*), count(v), sum(v), avg(v), min(v), max(v) ... WHERE body @@ '...'
 * [AND <pushed filter>] GROUP BY col, or the same without GROUP BY): per query and group, COUNT(*), COUNT(value), SUM, MIN
 * and MAX of column `value_field` over the docs sdbg_match_count_batch (sdbg_match_count_batch_groups_min) counts for it.
 * Deleted docs, the pushed filter, exclusions, groups and min-match apply exactly as there; identical at every pruning level.
 * Grouping: by `key_field` exactly as the facet entries group (int64 raw or bit-packed, or int32; the key_min / key_span
 * layout): out[q * key_span + (v - key_min)] is query q's group of key v, null_out[q] the group of the NULL key (docs past
 * the key column's rows included). key_field == UINT64_MAX: no GROUP BY, one group out[q]; key_min must be 0 and key_span
 * 1, and null_out[q] comes back zeroed.
 * The value column: int64 (raw or bit-packed), int32 or float64, NOT NULL or nullable, with one type in every segment; it
 * may be the key column or the filter's column. A doc past its rows has a NULL value.
 * count equals the facet entry's counts[q * key_span + b] (null_out[q].count its null_counts[q]) exactly; count_value
 * counts the non-NULL values. When count_value == 0, sum_i128, sum_f64, min and max are 0 and the caller emits SQL NULL
 * for them; AVG is the caller's SUM / count_value, as with sdbg_group_row.
 * Integer columns: sum_i128 is the exact two's-complement 128-bit sum ({low, high} words as in sdbg_group_row) for any
 * values and any number of matches; min / max the int64 (int32 sign-extended). sum_f64 is 0.
 * float64 columns: sum_f64 follows IEEE rules (NaN if any value is NaN or both infinities occur, else the infinity that
 * occurs); the order of the finite additions is unspecified. min / max are the float64 bits of the extremes under the
 * sorted scan's order: -0.0 equals +0.0, every NaN equals every NaN and sorts above +inf; a zero extreme comes back as
 * +0.0 and a NaN one as 0x7FF8000000000000. sum_i128 is 0.
 * Errors, all found before anything is queued: those of the facet entries for the key column and range; NULL out or
 * null_out, a value column whose type differs between segments, or key_field == UINT64_MAX with (key_min, key_span) !=
 * (0, 1): SDBG_EINVAL; a segment without the value column: SDBG_ENOTFOUND; key_span > 4096 (each CTA keeps key_span + 1
 * cells of 40 B in shared memory): SDBG_EUNSUPPORTED. Found after the scan: a matching doc whose key lies outside
 * [key_min, key_min + key_span): SDBG_EINVAL, and the outputs are unspecified. Synchronous on the context's stream.
 * Device scratch: (n_queries * (key_span + 1)) * 48 B + n_queries * 8 B (4096 queries x 2001 keys: 394 MB), and as
 * much pinned host memory for the copy back; a mixed-shape batch of the groups entry holds its per-shape rows in HBM (the
 * same bytes again) before they go to query order. Split larger batches.
 * Not supported: several value columns in one call (call once per column), key spans above 4096, float64 keys, HAVING,
 * COUNT(DISTINCT), the top-k and streaming entries. The multi-GPU merge: sdbg_dist_match_aggregate_batch_groups_min. */
typedef struct {
  uint64_t count;         /* COUNT(*) of the group's matches */
  uint64_t count_value;   /* COUNT(value): those whose value is not NULL */
  int64_t sum_i128[2];    /* integer value column: SUM(value), exact; {low, high} words as in sdbg_group_row */
  double sum_f64;         /* float64 value column: SUM(value) */
  int64_t min, max;       /* MIN / MAX(value): the integer (int32 sign-extended), or the float64's bits */
} sdbg_match_agg;
int sdbg_match_aggregate_batch(sdbg_segment* const* segs, size_t n_segs, int kind, const uint32_t* terms,
                               const uint32_t* term_off, size_t n_queries, const uint32_t* excl_terms,
                               const uint32_t* excl_off /* NULL: none */, const sdbg_col_pred* filt, uint64_t key_field,
                               int64_t key_min, uint32_t key_span, uint64_t value_field,
                               sdbg_match_agg* out /* n_queries * key_span */, sdbg_match_agg* null_out /* n_queries */);
int sdbg_match_aggregate_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                          const uint32_t* group_off, const uint32_t* query_group_off,
                                          const uint32_t* group_min /* NULL: all 1 */, size_t n_queries,
                                          const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                          const sdbg_col_pred* filt, uint64_t key_field, int64_t key_min, uint32_t key_span,
                                          uint64_t value_field, sdbg_match_agg* out /* n_queries * key_span */,
                                          sdbg_match_agg* null_out /* n_queries */);
/* Match scan (the Stream mode of the search scan: SELECT id [, bm25(...)] ... WHERE body @@ '...' [LIMIT n OFFSET o]
 * without ORDER BY): per query, its matches themselves, a page at a time. The query parameters are those of
 * sdbg_match_count_batch_groups_min (a flat OR is one group, a flat AND single-term groups); terms are sdbg_bm25_term.
 * Which docs: exactly the docs sdbg_match_count_batch_groups_min counts for the query, with the same normalisation and
 * degenerate shapes. Order: by (segment index in segs ascending, doc ascending).
 * Output: total[q] is the exact number of matches (that count). out[q * limit ..] holds the matches at ordinals
 * offset[q] .. offset[q] + limit - 1 of that order (offset NULL: all 0), n_out[q] = min(limit, total[q] - offset[q]),
 * and 0 when the offset is at or past the end. A hit is {score, doc, seg}: seg indexes segs, doc is segment-local.
 * Identical at every pruning level: nothing is pruned.
 * Scores: with scored != 0, a hit's score is bit for bit the score sdbg_bm25_topk_batch_groups_min gives that doc at
 * pruning level 0: the sum of the query's positive terms whose lists hold the doc, in ascending docs_count order in the
 * doc's segment (stable), from 0. k1 and b select BM25, BM15 (b = 0), BM1 (k1 = 0) or TFIDF (k1 = -1; b != 0:
 * normalised) as in the other batch entries; excluded terms never score. With scored == 0 no frequency, norm or scorer
 * parameter is read (k1, b and the terms' statistics are ignored) and every score is 0.
 * Errors, all found before anything is queued: those of sdbg_match_count_batch_groups_min; limit == 0, or NULL out, n_out
 * or total: SDBG_EINVAL; when scored, those of the top-k entries' limits (more than 65535 queries, or more than
 * 2^32 - 2 docs over the segments: SDBG_EUNSUPPORTED). Synchronous on the context's stream, with one wait per call.
 * Device scratch: n_queries * (limit * 12 + 12) B for the pages, totals and counts (4096 queries at limit 1000: 49 MB),
 * 12 B per work item (windows of one query in one segment, at most 2 x SMs per query and segment), and as much pinned
 * host memory as the pages for the copy back; a batch whose queries take several shapes also holds its per-shape rows in
 * HBM (the same bytes again) before they go to query order. Split larger batches.
 * sdbg_bm25_scan / sdbg_bm25_scan_excl stay the per-segment doc-window form with their own limits. */
int sdbg_match_scan_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const sdbg_bm25_term* terms,
                                     const uint32_t* group_off, const uint32_t* query_group_off,
                                     const uint32_t* group_min /* NULL: all 1 */, size_t n_queries,
                                     const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                     float k1, float b, const sdbg_col_pred* filt,
                                     const uint64_t* offset /* n_queries; NULL: all 0 */, uint32_t limit, int scored,
                                     sdbg_hit* out /* n_queries * limit */, uint32_t* n_out, uint64_t* total);
/* Exact phrase queries (`body @@ '"new york"'`: by_phrase / FixedPhraseQuery of plain terms, slop 0). Query q is the phrase
 * of slots phrase_off[q] .. phrase_off[q+1]) (1..16): slot i is term terms[i] at relative position rel_pos[i], rel_pos
 * starting at 0 in each phrase and strictly increasing (rel_pos NULL: 0, 1, 2, ..., adjacent words; gaps express removed
 * stop words). A term may repeat (`"to be or not to be"`); at most 16 distinct terms. Doc d matches when some anchor p has
 * p + rel_pos[i] among term terms[i]'s positions in d for every slot i, d is not deleted, passes the filter chain and is
 * in none of the lists of excl_terms[excl_off[q] .. excl_off[q+1]) (0..16 ids; excl_off NULL: none). The phrase frequency
 * is the number of such anchors, overlaps included (`"a a"` in `a a a`: 2). A term a segment holds no postings for makes
 * the phrase match nothing there. Every segment needs staged positions (sdbg_stage_positions).
 * sdbg_phrase_count_batch: counts[q] = the number of matching docs over the segments.
 * sdbg_phrase_topk_batch: the k best matches by score, scored bm25(phrase frequency, norm(d)) with phrase_stats[q] (one
 * per query, .term ignored; engine.py sums the terms' idfs), under BM25, BM15 (b = 0), BM1 (k1 = 0) or TFIDF (k1 = -1)
 * as in the other batch entries; out / n_out / total_matches / threshold_in as sdbg_bm25_topk_batch (score desc, segment
 * asc, doc asc; scores > threshold_in). Nothing is pruned: identical at every pruning level, total_matches exact and equal
 * to the count. A one-slot phrase gives exactly its term's flat result.
 * Errors, all found before anything is queued: an empty phrase, rel_pos not starting at 0 or not increasing, a
 * decreasing offset array, or NULL arrays with non-empty ranges: SDBG_EINVAL; more than 16 slots or 16 excluded ids:
 * SDBG_EUNSUPPORTED; a segment without positions: SDBG_ENOTFOUND; otherwise the errors and limits of
 * sdbg_match_count_batch (kind AND) and, for the top-k, of sdbg_bm25_topk_batch, with k capped at 4096 (each work item
 * keeps 2 * next_pow2(k) 16-byte candidate keys in shared memory): SDBG_EUNSUPPORTED above. Synchronous.
 * Device scratch: as sdbg_match_count_batch; the top-k adds k keys of 8 B per work item (a range of 65 536-doc windows of
 * one query in one segment, at most 2 x SMs per query and segment) and n_queries * (8k + 12) B for the results, with as
 * much pinned host memory for the copy back. */
int sdbg_phrase_count_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                            const uint32_t* rel_pos /* NULL: adjacent */, const uint32_t* phrase_off, size_t n_queries,
                            const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */, const sdbg_col_pred* filt,
                            uint64_t* counts);
int sdbg_phrase_topk_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                           const uint32_t* rel_pos /* NULL: adjacent */, const uint32_t* phrase_off, size_t n_queries,
                           const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                           const sdbg_bm25_term* phrase_stats /* n_queries */, float k1, float b, const sdbg_col_pred* filt,
                           uint32_t k, float threshold_in, sdbg_hit* out /* n_queries * k */, uint32_t* n_out,
                           uint64_t* total_matches);
/* Sorted scan, facet counts, aggregates and match scan of phrases (`WHERE body @@ '"new york"' ORDER BY col LIMIT k`,
 * `... GROUP BY col`, `SELECT id [, bm25(...)] ... LIMIT n OFFSET o`): the phrase parameters of sdbg_phrase_count_batch
 * (terms, rel_pos, phrase_off, n_queries, excl_terms, excl_off, filt), then the pass parameters and outputs of the flat
 * entry each mirrors: sdbg_match_topk_by_column_batch (k 1..4096), sdbg_match_facet_counts_batch,
 * sdbg_match_aggregate_batch and sdbg_match_scan_batch_groups_min. Which docs: exactly the docs sdbg_phrase_count_batch
 * counts for the query. Order, ties, NULL rules, key ranges, the dense layouts, the out-of-range report, pages and totals
 * are those of the mirrored entry; identical at every pruning level (the sorted scan prunes as its flat entry does).
 * sum(counts[q, :]) + null_counts[q], COUNT(*) over the groups and total[q] equal the phrase count. A one-slot phrase
 * gives exactly the flat AND entry's result for its term.
 * sdbg_phrase_scan_batch scores with phrase_stats, k1, b as sdbg_phrase_topk_batch does: with scored != 0 a hit's score is
 * bit for bit the score sdbg_phrase_topk_batch gives that doc; with scored == 0 every score is 0 and phrase_stats may be
 * NULL.
 * Errors, all found before anything is queued except the facet and aggregate passes' out-of-range key: those of
 * sdbg_phrase_count_batch (SDBG_ENOTFOUND for a segment without positions) and those of the mirrored entry; a scored scan
 * with NULL phrase_stats: SDBG_EINVAL. Synchronous on the context's stream.
 * Device scratch: the mirrored entry's, plus the slots' lists, 16 B per slot and segment; a scored scan stages the same
 * again with one PostingsDev and one 80-byte sink per segment and 16 B per query. The phrase check runs per doc that
 * survives the conjunction, the exclusions, the deleted docs and the filter chain (the sorted scan: once its key has
 * passed the threshold), and a page deep into the result repeats it in the scan's second pass. */
int sdbg_phrase_topk_by_column_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                     const uint32_t* rel_pos /* NULL: adjacent */, const uint32_t* phrase_off, size_t n_queries,
                                     const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                     const sdbg_col_pred* filt, uint64_t sort_field, int descending, int nulls_first,
                                     uint32_t k, sdbg_sort_hit* out /* n_queries * k */, uint32_t* n_out);
int sdbg_phrase_facet_counts_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                   const uint32_t* rel_pos /* NULL: adjacent */, const uint32_t* phrase_off, size_t n_queries,
                                   const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                   const sdbg_col_pred* filt, uint64_t key_field, int64_t key_min, uint32_t key_span,
                                   uint64_t* counts /* n_queries * key_span */, uint64_t* null_counts /* n_queries */);
int sdbg_phrase_aggregate_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                const uint32_t* rel_pos /* NULL: adjacent */, const uint32_t* phrase_off, size_t n_queries,
                                const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                const sdbg_col_pred* filt, uint64_t key_field, int64_t key_min, uint32_t key_span,
                                uint64_t value_field, sdbg_match_agg* out /* n_queries * key_span */,
                                sdbg_match_agg* null_out /* n_queries */);
int sdbg_phrase_scan_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                           const uint32_t* rel_pos /* NULL: adjacent */, const uint32_t* phrase_off, size_t n_queries,
                           const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */, const sdbg_col_pred* filt,
                           const sdbg_bm25_term* phrase_stats /* n_queries; NULL when scored == 0 */, float k1, float b,
                           const uint64_t* offset /* n_queries; NULL: all 0 */, uint32_t limit, int scored,
                           sdbg_hit* out /* n_queries * limit */, uint32_t* n_out, uint64_t* total);
/* Conjunctions of phrases, terms and negated phrases (`"new york" & pizza & !"deep dish"`). Query q is an AND of the
 * clauses query_clause_off[q] .. query_clause_off[q+1]) (at least one), plus excl_terms / excl_off and the filter chain
 * as above. Clause j is a phrase exactly as above, of slots clause_off[j] .. clause_off[j+1]) (at least one; rel_pos
 * starting at 0 in each clause and strictly increasing; rel_pos NULL: adjacent within each clause); a one-slot clause is a
 * plain term. Clause j is negated when clause_negated[j] != 0 (clause_negated NULL: none); a query needs a positive
 * clause. At most 16 slots per query, positive and negated clauses together. Doc d matches when every positive clause
 * has phrase frequency > 0 in d, every negated clause phrase frequency 0, d is not deleted, passes the filter chain and
 * holds none of the excluded terms. A term of a positive clause that a segment holds no postings for makes the query match
 * nothing there; a term of a negated clause that a segment does not hold makes that clause exclude nothing there (a
 * one-slot negated clause behaves exactly as that term among excl_terms).
 * Score (the top-k, and the scan with scored != 0): the fp32 sum, from 0, of bm25(phrase frequency, norm(d)) over the
 * positive clauses, each with its own statistics clause_stats[j] (one per clause, .term ignored, negated clauses' entries
 * ignored; engine.py sums each clause's idfs in slot order), in ascending cost order within d's segment: a clause costs the
 * smallest docs_count of its terms in that segment, ties in the query's clause order. For queries of one-slot clauses of
 * distinct terms that is the order of sdbg_bm25_topk_batch's conjunctions, whose results these entries then reproduce
 * bit for bit at pruning level 0; a query of one positive clause gives exactly the sdbg_phrase_* result for that phrase
 * (which is how those entries run). Nothing is pruned: identical at every pruning level, k <= 4096.
 * Each entry takes the parameters of its sdbg_phrase_* counterpart, with (terms, rel_pos, phrase_off) replaced by
 * (terms, rel_pos, clause_off, clause_negated, query_clause_off) and phrase_stats by clause_stats; outputs, orders, NULL
 * rules and scratch are the counterpart's (the clause tables add 16 B per clause and segment, and 16 B of statistics per
 * clause when scored). Errors, all found before anything is queued: an empty clause, a query without a clause or without
 * a positive clause, bad rel_pos, decreasing offsets, NULL arrays with non-empty ranges, NULL clause_stats where a score
 * is needed: SDBG_EINVAL; more than 16 slots in a query, more than 16 excluded ids, k > 4096: SDBG_EUNSUPPORTED; a
 * segment without staged positions: SDBG_ENOTFOUND; otherwise the counterpart's. Synchronous. */
int sdbg_phrase_and_count_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                const uint32_t* rel_pos /* NULL: adjacent within each clause */, const uint32_t* clause_off,
                                const uint8_t* clause_negated /* NULL: none */, const uint32_t* query_clause_off,
                                size_t n_queries, const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                const sdbg_col_pred* filt, uint64_t* counts);
int sdbg_phrase_and_topk_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                               const uint32_t* rel_pos /* NULL: adjacent within each clause */, const uint32_t* clause_off,
                               const uint8_t* clause_negated /* NULL: none */, const uint32_t* query_clause_off,
                               size_t n_queries, const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                               const sdbg_bm25_term* clause_stats /* one per clause */, float k1, float b,
                               const sdbg_col_pred* filt, uint32_t k, float threshold_in, sdbg_hit* out /* n_queries * k */,
                               uint32_t* n_out, uint64_t* total_matches);
int sdbg_phrase_and_topk_by_column_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                         const uint32_t* rel_pos /* NULL: adjacent within each clause */,
                                         const uint32_t* clause_off, const uint8_t* clause_negated /* NULL: none */,
                                         const uint32_t* query_clause_off, size_t n_queries, const uint32_t* excl_terms,
                                         const uint32_t* excl_off /* NULL: none */, const sdbg_col_pred* filt,
                                         uint64_t sort_field, int descending, int nulls_first, uint32_t k,
                                         sdbg_sort_hit* out /* n_queries * k */, uint32_t* n_out);
int sdbg_phrase_and_facet_counts_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                       const uint32_t* rel_pos /* NULL: adjacent within each clause */,
                                       const uint32_t* clause_off, const uint8_t* clause_negated /* NULL: none */,
                                       const uint32_t* query_clause_off, size_t n_queries, const uint32_t* excl_terms,
                                       const uint32_t* excl_off /* NULL: none */, const sdbg_col_pred* filt, uint64_t key_field,
                                       int64_t key_min, uint32_t key_span, uint64_t* counts /* n_queries * key_span */,
                                       uint64_t* null_counts /* n_queries */);
int sdbg_phrase_and_aggregate_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                    const uint32_t* rel_pos /* NULL: adjacent within each clause */,
                                    const uint32_t* clause_off, const uint8_t* clause_negated /* NULL: none */,
                                    const uint32_t* query_clause_off, size_t n_queries, const uint32_t* excl_terms,
                                    const uint32_t* excl_off /* NULL: none */, const sdbg_col_pred* filt, uint64_t key_field,
                                    int64_t key_min, uint32_t key_span, uint64_t value_field,
                                    sdbg_match_agg* out /* n_queries * key_span */, sdbg_match_agg* null_out /* n_queries */);
int sdbg_phrase_and_scan_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                               const uint32_t* rel_pos /* NULL: adjacent within each clause */, const uint32_t* clause_off,
                               const uint8_t* clause_negated /* NULL: none */, const uint32_t* query_clause_off,
                               size_t n_queries, const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                               const sdbg_col_pred* filt, const sdbg_bm25_term* clause_stats /* NULL when scored == 0 */,
                               float k1, float b, const uint64_t* offset /* n_queries; NULL: all 0 */, uint32_t limit,
                               int scored, sdbg_hit* out /* n_queries * limit */, uint32_t* n_out, uint64_t* total);
/* Conjunctions of OR groups of phrases and terms (`("new york" | nyc) & pizza & !"deep dish"`; the shape synonym
 * expansion of multi-word synonyms produces). Query q is an AND of the groups query_group_off[q] .. query_group_off[q+1])
 * (1..16), plus excl_terms / excl_off and the filter chain as above. Group g is an OR of the alternatives group_off[g] ..
 * group_off[g+1]) (1..16); it is negated when group_negated[g] != 0 (group_negated NULL: none), and a query needs a
 * positive group. Alternative j is a phrase exactly as a clause of sdbg_phrase_and_*: slots clause_off[j] ..
 * clause_off[j+1]) at rel_pos starting at 0 and strictly increasing (rel_pos NULL: adjacent), gaps and repeated terms
 * allowed; a one-slot alternative is a plain term. At most 16 slots per query, every alternative of every group counted.
 * Doc d matches when every positive group has an alternative with phrase frequency > 0 in d, no alternative of a negated
 * group has (`!(A | B)` is `!A & !B`), d is not deleted, passes the filter chain and holds none of the excluded terms. An
 * alternative with a term a segment holds no postings for matches nothing there (a positive group all of whose
 * alternatives are so matches nothing, so neither does the query) and, negated, excludes nothing there.
 * Score (the top-k, and the scan with scored != 0): the fp32 sum, from 0, of bm25(phrase frequency, norm(d)) over the
 * positive alternatives with frequency > 0 in d, whatever their group, each with its own statistics clause_stats[j] (one
 * per alternative, .term ignored, negated groups' entries ignored), in ascending cost order within d's segment: an
 * alternative costs the smallest docs_count of its terms there, ties in the query's alternative order, flattened group by
 * group. Duplicate alternatives are each scored; negated groups never score. Every group of one alternative gives exactly
 * sdbg_phrase_and_* (which, with sdbg_phrase_*, runs as this case); one-slot alternatives of distinct terms give exactly
 * the *_groups_min entries with every minimum 1 (the top-k bit for bit at pruning level 0); one group of one-slot
 * alternatives gives exactly the flat OR entries. Nothing is pruned: identical at every pruning level, k <= 4096.
 * Each entry takes the parameters of its sdbg_phrase_and_* counterpart, with (clause_off, clause_negated,
 * query_clause_off) replaced by (clause_off, group_off, group_negated, query_group_off); outputs, orders, NULL rules and
 * scratch are the counterpart's. Errors, all found before anything is queued: an empty group or clause, a query without
 * a group or without a positive group, bad rel_pos, decreasing offsets, NULL arrays with non-empty ranges, NULL
 * clause_stats where a score is needed: SDBG_EINVAL; more than 16 slots, groups or excluded ids in a query, k > 4096:
 * SDBG_EUNSUPPORTED; a segment without staged positions: SDBG_ENOTFOUND; otherwise the counterpart's. Synchronous. */
int sdbg_phrase_groups_count_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                   const uint32_t* rel_pos /* NULL: adjacent within each alternative */,
                                   const uint32_t* clause_off, const uint32_t* group_off,
                                   const uint8_t* group_negated /* NULL: none */, const uint32_t* query_group_off,
                                   size_t n_queries, const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                   const sdbg_col_pred* filt, uint64_t* counts);
int sdbg_phrase_groups_topk_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                  const uint32_t* rel_pos /* NULL: adjacent within each alternative */,
                                  const uint32_t* clause_off, const uint32_t* group_off,
                                  const uint8_t* group_negated /* NULL: none */, const uint32_t* query_group_off,
                                  size_t n_queries, const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                  const sdbg_bm25_term* clause_stats /* one per alternative */, float k1, float b,
                                  const sdbg_col_pred* filt, uint32_t k, float threshold_in, sdbg_hit* out /* n_queries * k */,
                                  uint32_t* n_out, uint64_t* total_matches);
int sdbg_phrase_groups_topk_by_column_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                            const uint32_t* rel_pos /* NULL: adjacent within each alternative */,
                                            const uint32_t* clause_off, const uint32_t* group_off,
                                            const uint8_t* group_negated /* NULL: none */, const uint32_t* query_group_off,
                                            size_t n_queries, const uint32_t* excl_terms,
                                            const uint32_t* excl_off /* NULL: none */, const sdbg_col_pred* filt,
                                            uint64_t sort_field, int descending, int nulls_first, uint32_t k,
                                            sdbg_sort_hit* out /* n_queries * k */, uint32_t* n_out);
int sdbg_phrase_groups_facet_counts_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                          const uint32_t* rel_pos /* NULL: adjacent within each alternative */,
                                          const uint32_t* clause_off, const uint32_t* group_off,
                                          const uint8_t* group_negated /* NULL: none */, const uint32_t* query_group_off,
                                          size_t n_queries, const uint32_t* excl_terms,
                                          const uint32_t* excl_off /* NULL: none */, const sdbg_col_pred* filt,
                                          uint64_t key_field, int64_t key_min, uint32_t key_span,
                                          uint64_t* counts /* n_queries * key_span */, uint64_t* null_counts /* n_queries */);
int sdbg_phrase_groups_aggregate_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                       const uint32_t* rel_pos /* NULL: adjacent within each alternative */,
                                       const uint32_t* clause_off, const uint32_t* group_off,
                                       const uint8_t* group_negated /* NULL: none */, const uint32_t* query_group_off,
                                       size_t n_queries, const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                       const sdbg_col_pred* filt, uint64_t key_field, int64_t key_min, uint32_t key_span,
                                       uint64_t value_field, sdbg_match_agg* out /* n_queries * key_span */,
                                       sdbg_match_agg* null_out /* n_queries */);
int sdbg_phrase_groups_scan_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                  const uint32_t* rel_pos /* NULL: adjacent within each alternative */,
                                  const uint32_t* clause_off, const uint32_t* group_off,
                                  const uint8_t* group_negated /* NULL: none */, const uint32_t* query_group_off,
                                  size_t n_queries, const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                  const sdbg_col_pred* filt, const sdbg_bm25_term* clause_stats /* NULL when scored == 0 */,
                                  float k1, float b, const uint64_t* offset /* n_queries; NULL: all 0 */, uint32_t limit,
                                  int scored, sdbg_hit* out /* n_queries * limit */, uint32_t* n_out, uint64_t* total);
/* Minimum match counts over OR groups of phrases and terms (`2 of ("new york" | nyc | "big apple") & pizza`; the shape a
 * minimum_should_match query with a multi-word synonym produces). Everything is as in sdbg_phrase_groups_*, with positive
 * group g holding doc d when at least group_min[g] of its s_g alternatives have phrase frequency > 0 in d (group_min
 * NULL: every minimum 1). Every alternative counts on its own: duplicate alternatives each count, as they are each
 * scored. 1 <= group_min[g] <= s_g; a negated group keeps minimum 1 (`!(A | B)` is `!A & !B`). The score is unchanged:
 * the fp32 sum, from 0, of bm25(phrase frequency, norm) over every positive alternative with frequency > 0 in d, in
 * ascending alternative cost within d's segment, ties in flattened query order; a doc holding more than group_min[g]
 * alternatives of a group is scored on all of them (as the term *_groups_min entries score). A positive group with
 * group_min == s_g is s_g groups of one alternative, and at most 16 slots per query still bound the groups after that
 * split. Every minimum 1 (or NULL) gives exactly sdbg_phrase_groups_* (which run as this case); group_min == s_g gives
 * exactly sdbg_phrase_and_* with that group's alternatives as separate positive clauses; one-slot alternatives of
 * distinct terms give exactly the term *_batch_groups_min entries (the top-k bit for bit at pruning level 0). Nothing is
 * pruned: identical at every pruning level, total_matches exact, k <= 4096.
 * Each entry takes the parameters of its sdbg_phrase_groups_* counterpart plus group_min right after group_negated;
 * outputs, orders, NULL rules and scratch are the counterpart's. Errors, all found before anything is queued: a
 * group_min[g] of 0 or above its group's size: SDBG_EINVAL; a negated group with group_min[g] != 1: SDBG_EUNSUPPORTED;
 * otherwise the counterpart's. Synchronous. */
int sdbg_phrase_groups_count_batch_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                       const uint32_t* rel_pos /* NULL: adjacent within each alternative */,
                                       const uint32_t* clause_off, const uint32_t* group_off,
                                       const uint8_t* group_negated /* NULL: none */,
                                       const uint32_t* group_min /* NULL: all 1 */, const uint32_t* query_group_off,
                                       size_t n_queries, const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                       const sdbg_col_pred* filt, uint64_t* counts);
int sdbg_phrase_groups_topk_batch_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                      const uint32_t* rel_pos /* NULL: adjacent within each alternative */,
                                      const uint32_t* clause_off, const uint32_t* group_off,
                                      const uint8_t* group_negated /* NULL: none */,
                                      const uint32_t* group_min /* NULL: all 1 */, const uint32_t* query_group_off,
                                      size_t n_queries, const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                      const sdbg_bm25_term* clause_stats /* one per alternative */, float k1, float b,
                                      const sdbg_col_pred* filt, uint32_t k, float threshold_in,
                                      sdbg_hit* out /* n_queries * k */, uint32_t* n_out, uint64_t* total_matches);
int sdbg_phrase_groups_topk_by_column_batch_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                const uint32_t* rel_pos /* NULL: adjacent within each alternative */,
                                                const uint32_t* clause_off, const uint32_t* group_off,
                                                const uint8_t* group_negated /* NULL: none */,
                                                const uint32_t* group_min /* NULL: all 1 */, const uint32_t* query_group_off,
                                                size_t n_queries, const uint32_t* excl_terms,
                                                const uint32_t* excl_off /* NULL: none */, const sdbg_col_pred* filt,
                                                uint64_t sort_field, int descending, int nulls_first, uint32_t k,
                                                sdbg_sort_hit* out /* n_queries * k */, uint32_t* n_out);
int sdbg_phrase_groups_facet_counts_batch_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                              const uint32_t* rel_pos /* NULL: adjacent within each alternative */,
                                              const uint32_t* clause_off, const uint32_t* group_off,
                                              const uint8_t* group_negated /* NULL: none */,
                                              const uint32_t* group_min /* NULL: all 1 */, const uint32_t* query_group_off,
                                              size_t n_queries, const uint32_t* excl_terms,
                                              const uint32_t* excl_off /* NULL: none */, const sdbg_col_pred* filt,
                                              uint64_t key_field, int64_t key_min, uint32_t key_span,
                                              uint64_t* counts /* n_queries * key_span */, uint64_t* null_counts /* n_queries */);
int sdbg_phrase_groups_aggregate_batch_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                           const uint32_t* rel_pos /* NULL: adjacent within each alternative */,
                                           const uint32_t* clause_off, const uint32_t* group_off,
                                           const uint8_t* group_negated /* NULL: none */,
                                           const uint32_t* group_min /* NULL: all 1 */, const uint32_t* query_group_off,
                                           size_t n_queries, const uint32_t* excl_terms,
                                           const uint32_t* excl_off /* NULL: none */,
                                           const sdbg_col_pred* filt, uint64_t key_field, int64_t key_min, uint32_t key_span,
                                           uint64_t value_field, sdbg_match_agg* out /* n_queries * key_span */,
                                           sdbg_match_agg* null_out /* n_queries */);
int sdbg_phrase_groups_scan_batch_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                      const uint32_t* rel_pos /* NULL: adjacent within each alternative */,
                                      const uint32_t* clause_off, const uint32_t* group_off,
                                      const uint8_t* group_negated /* NULL: none */,
                                      const uint32_t* group_min /* NULL: all 1 */, const uint32_t* query_group_off,
                                      size_t n_queries, const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                      const sdbg_col_pred* filt, const sdbg_bm25_term* clause_stats /* NULL when scored == 0 */,
                                      float k1, float b, const uint64_t* offset /* n_queries; NULL: all 0 */, uint32_t limit,
                                      int scored, sdbg_hit* out /* n_queries * limit */, uint32_t* n_out, uint64_t* total);
/* Multi-GPU: leave each query's top-k on the device as sortable 64-bit keys + a base ordinal so a
 * collective can gather them; merge gathered keys from `n_ranks` ranks (see INTEGRATION.md). */
int sdbg_bm25_topk_batch_device(sdbg_segment* const* segs, size_t n_segs, int kind,
                                const sdbg_bm25_term* terms, const uint32_t* term_off, size_t n_queries,
                                float k1, float b, const sdbg_col_pred* filt, uint32_t k, float threshold_in,
                                uint32_t rank, void* d_keys /* n_queries*k u64 */,
                                void* d_totals /* n_queries u64 */);
/* sdbg_bm25_topk_batch_device: rank < 15 and fewer than 2^28 docs over the rank's segments (each rank owns 2^28
 * ordinals of the merged key space), else SDBG_EUNSUPPORTED before anything is queued. Each query's k slots hold its
 * keys sorted descending, then zeros.
 * sdbg_topk_merge_gathered: the k best keys per query over all ranks' lists (a list's keys are its non-zero prefix).
 * k <= 8192 and n_queries <= 65535 as for the top-k entries, else SDBG_EUNSUPPORTED; a zero count: SDBG_EINVAL.
 * out may be NULL: the merged keys then stay in HBM (device-resident pipelines / timing). */
int sdbg_topk_merge_gathered(sdbg_ctx*, const void* d_keys_all /* n_ranks*n_queries*k u64 */,
                             uint32_t n_ranks, size_t n_queries, uint32_t k, sdbg_hit* out, uint32_t* n_out);
/* Test probe: decode+score one whole posting list (exhaustive, no top-k). Buffers sized docs_count. */
int sdbg_decode_score_term(sdbg_segment*, uint32_t term, float c0, float norm_const, float norm_length,
                           uint32_t* docs, uint32_t* freqs, float* scores);

/* Encoded int64 columns: frame-of-reference bit-packing in groups of 2048 rows -- per group a base (the minimum) and a
 * bit width, values stored as (v - base) in `bits` bits, little-endian, groups 8-byte aligned; bits = 0 is a constant
 * group. This is the algorithm of DuckDB's `bitpacking` codec in FOR mode, which the reference's column blocks name in
 * ColumnBlockMeta::codec (irs/formats/column/column_reader.hpp:90-96); DuckDB is not vendored in the reference tree, so
 * the byte layout is this library's. sdbg_pack_for is the host-side writer (returns SDBG_ECAPACITY with *n_words = the
 * room needed); sdbg_stage_column_for copies the packed stream to the GPU, so only the packed bytes cross PCIe.
 * HBM keeps an owned NOT NULL SDBG_I64 column in this form whenever it is smaller than the raw values (sdbg_stage_column
 * and sdbg_synth_column pack on the device; sdbg_stage_column_for keeps the caller's stream when every group starts at an
 * even word offset, as sdbg_pack_for writes it, and decodes it otherwise). The GROUP BY scan reads the packed words;
 * other readers see the raw values, decoded once on first use. sdbg_column_for_to_host copies a packed column's headers
 * and words back (the same bytes sdbg_pack_for writes for the same values); *n_words = 0 when the column is held raw. */
typedef struct { int64_t base; uint32_t bits; uint32_t off8; } sdbg_for_block;
int sdbg_pack_for(const int64_t* values, uint64_t rows, sdbg_for_block* headers /* (rows + 2047) / 2048 */, uint64_t* words,
                  uint64_t cap_words, uint64_t* n_words);
int sdbg_stage_column_for(sdbg_segment*, uint64_t field, const sdbg_for_block* headers, const uint64_t* words, uint64_t n_words,
                          uint64_t rows);
int sdbg_column_for_to_host(sdbg_segment*, uint64_t field, sdbg_for_block* headers, uint64_t* words, uint64_t cap_words,
                            uint64_t* n_words);

/* Late materialisation (HitBatcher::MaterializeColumn, irs/index/hit_batcher.hpp:39; FinalizeBatch of the search scan):
 * out_values[i] = column[docs[i] - 1] for n hit docs of the segment (element width = the staged type's), out_valid[i]
 * (nullable) = 0 for NULL or out-of-range rows, whose value is written as 0. */
int sdbg_gather_column(sdbg_segment*, uint64_t field, const uint32_t* docs, size_t n, void* out_values, uint8_t* out_valid);

/* ---- columnar filter / aggregate (boundary B3, iresearch_scan) ---- */
int sdbg_filter_bitmap(sdbg_segment*, const sdbg_col_pred* preds, size_t n_preds, uint64_t* mask_out);
int sdbg_filter_count_sum(sdbg_segment* const* segs, size_t n_segs, const sdbg_col_pred* preds,
                          size_t n_preds, uint64_t sum_field, uint64_t* count, int64_t sum_i128[2],
                          double* sum_f64);
typedef struct { int64_t key; uint64_t count; int64_t sum_i128[2]; double sum_f64; uint64_t cnt_f64; } sdbg_group_row;
/* SELECT key, COUNT(*), SUM(sum_int_field), SUM(avg_f64_field)/cnt_f64 ... GROUP BY key.
 * Rows come back sorted by key. Pass UINT64_MAX for an aggregate field that is not wanted. */
int sdbg_filter_groupby(sdbg_segment* const* segs, size_t n_segs, const sdbg_col_pred* preds,
                        size_t n_preds, uint64_t key_field, uint32_t n_groups_hint,
                        uint64_t sum_int_field, uint64_t avg_f64_field, sdbg_group_row* out, uint64_t cap,
                        uint64_t* n_out);
/* Multi-GPU split of the same: partial dense aggregates stay on the device in two flat buffers that
 * a SUM all-reduce can merge (int64 limbs + counts, and float64 sums), then finalize on any rank.
 * d_i64: 4*span int64 = [count | sum_lo | sum_hi | cnt_f64]; d_f64: span float64. */
int sdbg_filter_groupby_partial(sdbg_segment* const* segs, size_t n_segs, const sdbg_col_pred* preds,
                                size_t n_preds, uint64_t key_field, int64_t key_min, uint64_t key_span,
                                uint64_t sum_int_field, uint64_t avg_f64_field, void* d_i64, void* d_f64);
int sdbg_groupby_finalize(sdbg_ctx*, int64_t key_min, uint64_t key_span, const void* d_i64,
                          const void* d_f64, sdbg_group_row* out, uint64_t cap, uint64_t* n_out);
/* min/max of a staged int column (zonemap-style statistics gathered at staging). */
int sdbg_column_minmax_i64(sdbg_segment*, uint64_t field, int64_t* mn, int64_t* mx);

/* ---- host-side writer mirror + deterministic synthetic inputs (index-build side; not timed) ---- */
/* PostingsWriter mirror (irs/formats/posting/writer.hpp): builds a ".doc" stream on the host. segment_docs > 2^32 - 2:
 * SDBG_EINVAL. */
typedef struct sdbg_writer sdbg_writer;
int sdbg_writer_create(uint32_t segment_docs, int has_wand, float wand_b, const uint32_t* norms /* per doc, may be NULL */,
                       sdbg_writer** out);
void sdbg_writer_destroy(sdbg_writer*);
int sdbg_writer_add_term(sdbg_writer*, const uint32_t* docs, const uint32_t* freqs, uint32_t n);
int sdbg_writer_finish(sdbg_writer*, const uint8_t** doc_file, size_t* n, const sdbg_term_meta** terms, size_t* n_terms);
/* Synthetic corpus shard of SURVEY §8d: docs (doc0, doc0+n], terms [t0, t0+nt); fills norms (u8,
 * dl<=255) and stages everything into `seg`. Returns per-term docs_count and the shard's sum of dl. */
int sdbg_synth_corpus(sdbg_segment* seg, uint64_t doc0, uint32_t n_docs, uint32_t t0, uint32_t nt,
                      int threads, uint32_t* docs_count_out /* nt */, uint64_t* sum_dl_out);
/* Same with a probability floor: p_t = max(p_floor, min(0.5, 0.6 / (t + 1))) (flat tail; an index far larger than L2). */
int sdbg_synth_corpus_ex(sdbg_segment* seg, uint64_t doc0, uint32_t n_docs, uint32_t t0, uint32_t nt, int threads, double p_floor,
                         uint32_t* docs_count_out /* nt */, uint64_t* sum_dl_out);
/* Synthetic table column generated directly in HBM: kind as in SURVEY §8d (0 k,1 a,2 b,3 v,4 w,5+ raw),
 * or 6 = int32 n = h % 1000000 (hybrid INCLUDE column, stream 2). */
int sdbg_synth_column(sdbg_segment* seg, uint64_t field, uint64_t stream, int kind, uint64_t row0, uint64_t rows);
uint64_t sdbg_synth_hash(uint64_t stream, uint64_t index);
/* Host-only probe of the staging parser (no device): block table of a ".doc" stream, for tests. */
int sdbg_debug_stage_host(const uint8_t* doc_file, size_t n, const sdbg_term_meta* terms, size_t n_terms, int has_wand,
                          uint32_t cap, uint32_t* n_blocks, uint32_t* term_blk_begin, uint32_t* last_doc,
                          uint32_t* prev_last, uint32_t* packed, uint32_t* max_freq, uint32_t* max_norm,
                          uint64_t* arena_bytes);

/* ---- collectives over NVLink (NCCL, resolved at run time with dlopen: libsdbg.so does not link it) -------------
   One communicator per context, everything enqueued on the context's stream. A C++ host needs nothing but these
   calls: rank 0 creates the id, the host ships its 128 bytes to the other ranks by whatever channel it has
   (the reference's own RPC, MPI, a file), every rank calls sdbg_dist_init. */
#define SDBG_DIST_ID_BYTES 128
int sdbg_dist_unique_id(uint8_t* id128);
int sdbg_dist_init(sdbg_ctx*, const uint8_t* id128, int rank, int world);
int sdbg_dist_destroy(sdbg_ctx*);
int sdbg_dist_allreduce_i64(sdbg_ctx*, void* d_buf, size_t n);                          /* in place, SUM */
int sdbg_dist_allgather(sdbg_ctx*, const void* d_send, void* d_recv, size_t bytes_per_rank);
/* Dense GROUP BY partials (sdbg_filter_groupby_partial) of every rank -> global partials on every rank with ONE
   ncclAllReduce: counts, SUM(int) limbs (exact) and SUM(double) as 120-bit fixed point share one int64 buffer
   (independent of the rank order). abs_bound: finite, identical on every rank, and at least every rank's |partial
   SUM(double)| of every key -- not only the |total|: partials of opposite sign can be far larger than their sum.
   Σ|w| over all passing rows of all ranks is a safe choice. With abs_bound < 2^e, each partial is truncated toward zero
   to a multiple of 2^(e - 116) before the sum (a zero comes back as +0.0). NaN and +-inf partials are carried as counts:
   the merged value is NaN if any partial is NaN or both infinities occur, else the infinity that occurs. A finite partial
   above abs_bound on any rank makes the next sdbg_groupby_finalize / sdbg_sync return SDBG_EINVAL on every rank.
   A non-finite or negative abs_bound: SDBG_EINVAL. */
int sdbg_dist_groupby_merge(sdbg_ctx*, void* d_i64, void* d_f64, uint64_t span, double abs_bound);
/* BM25 top-k over the segments of ALL ranks: local scan -> one all-gather of the k best keys per query -> local
   selection, back to back on the context's stream. hit.seg = rank, hit.doc = ordinal within the rank. out == NULL:
   nothing is copied and nothing waits (results stay in HBM), except the once-per-column zonemap copy of a filter chain
   (SDBG_OP_AND_NEXT). */
int sdbg_dist_bm25_topk_batch(sdbg_segment* const* segs, size_t n_segs, int kind, const sdbg_bm25_term* terms,
                              const uint32_t* term_off, size_t n_queries, float k1, float b, const sdbg_col_pred* filt,
                              uint32_t k, float threshold_in, sdbg_hit* out, uint32_t* n_out);
/* Count, facet counts, aggregates and the sorted scan over the segments of ALL ranks (a corpus sharded by segment, one
   context per GPU): each rank runs the local pass over its own segments with the results left in HBM, then one collective
   and, for the aggregates and the sorted scan, a merge kernel, back to back on the context's stream; the one wait is the
   copy back at the end (the sorted scan's zonemap planning also waits for its own small copies, before its launches,
   and a filter chain's first use of a NOT NULL column waits once for its zonemap copy: SDBG_OP_AND_NEXT).
   The query parameters are those of the *_batch_groups_min entries. A flat query is a degenerate groups query (OR: one
   group, AND: single-term groups), which the groups entries run as the flat entries and with exactly their results
   (§ "Conjunctions of OR groups" above), so there are no flat-form dist entries. Results are those of the local entry
   over the union of all ranks' segments, the same on every rank.
   Caller's contract, as for any collective: every rank makes the same call with the same queries, key_field, key_min,
   key_span, value_field, sort_field, order and k (the collective's size follows from n_queries, key_span and k); every
   rank holds at least one segment (a rank without segments passes a segment with no docs); and every rank has the HBM
   for the scratch below (a failed allocation returns SDBG_ECUDA before the collective, like any CUDA failure).
   Errors: checks of the call's scalar arguments (NULL outputs or offsets, n_queries == 0, the key range as in the local
   entries, world > 1 without sdbg_dist_init) fail alike on every rank before anything is queued. Failures of a rank's
   own pass (a bad term id, a missing or mistyped column, a key outside the range, a value column whose type differs from
   other ranks') still join the collective with a failure flag in the exchanged buffer: the failing rank returns its own
   code, every other rank SDBG_EINVAL, and the outputs are unspecified.
   Without sdbg_dist_init the world is one rank: the all-reduce is a no-op, the all-gather a copy and the merge of one
   rank's buffer the identity on its cells and rows, so each entry gives its local entry's result: exactly for counts,
   facet counts, the integer aggregates, MIN / MAX and the sorted hits; for float64 sums the local pass's own sum, whose
   last bits vary from run to run (its atomics add in no fixed order).
   sdbg_dist_match_count_batch_groups_min / sdbg_dist_match_facet_counts_batch_groups_min: one ncclAllReduce(int64, sum)
   over [counts | NULL counts | out-of-range word | failure flag]; a key outside the range on any rank fails the call on
   every rank. Device scratch: the local entry's, plus (n_queries * (key_span + 2) + 2) * 8 B, plus for a batch
   of several query shapes (flat OR, flat AND, nested) one more set of per-query rows before they are scattered to query
   order.
   sdbg_match_aggregate_batch_groups_min_device: this rank's cells of sdbg_match_aggregate_batch_groups_min left in
   d_cells, with no wait: a 64-byte header {value type, key_span, n_queries, failure word, out-of-range word, 3 zero words}
   then n_queries * (key_span + 1) cells of 48 B (the per-key cells, then the NULL key's). A failure of the local pass
   returns its code and sets the header's failure word, so that a merge of the buffer fails on every rank.
   sdbg_match_aggregate_merge_gathered: the aggregates of n_ranks such buffers back to back (rank order). One thread per
   (query, key) cell: counts add, integer sums add in 128-bit two's complement with an exact carry, float64 sums are the
   ranks' partials added in rank order (bit-identical on every rank; IEEE NaN / inf rules hold), MIN / MAX are the largest
   order keys; then the local entry's conversion. The float64 sum therefore differs from the local entry's over the
   unsharded corpus only by the order of the additions. Headers that disagree (value type, key_span, n_queries) or any
   rank's failure or out-of-range word: SDBG_EINVAL. key_span > 4096: SDBG_EUNSUPPORTED.
   sdbg_dist_match_aggregate_batch_groups_min: the device form, one sdbg_dist_allgather, the merge. Device scratch:
   (1 + world) buffers of the device form plus one of merged cells: 4096 queries x 2002 keys x 48 B = 394 MB per buffer,
   3.9 GB at 8 ranks, a batch of several query shapes one more buffer of rows, and 394 MB of pinned host memory for the
   copy back. Split larger batches.
   sdbg_match_topk_by_column_batch_groups_min_device: this rank's min(k, matches) best rows per query of
   sdbg_match_topk_by_column_batch_groups_min, best first, left in d_rows with no wait: a 64-byte header {sort type, desc,
   nulls_first, k, n_queries, failure word, 2 zero words}, the row count of each query (u64 [n_queries]), then rows
   [n_queries][k] of 24 B: the 16-byte key of the sorted scan (bm25_sort.cuh) with ~rank in bits 32..62 of its low word, so
   that ties go to the lower rank, and the stored value's 8 bytes (the key canonicalises -0.0 and NaN). Each rank keeps up
   to 2^32 - 2 docs per call, as the local entry. rank >= 2^31: SDBG_EUNSUPPORTED; a failure of the local pass returns its
   code and sets the failure word.
   sdbg_match_topk_by_column_merge_gathered: per query (one CTA) the k best of n_ranks such buffers, in order, as
   sdbg_sort_hit: the value bits, doc = the hit's ordinal within its rank + 1 (the rank's earlier segments' docs plus the
   doc id), seg = the rank, is_null. Ties go to (rank asc, segment asc, doc asc): with ranks holding consecutive segments
   in corpus order, the order of the local entry over the unsharded corpus. Headers that disagree (sort type, desc,
   nulls_first, k, n_queries) or any rank's failure word: SDBG_EINVAL. k == 0: SDBG_EINVAL; k > 4096: SDBG_EUNSUPPORTED.
   sdbg_dist_match_topk_by_column_batch_groups_min: the device form, one sdbg_dist_allgather, the merge; hit.seg = rank.
   Device scratch: the local entry's, (1 + world) device-form buffers of 64 + n_queries * (8 + 24 k) B (8 ranks, 4096
   queries, k = 1000: 787 MB gathered), n_queries * k * 24 B of merged hits, and as much pinned host memory.
   sdbg_bm25_topk_batch_groups_min_device: this rank's result of sdbg_bm25_topk_batch_groups_min (same query and scorer
   parameters, threshold_in included: flat OR / AND, groups, min-match, exclusions, filter chains, deleted docs; BM25, BM15,
   BM1 and TFIDF) left in d_buf with no wait: a 64-byte header {k, n_queries, failure word, 5 zero words}, then the keys
   (u64 [n_queries][k], best first: score bits << 32 | ~ordinal, the ordinal being the docs of the rank's earlier segments
   plus the doc id, up to 2^32 - 2), total_matches (u64 [n_queries]) and the hit counts (u32 [n_queries]), padded to a multiple of 8 B: 64 +
   8 * ceil(n_queries * (8k + 12) / 8) B. The counts say how many keys are real: under BM1 every score is 0, so a key's value marks nothing. There is
   no rank parameter and no rank slot: a rank is its buffer's position in the gathered array, and a rank holds up to
   2^32 - 2 docs per call, as the local entry. Errors of the call's scalar arguments (NULL offsets or d_buf, k == 0,
   n_queries == 0: SDBG_EINVAL; k > 8192, n_queries > 65535: SDBG_EUNSUPPORTED) return before anything is queued; any
   other failure of the local pass returns its code and sets the failure word.
   sdbg_bm25_topk_merge_gathered: per query the k best hits of n_ranks such buffers back to back (rank order), ordered by
   (score desc, rank asc, ordinal asc), as sdbg_hit with seg = the rank and doc = the ordinal within the rank; n_out =
   min(k, hits) and total_matches (NULL: not wanted) the sum of the ranks' totals. With ranks holding consecutive segments
   in corpus order, the hits are those of the local entry over the unsharded corpus. The lists are re-keyed by position
   (score bits << 32 | ~(rank * k + index)), selected with the local merge kernel and mapped back, which is exact while
   n_ranks * k < 2^32 (k = 8192: 2^19 ranks). The headers are read first (one small copy and a wait): headers that
   disagree (k, n_queries) or any rank's failure word: SDBG_EINVAL with nothing queued. n_ranks == 0, k == 0, n_queries ==
   0: SDBG_EINVAL; k > 8192, n_queries > 65535, n_ranks * k >= 2^32: SDBG_EUNSUPPORTED. Synchronous on the context's stream.
   sdbg_dist_bm25_topk_batch_groups_min: the device form, one sdbg_dist_allgather, the merge, with the errors above; hit.seg
   = rank. Caller's contract, besides the one above: every rank passes the same term statistics (corpus-wide, as
   dist.global_term_stats computes them), scorer and threshold_in, so that a doc scores the same on every rank. Device
   scratch: the local entry's, (1 + world) device-form buffers (4096 queries at k = 1000: 33 MB per rank, 262 MB gathered
   at 8 ranks), the re-keyed lists (about one more gathered buffer), n_queries * k * 8 B of merged keys and n_queries * (12k
   + 12) B of hits, with as much pinned host memory for the copy back.
   sdbg_bm25_topk_batch_device and sdbg_dist_bm25_topk_batch keep their flat queries and 2^28-ordinal rank slots.
   Not supported: the streaming scan across ranks, a score or sort threshold exchanged between ranks during the scan. */
int sdbg_dist_match_count_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                           const uint32_t* group_off, const uint32_t* query_group_off,
                                           const uint32_t* group_min /* NULL: all 1 */, size_t n_queries,
                                           const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                           const sdbg_col_pred* filt, uint64_t* counts /* n_queries */);
int sdbg_dist_match_facet_counts_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                  const uint32_t* group_off, const uint32_t* query_group_off,
                                                  const uint32_t* group_min /* NULL: all 1 */, size_t n_queries,
                                                  const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                                  const sdbg_col_pred* filt, uint64_t key_field, int64_t key_min,
                                                  uint32_t key_span, uint64_t* counts /* n_queries * key_span */,
                                                  uint64_t* null_counts /* n_queries */);
int sdbg_match_aggregate_batch_groups_min_device(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                 const uint32_t* group_off, const uint32_t* query_group_off,
                                                 const uint32_t* group_min /* NULL: all 1 */, size_t n_queries,
                                                 const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                                 const sdbg_col_pred* filt, uint64_t key_field, int64_t key_min,
                                                 uint32_t key_span, uint64_t value_field,
                                                 void* d_cells /* 64 + n_queries * (key_span + 1) * 48 B */);
int sdbg_match_aggregate_merge_gathered(sdbg_ctx*, const void* d_all /* n_ranks device-form buffers */, uint32_t n_ranks,
                                        size_t n_queries, uint32_t key_span, sdbg_match_agg* out /* n_queries * key_span */,
                                        sdbg_match_agg* null_out /* n_queries */);
int sdbg_match_topk_by_column_batch_groups_min_device(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                      const uint32_t* group_off, const uint32_t* query_group_off,
                                                      const uint32_t* group_min /* NULL: all 1 */, size_t n_queries,
                                                      const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                                      const sdbg_col_pred* filt, uint64_t sort_field, int descending,
                                                      int nulls_first, uint32_t k, uint32_t rank,
                                                      void* d_rows /* 64 + n_queries * (8 + 24 * k) B */);
int sdbg_match_topk_by_column_merge_gathered(sdbg_ctx*, const void* d_all /* n_ranks device-form buffers */, uint32_t n_ranks,
                                             size_t n_queries, uint32_t k, sdbg_sort_hit* out /* n_queries * k */,
                                             uint32_t* n_out /* n_queries */);
int sdbg_dist_match_topk_by_column_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                    const uint32_t* group_off, const uint32_t* query_group_off,
                                                    const uint32_t* group_min /* NULL: all 1 */, size_t n_queries,
                                                    const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                                    const sdbg_col_pred* filt, uint64_t sort_field, int descending,
                                                    int nulls_first, uint32_t k, sdbg_sort_hit* out /* n_queries * k */,
                                                    uint32_t* n_out /* n_queries */);
int sdbg_dist_match_aggregate_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                               const uint32_t* group_off, const uint32_t* query_group_off,
                                               const uint32_t* group_min /* NULL: all 1 */, size_t n_queries,
                                               const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                               const sdbg_col_pred* filt, uint64_t key_field, int64_t key_min,
                                               uint32_t key_span, uint64_t value_field,
                                               sdbg_match_agg* out /* n_queries * key_span */,
                                               sdbg_match_agg* null_out /* n_queries */);
int sdbg_bm25_topk_batch_groups_min_device(sdbg_segment* const* segs, size_t n_segs, const sdbg_bm25_term* terms,
                                           const uint32_t* group_off, const uint32_t* query_group_off,
                                           const uint32_t* group_min /* NULL: all 1 */, size_t n_queries,
                                           const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                           float k1, float b, const sdbg_col_pred* filt, uint32_t k, float threshold_in,
                                           void* d_buf /* 64 + 8 * ceil(n_queries * (8 * k + 12) / 8) B */);
int sdbg_bm25_topk_merge_gathered(sdbg_ctx*, const void* d_all /* n_ranks device-form buffers */, uint32_t n_ranks,
                                  size_t n_queries, uint32_t k, sdbg_hit* out /* n_queries * k */,
                                  uint32_t* n_out /* n_queries */, uint64_t* total_matches /* n_queries, or NULL */);
int sdbg_dist_bm25_topk_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const sdbg_bm25_term* terms,
                                         const uint32_t* group_off, const uint32_t* query_group_off,
                                         const uint32_t* group_min /* NULL: all 1 */, size_t n_queries,
                                         const uint32_t* excl_terms, const uint32_t* excl_off /* NULL: none */,
                                         float k1, float b, const sdbg_col_pred* filt, uint32_t k, float threshold_in,
                                         sdbg_hit* out /* n_queries * k */, uint32_t* n_out /* n_queries */,
                                         uint64_t* total_matches /* n_queries, or NULL */);

#ifdef __cplusplus
}
#endif
#endif /* SDBG_H_ */
