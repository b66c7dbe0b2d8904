// gpu_adapters.hpp -- the two C++ adapters a SereneDB maintainer would add (INTEGRATION.md):
//
//  * GpuTopKIterator : irs::DocIterator -- returned from PostingsReaderImpl::WandIterator
//    (irs/formats/posting/reader.hpp:457-501) instead of MaxScoreIterator / SingleWandIterator when a
//    segment is staged on a GPU. Collect() runs the fused scan+score+top-k kernel for the segment and
//    feeds <= k (doc, score) pairs to the caller's ScoreCollector, honouring / publishing the
//    ScoreThresholdAttr exactly as CollectSegmentTopK expects
//    (server/connector/duckdb_search_full_scan.cpp:1898-1920).
//  * GpuAggScan -- the body of a new ScanMode::GpuAgg branch of IResearchScanFunction
//    (server/connector/duckdb_search_full_scan.cpp:1645-1709, modes :56-77 of the .hpp): the pushed
//    TableFilterSet + GROUP BY + SUM/AVG/COUNT run in one kernel and the scan emits already-aggregated
//    rows, <= STANDARD_VECTOR_SIZE per call, cardinality 0 = end of scan (like RunCountScan :2201-2239).
//
// Errors: the ABI returns codes; the adapters turn them into C++ exceptions like the reference's
// IoError / THROW_SQL_ERROR call sites.
#pragma once

#include <atomic>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/sdbg.h"
#include "irs_mock.hpp"

namespace sdbg_host {

struct GpuError : std::runtime_error {
  int code;
  GpuError(int c, const std::string& what) : std::runtime_error(what), code(c) {}
};

// A pushed filter as the adapters keep it: the whole chain at `table_filter` (sdbg.h, SDBG_OP_AND_NEXT; the conjunction
// of a ConjunctionAndFilter's comparison children), copied entry by entry up to the first without the bit or the 4th.
// data() is what the ABI takes: NULL for no filter.
struct FilterChain {
  std::vector<sdbg_col_pred> preds;
  FilterChain() = default;
  explicit FilterChain(const sdbg_col_pred* table_filter);
  const sdbg_col_pred* data() const { return preds.empty() ? nullptr : preds.data(); }
};

// One scored query over one staged segment.
class GpuTopKIterator final : public irs::DocIterator {
 public:
  GpuTopKIterator(sdbg_segment* segment, int kind /* SDBG_QUERY_OR | SDBG_QUERY_AND */,
                  std::vector<sdbg_bm25_term> terms /* BM25Stats per term + boost */, float k1 /* BM25::k() */,
                  float b /* BM25::b() */, uint32_t k /* 0 = streaming mode: every match, see EmitScoredDocs */,
                  const sdbg_col_pred* table_filter /* nullable: the ColFilter wrap */,
                  std::vector<uint32_t> excluded_terms = {} /* term ids of the And's Not children (irs exclusion.hpp) */,
                  std::vector<uint32_t> group_sizes = {} /* an And of Ors: consecutive OR groups over `terms`; empty = flat */,
                  std::vector<uint32_t> group_min_match = {} /* per group: Or::min_match_count, 1..its size; empty = all 1.
                    With phrase_positions: one per clause group (per clause_group_sizes, or per clause when that is
                    empty), 1..its clauses, 1 for a negated group; another size: GpuError(SDBG_EINVAL) */,

                  std::vector<uint32_t> phrase_positions = {} /* non-empty: `terms` are a by_phrase's slots at these
                                                                 relative positions (0 first, increasing); needs k > 0 */,
                  std::vector<uint32_t> clause_sizes = {} /* an And of clauses: consecutive clauses over `terms` /
                                                            phrase_positions (a one-slot clause is a term); empty: one phrase */,
                  std::vector<uint8_t> clause_negated = {} /* per clause: 1 for a Not child; empty: none */,
                  std::vector<uint32_t> clause_group_sizes = {} /* clauses per OR group, in order; empty: one per group */);

  // Scored top-k: the hot path.
  void Collect(const irs::ScoreFunction&, irs::ColumnArgsFetcher&, irs::ScoreCollector& collector) override;
  // Windowed variant used by TableFilterDocIterator / streaming callers (RunStreamingScan,
  // duckdb_search_full_scan.cpp:2370-2403): hits with doc in [min, max). With k = 0 the iterator holds every match
  // of the segment (sdbg_bm25_scan), so draining it window by window is the reference's streaming scan.
  uint32_t EmitScoredDocs(irs::doc_id_t* out, irs::score_t* scores, irs::doc_id_t max, const irs::ScoreFunction&,
                          irs::ColumnArgsFetcher*, irs::doc_id_t min) override;
  uint32_t EmitDocs(irs::doc_id_t* out, irs::doc_id_t min, irs::doc_id_t max) override;
  uint32_t count() override;  // total matches (exhaustive, like DocIterator::count)
  irs::doc_id_t advance() override;
  irs::doc_id_t seek(irs::doc_id_t target) override;
  // Bitmap + score window of [min, max) for callers that merge iterators (Conjunction / MaxScore windows,
  // iterators.hpp:322-337): bit (doc - min) per hit, score accumulated into score.score_window per merge_type,
  // match counts when match.matches is given. The hits are this iterator's top-k (its whole result set).
  std::pair<irs::doc_id_t, bool> FillBlock(irs::doc_id_t min, irs::doc_id_t max, uint64_t* mask, irs::FillBlockScoreContext score,
                                           irs::FillBlockMatchContext match) override;
  void FetchScoreArgs(uint16_t) override {}   // score arguments never leave the GPU
  // AttributeProvider: ScoreThresholdAttr (the caller seeds / reads the running threshold through it,
  // doc_collector.hpp:124-130, duckdb_search_full_scan.cpp:1910-1914) and CostAttr (conjunction ordering).
  irs::Attribute* GetMutable(irs::TypeInfo::type_id type) noexcept override;

  irs::ScoreThresholdAttr& threshold() noexcept { return threshold_; }
  const irs::CostAttr& cost() const noexcept { return cost_; }
  uint64_t total_matches() const noexcept { return total_; }

 private:
  void run();
  sdbg_segment* seg_;
  int kind_;
  std::vector<sdbg_bm25_term> terms_;
  std::vector<uint32_t> excluded_;
  std::vector<uint32_t> groups_;   // sizes of the OR groups over terms_ (empty: the flat `kind_` query)
  std::vector<uint32_t> group_min_;   // their minimum match counts (empty: all 1)
  std::vector<uint32_t> phrase_;      // a phrase's relative positions, one per term (empty: not a phrase)
  std::vector<uint32_t> clause_off_;  // the clauses over terms_ / phrase_ (a single phrase: one clause)
  std::vector<uint8_t> clause_neg_;   // per clause: negated
  std::vector<uint32_t> group_off_;   // the OR groups over the clauses (clause_group_sizes)
  std::vector<uint8_t> group_neg_;    // per group: negated
  float k1_, b_;
  uint32_t k_;
  FilterChain filter_;
  irs::ScoreThresholdAttr threshold_;
  irs::CostAttr cost_;
  std::vector<sdbg_hit> hits_;   // sorted by (score desc, doc asc) after run()
  std::vector<sdbg_hit> by_doc_; // same hits ordered by doc for advance()/seek()/Emit*
  size_t pos_ = 0;
  uint64_t total_ = 0;
  bool ran_ = false;
};

// SELECT key, COUNT(*), SUM(sum_int), AVG(avg_f64) FROM t WHERE preds GROUP BY key -- emitted in chunks.
class GpuAggScan {
 public:
  GpuAggScan(std::vector<sdbg_segment*> segments, std::vector<sdbg_col_pred> pushed_filters, uint64_t key_field,
             uint64_t sum_int_field, uint64_t avg_f64_field, uint32_t n_groups_hint);
  // IResearchScanFunction body for ScanMode::GpuAgg: fills `output`; output.size == 0 => exhausted.
  void Scan(duckdb::DataChunkMock& output);
  uint64_t rows_scanned() const noexcept { return rows_scanned_; }  // get_metrics hook (:860-864)

 private:
  std::vector<sdbg_segment*> segs_;
  std::vector<sdbg_col_pred> preds_;
  uint64_t key_, sum_i_, avg_f_;
  uint32_t hint_;
  std::vector<sdbg_group_row> groups_;
  size_t cursor_ = 0;
  bool ran_ = false;
  uint64_t rows_scanned_ = 0;
};

// SELECT count(*) FROM t WHERE body @@ '<query>' [AND <pushed filter>] -- the body of ScanMode::Count
// (duckdb_search_full_scan.cpp RunCountScan :2201-2239) for a text query: one row with the count, then cardinality 0.
// Nothing is scored (sdbg_match_count_batch); the count is exact whatever the pruning level.
class GpuCountScan {
 public:
  GpuCountScan(std::vector<sdbg_segment*> segments, int kind /* SDBG_QUERY_OR | SDBG_QUERY_AND */, std::vector<uint32_t> terms,
               std::vector<uint32_t> excluded_terms /* the And's Not children */, const sdbg_col_pred* table_filter /* nullable */,
               std::vector<uint32_t> group_sizes = {} /* an And of Ors: consecutive OR groups over `terms`; empty = flat */,
               std::vector<uint32_t> group_min_match = {} /* per group: Or::min_match_count, 1..its size; empty = all 1.
                 With phrase_positions: one per clause group (per clause_group_sizes, or per clause when that is
                 empty), 1..its clauses, 1 for a negated group; another size: GpuError(SDBG_EINVAL) */,

               std::vector<uint32_t> phrase_positions = {} /* non-empty: `terms` are a by_phrase's slots at these
                                                              relative positions (0 first, increasing) */,
               std::vector<uint32_t> clause_sizes = {} /* an And of clauses: consecutive clauses over `terms` /
                                                         phrase_positions (a one-slot clause is a term); empty: one phrase */,
               std::vector<uint8_t> clause_negated = {} /* per clause: 1 for a Not child; empty: none */,
                  std::vector<uint32_t> clause_group_sizes = {} /* clauses per OR group, in order; empty: one per group */);
  // Fills `output` with one row, count[0] = the number of matches; the next call leaves it empty (end of scan).
  void Scan(duckdb::DataChunkMock& output);

 private:
  std::vector<sdbg_segment*> segs_;
  int kind_;
  std::vector<uint32_t> terms_, excluded_, groups_, group_min_, phrase_, clause_off_;   // clause_off_: the phrase's clauses
  std::vector<uint8_t> clause_neg_, group_neg_;
  std::vector<uint32_t> group_off_;   // the OR groups over the clauses (clause_group_sizes)
  FilterChain filter_;
  bool done_ = false;
};

// SELECT ... FROM t WHERE body @@ '<query>' [AND <pushed filter>] ORDER BY col [DESC] [NULLS FIRST|LAST] LIMIT k -- the body
// of the TOP_N(col) <- IRESEARCH_SCAN(Stream) plan shape (duckdb_search_full_scan.cpp IResearchSetScanOrder :1711-1762 pushes
// only score orders; RunStreamingScan :2370-2403 serves the rest under TOP_N). One sdbg_match_topk_by_column_batch call
// (sdbg_match_topk_by_column_batch_groups_min with group_sizes, sdbg_phrase_topk_by_column_batch with phrase_positions) on the first Scan; then rows (doc, segment, value, valid) in TOP_N's order, <= STANDARD_VECTOR_SIZE per call,
// cardinality 0 at the end.
class GpuSortedScan {
 public:
  GpuSortedScan(std::vector<sdbg_segment*> segments, int kind /* SDBG_QUERY_OR | SDBG_QUERY_AND */, std::vector<uint32_t> terms,
                std::vector<uint32_t> excluded_terms /* the And's Not children */, const sdbg_col_pred* table_filter /* nullable */,
                uint64_t sort_field, bool descending, bool nulls_first /* the plan's resolved OrderByNullType */,
                uint32_t k /* LIMIT (+ OFFSET), 1..4096 */,
                std::vector<uint32_t> group_sizes = {} /* an And of Ors, as GpuCountScan takes it; kind is then unused */,
                std::vector<uint32_t> group_min_match = {} /* per group: Or::min_match_count, 1..its size; empty = all 1.
                  With phrase_positions: one per clause group (per clause_group_sizes, or per clause when that is
                  empty), 1..its clauses, 1 for a negated group; another size: GpuError(SDBG_EINVAL) */,

                std::vector<uint32_t> phrase_positions = {} /* non-empty: `terms` are a by_phrase's slots at these
                                                               relative positions (0 first, increasing) */,
                std::vector<uint32_t> clause_sizes = {} /* an And of clauses: consecutive clauses over `terms` /
                                                          phrase_positions (a one-slot clause is a term); empty: one phrase */,
                std::vector<uint8_t> clause_negated = {} /* per clause: 1 for a Not child; empty: none */,
                  std::vector<uint32_t> clause_group_sizes = {} /* clauses per OR group, in order; empty: one per group */);
  void Scan(duckdb::DataChunkMock& output);

 private:
  std::vector<sdbg_segment*> segs_;
  int kind_;
  std::vector<uint32_t> terms_, excluded_, group_sizes_, group_min_, phrase_, clause_off_;   // clause_off_: the phrase's clauses
  std::vector<uint8_t> clause_neg_, group_neg_;
  std::vector<uint32_t> group_off_;   // the OR groups over the clauses (clause_group_sizes)
  FilterChain filter_;
  uint64_t field_;
  bool desc_, nulls_first_;
  uint32_t k_;
  std::vector<sdbg_sort_hit> hits_;
  size_t cursor_ = 0;
  bool ran_ = false;
};

// SELECT id [, bm25(...)] FROM t WHERE body @@ '<query>' [AND <pushed filter>] [LIMIT n OFFSET o] without ORDER BY -- the
// body of the Stream scan mode (duckdb_search_full_scan.cpp RunStreamingScan :2370-2403) for flat, grouped and min-match
// queries and phrases over every segment. Pages of kPage matches come from sdbg_match_scan_batch_groups_min
// (sdbg_phrase_scan_batch with phrase_positions, scored with the phrase's summed idfs) (offset += kPage); Scan
// emits rows (doc, segment, score) of at most STANDARD_VECTOR_SIZE in (segment, doc) order, cardinality 0 at the end.
// Scores are those of the top-k at pruning level 0 when `scored`, else 0 (no frequency or norm is read).
class GpuMatchScan {
 public:
  static constexpr uint32_t kPage = 1u << 20;
  GpuMatchScan(std::vector<sdbg_segment*> segments, std::vector<sdbg_bm25_term> terms /* statistics unused when unscored */,
               std::vector<uint32_t> excluded_terms /* the And's Not children */, const sdbg_col_pred* table_filter /* nullable */,
               float k1, float b, bool scored,
               std::vector<uint32_t> group_sizes = {} /* an And of Ors over `terms`; empty = one group (a flat OR) */,
               std::vector<uint32_t> group_min_match = {} /* per group: Or::min_match_count, 1..its size; empty = all 1.
                 With phrase_positions: one per clause group (per clause_group_sizes, or per clause when that is
                 empty), 1..its clauses, 1 for a negated group; another size: GpuError(SDBG_EINVAL) */,

               std::vector<uint32_t> phrase_positions = {} /* non-empty: `terms` are a by_phrase's slots at these
                                                              relative positions (0 first, increasing) */,
               std::vector<uint32_t> clause_sizes = {} /* an And of clauses: consecutive clauses over `terms` /
                                                         phrase_positions (a one-slot clause is a term); empty: one phrase */,
               std::vector<uint8_t> clause_negated = {} /* per clause: 1 for a Not child; empty: none */,
                  std::vector<uint32_t> clause_group_sizes = {} /* clauses per OR group, in order; empty: one per group */);
  void Scan(duckdb::DataChunkMock& output);
  uint64_t total_matches() const { return total_; }

 private:
  void Fetch();
  std::vector<sdbg_segment*> segs_;
  std::vector<sdbg_bm25_term> terms_;
  std::vector<uint32_t> excluded_, group_sizes_, group_min_, phrase_, clause_off_;   // clause_off_: the phrase's clauses
  std::vector<uint8_t> clause_neg_, group_neg_;
  std::vector<uint32_t> group_off_;   // the OR groups over the clauses (clause_group_sizes)
  FilterChain filter_;
  float k1_, b_;
  bool scored_;
  std::vector<sdbg_hit> page_;
  uint64_t offset_ = 0, total_ = 0;   // ordinal of page_[0]'s successor page; the query's matches
  size_t cursor_ = 0;
  bool ran_ = false;
};

// SELECT col, count(*) FROM t WHERE body @@ '<query>' [AND <pushed filter>] GROUP BY col -- the body of the
// HASH_GROUP_BY(col; count_star()) <- IRESEARCH_SCAN(text query) plan shape (facet counts). The first Scan takes the key
// range from sdbg_column_minmax_i64 over the segments and runs one sdbg_match_facet_counts_batch call
// (sdbg_match_facet_counts_batch_groups_min with group_sizes, sdbg_phrase_facet_counts_batch with phrase_positions); then the non-empty
// groups as rows (key, count, valid) in ascending key order, the NULL group (valid = 0) last, <= STANDARD_VECTOR_SIZE per
// call, cardinality 0 at the end. A key range wider than 32768 throws GpuError(SDBG_EUNSUPPORTED): the plan stays on the CPU.
class GpuFacetScan {
 public:
  GpuFacetScan(std::vector<sdbg_segment*> segments, int kind /* SDBG_QUERY_OR | SDBG_QUERY_AND */, std::vector<uint32_t> terms,
               std::vector<uint32_t> excluded_terms /* the And's Not children */, const sdbg_col_pred* table_filter /* nullable */,
               uint64_t key_field /* int64 or int32 */,
               std::vector<uint32_t> group_sizes = {} /* an And of Ors, as GpuCountScan takes it; kind is then unused */,
               std::vector<uint32_t> group_min_match = {} /* per group: Or::min_match_count, 1..its size; empty = all 1.
                 With phrase_positions: one per clause group (per clause_group_sizes, or per clause when that is
                 empty), 1..its clauses, 1 for a negated group; another size: GpuError(SDBG_EINVAL) */,

               std::vector<uint32_t> phrase_positions = {} /* non-empty: `terms` are a by_phrase's slots at these
                                                              relative positions (0 first, increasing) */,
               std::vector<uint32_t> clause_sizes = {} /* an And of clauses: consecutive clauses over `terms` /
                                                         phrase_positions (a one-slot clause is a term); empty: one phrase */,
               std::vector<uint8_t> clause_negated = {} /* per clause: 1 for a Not child; empty: none */,
                  std::vector<uint32_t> clause_group_sizes = {} /* clauses per OR group, in order; empty: one per group */);
  void Scan(duckdb::DataChunkMock& output);

 private:
  std::vector<sdbg_segment*> segs_;
  int kind_;
  std::vector<uint32_t> terms_, excluded_, group_sizes_, group_min_, phrase_, clause_off_;   // clause_off_: the phrase's clauses
  std::vector<uint8_t> clause_neg_, group_neg_;
  std::vector<uint32_t> group_off_;   // the OR groups over the clauses (clause_group_sizes)
  FilterChain filter_;
  uint64_t field_;
  std::vector<std::pair<int64_t, uint64_t>> groups_;   // (key, count) of the non-empty groups
  uint64_t nulls_ = 0;                                 // the NULL group's count
  size_t cursor_ = 0;                                  // rows emitted; the NULL group is row groups_.size()
  bool ran_ = false;
};

// SELECT [col,] count(*), count(v), sum(v), avg(v), min(v), max(v) FROM t WHERE body @@ '<query>' [AND <pushed filter>]
// [GROUP BY col] -- the body of the HASH_GROUP_BY(col; count_star(), count(v), sum(v), avg(v), min(v), max(v)) and
// UNGROUPED_AGGREGATE(...) <- IRESEARCH_SCAN(text query) plan shapes, for one value column (two columns: two scans). The
// first Scan takes the key range as GpuFacetScan does and runs one sdbg_match_aggregate_batch call
// (sdbg_match_aggregate_batch_groups_min with group_sizes, sdbg_phrase_aggregate_batch with phrase_positions). Grouped, it then emits the non-empty groups as rows (key, count,
// count_value, sum_lo / sum_hi or sum_f64, avg, min, max, valid) in ascending key order, the NULL group (valid = 0) last;
// ungrouped (key_field UINT64_MAX), one row. <= STANDARD_VECTOR_SIZE rows per call, cardinality 0 at the end. A row with
// count_value 0 has NULL sum, avg, min and max (emitted as 0). A key range wider than 4096 values throws
// GpuError(SDBG_EUNSUPPORTED): the plan stays on the CPU.
class GpuMatchAggScan {
 public:
  GpuMatchAggScan(std::vector<sdbg_segment*> segments, int kind /* SDBG_QUERY_OR | SDBG_QUERY_AND */, std::vector<uint32_t> terms,
                  std::vector<uint32_t> excluded_terms /* the And's Not children */, const sdbg_col_pred* table_filter /* nullable */,
                  uint64_t key_field /* int64 or int32; UINT64_MAX: no GROUP BY */, uint64_t value_field,
                  sdbg_type value_type /* as staged: picks sum_f64 or the 128-bit sum for avg */,
                  std::vector<uint32_t> group_sizes = {} /* an And of Ors, as GpuCountScan takes it; kind is then unused */,
                  std::vector<uint32_t> group_min_match = {} /* per group: Or::min_match_count, 1..its size; empty = all 1.
                    With phrase_positions: one per clause group (per clause_group_sizes, or per clause when that is
                    empty), 1..its clauses, 1 for a negated group; another size: GpuError(SDBG_EINVAL) */,

                  std::vector<uint32_t> phrase_positions = {} /* non-empty: `terms` are a by_phrase's slots at these
                                                                 relative positions (0 first, increasing) */,
                  std::vector<uint32_t> clause_sizes = {} /* an And of clauses: consecutive clauses over `terms` /
                                                            phrase_positions (a one-slot clause is a term); empty: one phrase */,
                  std::vector<uint8_t> clause_negated = {} /* per clause: 1 for a Not child; empty: none */,
                  std::vector<uint32_t> clause_group_sizes = {} /* clauses per OR group, in order; empty: one per group */);
  void Scan(duckdb::DataChunkMock& output);

 private:
  std::vector<sdbg_segment*> segs_;
  int kind_;
  std::vector<uint32_t> terms_, excluded_, group_sizes_, group_min_, phrase_, clause_off_;   // clause_off_: the phrase's clauses
  std::vector<uint8_t> clause_neg_, group_neg_;
  std::vector<uint32_t> group_off_;   // the OR groups over the clauses (clause_group_sizes)
  FilterChain filter_;
  uint64_t key_field_, value_field_;
  sdbg_type value_type_;
  std::vector<std::pair<int64_t, sdbg_match_agg>> groups_;   // (key, cell) of the rows to emit
  bool null_row_ = false;                                    // the last row of groups_ is the NULL group
  size_t cursor_ = 0;
  bool ran_ = false;
};

// The same scan mode under DuckDB's threading contract (duckdb_search_full_scan.hpp:85-255, .cpp:99-268): ONE global
// state shared by all workers of the query -- touched through atomics only, like next_segment / next_unit there -- and
// one local state per worker. The first worker to arrive runs the aggregation on the GPU (the others wait on the
// once-flag, as they would wait for rows anyway); afterwards every worker claims chunks of <= STANDARD_VECTOR_SIZE
// result rows from an atomic cursor and fills its own DataChunk. Cardinality 0 = this worker is done.
struct GpuAggGlobalState {
  GpuAggGlobalState(std::vector<sdbg_segment*> segments, std::vector<sdbg_col_pred> pushed_filters, uint64_t key_field,
                    uint64_t sum_int_field, uint64_t avg_f64_field, uint32_t n_groups_hint);
  std::vector<sdbg_segment*> segs;
  std::vector<sdbg_col_pred> preds;
  uint64_t key, sum_i, avg_f;
  uint32_t hint;
  std::once_flag ran;
  std::vector<sdbg_group_row> groups;          // written once (under `ran`), read-only afterwards
  std::atomic<size_t> next_chunk{0};           // claim cursor, in units of STANDARD_VECTOR_SIZE rows
  std::atomic<uint64_t> rows_emitted{0};       // get_metrics hook
};
struct GpuAggLocalState {
  uint64_t chunks_claimed = 0;
};
// Body of IResearchScanFunction for ScanMode::GpuAgg (:1645-1709): safe to call from many threads at once.
void GpuAggScanFunction(GpuAggGlobalState& g, GpuAggLocalState& l, duckdb::DataChunkMock& output);

}  // namespace sdbg_host
