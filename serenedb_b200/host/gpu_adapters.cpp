#include "gpu_adapters.hpp"

#include <algorithm>
#include <cfloat>

namespace sdbg_host {

namespace {
void check(int rc, const char* what) {
  if (rc != SDBG_OK) throw GpuError(rc, std::string(what) + " failed with code " + std::to_string(rc));
}

// OR group sizes -> the group_off / query_group_off pair of one query (sdbg_*_batch_groups).
std::vector<uint32_t> group_offsets(const std::vector<uint32_t>& sizes, size_t n_terms) {
  std::vector<uint32_t> off(1, 0u);
  for (uint32_t n : sizes) off.push_back(off.back() + n);
  if (off.back() != n_terms) throw GpuError(SDBG_EINVAL, "OR group sizes must add up to the number of terms");
  return off;
}

// Per-group minimum match counts: one per group, or none (every group 1).
const uint32_t* group_minimums(const std::vector<uint32_t>& mins, size_t n_groups) {
  if (mins.empty()) return nullptr;
  if (mins.size() != n_groups) throw GpuError(SDBG_EINVAL, "one minimum match count per OR group");
  return mins.data();
}

// Per clause group of a phrase query (group_neg: one entry per group) its minimum match count, or none (every group 1).
const uint32_t* phrase_minimums(const std::vector<uint32_t>& mins, const std::vector<uint8_t>& group_neg) {
  if (mins.empty()) return nullptr;
  if (mins.size() != group_neg.size()) throw GpuError(SDBG_EINVAL, "one minimum match count per clause group");
  return mins.data();
}

// A phrase's relative positions: one per slot and no OR groups of terms (the library checks their order).
void check_phrase(const std::vector<uint32_t>& phrase, size_t n_terms, bool groups) {
  if (phrase.empty()) return;
  if (phrase.size() != n_terms) throw GpuError(SDBG_EINVAL, "one phrase position per term");
  if (groups) throw GpuError(SDBG_EUNSUPPORTED, "a phrase has no OR groups");
}

// The clauses of a phrase query over its n_terms slots for the sdbg_phrase_groups_* entries: clause_off (clause j is
// slots off[j] .. off[j + 1]), each clause's negation, and the OR groups over the clauses: group_off (group g is clauses
// goff[g] .. goff[g + 1]) and each group's negation, which all its clauses share. Empty sizes and negations: the slots are
// one positive clause (a single phrase); empty group sizes: one clause per group (an And of the clauses). Not a phrase
// (no positions): no clauses.
void phrase_clauses(const std::vector<uint32_t>& phrase, size_t n_terms, const std::vector<uint32_t>& sizes,
                    const std::vector<uint8_t>& negated, const std::vector<uint32_t>& group_sizes, std::vector<uint32_t>& off,
                    std::vector<uint8_t>& neg, std::vector<uint32_t>& goff, std::vector<uint8_t>& gneg) {
  if (phrase.empty()) {
    if (!sizes.empty() || !negated.empty() || !group_sizes.empty())
      throw GpuError(SDBG_EINVAL, "clause_sizes / clause_negated / clause_group_sizes need phrase_positions");
    return;
  }
  if (sizes.empty() && !negated.empty()) throw GpuError(SDBG_EINVAL, "clause_negated needs clause_sizes");
  const std::vector<uint32_t> one{uint32_t(n_terms)};
  const std::vector<uint32_t>& sz = sizes.empty() ? one : sizes;
  if (!negated.empty() && negated.size() != sz.size()) throw GpuError(SDBG_EINVAL, "one clause_negated entry per clause");
  off.assign(1, 0u);
  for (uint32_t x : sz) off.push_back(off.back() + x);
  if (off.back() != n_terms) throw GpuError(SDBG_EINVAL, "clause_sizes must cover the terms");
  neg.assign(sz.size(), 0u);
  for (size_t j = 0; j < negated.size(); ++j) neg[j] = negated[j] ? 1u : 0u;
  goff.assign(1, 0u);
  if (group_sizes.empty())
    for (size_t j = 0; j < sz.size(); ++j) goff.push_back(goff.back() + 1u);
  for (uint32_t x : group_sizes) {
    if (x == 0) throw GpuError(SDBG_EINVAL, "an empty OR group");
    goff.push_back(goff.back() + x);
  }
  if (goff.back() != sz.size()) throw GpuError(SDBG_EINVAL, "clause_group_sizes must cover the clauses");
  gneg.assign(goff.size() - 1, 0u);
  for (size_t g = 0; g + 1 < goff.size(); ++g) {
    gneg[g] = neg[goff[g]];
    for (uint32_t j = goff[g]; j < goff[g + 1]; ++j)
      if (neg[j] != gneg[g]) throw GpuError(SDBG_EINVAL, "the clauses of an OR group share their clause_negated flag");
  }
}

// The statistics of a phrase (collectors.cpp:116-128): the slots' idfs summed in float32 in slot order, a repeated term
// once per slot; the first slot's norm constants and boost (the field's, shared by every slot).
sdbg_bm25_term phrase_stats(const std::vector<sdbg_bm25_term>& slots) {
  sdbg_bm25_term s = slots[0];
  float idf = 0.f;
  for (const sdbg_bm25_term& t : slots) idf += t.idf;
  s.idf = idf;
  return s;
}

// One statistics entry per clause: the phrase statistics of its slots (a one-slot clause: its term's own); negated
// clauses never score and get zeros.
std::vector<sdbg_bm25_term> clause_stats(const std::vector<sdbg_bm25_term>& terms, const std::vector<uint32_t>& off,
                                         const std::vector<uint8_t>& neg) {
  std::vector<sdbg_bm25_term> out(neg.size(), sdbg_bm25_term{});
  for (size_t j = 0; j < neg.size(); ++j)
    if (!neg[j]) out[j] = phrase_stats(std::vector<sdbg_bm25_term>(terms.begin() + off[j], terms.begin() + off[j + 1]));
  return out;
}

std::vector<uint32_t> term_ids(const std::vector<sdbg_bm25_term>& terms) {
  std::vector<uint32_t> ids(terms.size());
  for (size_t i = 0; i < ids.size(); ++i) ids[i] = terms[i].term;
  return ids;
}
}  // namespace

FilterChain::FilterChain(const sdbg_col_pred* table_filter) {
  // a 4th entry that still carries the bit is kept: the library refuses the chain (SDBG_EUNSUPPORTED)
  for (const sdbg_col_pred* f = table_filter; f; f = (f->op & SDBG_OP_AND_NEXT) && preds.size() < 4 ? f + 1 : nullptr)
    preds.push_back(*f);
}

GpuTopKIterator::GpuTopKIterator(sdbg_segment* segment, int kind, std::vector<sdbg_bm25_term> terms, float k1, float b,
                                 uint32_t k, const sdbg_col_pred* table_filter, std::vector<uint32_t> excluded_terms,
                                 std::vector<uint32_t> group_sizes, std::vector<uint32_t> group_min_match,
                                 std::vector<uint32_t> phrase_positions,
    std::vector<uint32_t> clause_sizes, std::vector<uint8_t> clause_negated,
    std::vector<uint32_t> clause_group_sizes)
    : seg_(segment), kind_(kind), terms_(std::move(terms)), excluded_(std::move(excluded_terms)), groups_(std::move(group_sizes)),
      group_min_(std::move(group_min_match)), phrase_(std::move(phrase_positions)), k1_(k1), b_(b), k_(k), filter_(table_filter) {
  threshold_.value = FLT_MIN;  // doc_collector.hpp:102
  check_phrase(phrase_, terms_.size(), !groups_.empty());
  phrase_clauses(phrase_, terms_.size(), clause_sizes, clause_negated, clause_group_sizes, clause_off_, clause_neg_,
                 group_off_, group_neg_);
  if (!phrase_.empty()) phrase_minimums(group_min_, group_neg_);
  if (!phrase_.empty() && k_ == 0) throw GpuError(SDBG_EUNSUPPORTED, "phrases need k > 0: the streaming scan has no phrase form");
  // the streaming scan (sdbg_bm25_scan*) has no grouped form
  if (!groups_.empty() && k_ == 0) throw GpuError(SDBG_EUNSUPPORTED, "OR groups need k > 0: the streaming scan has no grouped form");
}

void GpuTopKIterator::run() {
  if (ran_) return;
  if (k_ == 0) {                   // streaming mode: every match, already in doc order
    uint64_t n = 0, cap = 0;
    std::vector<uint32_t> docs;
    std::vector<float> scores;
    for (;;) {
      const sdbg_col_pred* f = filter_.data();
      const int rc = excluded_.empty()
                         ? sdbg_bm25_scan(seg_, kind_, terms_.data(), terms_.size(), k1_, b_, f, 1, UINT32_MAX, docs.data(), scores.data(), cap, &n)
                         : sdbg_bm25_scan_excl(seg_, kind_, terms_.data(), terms_.size(), excluded_.data(), excluded_.size(), k1_, b_, f, 1,
                                               UINT32_MAX, docs.data(), scores.data(), cap, &n);
      if (rc == SDBG_ECAPACITY && n > cap) { cap = n; docs.resize(n); scores.resize(n); continue; }   // count-only call, then one with room
      check(rc, excluded_.empty() ? "sdbg_bm25_scan" : "sdbg_bm25_scan_excl");
      break;
    }
    by_doc_.resize(n);
    for (uint64_t i = 0; i < n; ++i) by_doc_[i] = sdbg_hit{scores[i], docs[i], 0};
    total_ = n;
    cost_.reset(total_);
    ran_ = true;
    return;
  }
  hits_.assign(k_, sdbg_hit{});
  uint32_t n = 0;
  float thr_out = 0;
  sdbg_segment* segs[1] = {seg_};
  if (!phrase_.empty()) {
    const std::vector<uint32_t> ids = term_ids(terms_);
    const std::vector<sdbg_bm25_term> stats = clause_stats(terms_, clause_off_, clause_neg_);
    const uint32_t query_group_off[2] = {0, uint32_t(group_neg_.size())}, excl_off[2] = {0, uint32_t(excluded_.size())};
    check(sdbg_phrase_groups_topk_batch_min(segs, 1, ids.data(), phrase_.data(), clause_off_.data(), group_off_.data(),
                                            group_neg_.data(), phrase_minimums(group_min_, group_neg_), query_group_off, 1,
                                            excluded_.data(), excl_off, stats.data(), k1_, b_, filter_.data(), k_, threshold_.value,
                                            hits_.data(), &n, &total_),
          "sdbg_phrase_groups_topk_batch_min");
    thr_out = n == k_ ? hits_[k_ - 1].score : threshold_.value;
  } else if (!groups_.empty()) {
    const std::vector<uint32_t> group_off = group_offsets(groups_, terms_.size());
    const uint32_t query_group_off[2] = {0, uint32_t(groups_.size())}, excl_off[2] = {0, uint32_t(excluded_.size())};
    check(sdbg_bm25_topk_batch_groups_min(segs, 1, terms_.data(), group_off.data(), query_group_off,
                                          group_minimums(group_min_, groups_.size()), 1, excluded_.data(), excl_off, k1_, b_,
                                          filter_.data(), k_, threshold_.value, hits_.data(), &n, &total_),
          "sdbg_bm25_topk_batch_groups_min");
    thr_out = n == k_ ? hits_[k_ - 1].score : threshold_.value;
  } else if (excluded_.empty()) {
    check(sdbg_bm25_topk(segs, 1, kind_, terms_.data(), terms_.size(), k1_, b_, filter_.data(), k_,
                         threshold_.value, hits_.data(), &n, &total_, &thr_out),
          "sdbg_bm25_topk");
  } else {
    const uint32_t term_off[2] = {0, uint32_t(terms_.size())}, excl_off[2] = {0, uint32_t(excluded_.size())};
    check(sdbg_bm25_topk_batch_excl(segs, 1, kind_, terms_.data(), term_off, 1, excluded_.data(), excl_off, k1_, b_,
                                    filter_.data(), k_, threshold_.value, hits_.data(), &n, &total_),
          "sdbg_bm25_topk_batch_excl");
    thr_out = n == k_ ? hits_[k_ - 1].score : threshold_.value;   // as sdbg_bm25_topk derives it
  }
  hits_.resize(n);
  by_doc_ = hits_;
  std::sort(by_doc_.begin(), by_doc_.end(), [](const sdbg_hit& a, const sdbg_hit& b) { return a.doc < b.doc; });
  if (n == k_ && thr_out > threshold_.value) threshold_.value = thr_out;  // raise the caller-visible threshold
  cost_.reset(total_);
  ran_ = true;
}

void GpuTopKIterator::Collect(const irs::ScoreFunction&, irs::ColumnArgsFetcher&, irs::ScoreCollector& collector) {
  run();
  if (k_ == 0) hits_ = by_doc_;    // a streaming iterator asked to Collect feeds everything it has
  if (hits_.empty()) { _doc = irs::doc_limits::eof(); return; }
  std::vector<irs::doc_id_t> docs(hits_.size());
  std::vector<irs::score_t> scores(hits_.size());
  for (size_t i = 0; i < hits_.size(); ++i) { docs[i] = hits_[i].doc; scores[i] = hits_[i].score; }
  collector.AddDocs(docs.data(), docs.size(), scores.data());  // iterators.hpp:176-207
  _doc = irs::doc_limits::eof();
}

uint32_t GpuTopKIterator::EmitScoredDocs(irs::doc_id_t* out, irs::score_t* scores, irs::doc_id_t max, const irs::ScoreFunction&,
                                         irs::ColumnArgsFetcher*, irs::doc_id_t min) {
  run();
  uint32_t n = 0;
  while (pos_ < by_doc_.size() && by_doc_[pos_].doc < min) ++pos_;
  while (pos_ < by_doc_.size() && by_doc_[pos_].doc < max) { out[n] = by_doc_[pos_].doc; scores[n] = by_doc_[pos_].score; ++n; ++pos_; }
  _doc = pos_ < by_doc_.size() ? by_doc_[pos_].doc : irs::doc_limits::eof();
  return n;
}

uint32_t GpuTopKIterator::EmitDocs(irs::doc_id_t* out, irs::doc_id_t min, irs::doc_id_t max) {
  run();
  uint32_t n = 0;
  while (pos_ < by_doc_.size() && by_doc_[pos_].doc < min) ++pos_;
  while (pos_ < by_doc_.size() && by_doc_[pos_].doc < max) out[n++] = by_doc_[pos_++].doc;
  _doc = pos_ < by_doc_.size() ? by_doc_[pos_].doc : irs::doc_limits::eof();
  return n;
}

uint32_t GpuTopKIterator::count() { run(); return uint32_t(total_); }

irs::Attribute* GpuTopKIterator::GetMutable(irs::TypeInfo::type_id type) noexcept {
  if (type == irs::Type<irs::ScoreThresholdAttr>::id()) return &threshold_;
  if (type == irs::Type<irs::CostAttr>::id()) return &cost_;
  return nullptr;
}

std::pair<irs::doc_id_t, bool> GpuTopKIterator::FillBlock(irs::doc_id_t min, irs::doc_id_t max, uint64_t* mask,
                                                          irs::FillBlockScoreContext score, irs::FillBlockMatchContext match) {
  run();
  bool empty = true;
  while (pos_ < by_doc_.size() && by_doc_[pos_].doc < min) ++pos_;
  for (; pos_ < by_doc_.size() && by_doc_[pos_].doc < max; ++pos_) {
    const uint32_t off = by_doc_[pos_].doc - min;
    bool set = true;
    if (match.matches) set = ++match.matches[off] >= match.min_match_count;   // TrackMatch: bit only when the threshold is met
    if (set) { mask[off >> 6] |= uint64_t(1) << (off & 63); empty = false; }
    if (score.score_window) {
      irs::score_t& w = score.score_window[off];
      switch (score.merge_type) {
        case irs::ScoreMergeType::Sum: w += by_doc_[pos_].score; break;
        case irs::ScoreMergeType::Max: w = std::max(w, by_doc_[pos_].score); break;
        default: w = by_doc_[pos_].score; break;
      }
    }
  }
  _doc = pos_ < by_doc_.size() ? by_doc_[pos_].doc : irs::doc_limits::eof();
  return {_doc, match.matches ? empty : false};
}

irs::doc_id_t GpuTopKIterator::advance() {
  run();
  if (_doc != irs::doc_limits::invalid() && pos_ < by_doc_.size() && by_doc_[pos_].doc == _doc) ++pos_;
  return _doc = pos_ < by_doc_.size() ? by_doc_[pos_].doc : irs::doc_limits::eof();
}

irs::doc_id_t GpuTopKIterator::seek(irs::doc_id_t target) {
  run();
  while (pos_ < by_doc_.size() && by_doc_[pos_].doc < target) ++pos_;
  return _doc = pos_ < by_doc_.size() ? by_doc_[pos_].doc : irs::doc_limits::eof();
}

GpuAggScan::GpuAggScan(std::vector<sdbg_segment*> segments, std::vector<sdbg_col_pred> pushed_filters, uint64_t key_field,
                       uint64_t sum_int_field, uint64_t avg_f64_field, uint32_t n_groups_hint)
    : segs_(std::move(segments)), preds_(std::move(pushed_filters)), key_(key_field), sum_i_(sum_int_field),
      avg_f_(avg_f64_field), hint_(n_groups_hint) {}

void GpuAggScan::Scan(duckdb::DataChunkMock& output) {
  output.Reset();
  if (!ran_) {
    uint64_t cap = std::max<uint64_t>(hint_, 1024), n = 0;
    for (;;) {
      groups_.resize(cap);
      const int rc = sdbg_filter_groupby(segs_.data(), segs_.size(), preds_.data(), preds_.size(), key_, hint_, sum_i_, avg_f_,
                                         groups_.data(), cap, &n);
      if (rc == SDBG_ECAPACITY && n > cap) { cap = n; continue; }  // the call reports how many groups exist: one retry with room for them
      if (rc != SDBG_OK) throw GpuError(rc, std::string("sdbg_filter_groupby: ") + sdbg_last_error(sdbg_segment_context(segs_[0])));
      break;
    }
    groups_.resize(n);
    for (const auto& g : groups_) rows_scanned_ += g.count;
    ran_ = true;
  }
  const size_t take = std::min<size_t>(duckdb::STANDARD_VECTOR_SIZE, groups_.size() - cursor_);
  for (size_t i = 0; i < take; ++i) {
    const sdbg_group_row& g = groups_[cursor_ + i];
    output.key.push_back(g.key);
    output.count.push_back(int64_t(g.count));
    output.sum_lo.push_back(g.sum_i128[0]);
    output.sum_hi.push_back(g.sum_i128[1]);
    output.avg.push_back(g.cnt_f64 ? g.sum_f64 / double(g.cnt_f64) : 0.0);
  }
  output.size = take;
  cursor_ += take;
}

GpuCountScan::GpuCountScan(std::vector<sdbg_segment*> segments, int kind, std::vector<uint32_t> terms,
                           std::vector<uint32_t> excluded_terms, const sdbg_col_pred* table_filter, std::vector<uint32_t> group_sizes,
                           std::vector<uint32_t> group_min_match, std::vector<uint32_t> phrase_positions,
    std::vector<uint32_t> clause_sizes, std::vector<uint8_t> clause_negated,
    std::vector<uint32_t> clause_group_sizes)
    : segs_(std::move(segments)), kind_(kind), terms_(std::move(terms)), excluded_(std::move(excluded_terms)),
      groups_(std::move(group_sizes)), group_min_(std::move(group_min_match)), phrase_(std::move(phrase_positions)),
      filter_(table_filter) {
  check_phrase(phrase_, terms_.size(), !groups_.empty());
  phrase_clauses(phrase_, terms_.size(), clause_sizes, clause_negated, clause_group_sizes, clause_off_, clause_neg_,
                 group_off_, group_neg_);
  if (!phrase_.empty()) phrase_minimums(group_min_, group_neg_);
}

void GpuCountScan::Scan(duckdb::DataChunkMock& output) {
  output.Reset();
  if (done_) return;                                          // cardinality 0: the count has been emitted
  const uint32_t term_off[2] = {0, uint32_t(terms_.size())};
  const uint32_t excl_off[2] = {0, uint32_t(excluded_.size())};
  uint64_t n = 0;
  int rc;
  const char* what;
  if (!phrase_.empty()) {
    const uint32_t query_group_off[2] = {0, uint32_t(group_neg_.size())};
    rc = sdbg_phrase_groups_count_batch_min(segs_.data(), segs_.size(), terms_.data(), phrase_.data(), clause_off_.data(),
                                            group_off_.data(), group_neg_.data(), phrase_minimums(group_min_, group_neg_),
                                            query_group_off, 1, excluded_.data(), excl_off, filter_.data(), &n);
    what = "sdbg_phrase_groups_count_batch_min: ";
  } else if (groups_.empty()) {
    rc = sdbg_match_count_batch(segs_.data(), segs_.size(), kind_, terms_.data(), term_off, 1, excluded_.data(), excl_off,
                                filter_.data(), &n);
    what = "sdbg_match_count_batch: ";
  } else {                                                    // an And of Ors: kind_ is not used
    const std::vector<uint32_t> group_off = group_offsets(groups_, terms_.size());
    const uint32_t query_group_off[2] = {0, uint32_t(groups_.size())};
    rc = sdbg_match_count_batch_groups_min(segs_.data(), segs_.size(), terms_.data(), group_off.data(), query_group_off,
                                           group_minimums(group_min_, groups_.size()), 1, excluded_.data(), excl_off,
                                           filter_.data(), &n);
    what = "sdbg_match_count_batch_groups_min: ";
  }
  if (rc != SDBG_OK) throw GpuError(rc, std::string(what) + sdbg_last_error(sdbg_segment_context(segs_[0])));
  output.count.push_back(int64_t(n));
  output.size = 1;
  done_ = true;
}

GpuSortedScan::GpuSortedScan(std::vector<sdbg_segment*> segments, int kind, std::vector<uint32_t> terms,
                             std::vector<uint32_t> excluded_terms, const sdbg_col_pred* table_filter, uint64_t sort_field,
                             bool descending, bool nulls_first, uint32_t k, std::vector<uint32_t> group_sizes,
                             std::vector<uint32_t> group_min_match, std::vector<uint32_t> phrase_positions,
    std::vector<uint32_t> clause_sizes, std::vector<uint8_t> clause_negated,
    std::vector<uint32_t> clause_group_sizes)
    : segs_(std::move(segments)), kind_(kind), terms_(std::move(terms)), excluded_(std::move(excluded_terms)),
      group_sizes_(std::move(group_sizes)), group_min_(std::move(group_min_match)), phrase_(std::move(phrase_positions)),
      filter_(table_filter), field_(sort_field), desc_(descending), nulls_first_(nulls_first), k_(k) {
  check_phrase(phrase_, terms_.size(), !group_sizes_.empty());
  phrase_clauses(phrase_, terms_.size(), clause_sizes, clause_negated, clause_group_sizes, clause_off_, clause_neg_,
                 group_off_, group_neg_);
  if (!phrase_.empty()) phrase_minimums(group_min_, group_neg_);
}

void GpuSortedScan::Scan(duckdb::DataChunkMock& output) {
  output.Reset();
  if (!ran_) {
    const uint32_t term_off[2] = {0, uint32_t(terms_.size())};
    const uint32_t excl_off[2] = {0, uint32_t(excluded_.size())};
    hits_.resize(k_);
    uint32_t n = 0;
    int rc;
    const char* what;
    if (!phrase_.empty()) {
      const uint32_t query_group_off[2] = {0, uint32_t(group_neg_.size())};
      rc = sdbg_phrase_groups_topk_by_column_batch_min(segs_.data(), segs_.size(), terms_.data(), phrase_.data(), clause_off_.data(),
                                                       group_off_.data(), group_neg_.data(), phrase_minimums(group_min_, group_neg_),
                                                       query_group_off, 1, excluded_.data(), excl_off, filter_.data(), field_,
                                                       desc_ ? 1 : 0, nulls_first_ ? 1 : 0, k_, hits_.data(), &n);
      what = "sdbg_phrase_groups_topk_by_column_batch_min: ";
    } else if (group_sizes_.empty()) {
      rc = sdbg_match_topk_by_column_batch(segs_.data(), segs_.size(), kind_, terms_.data(), term_off, 1, excluded_.data(), excl_off,
                                           filter_.data(), field_, desc_ ? 1 : 0, nulls_first_ ? 1 : 0, k_,
                                           hits_.data(), &n);
      what = "sdbg_match_topk_by_column_batch: ";
    } else {                                                  // an And of Ors: kind_ is not used
      const std::vector<uint32_t> group_off = group_offsets(group_sizes_, terms_.size());
      const uint32_t query_group_off[2] = {0, uint32_t(group_sizes_.size())};
      rc = sdbg_match_topk_by_column_batch_groups_min(segs_.data(), segs_.size(), terms_.data(), group_off.data(), query_group_off,
                                                      group_minimums(group_min_, group_sizes_.size()), 1, excluded_.data(),
                                                      excl_off, filter_.data(), field_, desc_ ? 1 : 0,
                                                      nulls_first_ ? 1 : 0, k_, hits_.data(), &n);
      what = "sdbg_match_topk_by_column_batch_groups_min: ";
    }
    if (rc != SDBG_OK) throw GpuError(rc, std::string(what) + sdbg_last_error(sdbg_segment_context(segs_[0])));
    hits_.resize(n);
    ran_ = true;
  }
  const size_t take = std::min<size_t>(duckdb::STANDARD_VECTOR_SIZE, hits_.size() - cursor_);   // 0: end of scan
  for (size_t i = 0; i < take; ++i) {
    const sdbg_sort_hit& h = hits_[cursor_ + i];
    output.doc.push_back(h.doc);
    output.segment.push_back(h.seg);
    output.value.push_back(h.value);
    output.valid.push_back(h.is_null ? 0 : 1);
  }
  output.size = take;
  cursor_ += take;
}

GpuMatchScan::GpuMatchScan(std::vector<sdbg_segment*> segments, std::vector<sdbg_bm25_term> terms,
                           std::vector<uint32_t> excluded_terms, const sdbg_col_pred* table_filter, float k1, float b, bool scored,
                           std::vector<uint32_t> group_sizes, std::vector<uint32_t> group_min_match,
                           std::vector<uint32_t> phrase_positions,
    std::vector<uint32_t> clause_sizes, std::vector<uint8_t> clause_negated,
    std::vector<uint32_t> clause_group_sizes)
    : segs_(std::move(segments)), terms_(std::move(terms)), excluded_(std::move(excluded_terms)),
      group_sizes_(group_sizes.empty() ? std::vector<uint32_t>{uint32_t(terms_.size())} : std::move(group_sizes)),
      group_min_(std::move(group_min_match)), phrase_(std::move(phrase_positions)), filter_(table_filter), k1_(k1), b_(b),
      scored_(scored) {
  check_phrase(phrase_, terms_.size(), group_sizes_.size() > 1);
  phrase_clauses(phrase_, terms_.size(), clause_sizes, clause_negated, clause_group_sizes, clause_off_, clause_neg_,
                 group_off_, group_neg_);
  if (!phrase_.empty()) phrase_minimums(group_min_, group_neg_);
}

void GpuMatchScan::Fetch() {   // the next page: matches offset_ .. offset_ + kPage - 1
  const std::vector<uint32_t> group_off = group_offsets(group_sizes_, terms_.size());
  const uint32_t query_group_off[2] = {0, uint32_t(group_sizes_.size())};
  const uint32_t excl_off[2] = {0, uint32_t(excluded_.size())};
  page_.resize(kPage);
  uint32_t n = 0;
  int rc;
  const char* what;
  if (!phrase_.empty()) {
    const std::vector<uint32_t> ids = term_ids(terms_);
    const std::vector<sdbg_bm25_term> stats = clause_stats(terms_, clause_off_, clause_neg_);
    const uint32_t query_group_off[2] = {0, uint32_t(group_neg_.size())};
    rc = sdbg_phrase_groups_scan_batch_min(segs_.data(), segs_.size(), ids.data(), phrase_.data(), clause_off_.data(),
                                           group_off_.data(), group_neg_.data(), phrase_minimums(group_min_, group_neg_),
                                           query_group_off, 1, excluded_.data(), excl_off, filter_.data(),
                                           scored_ ? stats.data() : nullptr, k1_, b_, &offset_, kPage, scored_ ? 1 : 0,
                                           page_.data(), &n, &total_);
    what = "sdbg_phrase_groups_scan_batch_min: ";
  } else {
    rc = sdbg_match_scan_batch_groups_min(segs_.data(), segs_.size(), terms_.data(), group_off.data(), query_group_off,
                                          group_minimums(group_min_, group_sizes_.size()), 1, excluded_.data(), excl_off,
                                          k1_, b_, filter_.data(), &offset_, kPage, scored_ ? 1 : 0, page_.data(), &n, &total_);
    what = "sdbg_match_scan_batch_groups_min: ";
  }
  if (rc != SDBG_OK) throw GpuError(rc, std::string(what) + sdbg_last_error(sdbg_segment_context(segs_[0])));
  page_.resize(n);
  offset_ += kPage;
  cursor_ = 0;
  ran_ = true;
}

void GpuMatchScan::Scan(duckdb::DataChunkMock& output) {
  output.Reset();
  if (!ran_ || (cursor_ == page_.size() && page_.size() == kPage && offset_ < total_)) Fetch();
  const size_t take = std::min<size_t>(duckdb::STANDARD_VECTOR_SIZE, page_.size() - cursor_);   // 0: end of scan
  for (size_t i = 0; i < take; ++i) {
    const sdbg_hit& h = page_[cursor_ + i];
    output.doc.push_back(h.doc);
    output.segment.push_back(h.seg);
    output.score.push_back(h.score);
  }
  output.size = take;
  cursor_ += take;
}

GpuFacetScan::GpuFacetScan(std::vector<sdbg_segment*> segments, int kind, std::vector<uint32_t> terms,
                           std::vector<uint32_t> excluded_terms, const sdbg_col_pred* table_filter, uint64_t key_field,
                           std::vector<uint32_t> group_sizes, std::vector<uint32_t> group_min_match,
                           std::vector<uint32_t> phrase_positions,
    std::vector<uint32_t> clause_sizes, std::vector<uint8_t> clause_negated,
    std::vector<uint32_t> clause_group_sizes)
    : segs_(std::move(segments)), kind_(kind), terms_(std::move(terms)), excluded_(std::move(excluded_terms)),
      group_sizes_(std::move(group_sizes)), group_min_(std::move(group_min_match)), phrase_(std::move(phrase_positions)),
      filter_(table_filter), field_(key_field) {
  check_phrase(phrase_, terms_.size(), !group_sizes_.empty());
  phrase_clauses(phrase_, terms_.size(), clause_sizes, clause_negated, clause_group_sizes, clause_off_, clause_neg_,
                 group_off_, group_neg_);
  if (!phrase_.empty()) phrase_minimums(group_min_, group_neg_);
}

void GpuFacetScan::Scan(duckdb::DataChunkMock& output) {
  output.Reset();
  if (!ran_) {
    sdbg_ctx* ctx = sdbg_segment_context(segs_[0]);
    int64_t lo = INT64_MAX, hi = INT64_MIN;
    for (sdbg_segment* s : segs_) {
      int64_t mn = 0, mx = 0;
      const int rc = sdbg_column_minmax_i64(s, field_, &mn, &mx);
      if (rc != SDBG_OK) throw GpuError(rc, std::string("sdbg_column_minmax_i64: ") + sdbg_last_error(ctx));
      lo = std::min(lo, mn);
      hi = std::max(hi, mx);
    }
    if (lo > hi) lo = hi = 0;   // every key NULL: one (empty) bin, every match in the NULL group
    const uint64_t span = uint64_t(hi) - uint64_t(lo) + 1;
    if (span == 0 || span > 32768) throw GpuError(SDBG_EUNSUPPORTED, "GpuFacetScan: the key range spans more than 32768 values");
    const uint32_t term_off[2] = {0, uint32_t(terms_.size())};
    const uint32_t excl_off[2] = {0, uint32_t(excluded_.size())};
    std::vector<uint64_t> counts(span);
    int rc;
    const char* what;
    if (!phrase_.empty()) {
      const uint32_t query_group_off[2] = {0, uint32_t(group_neg_.size())};
      rc = sdbg_phrase_groups_facet_counts_batch_min(segs_.data(), segs_.size(), terms_.data(), phrase_.data(), clause_off_.data(),
                                                     group_off_.data(), group_neg_.data(), phrase_minimums(group_min_, group_neg_),
                                                     query_group_off, 1, excluded_.data(), excl_off, filter_.data(), field_, lo,
                                                     uint32_t(span), counts.data(), &nulls_);
      what = "sdbg_phrase_groups_facet_counts_batch_min: ";
    } else if (group_sizes_.empty()) {
      rc = sdbg_match_facet_counts_batch(segs_.data(), segs_.size(), kind_, terms_.data(), term_off, 1, excluded_.data(), excl_off,
                                         filter_.data(), field_, lo, uint32_t(span), counts.data(), &nulls_);
      what = "sdbg_match_facet_counts_batch: ";
    } else {                                                  // an And of Ors: kind_ is not used
      const std::vector<uint32_t> group_off = group_offsets(group_sizes_, terms_.size());
      const uint32_t query_group_off[2] = {0, uint32_t(group_sizes_.size())};
      rc = sdbg_match_facet_counts_batch_groups_min(segs_.data(), segs_.size(), terms_.data(), group_off.data(), query_group_off,
                                                    group_minimums(group_min_, group_sizes_.size()), 1, excluded_.data(),
                                                    excl_off, filter_.data(), field_, lo, uint32_t(span),
                                                    counts.data(), &nulls_);
      what = "sdbg_match_facet_counts_batch_groups_min: ";
    }
    if (rc != SDBG_OK) throw GpuError(rc, std::string(what) + sdbg_last_error(ctx));
    for (uint64_t i = 0; i < span; ++i)
      if (counts[i]) groups_.emplace_back(int64_t(uint64_t(lo) + i), counts[i]);
    ran_ = true;
  }
  const size_t rows = groups_.size() + (nulls_ ? 1 : 0);
  const size_t take = std::min<size_t>(duckdb::STANDARD_VECTOR_SIZE, rows - cursor_);   // 0: end of scan
  for (size_t i = cursor_; i < cursor_ + take; ++i) {
    const bool null_group = i == groups_.size();
    output.key.push_back(null_group ? 0 : groups_[i].first);
    output.count.push_back(int64_t(null_group ? nulls_ : groups_[i].second));
    output.valid.push_back(null_group ? 0 : 1);
  }
  output.size = take;
  cursor_ += take;
}

GpuMatchAggScan::GpuMatchAggScan(std::vector<sdbg_segment*> segments, int kind, std::vector<uint32_t> terms,
                                 std::vector<uint32_t> excluded_terms, const sdbg_col_pred* table_filter, uint64_t key_field,
                                 uint64_t value_field, sdbg_type value_type, std::vector<uint32_t> group_sizes,
                                 std::vector<uint32_t> group_min_match, std::vector<uint32_t> phrase_positions,
    std::vector<uint32_t> clause_sizes, std::vector<uint8_t> clause_negated,
    std::vector<uint32_t> clause_group_sizes)
    : segs_(std::move(segments)), kind_(kind), terms_(std::move(terms)), excluded_(std::move(excluded_terms)),
      group_sizes_(std::move(group_sizes)), group_min_(std::move(group_min_match)), phrase_(std::move(phrase_positions)),
      filter_(table_filter), key_field_(key_field), value_field_(value_field), value_type_(value_type) {
  check_phrase(phrase_, terms_.size(), !group_sizes_.empty());
  phrase_clauses(phrase_, terms_.size(), clause_sizes, clause_negated, clause_group_sizes, clause_off_, clause_neg_,
                 group_off_, group_neg_);
  if (!phrase_.empty()) phrase_minimums(group_min_, group_neg_);
}

void GpuMatchAggScan::Scan(duckdb::DataChunkMock& output) {
  output.Reset();
  if (!ran_) {
    sdbg_ctx* ctx = sdbg_segment_context(segs_[0]);
    const bool grouped = key_field_ != UINT64_MAX;
    int64_t lo = 0;
    uint64_t span = 1;
    if (grouped) {
      int64_t mn_all = INT64_MAX, mx_all = INT64_MIN;
      for (sdbg_segment* s : segs_) {
        int64_t mn = 0, mx = 0;
        const int rc = sdbg_column_minmax_i64(s, key_field_, &mn, &mx);
        if (rc != SDBG_OK) throw GpuError(rc, std::string("sdbg_column_minmax_i64: ") + sdbg_last_error(ctx));
        mn_all = std::min(mn_all, mn);
        mx_all = std::max(mx_all, mx);
      }
      if (mn_all > mx_all) mn_all = mx_all = 0;   // every key NULL: one (empty) group, every match in the NULL group
      lo = mn_all;
      span = uint64_t(mx_all) - uint64_t(mn_all) + 1;
      if (span == 0 || span > 4096) throw GpuError(SDBG_EUNSUPPORTED, "GpuMatchAggScan: the key range spans more than 4096 values");
    }
    const uint32_t term_off[2] = {0, uint32_t(terms_.size())};
    const uint32_t excl_off[2] = {0, uint32_t(excluded_.size())};
    std::vector<sdbg_match_agg> cells(span);
    sdbg_match_agg null_cell{};
    int rc;
    const char* what;
    if (!phrase_.empty()) {
      const uint32_t query_group_off[2] = {0, uint32_t(group_neg_.size())};
      rc = sdbg_phrase_groups_aggregate_batch_min(segs_.data(), segs_.size(), terms_.data(), phrase_.data(), clause_off_.data(),
                                                  group_off_.data(), group_neg_.data(), phrase_minimums(group_min_, group_neg_),
                                                  query_group_off, 1, excluded_.data(), excl_off, filter_.data(), key_field_, lo,
                                                  uint32_t(span), value_field_, cells.data(), &null_cell);
      what = "sdbg_phrase_groups_aggregate_batch_min: ";
    } else if (group_sizes_.empty()) {
      rc = sdbg_match_aggregate_batch(segs_.data(), segs_.size(), kind_, terms_.data(), term_off, 1, excluded_.data(), excl_off,
                                      filter_.data(), key_field_, lo, uint32_t(span), value_field_, cells.data(),
                                      &null_cell);
      what = "sdbg_match_aggregate_batch: ";
    } else {                                                  // an And of Ors: kind_ is not used
      const std::vector<uint32_t> group_off = group_offsets(group_sizes_, terms_.size());
      const uint32_t query_group_off[2] = {0, uint32_t(group_sizes_.size())};
      rc = sdbg_match_aggregate_batch_groups_min(segs_.data(), segs_.size(), terms_.data(), group_off.data(), query_group_off,
                                                 group_minimums(group_min_, group_sizes_.size()), 1, excluded_.data(), excl_off,
                                                 filter_.data(), key_field_, lo, uint32_t(span), value_field_,
                                                 cells.data(), &null_cell);
      what = "sdbg_match_aggregate_batch_groups_min: ";
    }
    if (rc != SDBG_OK) throw GpuError(rc, std::string(what) + sdbg_last_error(ctx));
    for (uint64_t i = 0; i < span; ++i)
      if (cells[i].count || !grouped) groups_.emplace_back(int64_t(uint64_t(lo) + i), cells[i]);   // ungrouped: always one row
    if (grouped && null_cell.count) { groups_.emplace_back(0, null_cell); null_row_ = true; }
    ran_ = true;
  }
  const size_t take = std::min<size_t>(duckdb::STANDARD_VECTOR_SIZE, groups_.size() - cursor_);   // 0: end of scan
  for (size_t i = cursor_; i < cursor_ + take; ++i) {
    const sdbg_match_agg& a = groups_[i].second;
    const bool null_group = null_row_ && i + 1 == groups_.size();
    const __int128 sum = (static_cast<__int128>(a.sum_i128[1]) << 64) | static_cast<unsigned long long>(a.sum_i128[0]);
    output.key.push_back(null_group || key_field_ == UINT64_MAX ? 0 : groups_[i].first);
    output.valid.push_back(null_group ? 0 : 1);
    output.count.push_back(int64_t(a.count));
    output.count_value.push_back(int64_t(a.count_value));
    output.sum_lo.push_back(a.sum_i128[0]);
    output.sum_hi.push_back(a.sum_i128[1]);
    output.sum_f64.push_back(a.sum_f64);
    output.avg.push_back(!a.count_value ? 0.0 : (value_type_ == SDBG_F64 ? a.sum_f64 : double(sum)) / double(a.count_value));
    output.min.push_back(a.min);
    output.max.push_back(a.max);
  }
  output.size = take;
  cursor_ += take;
}

GpuAggGlobalState::GpuAggGlobalState(std::vector<sdbg_segment*> segments, std::vector<sdbg_col_pred> pushed_filters, uint64_t key_field,
                                     uint64_t sum_int_field, uint64_t avg_f64_field, uint32_t n_groups_hint)
    : segs(std::move(segments)), preds(std::move(pushed_filters)), key(key_field), sum_i(sum_int_field), avg_f(avg_f64_field),
      hint(n_groups_hint) {}

void GpuAggScanFunction(GpuAggGlobalState& g, GpuAggLocalState& l, duckdb::DataChunkMock& output) {
  output.Reset();
  std::call_once(g.ran, [&] {                 // an exception here leaves the flag unset: the next worker retries and rethrows
    uint64_t cap = std::max<uint64_t>(g.hint, 1024), n = 0;
    std::vector<sdbg_group_row> rows;
    for (;;) {
      rows.resize(cap);
      const int rc = sdbg_filter_groupby(g.segs.data(), g.segs.size(), g.preds.data(), g.preds.size(), g.key, g.hint, g.sum_i, g.avg_f,
                                         rows.data(), cap, &n);
      if (rc == SDBG_ECAPACITY && n > cap) { cap = n; continue; }
      if (rc != SDBG_OK) throw GpuError(rc, std::string("sdbg_filter_groupby: ") + sdbg_last_error(sdbg_segment_context(g.segs[0])));
      break;
    }
    rows.resize(n);
    g.groups = std::move(rows);
  });
  const size_t chunk = g.next_chunk.fetch_add(1, std::memory_order_relaxed);
  const size_t first = chunk * size_t(duckdb::STANDARD_VECTOR_SIZE);
  if (first >= g.groups.size()) return;                      // cardinality 0
  const size_t take = std::min<size_t>(duckdb::STANDARD_VECTOR_SIZE, g.groups.size() - first);
  for (size_t i = 0; i < take; ++i) {
    const sdbg_group_row& r = g.groups[first + i];
    output.key.push_back(r.key);
    output.count.push_back(int64_t(r.count));
    output.sum_lo.push_back(r.sum_i128[0]);
    output.sum_hi.push_back(r.sum_i128[1]);
    output.avg.push_back(r.cnt_f64 ? r.sum_f64 / double(r.cnt_f64) : 0.0);
  }
  output.size = take;
  ++l.chunks_claimed;
  g.rows_emitted.fetch_add(take, std::memory_order_relaxed);
}

}  // namespace sdbg_host
