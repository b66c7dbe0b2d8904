// adapter_selftest.cpp -- drives the two adapters the way the reference's callers would
// (ExecuteTopK's collector loop, IResearchScanFunction's chunk loop) and prints results as JSON lines
// for tests/test_gpu_adapters.py to compare with the oracle. Needs a GPU at run time. With a second argument "excl" it runs
// only the exclusion case instead (an And with a Not child, tests/test_gpu_exclusion.py); with "count", only the Count
// scan mode (GpuCountScan, tests/test_gpu_count.py); with "groups", only an And of Or groups through both adapters
// (tests/test_gpu_groups.py); with "minmatch", only an Or with min_match_count through both adapters
// (tests/test_gpu_min_match.py); with "sorted", only the sorted scan (GpuSortedScan, tests/test_gpu_sort_by_column.py); with
// "facet", only the facet counts (GpuFacetScan, tests/test_gpu_facets.py). "sorted groups" / "facet groups" run those two
// with group queries (tests/test_gpu_groups_column.py). "aggregate" / "aggregate groups" run the aggregates over the matches
// (GpuMatchAggScan, tests/test_gpu_match_aggregates.py). "chain" runs a pushed filter chain (SDBG_OP_AND_NEXT) through the
// top-k, streaming and count adapters next to the same calls filtered by an indicator column of the chain
// (tests/test_gpu_filter_chains.py). "scan" runs the Stream mode (GpuMatchScan) for flat, grouped and min-match queries
// (tests/test_gpu_match_scan.py). "phrase" runs a phrase through the top-k and count adapters on a token corpus of its own
// (tests/test_gpu_phrase.py); "phrase columns" runs the same phrases through the sorted, facet, aggregate and Stream
// adapters instead (tests/test_gpu_phrase_column.py); "phrase and" runs conjunctions of phrases, terms and negated phrases
// (clause_sizes / clause_negated) through all six phrase adapters (tests/test_gpu_phrase_and.py); "phrase groups" runs
// conjunctions of OR groups of phrases and terms (clause_group_sizes too) through them (tests/test_gpu_phrase_groups.py);
// "phrase min" runs OR groups of phrases and terms with minimum match counts (group_min_match per clause group) through
// them (tests/test_gpu_phrase_min_match.py).
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <thread>
#include <vector>

#include "gpu_adapters.hpp"

namespace {
struct ListCollector final : irs::ScoreCollector {  // a trivial ScoreCollector: keeps what it is fed
  ListCollector() : irs::ScoreCollector(Tag::Generic) {}
  std::vector<irs::ScoreDoc> docs;
  void Add(irs::score_t s, irs::doc_id_t d) override { docs.push_back({s, d, 0}); }
  void AddWindow(const irs::score_t*, const uint64_t*, irs::doc_id_t, size_t, bool) override {}
  void AddDocs(const irs::doc_id_t* d, size_t n, const irs::score_t* s) override { for (size_t i = 0; i < n; ++i) docs.push_back({s[i], d[i], 0}); }
};
// "phrase": a by_phrase through GpuTopKIterator (top-50) and GpuCountScan on a token corpus of its own, which
// tests/test_gpu_phrase.py rebuilds: doc i (1-based) has 1 + r % 16 tokens, each token r % 6, r the next value of
// r = r * 1664525 + 1013904223 (mod 2^32) >> 16 from state 12345, docs in order. Norms are the doc lengths. One line per
// phrase: its slots and positions, the excluded term, the hits, total_matches and the count.
// With `columns`, the int64 column 20 holds (d * 7919) % 23 - 11 for doc d, NULL when d % 5 == 0, and each line holds
// instead: GpuSortedScan ORDER BY column 20 DESC NULLS LAST LIMIT 30 (docs, values, valid), GpuFacetScan GROUP BY column 20
// (keys, counts, valid), GpuMatchAggScan of column 20 without GROUP BY (count, count_value, sum_lo, min, max), and the
// scored GpuMatchScan (docs, scores, total).
// With `clauses` ("phrase and"), the column is staged too and each case is an And of clauses (clause_sizes over the
// slots, clause_negated); each line holds its slots, positions, sizes, negations and excluded terms, then the top-50
// (GpuTopKIterator), total and count (GpuCountScan), the sorted docs, the facet keys and counts, the aggregate count
// and the scored scan's docs, scores and total, as above. With `groups` ("phrase groups") the cases are And of OR groups of
// clauses (clause_group_sizes), and each line also holds the group sizes ("gsizes"). With `mins` ("phrase min") the cases
// are And of OR groups with minimum match counts (group_min_match), and each line also holds them ("gmin").
int phrase_mode(sdbg_ctx* ctx, uint32_t n_docs, bool columns, bool clauses, bool groups, bool mins) {
  uint32_t state = 12345u;
  auto next = [&]() { state = state * 1664525u + 1013904223u; return state >> 16; };
  constexpr uint32_t kVocab = 6;
  std::vector<std::vector<uint32_t>> docs(kVocab), freqs(kVocab), pos(kVocab);
  std::vector<uint32_t> norms(n_docs);
  uint64_t sum_len = 0;
  for (uint32_t d = 1; d <= n_docs; ++d) {
    const uint32_t len = 1 + next() % 16;
    norms[d - 1] = len;
    sum_len += len;
    std::vector<std::vector<uint32_t>> at(kVocab);
    for (uint32_t p = 0; p < len; ++p) at[next() % kVocab].push_back(p);
    for (uint32_t t = 0; t < kVocab; ++t) {
      if (at[t].empty()) continue;
      docs[t].push_back(d); freqs[t].push_back(uint32_t(at[t].size()));
      pos[t].insert(pos[t].end(), at[t].begin(), at[t].end());
    }
  }
  sdbg_writer* w = nullptr;
  sdbg_segment* seg = nullptr;
  const uint8_t* doc_file = nullptr; const sdbg_term_meta* metas = nullptr;
  size_t n_bytes = 0, n_terms = 0;
  int rc = sdbg_writer_create(n_docs, 1, 0.75f, norms.data(), &w);
  for (uint32_t t = 0; t < kVocab && !rc; ++t) rc = sdbg_writer_add_term(w, docs[t].data(), freqs[t].data(), uint32_t(docs[t].size()));
  if (!rc) rc = sdbg_writer_finish(w, &doc_file, &n_bytes, &metas, &n_terms);
  if (!rc) rc = sdbg_segment_create(ctx, n_docs, &seg);
  if (!rc) rc = sdbg_stage_postings(seg, doc_file, n_bytes, metas, n_terms, 1);
  std::vector<uint8_t> nb(norms.begin(), norms.end());
  const sdbg_norm_rg rg{1, n_docs, 0};
  if (!rc) rc = sdbg_stage_norms(seg, nb.data(), nb.size(), &rg, 1);
  std::vector<uint32_t> flat;
  std::vector<uint64_t> off(1, 0);
  for (uint32_t t = 0; t < kVocab; ++t) { flat.insert(flat.end(), pos[t].begin(), pos[t].end()); off.push_back(flat.size()); }
  if (!rc) rc = sdbg_stage_positions(seg, flat.data(), off.data(), kVocab);
  if (w) sdbg_writer_destroy(w);
  std::vector<int64_t> key(n_docs);
  std::vector<uint64_t> valid_bits((n_docs + 63) / 64, 0);
  for (uint32_t d = 1; d <= n_docs; ++d) {
    key[d - 1] = int64_t((uint64_t(d) * 7919u) % 23u) - 11;
    if (d % 5u) valid_bits[(d - 1) / 64] |= uint64_t(1) << ((d - 1) % 64);
  }
  if (!rc && (columns || clauses)) rc = sdbg_stage_column(seg, 20, SDBG_I64, key.data(), valid_bits.data(), n_docs);
  if (rc) { std::printf("{\"error\": %d}\n", rc); return 1; }
  auto ints = [](const char* f, const auto& v) {
    std::printf(", \"%s\": [", f);
    for (size_t i = 0; i < v.size(); ++i) std::printf("%s%lld", i ? ", " : "", static_cast<long long>(v[i]));
    std::printf("]");
  };
  struct Case { std::vector<uint32_t> slots, rel, excl; };
  const Case cases[] = {{{1, 0}, {0, 1}, {}}, {{2, 2, 4}, {0, 1, 3}, {5}}};
  ListCollector col;
  irs::ScoreFunction sf; irs::ColumnArgsFetcher fetcher;
  if (clauses) {
    // "1 0" & 2;  "2 2" & 4 & !"3 1" & !5;  0 & 1 & !3
    struct AndCase { std::vector<uint32_t> slots, rel, sizes; std::vector<uint8_t> neg; std::vector<uint32_t> excl, gsizes, gmin; };
    const std::vector<AndCase> and_cases = {{{1, 0, 2}, {0, 1, 0}, {2, 1}, {0, 0}, {}, {}},
                                            {{2, 2, 4, 3, 1}, {0, 1, 0, 0, 1}, {2, 1, 2}, {0, 0, 1}, {5}, {}},
                                            {{0, 1, 3}, {0, 0, 0}, {1, 1, 1}, {0, 0, 1}, {}, {}}};
    // ("1 0" | 2) & 4;  ("2 2" | 3) & !("3 1" | 5);  (0 | "1 4") & (1 | 2) & !3 & !5
    const std::vector<AndCase> group_cases = {{{1, 0, 2, 4}, {0, 1, 0, 0}, {2, 1, 1}, {0, 0, 0}, {}, {2, 1}},
                                              {{2, 2, 3, 3, 1, 5}, {0, 1, 0, 0, 1, 0}, {2, 1, 2, 1}, {0, 0, 1, 1}, {}, {2, 2}},
                                              {{0, 1, 4, 1, 2, 3}, {0, 0, 1, 0, 0, 0}, {1, 2, 1, 1, 1}, {0, 0, 0, 0, 1}, {5}, {2, 2, 1}}};
    // 2 of ("1 0" | 2 | 4);  2 of ("2 2" | 3 | "1 4") & !("3 1" | 5);  3 of (0 | 1 | 2 | 3) & (4 | "5 0") & !5
    const std::vector<AndCase> min_cases = {
        {{1, 0, 2, 4}, {0, 1, 0, 0}, {2, 1, 1}, {0, 0, 0}, {}, {3}, {2}},
        {{2, 2, 3, 1, 4, 3, 1, 5}, {0, 1, 0, 0, 1, 0, 1, 0}, {2, 1, 2, 2, 1}, {0, 0, 0, 1, 1}, {}, {3, 2}, {2, 1}},
        {{0, 1, 2, 3, 4, 5, 0}, {0, 0, 0, 0, 0, 0, 1}, {1, 1, 1, 1, 1, 2}, {0, 0, 0, 0, 0, 0}, {5}, {4, 2}, {3, 1}}};
    for (const AndCase& cs : mins ? min_cases : groups ? group_cases : and_cases) {
      std::vector<sdbg_bm25_term> terms(cs.slots.size());
      for (size_t i = 0; i < terms.size(); ++i) {
        sdbg_bm25_collect(n_docs, sum_len, docs[cs.slots[i]].size(), 1.2f, 0.75f, &terms[i]);
        terms[i].term = cs.slots[i];
      }
      std::printf("{\"slots\": [");
      for (size_t i = 0; i < cs.slots.size(); ++i) std::printf("%s%u", i ? ", " : "", cs.slots[i]);
      std::printf("]");
      ints("rel", cs.rel); ints("sizes", cs.sizes); ints("neg", cs.neg); ints("excl", cs.excl);
      if (groups) ints("gsizes", cs.gsizes);
      if (mins) ints("gmin", cs.gmin);
      sdbg_host::GpuTopKIterator it(seg, SDBG_QUERY_AND, terms, 1.2f, 0.75f, 50, nullptr, cs.excl, {}, cs.gmin, cs.rel, cs.sizes,
                                  cs.neg, cs.gsizes);
      col.docs.clear();
      it.Collect(sf, fetcher, col);
      std::printf(", \"topk\": [");
      for (size_t i = 0; i < col.docs.size(); ++i) std::printf("%s[%u, %.9g]", i ? ", " : "", col.docs[i].doc, double(col.docs[i].score));
      std::printf("], \"total\": %llu", static_cast<unsigned long long>(it.total_matches()));
      duckdb::DataChunkMock out;
      sdbg_host::GpuCountScan cnt({seg}, SDBG_QUERY_AND, cs.slots, cs.excl, nullptr, {}, cs.gmin, cs.rel, cs.sizes, cs.neg, cs.gsizes);
      cnt.Scan(out);
      std::printf(", \"count\": %lld", static_cast<long long>(out.count.empty() ? -1 : out.count[0]));
      sdbg_host::GpuSortedScan sorted({seg}, SDBG_QUERY_AND, cs.slots, cs.excl, nullptr, 20, true, false, 30, {}, cs.gmin, cs.rel,
                                      cs.sizes, cs.neg, cs.gsizes);
      for (sorted.Scan(out); out.size; sorted.Scan(out)) ints("sorted_docs", out.doc);
      sdbg_host::GpuFacetScan facet({seg}, SDBG_QUERY_AND, cs.slots, cs.excl, nullptr, 20, {}, cs.gmin, cs.rel, cs.sizes, cs.neg,
                                    cs.gsizes);
      std::vector<int64_t> keys, counts;
      for (facet.Scan(out); out.size; facet.Scan(out)) {
        keys.insert(keys.end(), out.key.begin(), out.key.end());
        counts.insert(counts.end(), out.count.begin(), out.count.end());
      }
      ints("facet_keys", keys); ints("facet_counts", counts);
      sdbg_host::GpuMatchAggScan agg({seg}, SDBG_QUERY_AND, cs.slots, cs.excl, nullptr, UINT64_MAX, 20, SDBG_I64, {}, cs.gmin, cs.rel,
                                     cs.sizes, cs.neg, cs.gsizes);
      agg.Scan(out);
      ints("agg_count", out.count);
      sdbg_host::GpuMatchScan scan({seg}, terms, cs.excl, nullptr, 1.2f, 0.75f, true, {}, cs.gmin, cs.rel, cs.sizes, cs.neg,
                                   cs.gsizes);
      std::vector<uint32_t> sdocs;
      std::vector<float> sscores;
      for (scan.Scan(out); out.size; scan.Scan(out)) {
        sdocs.insert(sdocs.end(), out.doc.begin(), out.doc.end());
        sscores.insert(sscores.end(), out.score.begin(), out.score.end());
      }
      ints("scan_docs", sdocs);
      std::printf(", \"scan_scores\": [");
      for (size_t i = 0; i < sscores.size(); ++i) std::printf("%s%.9g", i ? ", " : "", double(sscores[i]));
      std::printf("], \"scan_total\": %llu}\n", static_cast<unsigned long long>(scan.total_matches()));
    }
  }
  for (const Case& cs : clauses ? std::vector<Case>{} : std::vector<Case>(std::begin(cases), std::end(cases))) {
    std::vector<sdbg_bm25_term> terms(cs.slots.size());
    for (size_t i = 0; i < terms.size(); ++i) {
      sdbg_bm25_collect(n_docs, sum_len, docs[cs.slots[i]].size(), 1.2f, 0.75f, &terms[i]);
      terms[i].term = cs.slots[i];
    }
    if (columns) {
      std::printf("{\"slots\": [");
      for (size_t i = 0; i < cs.slots.size(); ++i) std::printf("%s%u", i ? ", " : "", cs.slots[i]);
      std::printf("]");
      ints("rel", cs.rel);
      ints("excl", cs.excl);
      duckdb::DataChunkMock out;
      sdbg_host::GpuSortedScan sorted({seg}, SDBG_QUERY_AND, cs.slots, cs.excl, nullptr, 20, true, false, 30, {}, {}, cs.rel);
      for (sorted.Scan(out); out.size; sorted.Scan(out)) { ints("sorted_docs", out.doc); ints("sorted_values", out.value); ints("sorted_valid", out.valid); }
      sdbg_host::GpuFacetScan facet({seg}, SDBG_QUERY_AND, cs.slots, cs.excl, nullptr, 20, {}, {}, cs.rel);
      std::vector<int64_t> keys, counts, valid;
      for (facet.Scan(out); out.size; facet.Scan(out)) {
        keys.insert(keys.end(), out.key.begin(), out.key.end());
        counts.insert(counts.end(), out.count.begin(), out.count.end());
        valid.insert(valid.end(), out.valid.begin(), out.valid.end());
      }
      ints("facet_keys", keys); ints("facet_counts", counts); ints("facet_valid", valid);
      sdbg_host::GpuMatchAggScan agg({seg}, SDBG_QUERY_AND, cs.slots, cs.excl, nullptr, UINT64_MAX, 20, SDBG_I64, {}, {}, cs.rel);
      agg.Scan(out);
      ints("agg_count", out.count); ints("agg_count_value", out.count_value); ints("agg_sum_lo", out.sum_lo);
      ints("agg_min", out.min); ints("agg_max", out.max);
      sdbg_host::GpuMatchScan scan({seg}, terms, cs.excl, nullptr, 1.2f, 0.75f, true, {}, {}, cs.rel);
      std::vector<uint32_t> sdocs;
      std::vector<float> sscores;
      for (scan.Scan(out); out.size; scan.Scan(out)) {
        sdocs.insert(sdocs.end(), out.doc.begin(), out.doc.end());
        sscores.insert(sscores.end(), out.score.begin(), out.score.end());
      }
      ints("scan_docs", sdocs);
      std::printf(", \"scan_scores\": [");
      for (size_t i = 0; i < sscores.size(); ++i) std::printf("%s%.9g", i ? ", " : "", double(sscores[i]));
      std::printf("], \"scan_total\": %llu}\n", static_cast<unsigned long long>(scan.total_matches()));
      continue;
    }
    sdbg_host::GpuTopKIterator it(seg, SDBG_QUERY_AND, terms, 1.2f, 0.75f, 50, nullptr, cs.excl, {}, {}, cs.rel);
    col.docs.clear();
    it.Collect(sf, fetcher, col);
    sdbg_host::GpuCountScan cnt({seg}, SDBG_QUERY_AND, cs.slots, cs.excl, nullptr, {}, {}, cs.rel);
    duckdb::DataChunkMock out;
    cnt.Scan(out);
    std::printf("{\"slots\": [");
    for (size_t i = 0; i < cs.slots.size(); ++i) std::printf("%s%u", i ? ", " : "", cs.slots[i]);
    std::printf("], \"rel\": [");
    for (size_t i = 0; i < cs.rel.size(); ++i) std::printf("%s%u", i ? ", " : "", cs.rel[i]);
    std::printf("], \"excl\": [");
    for (size_t i = 0; i < cs.excl.size(); ++i) std::printf("%s%u", i ? ", " : "", cs.excl[i]);
    std::printf("], \"topk\": [");
    for (size_t i = 0; i < col.docs.size(); ++i) std::printf("%s[%u, %.9g]", i ? ", " : "", col.docs[i].doc, double(col.docs[i].score));
    std::printf("], \"total\": %llu, \"count\": %lld}\n", static_cast<unsigned long long>(it.total_matches()),
                static_cast<long long>(out.count.empty() ? -1 : out.count[0]));
  }
  sdbg_segment_destroy(seg);
  sdbg_destroy(ctx);
  return 0;
}
}  // namespace

int main(int argc, char** argv) {
  const uint32_t n_docs = argc > 1 ? uint32_t(std::atoi(argv[1])) : 200000;
  sdbg_ctx* ctx = nullptr;
  int rc = sdbg_init(0, &ctx);
  if (rc != SDBG_OK) { std::printf("{\"error\": %d}\n", rc); return rc == SDBG_ENODEVICE ? 3 : 1; }
  if (argc > 2 && std::string(argv[2]) == "phrase")
    return phrase_mode(ctx, n_docs, argc > 3 && std::string(argv[3]) == "columns",
                       argc > 3 && (std::string(argv[3]) == "and" || std::string(argv[3]) == "groups" || std::string(argv[3]) == "min"),
                       argc > 3 && (std::string(argv[3]) == "groups" || std::string(argv[3]) == "min"),
                       argc > 3 && std::string(argv[3]) == "min");
  sdbg_segment* seg = nullptr;
  sdbg_segment_create(ctx, n_docs, &seg);
  std::vector<uint32_t> dc(8);
  uint64_t sum_dl = 0;
  rc = sdbg_synth_corpus(seg, 0, n_docs, 0, 8, 4, dc.data(), &sum_dl);
  if (rc) { std::printf("{\"error\": %d}\n", rc); return 1; }
  sdbg_synth_column(seg, 9, 2, 6, 1, n_docs);
  // --- top-k through the DocIterator adapter ---
  std::vector<sdbg_bm25_term> terms(2);
  const uint32_t ids[2] = {2, 5};
  for (int i = 0; i < 2; ++i) { sdbg_bm25_collect(n_docs, sum_dl, dc[ids[i]], 1.2f, 0.75f, &terms[size_t(i)]); terms[size_t(i)].term = ids[i]; }
  sdbg_col_pred filt{}; filt.field = 9; filt.op = SDBG_OP_BETWEEN; filt.lo_i = 250000; filt.hi_i = 749999;
  if (argc > 2 && std::string(argv[2]) == "chain") {
    // `9 BETWEEN 250000 AND 749999 AND 20 < n_docs / 2 AND 9 <> 500000` (field 20: value = row, doc-ordered), then the
    // indicator column 21 = 1 where the chain holds (int32, nullable with every row valid) as the single predicate
    std::vector<int32_t> v9(n_docs);
    std::vector<int64_t> v20(n_docs);
    sdbg_column_to_host(seg, 9, v9.data(), n_docs);
    std::vector<int32_t> m(n_docs);
    for (uint32_t r = 0; r < n_docs; ++r) {
      v20[r] = int64_t(r);
      m[r] = v9[r] >= 250000 && v9[r] <= 749999 && v20[r] < int64_t(n_docs / 2) && v9[r] != 500000;
    }
    std::vector<uint64_t> valid((n_docs + 63) / 64, ~0ull);
    sdbg_stage_column(seg, 20, SDBG_I64, v20.data(), nullptr, n_docs);
    sdbg_stage_column(seg, 21, SDBG_I32, m.data(), valid.data(), n_docs);
    sdbg_col_pred chain[3] = {filt, {}, {}};
    chain[0].op |= SDBG_OP_AND_NEXT;
    chain[1].field = 20; chain[1].op = SDBG_OP_LT | SDBG_OP_AND_NEXT; chain[1].lo_i = n_docs / 2;
    chain[2].field = 9; chain[2].op = SDBG_OP_NE; chain[2].lo_i = 500000;
    sdbg_col_pred ind{}; ind.field = 21; ind.op = SDBG_OP_EQ; ind.lo_i = 1;
    irs::ScoreFunction sf; irs::ColumnArgsFetcher fetcher;
    for (int indicator = 0; indicator < 2; ++indicator) {
      const sdbg_col_pred* f = indicator ? &ind : chain;
      ListCollector col;
      sdbg_host::GpuTopKIterator it(seg, SDBG_QUERY_OR, terms, 1.2f, 0.75f, 100, f);
      it.Collect(sf, fetcher, col);
      std::printf("{\"indicator\": %d, \"topk\": [", indicator);
      for (size_t i = 0; i < col.docs.size(); ++i) std::printf("%s[%u, %.9g]", i ? ", " : "", col.docs[i].doc, double(col.docs[i].score));
      sdbg_host::GpuTopKIterator st(seg, SDBG_QUERY_OR, terms, 1.2f, 0.75f, 0, f);
      std::vector<irs::doc_id_t> d(2048);
      std::vector<irs::score_t> sc(2048);
      uint64_t n = 0, doc_sum = 0;
      for (irs::doc_id_t lo = 1; lo <= n_docs; lo += 2048) {
        const uint32_t got = st.EmitScoredDocs(d.data(), sc.data(), lo + 2048, sf, &fetcher, lo);
        for (uint32_t i = 0; i < got; ++i) doc_sum += d[i];
        n += got;
      }
      sdbg_host::GpuCountScan scan({seg}, SDBG_QUERY_OR, {2, 5}, {}, f);
      duckdb::DataChunkMock chunk;
      scan.Scan(chunk);
      std::printf("], \"total\": %llu, \"stream_n\": %llu, \"stream_doc_sum\": %llu, \"count\": %lld}\n",
                  static_cast<unsigned long long>(it.total_matches()), static_cast<unsigned long long>(n),
                  static_cast<unsigned long long>(doc_sum), chunk.size ? static_cast<long long>(chunk.count[0]) : -1ll);
    }
    sdbg_segment_destroy(seg);
    sdbg_destroy(ctx);
    return 0;
  }
  if (argc > 2 && std::string(argv[2]) == "excl") {
    // `t2 | t5` minus the docs of t3: Collect (top-100) and the streaming mode (k = 0), without and with the table filter
    ListCollector col;
    irs::ScoreFunction sf; irs::ColumnArgsFetcher fetcher;
    for (int with_filter = 0; with_filter < 2; ++with_filter) {
      sdbg_host::GpuTopKIterator it(seg, SDBG_QUERY_OR, terms, 1.2f, 0.75f, 100, with_filter ? &filt : nullptr, {3});
      col.docs.clear();
      it.Collect(sf, fetcher, col);
      std::printf("{\"filter\": %d, \"topk\": [", with_filter);
      for (size_t i = 0; i < col.docs.size(); ++i) std::printf("%s[%u, %.9g]", i ? ", " : "", col.docs[i].doc, double(col.docs[i].score));
      std::printf("], \"total\": %llu, \"threshold\": %.9g", static_cast<unsigned long long>(it.total_matches()), double(it.threshold().value));
      sdbg_host::GpuTopKIterator st(seg, SDBG_QUERY_OR, terms, 1.2f, 0.75f, 0, with_filter ? &filt : nullptr, {3});
      std::vector<irs::doc_id_t> d(2048);
      std::vector<irs::score_t> sc(2048);
      uint64_t n = 0, doc_sum = 0; double score_sum = 0;
      for (irs::doc_id_t lo = 1; lo <= n_docs; lo += 2048) {
        const uint32_t got = st.EmitScoredDocs(d.data(), sc.data(), lo + 2048, sf, &fetcher, lo);
        for (uint32_t i = 0; i < got; ++i) { doc_sum += d[i]; score_sum += sc[i]; }
        n += got;
      }
      std::printf(", \"stream_n\": %llu, \"stream_doc_sum\": %llu, \"stream_score_sum\": %.12g}\n", static_cast<unsigned long long>(n),
                  static_cast<unsigned long long>(doc_sum), score_sum);
    }
    sdbg_segment_destroy(seg);
    sdbg_destroy(ctx);
    return 0;
  }
  if (argc > 2 && std::string(argv[2]) == "groups") {
    // `t2 & (t5 | t6)` and `t2 & (t5 | t6) & !t3`, without and with the table filter: Collect (top-100) and count(*)
    std::vector<sdbg_bm25_term> g3(3);
    const uint32_t gids[3] = {2, 5, 6};
    for (int i = 0; i < 3; ++i) { sdbg_bm25_collect(n_docs, sum_dl, dc[gids[i]], 1.2f, 0.75f, &g3[size_t(i)]); g3[size_t(i)].term = gids[i]; }
    ListCollector col;
    irs::ScoreFunction sf; irs::ColumnArgsFetcher fetcher;
    for (int with_filter = 0; with_filter < 2; ++with_filter)
      for (int excl = 0; excl < 2; ++excl) {
        const std::vector<uint32_t> ex = excl ? std::vector<uint32_t>{3} : std::vector<uint32_t>{};
        sdbg_host::GpuTopKIterator it(seg, SDBG_QUERY_OR, g3, 1.2f, 0.75f, 100, with_filter ? &filt : nullptr, ex, {1, 2});
        col.docs.clear();
        it.Collect(sf, fetcher, col);
        std::printf("{\"filter\": %d, \"excl\": %d, \"topk\": [", with_filter, excl);
        for (size_t i = 0; i < col.docs.size(); ++i) std::printf("%s[%u, %.9g]", i ? ", " : "", col.docs[i].doc, double(col.docs[i].score));
        sdbg_host::GpuCountScan scan({seg}, SDBG_QUERY_OR, {2, 5, 6}, ex, with_filter ? &filt : nullptr, {1, 2});
        duckdb::DataChunkMock chunk;
        scan.Scan(chunk);
        const long long count = chunk.size ? chunk.count[0] : -1;
        scan.Scan(chunk);
        std::printf("], \"total\": %llu, \"threshold\": %.9g, \"count\": %lld, \"rows_after\": %llu}\n",
                    static_cast<unsigned long long>(it.total_matches()), double(it.threshold().value), count,
                    static_cast<unsigned long long>(chunk.size));
      }
    int code = 0;   // k = 0 (the streaming scan) has no grouped form
    try { sdbg_host::GpuTopKIterator st(seg, SDBG_QUERY_OR, g3, 1.2f, 0.75f, 0, nullptr, {}, {1, 2}); } catch (const sdbg_host::GpuError& e) { code = e.code; }
    std::printf("{\"stream_error\": %d}\n", code);
    sdbg_segment_destroy(seg);
    sdbg_destroy(ctx);
    return 0;
  }
  if (argc > 2 && std::string(argv[2]) == "minmatch") {
    // Or with min_match_count 2 over t2, t5, t6: alone (a root Or) and as the child of an And with t1, without and with the
    // table filter: Collect (top-100) and count(*)
    std::vector<sdbg_bm25_term> g4(4);
    const uint32_t gids[4] = {1, 2, 5, 6};
    for (int i = 0; i < 4; ++i) { sdbg_bm25_collect(n_docs, sum_dl, dc[gids[i]], 1.2f, 0.75f, &g4[size_t(i)]); g4[size_t(i)].term = gids[i]; }
    ListCollector col;
    irs::ScoreFunction sf; irs::ColumnArgsFetcher fetcher;
    for (int nested = 0; nested < 2; ++nested)
      for (int with_filter = 0; with_filter < 2; ++with_filter) {
        const std::vector<sdbg_bm25_term> t = nested ? g4 : std::vector<sdbg_bm25_term>(g4.begin() + 1, g4.end());
        const std::vector<uint32_t> ids = nested ? std::vector<uint32_t>{1, 2, 5, 6} : std::vector<uint32_t>{2, 5, 6};
        const std::vector<uint32_t> sizes = nested ? std::vector<uint32_t>{1, 3} : std::vector<uint32_t>{3};
        const std::vector<uint32_t> mins = nested ? std::vector<uint32_t>{1, 2} : std::vector<uint32_t>{2};
        sdbg_host::GpuTopKIterator it(seg, SDBG_QUERY_OR, t, 1.2f, 0.75f, 100, with_filter ? &filt : nullptr, {}, sizes, mins);
        col.docs.clear();
        it.Collect(sf, fetcher, col);
        std::printf("{\"nested\": %d, \"filter\": %d, \"topk\": [", nested, with_filter);
        for (size_t i = 0; i < col.docs.size(); ++i) std::printf("%s[%u, %.9g]", i ? ", " : "", col.docs[i].doc, double(col.docs[i].score));
        sdbg_host::GpuCountScan scan({seg}, SDBG_QUERY_OR, ids, {}, with_filter ? &filt : nullptr, sizes, mins);
        duckdb::DataChunkMock chunk;
        scan.Scan(chunk);
        const long long count = chunk.size ? chunk.count[0] : -1;
        scan.Scan(chunk);
        std::printf("], \"total\": %llu, \"threshold\": %.9g, \"count\": %lld, \"rows_after\": %llu}\n",
                    static_cast<unsigned long long>(it.total_matches()), double(it.threshold().value), count,
                    static_cast<unsigned long long>(chunk.size));
      }
    int code = 0;   // a minimum above the group's size
    try {
      sdbg_host::GpuCountScan scan({seg}, SDBG_QUERY_OR, {2, 5, 6}, {}, nullptr, {3}, {4});
      duckdb::DataChunkMock chunk;
      scan.Scan(chunk);
    } catch (const sdbg_host::GpuError& e) { code = e.code; }
    std::printf("{\"min_error\": %d}\n", code);
    sdbg_segment_destroy(seg);
    sdbg_destroy(ctx);
    return 0;
  }
  if (argc > 2 && std::string(argv[2]) == "scan") {
    // the Stream mode (GpuMatchScan): `t2 | t5` scored, `t1 & 2 of (t2 | t5 | t6)` unscored, `t2 & (t5 | t6)` scored; every
    // row in chunk order
    struct Case { std::vector<uint32_t> ids, sizes, mins; bool scored; };
    const Case cases[3] = {{{2, 5}, {2}, {1}, true}, {{1, 2, 5, 6}, {1, 3}, {1, 2}, false}, {{2, 5, 6}, {1, 2}, {1, 1}, true}};
    for (const Case& cs : cases) {
      std::vector<sdbg_bm25_term> t(cs.ids.size());
      for (size_t i = 0; i < t.size(); ++i) { sdbg_bm25_collect(n_docs, sum_dl, dc[cs.ids[i]], 1.2f, 0.75f, &t[i]); t[i].term = cs.ids[i]; }
      sdbg_host::GpuMatchScan scan({seg}, t, {}, nullptr, 1.2f, 0.75f, cs.scored, cs.sizes, cs.mins);
      std::vector<uint64_t> chunks;
      std::vector<uint32_t> docs, segs;
      std::vector<float> scores;
      duckdb::DataChunkMock chunk;
      for (scan.Scan(chunk); chunk.size; scan.Scan(chunk)) {
        chunks.push_back(chunk.size);
        docs.insert(docs.end(), chunk.doc.begin(), chunk.doc.end());
        segs.insert(segs.end(), chunk.segment.begin(), chunk.segment.end());
        scores.insert(scores.end(), chunk.score.begin(), chunk.score.end());
      }
      scan.Scan(chunk);
      std::printf("{\"groups\": [");
      for (size_t g = 0, o = 0; g < cs.sizes.size(); o += cs.sizes[g++]) {
        std::printf("%s[", g ? ", " : "");
        for (uint32_t i = 0; i < cs.sizes[g]; ++i) std::printf("%s%u", i ? ", " : "", cs.ids[o + i]);
        std::printf("]");
      }
      std::printf("], \"mins\": [");
      for (size_t g = 0; g < cs.mins.size(); ++g) std::printf("%s%u", g ? ", " : "", cs.mins[g]);
      std::printf("], \"scored\": %d, \"chunks\": [", cs.scored ? 1 : 0);
      for (size_t i = 0; i < chunks.size(); ++i) std::printf("%s%llu", i ? ", " : "", static_cast<unsigned long long>(chunks[i]));
      std::printf("], \"docs\": [");
      for (size_t i = 0; i < docs.size(); ++i) std::printf("%s%u", i ? ", " : "", docs[i]);
      std::printf("], \"segs\": [");
      for (size_t i = 0; i < segs.size(); ++i) std::printf("%s%u", i ? ", " : "", segs[i]);
      std::printf("], \"scores\": [");
      for (size_t i = 0; i < scores.size(); ++i) std::printf("%s%.9g", i ? ", " : "", double(scores[i]));
      std::printf("], \"total\": %llu, \"rows_after\": %llu}\n", static_cast<unsigned long long>(scan.total_matches()),
                  static_cast<unsigned long long>(chunk.size));
    }
    sdbg_segment_destroy(seg);
    sdbg_destroy(ctx);
    return 0;
  }
  // With a third argument "groups", the sorted and facet modes run group queries instead of `t2 | t5` (and `t2 & t5`):
  // query 0 is `t2 & (t5 | t6)`, query 1 `2 of (t2 | t5 | t6)`.
  const bool grouped = argc > 3 && std::string(argv[3]) == "groups";
  const std::vector<uint32_t> flat_ids{2, 5}, group_ids{2, 5, 6};
  auto group_sizes = [&](int q) { return !grouped ? std::vector<uint32_t>{} : q ? std::vector<uint32_t>{3} : std::vector<uint32_t>{1, 2}; };
  auto group_mins = [&](int q) { return grouped && q ? std::vector<uint32_t>{2} : std::vector<uint32_t>{}; };
  if (argc > 2 && std::string(argv[2]) == "sorted") {
    // `t2 | t5` and `(t2 | t5) & !t3` ORDER BY the int32 column 9, LIMIT 4096 (two chunks), every direction and NULL
    // placement, without and with the table filter: every row in order, then end of scan
    for (int query = 0; query < (grouped ? 2 : 1); ++query)
    for (int with_filter = 0; with_filter < 2; ++with_filter)
      for (int excl = 0; excl < 2; ++excl)
        for (int desc = 0; desc < 2; ++desc)
          for (int nf = 0; nf < 2; ++nf) {
            sdbg_host::GpuSortedScan scan({seg}, SDBG_QUERY_OR, grouped ? group_ids : flat_ids,
                                          excl ? std::vector<uint32_t>{3} : std::vector<uint32_t>{}, with_filter ? &filt : nullptr, 9,
                                          desc != 0, nf != 0, 4096, group_sizes(query), group_mins(query));
            duckdb::DataChunkMock chunk;
            std::vector<uint32_t> docs, segs;
            std::vector<int64_t> vals;
            std::vector<uint8_t> valid;
            uint64_t chunks = 0, max_chunk = 0;
            for (;;) {
              scan.Scan(chunk);
              if (chunk.size == 0) break;
              ++chunks;
              max_chunk = std::max<uint64_t>(max_chunk, chunk.size);
              docs.insert(docs.end(), chunk.doc.begin(), chunk.doc.end());
              segs.insert(segs.end(), chunk.segment.begin(), chunk.segment.end());
              vals.insert(vals.end(), chunk.value.begin(), chunk.value.end());
              valid.insert(valid.end(), chunk.valid.begin(), chunk.valid.end());
            }
            scan.Scan(chunk);
            if (grouped) std::printf("{\"query\": %d, ", query);
            std::printf("%s\"filter\": %d, \"excl\": %d, \"desc\": %d, \"nulls_first\": %d, \"chunks\": %llu, \"max_chunk\": %llu, "
                        "\"rows_after\": %llu, \"docs\": [", grouped ? "" : "{", with_filter, excl, desc, nf, static_cast<unsigned long long>(chunks),
                        static_cast<unsigned long long>(max_chunk), static_cast<unsigned long long>(chunk.size));
            for (size_t i = 0; i < docs.size(); ++i) std::printf("%s%u", i ? ", " : "", docs[i]);
            std::printf("], \"segs\": [");
            for (size_t i = 0; i < segs.size(); ++i) std::printf("%s%u", i ? ", " : "", segs[i]);
            std::printf("], \"values\": [");
            for (size_t i = 0; i < vals.size(); ++i) std::printf("%s%lld", i ? ", " : "", static_cast<long long>(vals[i]));
            std::printf("], \"valid\": [");
            for (size_t i = 0; i < valid.size(); ++i) std::printf("%s%u", i ? ", " : "", unsigned(valid[i]));
            std::printf("]}\n");
          }
    sdbg_segment_destroy(seg);
    sdbg_destroy(ctx);
    return 0;
  }
  if (argc > 2 && std::string(argv[2]) == "facet") {
    // `t2 | t5`, `t2 & t5` and `(t2 | t5) & !t3` GROUP BY the 2001-key int64 column 15 (count(*)), without and with the
    // table filter: every group in key order, then end of scan. Then the int32 column 9, whose range is too wide.
    // (grouped: "kind" 0 / 1 is query 0 / 1)
    sdbg_synth_column(seg, 15, 15, 3, 1, n_docs);
    for (int with_filter = 0; with_filter < 2; ++with_filter)
      for (int kind : {int(SDBG_QUERY_OR), int(SDBG_QUERY_AND)})
        for (int excl = 0; excl < 2; ++excl) {
          sdbg_host::GpuFacetScan scan({seg}, kind, grouped ? group_ids : flat_ids,
                                       excl ? std::vector<uint32_t>{3} : std::vector<uint32_t>{}, with_filter ? &filt : nullptr, 15,
                                       group_sizes(kind), group_mins(kind));
          duckdb::DataChunkMock chunk;
          std::vector<int64_t> keys, counts;
          std::vector<uint8_t> valid;
          uint64_t chunks = 0, max_chunk = 0;
          for (;;) {
            scan.Scan(chunk);
            if (chunk.size == 0) break;
            ++chunks;
            max_chunk = std::max<uint64_t>(max_chunk, chunk.size);
            keys.insert(keys.end(), chunk.key.begin(), chunk.key.end());
            counts.insert(counts.end(), chunk.count.begin(), chunk.count.end());
            valid.insert(valid.end(), chunk.valid.begin(), chunk.valid.end());
          }
          scan.Scan(chunk);
          std::printf("{\"filter\": %d, \"kind\": %d, \"excl\": %d, \"chunks\": %llu, \"max_chunk\": %llu, \"rows_after\": %llu, "
                      "\"keys\": [", with_filter, kind, excl, static_cast<unsigned long long>(chunks),
                      static_cast<unsigned long long>(max_chunk), static_cast<unsigned long long>(chunk.size));
          for (size_t i = 0; i < keys.size(); ++i) std::printf("%s%lld", i ? ", " : "", static_cast<long long>(keys[i]));
          std::printf("], \"counts\": [");
          for (size_t i = 0; i < counts.size(); ++i) std::printf("%s%lld", i ? ", " : "", static_cast<long long>(counts[i]));
          std::printf("], \"valid\": [");
          for (size_t i = 0; i < valid.size(); ++i) std::printf("%s%u", i ? ", " : "", unsigned(valid[i]));
          std::printf("]}\n");
        }
    int code = 0;
    try {
      sdbg_host::GpuFacetScan wide({seg}, SDBG_QUERY_OR, {2, 5}, {}, nullptr, 9);
      duckdb::DataChunkMock chunk;
      wide.Scan(chunk);
    } catch (const sdbg_host::GpuError& e) { code = e.code; }
    std::printf("{\"wide_error\": %d}\n", code);
    sdbg_segment_destroy(seg);
    sdbg_destroy(ctx);
    return 0;
  }
  if (argc > 2 && std::string(argv[2]) == "aggregate") {
    // `t2 | t5`, `t2 & t5` and `(t2 | t5) & !t3` (grouped: "kind" 0 / 1 is query 0 / 1), without and with the table filter:
    // count, count(v), sum, avg, min, max of the int32 column 9 GROUP BY the 2001-key int64 column 15 (every group in key
    // order, then end of scan), and of the float64 column 16 without GROUP BY (one row). Then column 9 as the key, whose
    // range is too wide.
    sdbg_synth_column(seg, 15, 15, 3, 1, n_docs);
    sdbg_synth_column(seg, 16, 16, 4, 1, n_docs);
    auto run = [&](sdbg_host::GpuMatchAggScan& scan, const char* name) {
      duckdb::DataChunkMock chunk;
      std::vector<long long> keys, cnt, cntv, lo, hi, mn, mx;
      std::vector<double> sf, avg;
      std::vector<unsigned> valid;
      uint64_t chunks = 0, max_chunk = 0;
      for (;;) {
        scan.Scan(chunk);
        if (chunk.size == 0) break;
        ++chunks;
        max_chunk = std::max<uint64_t>(max_chunk, chunk.size);
        for (size_t i = 0; i < chunk.size; ++i) {
          keys.push_back(chunk.key[i]); cnt.push_back(chunk.count[i]); cntv.push_back(chunk.count_value[i]);
          lo.push_back(chunk.sum_lo[i]); hi.push_back(chunk.sum_hi[i]); sf.push_back(chunk.sum_f64[i]); avg.push_back(chunk.avg[i]);
          mn.push_back(chunk.min[i]); mx.push_back(chunk.max[i]); valid.push_back(chunk.valid[i]);
        }
      }
      scan.Scan(chunk);
      std::printf("\"%s\": {\"chunks\": %llu, \"max_chunk\": %llu, \"rows_after\": %llu", name, static_cast<unsigned long long>(chunks),
                  static_cast<unsigned long long>(max_chunk), static_cast<unsigned long long>(chunk.size));
      auto ints = [](const char* f, const std::vector<long long>& v) {
        std::printf(", \"%s\": [", f);
        for (size_t i = 0; i < v.size(); ++i) std::printf("%s%lld", i ? ", " : "", v[i]);
        std::printf("]");
      };
      auto dbls = [](const char* f, const std::vector<double>& v) {
        std::printf(", \"%s\": [", f);
        for (size_t i = 0; i < v.size(); ++i) std::printf("%s%.17g", i ? ", " : "", v[i]);
        std::printf("]");
      };
      ints("keys", keys); ints("count", cnt); ints("count_value", cntv); ints("sum_lo", lo); ints("sum_hi", hi);
      dbls("sum_f64", sf); dbls("avg", avg); ints("min", mn); ints("max", mx);
      std::printf(", \"valid\": [");
      for (size_t i = 0; i < valid.size(); ++i) std::printf("%s%u", i ? ", " : "", valid[i]);
      std::printf("]}");
    };
    for (int with_filter = 0; with_filter < 2; ++with_filter)
      for (int kind : {int(SDBG_QUERY_OR), int(SDBG_QUERY_AND)})
        for (int excl = 0; excl < 2; ++excl) {
          const std::vector<uint32_t> ex = excl ? std::vector<uint32_t>{3} : std::vector<uint32_t>{};
          sdbg_host::GpuMatchAggScan by_key({seg}, kind, grouped ? group_ids : flat_ids, ex, with_filter ? &filt : nullptr, 15, 9,
                                            SDBG_I32, group_sizes(kind), group_mins(kind));
          sdbg_host::GpuMatchAggScan whole({seg}, kind, grouped ? group_ids : flat_ids, ex, with_filter ? &filt : nullptr, UINT64_MAX,
                                           16, SDBG_F64, group_sizes(kind), group_mins(kind));
          std::printf("{\"filter\": %d, \"kind\": %d, \"excl\": %d, ", with_filter, kind, excl);
          run(by_key, "grouped");
          std::printf(", ");
          run(whole, "ungrouped");
          std::printf("}\n");
        }
    int code = 0;
    try {
      sdbg_host::GpuMatchAggScan wide({seg}, SDBG_QUERY_OR, {2, 5}, {}, nullptr, 9, 16, SDBG_F64);
      duckdb::DataChunkMock chunk;
      wide.Scan(chunk);
    } catch (const sdbg_host::GpuError& e) { code = e.code; }
    std::printf("{\"wide_error\": %d}\n", code);
    sdbg_segment_destroy(seg);
    sdbg_destroy(ctx);
    return 0;
  }
  if (argc > 2 && std::string(argv[2]) == "count") {
    // count(*) of `t2 | t5`, `t2 & t5` and `(t2 | t5) & !t3`, without and with the table filter: one row, then end of scan
    for (int with_filter = 0; with_filter < 2; ++with_filter)
      for (int kind : {int(SDBG_QUERY_OR), int(SDBG_QUERY_AND)})
        for (int excl = 0; excl < 2; ++excl) {
          sdbg_host::GpuCountScan scan({seg}, kind, {2, 5}, excl ? std::vector<uint32_t>{3} : std::vector<uint32_t>{},
                                       with_filter ? &filt : nullptr);
          duckdb::DataChunkMock chunk;
          scan.Scan(chunk);
          const uint64_t rows = chunk.size;
          const long long count = rows ? chunk.count[0] : -1;
          scan.Scan(chunk);
          std::printf("{\"filter\": %d, \"kind\": %d, \"excl\": %d, \"rows\": %llu, \"count\": %lld, \"rows_after\": %llu}\n", with_filter,
                      kind, excl, static_cast<unsigned long long>(rows), count, static_cast<unsigned long long>(chunk.size));
        }
    sdbg_segment_destroy(seg);
    sdbg_destroy(ctx);
    return 0;
  }
  sdbg_host::GpuTopKIterator it(seg, SDBG_QUERY_OR, terms, 1.2f, 0.75f, 100, &filt);
  ListCollector col;
  irs::ScoreFunction sf; irs::ColumnArgsFetcher fetcher;
  it.Collect(sf, fetcher, col);
  std::printf("{\"topk\": [");
  for (size_t i = 0; i < col.docs.size(); ++i) std::printf("%s[%u, %.9g]", i ? ", " : "", col.docs[i].doc, double(col.docs[i].score));
  // attributes through the reference's accessor, and the bitmap window of the first 4096 docs
  const auto* thr = irs::get<irs::ScoreThresholdAttr>(it);
  const auto* cost = irs::get<irs::CostAttr>(it);
  sdbg_host::GpuTopKIterator it2(seg, SDBG_QUERY_OR, terms, 1.2f, 0.75f, 100, &filt);
  std::vector<uint64_t> mask(64, 0);
  std::vector<irs::score_t> window(4096, 0.f);
  irs::FillBlockScoreContext sc; sc.score_window = window.data(); sc.merge_type = irs::ScoreMergeType::Sum;
  const auto fb = it2.FillBlock(1, 4097, mask.data(), sc, irs::FillBlockMatchContext{});
  unsigned bits = 0; double wsum = 0;
  for (uint64_t w : mask) bits += unsigned(__builtin_popcountll(w));
  for (float w : window) wsum += w;
  std::printf("], \"total\": %llu, \"threshold\": %.9g, \"attr_threshold\": %.9g, \"attr_cost\": %llu, \"fill_bits\": %u, \"fill_sum\": %.9g, \"fill_next\": %u}\n",
              static_cast<unsigned long long>(it.total_matches()), double(it.threshold().value), double(thr ? thr->value : -1.f),
              static_cast<unsigned long long>(cost ? cost->estimate() : 0), bits, wsum, fb.first);
  // --- streaming mode: drain EmitScoredDocs in STANDARD_VECTOR_SIZE-bounded windows like StreamScanLocalState::EmitChunk ---
  {
    sdbg_host::GpuTopKIterator st(seg, SDBG_QUERY_OR, terms, 1.2f, 0.75f, 0, &filt);
    std::vector<irs::doc_id_t> d(2048);
    std::vector<irs::score_t> sc(2048);
    uint64_t n = 0, chunks = 0, doc_sum = 0; double score_sum = 0; bool ordered = true; irs::doc_id_t last = 0;
    for (irs::doc_id_t lo = 1; lo <= n_docs; lo += 2048) {      // a 2048-doc window can hold at most 2048 matches
      const uint32_t got = st.EmitScoredDocs(d.data(), sc.data(), lo + 2048, sf, &fetcher, lo);
      if (got) ++chunks;
      for (uint32_t i = 0; i < got; ++i) { ordered = ordered && d[i] > last; last = d[i]; doc_sum += d[i]; score_sum += sc[i]; }
      n += got;
    }
    std::printf("{\"stream_n\": %llu, \"stream_chunks\": %llu, \"stream_doc_sum\": %llu, \"stream_score_sum\": %.12g, \"stream_ordered\": %d, \"stream_count\": %u}\n",
                static_cast<unsigned long long>(n), static_cast<unsigned long long>(chunks), static_cast<unsigned long long>(doc_sum), score_sum,
                ordered ? 1 : 0, st.count());
  }
  // --- aggregate scan through the table-function adapter ---
  for (uint64_t f = 10; f <= 14; ++f) sdbg_synth_column(seg, f, f, int(f - 10), 0, n_docs);
  std::vector<sdbg_col_pred> preds(2);
  preds[0].field = 11; preds[0].op = SDBG_OP_LT; preds[0].lo_i = 500000;
  preds[1].field = 12; preds[1].op = SDBG_OP_GE; preds[1].is_float = 1; preds[1].lo_f = 0.25;
  sdbg_host::GpuAggScan scan({seg}, preds, 10, 13, 14, 100000);
  duckdb::DataChunkMock chunk;
  uint64_t groups = 0, rows = 0, chunks = 0; __int128 sum = 0; double avg_sum = 0;
  for (;;) {
    scan.Scan(chunk);
    if (chunk.size == 0) break;
    ++chunks;
    for (size_t i = 0; i < chunk.size; ++i) { ++groups; rows += uint64_t(chunk.count[i]); sum += (static_cast<__int128>(chunk.sum_hi[i]) << 64) + static_cast<unsigned long long>(chunk.sum_lo[i]); avg_sum += chunk.avg[i]; }
    if (chunk.size > duckdb::STANDARD_VECTOR_SIZE) return 2;
  }
  std::printf("{\"groups\": %llu, \"rows\": %llu, \"chunks\": %llu, \"sum_v\": %lld, \"avg_sum\": %.12g}\n", static_cast<unsigned long long>(groups),
              static_cast<unsigned long long>(rows), static_cast<unsigned long long>(chunks), static_cast<long long>(sum), avg_sum);
  // --- the same scan mode driven by four concurrent workers (one global state, a local state each) ---
  {
    sdbg_host::GpuAggGlobalState gs({seg}, preds, 10, 13, 14, 100000);
    constexpr int kWorkers = 4;
    uint64_t w_groups[kWorkers] = {}, w_rows[kWorkers] = {}, w_chunks[kWorkers] = {};
    long long w_sum[kWorkers] = {};
    bool w_ok[kWorkers] = {};
    std::vector<std::thread> pool;
    for (int w = 0; w < kWorkers; ++w)
      pool.emplace_back([&, w] {
        sdbg_host::GpuAggLocalState ls;
        duckdb::DataChunkMock out;
        bool ok = true;
        for (;;) {
          sdbg_host::GpuAggScanFunction(gs, ls, out);
          if (out.size == 0) break;
          ok = ok && out.size <= duckdb::STANDARD_VECTOR_SIZE;
          for (size_t i = 0; i < out.size; ++i) { ++w_groups[w]; w_rows[w] += uint64_t(out.count[i]); w_sum[w] += out.sum_lo[i]; }
        }
        w_chunks[w] = ls.chunks_claimed;
        w_ok[w] = ok;
      });
    for (auto& th : pool) th.join();
    uint64_t tg = 0, tr = 0, tc = 0; long long ts = 0; bool ok = true;
    for (int w = 0; w < kWorkers; ++w) { tg += w_groups[w]; tr += w_rows[w]; tc += w_chunks[w]; ts += w_sum[w]; ok = ok && w_ok[w]; }
    std::printf("{\"mt_groups\": %llu, \"mt_rows\": %llu, \"mt_chunks\": %llu, \"mt_sum_v\": %lld, \"mt_ok\": %d, \"mt_emitted\": %llu}\n",
                static_cast<unsigned long long>(tg), static_cast<unsigned long long>(tr), static_cast<unsigned long long>(tc), ts, ok ? 1 : 0,
                static_cast<unsigned long long>(gs.rows_emitted.load()));
  }
  sdbg_segment_destroy(seg);
  sdbg_destroy(ctx);
  return 0;
}
