// bm25_emit.cuh -- sm_90a kernels of the match scan (sdbg_match_scan_batch_groups_min): the matches of a full-text query
// in (segment, doc) order, the page [offset, offset + limit) of them per query, optionally scored. The Stream mode of the
// search scan (duckdb_search_full_scan RunStreamingScan) for every query shape the count pass takes.
//
// The match set comes from bm25_count_kernel's emit sink (kEmit), launched twice over the same work items:
//   pass A  each item writes its match count to its own slot (item.w);
//   bases   emit_bases_kernel scans each query's item counts in (segment, first window) order into each item's first
//           ordinal, total[q] and n_out[q], on the device;
//   pass B  an item whose ordinals miss the page exits before it decodes anything; the others walk their windows again and
//           write the docs whose ordinal falls in the page, and stop once it is full.
// Scored calls then run emit_score_kernel over the page: each hit is probed in every positive list of its query, in the
// order the top-k sums them (ascending docs_count per segment), and the scores are added from 0 with __fadd_rn. Scored
// phrase scans (sdbg_phrase_scan_batch, sdbg_phrase_and_scan_batch, sdbg_phrase_groups_scan_batch) run
// phrase_score_kernel instead: the scores of each hit's positive alternatives that occur in it, summed as the phrase top-k
// sums them.
#pragma once

#include "bm25_kernels.cuh"
#include "bm25_phrase.cuh"

namespace sdbg {

struct EmitHit { float score; uint32_t doc; uint32_t seg; };   // sdbg_hit

// bm25_count_kernel's emit sink. base null: pass A.
struct EmitSink {
  uint32_t* item_n = nullptr;                    // [work items] match count of each item (item.w)
  const unsigned long long* base = nullptr;      // [work items] ordinal of each item's first match
  const unsigned long long* offset = nullptr;    // [queries] first ordinal of the page
  EmitHit* out = nullptr;                        // [queries][limit]
  uint32_t limit = 0;
  uint32_t seg = 0;                              // index of the launch's segment in the call
};

// One warp per query: the items slots[slot_off[q] .. slot_off[q + 1]) in (segment, first window) order get their first
// ordinals (an exclusive scan of item_n); total[q] is the sum, n_out[q] = min(limit, total - offset[q]), 0 past the end.
__global__ void __launch_bounds__(32) emit_bases_kernel(const uint32_t* __restrict__ item_n, const uint32_t* __restrict__ slot_off,
                                                        const uint32_t* __restrict__ slots, const unsigned long long* __restrict__ offset,
                                                        uint32_t limit, unsigned long long* __restrict__ base,
                                                        unsigned long long* __restrict__ total, uint32_t* __restrict__ n_out) {
  const uint32_t q = blockIdx.x, lane = threadIdx.x;
  const uint32_t end = slot_off[q + 1];
  unsigned long long run = 0;
  for (uint32_t i0 = slot_off[q]; i0 < end; i0 += 32u) {
    const uint32_t i = i0 + lane;
    const uint32_t slot = i < end ? slots[i] : 0u;
    const unsigned long long n = i < end ? item_n[slot] : 0u;
    unsigned long long incl = n;
#pragma unroll
    for (uint32_t o = 1; o < 32u; o <<= 1) {
      const unsigned long long t = __shfl_up_sync(kFull, incl, o);
      if (lane >= o) incl += t;
    }
    if (i < end) base[slot] = run + incl - n;
    run += __shfl_sync(kFull, incl, 31);
  }
  if (lane == 0) {
    const unsigned long long off = offset[q];
    total[q] = run;
    n_out[q] = off < run ? uint32_t(min(run - off, static_cast<unsigned long long>(limit))) : 0u;
  }
}

constexpr uint32_t kEmitScoreThreads = 256;
constexpr uint32_t kEmitScoreRun = 8;   // hits per lane: a warp scores 32 * kEmitScoreRun consecutive hits
constexpr uint32_t kEmitScoreHits = kEmitScoreThreads * kEmitScoreRun;

struct EmitScoreParams {
  const PostingsDev* segs;    // [segments]
  const QTermDev* qterms;     // [segment][term], each query's terms by ascending docs_count in that segment
  const uint32_t* qterm_off;  // [queries + 1]
  uint32_t n_terms;           // qterm_off[queries]
  uint32_t blocks_per_query;  // ceil(limit / kEmitScoreHits)
  uint32_t limit;
  EmitHit* out;               // [queries][limit], n_out[q] hits each, ascending (segment, doc)
  const uint32_t* n_out;
};

// Frequency of doc d in the list of qt, or false when the list does not hold it. hint: a block of the list not behind
// d's block, moved to the block searched (a lane's docs ascend, so it only moves forward).
__device__ __forceinline__ bool emit_probe(const PostingsDev& S, const QTermDev& qt, uint32_t d, uint32_t& hint, uint32_t& f) {
  const uint4* B = S.blocks + qt.blk_begin;
  const uint32_t n = qt.nblk;
  if (n == 0u) return false;
  const uint32_t l = find_block_from(B, 0u, n, min(hint, n - 1u), d);
  hint = min(l, n - 1u);
  if (l >= n) return false;
  const uint4 desc = __ldg(B + l);
  if (d <= desc.z) return false;                       // d lies between two blocks
  uint32_t idx = 0;
  if (!block_find_doc(S, desc, qt.blk_begin + l, d, idx)) return false;
  if (!freq_at(S.arena, desc, idx, f))                 // StreamVByte frequencies: scalar walk
    f = svb_value_at(reinterpret_cast<const uint8_t*>(S.arena + desc.x + desc_fdelta(desc.w)), desc_len(desc.w), idx, false, false, 0u, &idx);
  return true;
}

// Grid: queries x blocks_per_query. Lane l of a warp scores hits first + l + 32 j (j < kEmitScoreRun) of its query: the
// sum of bm25() over the positive lists that hold the doc, in qterms order, from 0. A list that misses the doc adds
// nothing (for a conjunction every list holds it; excluded lists are not among the positive ones).
__global__ void __launch_bounds__(kEmitScoreThreads) emit_score_kernel(EmitScoreParams P) {
  __shared__ uint32_t hint[kMaxQueryTerms][kEmitScoreThreads];
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const uint32_t q = blockIdx.x / P.blocks_per_query, b = blockIdx.x % P.blocks_per_query;
  const uint32_t n = P.n_out[q];
  const uint32_t first = b * kEmitScoreHits + warp * (32u * kEmitScoreRun);
  if (first >= n) return;   // no block-wide barrier below
  const uint32_t t0 = P.qterm_off[q], nt = P.qterm_off[q + 1] - t0;
  EmitHit* H = P.out + size_t(q) * P.limit;
  uint32_t cur = 0xFFFFFFFFu;   // segment of this lane's hints
  for (uint32_t j = 0; j < kEmitScoreRun; ++j) {
    const uint32_t i = first + 32u * j + lane;
    if (i >= n) break;
    const uint32_t d = H[i].doc, si = H[i].seg;
    if (si != cur) {
      for (uint32_t u = 0; u < nt; ++u) hint[u][tid] = 0u;
      cur = si;
    }
    const PostingsDev& S = P.segs[si];
    const QTermDev* qt = P.qterms + size_t(si) * P.n_terms + t0;
    float s = 0.f;
    for (uint32_t u = 0; u < nt; ++u) {
      uint32_t f = 0, h = hint[u][tid];
      const bool found = emit_probe(S, qt[u], d, h, f);
      hint[u][tid] = h;
      if (found) s = __fadd_rn(s, bm25(f, load_norm(S.norms, S.norm_width, d), qt[u].c0, qt[u].norm_const, qt[u].norm_length));
    }
    H[i].score = s;
  }
}

struct PhraseScoreParams {
  const PostingsDev* segs;    // [segments]
  const PhraseSink* sinks;    // [segments]: positions, that segment's slots and alternative tables, offsets, masks, consts
  uint32_t blocks_per_query;  // ceil(limit / kEmitScoreThreads)
  uint32_t limit;
  EmitHit* out;               // [queries][limit], n_out[q] hits each
  const uint32_t* n_out;
};

// Grid: queries x blocks_per_query, one thread per hit: phrase_clauses of the hit's doc over its segment's alternative
// table, scored as the phrase top-k scores it (negated entries skipped, alternatives of frequency 0 add nothing). At least 4 CTAs per SM (64 registers): no spill around the position walk.
__global__ void __launch_bounds__(kEmitScoreThreads, 4) phrase_score_kernel(PhraseScoreParams P) {
  const uint32_t q = blockIdx.x / P.blocks_per_query;
  const uint32_t i = (blockIdx.x % P.blocks_per_query) * kEmitScoreThreads + threadIdx.x;
  if (i >= P.n_out[q]) return;
  EmitHit& h = P.out[size_t(q) * P.limit + i];
  const uint32_t d = h.doc;
  const PostingsDev& S = P.segs[h.seg];
  const PhraseSink& F = P.sinks[h.seg];
  float s;
  phrase_clauses<true>(S, F, phrase_query(F, q), d, PhraseMode::score_match, s);   // the hit matched: every group holds
  h.score = s;
}

}  // namespace sdbg
