// bm25_count.cuh -- sm_90a kernel for the Count mode of the search scan: the number of docs that match a full-text query
// (OR / AND of 1..16 terms), minus deleted docs, minus docs that fail the pushed column predicate, minus the docs of up to
// 16 excluded terms. Nothing is scored: the kernel reads block descriptors, doc payloads, the deleted bitmap, the filter
// column and the excluded lists' doc payloads -- never frequencies, norms or block-max pairs.
//
// Mapping: one CTA per work item {query, first window, windows} of one segment. A window is kCountWindow docs aligned to
// a multiple of kCountWindow, held as a bitmap `acc` in shared memory (bit i = doc ws + i). Because windows are aligned,
// word i of `acc` is word ws / 32 + i of the deleted-docs bitmap.
//   OR   warps decode every positive list's blocks that overlap the window and set their docs in `acc`.
//   AND  the shortest list fills `acc`; each further list (ascending docs_count) decodes only the blocks whose doc range
//        (prev_last, last_doc] holds a bit of `acc`, sets their docs in `tmp`, then acc &= tmp; the window ends early
//        once `acc` is empty.
//   GROUPS  an AND of OR groups (kGroups): the lead group (smallest summed docs_count) fills `acc` like an OR; each further
//        group ORs into `tmp` the docs of its lists' blocks whose range holds a bit of `acc`, then acc &= tmp, with the
//        same early end. A group that needs m >= 2 of its s lists (`2 of (a | b | c)`) leads with its s - m + 1 shortest
//        lists; it decodes each list into `tmp` the same way, adds it into a bit-sliced counter, then acc &= counter >= m.
//   NOT  the excluded lists' blocks whose range holds a bit of `acc` are decoded and their docs cleared.
// Then acc &= ~deleted, the filter chain runs per remaining bit, and popcounts are summed: one 64-bit atomicAdd per CTA.
// With the chain's zone verdicts (ChainDev::zone), a window whose zones are all dead is skipped before any list is
// decoded, the docs of dead zones are cleared before any column is read, and docs of pass zones skip the chain.
// The facet pass (kFacet, bm25_facet.cuh) also counts each remaining bit in its key's shared-memory bin; the aggregate pass
// (kAgg, bm25_agg.cuh) also adds its value to its key's shared-memory cell. The match scan (kEmit, bm25_emit.cuh) counts
// each item's matches, then writes the docs whose ordinal falls in the query's page.
// A window that no positive list reaches (OR), that the shortest list does not reach (AND) or that no list of the lead
// group reaches (GROUPS) is never touched: the CTA
// jumps to the window of the next block's first possible doc, so a sparse query costs in proportion to its blocks.
#pragma once

#include "bm25_kernels.cuh"
#include "bm25_agg.cuh"
#include "bm25_emit.cuh"
#include "bm25_facet.cuh"
#include "bm25_phrase.cuh"
#include "bm25_sort.cuh"

namespace sdbg {

constexpr uint32_t kCountWindowLog = 16;
constexpr uint32_t kCountWindow = 1u << kCountWindowLog;   // docs per window
constexpr uint32_t kCountWords = kCountWindow / 32u;        // 2048 words: an 8 KB bitmap
constexpr uint32_t kCountThreads = 256;
constexpr uint32_t kCountWarps = kCountThreads / 32u;
constexpr uint32_t kCountMaxLists = 2u * kMaxQueryTerms;   // positive + excluded lists of one query

struct CountParams {
  PostingsDev seg;              // arena, blocks, deleted, n_docs
  ChainDev filt;
  // Per query q of this segment: positive lists lists[term_off[q] .. term_off[q + 1]) as {first BlockDesc, blocks},
  // ascending by docs_count; excluded lists lists[n_pos + excl_off[q] .. n_pos + excl_off[q + 1]) (0 blocks: a term the
  // segment does not hold). excl_off null: no exclusions.
  const uint2* lists;
  const uint32_t* term_off;
  const uint32_t* excl_off;
  // kGroups: query q's positive lists form consecutive OR groups, lead group first, each group's lists by ascending
  // docs_count; group g of q ends (exclusive, relative to term_off[q]) at grp_end[grp_off[q] + g] & 0xFF, and needs
  // m_g = (grp_end[grp_off[q] + g] >> 8) + 1 of its lists to hold a doc. Per segment, since the lead group and the list
  // order depend on it. A group with m_g >= 2 counts in a bit-sliced counter of bits(m_g) planes of kCountWords words in
  // dynamic shared memory; the launch provides the batch's largest.
  const uint32_t* grp_end = nullptr;
  const uint32_t* grp_off = nullptr;
  uint32_t n_pos;               // term_off[n_queries]
  const uint4* work;            // {query, first window, windows, 0}
  unsigned long long* counts;   // per query, summed over items and segments
  SortSink sort;                // kSort: the sorted scan's sink (work item .w = its output slot)
  FacetSink facet;              // kFacet: the facet pass's sink
  AggSink agg;                  // kAgg: the aggregate pass's sink
  EmitSink emit;                // kEmit: the match scan's sink (work item .w = its count and base slot)
  PhraseSink phrase;            // kPhrase: the phrase check and its top-k (work item .w = its output slot)
};

__device__ __forceinline__ uint32_t warp_min(uint32_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(kFull, v, o));
  return v;
}

// Sets (clear = false) or clears (clear = true) the bits of block `d`'s docs that fall in the window [ws, ws + W) of
// `bm`. Whole warp. Bitset blocks are merged word by word without expanding them; the other encodings are decoded.
// Returns the block's first doc past the window (0xFFFFFFFF: none), where the next window of a straddling block starts.
__device__ __forceinline__ uint32_t block_to_bitmap(const uint4* arena, const uint4& d, uint32_t lane, uint32_t* stage,
                                                    uint32_t ws, uint32_t* bm, bool clear) {
  const long long wend = static_cast<long long>(ws) + kCountWindow;
  uint32_t beyond = 0xFFFFFFFFu;
  if (desc_doc_enc(d.w) == 4u) {   // de_for_bitset: bit j of the payload <=> doc prev + j
    const uint32_t* w = reinterpret_cast<const uint32_t*>(arena + d.x);
    const uint32_t chunks = 2u * desc_words(d.w);
    for (uint32_t c = lane; c < chunks; c += 32u) {
      const uint32_t v = __ldg(w + c);
      const long long r = static_cast<long long>(d.z) + 32ll * c - static_cast<long long>(ws);   // bit 0 of v, window-relative
      if (v == 0u || r <= -32) continue;
      if (r + 31 >= static_cast<long long>(kCountWindow)) {                                      // bits past the window
        const uint32_t past = r >= static_cast<long long>(kCountWindow) ? v : v & (0xFFFFFFFFu << uint32_t(kCountWindow - r));
        if (past) beyond = min(beyond, uint32_t(wend - static_cast<long long>(kCountWindow) + r) + uint32_t(__ffs(past) - 1));
        if (r >= static_cast<long long>(kCountWindow)) continue;
      }
      const uint32_t sh = static_cast<uint32_t>(r & 31);
      const long long wi = r >> 5;                                                               // floor
      const uint32_t lo = v << sh, hi = sh ? v >> (32u - sh) : 0u;
      if (wi >= 0 && lo) { if (clear) atomicAnd(&bm[wi], ~lo); else atomicOr(&bm[wi], lo); }
      if (wi + 1 < static_cast<long long>(kCountWords) && hi) { if (clear) atomicAnd(&bm[wi + 1], ~hi); else atomicOr(&bm[wi + 1], hi); }
    }
    return warp_min(beyond);
  }
  uint32_t doc[4];
  decode_docs(arena, d, lane, stage, doc);
  const uint32_t len = desc_len(d.w);
  uint32_t word = 0xFFFFFFFFu, bits = 0u;   // a lane's four docs ascend: one atomic per distinct word
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (4u * lane + j >= len) continue;
    const uint32_t rel = doc[j] - ws;
    if (rel >= kCountWindow) {
      if (static_cast<long long>(doc[j]) >= wend) beyond = min(beyond, doc[j]);
      continue;
    }
    if ((rel >> 5) != word) {
      if (bits) { if (clear) atomicAnd(&bm[word], ~bits); else atomicOr(&bm[word], bits); }
      word = rel >> 5; bits = 0u;
    }
    bits |= 1u << (rel & 31u);
  }
  if (bits) { if (clear) atomicAnd(&bm[word], ~bits); else atomicOr(&bm[word], bits); }
  return warp_min(beyond);
}

// Does `bm` hold a bit for a doc in (prev_last, last_doc] within the window [ws, wlast]? Whole warp.
__device__ __forceinline__ bool range_has_bits(const uint32_t* bm, const uint4& d, uint32_t ws, uint32_t wlast, uint32_t lane) {
  const uint32_t a = max(d.z + 1u, ws) - ws, b = min(d.y, wlast) - ws;   // d.z < wlast, d.y >= ws: a <= b
  const uint32_t wa = a >> 5, wb = b >> 5;
  uint32_t any = 0u;
  for (uint32_t i = wa + lane; i <= wb; i += 32u) {
    uint32_t v = bm[i];
    if (i == wa) v &= 0xFFFFFFFFu << (a & 31u);
    if (i == wb) v &= 0xFFFFFFFFu >> (31u - (b & 31u));
    any |= v;
  }
  return __any_sync(kFull, any != 0u);
}

// The clause check inlined into the phrase instantiations spills under ptxas's own register choice (the phrase sink, the
// sorted scan's and the facet pass's); at least 4 CTAs per SM (64 registers) none does. Every other instantiation has no
// minimum.
constexpr int kPhraseMinBlocks = 4;

// kAnd: conjunction (else disjunction). kGroups: conjunction of OR groups (CountParams::grp_end). The term loops are not
// unrolled: 1..16 terms share one instantiation.
// kSort: the sorted scan (bm25_sort.cuh). Instead of popcounting, every surviving doc's sort key enters a buffer of
// P.sort.cap keys in dynamic shared memory; a full buffer is sorted and cut to the k best, whose k-th hi raises the
// query's threshold word. With a threshold word (pruning level >= 1), a key whose hi is below the threshold never enters,
// and with a zonemap each window is judged before any list is decoded: a window none of whose zones can reach the
// threshold is skipped, and in a kept window the docs of such zones are cleared before the column is read. The item's
// k best go to output slot item.w.
// kFacet: the facet pass (bm25_facet.cuh). Besides the popcount, every surviving doc's key is counted in the item's
// histogram of P.facet.span u32 bins in dynamic shared memory, flushed to the query's row of P.facet.counts at the end.
// kAgg: the aggregate pass (bm25_agg.cuh). Besides the popcount, every surviving doc's value is added to its key's cell
// among the item's P.agg.key.span + 1 cells in dynamic shared memory (ungrouped: to the thread's register cell), flushed
// to the query's output cells at the end.
// kEmit: the match scan (bm25_emit.cuh). Pass A (P.emit.base null) writes the item's match count to
// P.emit.item_n[item.w] instead of adding it to P.counts. Pass B ranks the surviving docs of each window in doc order:
// each thread takes kCountWords / kCountThreads consecutive words, and a block-wide exclusive scan of their popcounts
// gives each doc its ordinal, base[item.w] plus the matches of the item's earlier windows; the docs whose ordinal lies in
// [offset[q], offset[q] + limit) go to their row of P.emit.out, unscored. An item whose ordinals miss the page exits
// before it decodes anything, and an item stops after the window that fills the page.
// kPhrase (on any candidate shape: the AND, the flat OR or the OR groups (m >= 1) of the alternatives' proxy terms): the
// alternative check (phrase_clauses, bm25_phrase.cuh). Every doc that survives the candidate scan, the exclusions, the
// deleted docs and the filter chain is probed, entry after entry of the query's alternative table, in each slot's list
// for its positions; a doc that fails its groups is dropped, the others are counted and, with P.phrase.cap, scored as the
// sum of their matching positive alternatives' scores and kept in a buffer of P.phrase.cap keys in dynamic shared memory
// as the sorted scan keeps its keys; the item's k best go to slot item.w. Without a score the entries of groups that the
// candidate scan guarantees, or that an earlier entry satisfied, are skipped.
// kPhrase with one other sink: with kFacet, kAgg or kEmit the clause check is a stage that narrows `acc` after the
// exclusions (deleted docs, filter chain, then the check per surviving bit, written back), so the sink reads only
// matches and emit passes A and B see the same set. With kSort it runs inside the sink, on a doc whose key has passed
// s_thr: a doc that cannot enter the buffer is never probed for positions.
// The sinks take kGroups queries: the groups narrow `acc` before the sink reads the column, and the bit-sliced counter
// planes follow the sink's region of dynamic shared memory (16 * cap B of the sorted scan or the phrase sink, 4 * span B
// or agg_cells_bytes(span), rounded up to 16 B).
template <bool kAnd, bool kGroups = false, bool kSort = false, bool kFacet = false, bool kAgg = false, bool kEmit = false,
          bool kPhrase = false>
__global__ void __launch_bounds__(kCountThreads, kPhrase ? kPhraseMinBlocks : 0) bm25_count_kernel(CountParams P) {
  static_assert(!(kAnd && kGroups), "groups generalise the conjunction");
  static_assert(!(kFacet && kSort), "the facet pass has its own sink");
  static_assert(!(kAgg && (kSort || kFacet)), "the aggregate pass has its own sink");
  static_assert(!(kEmit && (kSort || kFacet || kAgg)), "the match scan has its own sink");
  static_assert(!kPhrase || int(kSort) + int(kFacet) + int(kAgg) + int(kEmit) <= 1, "the phrase check serves one sink");
  constexpr bool kPhraseSink = kPhrase && !kSort && !kFacet && !kAgg && !kEmit;   // count / top-k of phrase matches
  constexpr bool kPhraseStage = kPhrase && (kFacet || kAgg || kEmit);           // narrows acc before the sink
  __shared__ uint32_t acc[kCountWords];
  __shared__ uint32_t tmp[kAnd || kGroups ? kCountWords : 1];
  __shared__ uint32_t stage[kCountWarps][128];
  // per list: blocks [s_cur, s_end) overlap the current window; s_next = first block that reaches past it
  __shared__ uint32_t s_cur[kCountMaxLists], s_end[kCountMaxLists], s_next[kCountMaxLists];
  // per lead list: first doc of block s_next past the window, when that block straddled it and was decoded (else 0)
  __shared__ uint32_t s_resume[kCountMaxLists];
  __shared__ uint2 s_list[kCountMaxLists];
  __shared__ uint32_t s_gend[kGroups ? kMaxQueryTerms : 1];
  __shared__ uint32_t s_ws, s_done;
  __shared__ unsigned long long s_sum[kCountWarps];
  __shared__ unsigned long long s_thr[1];   // kSort: this item's best known k-th hi (kPhrase: k-th key)
  __shared__ uint32_t s_fill[1];  // kSort: keys in the buffer (kFacet: NULL keys)
  // the window's zones that hold docs that can count: not dead for the filter chain and (kSort) able to reach s_thr;
  // the zones where the chain holds for every row; (kSort) the zones that can reach s_thr
  __shared__ uint32_t s_zmask[2], s_pmask[2], s_smask[2];
  // kSort: hi[cap] | lo[cap]; kFacet: the u32 bins, padded to 16 B; kAgg: the cells; then (kGroups) the bit-sliced
  // counter planes
  extern __shared__ unsigned long long sort_buf[];
  uint32_t* const bins = reinterpret_cast<uint32_t*>(sort_buf);
  AggSmemCell* const cells = reinterpret_cast<AggSmemCell*>(sort_buf);

  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const uint4 item = P.work[blockIdx.x];
  const uint32_t q = item.x, w_end = item.y + item.z;   // windows [item.y, w_end)
  const uint32_t n_pos = P.term_off[q + 1] - P.term_off[q];
  const uint32_t n_excl = P.excl_off ? P.excl_off[q + 1] - P.excl_off[q] : 0u;
  const uint32_t n_lists = n_pos + n_excl;
  const uint32_t n_groups = kGroups ? P.grp_off[q + 1] - P.grp_off[q] : 0u;
  if (kGroups && tid < n_groups) s_gend[tid] = P.grp_end[P.grp_off[q] + tid];
  // lists that decide which windows hold matches; for groups the lead group's s - m + 1 shortest (a doc that m of its s
  // lists hold is in one of them)
  const uint32_t gend0 = kGroups ? P.grp_end[P.grp_off[q]] : 0u;
  const uint32_t n_lead = kGroups ? (gend0 & 0xFFu) - (gend0 >> 8) : kAnd ? 1u : n_pos;
  const uint4* const B = P.seg.blocks;
  const uint32_t del_words = (P.seg.n_docs >> 5) + 2u;   // (n_docs + 32) / 32 + 1, the host bitmap's words, without wrapping
  // kEmit pass B: the ordinal of the item's next match and the end of the query's page
  unsigned long long e_run = 0, e_end = 0;
  if constexpr (kEmit) {
    if (P.emit.base) {
      const unsigned long long b = P.emit.base[item.w], n = P.emit.item_n[item.w], off = P.emit.offset[q];
      e_run = b;
      e_end = off + P.emit.limit;
      if (b + n <= off || b >= e_end) return;   // the whole block: nothing has been read or synchronised yet
    }
  }

  if (tid < n_lists) {
    const uint2 l = tid < n_pos ? P.lists[P.term_off[q] + tid] : P.lists[P.n_pos + P.excl_off[q] + (tid - n_pos)];
    s_list[tid] = l;
    s_resume[tid] = 0u;
    // first block whose last doc reaches the item's first window
    s_next[tid] = l.y ? find_block_from(B + l.x, 0u, l.y, 0u, item.y << kCountWindowLog) : 0u;
  }
  unsigned long long count = 0;
  bool oor = false;                                     // kFacet, kAgg: this thread met a key outside the bins
  AggSmemCell mine{};                                   // kAgg without a key column: this thread's group
  uint32_t ws = item.y << kCountWindowLog;              // start of the window being looked at
  uint32_t judged = 0, skipped = 0;                     // kSort: windows judged / skipped by the zonemap
  if constexpr (kSort) {
    for (uint32_t i = tid; i < 2u * P.sort.cap; i += kCountThreads) sort_buf[i] = 0ull;
    if (tid == 0) { s_thr[0] = 0ull; s_fill[0] = 0u; }
  }
  if constexpr (kPhraseSink) {
    for (uint32_t i = tid; i < 2u * P.phrase.cap; i += kCountThreads) sort_buf[i] = 0ull;
    if (tid == 0) { s_thr[0] = P.phrase.cap ? P.phrase.thr[q] : 0ull; s_fill[0] = 0u; }
  }
  if constexpr (kFacet) {
    for (uint32_t i = tid; i < P.facet.span; i += kCountThreads) bins[i] = 0u;
    if (tid == 0) s_fill[0] = 0u;
  }
  if constexpr (kAgg) {
    for (uint32_t i = tid; i < agg_cells_bytes(P.agg.key.span) / 4u; i += kCountThreads) bins[i] = 0u;
  }
  __syncthreads();
  for (;;) {
    // ---- next window: the first possible doc of the lead lists' current blocks ----
    if (tid == 0) {
      uint32_t nxt = 0xFFFFFFFFu;
      bool any = false;
      for (uint32_t i = 0; i < n_lead; ++i) {
        const uint2 l = s_list[i];
        if (s_next[i] >= l.y) continue;
        const uint4 d = __ldg(B + l.x + s_next[i]);
        nxt = min(nxt, max(max(d.z + 1u, ws), s_resume[i]));
        any = true;
      }
      s_done = (!any || (nxt >> kCountWindowLog) >= w_end) ? 1u : 0u;
      s_ws = (nxt >> kCountWindowLog) << kCountWindowLog;
      if constexpr (kSort) {
        if (P.sort.thr) s_thr[0] = max(s_thr[0], *reinterpret_cast<volatile unsigned long long*>(P.sort.thr + q));
      }
      if constexpr (kPhraseSink) {
        if (P.phrase.cap) s_thr[0] = max(s_thr[0], *reinterpret_cast<volatile unsigned long long*>(P.phrase.thr + q));
      }
    }
    __syncthreads();
    if (s_done) break;
    ws = s_ws;
    const uint32_t wlast = ws + (kCountWindow - 1u);
    if (tid < n_lists) {
      const uint2 l = s_list[tid];
      const uint4* LB = B + l.x;
      uint32_t c = s_next[tid], e = l.y;
      if (c < l.y) c = find_block_from(LB, c, l.y, c, ws);
      if (c < l.y && wlast != 0xFFFFFFFFu) e = find_block_from(LB, c, l.y, c, wlast + 1u);
      s_cur[tid] = c;
      s_next[tid] = e;
      s_resume[tid] = 0u;
      s_end[tid] = (e < l.y && __ldg(&LB[e].z) < wlast) ? e + 1u : e;   // block e straddles the window's end
    }
    // Zone verdicts (the sort column's zonemap, the filter chain's): zones zb .. zb + 32 hold the window's rows
    // ws - 1 .. ws + 65534 (32 zones for ws = 0)
    const uint32_t zb = ws == 0u ? 0u : (ws >> 11) - 1u;
    const bool sort_zoned = kSort && P.sort.zone;
    const bool zoned = sort_zoned || P.filt.zone;
    if (zoned && tid < 64u) {
      const uint32_t z = zb + tid;
      const bool in = tid < (ws == 0u ? 32u : 33u);
      bool comp = in, pass = false;
      if constexpr (kSort) {
        if (P.sort.zone) comp = in && sort_zone_bound(P.sort, z) >= s_thr[0];
      }
      const uint32_t sm = __ballot_sync(kFull, comp);
      if (P.filt.zone) {
        const uint8_t v = in && z < P.filt.n_zones ? P.filt.zone[z] : kZoneDead;   // zones past the segment hold no doc
        comp = comp && v != kZoneDead;
        pass = v == kZonePass;
      }
      const uint32_t m = __ballot_sync(kFull, comp), p = __ballot_sync(kFull, pass);
      if (lane == 0) { s_zmask[warp] = m; s_pmask[warp] = p; s_smask[warp] = sm; }
    }
    for (uint32_t i = tid; i < kCountWords; i += kCountThreads) acc[i] = 0u;
    __syncthreads();
    bool skip = false;
    if (zoned) {
      skip = (s_zmask[0] | s_zmask[1]) == 0u;
      if (sort_zoned) { ++judged; skipped += (s_smask[0] | s_smask[1]) == 0u; }
    }
    // the bits of acc word i whose zone is set in the zone mask zm: bit 0 is row ws + 32i - 1, which starts a zone when
    // ws + 32i does
    auto zone_bits = [&](const uint32_t* zm, uint32_t i) {
      auto has = [&](uint32_t zr) { return (zm[zr >> 5] >> (zr & 31u)) & 1u; };
      const uint32_t d0 = ws + 32u * i;
      uint32_t bits = has((d0 >> 11) - zb) ? 0xFFFFFFFEu : 0u;
      if (d0 != 0u && has(((d0 - 1u) >> 11) - zb)) bits |= 1u;
      return bits;
    };
    // the docs of word i's bits v that pass the filter chain: dead zones are cleared first, pass zones are not read
    auto chain_bits = [&](uint32_t v, uint32_t i) {
      if (v && zoned) v &= zone_bits(s_zmask, i);
      if (v && P.filt.ps.n) {
        const uint32_t check = P.filt.zone ? v & ~zone_bits(s_pmask, i) : v;
        for (uint32_t r = check; r; r &= r - 1u) {
          const uint32_t bit = __ffs(r) - 1u;
          if (!preds_row(P.filt.ps, uint64_t(ws + 32u * i + bit) - 1u)) v &= ~(1u << bit);
        }
      }
      return v;
    };
    if (!skip) {

    // Blocks [s_cur, s_end) of lists [lo, hi) spread over the warps; `filter`: only blocks whose range holds a bit of acc.
    auto run_lists = [&](uint32_t lo, uint32_t hi, uint32_t* bm, bool clear, bool filter) {
      const uint32_t li = lo + lane;
      const uint32_t n = li < hi ? s_end[li] - s_cur[li] : 0u;
      const uint32_t incl = warp_incl_scan(n, lane);
      const uint32_t total = __shfl_sync(kFull, incl, 31);
      for (uint32_t it = warp; it < total; it += kCountWarps) {
        const uint32_t src = __ffs(__ballot_sync(kFull, incl > it)) - 1u;
        const uint32_t before = __shfl_sync(kFull, incl - n, src);
        const uint32_t li2 = lo + src, blk = s_cur[li2] + (it - before);
        const uint4 d = __ldg(B + s_list[li2].x + blk);
        if (filter && !range_has_bits(acc, d, ws, wlast, lane)) continue;
        const uint32_t beyond = block_to_bitmap(P.seg.arena, d, lane, stage[warp], ws, bm, clear);
        if (lane == 0 && blk == s_next[li2]) s_resume[li2] = beyond;   // the block that straddles the window's end
      }
    };

    run_lists(0u, n_lead, acc, false, false);
    __syncthreads();
    bool live = true;
    if constexpr (kAnd) {
      for (uint32_t t = 1; t < n_pos; ++t) {
        for (uint32_t i = tid; i < kCountWords; i += kCountThreads) tmp[i] = 0u;
        __syncthreads();
        run_lists(t, t + 1u, tmp, false, true);
        __syncthreads();
        uint32_t nz = 0u;
        for (uint32_t i = tid; i < kCountWords; i += kCountThreads) { const uint32_t v = acc[i] & tmp[i]; acc[i] = v; nz |= v; }
        if (!__syncthreads_or(nz != 0u)) { live = false; break; }
      }
    }
    if constexpr (kGroups) {
      // the lead group is already in acc unless it needs m >= 2 of its lists
      for (uint32_t g = (gend0 >> 8) ? 0u : 1u; g < n_groups; ++g) {
        const uint32_t lo = g ? s_gend[g - 1] & 0xFFu : 0u, hi = s_gend[g] & 0xFFu, m = (s_gend[g] >> 8) + 1u;
        uint32_t nz = 0u;
        if (m == 1u) {
          for (uint32_t i = tid; i < kCountWords; i += kCountThreads) tmp[i] = 0u;
          __syncthreads();
          run_lists(lo, hi, tmp, false, true);
          __syncthreads();
          for (uint32_t i = tid; i < kCountWords; i += kCountThreads) { const uint32_t v = acc[i] & tmp[i]; acc[i] = v; nz |= v; }
        } else {
          // at least m of the lists: each list's bitmap is added into a saturating bit-sliced counter (plane p = bit p)
          const uint32_t np = 32u - __clz(m);
          uint32_t* const plane = bins + (kSort ? 4u * P.sort.cap : kFacet ? (P.facet.span + 3u) & ~3u
                                          : kAgg ? agg_cells_bytes(P.agg.key.span) / 4u : kPhraseSink ? 4u * P.phrase.cap : 0u);
          for (uint32_t i = tid; i < np * kCountWords; i += kCountThreads) plane[i] = 0u;
          for (uint32_t i = tid; i < kCountWords; i += kCountThreads) tmp[i] = 0u;
          for (uint32_t li = lo; li < hi; ++li) {
            __syncthreads();
            run_lists(li, li + 1u, tmp, false, true);
            __syncthreads();
            for (uint32_t i = tid; i < kCountWords; i += kCountThreads) {
              uint32_t c = tmp[i];
              tmp[i] = 0u;
              for (uint32_t p = 0; p < np && c; ++p) { const uint32_t t = plane[p * kCountWords + i] & c; plane[p * kCountWords + i] ^= c; c = t; }
              if (c) for (uint32_t p = 0; p < np; ++p) plane[p * kCountWords + i] |= c;   // 2^np - 1 >= m: saturate
            }
          }
          __syncthreads();
          for (uint32_t i = tid; i < kCountWords; i += kCountThreads) {
            uint32_t gt = 0u, eq = 0xFFFFFFFFu;   // counter > m / == m on the bits above p
            for (uint32_t p = np; p-- > 0;) {
              const uint32_t v = plane[p * kCountWords + i];
              if ((m >> p) & 1u) eq &= v;
              else { gt |= eq & v; eq &= ~v; }
            }
            const uint32_t v = acc[i] & (gt | eq);
            acc[i] = v; nz |= v;
          }
        }
        if (!__syncthreads_or(nz != 0u)) { live = false; break; }
      }
    }
    if (live && n_excl) {
      run_lists(n_pos, n_lists, acc, true, true);
      __syncthreads();
    }
    if constexpr (kPhraseStage) {
      if (live) {
        const uint32_t wbase = ws >> 5;
        const PhraseQuery PQ = phrase_query(P.phrase, q);
        float unused;
        for (uint32_t i = tid; i < kCountWords; i += kCountThreads) {
          uint32_t v = acc[i];
          if (v && P.seg.deleted && wbase + i < del_words) v &= ~__ldg(P.seg.deleted + wbase + i);
          v = chain_bits(v, i);
          for (uint32_t r = v; r; r &= r - 1u) {
            const uint32_t bit = __ffs(r) - 1u;
            if (!phrase_clauses<!kAnd>(P.seg, P.phrase, PQ, ws + 32u * i + bit, PhraseMode::check, unused)) v &= ~(1u << bit);
          }
          acc[i] = v;
        }
        __syncthreads();
      }
    }
    if (live && !kSort && !kPhraseSink && !(kEmit && P.emit.base)) {
      const uint32_t wbase = ws >> 5;
      for (uint32_t i = tid; i < kCountWords; i += kCountThreads) {
        uint32_t v = acc[i];
        if constexpr (!kPhraseStage) {   // else the stage has applied them
          if (v && P.seg.deleted && wbase + i < del_words) v &= ~__ldg(P.seg.deleted + wbase + i);
          v = chain_bits(v, i);
        }
        if constexpr (kFacet) {
          for (uint32_t r = v; r; r &= r - 1u) oor |= facet_add(P.facet, ws + 32u * i + (__ffs(r) - 1u), bins, &s_fill[0]);
        }
        if constexpr (kAgg) {
          for (uint32_t r = v; r; r &= r - 1u) oor |= agg_add(P.agg, ws + 32u * i + (__ffs(r) - 1u), cells, mine);
        }
        count += __popc(v);
      }
    }
    if constexpr (kEmit) {
      if (live && P.emit.base) {
        constexpr uint32_t kRun = kCountWords / kCountThreads;
        const uint32_t wbase = ws >> 5, i0 = tid * kRun;
        uint32_t v[kRun], n = 0;
#pragma unroll
        for (uint32_t j = 0; j < kRun; ++j) {
          uint32_t x = acc[i0 + j];
          if constexpr (!kPhraseStage) {
            if (x && P.seg.deleted && wbase + i0 + j < del_words) x &= ~__ldg(P.seg.deleted + wbase + i0 + j);
            x = chain_bits(x, i0 + j);
          }
          v[j] = x;
          n += __popc(v[j]);
        }
        const uint32_t incl = warp_incl_scan(n, lane);
        if (lane == 31u) s_sum[warp] = incl;   // s_sum is free until the end of the kernel
        __syncthreads();
        unsigned long long before = 0, all = 0;
        for (uint32_t w = 0; w < kCountWarps; ++w) { before += w < warp ? s_sum[w] : 0ull; all += s_sum[w]; }
        unsigned long long r = e_run + before + (incl - n);   // ordinal of this thread's first doc
        const unsigned long long off = P.emit.offset[q];
        if (r < e_end && r + n > off) {
          EmitHit* out = P.emit.out + size_t(q) * P.emit.limit;
#pragma unroll
          for (uint32_t j = 0; j < kRun; ++j)
            for (uint32_t x = v[j]; x && r < e_end; x &= x - 1u, ++r)
              if (r >= off) out[r - off] = EmitHit{0.f, ws + 32u * (i0 + j) + uint32_t(__ffs(x) - 1), P.emit.seg};
        }
        e_run += all;
      }
    }
    if constexpr (kSort) {
      if (live) {
        const uint32_t wbase = ws >> 5, cap = P.sort.cap;
        PhraseQuery PQ{};
        if constexpr (kPhrase) PQ = phrase_query(P.phrase, q);
        unsigned long long* hi = sort_buf;
        unsigned long long* lo = sort_buf + cap;
        for (uint32_t base = 0; base < kCountWords; base += kCountThreads) {   // uniform trip count
          const uint32_t i = base + tid;
          uint32_t v = acc[i];
          if (v && P.seg.deleted && wbase + i < del_words) v &= ~__ldg(P.seg.deleted + wbase + i);
          v = chain_bits(v, i);
          for (;;) {   // a full buffer is cut to the k best and the remaining bits go on
            const unsigned long long thr = s_thr[0];
            for (; v; v &= v - 1u) {
              const uint32_t doc = ws + 32u * i + (__ffs(v) - 1u);
              const ulonglong2 key = sort_key(P.sort, doc);
              if (key.x < thr) continue;
              if constexpr (kPhrase) {
                float unused;
                if (!phrase_clauses<!kAnd>(P.seg, P.phrase, PQ, doc, PhraseMode::check, unused)) continue;
              }
              const uint32_t slot = atomicAdd(&s_fill[0], 1u);
              if (slot >= cap) break;
              hi[slot] = key.x; lo[slot] = key.y;
            }
            if (!__syncthreads_or(v != 0u)) break;
            const unsigned long long kth = sort_select(hi, lo, cap, P.sort.k, &s_fill[0]);
            if (P.sort.thr && tid == 0 && kth > s_thr[0]) { s_thr[0] = kth; atomicMax(P.sort.thr + q, kth); }
            __syncthreads();
          }
        }
      }
    }
    if constexpr (kPhraseSink) {
      if (live) {
        const PhraseSink& F = P.phrase;
        const uint32_t wbase = ws >> 5, cap = F.cap;
        const PhraseQuery PQ = phrase_query(F, q);
        const PhraseMode mode = cap ? PhraseMode::score : PhraseMode::check;
        unsigned long long* hi = sort_buf;
        unsigned long long* lo = sort_buf + cap;
        for (uint32_t base = 0; base < kCountWords; base += kCountThreads) {   // uniform trip count
          const uint32_t i = base + tid;
          uint32_t v = acc[i];
          if (v && P.seg.deleted && wbase + i < del_words) v &= ~__ldg(P.seg.deleted + wbase + i);
          v = chain_bits(v, i);
          for (;;) {   // a full buffer is cut to the k best and the remaining bits go on
            const unsigned long long thr = s_thr[0];
            for (; v; v &= v - 1u) {
              const uint32_t doc = ws + 32u * i + (__ffs(v) - 1u);
              float s;
              if (!phrase_clauses<!kAnd>(P.seg, F, PQ, doc, mode, s)) continue;
              if (cap) {
                const unsigned long long key = phrase_key(F, doc, s);
                if (key > thr) {
                  const uint32_t slot = atomicAdd(&s_fill[0], 1u);
                  if (slot >= cap) break;   // this bit is checked again after the cut
                  hi[slot] = key;
                }
              }
              ++count;
            }
            if (!cap || !__syncthreads_or(v != 0u)) break;
            const unsigned long long kth = sort_select(hi, lo, cap, F.k, &s_fill[0]);
            if (tid == 0 && kth > s_thr[0]) { s_thr[0] = kth; atomicMax(F.thr + q, kth); }
            __syncthreads();
          }
        }
      }
    }
    }   // !skip
    __syncthreads();   // acc / tmp / cursors (kEmit: s_sum) are rewritten by the next window
    if constexpr (kEmit) {
      if (P.emit.base && e_run >= e_end) return;   // the page is full
    }
    if (wlast == 0xFFFFFFFFu || (wlast >> kCountWindowLog) + 1u >= w_end) break;
    ws = wlast + 1u;
  }
  if constexpr (kSort) {
    unsigned long long* hi = sort_buf;
    unsigned long long* lo = sort_buf + P.sort.cap;
    const unsigned long long kth = sort_select(hi, lo, P.sort.cap, P.sort.k, &s_fill[0]);
    const uint32_t n = s_fill[0];
    ulonglong2* out = P.sort.out + size_t(item.w) * P.sort.k;
    for (uint32_t i = tid; i < n; i += kCountThreads) out[i] = make_ulonglong2(hi[i], lo[i]);
    if (tid == 0) {
      P.sort.out_n[item.w] = n;
      if (P.sort.thr && kth) atomicMax(P.sort.thr + q, kth);
      if (judged) { atomicAdd(P.sort.stats, judged); if (skipped) atomicAdd(P.sort.stats + 1, skipped); }
    }
    return;
  }
  if constexpr (kFacet) {
    // A work item covers docs of one segment, fewer than 2^32, so no u32 bin can wrap before this flush.
    unsigned long long* out = P.facet.counts + size_t(q) * P.facet.span;
    for (uint32_t i = tid; i < P.facet.span; i += kCountThreads)
      if (bins[i]) atomicAdd(out + i, static_cast<unsigned long long>(bins[i]));
    if (oor) *P.facet.out_of_range = 1u;
    if (tid == 0 && s_fill[0]) atomicAdd(P.facet.nulls + q, static_cast<unsigned long long>(s_fill[0]));
  }
  if constexpr (kAgg) {
    // A work item covers docs of one segment, fewer than 2^32, so no u32 count or 64-bit limb can wrap before this flush.
    const uint32_t span = P.agg.key.span;
    if (!P.agg.key.values) {
      agg_merge(&cells[0], mine, P.agg.type);
      __syncthreads();
    }
    AggCell* out = P.agg.cells + size_t(q) * span;
    for (uint32_t i = tid; i <= span; i += kCountThreads) {
      const AggSmemCell c = cells[i];
      if (c.n) agg_flush(i < span ? out + i : P.agg.nulls + q, c, P.agg.type);
    }
    if (oor) *P.agg.out_of_range = 1u;
  }
  if constexpr (kEmit) {
    if (P.emit.base) return;
  }
  if constexpr (kPhraseSink) {
    if (P.phrase.cap) {
      const unsigned long long kth = sort_select(sort_buf, sort_buf + P.phrase.cap, P.phrase.cap, P.phrase.k, &s_fill[0]);
      const uint32_t n = s_fill[0];
      for (uint32_t i = tid; i < n; i += kCountThreads) P.phrase.out[size_t(item.w) * P.phrase.k + i] = sort_buf[i];
      if (tid == 0) {
        P.phrase.out_n[item.w] = n;
        if (kth) atomicMax(P.phrase.thr + q, kth);
      }
    }
  }
  count = warp_sum64(count);
  if (lane == 0) s_sum[warp] = count;
  __syncthreads();
  if (tid == 0) {
    unsigned long long s = 0;
    for (uint32_t w = 0; w < kCountWarps; ++w) s += s_sum[w];
    if constexpr (kEmit) P.emit.item_n[item.w] = uint32_t(s);   // an item's docs lie in one segment: fewer than 2^32
    else if (s) atomicAdd(P.counts + q, s);
  }
}

}  // namespace sdbg
