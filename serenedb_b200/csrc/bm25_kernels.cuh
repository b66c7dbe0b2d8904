// bm25_kernels.cuh -- sm_90a kernels for the BM25 posting scan + top-k.
//
// Reference behaviour being reproduced (paths relative to /root/reference/libs/iresearch/include/iresearch):
//   decode      formats/posting/format_block_128.hpp:475-636 (ReadTailDelta / ReadTail)
//   norms       search/column_collector.hpp:52-74, formats/column/norm_column_reader.hpp:99-108
//   score       search/bm25.cpp:90-107  (c1 = nc + nl*norm; r = c0 - c0*c1/(c1+freq), no FMA contraction)
//   windows     search/max_score_iterator.hpp:311-356 (score window + bitmap, Sum merge)
//   collector   index/iterators.hpp:103-250 (buffer of 2k, select when full, threshold = k-th)
//   conjunction search/conjunction.hpp:248-505 (all terms must match), score = sum of sub-scores
//   hybrid      index/table_filter_iterator.cpp:381-475 (column predicate on matched docs)
//
// Mapping: one CTA owns a chain of doc-id windows of one query; within a window every warp decodes
// one 128-posting block at a time (lane l holds postings 4l..4l+3 -- the four 32-bit lanes of the
// simdcomp layout are one 16-byte vector per row, so a lane reads at most two uint4 per block),
// scores it and adds into a shared-memory score window; matched slots are then compared with the
// query's running threshold and appended to a per-CTA candidate buffer that is compacted by a
// CTA-wide bitonic sort when full (the GPU analogue of nth_element at 2k).
#pragma once

#include "column_kernels.cuh"

namespace sdbg {

// ---- device views ----
struct PostingsDev {
  const uint4* arena;     // block payloads, 16-byte units
  const uint4* blocks;    // BlockDesc {off16, last_doc, prev_last, packed}
  const uint2* blk_max;   // {freq, norm} per block (block-max pairs), may be null
  const uint4* anchors;   // per block: doc ids of postings 31, 63, 95 (probe acceleration, see posting_format.hpp)
  const uint8_t* norms;   // fixed-width field lengths, row = doc-1; null => norm = 1
  const uint32_t* deleted; // DocumentMask as a bitmap, bit `doc` set = deleted (SegmentReaderImpl::mask, segment_reader_impl.cpp:318-326); null = none
  uint32_t norm_width;    // 1, 2 or 4
  uint32_t n_docs;
  uint32_t ordinal_base;  // first global ordinal of this segment (keys carry base + doc)
};

struct QTermDev {  // one term of one query over one segment, 40 bytes
  uint32_t blk_begin;  // first BlockDesc of the term
  uint32_t nblk;
  float c0;            // boost*(k1+1)*idf   (bm25.cpp:224)
  float norm_const;
  float norm_length;
  uint32_t docs_count;
  uint32_t root_freq, root_norm;   // block-max pair of the whole list (0,0 = unknown); bit 31 of root_freq: the list's blocks
                                   // are bitsets with random-access freqs, i.e. cheap to probe (driver mode is worth it)
  // norm_const / norm_length for scoring a block-max pair as an upper bound (fill_qterm, sdbg_abi.cu): the pair maximises
  // BM25 under the segment's own average length, which need not be the query's corpus-wide one
  float bound_const, bound_length;
};

constexpr uint32_t kMaxQueryTerms = 16;
// Per-doc list checks of a query (TopkParams::excl): up to 16 excluded lists plus up to 16 lists of required OR groups.
constexpr uint32_t kMaxCheckLists = 2u * kMaxQueryTerms;
// Tag of an excluded list. A group list's tag holds its group index g (0..15) in the low nibble and the group's minimum
// match count m_g - 1 in the high nibble (0 for a plain OR group; m_g <= 15, so no group tag equals kCheckExcl).
constexpr uint8_t kCheckExcl = 0xFF;
constexpr uint32_t kTopkThreads = 256;
constexpr uint32_t kTopkWarps = kTopkThreads / 32;
constexpr uint32_t kTopkBudget = 32;   // bm25_topk_kernel: posting blocks per window, one planner lane each

__device__ __forceinline__ uint32_t desc_doc_enc(uint32_t p) { return p & 63u; }
__device__ __forceinline__ uint32_t desc_freq_enc(uint32_t p) { return (p >> 6) & 63u; }
__device__ __forceinline__ uint32_t desc_len(uint32_t p) { return ((p >> 12) & 127u) + 1u; }
__device__ __forceinline__ uint32_t desc_fdelta(uint32_t p) { return (p >> 19) & 63u; }
__device__ __forceinline__ uint32_t desc_words(uint32_t p) { return p >> 25; }

// ---- block decode: lane holds values 4*lane .. 4*lane+3 ----
// Bit-packed payload (simdunpack layout): row = lane, the four 32-bit lanes of that row are the
// four components of one uint4; row r occupies bits [r*b, r*b+b) of every lane stream.
__device__ __forceinline__ void unpack4(const uint4* p, uint32_t b, uint32_t lane, uint32_t v[4]) {
  const uint32_t bit = lane * b;
  const uint32_t w = bit >> 5, sh = bit & 31u;
  const uint4 lo = ld_ro_v4(p + w);
  const uint4 hi = ld_ro_v4(p + min(w + 1u, b - 1u));
  const uint32_t mask = (1u << b) - 1u;  // b <= 31
  v[0] = __funnelshift_r(lo.x, hi.x, sh) & mask;
  v[1] = __funnelshift_r(lo.y, hi.y, sh) & mask;
  v[2] = __funnelshift_r(lo.z, hi.z, sh) & mask;
  v[3] = __funnelshift_r(lo.w, hi.w, sh) & mask;
}

// StreamVByte 1234 (tails only): control byte `lane` describes this lane's four values.
__device__ __forceinline__ void svb4(const uint4* p, uint32_t len, uint32_t lane, uint32_t v[4]) {
  const uint8_t* bytes = reinterpret_cast<const uint8_t*>(p);
  const uint32_t nctl = (len + 3u) >> 2;
  const uint32_t ctl = lane < nctl ? uint32_t(__ldg(bytes + lane)) : 0u;
  uint32_t n[4], mine = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    n[j] = (4u * lane + j < len) ? ((ctl >> (2 * j)) & 3u) + 1u : 0u;
    mine += n[j];
  }
  uint32_t pos = nctl + warp_incl_scan(mine, lane) - mine;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    uint32_t x = 0;
    for (uint32_t k = 0; k < n[j]; ++k) x |= uint32_t(__ldg(bytes + pos + k)) << (8 * k);
    pos += n[j];
    v[j] = x;
  }
}

__device__ __forceinline__ uint32_t same_value(const uint4* p, uint32_t width_code /*1,2,3*/) {
  const uint32_t raw = __ldg(reinterpret_cast<const uint32_t*>(p));
  return width_code == 1 ? (raw & 0xFFu) : width_code == 2 ? (raw & 0xFFFFu) : raw;
}

// Turns four per-lane gaps into absolute ids: running sum across the warp in value order.
__device__ __forceinline__ void prefix_from_gaps(uint32_t prev, uint32_t lane, uint32_t v[4]) {
  v[1] += v[0]; v[2] += v[1]; v[3] += v[2];
  const uint32_t base = prev + warp_incl_scan(v[3], lane) - v[3];
  v[0] += base; v[1] += base; v[2] += base; v[3] += base;
}

// Doc ids of one block. `stage` = 128 u32 of per-warp shared scratch (bitset rank scatter).
__device__ __forceinline__ void decode_docs(const uint4* arena, const uint4& d, uint32_t lane,
                                            uint32_t* stage, uint32_t doc[4]) {
  const uint4* p = arena + d.x;
  const uint32_t enc = desc_doc_enc(d.w), len = desc_len(d.w), prev = d.z;
  if (enc >= 8u) {  // de_delta_bitpack_b, b = enc - 6
    unpack4(p, enc - 6u, lane, doc);
    prefix_from_gaps(prev, lane, doc);
  } else if (enc == 4u) {  // de_for_bitset: bit j set => id prev + j
    // Position-parallel expansion: in iteration i every lane tests bit 32*i + lane of the bitset (the
    // 32-bit chunk is broadcast from the lane that loaded it) and a set bit is written to its rank
    // (= set bits before it). All lanes run the same trip count, unlike a per-lane "next set bit" loop.
    const uint32_t words = desc_words(d.w);             // 64-bit words, <= 64
    uint4 x = make_uint4(0, 0, 0, 0);                    // lane l holds 32-bit chunks 4l .. 4l+3
    if (2u * lane < words) x = ld_ro_v4(p + lane);
    const uint32_t lt = (1u << lane) - 1u;
    uint32_t base = 0;
    const uint32_t chunks = 2u * words;
    for (uint32_t i = 0; i < chunks; i += 4u) {
      const uint32_t src = i >> 2;
      const uint32_t c0 = __shfl_sync(kFull, x.x, src), c1 = __shfl_sync(kFull, x.y, src);
      const uint32_t c2 = __shfl_sync(kFull, x.z, src), c3 = __shfl_sync(kFull, x.w, src);
      const uint32_t id = prev + 32u * i + lane;
      if ((c0 >> lane) & 1u) stage[base + __popc(c0 & lt)] = id;
      base += __popc(c0);
      if ((c1 >> lane) & 1u) stage[base + __popc(c1 & lt)] = id + 32u;
      base += __popc(c1);
      if ((c2 >> lane) & 1u) stage[base + __popc(c2 & lt)] = id + 64u;
      base += __popc(c2);
      if ((c3 >> lane) & 1u) stage[base + __popc(c3 & lt)] = id + 96u;
      base += __popc(c3);
    }
    __syncwarp();
    const uint4 o = reinterpret_cast<const uint4*>(stage)[lane];
    doc[0] = o.x; doc[1] = o.y; doc[2] = o.z; doc[3] = o.w;
    __syncwarp();
  } else if (enc >= 1u && enc <= 3u) {  // de_delta_all_same_{08,16,32}
    const uint32_t g = same_value(p, enc);
#pragma unroll
    for (int j = 0; j < 4; ++j) doc[j] = prev + g * (4u * lane + j + 1u);
  } else if (enc == 0u) {  // de_values
    uint4 x = make_uint4(0, 0, 0, 0);
    if (4u * lane < len) x = ld_ro_v4(p + lane);
    doc[0] = x.x; doc[1] = x.y; doc[2] = x.z; doc[3] = x.w;
  } else {  // 5 de_streamvbyte1234, 7 de_delta_streamvbyte1234 (tails)
    svb4(p, len, lane, doc);
    if (enc == 7u) prefix_from_gaps(prev, lane, doc);
  }
}

__device__ __forceinline__ void decode_freqs(const uint4* arena, const uint4& d, uint32_t lane, uint32_t f[4]) {
  const uint4* p = arena + d.x + desc_fdelta(d.w);
  const uint32_t enc = desc_freq_enc(d.w), len = desc_len(d.w);
  if (enc >= 5u) {  // e_bitpack_b, b = enc - 4
    unpack4(p, enc - 4u, lane, f);
  } else if (enc >= 1u && enc <= 3u) {
    const uint32_t g = same_value(p, enc);
    f[0] = f[1] = f[2] = f[3] = g;
  } else if (enc == 0u) {
    uint4 x = make_uint4(0, 0, 0, 0);
    if (4u * lane < len) x = ld_ro_v4(p + lane);
    f[0] = x.x; f[1] = x.y; f[2] = x.z; f[3] = x.w;
  } else {
    svb4(p, len, lane, f);
  }
}

__device__ __forceinline__ uint32_t load_norm(const uint8_t* norms, uint32_t width, uint32_t doc) {
  if (norms == nullptr) return 1u;  // bm25.cpp:353-360
  const size_t row = size_t(doc) - 1u;
  if (width == 1u) return __ldg(norms + row);
  if (width == 2u) return __ldg(reinterpret_cast<const uint16_t*>(norms) + row);
  return __ldg(reinterpret_cast<const uint32_t*>(norms) + row);
}

// bm25.cpp:105-106 with the reference's operation order; intrinsics forbid FMA contraction so the
// result is bit-identical to the g++ -ffp-contract=off oracle. A NaN norm_length is the host's marker for
// the BM15 form (b == 0, bm25.cpp:70-87: c0 - c0 / (1 + freq / c1) with c1 = k, norms unused); the test is
// uniform per posting list. BM1 (k == 0) arrives as c0 == 0 and scores 0 through the BM25 form.
__device__ __forceinline__ float bm25(uint32_t freq, uint32_t norm, float c0, float nc, float nl) {
  if (nc != nc) {
    // TFIDF (search/tfidf.cpp:59-80): a NaN norm_const is the host's marker; c0 = boost * idf, nl != 0 = normalised.
    // sqrt(freq) * idf [/ sqrt(norm)], every operation correctly rounded like the reference's std::sqrt / * / /.
    float r = __fmul_rn(__fsqrt_rn(static_cast<float>(freq)), c0);
    if (nl != 0.f) r = __fdiv_rn(r, __fsqrt_rn(static_cast<float>(norm)));
    return r;
  }
  if (nl != nl) return __fsub_rn(c0, __fdiv_rn(c0, __fadd_rn(1.f, __fdiv_rn(static_cast<float>(freq), nc))));
  const float c1 = __fadd_rn(nc, __fmul_rn(nl, static_cast<float>(norm)));
  return __fsub_rn(c0, __fdiv_rn(__fmul_rn(c0, c1), __fadd_rn(c1, static_cast<float>(freq))));
}

// Upper bound of the query-time score of every posting that a block-max pair (freq, norm) stands for. Pruning runs
// only for the BM25 form, so the bound constants are always finite.
__device__ __forceinline__ float pair_bound(uint32_t freq, uint32_t norm, const QTermDev& qt) {
  return bm25(freq, norm, qt.c0, qt.bound_const, qt.bound_length);
}

// The BM25 form alone (bm25.cpp:105-106), for kernels the host only dispatches with k != 0, b != 0 (bm25_merge_kernel,
// bm25_stream_kernel): same operations as the last two lines of bm25(), without the per-posting form tests and without
// the other forms' divides and square roots in the instruction stream.
__device__ __forceinline__ float bm25_plain(uint32_t freq, uint32_t norm, float c0, float nc, float nl) {
  const float c1 = __fadd_rn(nc, __fmul_rn(nl, static_cast<float>(norm)));
  return __fsub_rn(c0, __fdiv_rn(__fmul_rn(c0, c1), __fadd_rn(c1, static_cast<float>(freq))));
}

// ------------------------------------------------------------------------------------------
// Probe kernel: decode + score one whole posting list (exhaustive). One warp per block.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTopkThreads)
decode_score_kernel(PostingsDev seg, uint32_t blk_begin, uint32_t nblk, float c0, float nc, float nl,
                    uint32_t* __restrict__ docs, uint32_t* __restrict__ freqs, float* __restrict__ scores) {
  __shared__ __align__(16) uint32_t stage[kTopkWarps][128];
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  for (uint32_t b = blockIdx.x * kTopkWarps + warp; b < nblk; b += gridDim.x * kTopkWarps) {
    const uint4 d = ld_ro_v4(seg.blocks + blk_begin + b);
    uint32_t doc[4], f[4];
    decode_docs(seg.arena, d, lane, stage[warp], doc);
    decode_freqs(seg.arena, d, lane, f);
    const uint32_t len = desc_len(d.w);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t i = 4u * lane + j;
      if (i < len) {
        const size_t o = size_t(b) * 128u + i;
        docs[o] = doc[j]; freqs[o] = f[j];
        scores[o] = bm25(f[j], load_norm(seg.norms, seg.norm_width, doc[j]), c0, nc, nl);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Fused scan + score + top-k kernel.
//
// grid = (chains G, queries Q). CTA (g, q) owns the doc range [1 + g*chunk, min(N, (g+1)*chunk)] of
// query q and walks it in WINDOWS DEFINED BY A BLOCK BUDGET, not by a doc count: every window holds
// at most kTopkBudget posting blocks in total (kTopkBudget / T per term), so the fixed per-window costs are
// amortised over up to kTopkBudget*128 postings whether the lists are dense (p = 0.5: a window spans a
// few hundred docs) or sparse (p = 0.002: hundreds of thousands). The reference gets the same effect
// from ComputeOuterWindow, which aligns windows with the essential lists' block boundaries
// (search/max_score_iterator.hpp:510-539).
//
// Planning is one round of parallel loads: lane (t, j) of warp 0 reads the descriptor of block
// cursor_t + j; the window ends at the earliest "m-th block end" over the terms that still have m
// blocks (so no term can overlap the window with more than m blocks); a ballot yields the item list
// and popcounts advance the cursors. The plan for window i+1 is computed while window i is processed.
//
// Window body (no shared-memory atomics, every loop is dense over lanes):
//   1. decode: one warp per block; docs + BM25 scores land in shared memory as per-term arrays that
//      are sorted by doc id (blocks of a term are consecutive, padding = 0xFFFFFFFF).
//   2. fold: for t = 0 .. T-2 every live entry of terms <= t binary-searches term t+1; on a hit its
//      score is added into the hit slot and the entry dies. A doc has at most one live entry at any
//      step, so each slot has a unique writer and the sum is formed in ascending-cost order
//      ((s0+s1)+s2..., ConjunctionScore's order, search/conjunction.hpp:185-195) -- bit-reproducible.
//      For conjunctions an entry that misses dies too, so only the shortest list keeps searching.
//   3. emit: live in-window entries -> column filter -> threshold -> ballot-compacted append to the
//      per-CTA candidate buffer (bitonic select when full = nth_element at 2k, iterators.hpp:216-228).
//
// Shared memory (dynamic): docs[E] u32 | score[E] f32 | cnt[E] u8 (AND only) | cand[cap] u64, E = kTopkBudget*128.
// ------------------------------------------------------------------------------------------
struct TopkParams {
  PostingsDev seg;
  ChainDev filt;
  const QTermDev* qterms;      // flattened, per query sorted by ascending docs_count
  const uint32_t* qterm_off;   // n_queries + 1
  unsigned long long* theta;   // per query running threshold key (shared by all chains / segments)
  unsigned long long* total;   // per query matched-doc count
  unsigned long long* cand;    // [lists][cap] candidate keys, sorted descending on exit
  uint32_t* cand_n;            // [lists]
  // One CTA per work item {query, first doc, docs, candidate list}: a query is cut into as many chains
  // (contiguous doc ranges) as its posting count warrants, and the items are ordered largest first so that
  // the long chains do not end up running alone at the tail of the launch.
  const uint4* work;
  // Stream kernels only: one word per work item, or null. An item that can be run either as an exhaustive merge
  // (bm25_merge_kernel) or as lead list + probes (bm25_stream_kernel in lead mode) is launched into BOTH; the
  // first CTA to arrive looks at the query's threshold, decides, and records 1 = merge / 2 = lead here; the other
  // one reads the verdict and exits.
  uint32_t* claim;
  // Scored scan (the reference's streaming mode, duckdb_search_full_scan.cpp RunStreamingScan): when emit_docs is set the
  // stream kernel writes EVERY match (segment-local doc, score) through a global cursor instead of keeping a top-k;
  // emit_count keeps counting past emit_cap so that the host can report the room needed.
  uint32_t* emit_docs = nullptr;
  float* emit_scores = nullptr;
  unsigned long long* emit_count = nullptr;
  unsigned long long emit_cap = 0;
  // Excluded terms (the NOT children of an And, irs search/exclusion.hpp): query q rejects every doc that occurs in one
  // of the lists excl[excl_off[q] .. excl_off[q + 1]), each {first BlockDesc, blocks} in this segment (0 blocks: a term
  // the segment does not hold). Excluded terms never score. Null: no query of the call excludes anything.
  // excl_grp, when set, tags each of those lists: kCheckExcl for an excluded list, else a required OR group of the query
  // (`a & (b | c)`, `2 of (a | b | c)`; kCheckExcl's comment gives the layout): a doc then also needs, for every group
  // present, at least m_g of the group's tagged lists that hold it.
  // Set only for the kGroups instantiations, whose queries have at most kMaxCheckLists lists.
  const uint2* excl = nullptr;
  const uint32_t* excl_off = nullptr;
  const uint8_t* excl_grp = nullptr;
  uint32_t k;
  uint32_t cap;                // candidate buffer capacity, power of two, > k
  int32_t conjunction;         // 0 OR, 1 AND
  int32_t wand;                // 1: block-max pruning on (total_matches becomes a lower bound, like the reference with WAND)
};

constexpr uint32_t kPadDoc = 0xFFFFFFFFu;
// Doc ids are 1 .. 2^32 - 2 (doc_limits::eof() = 2^32 - 1 is never a doc): the largest segment, and the most docs one
// top-k or sorted call takes summed over its segments (ordinal_base + doc stays a valid id).
constexpr uint32_t kMaxDocId = 0xFFFFFFFEu;

// First index in sorted a[0..n) with a[i] >= d (n > 0 is a multiple of 128).
__device__ __forceinline__ uint32_t lower_bound_u32(const uint32_t* a, uint32_t n, uint32_t d) {
  uint32_t pos = 0;
  for (uint32_t step = 1u << (31 - __clz(n)); step; step >>= 1) {
    const uint32_t nxt = pos + step;
    if (nxt <= n && a[nxt - 1u] < d) pos = nxt;
  }
  return pos;
}

// ---- random access into one block (driver-mode probes) ----
// Frequency of posting `i` of the block without decoding the rest; false when the encoding is sequential
// (StreamVByte tails) and the caller has to decode the block.
__device__ __forceinline__ bool freq_at(const uint4* arena, const uint4& d, uint32_t i, uint32_t& f) {
  const uint4* p = arena + d.x + desc_fdelta(d.w);
  const uint32_t enc = desc_freq_enc(d.w);
  if (enc >= 5u) {                                   // e_bitpack_b: value i = row i>>2 of lane stream i&3
    const uint32_t b = enc - 4u, bit = (i >> 2) * b, w = bit >> 5, sh = bit & 31u;
    const uint32_t* q = reinterpret_cast<const uint32_t*>(p) + (i & 3u);
    const uint32_t lo = __ldg(q + 4u * w), hi = __ldg(q + 4u * min(w + 1u, b - 1u));
    f = __funnelshift_r(lo, hi, sh) & ((1u << b) - 1u);
    return true;
  }
  if (enc >= 1u && enc <= 3u) { f = same_value(p, enc); return true; }
  if (enc == 0u) { f = __ldg(reinterpret_cast<const uint32_t*>(p) + i); return true; }
  return false;
}
// Membership + rank of doc `doc` in a de_for_bitset block (bit j set <=> id prev + j): O(words) popcounts.
__device__ __forceinline__ bool bitset_rank(const uint4* arena, const uint4& d, uint32_t doc, uint32_t& rank) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(arena + d.x);
  const uint32_t j = doc - d.z, chunk = j >> 5;
  if (chunk >= 2u * desc_words(d.w)) return false;
  const uint32_t mine = __ldg(w + chunk);
  if (!((mine >> (j & 31u)) & 1u)) return false;
  uint32_t r = __popc(mine & ((1u << (j & 31u)) - 1u));
  for (uint32_t c = 0; c < chunk; ++c) r += __popc(__ldg(w + c));
  rank = r;
  return true;
}
// First block in [b0, b1) whose last doc is >= doc, searched outwards from `guess` (b1 when none).
__device__ __forceinline__ uint32_t find_block_from(const uint4* LB, uint32_t b0, uint32_t b1, uint32_t guess, uint32_t doc) {
  uint32_t l, r;                                       // answer in [l, r]
  if (__ldg(&LB[guess].y) >= doc) {                    // answer <= guess: gallop down
    r = guess; l = b0;
    for (uint32_t step = 1u; r - b0 >= step; step <<= 1) {
      if (__ldg(&LB[r - step].y) >= doc) r -= step; else { l = r - step + 1u; break; }
    }
  } else {                                             // answer > guess: gallop up
    l = guess + 1u; r = b1;
    for (uint32_t step = 1u; l + step - 1u < b1; step <<= 1) {
      if (__ldg(&LB[l + step - 1u].y) < doc) l += step; else { r = l + step - 1u; break; }
    }
    l = min(l, b1);
  }
  while (l < r) { const uint32_t mid = (l + r) >> 1; if (__ldg(&LB[mid].y) < doc) l = mid + 1u; else r = mid; }
  return l;
}

__device__ __forceinline__ uint32_t svb_value_at(const uint8_t* bytes, uint32_t len, uint32_t idx_or_doc, bool by_doc, bool delta,
                                                 uint32_t prev, uint32_t* idx_out) {
  // by_doc: walks the doc stream until the running id reaches idx_or_doc (returns the id found or 0xFFFFFFFF);
  // else returns value number idx_or_doc.
  const uint32_t nctl = (len + 3u) >> 2;
  uint32_t pos = nctl, acc = prev;
  for (uint32_t i = 0; i < len; ++i) {
    const uint32_t c = (uint32_t(__ldg(bytes + (i >> 2))) >> (2u * (i & 3u))) & 3u;
    uint32_t x = 0;
    for (uint32_t k = 0; k <= c; ++k) x |= uint32_t(__ldg(bytes + pos + k)) << (8u * k);
    pos += c + 1u;
    if (by_doc) {
      acc = delta ? acc + x : x;
      if (acc >= idx_or_doc) { *idx_out = i; return acc; }
    } else if (i == idx_or_doc) {
      return x;
    }
  }
  return 0xFFFFFFFFu;
}

// Position of doc `d` inside block `desc` (prev_last < d <= last_doc), or false when the block does not hold it.
__device__ __forceinline__ bool block_find_doc(const PostingsDev& S, const uint4& desc, uint32_t gblk, uint32_t d, uint32_t& idx) {
  const uint4* p = S.arena + desc.x;
  const uint32_t enc = desc_doc_enc(desc.w), len = desc_len(desc.w), prev = desc.z;
  if (enc >= 8u) {                                   // bit-packed gaps: row r = postings 4r .. 4r+3
    const uint32_t b = enc - 6u;
    const uint4 an = __ldg(S.anchors + gblk);
    const uint32_t qd = (d > an.x ? 1u : 0u) + (d > an.y ? 1u : 0u) + (d > an.z ? 1u : 0u);
    uint32_t acc = qd == 0u ? prev : qd == 1u ? an.x : qd == 2u ? an.y : an.z;
    const uint32_t mask = (1u << b) - 1u;
    for (uint32_t r = 8u * qd; r < 8u * qd + 8u; ++r) {
      const uint32_t bit = r * b, w = bit >> 5, sh = bit & 31u;
      const uint4 lo = __ldg(p + w), hi = __ldg(p + min(w + 1u, b - 1u));
      acc += __funnelshift_r(lo.x, hi.x, sh) & mask; if (acc >= d) { idx = 4u * r; return acc == d; }
      acc += __funnelshift_r(lo.y, hi.y, sh) & mask; if (acc >= d) { idx = 4u * r + 1u; return acc == d; }
      acc += __funnelshift_r(lo.z, hi.z, sh) & mask; if (acc >= d) { idx = 4u * r + 2u; return acc == d; }
      acc += __funnelshift_r(lo.w, hi.w, sh) & mask; if (acc >= d) { idx = 4u * r + 3u; return acc == d; }
    }
    return false;
  }
  if (enc == 4u) return bitset_rank(S.arena, desc, d, idx);
  if (enc >= 1u && enc <= 3u) {                       // constant gap g: ids prev + g, prev + 2g, ...
    const uint32_t g = same_value(p, enc);
    const uint32_t off = d - prev;
    if (g == 0u || off % g != 0u) return false;
    idx = off / g - 1u;
    return idx < len;
  }
  if (enc == 0u) {                                    // raw ids
    const uint32_t* a = reinterpret_cast<const uint32_t*>(p);
    uint32_t l = 0, r = len;
    while (l < r) { const uint32_t m = (l + r) >> 1; if (__ldg(a + m) < d) l = m + 1u; else r = m; }
    idx = l;
    return l < len && __ldg(a + l) == d;
  }
  return svb_value_at(reinterpret_cast<const uint8_t*>(p), len, d, true, enc == 7u, prev, &idx) == d;
}

// Membership only: does the list {first BlockDesc, blocks} hold doc d? Block search from `hint` (a block index within the
// list; on return the block that was searched), then the in-block search -- no frequency, no score. Excluded terms.
__device__ __forceinline__ bool probe_contains(const PostingsDev& S, uint2 list, uint32_t d, uint32_t hint, uint32_t& found_blk) {
  const uint4* B = S.blocks + list.x;
  const uint32_t n = list.y;
  if (n == 0u) { found_blk = 0u; return false; }
  const uint32_t l = find_block_from(B, 0u, n, min(hint, n - 1u), d);
  found_blk = min(l, n - 1u);
  if (l >= n) return false;
  const uint4 desc = __ldg(B + l);
  if (d <= desc.z) return false;                       // d lies between two blocks
  uint32_t idx = 0;
  return block_find_doc(S, desc, list.x + l, d, idx);
}

// Per-doc state of the OR-group check, one 4-bit counter per group g at bits 4g .. 4g + 3: `need` = lists that must still
// hold the doc (m_g at first), `slack` = lists that may still miss it (s_g - m_g at first, s_g = the group's lists).
// A group is satisfied once its need is 0 and fails once a list misses with its slack at 0.
struct GroupNeed { unsigned long long need, slack; };
__device__ __forceinline__ GroupNeed check_group_need(const uint8_t* grp, uint32_t n) {
  unsigned long long need = 0ull, lists = 0ull;
  for (uint32_t x = 0; x < n; ++x) {
    if (grp[x] == kCheckExcl) continue;
    const uint32_t g4 = 4u * (grp[x] & 15u);
    need |= static_cast<unsigned long long>((grp[x] >> 4) + 1u) << g4;
    lists += 1ull << g4;   // s_g = 16 carries into the next nibble; lists - need is still exact per nibble
  }
  return {need, lists - need};
}

// One group list's verdict for one doc: counts a hit towards the group's minimum, a miss against its slack. False when
// the group can no longer reach its minimum.
__device__ __forceinline__ bool group_step(GroupNeed& st, uint32_t g4, bool hit) {
  if (hit) { st.need -= 1ull << g4; return true; }
  if (((st.slack >> g4) & 15ull) == 0ull) return false;
  st.slack -= 1ull << g4;
  return true;
}

// One thread: does any of the n excluded lists hold doc d (legacy window kernel's emit step)? Each list is searched from
// its first block. Takes the views by value so that the kernel's parameter block is not copied to local memory.
__device__ __noinline__ bool excluded_doc(const uint4* arena, const uint4* blocks, const uint4* anchors, const uint2* ex, uint32_t n,
                                          uint32_t d) {
  PostingsDev S{};
  S.arena = arena; S.blocks = blocks; S.anchors = anchors;
  for (uint32_t x = 0; x < n; ++x) {
    uint32_t blk = 0;
    if (probe_contains(S, ex[x], d, 0u, blk)) return true;
  }
  return false;
}

// The same with OR groups: is doc d rejected because an excluded list holds it, or because some group tagged in `grp`
// has fewer than m_g lists that hold it? A group's remaining lists are skipped once m_g of them hold d, and d is rejected
// as soon as a group's remaining lists cannot reach m_g.
__device__ __noinline__ bool excluded_doc(const uint4* arena, const uint4* blocks, const uint4* anchors, const uint2* ex,
                                          const uint8_t* grp, uint32_t n, uint32_t d) {
  GroupNeed st = check_group_need(grp, n);
  PostingsDev S{};
  S.arena = arena; S.blocks = blocks; S.anchors = anchors;
  for (uint32_t x = 0; x < n; ++x) {
    const uint32_t g = grp[x];
    const uint32_t g4 = 4u * (g & 15u);
    if (g != kCheckExcl && ((st.need >> g4) & 15ull) == 0ull) continue;
    uint32_t blk = 0;
    const bool hit = probe_contains(S, ex[x], d, 0u, blk);
    if (g == kCheckExcl) {
      if (hit) return true;
    } else if (!group_step(st, g4, hit)) {
      return true;
    }
  }
  return st.need != 0ull;
}

// kDrive compiles the driver-mode code (pruning level 2) in; the default kernel stays free of its registers. kExcl: the
// queries of the launch exclude terms (TopkParams::excl); with kGroups they also require OR groups (TopkParams::excl_grp).
// Likewise kept out of the other instantiations.
template <bool kDrive, bool kExcl = false, bool kGroups = false>
__global__ void __launch_bounds__(kTopkThreads)
bm25_topk_kernel(const TopkParams P) {
  constexpr uint32_t kEntries = kTopkBudget * 128u;
  static_assert(kTopkBudget <= 32, "one planner lane per block");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint32_t* e_doc = reinterpret_cast<uint32_t*>(smem_raw);
  float* e_score = reinterpret_cast<float*>(e_doc + kEntries);
  uint8_t* e_cnt = reinterpret_cast<uint8_t*>(e_score + kEntries);
  unsigned long long* cand = reinterpret_cast<unsigned long long*>(e_cnt + (P.conjunction ? kEntries : 0u));
  uint16_t* s_probe = reinterpret_cast<uint16_t*>(cand + P.cap);   // 2 * kEntries u16 (probe list | decode-fallback list), only present at wand level 2

  __shared__ __align__(16) uint32_t stage[kTopkWarps][128];
  __shared__ __align__(16) uint4 s_item[2][32];        // descriptors of the window's blocks, term-major
  __shared__ uint32_t s_item_term[2][32];
  __shared__ uint32_t s_phase[2][kMaxQueryTerms + 1];  // first item of each term
  __shared__ uint32_t s_lo[2], s_hi[2], s_valid[2];
  __shared__ float s_item_bound[2][32];                // block-max upper bound of each item (+inf when unknown)
  __shared__ uint32_t s_driver;                        // 1: the largest list is probed per candidate instead of scanned
  __shared__ uint32_t s_Lb0[2], s_Lb1[2];              // block range of the largest list that covers the window (driver mode)
  __shared__ uint32_t s_nprobe, s_nslow;
  __shared__ float s_ubL;                              // global block-max bound of the largest list
  __shared__ float s_term_ub[2][kMaxQueryTerms];       // max bound over the term's blocks in the window (0 if none)
  __shared__ uint32_t s_cursor[kMaxQueryTerms];
  __shared__ QTermDev s_qt[kMaxQueryTerms];
  __shared__ uint32_t s_ncand, s_matched;
  __shared__ unsigned long long s_theta;
  __shared__ uint32_t s_hist[258];
  __shared__ uint2 s_ex[kGroups ? kMaxCheckLists : kExcl ? kMaxQueryTerms : 1];   // check lists of the query (TopkParams::excl)
  __shared__ uint8_t s_exg[kGroups ? kMaxCheckLists : 1];                          // and their tags (kGroups)

  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const uint4 work = P.work[blockIdx.x];
  const uint32_t q = work.x, chunk = work.z;   // work item = {query, first doc, docs, candidate list}
  const uint32_t t0 = P.qterm_off[q];
  const uint32_t T = min(P.qterm_off[q + 1] - t0, kMaxQueryTerms);
  const uint32_t x0 = kExcl ? P.excl_off[q] : 0u;
  const uint32_t n_ex = kExcl ? min(P.excl_off[q + 1] - x0, kGroups ? kMaxCheckLists : kMaxQueryTerms) : 0u;
  const uint32_t m = max(1u, kTopkBudget / T);                      // block budget per term
  const unsigned long long first64 = work.y;
  const bool chain_empty = first64 > P.seg.n_docs;
  const uint32_t chain_lo = chain_empty ? 1u : uint32_t(first64);
  const uint32_t chain_hi = chain_empty ? 0u : uint32_t(min(static_cast<unsigned long long>(P.seg.n_docs), first64 + chunk - 1ull));

  for (uint32_t i = tid; i < P.cap; i += blockDim.x) cand[i] = 0ull;
  if (tid < T) s_qt[tid] = P.qterms[t0 + tid];
  if (kExcl && tid < n_ex) s_ex[tid] = P.excl[x0 + tid];
  if (kGroups && tid < n_ex) s_exg[tid] = P.excl_grp[x0 + tid];
  if (tid == 0) { s_ncand = 0u; s_matched = 0u; s_theta = 0ull; }
  __syncthreads();

  // Warp 0, lane t: first block of term t whose last doc reaches the chain (binary search, once).
  if (warp == 0 && lane < T) {
    const uint4* B = P.seg.blocks + s_qt[lane].blk_begin;
    uint32_t l = 0, r = s_qt[lane].nblk;
    while (l < r) { const uint32_t mid = (l + r) >> 1; if (__ldg(&B[mid].y) < chain_lo) l = mid + 1u; else r = mid; }
    s_cursor[lane] = l;
  }
  __syncwarp();

  // level 1 prunes single-term queries only (planner-level block skip is free there); with several terms the
  // other terms' window bounds almost always keep every block alive, so the test would be pure overhead.
  // level 2 adds DRIVER MODE for disjunctions: once the threshold exceeds the global block-max bound of the
  // largest list L, a doc that occurs only in L can no longer qualify (L is "non-essential",
  // max_score_iterator.hpp:450-508). From then on windows are planned over the other lists only and L is
  // probed per surviving candidate (ProcessNonEssentialFromCandidates, :406-429) instead of being scanned.
  const bool prune = P.wand && !P.conjunction && P.seg.blk_max != nullptr && (T == 1u || P.wand >= 2);
  const bool can_drive = kDrive && prune && P.wand >= 2 && T >= 2u;
  if (tid == 0) {
    s_driver = 0u;
    const QTermDev& L = s_qt[T - 1u];
    // driver mode only for a probe-friendly largest list: a probe into a bit-packed block costs a block decode
    s_ubL = (can_drive && (L.root_freq >> 31) && (L.root_freq & 0x7FFFFFFFu) != 0u)
                ? pair_bound(L.root_freq & 0x7FFFFFFFu, L.root_norm, L)
                                              : __int_as_float(0x7f800000);
  }
  __syncthreads();

  // Plans the window starting at doc `lo` into buffer `buf` (warp 0 only); returns the next lo.
  // With pruning on, blocks / windows whose block-max bound cannot beat the current threshold are consumed
  // without being handed to the decoders (UpdateWindowScores, max_score_iterator.hpp:437).
  auto plan = [&](uint32_t lo, uint32_t buf) -> uint32_t {
    const float thr = __uint_as_float(uint32_t(s_theta >> 32));
    // one-way switch (the threshold only rises); every bound test carries the stream kernels' rounding margin
    if (can_drive && !s_driver && thr > __fmul_rn(s_ubL, 1.000001f)) { if (lane == 0) s_driver = 1u; }
    __syncwarp();
    const bool driver = kDrive && s_driver != 0u;
    const uint32_t Tp = driver ? T - 1u : T;             // lists that get planner lanes
    const uint32_t mp = max(1u, kTopkBudget / Tp);
    for (uint32_t tries = 0;; ++tries) {
      if (lo > chain_hi || lo == 0u) {  // lo == 0: wrapped past 2^32-1
        if (lane == 0) s_valid[buf] = 0u;
        return 0u;
      }
      const uint32_t t = lane / mp, j = lane - t * mp;
      const bool mine = t < Tp && lane < Tp * mp;
      uint4 d = make_uint4(0, 0, 0, 0);
      bool exists = false;
      uint32_t gblk = 0;
      if (mine) {
        const uint32_t b = s_cursor[t] + j;
        exists = b < s_qt[t].nblk;
        gblk = s_qt[t].blk_begin + b;
        if (exists) d = ld_ro_v4(P.seg.blocks + gblk);
      }
      // a term that still has mp blocks bounds the window at the end of its mp-th block
      uint32_t hi = (exists && j == mp - 1u) ? d.y : 0xFFFFFFFFu;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) hi = min(hi, __shfl_xor_sync(kFull, hi, o));
      hi = min(hi, chain_hi);
      bool overlap = exists && d.z < hi;                 // first doc of the block (prev_last + 1) <= hi
      const bool consumed = exists && d.y <= hi;          // block ends inside the window
      const uint32_t co = __ballot_sync(kFull, consumed);
      float bound = __int_as_float(0x7f800000);           // +inf: no block-max data => never skipped
      if (prune) {
        if (overlap) {
          const uint2 fn = __ldg(P.seg.blk_max + gblk);
          if (fn.x != 0u) bound = pair_bound(fn.x, fn.y, s_qt[t]);
        }
        // per-term window bound = max over the term's blocks that reach into the window (0 if none)
        s_item_bound[buf][lane] = overlap ? bound : 0.f;
        __syncwarp();
        if (lane < Tp) {
          float ub = 0.f;
          for (uint32_t i = lane * mp; i < min(lane * mp + mp, 32u); ++i) ub = fmaxf(ub, s_item_bound[buf][i]);
          s_term_ub[buf][lane] = ub;
        }
        __syncwarp();
        // A block is dropped when even its own block-max plus the best the OTHER lists can add inside this
        // window stays below the threshold (SingleWandIterator's block skip, iterator_score.hpp:218-233, for
        // one term; the window-level test of MaxScore for several). Strict '<': an equal score could still
        // win on doc id. Sum in ascending-cost order with this term's contribution replaced by the bound.
        float sum = 0.f;
        for (uint32_t u = 0; u < Tp; ++u) sum = __fadd_rn(sum, u == t ? bound : s_term_ub[buf][u]);
        if (driver) sum = __fadd_rn(sum, s_ubL);
        if (overlap && __fmul_rn(sum, 1.000001f) < thr) overlap = false;
        __syncwarp();
      }
      const uint32_t ov = __ballot_sync(kFull, overlap);
      const bool skip_window = prune && ov == 0u && tries < 64u;
      if (overlap) {
        const uint32_t idx = __popc(ov & ((1u << lane) - 1u));
        s_item[buf][idx] = d;
        s_item_term[buf][idx] = t;
      }
      __syncwarp();
      if (overlap) s_item_bound[buf][__popc(ov & ((1u << lane) - 1u))] = bound;   // re-indexed by item
      if (lane <= Tp) {  // first item of term `lane` = overlapping lanes below the term's first lane
        const uint32_t first_lane = min(lane * mp, 32u);
        s_phase[buf][lane] = first_lane >= 32u ? __popc(ov) : __popc(ov & ((1u << first_lane) - 1u));
      }
      if (lane > Tp && lane <= T) s_phase[buf][lane] = __popc(ov);     // driver mode: the probed list owns no items
      if (lane < Tp) {
        const uint32_t lo_l = lane * mp, n = min(mp, 32u - lo_l);
        const uint32_t bits = n >= 32u ? 0xFFFFFFFFu : (((1u << n) - 1u) << lo_l);
        s_cursor[lane] += __popc(co & bits);
      }
      if (kDrive && driver && lane == 31u) {
        // block range of L covering [lo, hi]: gallop from its cursor (windows only move forward)
        const uint4* B = P.seg.blocks + s_qt[T - 1u].blk_begin;
        const uint32_t nblk = s_qt[T - 1u].nblk;
        uint32_t a = s_cursor[T - 1u], step = 1u;          // first block with last_doc >= lo
        while (a + step <= nblk && __ldg(&B[a + step - 1u].y) < lo) { a += step; step <<= 1; }
        uint32_t l = a, r = min(a + step - 1u, nblk);
        while (l < r) { const uint32_t mid = (l + r) >> 1; if (__ldg(&B[mid].y) < lo) l = mid + 1u; else r = mid; }
        const uint32_t b0 = l;
        uint32_t e = b0; step = 1u;                         // first block that starts after hi
        while (e + step <= nblk && __ldg(&B[e + step - 1u].z) < hi) { e += step; step <<= 1; }
        l = e; r = min(e + step - 1u, nblk);
        while (l < r) { const uint32_t mid = (l + r) >> 1; if (__ldg(&B[mid].z) < hi) l = mid + 1u; else r = mid; }
        s_cursor[T - 1u] = b0;
        s_Lb0[buf] = b0; s_Lb1[buf] = l;
      }
      __syncwarp();
      if (!skip_window) {
        if (lane == 0) { s_lo[buf] = lo; s_hi[buf] = hi; s_valid[buf] = driver ? 2u : 1u; }
        __syncwarp();
        return hi + 1u;  // wraps to 0 at 2^32-1: treated as "past the end"
      }
      lo = hi + 1u;      // nothing in [lo, hi] can reach the threshold: plan the next window straight away
      __syncwarp();
    }
  };

  // Candidate buffer full: exact radix select keeps the best k and raises the thresholds (the GPU
  // analogue of nth_element at 2k, iterators.hpp:216-228). All threads call it.
  auto compact = [&]() {
    if (min(s_ncand, P.cap) > P.k) {       // uniform (shared value, read after a barrier)
      const unsigned long long kth = block_select_topk(cand, P.cap, P.k, s_hist);
      if (tid == 0) {
        if (kth > s_theta) s_theta = kth;
        atomicMax(P.theta + q, kth);
        s_ncand = P.k;
      }
    } else if (tid == 0) {
      s_ncand = min(s_ncand, P.cap);
    }
    __syncthreads();
  };

  uint32_t next_lo = 0;  // meaningful in warp 0 only
  if (warp == 0) next_lo = plan(chain_lo, 0);
  __syncthreads();

  for (uint32_t buf = 0; s_valid[buf]; buf ^= 1u) {
    const uint32_t lo = s_lo[buf], hi = s_hi[buf];
    const bool driver = kDrive && s_valid[buf] == 2u;               // this window was planned without the largest list
    const uint32_t Tw = driver ? T - 1u : T;              // lists decoded into entry arrays in this window
    const uint32_t n_items = s_phase[buf][Tw];
    if (tid == 0) {  // pick up thresholds published by other chains / earlier segments
      const unsigned long long gt = *reinterpret_cast<volatile unsigned long long*>(P.theta + q);
      if (gt > s_theta) s_theta = gt;
      s_nprobe = 0u;
    }
    if (warp == 0) next_lo = plan(next_lo, buf ^ 1u);  // next window's plan overlaps this window's work

    // ---- 1. decode + score: one 128-posting block per warp iteration -> entries [it*128, it*128+128) ----
    for (uint32_t it = warp; it < n_items; it += kTopkWarps) {
      const uint4 d = s_item[buf][it];
      const uint32_t t = s_item_term[buf][it];
      uint32_t doc[4], f[4];
      decode_docs(P.seg.arena, d, lane, stage[warp], doc);
      decode_freqs(P.seg.arena, d, lane, f);
      const uint32_t len = desc_len(d.w);
      const float c0 = s_qt[t].c0, nc = s_qt[t].norm_const, nl = s_qt[t].norm_length;
      uint32_t nrm[4]; bool in[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (4u * lane + j >= len) doc[j] = kPadDoc;       // short (last) block of a list: pad sorts last
        in[j] = doc[j] >= lo && doc[j] <= hi;               // docs of a straddling block outside the window stay
        nrm[j] = in[j] ? load_norm(P.seg.norms, P.seg.norm_width, doc[j]) : 1u;   // in the array (sortedness) but are never emitted
      }
      uint4 od; float4 os;
      od.x = doc[0]; od.y = doc[1]; od.z = doc[2]; od.w = doc[3];
      os.x = in[0] ? bm25(f[0], nrm[0], c0, nc, nl) : 0.f;
      os.y = in[1] ? bm25(f[1], nrm[1], c0, nc, nl) : 0.f;
      os.z = in[2] ? bm25(f[2], nrm[2], c0, nc, nl) : 0.f;
      os.w = in[3] ? bm25(f[3], nrm[3], c0, nc, nl) : 0.f;
      reinterpret_cast<uint4*>(e_doc + it * 128u)[lane] = od;
      reinterpret_cast<float4*>(e_score + it * 128u)[lane] = os;
      if (P.conjunction) reinterpret_cast<uint32_t*>(e_cnt + it * 128u)[lane] = 0u;
    }
    __syncthreads();

    // ---- 2. fold term t into term t+1 (sources: live entries of terms 0..t) ----
    for (uint32_t t = 0; t + 1u < Tw; ++t) {
      const uint32_t src_end = s_phase[buf][t + 1u] * 128u;
      const uint32_t dst_begin = src_end, dst_n = (s_phase[buf][t + 2u] - s_phase[buf][t + 1u]) * 128u;
      // Conjunction: the only candidates still alive at step t sit in term t's own slots and have
      // collected every earlier term (cnt == t); anything else can never complete.
      const uint32_t src_begin = P.conjunction ? s_phase[buf][t] * 128u : 0u;
      for (uint32_t e = src_begin + tid; e < src_end; e += blockDim.x) {
        const uint32_t d = e_doc[e];
        if (d - lo > hi - lo) continue;     // padding (0xFFFFFFFF), folded entries, docs of straddling blocks outside the window
        if (P.conjunction && e_cnt[e] != t) { e_doc[e] = kPadDoc; continue; }
        uint32_t pos = dst_n;
        if (dst_n) pos = lower_bound_u32(e_doc + dst_begin, dst_n, d);
        if (pos < dst_n && e_doc[dst_begin + pos] == d) {
          e_score[dst_begin + pos] = __fadd_rn(e_score[e], e_score[dst_begin + pos]);
          if (P.conjunction) e_cnt[dst_begin + pos] = uint8_t(e_cnt[e] + 1u);
          e_doc[e] = kPadDoc;                 // folded: the target slot now carries this doc
        } else if (P.conjunction) {
          e_doc[e] = kPadDoc;                 // conjunction: a miss kills the candidate
        }
      }
      __syncthreads();
    }

    // ---- 2b. driver mode: probe the largest list L for the candidates that can still qualify ----
    if (kDrive && driver) {
      const uint32_t n_ent = n_items * 128u;
      const float thr = __uint_as_float(uint32_t(s_theta >> 32));
      const float ubL = s_ubL;
      for (uint32_t e0 = 0; e0 < n_ent; e0 += blockDim.x) {
        const uint32_t e = e0 + tid;
        const uint32_t d = e < n_ent ? e_doc[e] : kPadDoc;
        const bool live = d - lo <= hi - lo;
        // even with L's best possible contribution this doc stays below the threshold: drop it
        const bool cand = live && !(__fadd_rn(e_score[live ? e : 0u], ubL) < thr);
        if (live && !cand) e_doc[e] = kPadDoc;
        const uint32_t cb = __ballot_sync(kFull, cand);
        if (cb) {
          uint32_t base = 0;
          if (lane == 0) base = atomicAdd(&s_nprobe, uint32_t(__popc(cb)));
          base = __shfl_sync(kFull, base, 0);
          if (cand) s_probe[base + __popc(cb & ((1u << lane) - 1u))] = uint16_t(e);
        }
      }
      __syncthreads();
      const QTermDev& L = s_qt[T - 1u];
      const uint4* LB = P.seg.blocks + L.blk_begin;
      const uint32_t Lb0 = s_Lb0[buf], Lb1 = s_Lb1[buf];
      const uint32_t n_probe = s_nprobe;
      // (i) one candidate per lane: locate its block of L (interpolated guess + gallop: L's blocks are near
      // uniform in doc space), block-max test, then membership + rank straight from the bitset and a
      // random-access frequency -- no block decode. Candidates in blocks with other encodings are queued
      // (second half of s_probe) for the warp-cooperative decode below.
      if (tid == 0) s_nslow = 0u;
      __syncthreads();
      for (uint32_t c = tid; c < n_probe; c += blockDim.x) {
        const uint32_t e = s_probe[c];
        const uint32_t d = e_doc[e];
        const float partial = e_score[e];
        if (Lb1 == Lb0) continue;
        const uint32_t nb = Lb1 - Lb0;
        const uint32_t guess = Lb0 + min(nb - 1u, uint32_t((static_cast<unsigned long long>(d - lo) * nb) / (static_cast<unsigned long long>(hi - lo) + 1ull)));
        const uint32_t bl = find_block_from(LB, Lb0, Lb1, guess, d);
        if (bl >= Lb1) continue;                                          // beyond L's last block in the window
        const uint4 pd = ld_ro_v4(LB + bl);
        if (!(pd.z < d)) continue;
        const uint2 fn = __ldg(P.seg.blk_max + L.blk_begin + bl);
        if (fn.x != 0u && __fmul_rn(__fadd_rn(partial, pair_bound(fn.x, fn.y, L)), 1.000001f) < thr) {
          e_doc[e] = kPadDoc;                                             // cannot qualify even with this block's best
          continue;
        }
        uint32_t rank = 0, fr = 0;
        bool fast = false;
        if (desc_doc_enc(pd.w) == 4u) {
          if (!bitset_rank(P.seg.arena, pd, d, rank)) continue;           // doc not in L: the driver score stands
          fast = freq_at(P.seg.arena, pd, rank, fr);
        }
        if (fast) {
          const float sL = bm25(fr, load_norm(P.seg.norms, P.seg.norm_width, d), L.c0, L.norm_const, L.norm_length);
          e_score[e] = __fadd_rn(partial, sL);                            // L is last in ascending-cost order
        } else {
          s_probe[kEntries + atomicAdd(&s_nslow, 1u)] = uint16_t(e);      // second half of s_probe
        }
      }
      __syncthreads();
      const uint32_t n_slow = s_nslow;
      uint32_t have_blk = 0xFFFFFFFFu;
      uint32_t pdoc[4], pf[4];
      bool have_f = false;
      uint4 pd = make_uint4(0, 0, 0, 0);
      // (ii) warp per remaining candidate: decode its block
      for (uint32_t c = warp; c < n_slow; c += kTopkWarps) {
        const uint32_t e = s_probe[kEntries + c];
        const uint32_t d = e_doc[e];
        const float partial = e_score[e];
        // 32-ary search over L's blocks [Lb0, Lb1): first block with last_doc >= d
        uint32_t bl = Lb0, bn = Lb1 - Lb0;
        while (bn > 1u) {
          const uint32_t step = (bn + 31u) >> 5;
          const uint32_t idx = min((lane + 1u) * step, bn) - 1u;        // lane i looks at the last block of its slice
          const bool ge = __ldg(&LB[bl + idx].y) >= d;
          const uint32_t m = __ballot_sync(kFull, ge);
          if (m == 0u) { bl += bn; bn = 0u; break; }                     // beyond every block of the range
          const uint32_t fsl = uint32_t(__ffs(m) - 1);
          const uint32_t nb = min((fsl + 1u) * step, bn) - fsl * step;
          bl += fsl * step; bn = nb;
        }
        if (bn == 0u) continue;
        if (have_blk != bl) {
          pd = ld_ro_v4(LB + bl);
          have_blk = bl; have_f = false;
          if (!(pd.z < d && d <= pd.y)) { have_blk = 0xFFFFFFFFu; continue; }   // d falls between blocks: not in L
          const uint2 fn = __ldg(P.seg.blk_max + L.blk_begin + bl);
          if (fn.x != 0u && __fmul_rn(__fadd_rn(partial, pair_bound(fn.x, fn.y, L)), 1.000001f) < thr) {
            e_doc[e] = kPadDoc;                                          // cannot qualify even with this block's best
            have_blk = 0xFFFFFFFFu;
            continue;
          }
          decode_docs(P.seg.arena, pd, lane, stage[warp], pdoc);
          const uint32_t len = desc_len(pd.w);
#pragma unroll
          for (int j = 0; j < 4; ++j) if (4u * lane + j >= len) pdoc[j] = kPadDoc;
        } else if (!(pd.z < d && d <= pd.y)) {
          continue;
        }
        const bool h0 = pdoc[0] == d, h1 = pdoc[1] == d, h2 = pdoc[2] == d, h3 = pdoc[3] == d;
        const uint32_t hit = __ballot_sync(kFull, h0 | h1 | h2 | h3);
        if (!hit) continue;                                              // doc not in L
        if (!have_f) { decode_freqs(P.seg.arena, pd, lane, pf); have_f = true; }
        if (h0 | h1 | h2 | h3) {
          const uint32_t fr = h0 ? pf[0] : h1 ? pf[1] : h2 ? pf[2] : pf[3];
          const float sL = bm25(fr, load_norm(P.seg.norms, P.seg.norm_width, d), L.c0, L.norm_const, L.norm_length);
          e_score[e] = __fadd_rn(partial, sL);                           // L is last in ascending-cost order
        }
      }
      __syncthreads();
    }

    // ---- 3. emit live in-window entries ----
    const uint32_t n_entries = n_items * 128u;
    const uint32_t emit_begin = P.conjunction ? s_phase[buf][T - 1u] * 128u : 0u;  // AND: only the last term's slots can be complete (never in driver mode)
    bool first_pass = true;
    const bool plain = !P.conjunction && P.filt.ps.n == 0 && P.seg.deleted == nullptr && !kExcl;   // disjunction, no table filter, no deletes, no exclusions: 4 entries per lane
    for (;;) {
      const unsigned long long theta = s_theta;
      const uint32_t theta_hi = uint32_t(theta >> 32);
      uint32_t matched = 0;
      bool pending = false;
      if (plain) {
        // Vector pass: one 16-byte load of docs and of scores per lane; the score bits are tested against the
        // threshold's score half, and only a warp that holds at least one possible candidate enters the append path.
        for (uint32_t e0 = 0; e0 < n_entries; e0 += blockDim.x * 4u) {
          const uint32_t e = e0 + tid * 4u;                    // n_entries is a multiple of 128
          uint4 d4 = make_uint4(kPadDoc, kPadDoc, kPadDoc, kPadDoc);
          uint4 s4 = make_uint4(0u, 0u, 0u, 0u);
          if (e < n_entries) {
            d4 = *reinterpret_cast<const uint4*>(e_doc + e);
            s4 = *reinterpret_cast<const uint4*>(e_score + e);
          }
          const uint32_t span = hi - lo;
          const bool l0 = d4.x - lo <= span, l1 = d4.y - lo <= span, l2 = d4.z - lo <= span, l3 = d4.w - lo <= span;
          if (first_pass) matched += uint32_t(l0) + uint32_t(l1) + uint32_t(l2) + uint32_t(l3);
          const bool w0 = l0 && s4.x >= theta_hi, w1 = l1 && s4.y >= theta_hi, w2 = l2 && s4.z >= theta_hi, w3 = l3 && s4.w >= theta_hi;
          if (!__any_sync(kFull, w0 | w1 | w2 | w3)) continue;   // the common case once the threshold is up
          const uint32_t dd[4] = {d4.x, d4.y, d4.z, d4.w}, ss[4] = {s4.x, s4.y, s4.z, s4.w};
          const bool ww[4] = {w0, w1, w2, w3};
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            bool want = ww[j];
            unsigned long long key = 0ull;
            if (want) { key = make_key(__uint_as_float(ss[j]), P.seg.ordinal_base + dd[j]); want = key > theta; }
            const uint32_t wb = __ballot_sync(kFull, want);
            if (!wb) continue;
            uint32_t base = 0;
            if (lane == 0) base = atomicAdd(&s_ncand, uint32_t(__popc(wb)));
            base = __shfl_sync(kFull, base, 0);
            if (want) {
              const uint32_t pos = base + __popc(wb & ((1u << lane) - 1u));
              if (pos < P.cap) { cand[pos] = key; e_doc[e + j] = kPadDoc; }   // stored: tombstone so that a retry skips it
              else pending = true;
            }
          }
        }
      } else {
      for (uint32_t e0 = emit_begin; e0 < n_entries; e0 += blockDim.x) {
        const uint32_t e = e0 + tid;
        const uint32_t d = e < n_entries ? e_doc[e] : kPadDoc;
        bool live = d - lo <= hi - lo;                       // in window, not padding / folded / already stored
        if (live && P.conjunction) live = e_cnt[e] == T - 1u;
        if (live && P.seg.deleted != nullptr) live = ((__ldg(P.seg.deleted + (d >> 5)) >> (d & 31u)) & 1u) == 0u;   // MaskDocIterator: neither scored nor counted
        if (live && P.filt.ps.n) live = chain_pass(P.filt, d);
        if (kGroups && live) live = !excluded_doc(P.seg.arena, P.seg.blocks, P.seg.anchors, s_ex, s_exg, n_ex, d);
        else if (kExcl && live) live = !excluded_doc(P.seg.arena, P.seg.blocks, P.seg.anchors, s_ex, n_ex, d);   // neither collected nor counted
        // cheap pre-test on the score bits alone; the full 64-bit key only for the few that may qualify
        const uint32_t sbits = live ? __float_as_uint(e_score[e]) : 0u;
        matched += (live && first_pass) ? 1u : 0u;
        bool want = live && sbits >= theta_hi;
        unsigned long long key = 0ull;
        if (want) { key = make_key(__uint_as_float(sbits), P.seg.ordinal_base + d); want = key > theta; }
        const uint32_t wb = __ballot_sync(kFull, want);
        if (wb) {                                            // uniform: most iterations append nothing once the threshold is up
          uint32_t base = 0;
          if (lane == 0) base = atomicAdd(&s_ncand, uint32_t(__popc(wb)));
          base = __shfl_sync(kFull, base, 0);
          if (want) {
            const uint32_t pos = base + __popc(wb & ((1u << lane) - 1u));
            if (pos < P.cap) { cand[pos] = key; e_doc[e] = kPadDoc; }   // stored: tombstone so that a retry skips it
            else pending = true;
          }
        }
      }
      }
      matched = warp_sum(matched);
      if (lane == 0 && matched) atomicAdd(&s_matched, matched);
      if (!__syncthreads_or(int(pending))) break;
      compact();  // buffer overflowed: select, raise the threshold, retry the entries that did not fit
      first_pass = false;
    }
  }

  // ---- chain epilogue: best k, sorted descending (only the first pow2(k) slots need the sort) ----
  __syncthreads();
  compact();
  const uint32_t n_out = min(s_ncand, P.k);
  uint32_t sort_n = 256u;
  while (sort_n < n_out) sort_n <<= 1;      // compact() left the survivors in [0, n_out) and zeros behind them
  block_sort_desc(cand, sort_n);
  const size_t list = work.w;
  unsigned long long* out = P.cand + list * P.cap;
  for (uint32_t i = tid; i < n_out; i += blockDim.x) out[i] = cand[i];   // the merge reads cand_n entries only
  if (tid == 0) {
    P.cand_n[list] = n_out;
    if (s_matched) atomicAdd(P.total + q, static_cast<unsigned long long>(s_matched));
  }
}

// ------------------------------------------------------------------------------------------
// Merge the candidate lists of each query into its final top-k (one CTA per query).
// keys_out[q][k] sorted descending, zero-padded. Streaming: buffer = [best so far | next chunk];
// when the buffer is full an exact radix select keeps the best k; one bitonic sort at the end.
// Lists are sorted descending, so a list whose head is below the current k-th is skipped outright.
// ------------------------------------------------------------------------------------------
struct MergeParams {
  const unsigned long long* cand;  // [lists][stride]; query q owns lists [list_off[q], list_off[q+1]), or [q*G, (q+1)*G) when list_off is null
  const uint32_t* cand_n;          // [lists] (null => every list holds `stride` slots: its keys, then zeros)
  const uint32_t* list_off;        // [Q+1] or null
  uint32_t G, stride, k, cap;      // cap = power of two > k, multiple of the CTA size
  unsigned long long* keys_out;    // [Q][k]
  uint32_t* n_out;                 // [Q]
};

__global__ void __launch_bounds__(kTopkThreads)
topk_merge_kernel(const MergeParams P) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* buf = reinterpret_cast<unsigned long long*>(smem_raw);
  __shared__ uint32_t s_n;
  __shared__ unsigned long long s_kth;
  __shared__ uint32_t s_hist[258];
  const uint32_t q = blockIdx.x, tid = threadIdx.x;
  for (uint32_t i = tid; i < P.cap; i += blockDim.x) buf[i] = 0ull;
  if (tid == 0) { s_n = 0u; s_kth = 0ull; }
  __syncthreads();
  const uint32_t l_begin = P.list_off ? P.list_off[q] : q * P.G, l_end = P.list_off ? P.list_off[q + 1] : (q + 1u) * P.G;
  if (l_end - l_begin == 1u && P.cand_n != nullptr) {
    // one chain: its list is already the query's answer (<= k keys, sorted descending by the chain's epilogue)
    const unsigned long long* src = P.cand + size_t(l_begin) * P.stride;
    const uint32_t n = min(min(P.cand_n[l_begin], P.stride), P.k);
    for (uint32_t i = tid; i < P.k; i += blockDim.x) P.keys_out[size_t(q) * P.k + i] = i < n ? src[i] : 0ull;
    if (tid == 0) P.n_out[q] = n;
    return;
  }
  for (uint32_t g = l_begin; g < l_end; ++g) {
    const unsigned long long* src = P.cand + size_t(g) * P.stride;
    uint32_t n;
    if (P.cand_n) {
      n = min(P.cand_n[g], P.stride);
    } else {
      // zero-padded list: only its non-zero prefix counts (sorted descending, so the zeros are the tail). A zero taken
      // into the buffer would count as a key and could stop the select below from compacting.
      uint32_t lo = 0, hi = P.stride;
      while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (src[mid] != 0ull) lo = mid + 1; else hi = mid;
      }
      n = lo;
    }
    uint32_t base = 0;
    while (base < n) {
      const uint32_t have = s_n;
      const unsigned long long kth = s_kth;
      __syncthreads();
      if (src[base] <= kth) break;                       // sorted list: nothing below can matter
      const uint32_t take = min(P.cap - have, n - base);
      for (uint32_t i = tid; i < take; i += blockDim.x) buf[have + i] = src[base + i];
      __syncthreads();
      base += take;
      if (have + take == P.cap) {                        // full: keep the best k
        const unsigned long long nk = block_select_topk(buf, P.cap, P.k, s_hist);
        if (tid == 0) { s_n = P.k; if (nk > s_kth) s_kth = nk; }
      } else if (tid == 0) {
        s_n = have + take;
      }
      __syncthreads();
    }
  }
  if (s_n > P.k) {
    block_select_topk(buf, P.cap, P.k, s_hist);
    if (tid == 0) s_n = P.k;
    __syncthreads();
  }
  uint32_t sort_n = 256u;
  while (sort_n < min(s_n, P.k)) sort_n <<= 1;
  // entries beyond s_n may be stale-free zeros only when a select ran; make sure of it before sorting
  for (uint32_t i = s_n + tid; i < sort_n; i += blockDim.x) buf[i] = 0ull;
  __syncthreads();
  block_sort_desc(buf, sort_n);
  uint32_t real = 0;
  for (uint32_t i = tid; i < P.k; i += blockDim.x) {
    const unsigned long long v = i < s_n ? buf[i] : 0ull;
    P.keys_out[size_t(q) * P.k + i] = v;
    real += v != 0ull;
  }
  real = warp_sum(real);
  __shared__ uint32_t s_real;
  if (tid == 0) s_real = 0u;
  __syncthreads();
  if ((tid & 31u) == 0 && real) atomicAdd(&s_real, real);
  __syncthreads();
  if (tid == 0) P.n_out[q] = s_real;
}

// ---- the BM25 top-k across ranks ----
// A rank's buffer (sdbg_bm25_topk_batch_groups_min_device): this header, then the region the local entries fill, keys
// [nq][k] (score bits << 32 | ~ordinal within the rank, best first) | total_matches u64 [nq] | hit counts u32 [nq], padded
// to a multiple of 8 bytes so that every rank's keys stay 8-byte aligned in the gathered array.
struct TopkDistHeader {
  unsigned long long k, nq;
  unsigned long long failed;   // non-zero: this rank's local pass failed
  unsigned long long pad[5];
};
static_assert(sizeof(TopkDistHeader) == 64, "the keys stay 8-byte aligned");

__host__ __device__ __forceinline__ size_t topk_dist_bytes(size_t nq, uint32_t k) {
  return sizeof(TopkDistHeader) + ((nq * (size_t(k) * 8 + 12) + 7) & ~size_t(7));
}

// Rank and ordinal do not fit in 32 bits together, so the merge orders by position instead: list (q, r) of the gathered
// buffers becomes row q * n_ranks + r of `keys`, key i of it score_bits << 32 | ~(r * k + i). Within a rank the keys are
// sorted by (score desc, ordinal asc), so the positional keys order by (score desc, rank asc, ordinal asc) and are never
// zero while n_ranks * k < 2^32. cand_n[row] = the list's hit count (at most k).
__global__ void __launch_bounds__(256) topk_rekey_gathered_kernel(const char* __restrict__ all, size_t rank_bytes, uint32_t n_ranks,
                                                                  uint32_t nq, uint32_t k, unsigned long long* __restrict__ keys,
                                                                  uint32_t* __restrict__ cand_n) {
  const size_t rows = size_t(nq) * n_ranks;
  for (size_t row = blockIdx.x; row < rows; row += gridDim.x) {
    const uint32_t q = uint32_t(row / n_ranks), r = uint32_t(row - size_t(q) * n_ranks);
    const char* b = all + r * rank_bytes + sizeof(TopkDistHeader);
    const auto* src = reinterpret_cast<const unsigned long long*>(b) + size_t(q) * k;
    const uint32_t n = min(reinterpret_cast<const uint32_t*>(b + size_t(nq) * (size_t(k) * 8 + 8))[q], k);
    unsigned long long* dst = keys + row * k;
    const uint32_t pos0 = r * k;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x)
      dst[i] = (src[i] & 0xFFFFFFFF00000000ull) | static_cast<unsigned long long>(~(pos0 + i));
    if (threadIdx.x == 0) cand_n[row] = n;
  }
}

// One CTA per query: the merged positional keys back to hits {score, ordinal within the rank, rank} (the layout of
// sdbg_hit), and the query's total_matches summed over the ranks.
__global__ void __launch_bounds__(256) topk_hits_gathered_kernel(const char* __restrict__ all, size_t rank_bytes, uint32_t n_ranks,
                                                                 uint32_t nq, uint32_t k, const unsigned long long* __restrict__ merged,
                                                                 const uint32_t* __restrict__ n_out, uint3* __restrict__ hits,
                                                                 unsigned long long* __restrict__ totals) {
  __shared__ unsigned long long s_total;
  const uint32_t q = blockIdx.x;
  if (threadIdx.x == 0) s_total = 0ull;
  __syncthreads();
  const uint32_t n = n_out[q];
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    const unsigned long long key = merged[size_t(q) * k + i];
    const uint32_t pos = ~uint32_t(key), r = pos / k, j = pos - r * k;
    const auto* src = reinterpret_cast<const unsigned long long*>(all + r * rank_bytes + sizeof(TopkDistHeader));
    hits[size_t(q) * k + i] = make_uint3(uint32_t(key >> 32), ~uint32_t(src[size_t(q) * k + j]), r);
  }
  unsigned long long t = 0;
  for (uint32_t r = threadIdx.x; r < n_ranks; r += blockDim.x)
    t += reinterpret_cast<const unsigned long long*>(all + r * rank_bytes + sizeof(TopkDistHeader) + size_t(nq) * k * 8)[q];
  if (t) atomicAdd(&s_total, t);
  __syncthreads();
  if (threadIdx.x == 0) totals[q] = s_total;
}

}  // namespace sdbg
