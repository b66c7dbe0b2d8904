// bm25_stream.cuh -- warp-autonomous BM25 scan + score + top-k for disjunctions of 1..4 terms (sm_90a).
//
// Reference behaviour being reproduced (paths relative to /root/reference/libs/iresearch/include/iresearch):
//   block walk    formats/posting/iterator_doc.hpp:309-430 (Collect / ScoreBlock / ProcessBatch: one 128-posting
//                 block at a time: decode -> norms -> score -> collector)
//   disjunction   search/max_score_iterator.hpp:311-356 (ScoreAndCollectWindow: Sum merge of the lists' scores)
//   sum order     search/conjunction.hpp:185-195 (sub-scores added in ascending-cost order)
//   collector     index/iterators.hpp:103-250 (buffer, select at capacity, threshold = k-th)
//
// Why a second kernel: bm25_topk_kernel (bm25_kernels.cuh) moves every window through CTA-wide phases (decode ->
// barrier -> fold by binary search over up to 4096 entries -> barrier -> emit -> barrier); ncu showed it bound by
// instruction issue with the block barrier as the largest stall. Here nothing in the scan is CTA-wide:
//
//   * a CTA is eight independent WARPS, each owning a contiguous doc sub-range of the work item's chain; the only
//     CTA-wide events are the candidate-buffer compactions (a rendezvous every ~1000 accepted candidates);
//   * every term has one LIVE block per warp (128 sorted doc ids + scores in shared memory). A step replaces the
//     live block(s) that ended at the previous frontier and then finalises the docs up to phi = min over terms of the
//     live block's last doc -- every list has been decoded at least that far. Each step retires at least one block;
//     each posting is decoded, scored and finalised exactly once;
//   * the pending entries of a live block are an index range [a0, a1) of its sorted ids, handled 32 at a time, one
//     entry per lane: an entry of term t looks for its doc in the live block of term t+1, t+2, ... (7-step binary
//     search over 128 ids); on a hit it adds its score INTO that slot (acc + s_u: the reference's ascending-cost sum
//     order, bit-reproducible for any number of terms) and dies; an entry nobody absorbs is final and is tested
//     against the threshold;
//   * block payloads arrive through the TMA engine: per warp and term two 512-byte slots, filled two blocks ahead by
//     cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes (SASS UBLKCP) and awaited on an mbarrier
//     (SYNCS), so the decode reads shared memory and does not wait for L2 / HBM;
//   * BM25 per posting is computed (bm25_plain: the __f*_rn sequence of bm25.cpp:105-106).
// The term count is a run-time value and every per-term loop is rolled: the whole scan is ~2 k instructions, so the
// eight warps of a CTA, which are all at different places of it, stay inside the instruction cache (the first
// version unrolled everything per term: 17 k instructions for two terms and `no_instruction` as its top stall).
#pragma once

#include "bm25_kernels.cuh"

namespace sdbg {

constexpr uint32_t kStreamMaxTerms = 4;
constexpr uint32_t kSlotUnits = 32;    // prefetch slot = 32 x 16 B
constexpr uint32_t kNoDoc = 0xFFFFFFFFu;
constexpr int kStreamMinBlocks = 3;    // CTAs per SM in __launch_bounds__ of the stream and merge kernels (80 registers)
// per warp and term: docs[128] u32 | scores[128] f32 | slots[2][32] uint4 | descriptor window[32] uint4
constexpr uint32_t kStreamTermBytes = 512u + 512u + 1024u + 512u;

struct StreamCtl {   // CTA-wide control block (shared memory)
  unsigned long long theta;
  uint32_t ncand, matched, full, active;
  uint32_t hist[258];
};

// A block is prefetched into its slot unless it is larger than a slot. Its size is exact: payloads are contiguous in
// the arena in block order, so units = off16 of the next block - off16 of this one (the block table ends with a
// sentinel).
__device__ __forceinline__ void unpack4s(const uint4* p, uint32_t b, uint32_t lane, uint32_t v[4]) {
  const uint32_t bit = lane * b;
  const uint32_t w = bit >> 5, sh = bit & 31u;
  const uint4 lo = p[w];
  const uint4 hi = p[min(w + 1u, b - 1u)];
  const uint32_t mask = (1u << b) - 1u;  // b <= 31
  v[0] = __funnelshift_r(lo.x, hi.x, sh) & mask;
  v[1] = __funnelshift_r(lo.y, hi.y, sh) & mask;
  v[2] = __funnelshift_r(lo.z, hi.z, sh) & mask;
  v[3] = __funnelshift_r(lo.w, hi.w, sh) & mask;
}

// StreamVByte 1234 from shared memory (tails only): control byte `lane` describes this lane's four values.
// Scored scan: every match goes out through a global cursor, one atomic per warp.
__device__ __noinline__ void stream_emit(uint32_t* docs, float* scores, unsigned long long* count, unsigned long long cap,
                                         bool alive, uint32_t dv, float sv) {
  const uint32_t bal = __ballot_sync(kFull, alive);
  if (!bal) return;
  const uint32_t lane = threadIdx.x & 31u;
  unsigned long long base = 0ull;
  if (lane == uint32_t(__ffs(int(bal)) - 1)) base = atomicAdd(count, static_cast<unsigned long long>(__popc(bal)));
  base = __shfl_sync(kFull, base, __ffs(int(bal)) - 1);
  const unsigned long long pos = base + __popc(bal & ((1u << lane) - 1u));
  if (alive && pos < cap) { docs[pos] = dv; scores[pos] = sv; }
}

__device__ __noinline__ void svb4s(const uint4* p, uint32_t len, uint32_t lane, uint32_t* v_out /* shared: 128 u32 */) {
  const uint8_t* bytes = reinterpret_cast<const uint8_t*>(p);
  const uint32_t nctl = (len + 3u) >> 2;
  const uint32_t ctl = lane < nctl ? uint32_t(bytes[lane]) : 0u;
  uint32_t n[4], mine = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    n[j] = (4u * lane + j < len) ? ((ctl >> (2 * j)) & 3u) + 1u : 0u;
    mine += n[j];
  }
  uint32_t pos = nctl + warp_incl_scan(mine, lane) - mine;
  uint32_t v[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    uint32_t x = 0;
    for (uint32_t k = 0; k < n[j]; ++k) x |= uint32_t(bytes[pos + k]) << (8 * k);
    pos += n[j];
    v[j] = x;
  }
  __syncwarp();
  reinterpret_cast<uint4*>(v_out)[lane] = make_uint4(v[0], v[1], v[2], v[3]);
  __syncwarp();
}

// Doc ids of one prefetched block; `pd` points at the doc payload in SHARED memory. `stage` = 128 u32 of per-warp
// shared scratch (bitset rank scatter, svb). Lane l gets postings 4l .. 4l+3.
__device__ __forceinline__ void decode_docs_smem(const uint4* pd, const uint4& d, uint32_t lane, uint32_t* stage, uint32_t doc[4]) {
  const uint32_t enc = desc_doc_enc(d.w), len = desc_len(d.w), prev = d.z;
  if (enc >= 8u) {                                  // de_delta_bitpack_b, b = enc - 6
    unpack4s(pd, enc - 6u, lane, doc);
    prefix_from_gaps(prev, lane, doc);
  } else if (enc == 4u) {                           // de_for_bitset (position-parallel expansion, see decode_docs)
    const uint32_t words = desc_words(d.w);
    uint4 x = make_uint4(0, 0, 0, 0);
    if (2u * lane < words) x = pd[lane];
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
  } else if (enc >= 1u && enc <= 3u) {              // de_delta_all_same_{08,16,32}
    const uint32_t raw = *reinterpret_cast<const uint32_t*>(pd);
    const uint32_t g = enc == 1u ? (raw & 0xFFu) : enc == 2u ? (raw & 0xFFFFu) : raw;
#pragma unroll
    for (int j = 0; j < 4; ++j) doc[j] = prev + g * (4u * lane + j + 1u);
  } else if (enc == 0u) {                           // de_values
    uint4 x = make_uint4(0, 0, 0, 0);
    if (4u * lane < len) x = pd[lane];
    doc[0] = x.x; doc[1] = x.y; doc[2] = x.z; doc[3] = x.w;
  } else {                                          // 5 de_streamvbyte1234, 7 de_delta_streamvbyte1234 (tails)
    svb4s(pd, len, lane, stage);
    const uint4 o = reinterpret_cast<const uint4*>(stage)[lane];
    doc[0] = o.x; doc[1] = o.y; doc[2] = o.z; doc[3] = o.w;
    __syncwarp();
    if (enc == 7u) prefix_from_gaps(prev, lane, doc);
  }
}
__device__ __forceinline__ void decode_freqs_smem(const uint4* pf, const uint4& d, uint32_t lane, uint32_t* stage, uint32_t f[4]) {
  const uint32_t fenc = desc_freq_enc(d.w), len = desc_len(d.w);
  if (fenc >= 5u) {
    unpack4s(pf, fenc - 4u, lane, f);
  } else if (fenc >= 1u && fenc <= 3u) {
    const uint32_t raw = *reinterpret_cast<const uint32_t*>(pf);
    f[0] = f[1] = f[2] = f[3] = fenc == 1u ? (raw & 0xFFu) : fenc == 2u ? (raw & 0xFFFFu) : raw;
  } else if (fenc == 0u) {
    uint4 x = make_uint4(0, 0, 0, 0);
    if (4u * lane < len) x = pf[lane];
    f[0] = x.x; f[1] = x.y; f[2] = x.z; f[3] = x.w;
  } else {
    svb4s(pf, len, lane, stage);
    const uint4 o = reinterpret_cast<const uint4*>(stage)[lane];
    f[0] = o.x; f[1] = o.y; f[2] = o.z; f[3] = o.w;
    __syncwarp();
  }
}

// Blocks that are not prefetched (StreamVByte tails, oversized raw blocks): decoded straight from the arena.
// Results go through shared memory (out_docs / out_freqs, 128 u32 each) so that the caller's registers stay registers.
__device__ __noinline__ void decode_block_global(const uint4* arena, uint4 d, uint32_t lane, uint32_t* out_docs,
                                                 uint32_t* out_freqs) {
  uint32_t doc[4], f[4];
  decode_docs(arena, d, lane, out_docs, doc);
  decode_freqs(arena, d, lane, f);
  __syncwarp();
  reinterpret_cast<uint4*>(out_docs)[lane] = make_uint4(doc[0], doc[1], doc[2], doc[3]);
  reinterpret_cast<uint4*>(out_freqs)[lane] = make_uint4(f[0], f[1], f[2], f[3]);
  __syncwarp();
}

// First block in B[0, n) whose last doc is >= x (n when none): 32-ary search, one descriptor per lane and round.
__device__ __forceinline__ uint32_t warp_first_block(const uint4* B, uint32_t n, uint32_t x, uint32_t lane) {
  uint32_t lo = 0;
  while (n > 32u) {
    const uint32_t step = (n + 31u) >> 5;
    const uint32_t idx = min((lane + 1u) * step, n) - 1u;      // last block of this lane's slice
    const bool ge = __ldg(&B[lo + idx].y) >= x;
    const uint32_t m = __ballot_sync(kFull, ge);
    if (m == 0u) return lo + n;
    const uint32_t fs = uint32_t(__ffs(m) - 1);
    const uint32_t nn = min((fs + 1u) * step, n) - fs * step;
    lo += fs * step; n = nn;
  }
  const bool ge = lane < n && __ldg(&B[lo + lane].y) >= x;
  const uint32_t m = __ballot_sync(kFull, ge);
  return m ? lo + uint32_t(__ffs(m) - 1) : lo + n;
}

// ------------------------------------------------------------------------------------------
// Probes: "does list u contain doc d, and with which frequency?" answered by ONE lane without decoding the block
// for the whole warp -- 32 candidates are looked up at once. This is what the reference does with
// it.seek(doc) on a non-essential iterator (ProcessNonEssentialFromCandidates, search/max_score_iterator.hpp:406-429)
// and on the non-lead iterators of a conjunction (Conjunction::converge / LazySeek, search/conjunction.hpp:248-340,
// PostingIteratorBase::seek, formats/posting/iterator_doc.hpp:233-306): skip-list to the block, search inside it.
// Here: gallop + binary search over the block table's last_doc column, then inside the block
//   bit-packed gaps  the staged anchors (doc ids of postings 31 / 63 / 95) pick a quarter, <= 32 gaps are summed
//   bitset           one bit test, rank by popcount
//   all-same / raw   arithmetic / binary search
//   StreamVByte      scalar walk (tail blocks only)
// followed by a random-access read of the frequency.
// ------------------------------------------------------------------------------------------
// One lane: score of doc d in the posting list of `qt`, or false when the list does not contain d. `hint` = a block
// of the list (index within the term) that is not behind d's block; on return the block that was searched.
__device__ __forceinline__ bool probe_term(const PostingsDev& S, const QTermDev& qt, uint32_t d, uint32_t hint, uint32_t& found_blk,
                                           float& score) {
  const uint4* B = S.blocks + qt.blk_begin;
  const uint32_t n = qt.nblk;
  if (n == 0u) { found_blk = 0u; return false; }
  const uint32_t l = find_block_from(B, 0u, n, min(hint, n - 1u), d);   // first block whose last doc is >= d, searched outwards from the hint
  found_blk = min(l, n - 1u);
  if (l >= n) return false;
  const uint4 desc = __ldg(B + l);
  if (d <= desc.z) return false;                       // d lies between two blocks
  uint32_t idx = 0, f = 0;
  if (!block_find_doc(S, desc, qt.blk_begin + l, d, idx)) return false;
  if (!freq_at(S.arena, desc, idx, f)) {               // StreamVByte frequencies: scalar walk
    f = svb_value_at(reinterpret_cast<const uint8_t*>(S.arena + desc.x + desc_fdelta(desc.w)), desc_len(desc.w), idx, false, false, 0u, &idx);
  }
  score = bm25_plain(f, load_norm(S.norms, S.norm_width, d), qt.c0, qt.norm_const, qt.norm_length);
  return true;
}

// One probe round of a warp: lane i takes ring entry qhead + i (i < n) and visits the probed lists u0 .. n_terms-1 in
// ascending-cost order. Outlined on purpose: the probe code is large and cold for exhaustive scans, and the scan loop
// has to stay inside the instruction cache. `wand` = TopkParams::wand: disjunctions drop candidates on bounds only when
// pruning is on.
struct ProbeResult { uint32_t d; float s; uint32_t alive; };
template <bool kAnd>
__device__ __noinline__ ProbeResult stream_probe_round(const PostingsDev* S, const QTermDev* qt, const float* sfx, uint32_t* hint,
                                                      const uint32_t* qd, const float* qs, uint32_t qhead, uint32_t n, uint32_t u0,
                                                      uint32_t n_terms, float theta_score, int wand) {
  const uint32_t lane = threadIdx.x & 31u;
  bool alive = lane < n;
  const uint32_t d = alive ? qd[(qhead + lane) & 127u] : kNoDoc;
  float s = alive ? qs[(qhead + lane) & 127u] : 0.f;
  for (uint32_t u = u0; u < n_terms; ++u) {
    if (!__any_sync(kFull, alive)) break;
    uint32_t fb = 0u;
    float su = 0.f;
    bool found = false;
    if (alive) found = probe_term(*S, qt[u], d, hint[u], fb, su);
    const uint32_t who = __ballot_sync(kFull, alive);
    fb = __shfl_sync(kFull, fb, __ffs(who) - 1);
    __syncwarp();
    if (lane == 0) hint[u] = fb;
    __syncwarp();
    if (kAnd) {
      alive = alive && found;
      if (found) s = __fadd_rn(s, su);
    } else {
      if (found) s = __fadd_rn(s, su);                       // ascending-cost order: probed lists come last
      // even with the best the remaining lists can add this doc stays below the threshold
      if (wand && alive && __fmul_rn(__fadd_rn(s, sfx[u + 1u]), 1.000001f) < theta_score) alive = false;
    }
  }
  ProbeResult r;
  r.d = d; r.s = s; r.alive = alive ? 1u : 0u;
  return r;
}

// Excluded lists of a CTA's query (TopkParams::excl), in shared memory.
struct StreamExcl {
  uint2 list[kMaxQueryTerms];
  uint32_t n;
  uint32_t hint[kTopkWarps][kMaxQueryTerms];      // per warp and list: block where the warp's last probe ended
};

// Exclusion (NOT clauses): false for lanes whose doc occurs in one of the excluded lists, else `alive`. It votes, so all
// 32 lanes call it, with `alive` as an argument. The hints advance like s_hint in stream_probe_round. Outlined for the
// same reason as that function.
__device__ __noinline__ bool stream_excl_pass(const PostingsDev* S, StreamExcl* X, bool alive, uint32_t d) {
  const uint32_t lane = threadIdx.x & 31u;
  uint32_t* const hint = X->hint[threadIdx.x >> 5];
  for (uint32_t x = 0; x < X->n; ++x) {
    if (!__any_sync(kFull, alive)) break;
    uint32_t fb = 0u;
    bool hit = false;
    if (alive) hit = probe_contains(*S, X->list[x], d, hint[x], fb);
    const uint32_t who = __ballot_sync(kFull, alive);
    fb = __shfl_sync(kFull, fb, __ffs(who) - 1);
    __syncwarp();
    if (lane == 0) hint[x] = fb;
    __syncwarp();
    alive = alive && !hit;
  }
  return alive;
}

// Check lists of a CTA's query with OR groups (TopkParams::excl / excl_grp: excluded lists and the groups' lists), in
// shared memory.
struct StreamGroups {
  uint2 list[kMaxCheckLists];
  uint8_t grp[kMaxCheckLists];                    // kCheckExcl or the list's group tag
  uint32_t n;
  uint32_t e0;                                    // live terms at the start of the scan (pigeonhole lead; else T)
  GroupNeed need;                                 // per-group counters at the start of a doc's check
  uint32_t hint[kTopkWarps][kMaxCheckLists];      // per warp and list: block where the warp's last probe ended
};

// The same with OR groups: false for lanes whose doc occurs in an excluded list, or whose doc fewer than m_g lists of
// some required group hold; else `alive`. A lane stops probing a group once m_g of its lists hold the doc, and rejects
// the doc once the group's remaining lists cannot reach m_g.
__device__ __noinline__ bool stream_excl_pass(const PostingsDev* S, StreamGroups* X, bool alive, uint32_t d) {
  const uint32_t lane = threadIdx.x & 31u;
  uint32_t* const hint = X->hint[threadIdx.x >> 5];
  GroupNeed st = X->need;
  for (uint32_t x = 0; x < X->n; ++x) {
    if (!__any_sync(kFull, alive)) break;
    const uint32_t g = X->grp[x];
    const uint32_t g4 = 4u * (g & 15u);
    const bool excl = g == kCheckExcl;
    const bool probe = alive && (excl || ((st.need >> g4) & 15ull) != 0ull);
    uint32_t fb = 0u;
    bool hit = false;
    if (probe) hit = probe_contains(*S, X->list[x], d, hint[x], fb);
    const uint32_t who = __ballot_sync(kFull, probe);
    if (who) {
      fb = __shfl_sync(kFull, fb, __ffs(who) - 1);
      __syncwarp();
      if (lane == 0) hint[x] = fb;
      __syncwarp();
    }
    if (excl) alive = alive && !hit;
    else if (probe) alive = group_step(st, g4, hit);
  }
  return alive && st.need == 0ull;
}

// Candidate buffer full: exact radix select keeps the best k and raises the thresholds. Called by every thread of the
// CTA between two barriers of the rendezvous.
__device__ __noinline__ void stream_compact(StreamCtl* ctl, unsigned long long* cand, uint32_t cap, uint32_t k,
                                            unsigned long long* theta_global) {
  if (min(ctl->ncand, cap) > k) {       // uniform (shared value, read after a barrier)
    const unsigned long long kth = block_select_topk(cand, cap, k, ctl->hist);
    if (threadIdx.x == 0) {
      if (kth > ctl->theta) ctl->theta = kth;
      atomicMax(theta_global, kth);
      ctl->ncand = k;
    }
  } else if (threadIdx.x == 0) {
    ctl->ncand = min(ctl->ncand, cap);
  }
  if (threadIdx.x == 0) ctl->full = 0u;
  __syncthreads();
}

// Every warp passes through here when the buffer overflowed (ctl->full): active warps look at the flag once per step
// and inside an overflowing append; finished warps wait here until the whole CTA is done. Returns true when every
// warp of the CTA has finished its scan.
__device__ __noinline__ bool stream_rendezvous(StreamCtl* ctl, unsigned long long* cand, uint32_t cap, uint32_t k,
                                               unsigned long long* theta_global) {
  __syncthreads();
  if (ctl->full) stream_compact(ctl, cand, cap, k, theta_global);   // uniform after the barrier
  const bool done = *reinterpret_cast<volatile uint32_t*>(&ctl->active) == 0u;
  __syncthreads();
  return done;
}

// Dynamic shared memory: cand[cap] u64 | per warp: T x kStreamTermBytes.
// Terms are in ascending-cost order (the host sorts them); T-1 is the "top" term.
// kAnd: conjunction -- term 0 (the shortest list) is streamed, every other list is probed per candidate and must
// contain it (T = 1 live term, any number of probed terms). Disjunctions stream all T terms until the running
// threshold exceeds the summed block-max bounds of a suffix of them (MaxScore's non-essential lists, P.wand != 0).
// kMode: 0 = disjunction, all T lists live at first; 1 = conjunction (kAnd); 2 = disjunction in LEAD mode: only the
// shortest list is live from the start and every other list is probed -- valid once the query's threshold exceeds the
// summed bounds of those lists, which the CTA checks when it claims its work item (TopkParams::claim).
// kExcl: the queries of the launch exclude terms (TopkParams::excl); with kGroups they also require OR groups
// (TopkParams::excl_grp). Separate instantiations, so that the others carry none of their code or registers.
constexpr int kModeOr = 0, kModeAnd = 1, kModeLead = 2;
template <uint32_t T, int kMode, bool kExcl = false, bool kGroups = false>
__global__ void __launch_bounds__(kTopkThreads, kStreamMinBlocks)
bm25_stream_kernel(const __grid_constant__ TopkParams P) {
  constexpr bool kAnd = kMode == kModeAnd;
  constexpr bool kProbeRest = kMode != kModeOr;        // the query has more terms than live lists
  static_assert(T >= 1 && T <= kStreamMaxTerms, "1..4 live terms");
  static_assert(!kProbeRest || T == 1, "conjunctions and lead mode stream one list");
  static_assert(!kExcl || kMode != kModeLead, "lead mode has no per-doc checks");
  static_assert(!kGroups || (kExcl && kMode == kModeOr), "OR groups run as the disjunction of their terms");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* cand = reinterpret_cast<unsigned long long*>(smem_raw);
  unsigned char* warp_area = reinterpret_cast<unsigned char*>(cand + P.cap);

  __shared__ __align__(16) StreamCtl ctl;
  __shared__ uint64_t s_bar[kTopkWarps][kStreamMaxTerms][2];
  __shared__ QTermDev s_qt[kMaxQueryTerms];
  __shared__ float s_sfx[kMaxQueryTerms + 1];          // s_sfx[e] = sum of the list-wide block-max bounds of terms e .. (inf when unknown)
  __shared__ uint32_t s_hint[kTopkWarps][kMaxQueryTerms];   // per warp and probed term: block where the last probe ended
  __shared__ std::conditional_t<kExcl, std::conditional_t<kGroups, StreamGroups, StreamExcl>, uint32_t> s_x;   // kExcl only

  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  constexpr uint32_t kWarpBytes = T * kStreamTermBytes + (kProbeRest ? 1024u : 0u);
  unsigned char* mine = warp_area + warp * kWarpBytes;
  auto live_docs = [&](uint32_t t) { return reinterpret_cast<uint32_t*>(mine + t * kStreamTermBytes); };
  auto live_scores = [&](uint32_t t) { return reinterpret_cast<float*>(mine + t * kStreamTermBytes + 512u); };
  auto slot_of = [&](uint32_t t, uint32_t s) { return reinterpret_cast<uint4*>(mine + t * kStreamTermBytes + 1024u + s * 512u); };
  auto desc_win = [&](uint32_t t) { return reinterpret_cast<uint4*>(mine + t * kStreamTermBytes + 2048u); };

  const uint4 work = P.work[blockIdx.x];
  const uint32_t q = work.x, chunk = work.z;   // work item = {query, first doc, docs, candidate list}
  const uint32_t t0 = P.qterm_off[q];
  const uint32_t n_terms = kProbeRest ? min(P.qterm_off[q + 1] - t0, kMaxQueryTerms) : T;   // live + probed
  const unsigned long long first64 = work.y;
  const bool chain_empty = first64 > P.seg.n_docs;
  const uint32_t chain_lo = chain_empty ? 1u : uint32_t(first64);
  const uint32_t chain_hi = chain_empty ? 0u : uint32_t(min(static_cast<unsigned long long>(P.seg.n_docs), first64 + chunk - 1ull));
  const uint32_t clen = chain_empty ? 0u : chain_hi - chain_lo + 1u;
  const uint32_t sub = uint32_t((clen + (kTopkWarps - 1ull)) / kTopkWarps);   // 64-bit: clen reaches 2^32 - 2
  const bool warp_empty = clen == 0u || warp * sub >= clen;
  const uint32_t lo_w = warp_empty ? 1u : chain_lo + warp * sub;
  // 64-bit: the last warp's sub-range may end past 2^32 - 1 before it is cut to the chain
  const uint32_t hi_w = warp_empty ? 0u : uint32_t(min(static_cast<unsigned long long>(chain_hi), lo_w + (sub - 1ull)));

  for (uint32_t i = tid; i < P.cap; i += blockDim.x) cand[i] = 0ull;
  if (tid < n_terms) s_qt[tid] = P.qterms[t0 + tid];
  if constexpr (kGroups) {
    const uint32_t x0 = P.excl_off[q];
    const uint32_t n_ex = min(P.excl_off[q + 1] - x0, kMaxCheckLists);
    if (tid < n_ex) { s_x.list[tid] = P.excl[x0 + tid]; s_x.grp[tid] = P.excl_grp[x0 + tid]; }
    for (uint32_t i = tid; i < kTopkWarps * kMaxCheckLists; i += blockDim.x) (&s_x.hint[0][0])[i] = 0u;
    if (tid == 0) {
      s_x.n = n_ex;
      s_x.need = check_group_need(P.excl_grp + x0, n_ex);
      // Pigeonhole lead: a query of one group with m >= 2 ("m of n") matches only docs that one of its n - m + 1
      // shortest lists holds. Only those are streamed; its m - 1 longest lists are probed per candidate from the start.
      const unsigned long long nd = s_x.need.need;
      s_x.e0 = (nd >> 4) == 0ull && nd >= 2ull ? T + 1u - uint32_t(nd) : T;
    }
  } else if constexpr (kExcl) {
    const uint32_t x0 = P.excl_off[q];
    const uint32_t n_ex = min(P.excl_off[q + 1] - x0, kMaxQueryTerms);
    if (tid < n_ex) s_x.list[tid] = P.excl[x0 + tid];
    if (tid < kTopkWarps * kMaxQueryTerms) (&s_x.hint[0][0])[tid] = 0u;
    if (tid == 0) s_x.n = n_ex;
  }
  if (tid == 0) { ctl.ncand = 0u; ctl.matched = 0u; ctl.full = 0u; ctl.active = kTopkWarps; ctl.theta = 0ull; }
  if (lane == 0) {
#pragma unroll
    for (uint32_t t = 0; t < T; ++t) { mbar_init(&s_bar[warp][t][0], 1u); mbar_init(&s_bar[warp][t][1], 1u); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    // suffix sums of the list-wide upper bounds (root block-max pair scored with the query's statistics)
    float acc = 0.f;
    s_sfx[n_terms] = 0.f;
    for (uint32_t t = n_terms; t-- > 0;) {
      const uint32_t rf = s_qt[t].root_freq & 0x7FFFFFFFu;
      const float ub = (P.wand && P.seg.blk_max != nullptr && rf != 0u) ? pair_bound(rf, s_qt[t].root_norm, s_qt[t])
                                                                       : __int_as_float(0x7f800000);
      acc = __fadd_rn(acc, ub);
      s_sfx[t] = acc;
    }
  }
  __syncthreads();
  unsigned long long* const theta_global = P.theta + q;
  if (P.claim != nullptr) {
    // Lead mode is valid only if a doc outside the lead list can no longer qualify: threshold above the summed bounds
    // of all the other lists (strict, with the rounding margin). First arrival decides for both kernels.
    if (tid == 0) {
      const float th = __uint_as_float(uint32_t(*reinterpret_cast<volatile unsigned long long*>(theta_global) >> 32));
      const uint32_t mine_mode = (__fmul_rn(s_sfx[1], 1.000001f) < th) ? 2u : 1u;
      const uint32_t old = atomicCAS(P.claim + blockIdx.x, 0u, mine_mode);
      ctl.full = (old ? old : mine_mode) == (kMode == kModeLead ? 2u : 1u) ? 0u : 0xFFFFFFFFu;
    }
    __syncthreads();
    if (ctl.full == 0xFFFFFFFFu) return;                 // the merge kernel owns this item
  }
  // The buffer is compacted when it holds k + max(k, 256) candidates (rounded up to the CTA size, at most its
  // capacity): for small k the threshold then follows the running k-th best closely instead of waiting for 2048
  // accepted candidates, which is what block-max skipping lives on.
  const uint32_t lim = min(P.cap, (P.k + max(P.k, 256u) + kTopkThreads - 1u) / kTopkThreads * kTopkThreads);
  const bool doc_checks = P.filt.ps.n != 0 || P.seg.deleted != nullptr;   // hybrid filter / DocumentMask on final docs
  // Per-doc list checks (excluded terms, OR groups): a probe per doc costs a few dependent loads. With pruning and a top-k
  // sink only docs whose final score passes the threshold pre-test are probed (late): a rejected doc then never enters the
  // candidate buffer, so the threshold is raised by real results only and pruned == exhaustive, and `matched` counts only
  // docs known to survive (a lower bound). Otherwise every match is probed before it is counted (early: exact count).
  const bool excl_late = kExcl && P.wand != 0 && P.emit_docs == nullptr;
  const bool excl_early = kExcl && !excl_late;

  if (!warp_empty) {
    // ---- per-term stream state: registers (every loop over t is unrolled) ----
    uint32_t cur[T] = {};     // next block to load (index within the term)
    uint32_t widx[T] = {};    // its position in the descriptor window
    uint32_t rr[T] = {};      // blocks consumed so far, mod 4: prefetch slot = rr & 1, barrier parity = rr >> 1
    uint32_t fr[T] = {};      // last doc of the live block (kNoDoc: list exhausted for this warp)
    uint32_t a0[T] = {};      // first pending entry of the live block
    uint32_t nxt[T] = {};     // its doc id (kNoDoc: none) -- lower terms only
    uint32_t matched = 0;     // per lane; summed at the end
    uint32_t skip0 = 0u;      // term 0, bit i: window block i cannot reach the threshold
    uint32_t skip_theta = 0u; // threshold (score bits) the verdicts were made with
    unsigned long long theta = 0ull;
    uint32_t theta_hi = 0u;

    // Appends the lanes' keys (want) to the candidate buffer; on overflow: compaction, then the rest is retried.
    auto append = [&](bool want, unsigned long long key) {
      for (;;) {
        const uint32_t wbal = __ballot_sync(kFull, want);
        if (!wbal) break;
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(&ctl.ncand, uint32_t(__popc(wbal)));
        base = __shfl_sync(kFull, base, 0);
        const uint32_t pos = base + __popc(wbal & ((1u << lane) - 1u));
        if (want && pos < lim) { cand[pos] = key; want = false; }
        if (!__any_sync(kFull, want)) break;
        if (lane == 0) *reinterpret_cast<volatile uint32_t*>(&ctl.full) = 1u;
        stream_rendezvous(&ctl, cand, lim, P.k, theta_global);
        want = want && key > *reinterpret_cast<volatile unsigned long long*>(&ctl.theta);
      }
    };

    // ---- candidates that still have lists to visit (probed terms) wait in a per-warp ring of 128 (doc, partial score);
    // a round looks 32 of them up at once, one per lane ----
    uint32_t E = T;                      // live terms 0 .. E-1 are streamed; terms E .. n_terms-1 are probed
    if constexpr (kGroups) E = s_x.e0;
    uint32_t qhead = 0u, qcount = 0u;
    uint32_t* const qd = kProbeRest ? reinterpret_cast<uint32_t*>(mine + T * kStreamTermBytes) : live_docs(T - 1u);   // plain OR: the ring
    float* const qs = kProbeRest ? reinterpret_cast<float*>(mine + T * kStreamTermBytes + 512u) : live_scores(T - 1u);  // reuses the dropped top list's arrays

    auto doc_ok = [&](uint32_t d) {
      if (P.seg.deleted != nullptr && ((__ldg(P.seg.deleted + (d >> 5)) >> (d & 31u)) & 1u)) return false;   // MaskDocIterator
      return chain_pass(P.filt, d);
    };
    auto test_and_append = [&](bool alive, uint32_t dv, float sv) {
      if (P.emit_docs != nullptr) { stream_emit(P.emit_docs, P.emit_scores, P.emit_count, P.emit_cap, alive, dv, sv); return; }
      bool want = alive && __float_as_uint(sv) >= theta_hi;
      if constexpr (kExcl) {
        if (excl_late && __any_sync(kFull, want)) {
          want = stream_excl_pass(&P.seg, &s_x, want, dv);
          matched += want ? 1u : 0u;
        }
      }
      if (__any_sync(kFull, want)) {
        unsigned long long key = 0ull;
        if (want) { key = make_key(sv, P.seg.ordinal_base + dv); want = key > theta; }
        append(want, key);
      }
    };
    auto probe_round = [&]() {
      const uint32_t n = min(32u, qcount);
      const ProbeResult r = stream_probe_round<kAnd>(&P.seg, s_qt, s_sfx, s_hint[warp], qd, qs, qhead, n, E, n_terms,
                                                     __uint_as_float(theta_hi), P.wand);
      qhead = (qhead + n) & 127u; qcount -= n;
      bool alive = r.alive != 0u;
      if (kAnd) {
        if (doc_checks && alive) alive = doc_ok(r.d);
        if constexpr (kExcl) {
          if (excl_early) alive = stream_excl_pass(&P.seg, &s_x, alive, r.d);
          if (!excl_late) matched += alive ? 1u : 0u;
        } else {
          matched += alive ? 1u : 0u;
        }
      }
      test_and_append(alive, r.d, r.s);
    };
    // Entries that no live list absorbs any more.
    auto finalize_entries = [&](bool alive, uint32_t dv, float sv) {
      if (!kAnd) {
        if (doc_checks && alive) alive = doc_ok(dv);
        if constexpr (kExcl) {
          if (excl_early) alive = stream_excl_pass(&P.seg, &s_x, alive, dv);
          if (!excl_late) matched += alive ? 1u : 0u;
        } else {
          matched += alive ? 1u : 0u;
        }
        if (E == n_terms) { test_and_append(alive, dv, sv); return; }   // nothing left to probe
        // MaxScore: a doc that cannot reach the threshold even with every probed list's bound is dropped unprobed
        alive = alive && !(__fmul_rn(__fadd_rn(sv, s_sfx[E]), 1.000001f) < __uint_as_float(theta_hi));
      }
      const uint32_t bal = __ballot_sync(kFull, alive);
      if (bal) {
        if (alive) {
          const uint32_t pos = (qhead + qcount + __popc(bal & ((1u << lane) - 1u))) & 127u;
          qd[pos] = dv; qs[pos] = sv;
        }
        qcount += __popc(bal);
        __syncwarp();
        while (qcount >= 32u) probe_round();
      }
    };

    // Top live term: entries [a0, ...) with doc <= limit of its live block, lane l holding entries 4l .. 4l+3.
    auto finalize_top = [&](const uint32_t t, uint32_t limit) {
      const uint4 dd = reinterpret_cast<const uint4*>(live_docs(t))[lane];
      const float4 ss = reinterpret_cast<const float4*>(live_scores(t))[lane];
      const uint32_t dv[4] = {dd.x, dd.y, dd.z, dd.w};
      const float sv[4] = {ss.x, ss.y, ss.z, ss.w};
      bool alive[4];
      bool want_any = false;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        alive[j] = dv[j] <= limit && 4u * lane + j >= a0[t];       // pads are kNoDoc > limit
        want_any |= alive[j] && __float_as_uint(sv[j]) >= theta_hi;
      }
      if (!kAnd && E == n_terms && !doc_checks && !kExcl) {
        // common case: nothing to probe, nothing to check -- count, and touch the append path only when some score
        // reaches the threshold
#pragma unroll
        for (int j = 0; j < 4; ++j) matched += alive[j] ? 1u : 0u;
        if (__any_sync(kFull, want_any)) {
#pragma unroll 1
          for (int j = 0; j < 4; ++j) {
            const uint32_t d1 = j == 0 ? dv[0] : j == 1 ? dv[1] : j == 2 ? dv[2] : dv[3];
            const float s1 = j == 0 ? sv[0] : j == 1 ? sv[1] : j == 2 ? sv[2] : sv[3];
            const bool al = j == 0 ? alive[0] : j == 1 ? alive[1] : j == 2 ? alive[2] : alive[3];
            test_and_append(al, d1, s1);
          }
        }
      } else {
#pragma unroll 1
        for (int j = 0; j < 4; ++j) {
          const uint32_t d1 = j == 0 ? dv[0] : j == 1 ? dv[1] : j == 2 ? dv[2] : dv[3];
          const float s1 = j == 0 ? sv[0] : j == 1 ? sv[1] : j == 2 ? sv[2] : sv[3];
          const bool al = j == 0 ? alive[0] : j == 1 ? alive[1] : j == 2 ? alive[2] : alive[3];
          finalize_entries(al, d1, s1);
        }
      }
    };

    // Issues the bulk copy of the block at window position wi of term t into slot `sl`; every block gets exactly one
    // arrival on its slot's barrier, in block order (a block larger than a slot arrives with 0 bytes and is decoded
    // from the arena). The window holds the block's descriptor and its successor's (possibly the table's sentinel).
    auto prefetch = [&](const uint32_t t, uint32_t wi, uint32_t sl) {
      if (lane == 0) {
        const uint4* w = desc_win(t) + wi;
        const uint32_t off = w[0].x;
        uint32_t units = w[1].x - off;
        if (units > kSlotUnits || (t == 0u && ((skip0 >> wi) & 1u))) units = 0u;
        uint64_t* bar = &s_bar[warp][t][sl];
        mbar_arrive_expect_tx(bar, units * 16u);
        if (units) bulk_g2s(slot_of(t, sl), P.seg.arena + off, units * 16u, bar);
      }
    };
    // Single live list (one term, or MaxScore has demoted the others): a block whose block-max bound plus the probed
    // lists' bounds stays below the threshold is never decoded -- SingleWandIterator's block skip
    // (formats/posting/iterator_score.hpp:218-233, 513-632). Judged for the 32 blocks of term 0's descriptor window
    // whenever the window moves or the threshold has risen; the threshold only rises, so a verdict stays valid.
    auto judge_window = [&](uint32_t first) {
      bool skip = false;
      if (!kAnd && P.wand && E == 1u && first + lane < s_qt[0].nblk) {
        const uint2 fn = __ldg(P.seg.blk_max + s_qt[0].blk_begin + first + lane);
        if (fn.x != 0u) {
          const float bound = pair_bound(fn.x, fn.y, s_qt[0]);
          skip = __fmul_rn(__fadd_rn(bound, s_sfx[1]), 1.000001f) < __uint_as_float(theta_hi);
        }
      }
      skip0 = __ballot_sync(kFull, skip);
      skip_theta = theta_hi;
    };
    // Window = descriptors [first, first + 32) of the term (zeros past the sentinel).
    auto load_window = [&](const uint32_t t, uint32_t first) {
      __syncwarp();
      desc_win(t)[lane] = (first + lane <= s_qt[t].nblk) ? __ldg(P.seg.blocks + s_qt[t].blk_begin + first + lane) : make_uint4(0, 0, 0, 0);
      if (t == 0u) judge_window(first);
      __syncwarp();
    };

    // Makes block cur[t] the live block of term t: wait for its payload, decode, gather norms, score, publish.
    auto advance = [&](const uint32_t t, uint32_t plo, bool first_block) {
      uint32_t* ld = live_docs(t);
      float* ls = live_scores(t);
      const uint32_t nblk = s_qt[t].nblk;
      bool have = cur[t] < nblk;
      uint4 d = make_uint4(0, 0, 0, 0);
      if (have) {
        if (widx[t] >= 28u) { load_window(t, cur[t]); widx[t] = 0u; }   // keeps positions widx .. widx + 3 inside the window
        d = desc_win(t)[widx[t]];
        have = d.z < hi_w;                                         // first doc of the block (prev_last + 1) inside the sub-range
      }
      if (!have) {
        reinterpret_cast<uint4*>(ld)[lane] = make_uint4(kNoDoc, kNoDoc, kNoDoc, kNoDoc);
        fr[t] = kNoDoc; a0[t] = 128u; nxt[t] = kNoDoc;
        return;
      }
      const uint32_t units = desc_win(t)[widx[t] + 1u].x - d.x;
      const uint32_t sl = rr[t] & 1u;
      mbar_wait(&s_bar[warp][t][sl], (rr[t] >> 1) & 1u);
      if (t == 0u && ((skip0 >> widx[0]) & 1u)) {
        // block-max says no doc of this block can qualify: consume it without decoding
        __syncwarp();
        if (cur[t] + 2u < nblk) prefetch(t, widx[t] + 2u, sl);
        reinterpret_cast<uint4*>(ld)[lane] = make_uint4(kNoDoc, kNoDoc, kNoDoc, kNoDoc);
        fr[t] = d.y; a0[t] = 128u; nxt[t] = kNoDoc;
        ++cur[t]; ++widx[t]; rr[t] = (rr[t] + 1u) & 3u;
        return;
      }
      const uint32_t len = desc_len(d.w);
      uint32_t doc[4], f[4], nrm[4];
      const uint4* p = slot_of(t, sl);
      if (units <= kSlotUnits) {
        decode_docs_smem(p, d, lane, ld, doc);
      } else {
        decode_block_global(P.seg.arena, d, lane, ld, reinterpret_cast<uint32_t*>(ls));
        const uint4 x = reinterpret_cast<const uint4*>(ld)[lane], y = reinterpret_cast<const uint4*>(ls)[lane];
        doc[0] = x.x; doc[1] = x.y; doc[2] = x.z; doc[3] = x.w;
        f[0] = y.x; f[1] = y.y; f[2] = y.z; f[3] = y.w;
      }
      // norm gathers go out before the rest of the decode: their L2 latency overlaps the frequency unpack + prefetch
      if (len == 128u) {
#pragma unroll
        for (int j = 0; j < 4; ++j) nrm[j] = load_norm(P.seg.norms, P.seg.norm_width, doc[j]);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const bool valid = 4u * lane + j < len;
          if (!valid) doc[j] = kNoDoc;
          nrm[j] = valid ? load_norm(P.seg.norms, P.seg.norm_width, doc[j]) : 1u;
        }
      }
      if (units <= kSlotUnits) decode_freqs_smem(p + desc_fdelta(d.w), d, lane, reinterpret_cast<uint32_t*>(ls), f);
      __syncwarp();                                                // every lane is done with the slot
      if (cur[t] + 2u < nblk) prefetch(t, widx[t] + 2u, sl);
      if (len != 128u) {
#pragma unroll
        for (int j = 0; j < 4; ++j) if (4u * lane + j >= len) f[j] = 1u;
      }
      float s[4];
      const float c0 = s_qt[t].c0, nc = s_qt[t].norm_const, nl = s_qt[t].norm_length;
#pragma unroll
      for (int j = 0; j < 4; ++j) s[j] = bm25_plain(f[j], nrm[j], c0, nc, nl);
      reinterpret_cast<uint4*>(ld)[lane] = make_uint4(doc[0], doc[1], doc[2], doc[3]);
      reinterpret_cast<float4*>(ls)[lane] = make_float4(s[0], s[1], s[2], s[3]);
      a0[t] = 0u;
      if (first_block) {
        // the first block of a warp may hold docs below its sub-range: they are not pending
        a0[t] = __popc(__ballot_sync(kFull, doc[0] <= plo)) + __popc(__ballot_sync(kFull, doc[1] <= plo)) +
                __popc(__ballot_sync(kFull, doc[2] <= plo)) + __popc(__ballot_sync(kFull, doc[3] <= plo));
      }
      if (t + 1u < T) {
        __syncwarp();
        nxt[t] = a0[t] < 128u ? ld[a0[t]] : kNoDoc;
      }
      fr[t] = d.y;
      ++cur[t]; ++widx[t]; rr[t] = (rr[t] + 1u) & 3u;
    };

#pragma unroll
    for (uint32_t t = 0; t < T; ++t) {
      const uint32_t st = warp_first_block(P.seg.blocks + s_qt[t].blk_begin, s_qt[t].nblk, lo_w, lane);
      if (kGroups && t >= E) {
        // probed from the start (pigeonhole lead): never loaded, so nothing to drain; the top list's arrays hold the ring
        if (lane == 0) s_hint[warp][t] = st;
        cur[t] = s_qt[t].nblk; widx[t] = 0u; rr[t] = 0u;
        fr[t] = kNoDoc; nxt[t] = kNoDoc; a0[t] = 128u;
        continue;
      }
      cur[t] = st; widx[t] = 0u; rr[t] = 0u;
      load_window(t, st);
      if (st < s_qt[t].nblk) prefetch(t, 0u, 0u);
      if (st + 1u < s_qt[t].nblk) prefetch(t, 1u, 1u);
      fr[t] = lo_w - 1u;
    }

    if (kProbeRest) {
      for (uint32_t u = 1u; u < n_terms; ++u) {
        const uint32_t hb = warp_first_block(P.seg.blocks + s_qt[u].blk_begin, s_qt[u].nblk, lo_w, lane);
        if (lane == 0) s_hint[warp][u] = hb;
      }
      __syncwarp();
    }

    uint32_t plo = lo_w - 1u;   // docs <= plo are final
    for (uint32_t step = 0;; ++step) {
      // ---- replace the live blocks that ended at plo (first step: every term) ----
#pragma unroll
      for (uint32_t t = 0; t < T; ++t)
        if (fr[t] == plo) advance(t, plo, step == 0u);
      __syncwarp();

      uint32_t phi = hi_w;
#pragma unroll
      for (uint32_t t = 0; t < T; ++t) phi = min(phi, fr[t]);
      theta = *reinterpret_cast<volatile unsigned long long*>(&ctl.theta);
      if ((step & 15u) == 0u) {   // thresholds published by other chains / earlier segments of this query
        const unsigned long long gt = *reinterpret_cast<volatile unsigned long long*>(theta_global);
        if (gt > theta) { theta = gt; if (lane == 0) atomicMax(&ctl.theta, gt); }
      }
      theta_hi = uint32_t(theta >> 32);

      // ---- MaxScore: lists whose summed bounds stay below the threshold stop being streamed (they are probed for the
      // candidates the remaining lists produce). Strict, with a margin for the rounding of the canonical sum. ----
      if (!kAnd && T > 1u && P.wand) {
        while (E > 1u && __fmul_rn(s_sfx[E - 1u], 1.000001f) < __uint_as_float(theta_hi)) {
#pragma unroll
          for (uint32_t t = 1; t < T; ++t)
            if (t + 1u == E) {
              // entries of the departing top list up to plo are complete (they may carry scores folded in from the
              // lower lists): finalise them before its live block is abandoned
              finalize_top(t, plo);
              while (qcount) probe_round();   // ring entries are owed the lists E .. : empty it before E changes
              __syncwarp();
              if (lane == 0) s_hint[warp][t] = cur[t] ? cur[t] - 1u : 0u;
              fr[t] = kNoDoc; nxt[t] = kNoDoc; a0[t] = 128u;
            }
          --E;
          __syncwarp();
        }
      }

      if (!kAnd && P.wand && E == 1u && theta_hi != skip_theta) judge_window(cur[0] - widx[0]);

#pragma unroll
      for (uint32_t t = 0; t < T; ++t) {
        if (t + 1u < E) {
          // ---- lower live terms: pending entries [a0, a1) with doc <= phi, 32 at a time, one entry per lane ----
          if (nxt[t] > phi) continue;                              // uniform: nothing of this term is due
          const uint32_t* ld = live_docs(t);
          const float* ls = live_scores(t);
          const uint4 dd = reinterpret_cast<const uint4*>(ld)[lane];
          const uint32_t a1 = __popc(__ballot_sync(kFull, dd.x <= phi)) + __popc(__ballot_sync(kFull, dd.y <= phi)) +
                              __popc(__ballot_sync(kFull, dd.z <= phi)) + __popc(__ballot_sync(kFull, dd.w <= phi));
          for (uint32_t e0 = a0[t]; e0 < a1; e0 += 32u) {
            const uint32_t e = e0 + lane;
            bool alive = e < a1;
            const uint32_t dv = alive ? ld[e] : kNoDoc;
            const float sv = alive ? ls[e] : 0.f;
#pragma unroll
            for (uint32_t u = t + 1u; u < T; ++u) {
              // absorbed by a later live term's block? (a pending doc can only sit in live blocks: everything a list
              // holds before its live block is <= plo)
              if (fr[u] == kNoDoc) continue;                       // uniform: nothing live in term u (exhausted / probed)
              const uint32_t* a = live_docs(u);
              uint32_t pos = 0;
#pragma unroll
              for (uint32_t stp = 64u; stp; stp >>= 1) pos += (a[pos + stp - 1u] < dv) ? stp : 0u;
              if (alive && a[pos] == dv) {
                float* as = live_scores(u);
                as[pos] = __fadd_rn(sv, as[pos]);                  // unique writer: docs are unique within term t
                alive = false;
              }
            }
            finalize_entries(alive, dv, sv);                       // whatever is still alive is final
          }
          a0[t] = a1;
          __syncwarp();   // folds into later terms are visible before those terms are read
          nxt[t] = a1 < 128u ? ld[a1] : kNoDoc;
        } else if (t + 1u == E) {
          // ---- top live term: its block is finalised as a whole when it retires (every lower term has been folded in
          // up to its last doc by then); lane l holds entries 4l .. 4l+3 ----
          if (fr[t] == phi || phi >= hi_w) { finalize_top(t, phi); a0[t] = 128u; }   // nothing of this block is pending any more
        }
      }
      plo = phi;
      if (phi >= hi_w) break;
      if (*reinterpret_cast<volatile uint32_t*>(&ctl.full)) stream_rendezvous(&ctl, cand, lim, P.k, theta_global);
    }
    while (qcount) probe_round();
    // drain bulk copies that were issued but never consumed (they must not outlive the CTA's shared memory):
    // blocks cur and cur + 1 of every term
#pragma unroll
    for (uint32_t t = 0; t < T; ++t) {
      for (uint32_t i = 0; i < 2u; ++i)
        if (cur[t] + i < s_qt[t].nblk) { const uint32_t r = (rr[t] + i) & 3u; mbar_wait(&s_bar[warp][t][r & 1u], (r >> 1) & 1u); }
    }
    matched = warp_sum(matched);
    if (lane == 0 && matched) atomicAdd(&ctl.matched, matched);
  }
  __syncwarp();
  if (lane == 0) atomicSub(&ctl.active, 1u);
  // finished warps keep serving compactions until every warp of the CTA is done
  while (!stream_rendezvous(&ctl, cand, lim, P.k, theta_global)) {}

  // ---- chain epilogue: best k, sorted descending ----
  stream_compact(&ctl, cand, lim, P.k, theta_global);
  const uint32_t n_out = min(ctl.ncand, P.k);
  uint32_t sort_n = 256u;
  while (sort_n < n_out) sort_n <<= 1;
  block_sort_desc(cand, sort_n);
  const size_t list = work.w;
  unsigned long long* out = P.cand + list * P.cap;
  for (uint32_t i = tid; i < n_out; i += blockDim.x) out[i] = cand[i];
  if (tid == 0) {
    P.cand_n[list] = n_out;
    if (ctl.matched) atomicAdd(P.total + q, static_cast<unsigned long long>(ctl.matched));
  }
}

}  // namespace sdbg
