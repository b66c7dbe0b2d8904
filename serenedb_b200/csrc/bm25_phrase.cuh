// bm25_phrase.cuh -- exact phrase queries, conjunctions of phrase clauses and conjunctions of OR groups of phrases
// (sdbg_phrase_*_batch, sdbg_phrase_and_*_batch, sdbg_phrase_groups_*_batch): the positions layout in HBM, the kernels
// that build it at staging, and the per-doc check of a query's alternatives that bm25_count_kernel runs (kPhrase) on the
// docs that survive its candidate scan (the AND, the flat OR or the OR groups of the alternatives' proxy terms), the
// deleted docs, the filter chain and the exclusions: in its own sink (count, top-k), as a stage that narrows the window
// before the facet, aggregate and match-scan sinks, or inside the sorted scan's sink once a doc's key has passed the
// threshold. A single phrase is a query of one positive group of one alternative; a clause conjunction is a query of
// groups of one alternative each.
//
// Positions layout (DESIGN.md §3): per posting block g a 64-bit base pos_base[g] into the u32 arena `pos` (one sentinel
// behind the last block), and at pos[pos_base[g] ..] first the block's len exclusive prefix sums of its frequencies, then
// its positions, posting after posting, each posting's ascending. A probe that knows (block, index in block) finds its
// positions with two 64-bit and two 32-bit loads, without decoding the block's frequencies:
//   first = pos_base[g] + len + pos[pos_base[g] + i], count = next prefix (or the block's end) - pos[pos_base[g] + i].
// 8 B per block, 4 B per posting and 4 B per position.
#pragma once

#include "bm25_kernels.cuh"
#include "bm25_sort.cuh"

namespace sdbg {

constexpr uint32_t kMaxPhraseSlots = 16;

// bm25_count_kernel's phrase sink (kPhrase). cap == 0: count only; else the top-k of the matches by score. With another
// sink (kSort, kFacet, kAgg, kEmit) only the positions, slots and clauses are read.
struct PhraseSink {
  const unsigned long long* pos_base = nullptr;   // per block + sentinel
  const uint32_t* pos = nullptr;
  const uint4* slots = nullptr;                   // this segment's slots: {first BlockDesc, blocks, rel_pos, 0}
  // query q's alternatives clauses[clause_off[q] .. clause_off[q + 1]) in this segment's cost order (ascending smallest
  // docs_count of the alternative's terms, ties in query order, flattened group by group): {first slot, slots, flags
  // (kAlt*), statistics index}
  const uint4* clauses = nullptr;
  const uint32_t* clause_off = nullptr;
  const float4* consts = nullptr;                 // per statistics index {c0, norm_const, norm_length, 0} of a positive alternative
  uint32_t ordinal_base = 0;                      // docs of the earlier segments: key = score bits << 32 | ~(base + doc)
  uint32_t k = 0, cap = 0;                        // cap: buffer slots, a power of two >= 2k (0: count only)
  unsigned long long* thr = nullptr;              // per query: the best known k-th key, seeded with the threshold
  unsigned long long* out = nullptr;              // per work item slot: k keys, best first
  uint32_t* out_n = nullptr;                      // per work item slot: keys written
};

// The positions of doc d in the list of slot `sl`: F.pos[first .. first + n). False when the list does not hold d.
__device__ __forceinline__ bool phrase_positions(const PostingsDev& S, const PhraseSink& F, const uint4& sl, uint32_t d,
                                                 unsigned long long& first, uint32_t& n) {
  const uint4* B = S.blocks + sl.x;
  if (sl.y == 0u) return false;
  const uint32_t l = find_block_from(B, 0u, sl.y, 0u, d);
  if (l >= sl.y) return false;
  const uint4 desc = __ldg(B + l);
  if (d <= desc.z) return false;
  uint32_t idx = 0;
  if (!block_find_doc(S, desc, sl.x + l, d, idx)) return false;
  const unsigned long long base = __ldg(F.pos_base + sl.x + l), end = __ldg(F.pos_base + sl.x + l + 1u);
  const uint32_t len = desc_len(desc.w);
  const uint32_t p0 = __ldg(F.pos + base + idx);
  const uint32_t p1 = idx + 1u < len ? __ldg(F.pos + base + idx + 1u) : uint32_t(end - base - len);
  first = base + len + p0;
  n = p1 - p0;
  return true;
}

// Phrase frequency of doc d: the anchors p (positions of slot 0, whose rel_pos is 0) with p + rel_i among slot i's
// positions for every slot i. One cursor per slot walks its positions forward as the anchors ascend.
__device__ __forceinline__ uint32_t phrase_freq(const PostingsDev& S, const PhraseSink& F, uint32_t s0, uint32_t ns, uint32_t d) {
  unsigned long long at[kMaxPhraseSlots];
  uint32_t cnt[kMaxPhraseSlots], cur[kMaxPhraseSlots], rel[kMaxPhraseSlots];
  for (uint32_t i = 0; i < ns; ++i) {
    const uint4 sl = __ldg(F.slots + s0 + i);
    if (!phrase_positions(S, F, sl, d, at[i], cnt[i])) return 0u;
    rel[i] = sl.z;
    cur[i] = 0u;
  }
  if (ns == 1u) return cnt[0];   // a term: its frequency, without walking its positions
  uint32_t freq = 0;
  for (uint32_t j = 0; j < cnt[0]; ++j) {
    const unsigned long long p = __ldg(F.pos + at[0] + j);
    bool ok = true;
    for (uint32_t i = 1; i < ns && ok; ++i) {
      const unsigned long long want = p + rel[i];
      while (cur[i] < cnt[i] && __ldg(F.pos + at[i] + cur[i]) < want) ++cur[i];
      if (cur[i] == cnt[i]) return freq;   // later anchors want later positions still
      ok = __ldg(F.pos + at[i] + cur[i]) == want;
    }
    freq += ok ? 1u : 0u;
  }
  return freq;
}

// The flags of an alternative table entry: negated; its group (bits 1..4) of the query; the candidate scan guarantees its
// group (check mode need not look); `need` (bits 6..9), the count of matched entries its group must have before this
// entry for the doc to survive this entry's frequency 0: max(0, m - rest), rest the positive entries of the group after
// this one in table order (for m = 1: 1 on the group's last entry, else 0; negated entries 0); the group's minimum match
// count m - 1 (bits 10..13; negated groups 0).
constexpr uint32_t kAltNegated = 1u, kAltGuaranteed = 1u << 5, kAltNeedShift = 6, kAltMinShift = 10;

// Query q's alternative range and its first alternative, read once per window outside the per-doc loops: a single phrase
// (one alternative) then reads no table per doc.
struct PhraseQuery {
  uint32_t c0, c1;
  uint4 first;
};

__device__ __forceinline__ PhraseQuery phrase_query(const PhraseSink& F, uint32_t q) {
  PhraseQuery Q;
  Q.c0 = __ldg(F.clause_off + q);
  Q.c1 = __ldg(F.clause_off + q + 1);
  Q.first = __ldg(F.clauses + Q.c0);
  return Q;
}

// How phrase_clauses treats doc d: check only (entries of a group that the candidate scan guarantees or that an earlier
// entry satisfied are skipped), check and score, or score a doc known to match (negated entries skipped).
enum class PhraseMode { check, score, score_match };

// The check of doc d for query Q, entry after entry in table order. kAlts false, for the candidate AND (every positive
// group one alternative, table flags only kAltNegated): a clause conjunction's walk, dropping d at the first entry that
// fails (positive: frequency 0; negated: frequency > 0); check mode skips the one-slot positive entries, which the AND
// holds. kAlts true, for the flat OR and OR-group candidates, with per positive group a 4-bit count `have` of its
// entries of frequency > 0 so far (16 counters in `cnt`, counted until they reach m <= 15; a group is satisfied when
// have == m): a negated entry with phrase frequency > 0 drops d; a positive entry with frequency > 0 counts for its
// group, and one with frequency 0 drops d when have < need, i.e. the group's count plus the entries after this one cannot
// reach m (for m = 1: the last entry of an unsatisfied group). A positive group's last entry has need m, so a doc that
// reaches the table's end has every positive group satisfied (or guaranteed): it matches, and no state of the query's
// groups needs to stay live. Scoring modes evaluate every positive entry: s = the
// sum of bm25(frequency, norm(d)) of those with frequency > 0, with their statistics, in table order from 0 (a one-slot
// entry's frequency is its term's position count). The kAlts walk scores a conjunction's table too, so phrase_score_kernel takes every shape.
template <bool kAlts>
__device__ __forceinline__ bool phrase_clauses(const PostingsDev& S, const PhraseSink& F, const PhraseQuery& Q, uint32_t d,
                                               PhraseMode mode, float& s) {
  s = 0.f;
  if constexpr (!kAlts) {
    uint4 cl = Q.first;
    for (uint32_t c = Q.c0;;) {
      const bool skip = cl.z ? mode == PhraseMode::score_match : mode == PhraseMode::check && cl.y == 1u;
      if (!skip) {
        const uint32_t f = phrase_freq(S, F, cl.x, cl.y, d);
        if ((f != 0u) == (cl.z != 0u)) return false;
        if (mode != PhraseMode::check && !cl.z) {
          const float4 k = __ldg(F.consts + cl.w);
          s = __fadd_rn(s, bm25(f, load_norm(S.norms, S.norm_width, d), k.x, k.y, k.z));
        }
      }
      if (++c >= Q.c1) return true;
      cl = __ldg(F.clauses + c);
    }
  } else {
    uint4 cl = __ldg(F.clauses + Q.c0);   // Q.first is not kept live across the window: the candidate scan's state is
    unsigned long long cnt = 0ull;
    for (uint32_t c = Q.c0;;) {
      const bool neg = cl.z & kAltNegated;
      const uint32_t sh = 4u * ((cl.z >> 1) & 15u), have = uint32_t(cnt >> sh) & 15u;
      const bool open = have <= ((cl.z >> kAltMinShift) & 15u);   // have < m
      const bool skip = neg ? mode == PhraseMode::score_match
                            : mode == PhraseMode::check && ((cl.z & kAltGuaranteed) || !open);
      if (!skip) {
        const uint32_t f = phrase_freq(S, F, cl.x, cl.y, d);
        if (f != 0u ? neg : have < ((cl.z >> kAltNeedShift) & 15u)) return false;
        if (f != 0u) {
          cnt += static_cast<unsigned long long>(open) << sh;
          if (mode != PhraseMode::check) {
            const float4 k = __ldg(F.consts + cl.w);
            s = __fadd_rn(s, bm25(f, load_norm(S.norms, S.norm_width, d), k.x, k.y, k.z));
          }
        }
      }
      if (++c >= Q.c1) return true;
      cl = __ldg(F.clauses + c);
    }
  }
}

// The top-k key of a match of score s: score bits, then ~ordinal (ties: segment asc, doc asc), as bm25_topk's keys.
__device__ __forceinline__ unsigned long long phrase_key(const PhraseSink& F, uint32_t d, float s) {
  return (static_cast<unsigned long long>(__float_as_uint(s)) << 32) | (~(F.ordinal_base + d) & 0xFFFFFFFFull);
}

// ---- staging ----
// One warp per block: the sum of its frequencies.
__global__ void __launch_bounds__(256) phrase_freq_sums_kernel(const uint4* __restrict__ arena, const uint4* __restrict__ blocks,
                                                               uint64_t n_blocks, unsigned long long* __restrict__ sums) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint64_t g = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (g >= n_blocks) return;
  const uint4 d = __ldg(blocks + g);
  uint32_t f[4];
  decode_freqs(arena, d, lane, f);
  const uint32_t len = desc_len(d.w);
  unsigned long long s = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) s += 4u * lane + j < len ? f[j] : 0u;
  s = warp_sum64(s);
  if (lane == 0) sums[g] = s;
}

// One warp per block: writes the block's frequency prefixes and copies its positions (src[src_off[g] ..], in posting
// order) behind them; sets *bad when a posting's positions do not ascend strictly.
__global__ void __launch_bounds__(256) phrase_fill_kernel(const uint4* __restrict__ arena, const uint4* __restrict__ blocks,
                                                          uint64_t n_blocks, const unsigned long long* __restrict__ pos_base,
                                                          const unsigned long long* __restrict__ src_off,
                                                          const uint32_t* __restrict__ src, uint32_t* __restrict__ pos,
                                                          unsigned int* __restrict__ bad) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint64_t g = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (g >= n_blocks) return;
  const uint4 d = __ldg(blocks + g);
  uint32_t f[4];
  decode_freqs(arena, d, lane, f);
  const uint32_t len = desc_len(d.w);
#pragma unroll
  for (int j = 0; j < 4; ++j) if (4u * lane + j >= len) f[j] = 0u;
  const uint32_t mine = f[0] + f[1] + f[2] + f[3];
  uint32_t pre = warp_incl_scan(mine, lane) - mine;
  const unsigned long long base = pos_base[g], from = src_off[g];
  const unsigned long long total = pos_base[g + 1] - base - len;
  for (unsigned long long i = lane; i < total; i += 32u) pos[base + len + i] = src[from + i];
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (4u * lane + j < len) {
      pos[base + 4u * lane + j] = pre;
      for (uint32_t x = 1; x < f[j]; ++x) ok &= src[from + pre + x] > src[from + pre + x - 1u];
    }
    pre += f[j];
  }
  if (!ok) atomicExch(bad, 1u);
}

// ---- top-k merge ----
// One CTA per query: the k best of its work items' keys (slots[slot_off[q] .. slot_off[q + 1])), best first, into
// out[q][k] with n_out[q]. The keys are unique, so the buffer's lo words stay 0 (merge_item_keys, bm25_sort.cuh).
__global__ void __launch_bounds__(256) phrase_merge_kernel(const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ keys_n,
                                                           const uint32_t* __restrict__ slot_off, const uint32_t* __restrict__ slots,
                                                           uint32_t k, uint32_t cap, unsigned long long* __restrict__ out,
                                                           uint32_t* __restrict__ n_out) {
  extern __shared__ unsigned long long sm_keys[];
  __shared__ uint32_t s_fill;
  unsigned long long* hi = sm_keys;
  unsigned long long* lo = sm_keys + cap;
  const uint32_t q = blockIdx.x;
  merge_item_keys(hi, lo, cap, k, q, slot_off, slots, keys_n, &s_fill,
                  [&](uint32_t slot, uint32_t i) { return make_ulonglong2(keys[size_t(slot) * k + i], 0ull); });
  const uint32_t n = s_fill;
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) out[size_t(q) * k + i] = hi[i];
  if (threadIdx.x == 0) n_out[q] = n;
}

}  // namespace sdbg
