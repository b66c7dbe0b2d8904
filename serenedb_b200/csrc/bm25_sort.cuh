// bm25_sort.cuh -- the sink of the sorted scan (`WHERE body @@ '...' ORDER BY col LIMIT k`): the Count-mode kernel
// (bm25_count.cuh, kSort) builds each window's exact match bitmap, then reads the sort column for every surviving bit
// and keeps the k best in a per-CTA buffer of wide keys; sort_merge_kernel merges the work items' survivors per query.
//
// Key (larger = better, unique): hi = class (1 bit) | vkey >> 1, lo = (vkey & 1) << 63 | ~ordinal (32 bits).
//   class   1 for the group that sorts first: the values under NULLS LAST, the NULLs under NULLS FIRST.
//   vkey    the value mapped onto uint64 in ascending order (int64 / int32 with the sign bit flipped; float64 with -0.0
//           as +0.0, every NaN as the one canonical NaN above +inf, then the usual sign-magnitude flip), negated for ASC.
//           0 for a NULL, so all NULLs tie.
//   ordinal ordinal_base (docs of the earlier segments) + doc - 1: ties go to (segment asc, doc asc). Ordinals stay below
//           2^32 - 1, so a real key has lo != 0 and (0, 0) marks an empty slot.
// The per-query threshold word holds the hi of the best known k-th key: a match whose hi is below it cannot be in the
// result; an equal hi can (ties are decided by lo), so it enters the buffer.
#pragma once

#include "bm25_kernels.cuh"
#include "column_kernels.cuh"

namespace sdbg {

constexpr uint32_t kSortMaxK = 4096;   // the candidate buffer holds 2 * next_pow2(k) keys of 16 B: 128 KB at this k

struct SortSink {
  const void* values = nullptr;                  // raw sort column (packed int64 columns: their raw view)
  const unsigned long long* validity = nullptr;  // null: NOT NULL
  uint64_t rows = 0;                             // docs past row `rows - 1` sort as NULL
  const long long* zone = nullptr;               // {min, max} per kZoneRows rows (predicate key space); null: no zone pruning
  uint32_t n_zones = 0;
  uint32_t type = 0;                             // 0 int64, 1 float64, 2 int32 (sdbg_type)
  uint32_t desc = 0, nulls_first = 0;
  uint32_t ordinal_base = 0;
  uint32_t k = 0, cap = 0;                       // cap: buffer slots, a power of two >= 2k
  unsigned long long* thr = nullptr;             // per query: hi of the best known k-th key; null: no pruning (level 0)
  ulonglong2* out = nullptr;                     // per work item slot: k keys {hi, lo}, best first
  uint32_t* out_n = nullptr;                     // per work item slot: keys written
  unsigned long long* stats = nullptr;           // {windows judged, windows skipped} by the zonemap
};

// Value (raw bits, int32 sign-extended) -> ascending uint64 order.
__host__ __device__ __forceinline__ unsigned long long sort_order(unsigned long long bits, uint32_t type) {
  constexpr unsigned long long kSign = 0x8000000000000000ull;
  if (type != 1u) return bits ^ kSign;
  if ((bits & ~kSign) > 0x7FF0000000000000ull) bits = 0x7FF8000000000000ull;   // any NaN: the canonical one, above +inf
  else if (bits == kSign) bits = 0ull;                                         // -0.0 == +0.0
  return (bits & kSign) ? ~bits : (bits | kSign);
}

__host__ __device__ __forceinline__ unsigned long long sort_hi(const SortSink& S, unsigned long long order) {
  const unsigned long long vkey = S.desc ? order : ~order;
  return (static_cast<unsigned long long>(S.nulls_first ^ 1u) << 63) | (vkey >> 1);
}

__host__ __device__ __forceinline__ unsigned long long sort_null_hi(const SortSink& S) {
  return static_cast<unsigned long long>(S.nulls_first) << 63;
}

// The key of doc `doc` (row doc - 1).
__device__ __forceinline__ ulonglong2 sort_key(const SortSink& S, uint32_t doc) {
  const uint64_t r = uint64_t(doc) - 1ull;
  const unsigned long long ord = ~static_cast<unsigned long long>(S.ordinal_base + doc - 1u) & 0xFFFFFFFFull;
  const bool valid = r < S.rows && (S.validity == nullptr || ((__ldg(S.validity + (r >> 6)) >> (r & 63ull)) & 1ull));
  if (!valid) return make_ulonglong2(sort_null_hi(S), ord);
  const unsigned long long bits = S.type == 2u ? static_cast<unsigned long long>(static_cast<long long>(__ldg(static_cast<const int*>(S.values) + r)))
                                               : __ldg(static_cast<const unsigned long long*>(S.values) + r);
  const unsigned long long vkey = S.desc ? sort_order(bits, S.type) : ~sort_order(bits, S.type);
  return make_ulonglong2(sort_hi(S, sort_order(bits, S.type)), ((vkey & 1ull) << 63) | ord);
}

// Upper bound of the hi of any key in zone z (the host plans with it too) (rows [z * kZoneRows, (z + 1) * kZoneRows)). Zones past the column, and
// the last zone when it is partial, hold docs that sort as NULL.
__host__ __device__ __forceinline__ unsigned long long sort_zone_bound(const SortSink& S, uint32_t z) {
  if (z >= S.n_zones) return sort_null_hi(S);
  const long long mn = S.zone[2 * z], mx = S.zone[2 * z + 1];   // also run on the host, over a copy
  unsigned long long lo_o, hi_o;   // ascending order of the zone's smallest / largest value
  if (S.type == 1u) {
    // Doubles are zoned through fkey(): a NaN with the sign bit set lies below fkey(-inf), one without above fkey(+inf),
    // and -0.0 just below +0.0. The sort ranks every NaN above +inf.
    const long long ninf = fkey(static_cast<long long>(0xFFF0000000000000ull)), pinf = 0x7FF0000000000000ll;
    const bool neg_nan = mn < ninf;
    lo_o = sort_order(neg_nan ? 0xFFF0000000000000ull : static_cast<unsigned long long>(fkey(mn)), 1u);
    hi_o = (neg_nan || mx > pinf) ? sort_order(0x7FF8000000000000ull, 1u) : sort_order(static_cast<unsigned long long>(fkey(mx)), 1u);
  } else {
    lo_o = sort_order(static_cast<unsigned long long>(mn), 0u);
    hi_o = sort_order(static_cast<unsigned long long>(mx), 0u);
  }
  unsigned long long b = sort_hi(S, S.desc ? hi_o : lo_o);
  if (uint64_t(z + 1u) * kZoneRows > S.rows && sort_null_hi(S) > b) b = sort_null_hi(S);
  return b;
}

__device__ __forceinline__ bool key_less(unsigned long long ah, unsigned long long al, unsigned long long bh, unsigned long long bl) {
  return ah < bh || (ah == bh && al < bl);
}

// Sorts n (a power of two) keys best first. Whole CTA; starts and ends with a barrier.
__device__ __forceinline__ void sort_keys_desc(unsigned long long* hi, unsigned long long* lo, uint32_t n) {
  __syncthreads();
  for (uint32_t k = 2; k <= n; k <<= 1) {
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
      for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t p = i ^ j;
        if (p <= i) continue;
        const unsigned long long ah = hi[i], al = lo[i], bh = hi[p], bl = lo[p];
        const bool first_desc = (i & k) == 0;   // this run ends up best first
        if (first_desc == key_less(ah, al, bh, bl)) { hi[i] = bh; lo[i] = bl; hi[p] = ah; lo[p] = al; }
      }
      __syncthreads();
    }
  }
}

// Keeps the k best of the first min(*fill, cap) keys: sorts, empties slots k.., sets *fill to the keys kept and returns
// the hi of the k-th key (0 when fewer than k are held). Whole CTA.
__device__ __forceinline__ unsigned long long sort_select(unsigned long long* hi, unsigned long long* lo, uint32_t cap, uint32_t k,
                                                          uint32_t* fill) {
  sort_keys_desc(hi, lo, cap);
  const uint32_t held = min(*fill, cap);
  for (uint32_t i = k + threadIdx.x; i < cap; i += blockDim.x) { hi[i] = 0ull; lo[i] = 0ull; }
  const unsigned long long kth = held >= k ? hi[k - 1] : 0ull;
  __syncthreads();
  if (threadIdx.x == 0) *fill = min(held, k);
  __syncthreads();
  return kth;
}

// Gathers the keys of query q's work items (slots[slot_off[q] .. slot_off[q + 1]), keys_n[slot] keys each, load(slot, i)
// the i-th as {hi, lo}) into hi / lo and keeps the k best (sort_select); *fill ends at their number. Whole CTA; the
// buffer of cap >= 2k slots is zeroed first.
template <class Load>
__device__ __forceinline__ void merge_item_keys(unsigned long long* hi, unsigned long long* lo, uint32_t cap, uint32_t k, uint32_t q,
                                                const uint32_t* slot_off, const uint32_t* slots, const uint32_t* keys_n,
                                                uint32_t* fill, Load load) {
  for (uint32_t i = threadIdx.x; i < cap; i += blockDim.x) { hi[i] = 0ull; lo[i] = 0ull; }
  if (threadIdx.x == 0) *fill = 0u;
  __syncthreads();
  for (uint32_t si = slot_off[q]; si < slot_off[q + 1]; ++si) {
    const uint32_t slot = slots[si], n = keys_n[slot];
    if (*fill + n > cap) sort_select(hi, lo, cap, k, fill);   // n <= k and cap >= 2k: room after a select
    const uint32_t f = *fill;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
      const ulonglong2 v = load(slot, i);
      hi[f + i] = v.x; lo[f + i] = v.y;
    }
    __syncthreads();
    if (threadIdx.x == 0) *fill = f + n;
    __syncthreads();
  }
  sort_select(hi, lo, cap, k, fill);
}

// One row of sdbg_sort_hit.
struct SortHitDev {
  long long value;
  uint32_t doc, seg;
  uint8_t is_null, pad[7];
};

struct SortSegDev {   // per segment: the sort column and the segment's first ordinal
  const void* values;
  const unsigned long long* validity;
  uint64_t rows;
  uint32_t ordinal_base, pad;
};

struct SortMergeParams {
  const ulonglong2* keys;       // per work item slot: k keys
  const uint32_t* keys_n;
  const uint32_t* slot_off;     // query q's slots: slots[slot_off[q] .. slot_off[q + 1])
  const uint32_t* slots;
  const SortSegDev* segs;
  uint32_t n_segs, type, nulls_first, k, cap;
  SortHitDev* out;              // [Q][k]
  uint32_t* n_out;
};

// One CTA per query: merges the survivors of its work items into the k best, in order, and reads each hit's stored value.
__global__ void __launch_bounds__(256) sort_merge_kernel(SortMergeParams P) {
  extern __shared__ unsigned long long sm_keys[];
  __shared__ uint32_t s_fill;
  unsigned long long* hi = sm_keys;
  unsigned long long* lo = sm_keys + P.cap;
  const uint32_t q = blockIdx.x, k = P.k, cap = P.cap;
  merge_item_keys(hi, lo, cap, k, q, P.slot_off, P.slots, P.keys_n, &s_fill,
                  [&](uint32_t slot, uint32_t i) { return P.keys[size_t(slot) * k + i]; });
  const uint32_t n = s_fill;
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    const uint32_t ord = ~static_cast<uint32_t>(lo[i]);
    uint32_t s = 0;
    while (s + 1u < P.n_segs && P.segs[s + 1u].ordinal_base <= ord) ++s;
    const SortSegDev& G = P.segs[s];
    SortHitDev h{};
    h.doc = ord - G.ordinal_base + 1u;
    h.seg = s;
    h.is_null = static_cast<uint8_t>((hi[i] >> 63) == P.nulls_first);
    if (!h.is_null) {
      const uint64_t r = uint64_t(h.doc) - 1ull;
      h.value = P.type == 2u ? static_cast<long long>(__ldg(static_cast<const int*>(G.values) + r))
                             : __ldg(static_cast<const long long*>(G.values) + r);
    }
    P.out[size_t(q) * k + i] = h;
  }
  if (threadIdx.x == 0) P.n_out[q] = n;
}

// ---- the sorted scan across ranks ----
// A rank's buffer: SortDistHeader, then its per-query row counts (u64 [nq]), then rows [nq][k], best first. A row is the
// key above with the rank folded into lo bits 32..62 as ~rank (ties go to the lower rank, then the lower ordinal), and
// the stored value: the key canonicalises -0.0 and NaN, so the value cannot be rebuilt from it.
struct SortDistHeader {
  unsigned long long type, desc, nulls_first, k, nq;   // the sort column's sdbg_type (UINT64_MAX: not found), the call's order
  unsigned long long failed;                           // non-zero: this rank's local pass failed
  unsigned long long pad[2];
};
static_assert(sizeof(SortDistHeader) == 64, "the rows stay 16-byte aligned");

struct SortDistRow { unsigned long long hi, lo, value; };

__host__ __device__ __forceinline__ unsigned long long sort_rank_bits(uint32_t rank) {
  return static_cast<unsigned long long>(~rank & 0x7FFFFFFFu) << 32;
}

// One CTA per query: the local result's hits (sort_merge_kernel's output) -> this rank's rows.
__global__ void __launch_bounds__(256) sort_dist_rows_kernel(const SortHitDev* __restrict__ hits, const uint32_t* __restrict__ n_out,
                                                             const SortSegDev* __restrict__ segs, uint32_t k, uint32_t type,
                                                             uint32_t desc, uint32_t nulls_first, uint32_t rank,
                                                             unsigned long long* __restrict__ rows_n, SortDistRow* __restrict__ rows) {
  const uint32_t q = blockIdx.x, n = n_out[q];
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    const SortHitDev h = hits[size_t(q) * k + i];
    const uint32_t ord = segs[h.seg].ordinal_base + h.doc - 1u;
    const unsigned long long rlo = sort_rank_bits(rank) | (~static_cast<unsigned long long>(ord) & 0xFFFFFFFFull);
    SortDistRow w;
    if (h.is_null) {
      w = {static_cast<unsigned long long>(nulls_first) << 63, rlo, 0ull};
    } else {
      const unsigned long long o = sort_order(static_cast<unsigned long long>(h.value), type), vkey = desc ? o : ~o;
      w = {(static_cast<unsigned long long>(nulls_first ^ 1u) << 63) | (vkey >> 1), ((vkey & 1ull) << 63) | rlo,
           static_cast<unsigned long long>(h.value)};
    }
    rows[size_t(q) * k + i] = w;
  }
  if (threadIdx.x == 0) rows_n[q] = n;
}

// One CTA per query: the k best of n_ranks ranks' rows (buffers of rank_bytes back to back), in order, as sdbg_sort_hit
// (doc = ordinal within the rank + 1, seg = rank). Each selected key's value is found by a binary search of its rank's
// list, which is sorted best first with unique keys. Block 0 also checks the headers: status = {headers disagree, some
// rank failed}.
__global__ void __launch_bounds__(256) sort_merge_gathered_kernel(const char* __restrict__ all, size_t rank_bytes, uint32_t n_ranks,
                                                                  uint32_t nq, uint32_t k, uint32_t cap,
                                                                  unsigned long long* __restrict__ status, SortHitDev* __restrict__ out,
                                                                  uint32_t* __restrict__ n_out) {
  extern __shared__ unsigned long long sm_keys[];
  __shared__ uint32_t s_fill;
  unsigned long long* hi = sm_keys;
  unsigned long long* lo = sm_keys + cap;
  const uint32_t q = blockIdx.x;
  const auto* h0 = reinterpret_cast<const SortDistHeader*>(all);
  if (q == 0 && threadIdx.x == 0) {
    unsigned long long bad = 0, failed = 0;
    for (uint32_t r = 0; r < n_ranks; ++r) {
      const auto* h = reinterpret_cast<const SortDistHeader*>(all + r * rank_bytes);
      bad |= h->type != h0->type || h->desc != h0->desc || h->nulls_first != h0->nulls_first || h->k != k || h->nq != nq;
      failed |= h->failed;
    }
    status[0] = bad; status[1] = failed;
  }
  const size_t rows_pos = sizeof(SortDistHeader) + size_t(nq) * 8;
  for (uint32_t i = threadIdx.x; i < cap; i += blockDim.x) { hi[i] = 0ull; lo[i] = 0ull; }
  if (threadIdx.x == 0) s_fill = 0u;
  __syncthreads();
  for (uint32_t r = 0; r < n_ranks; ++r) {
    const char* b = all + r * rank_bytes;
    const uint32_t n = static_cast<uint32_t>(min(reinterpret_cast<const unsigned long long*>(b + sizeof(SortDistHeader))[q],
                                                 static_cast<unsigned long long>(k)));
    if (s_fill + n > cap) sort_select(hi, lo, cap, k, &s_fill);   // n <= k and cap >= 2k: room after a select
    const uint32_t f = s_fill;
    const auto* rows = reinterpret_cast<const SortDistRow*>(b + rows_pos) + size_t(q) * k;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) { hi[f + i] = rows[i].hi; lo[f + i] = rows[i].lo; }
    __syncthreads();
    if (threadIdx.x == 0) s_fill = f + n;
    __syncthreads();
  }
  sort_select(hi, lo, cap, k, &s_fill);
  const uint32_t n = s_fill;
  const uint32_t nulls_first = static_cast<uint32_t>(h0->nulls_first);
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    const unsigned long long kh = hi[i], kl = lo[i];
    const uint32_t r = ~static_cast<uint32_t>(kl >> 32) & 0x7FFFFFFFu;
    SortHitDev h{};
    h.doc = ~static_cast<uint32_t>(kl) + 1u;
    h.seg = r;
    h.is_null = static_cast<uint8_t>((kh >> 63) == nulls_first);
    if (!h.is_null && r < n_ranks) {
      const char* b = all + r * rank_bytes;
      const auto* rows = reinterpret_cast<const SortDistRow*>(b + rows_pos) + size_t(q) * k;
      const uint32_t cnt = static_cast<uint32_t>(min(reinterpret_cast<const unsigned long long*>(b + sizeof(SortDistHeader))[q],
                                                     static_cast<unsigned long long>(k)));
      uint32_t a = 0, e = cnt;
      while (a < e) {   // first row not better than the key: the key itself
        const uint32_t m = (a + e) >> 1;
        if (key_less(kh, kl, rows[m].hi, rows[m].lo)) a = m + 1u; else e = m;
      }
      if (a < cnt) h.value = static_cast<long long>(rows[a].value);
    }
    out[size_t(q) * k + i] = h;
  }
  if (threadIdx.x == 0) n_out[q] = n;
}

}  // namespace sdbg
