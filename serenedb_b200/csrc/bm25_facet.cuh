// bm25_facet.cuh -- the sink of the facet pass (`WHERE body @@ '...' GROUP BY col`, count per value): the Count-mode kernel
// (bm25_count.cuh, kFacet) builds each window's exact match bitmap, then reads the key column once for every surviving
// bit and counts it in a per-CTA histogram of `span` u32 bins in dynamic shared memory; at the end of its work item the
// CTA adds the non-zero bins to the query's row of the dense u64 output with one atomic each.
#pragma once

#include "bm25_kernels.cuh"

namespace sdbg {

constexpr uint32_t kFacetMaxSpan = 32768;   // 128 KB of u32 bins: with the kernel's static shared memory, under 227 KB

struct FacetSink {
  const void* values = nullptr;                  // raw key column (packed int64 columns: their raw view)
  const unsigned long long* validity = nullptr;  // null: NOT NULL
  uint64_t rows = 0;                             // docs past row `rows - 1` have a NULL key
  uint32_t type = 0;                             // 0 int64, 2 int32 (sdbg_type)
  uint32_t span = 0;                             // bins: keys key_min .. key_min + span - 1
  long long key_min = 0;
  unsigned long long* counts = nullptr;          // [query][span]
  unsigned long long* nulls = nullptr;           // [query]
  unsigned int* out_of_range = nullptr;          // set to 1 when a counted doc's key lies outside the bins
};

// Groups doc `doc` (row doc - 1) by its key: calls on_null() for a NULL key, else on_bin(bin) with bin = key - key_min
// when the key lies in the bins. Returns true when it does not. The facet pass and the aggregate sink (bm25_agg.cuh)
// both group through it.
template <class OnNull, class OnBin>
__device__ __forceinline__ bool facet_key(const FacetSink& F, uint32_t doc, OnNull on_null, OnBin on_bin) {
  const uint64_t r = uint64_t(doc) - 1ull;
  if (r >= F.rows || (F.validity && !((__ldg(F.validity + (r >> 6)) >> (r & 63ull)) & 1ull))) {
    on_null();
    return false;
  }
  const long long v = F.type == 2u ? static_cast<long long>(__ldg(static_cast<const int*>(F.values) + r))
                                   : __ldg(static_cast<const long long*>(F.values) + r);
  // key_min + span - 1 does not overflow (checked on the host), so the wrapped difference is below span exactly for the
  // keys in range
  const unsigned long long bin = static_cast<unsigned long long>(v) - static_cast<unsigned long long>(F.key_min);
  if (bin >= F.span) return true;
  on_bin(static_cast<uint32_t>(bin));
  return false;
}

// Counts doc `doc` in its key's bin or the NULL counter. Returns true when its key lies outside the bins.
__device__ __forceinline__ bool facet_add(const FacetSink& F, uint32_t doc, uint32_t* bins, uint32_t* nulls) {
  return facet_key(F, doc, [&] { atomicAdd(nulls, 1u); }, [&](uint32_t bin) { atomicAdd(&bins[bin], 1u); });
}

}  // namespace sdbg
