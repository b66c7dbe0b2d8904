// bm25_agg.cuh -- the sink of the aggregate pass (`SELECT col, count(*), sum(v), avg(v), min(v), max(v) ... WHERE body @@
// '...' GROUP BY col`, or the same without GROUP BY): the Count-mode kernel (bm25_count.cuh, kAgg) builds each window's
// exact match bitmap, then for every surviving bit finds the doc's group through the facet pass's facet_key and reads its
// value once.
//
// Per CTA, one 40-byte cell per key, plus one for the NULL key, in dynamic shared memory (AggSmemCell). Integer sums are
// kept in two 64-bit limbs, the sum of the low 32 bits and the signed sum of v >> 32: a work item spans fewer than 2^32
// docs, so neither limb can overflow before the flush. A float64 column keeps one double instead. MIN and MAX are kept
// as maxima of ~sort_order(v) and sort_order(v) (bm25_sort.cuh), so every cell, in shared memory and in HBM, starts as
// zeros. Ungrouped (no key column) each thread accumulates in registers and merges into cell 0 once per item.
// At the end of its item the CTA adds every non-empty cell to the query's output cell (AggCell): 64-bit atomics, the
// 128-bit sum with an exact carry, atomicMax for the extremes, so the result does not depend on the order of the atomics
// (the float64 sum excepted).
#pragma once

#include "bm25_facet.cuh"
#include "bm25_sort.cuh"

namespace sdbg {

constexpr uint32_t kAggMaxSpan = 4096;   // 4097 cells of 40 B: 160 KB, with 32 KB of counter planes and the kernel's
                                         // 17.4 KB of static shared memory under 227 KB

struct AggSmemCell {           // one group of one work item
  uint32_t n, nv;              // COUNT(*), COUNT(value)
  unsigned long long lo;       // integer: sum of (v & 0xFFFFFFFF); float64: the double sum's bits
  unsigned long long hi;       // integer: sum of (v >> 32), two's complement
  unsigned long long nmin;     // max of ~sort_order(v): the MIN
  unsigned long long max;      // max of sort_order(v)
};
static_assert(sizeof(AggSmemCell) == 40, "40 B per key");

struct AggCell {               // one group of one query, summed over items and segments
  unsigned long long count, count_value;
  unsigned long long sum_lo, sum_hi;   // integer: the 128-bit two's-complement sum; float64: sum_lo holds the double
  unsigned long long nmin, max;
};

struct AggSink {
  FacetSink key;                                 // the key column and its bins (key.values null: one group, cell 0)
  const void* values = nullptr;                  // raw value column (packed int64 columns: their raw view)
  const unsigned long long* validity = nullptr;  // null: NOT NULL
  uint64_t rows = 0;                             // docs past row `rows - 1` have a NULL value
  uint32_t type = 0;                             // 0 int64, 1 float64, 2 int32 (sdbg_type)
  AggCell* cells = nullptr;                      // [query][key.span]
  AggCell* nulls = nullptr;                      // [query]: the NULL key's group
  unsigned int* out_of_range = nullptr;          // set to 1 when a matching doc's key lies outside the bins
};

// Dynamic shared memory of the cells for `span` keys and the NULL key, rounded up to 16 B.
__host__ __device__ __forceinline__ uint32_t agg_cells_bytes(uint32_t span) {
  return ((span + 1u) * uint32_t(sizeof(AggSmemCell)) + 15u) & ~15u;
}

// Inverse of sort_order: the value's bits (a zero comes back as +0.0, a NaN as 0x7FF8000000000000).
__host__ __device__ __forceinline__ unsigned long long sort_order_value(unsigned long long order, uint32_t type) {
  constexpr unsigned long long kSign = 0x8000000000000000ull;
  if (type != 1u) return order ^ kSign;
  return (order & kSign) ? order ^ kSign : ~order;
}

// The one-doc cell of doc `doc` (row doc - 1).
__device__ __forceinline__ AggSmemCell agg_one(const AggSink& S, uint32_t doc) {
  AggSmemCell c{1u, 0u, 0ull, 0ull, 0ull, 0ull};
  const uint64_t r = uint64_t(doc) - 1ull;
  if (r >= S.rows || (S.validity && !((__ldg(S.validity + (r >> 6)) >> (r & 63ull)) & 1ull))) return c;
  const unsigned long long bits = S.type == 2u ? static_cast<unsigned long long>(static_cast<long long>(__ldg(static_cast<const int*>(S.values) + r)))
                                               : __ldg(static_cast<const unsigned long long*>(S.values) + r);
  const unsigned long long o = sort_order(bits, S.type);
  c.nv = 1u;
  c.lo = S.type == 1u ? bits : bits & 0xFFFFFFFFull;
  c.hi = S.type == 1u ? 0ull : static_cast<unsigned long long>(static_cast<long long>(bits) >> 32);
  c.nmin = ~o;
  c.max = o;
  return c;
}

// a += b, in registers.
__device__ __forceinline__ void agg_accum(AggSmemCell& a, const AggSmemCell& b, uint32_t type) {
  a.n += b.n;
  a.nv += b.nv;
  if (type == 1u) a.lo = __double_as_longlong(__longlong_as_double(a.lo) + __longlong_as_double(b.lo));
  else { a.lo += b.lo; a.hi += b.hi; }
  a.nmin = a.nmin > b.nmin ? a.nmin : b.nmin;
  a.max = a.max > b.max ? a.max : b.max;
}

// *a += b, with shared-memory atomics.
__device__ __forceinline__ void agg_merge(AggSmemCell* a, const AggSmemCell& b, uint32_t type) {
  if (!b.n) return;
  atomicAdd(&a->n, b.n);
  if (!b.nv) return;
  atomicAdd(&a->nv, b.nv);
  if (type == 1u) atomicAdd(reinterpret_cast<double*>(&a->lo), __longlong_as_double(b.lo));
  else { atomicAdd(&a->lo, b.lo); atomicAdd(&a->hi, b.hi); }
  atomicMax(&a->nmin, b.nmin);
  atomicMax(&a->max, b.max);
}

// Counts doc `doc` in its group: ungrouped in the thread's register cell `mine`, else in its key's shared cell (cell span
// for the NULL key). Returns true when its key lies outside the bins.
__device__ __forceinline__ bool agg_add(const AggSink& S, uint32_t doc, AggSmemCell* cells, AggSmemCell& mine) {
  if (!S.key.values) {
    agg_accum(mine, agg_one(S, doc), S.type);
    return false;
  }
  return facet_key(S.key, doc, [&] { agg_merge(&cells[S.key.span], agg_one(S, doc), S.type); },
                   [&](uint32_t bin) { agg_merge(&cells[bin], agg_one(S, doc), S.type); });
}

// *g += c over global memory. The integer sum c.lo + c.hi * 2^32 is added as a 128-bit number: the carry out of the low
// word is taken from the value the atomic returns, so the total is exact whatever the order of the flushes.
__device__ __forceinline__ void agg_flush(AggCell* g, const AggSmemCell& c, uint32_t type) {
  atomicAdd(&g->count, static_cast<unsigned long long>(c.n));
  if (!c.nv) return;
  atomicAdd(&g->count_value, static_cast<unsigned long long>(c.nv));
  if (type == 1u) {
    atomicAdd(reinterpret_cast<double*>(&g->sum_lo), __longlong_as_double(c.lo));
  } else {
    const unsigned long long wlo = c.lo + (c.hi << 32);
    const unsigned long long whi = static_cast<unsigned long long>(static_cast<long long>(c.hi) >> 32) + (wlo < c.lo ? 1ull : 0ull);
    const unsigned long long old = atomicAdd(&g->sum_lo, wlo);
    atomicAdd(&g->sum_hi, whi + (old + wlo < old ? 1ull : 0ull));
  }
  atomicMax(&g->nmin, c.nmin);
  atomicMax(&g->max, c.max);
}

}  // namespace sdbg
