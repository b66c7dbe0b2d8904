// column_kernels.cuh -- sm_90a kernels for the columnar filter / aggregate path.
//
// Reference behaviour (paths relative to /root/reference):
//   scan+filter   server/connector/full_scanner.cpp:81-147 (FullScanner::Scan: FilterWindow narrows a
//                 selection vector, survivors' columns are gathered, 2048 rows per call)
//                 libs/iresearch/include/iresearch/index/table_filter_iterator.cpp:147-264
//   NULL logic    server/connector/duckdb_search_full_scan.cpp:1785-1786 (NULL never passes)
//   aggregates    DuckDB HASH_GROUP_BY / UNGROUPED_AGGREGATE above the scan (not in the tree):
//                 COUNT u64, SUM(BIGINT) exact 128-bit, SUM/AVG(DOUBLE) double sum + one division.
//
// All kernels are HBM-streaming: every referenced column byte is read exactly once with 16-byte
// no-allocate loads, predicates are evaluated in registers, and only aggregates leave the SM
// (warp-shuffle + block reduction for ungrouped, L2-resident RED atomics for grouped).
#pragma once

#include "device_common.cuh"

namespace sdbg {

constexpr int kMaxPreds = 4;

struct ColDev {
  const void* values;        // 8-byte (i64/f64) or 4-byte (i32) elements
  const uint64_t* validity;  // null => NOT NULL
  int32_t type;              // 0 i64, 1 f64, 2 i32
  int32_t pad;
};
struct PredDev {
  ColDev col;
  int32_t op;
  int32_t pad;
  int64_t lo_i, hi_i;
  double lo_f, hi_f;
};
struct PredSet {
  PredDev p[kMaxPreds];
  int32_t n;
  int32_t pad;
};

__device__ __forceinline__ bool col_valid(const ColDev& c, uint64_t r) {
  return c.validity == nullptr || ((__ldg(c.validity + (r >> 6)) >> (r & 63)) & 1ull);
}
__device__ __forceinline__ bool cmp_i64(int op, long long v, long long lo, long long hi) {
  switch (op) {
    case 0: return v < lo; case 1: return v <= lo; case 2: return v > lo; case 3: return v >= lo;
    case 4: return v == lo; case 5: return v != lo; default: return v >= lo && v <= hi;
  }
}
__device__ __forceinline__ bool cmp_f64(int op, double v, double lo, double hi) {
  switch (op) {
    case 0: return v < lo; case 1: return v <= lo; case 2: return v > lo; case 3: return v >= lo;
    case 4: return v == lo; case 5: return v != lo; default: return v >= lo && v <= hi;
  }
}

// Evaluates predicate `p` on rows r, r+1 (r even). Returns a 2-bit mask. 8-byte columns are read
// with one 16-byte streaming load; i32 columns with one 8-byte load.
__device__ __forceinline__ uint32_t pred2(const PredDev& p, uint64_t r, uint64_t rows) {
  uint32_t valid = 3u;
  if (p.col.validity) valid = (col_valid(p.col, r) ? 1u : 0u) | ((r + 1 < rows && col_valid(p.col, r + 1)) ? 2u : 0u);
  if (p.op == 7) return (~valid) & 3u;
  if (p.op == 8) return valid;
  uint32_t m = 0;
  if (p.col.type == 2) {
    const int2 v = *reinterpret_cast<const int2*>(static_cast<const int*>(p.col.values) + r);
    m = (cmp_i64(p.op, v.x, p.lo_i, p.hi_i) ? 1u : 0u) | (cmp_i64(p.op, v.y, p.lo_i, p.hi_i) ? 2u : 0u);
  } else {
    const uint4 raw = ld_stream_v4(static_cast<const char*>(p.col.values) + r * 8);
    if (p.col.type == 1) {
      const double a = __longlong_as_double((static_cast<long long>(raw.y) << 32) | raw.x);
      const double b = __longlong_as_double((static_cast<long long>(raw.w) << 32) | raw.z);
      m = (cmp_f64(p.op, a, p.lo_f, p.hi_f) ? 1u : 0u) | (cmp_f64(p.op, b, p.lo_f, p.hi_f) ? 2u : 0u);
    } else {
      const long long a = (static_cast<long long>(raw.y) << 32) | raw.x;
      const long long b = (static_cast<long long>(raw.w) << 32) | raw.z;
      m = (cmp_i64(p.op, a, p.lo_i, p.hi_i) ? 1u : 0u) | (cmp_i64(p.op, b, p.lo_i, p.hi_i) ? 2u : 0u);
    }
  }
  return m & valid;
}

// All predicates on a row pair. Rows are padded to even counts by the host allocation (8-byte
// columns are allocated with 16 bytes of slack), the (r+1 < rows) test masks the phantom row.
__device__ __forceinline__ uint32_t preds2(const PredSet& ps, uint64_t r, uint64_t rows) {
  uint32_t m = (r + 1 < rows) ? 3u : 1u;
#pragma unroll
  for (int i = 0; i < kMaxPreds; ++i) {
    if (i < ps.n) m &= pred2(ps.p[i], r, rows);
  }
  return m;
}

// Predicate `p` of a filter chain on row r alone (the full-text kernels' per-doc test). The host hands chain predicates
// over as `lo <= v <= hi` (SDBG_OP_BETWEEN), `NOT (lo <= v <= hi)` (SDBG_OP_NE) or a NULL test (filter_view).
__device__ __forceinline__ bool pred1(const PredDev& p, uint64_t r) {
  const bool valid = col_valid(p.col, r);
  if (p.op >= 7) return (p.op == 8) == valid;
  if (!valid) return false;
  bool in;
  if (p.col.type == 1) {
    const double v = __ldg(static_cast<const double*>(p.col.values) + r);
    in = v >= p.lo_f && v <= p.hi_f;
  } else {
    const long long v = p.col.type == 2 ? static_cast<long long>(__ldg(static_cast<const int*>(p.col.values) + r))
                                        : __ldg(static_cast<const long long*>(p.col.values) + r);
    in = v >= p.lo_i && v <= p.hi_i;
  }
  return in != (p.op == 5);
}

// Every predicate of `ps` on row r, in the caller's order, up to the first that fails.
// The first predicate is read from fixed parameter offsets like a single one; the loop over the others is not unrolled,
// so the callers' instruction streams hold two copies of pred1, not four.
__device__ __forceinline__ bool preds_row(const PredSet& ps, uint64_t r) {
  if (ps.n == 0) return true;
  if (!pred1(ps.p[0], r)) return false;
#pragma unroll 1
  for (int i = 1; i < ps.n; ++i)
    if (!pred1(ps.p[i], r)) return false;
  return true;
}

__device__ __forceinline__ void load2_i64(const ColDev& c, uint64_t r, long long& a, long long& b) {
  if (c.type == 2) {
    const int2 v = *reinterpret_cast<const int2*>(static_cast<const int*>(c.values) + r);
    a = v.x; b = v.y;
  } else {
    const uint4 raw = ld_stream_v4(static_cast<const char*>(c.values) + r * 8);
    a = (static_cast<long long>(raw.y) << 32) | raw.x;
    b = (static_cast<long long>(raw.w) << 32) | raw.z;
  }
}
__device__ __forceinline__ void load2_f64(const ColDev& c, uint64_t r, double& a, double& b) {
  const uint4 raw = ld_stream_v4(static_cast<const char*>(c.values) + r * 8);
  a = __longlong_as_double((static_cast<long long>(raw.y) << 32) | raw.x);
  b = __longlong_as_double((static_cast<long long>(raw.w) << 32) | raw.z);
}

// ------------------------------------------------------------------------------------------
// Filter bitmap (parity probe, and the FilterWindow analogue). One thread per 2 rows, a warp
// produces one 64-bit mask word.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
filter_bitmap_kernel(const PredSet ps, uint64_t rows, unsigned long long* __restrict__ mask_out) {
  const uint64_t words = (rows + 63) / 64;
  const uint32_t lane = threadIdx.x & 31u;
  for (uint64_t w = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; w < words;
       w += (uint64_t(gridDim.x) * blockDim.x) >> 5) {
    const uint64_t r = w * 64 + 2ull * lane;
    const uint32_t m = r < rows ? preds2(ps, r, rows) : 0u;
    const uint32_t b0 = __ballot_sync(kFull, m & 1u);
    const uint32_t b1 = __ballot_sync(kFull, m & 2u);
    if (lane == 0) {
      // interleave: bit 2l = row pair l first row, bit 2l+1 = second row
      unsigned long long x = 0;
      for (int l = 0; l < 32; ++l) {
        x |= static_cast<unsigned long long>((b0 >> l) & 1u) << (2 * l);
        x |= static_cast<unsigned long long>((b1 >> l) & 1u) << (2 * l + 1);
      }
      mask_out[w] = x;
    }
  }
}

// ------------------------------------------------------------------------------------------
// filter -> COUNT(*), SUM(col).  Block partials are combined by the last block to finish
// (fixed order => deterministic double sum for a given grid).
// ------------------------------------------------------------------------------------------
struct CountSumOut {  // one per block, plus the final result in slot [gridDim.x]
  unsigned long long count;
  unsigned long long sum_lo;  // 128-bit two's complement
  long long sum_hi;
  double sum_f;
};

__device__ __forceinline__ void add128(unsigned long long& lo, long long& hi, long long v) {
  const unsigned long long nlo = lo + static_cast<unsigned long long>(v);
  hi += (v < 0 ? -1ll : 0ll) + (nlo < lo ? 1ll : 0ll);
  lo = nlo;
}
__device__ __forceinline__ void add128u(unsigned long long& lo, long long& hi, unsigned long long alo, long long ahi) {
  const unsigned long long nlo = lo + alo;
  hi += ahi + (nlo < lo ? 1ll : 0ll);
  lo = nlo;
}

__global__ void __launch_bounds__(256)
filter_count_sum_kernel(const PredSet ps, const ColDev sum_col, int has_sum, uint64_t rows,
                        CountSumOut* __restrict__ partials, unsigned int* __restrict__ done_counter, CountSumOut* host_out,
                        unsigned long long* host_seq, unsigned long long seq) {
  unsigned long long cnt = 0, lo = 0;
  long long hi = 0;
  double sf = 0.0;
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x * 2ull;
  for (uint64_t r = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) * 2ull; r < rows; r += stride) {
    const uint32_t m = preds2(ps, r, rows);
    if (has_sum) {
      uint32_t mv = m;
      if (sum_col.validity) mv &= (col_valid(sum_col, r) ? 1u : 0u) | ((r + 1 < rows && col_valid(sum_col, r + 1)) ? 2u : 0u);
      if (sum_col.type == 1) {
        double a, b; load2_f64(sum_col, r, a, b);
        if (mv & 1u) sf += a;
        if (mv & 2u) sf += b;
      } else {
        long long a, b; load2_i64(sum_col, r, a, b);
        if (mv & 1u) add128(lo, hi, a);
        if (mv & 2u) add128(lo, hi, b);
      }
    }
    cnt += __popc(m);
  }
  // warp reduce (128-bit add is associative; carry handled per step)
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    cnt += __shfl_xor_sync(kFull, cnt, o);
    const unsigned long long olo = __shfl_xor_sync(kFull, lo, o);
    const long long ohi = __shfl_xor_sync(kFull, hi, o);
    add128u(lo, hi, olo, ohi);
    sf += __shfl_xor_sync(kFull, sf, o);
  }
  __shared__ CountSumOut s[8];
  __shared__ bool s_last;
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  if (lane == 0) { s[warp].count = cnt; s[warp].sum_lo = lo; s[warp].sum_hi = hi; s[warp].sum_f = sf; }
  __syncthreads();
  if (threadIdx.x == 0) {
    CountSumOut t = s[0];
    for (uint32_t w = 1; w < blockDim.x / 32u; ++w) {
      t.count += s[w].count; add128u(t.sum_lo, t.sum_hi, s[w].sum_lo, s[w].sum_hi); t.sum_f += s[w].sum_f;
    }
    partials[blockIdx.x] = t;
    __threadfence();
    s_last = atomicAdd(done_counter, 1u) == gridDim.x - 1u;
  }
  __syncthreads();
  if (s_last) {
    // Last block to finish: combine the block partials with all 256 threads (thread i takes partials i, i + 256, ... in
    // index order, then a fixed shuffle / shared-memory tree): one pass of parallel loads instead of gridDim.x dependent
    // ones, and still a deterministic double sum for a given grid. The result also goes to `host_out` (mapped pinned
    // memory) when given, so a point query needs no device-to-host copy after the launch.
    __threadfence();
    CountSumOut t = {0, 0, 0, 0.0};
    for (uint32_t b = threadIdx.x; b < gridDim.x; b += blockDim.x) {
      const volatile CountSumOut* p = partials + b;
      t.count += p->count; add128u(t.sum_lo, t.sum_hi, p->sum_lo, p->sum_hi); t.sum_f += p->sum_f;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      t.count += __shfl_xor_sync(kFull, t.count, o);
      const unsigned long long olo = __shfl_xor_sync(kFull, t.sum_lo, o);
      const long long ohi = __shfl_xor_sync(kFull, t.sum_hi, o);
      add128u(t.sum_lo, t.sum_hi, olo, ohi);
      t.sum_f += __shfl_xor_sync(kFull, t.sum_f, o);
    }
    __syncthreads();                       // s[] is free again (thread 0 read it before the counter increment)
    if (lane == 0) s[warp] = t;
    __syncthreads();
    if (threadIdx.x == 0) {
      CountSumOut r = s[0];
      for (uint32_t w = 1; w < blockDim.x / 32u; ++w) {
        r.count += s[w].count; add128u(r.sum_lo, r.sum_hi, s[w].sum_lo, s[w].sum_hi); r.sum_f += s[w].sum_f;
      }
      partials[gridDim.x] = r;
      if (host_out != nullptr) {
        *host_out = r;
        __threadfence_system();
        // the caller spins on this word instead of synchronising the stream: the result above is visible before it
        if (host_seq != nullptr) *reinterpret_cast<volatile unsigned long long*>(host_seq) = seq;
      }
      *done_counter = 0u;
    }
  }
}

// ------------------------------------------------------------------------------------------
// Fused filter -> GROUP BY key -> COUNT(*), SUM(int), SUM(double)/COUNT(double).
// Dense group table indexed by key - key_min (DuckDB's perfect-hash aggregate when column
// statistics bound the key range; the min/max come from the staged column's zonemap). The table is
// 32 bytes per group = one L2 sector, updated with fire-and-forget RED atomics; at 1e5 groups it is
// 3.2 MB and stays L2-resident while the 40 B/row column stream goes by.
// ------------------------------------------------------------------------------------------
struct GroupSlot {            // 32 bytes = one L2 sector per group
  unsigned long long count;   // COUNT(*)
  long long sum_lo;           // SUM(int): low limb  (narrow mode: the whole sum)
  long long sum_hi;           // SUM(int): high limb (wide mode: sum of v >> 32)
  double sum_f;               // SUM(double)
};
static_assert(sizeof(GroupSlot) == 32, "one L2 sector per group");

struct GroupByParams {
  PredSet ps;
  ColDev key, sum_i, sum_f;
  int32_t has_sum_i, has_sum_f;
  int32_t wide_int;      // 1: values may exceed 32 bits => two limbs (lo = v & 0xFFFFFFFF, hi = v >> 32)
  int32_t count_f;       // 1: avg column nullable => cnt_f64 kept in a side array
  int64_t key_min;
  uint64_t key_span;
  uint64_t rows;
  GroupSlot* table;
  unsigned long long* cnt_f;   // [span] only when count_f
  unsigned long long* out_of_range;  // rows whose key fell outside [key_min, key_min+span): must stay 0
};

__device__ __forceinline__ void group_update(const GroupByParams& P, long long key, long long v, bool v_ok,
                                             double w, bool w_ok) {
  const unsigned long long idx = static_cast<unsigned long long>(key - P.key_min);
  if (idx >= P.key_span) { atomicAdd(P.out_of_range, 1ull); return; }
  GroupSlot* g = P.table + idx;
  atomicAdd(&g->count, 1ull);
  if (P.has_sum_i && v_ok) {
    if (P.wide_int) {
      atomicAdd(reinterpret_cast<unsigned long long*>(&g->sum_lo), static_cast<unsigned long long>(v) & 0xFFFFFFFFull);
      atomicAdd(reinterpret_cast<unsigned long long*>(&g->sum_hi), static_cast<unsigned long long>(v >> 32));
    } else {
      atomicAdd(reinterpret_cast<unsigned long long*>(&g->sum_lo), static_cast<unsigned long long>(v));
    }
  }
  if (P.has_sum_f && w_ok) {
    atomicAdd(&g->sum_f, w);
    if (P.count_f) atomicAdd(P.cnt_f + idx, 1ull);
  }
}

template <int kUnroll>
__global__ void __launch_bounds__(256)
filter_groupby_kernel(const GroupByParams P) {
  const uint64_t tile = uint64_t(blockDim.x) * 2ull * kUnroll;
  for (uint64_t base = uint64_t(blockIdx.x) * tile; base < P.rows; base += uint64_t(gridDim.x) * tile) {
    uint32_t m[kUnroll];
    long long k0[kUnroll], k1[kUnroll], v0[kUnroll], v1[kUnroll];
    double w0[kUnroll], w1[kUnroll];
    // Issue every load of the tile before the first use (kUnroll * 5 independent 16-byte loads).
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const uint64_t r = base + (uint64_t(u) * blockDim.x + threadIdx.x) * 2ull;
      m[u] = 0; k0[u] = k1[u] = v0[u] = v1[u] = 0; w0[u] = w1[u] = 0.0;
      if (r < P.rows) {
        m[u] = preds2(P.ps, r, P.rows);
        load2_i64(P.key, r, k0[u], k1[u]);
        if (P.has_sum_i) load2_i64(P.sum_i, r, v0[u], v1[u]);
        if (P.has_sum_f) load2_f64(P.sum_f, r, w0[u], w1[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      if (!m[u]) continue;
      const uint64_t r = base + (uint64_t(u) * blockDim.x + threadIdx.x) * 2ull;
      bool vi0 = true, vi1 = true, wf0 = true, wf1 = true;
      if (P.has_sum_i && P.sum_i.validity) { vi0 = col_valid(P.sum_i, r); vi1 = r + 1 < P.rows && col_valid(P.sum_i, r + 1); }
      if (P.has_sum_f && P.sum_f.validity) { wf0 = col_valid(P.sum_f, r); wf1 = r + 1 < P.rows && col_valid(P.sum_f, r + 1); }
      if (m[u] & 1u) group_update(P, k0[u], v0[u], vi0, w0[u], wf0);
      if (m[u] & 2u) group_update(P, k1[u], v1[u], vi1, w1[u], wf1);
    }
  }
}

// ------------------------------------------------------------------------------------------
// TMA-pipelined variant of the fused filter -> GROUP BY kernel (NOT NULL columns).
//
// The register-staged kernel above is latency-bound: bytes in flight are tied to resident warps, and a
// warp that is busy issuing its RED atomics is not loading. Here a single producer thread streams
// column tiles into a kStages-deep shared-memory ring with 1-D bulk async copies
// (cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes -> SASS UBLKCP) signalled through
// mbarriers, and the consumer warps evaluate predicates from shared memory and issue the REDs. In-flight
// bytes per SM = CTAs/SM * kStages * tile bytes (3 * 3 * 20 KB = 180 KB), independent of how far the
// consumers have got. Persistent CTAs, tiles handed out round-robin.
// ------------------------------------------------------------------------------------------
constexpr int kMaxStreams = 7;   // up to 4 predicate columns + key + sum_int + sum_f64 (deduplicated)

// Frame-of-reference bit-packed int64 column (DuckDB's `bitpacking` codec in FOR mode): per 2048-row group a base and a
// bit width; value i of the group sits at bit i * bits of the group's word run, little-endian; bits == 0 is a constant
// group. Staged columns keep every group 16-byte aligned (off8 even), so a 512-row tile of a group is 64 * bits bytes at
// byte offset (tile % 4) * 64 * bits of the group: one bulk copy.
struct ForBlockDev { long long base; uint32_t bits; uint32_t off8; };
constexpr uint32_t kForGroupRows = 2048;
constexpr int kTypeFor = 3;      // stream / predicate / key / sum type: FOR bit-packed int64 (TMA GROUP BY only)

// Everything the row loop needs is resolved on the host into plain scalars (direct constant-bank operands):
// no stream indirection, no per-row type switch over parameter arrays.
struct TmaGroupByParams {
  const void* src[kMaxStreams];   // distinct referenced columns
  int32_t elem[kMaxStreams];      // 8 (int64 / float64) or 4 (int32)
  uint32_t off[kMaxStreams + 1];  // byte offset of each stream inside a stage; off[n_streams] = stage bytes
  int32_t n_streams;
  int32_t n_preds;
  // Predicate i: pass = ((key(v) - pred_lo) <=u pred_span) != pred_negate, where key() maps the column type
  // onto int64 order: integers as they are, doubles through fkey() below. The host normalises every
  // comparison to a closed range in that key space and removes predicates that are always true / aborts
  // on ones that are always false, so lo <= lo + span always holds here.
  uint32_t pred_off[kMaxPreds];
  int32_t pred_type[kMaxPreds];     // 0 i64, 1 f64, 2 i32
  int32_t pred_negate[kMaxPreds];   // 1: SQL <>
  int64_t pred_lo[kMaxPreds];
  uint64_t pred_span[kMaxPreds];
  uint32_t key_off, sum_i_off, sum_f_off;
  int32_t key_type, sum_i_type;     // 0 i64, 2 i32
  int32_t has_sum_i, has_sum_f;
  int32_t wide_int;
  int32_t debug_skip;   // timing experiments only (SDBG_GROUPBY_DEBUG): bits 1/2/4 drop the count / sum_int / sum_f64 RED
  // Packed accumulators (kPacked kernels): COUNT and SUM(int) share one 64-bit word, count << pack_shift |
  // sum of (v - pack_bias), so a passing row costs one integer RED instead of two. The host proves from the
  // column's min/max and the row count that neither field can overflow; rows are dealt to pack_tables
  // (1..3) words of the slot by tile index when one word would not be enough.
  int32_t pack_shift, pack_tables;
  int64_t pack_bias;
  int64_t key_min;
  uint64_t key_span;
  uint64_t rows;
  GroupSlot* table;
  unsigned long long* out_of_range;
  // Zonemap verdicts (or null): skip[b] != 0 means no row of the 2048-row block b can pass the pushed predicates
  // (per-block min / max against every predicate's range: ColFilterChain::FilterWindow / DeadUntil,
  // irs/index/table_filter_iterator.cpp:147-286). Such tiles are neither copied nor looked at.
  const uint8_t* skip;
  // kFor kernels: hdr[s] != null marks stream s as FOR bit-packed (src[s] = its word stream, elem[s] = 8 keeps the raw
  // stage size). The producer copies only the tile's packed bytes and puts the group header into the stage; the
  // consumers decode from shared memory. *_stream: which stream feeds predicate i / the key / the integer sum.
  const ForBlockDev* hdr[kMaxStreams];
  int32_t pred_stream[kMaxPreds];
  int32_t key_stream, sum_i_stream;
};
constexpr uint32_t kZoneRows = 2048;   // rows per zonemap block = the reference's filter window (STANDARD_VECTOR_SIZE)

// Order-preserving map from the bits of a double to int64 (negative doubles reversed). -0.0 maps just
// below +0.0 (the host widens range ends that are zeros accordingly); NaNs land beyond +-inf, outside
// every closed range, which is the SQL comparison result.
__host__ __device__ __forceinline__ long long fkey(long long bits) { return bits ^ ((bits >> 63) & 0x7FFFFFFFFFFFFFFFll); }

// |w| / 2^eunit truncated to an integer below 2^(2*limb), split into two limbs carrying w's sign.
// Requires |w| < 2^(eunit + 2*limb) and w finite (the caller checks both).
__device__ __forceinline__ void fix_limbs(double w, int limb, int eunit, long long& l0, long long& l1) {
  const long long bits = __double_as_longlong(w);
  const int ex = int((bits >> 52) & 0x7FF);
  unsigned long long mant = static_cast<unsigned long long>(bits) & 0xFFFFFFFFFFFFFull;
  if (ex) mant |= 1ull << 52;
  const int s = (ex ? ex : 1) - 1075 - eunit;          // |w| = mant * 2^(s + eunit); s <= 2*limb - 53 <= 21
  unsigned long long lo, hi = 0ull;
  if (s >= 0) { lo = mant << s; if (s) hi = mant >> (64 - s); }
  else lo = s > -64 ? mant >> (-s) : 0ull;
  l0 = static_cast<long long>(lo & ((1ull << limb) - 1ull));
  l1 = static_cast<long long>((lo >> limb) | (hi << (64 - limb)));
  if (bits < 0) { l0 = -l0; l1 = -l1; }
}
// (s1 * 2^limb + s0) * 2^eunit as a double; the 128-bit integer is formed exactly, then rounded.
__host__ __device__ __forceinline__ double fix_total(long long s0, long long s1, int limb, int eunit) {
  long long hi = s1 >> (64 - limb);
  unsigned long long lo = static_cast<unsigned long long>(s1) << limb;
  const unsigned long long lo2 = lo + static_cast<unsigned long long>(s0);
  hi += (s0 >> 63) + (lo2 < lo ? 1 : 0);
  lo = lo2;
  const bool neg = hi < 0;
  if (neg) { lo = ~lo + 1ull; hi = ~hi + (lo == 0ull ? 1 : 0); }
  const double mag = static_cast<double>(static_cast<unsigned long long>(hi)) * 18446744073709551616.0 + static_cast<double>(lo);
  return scalbn(neg ? -mag : mag, eunit);
}

// Rows r, r+1 (r even) of a staged column as int64 values: one 16-byte (int32: 8-byte) shared load.
// kType: 0 i64, 1 f64 (raw bits), 2 i32 (sign-extended).
template <int kType>
__device__ __forceinline__ void load2(const unsigned char* col, uint32_t r, long long (&v)[2]) {
  if (kType == 2) {
    const int2 x = *reinterpret_cast<const int2*>(col + size_t(r) * 4u);
    v[0] = x.x; v[1] = x.y;
  } else {
    const longlong2 x = *reinterpret_cast<const longlong2*>(col + size_t(r) * 8u);
    v[0] = x.x; v[1] = x.y;
  }
}
// Bit j: row r + j lies in the closed key-space range [lo, lo + span].
template <int kType>
__device__ __forceinline__ uint32_t range2(const unsigned char* col, uint32_t r, long long lo, unsigned long long span) {
  long long v[2];
  load2<kType>(col, r, v);
  if (kType == 1) { v[0] = fkey(v[0]); v[1] = fkey(v[1]); }
  return (static_cast<unsigned long long>(v[0] - lo) <= span ? 1u : 0u) | (static_cast<unsigned long long>(v[1] - lo) <= span ? 2u : 0u);
}
// Rows r, r+1 (r even) of a FOR bit-packed tile in shared memory: `col` holds the tile's slice of its group's words, `h`
// the group header {base lo, base hi, bits, off8}. bits is warp-uniform; any width 0..64 (0: the constant `base`).
__device__ __forceinline__ void unpack2(const unsigned char* col, uint32_t r, const uint4 h, long long (&v)[2]) {
  const unsigned long long* w = reinterpret_cast<const unsigned long long*>(col);
  const uint32_t bits = h.z;
  const long long base = static_cast<long long>((static_cast<unsigned long long>(h.y) << 32) | h.x);
  const unsigned long long mask = bits >= 64u ? ~0ull : (1ull << bits) - 1ull;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const uint32_t bit = (r + uint32_t(j)) * bits, wi = bit >> 6, sh = bit & 63u;
    unsigned long long x = w[wi] >> sh;
    if (sh + bits > 64u) x |= w[wi + 1] << (64u - sh);    // the value straddles two words (never past the tile's data)
    v[j] = base + static_cast<long long>(x & mask);        // two's complement wrap-around undoes the encoder's subtraction
  }
}
__device__ __forceinline__ uint32_t range2_for(const unsigned char* col, uint32_t r, const uint4 h, long long lo, unsigned long long span) {
  long long v[2];
  unpack2(col, r, h, v);
  return (static_cast<unsigned long long>(v[0] - lo) <= span ? 1u : 0u) | (static_cast<unsigned long long>(v[1] - lo) <= span ? 2u : 0u);
}

// Shape of filter_groupby_tma_kernel: a ring of kGroupByStages tiles of kGroupByTileRows rows, filled by one producer
// warp and read by kGroupByConsumerWarps consumer warps. 3 x 20 KB stages -> 3 CTAs (24 consumer warps) per SM; on an
// H100 (400 W) ring depths 3 and 4 tie, 2 is 7 % slower.
constexpr int kGroupByStages = 3;
constexpr int kGroupByTileRows = 512;
constexpr int kGroupByConsumerWarps = 8;
// kFor: some streams are FOR bit-packed (TmaGroupByParams::hdr); needs kTileRows to divide kForGroupRows with 16-byte
// aligned tile slices. The group headers of the stages live behind the ring: kStages * kMaxStreams * 16 bytes.
template <bool kPacked, bool kFor>
__global__ void __launch_bounds__((kGroupByConsumerWarps + 1) * 32)
filter_groupby_tma_kernel(const TmaGroupByParams P) {
  constexpr int kStages = kGroupByStages, kTileRows = kGroupByTileRows, kConsumerWarps = kGroupByConsumerWarps;
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ __align__(8) uint64_t full_bar[kStages], empty_bar[kStages];
  static_assert(!kFor || (kForGroupRows % kTileRows == 0 && kTileRows % 128 == 0), "a tile's packed slice must be 16-byte aligned");

  const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31u;
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&full_bar[s], 1u); mbar_init(&empty_bar[s], kConsumerWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const uint32_t stage_bytes = P.off[P.n_streams];
  const uint64_t n_tiles = (P.rows + kTileRows - 1) / kTileRows;
  uint4* const pk_hdr = reinterpret_cast<uint4*>(smem + size_t(kStages) * stage_bytes);

  if (warp == kConsumerWarps) {
    if (kFor) {
      // ===== producer over packed streams: lane s moves stream s =====
      // Each lane loads the group header of its stream for the NEXT tile while this one waits for its stage, so no copy
      // address waits on a dependent global load; lane 0 puts the headers into the stage before its arrive (release).
      const bool mine = lane < uint32_t(P.n_streams);
      const ForBlockDev* hp = mine ? P.hdr[lane] : nullptr;
      const char* src = mine ? static_cast<const char*>(P.src[lane]) : nullptr;
      const uint32_t elem = mine ? uint32_t(P.elem[lane]) : 0u, soff = mine ? P.off[lane] : 0u;
      auto header = [&](uint64_t t) { return __ldg(reinterpret_cast<const uint4*>(hp + (t * kTileRows) / kForGroupRows)); };
      uint4 nh = make_uint4(0u, 0u, 0u, 0u);
      uint64_t nh_tile = ~0ull;                              // the tile `nh` belongs to
      uint32_t it = 0;
      for (uint64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        if (P.skip != nullptr && P.skip[(tile * kTileRows) / kZoneRows]) continue;   // zonemap verdict (warp-uniform): no header
        uint4 h = make_uint4(0u, 0u, 0u, 0u);
        if (hp != nullptr) h = nh_tile == tile ? nh : header(tile);   // not prefetched only after a skipped tile
        const uint64_t next = tile + gridDim.x;
        if (hp != nullptr && next < n_tiles && (P.skip == nullptr || !P.skip[(next * kTileRows) / kZoneRows])) { nh = header(next); nh_tile = next; }
        const uint32_t st = it % kStages, use = it / kStages;
        ++it;
        const uint64_t row0 = tile * kTileRows;
        const uint32_t nrows = uint32_t(min(static_cast<unsigned long long>(kTileRows), static_cast<unsigned long long>(P.rows - row0)));
        uint32_t bytes = 0u;
        const char* g = nullptr;
        if (hp != nullptr) {
          // the tile's slice of its group's words, rounded up to 16 bytes (covered by the column's slack); none when bits == 0
          bytes = (nrows * h.z + 127u) / 128u * 16u;
          g = src + uint64_t(h.w) * 8u + (row0 % kForGroupRows) * h.z / 8u;
        } else if (mine) {
          bytes = (nrows * elem + 15u) & ~15u;
          g = src + row0 * elem;
        }
        const uint32_t total = __reduce_add_sync(kFull, bytes);
        if (lane == 0) mbar_wait(&empty_bar[st], (use & 1u) ^ 1u);   // consumers released the previous use of this stage
        for (int s = 0; s < P.n_streams; ++s) {                // every lane shuffles, lane 0 writes
          uint4 x;
          x.x = __shfl_sync(kFull, h.x, s); x.y = __shfl_sync(kFull, h.y, s); x.z = __shfl_sync(kFull, h.z, s); x.w = __shfl_sync(kFull, h.w, s);
          if (lane == 0) pk_hdr[st * kMaxStreams + s] = x;
        }
        if (lane == 0) mbar_arrive_expect_tx(&full_bar[st], total);   // counts only the bytes issued below
        __syncwarp();
        if (bytes != 0u) bulk_g2s(smem + size_t(st) * stage_bytes + soff, g, bytes, &full_bar[st]);
      }
      return;
    }
    // ===== producer: one thread keeps the ring full =====
    if (lane == 0) {
      uint32_t it = 0;
      for (uint64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        if (P.skip != nullptr && P.skip[(tile * kTileRows) / kZoneRows]) continue;   // zonemap: nothing in this tile can pass
        const uint32_t st = it % kStages, use = it / kStages;
        ++it;
        mbar_wait(&empty_bar[st], (use & 1u) ^ 1u);           // consumers released the previous use of this stage
        const uint64_t row0 = tile * kTileRows;
        const uint32_t nrows = uint32_t(min(static_cast<unsigned long long>(kTileRows), static_cast<unsigned long long>(P.rows - row0)));
        uint32_t total = 0;
        for (int s = 0; s < P.n_streams; ++s) total += (nrows * uint32_t(P.elem[s]) + 15u) & ~15u;
        mbar_arrive_expect_tx(&full_bar[st], total);
        unsigned char* dst = smem + size_t(st) * stage_bytes;
        for (int s = 0; s < P.n_streams; ++s) {
          const uint32_t bytes = (nrows * uint32_t(P.elem[s]) + 15u) & ~15u;   // columns carry >= 64 B of slack
          bulk_g2s(dst + P.off[s], static_cast<const char*>(P.src[s]) + row0 * uint64_t(P.elem[s]), bytes, &full_bar[st]);
        }
      }
    }
    return;
  }

  // ===== consumers =====
  // Each lane owns two consecutive rows of a 64-row strip, so every staged column is read with one
  // 16-byte (8-byte for int32) shared load per lane and the column type is a warp-uniform switch
  // outside the per-row work.
  uint32_t it = 0;
  for (uint64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    if (P.skip != nullptr && P.skip[(tile * kTileRows) / kZoneRows]) continue;       // same verdict as the producer's
    const uint32_t st = it % kStages, use = it / kStages;
    ++it;
    mbar_wait(&full_bar[st], use & 1u);
    const unsigned char* base = smem + size_t(st) * stage_bytes;
    const uint64_t row0 = tile * kTileRows;
    const uint32_t nrows = uint32_t(min(static_cast<unsigned long long>(kTileRows), static_cast<unsigned long long>(P.rows - row0)));
    const uint32_t pack_word = kPacked ? uint32_t(tile % uint64_t(P.pack_tables)) : 0u;   // words 0..2 of a slot: count / sum_lo / sum_hi
    const uint4* const hst = pk_hdr + st * kMaxStreams;       // kFor: this stage's group headers, one per stream
    for (uint32_t rb = warp * 64u; rb < nrows; rb += kConsumerWarps * 64u) {   // warp-uniform trip count
      const uint32_t r = rb + 2u * lane;
      uint32_t m = r + 1u < nrows ? 3u : r < nrows ? 1u : 0u;   // bit j: row r + j exists and still passes
#pragma unroll
      for (int i = 0; i < kMaxPreds; ++i) {
        if (i < P.n_preds) {
          const unsigned char* col = base + P.pred_off[i];
          uint32_t in;
          if (kFor && P.pred_type[i] == kTypeFor) in = range2_for(col, r, hst[P.pred_stream[i]], P.pred_lo[i], P.pred_span[i]);
          else switch (P.pred_type[i]) {
            case 0: in = range2<0>(col, r, P.pred_lo[i], P.pred_span[i]); break;
            case 1: in = range2<1>(col, r, P.pred_lo[i], P.pred_span[i]); break;
            default: in = range2<2>(col, r, P.pred_lo[i], P.pred_span[i]); break;
          }
          m &= P.pred_negate[i] ? ~in : in;
        }
      }
      if (m == 0u) continue;
      long long key[2], v[2] = {0, 0};
      double w[2] = {0.0, 0.0};
      if (kFor && P.key_type == kTypeFor) unpack2(base + P.key_off, r, hst[P.key_stream], key);
      else if (P.key_type == 2) load2<2>(base + P.key_off, r, key); else load2<0>(base + P.key_off, r, key);
      if (kPacked || P.has_sum_i) {
        if (kFor && P.sum_i_type == kTypeFor) unpack2(base + P.sum_i_off, r, hst[P.sum_i_stream], v);
        else if (P.sum_i_type == 2) load2<2>(base + P.sum_i_off, r, v); else load2<0>(base + P.sum_i_off, r, v);
      }
      if (P.has_sum_f) {
        const double2 x = *reinterpret_cast<const double2*>(base + P.sum_f_off + size_t(r) * 8u);
        w[0] = x.x; w[1] = x.y;
      }
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        if (!(m & (1u << j))) continue;
        // a passing row issues its REDs (fire-and-forget) into the L2-resident group table
        const unsigned long long idx = static_cast<unsigned long long>(key[j] - P.key_min);
        if (idx >= P.key_span) { atomicAdd(P.out_of_range, 1ull); continue; }
        unsigned long long* g = reinterpret_cast<unsigned long long*>(P.table + idx);   // words: count, sum_lo, sum_hi, sum_f
        if (kPacked) {
          if (!(P.debug_skip & 3)) atomicAdd(g + pack_word, (1ull << P.pack_shift) + static_cast<unsigned long long>(v[j] - P.pack_bias));
        } else {
          if (!(P.debug_skip & 1)) atomicAdd(g, 1ull);
          if (P.has_sum_i && !(P.debug_skip & 2)) {
            if (P.wide_int) {
              atomicAdd(g + 1, static_cast<unsigned long long>(v[j]) & 0xFFFFFFFFull);
              atomicAdd(g + 2, static_cast<unsigned long long>(v[j] >> 32));
            } else {
              atomicAdd(g + 1, static_cast<unsigned long long>(v[j]));
            }
          }
        }
        if (P.has_sum_f && !(P.debug_skip & 4)) atomicAdd(reinterpret_cast<double*>(g + 3), w[j]);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[st]);   // this warp is done reading the stage
  }
}

// ------------------------------------------------------------------------------------------
// Zonemaps: min / max per 2048-row block of a NOT NULL column, in the int64 key space the predicates are resolved into
// (integers as they are, doubles through fkey()). Built once per column on first use (the reference keeps them in
// ColumnBlockMeta::statistics, irs/formats/column/column_reader.hpp:90-96). One warp per block.
// ------------------------------------------------------------------------------------------
template <int kType>
__global__ void __launch_bounds__(256)
zonemap_kernel(const unsigned char* __restrict__ values, uint64_t rows, long long* __restrict__ zone /* [blocks][2] */) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint64_t n_blocks = (rows + kZoneRows - 1) / kZoneRows;
  for (uint64_t b = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; b < n_blocks; b += (uint64_t(gridDim.x) * blockDim.x) >> 5) {
    long long mn = 0x7FFFFFFFFFFFFFFFll, mx = -0x7FFFFFFFFFFFFFFFll - 1;
    const uint64_t r0 = b * kZoneRows, r1 = min(rows, r0 + kZoneRows);
    for (uint64_t r = r0 + lane; r < r1; r += 32u) {
      long long v;
      if (kType == 2) v = reinterpret_cast<const int*>(values)[r];
      else v = reinterpret_cast<const long long*>(values)[r];
      if (kType == 1) v = fkey(v);
      mn = min(mn, v); mx = max(mx, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { mn = min(mn, __shfl_xor_sync(kFull, mn, o)); mx = max(mx, __shfl_xor_sync(kFull, mx, o)); }
    if (lane == 0) { zone[2 * b] = mn; zone[2 * b + 1] = mx; }
  }
}

constexpr uint8_t kZoneCheck = 0, kZoneDead = 1, kZonePass = 2;   // zone verdicts

struct ZoneVerdictParams {
  const long long* zone[kMaxPreds];   // per predicate: the column's zonemap (null: no verdict from this predicate)
  long long lo[kMaxPreds];
  unsigned long long span[kMaxPreds];
  int negate[kMaxPreds];
  int n_preds;
  int pass;                           // 1: also judge zones where every predicate holds for every row
  uint64_t n_blocks;
};
// The verdict of block b from the blocks' [min, max] in zone[i] (per predicate; null: no verdict from it): kZoneDead when
// some predicate's range [lo, lo + span] misses the block entirely (a negated predicate, SQL <>, only when the whole
// block equals the excluded value); with Z.pass, kZonePass when every predicate has a zonemap and its range covers
// [min, max] (negated: misses it); else kZoneCheck. zone is Z.zone on the device and host copies on the host.
__host__ __device__ __forceinline__ uint8_t zone_verdict(const ZoneVerdictParams& Z, const long long* const* zone, uint64_t b) {
  bool dead = false, all = Z.pass != 0;
  for (int i = 0; i < Z.n_preds; ++i) {
    if (zone[i] == nullptr) { all = false; continue; }
    const long long mn = zone[i][2 * b], mx = zone[i][2 * b + 1];
    const long long lo = Z.lo[i];
    const bool hi_below = static_cast<unsigned long long>(mn - lo) > Z.span[i] && mn > lo;   // block starts beyond lo + span
    const bool lo_above = mx < lo;                                                             // block ends before lo
    const bool inside = mn >= lo && static_cast<unsigned long long>(mx - lo) <= Z.span[i];    // block within the range
    if (Z.negate[i]) { dead |= Z.span[i] == 0ull && mn == lo && mx == lo; all &= hi_below || lo_above; }
    else { dead |= hi_below || lo_above; all &= inside; }
  }
  return dead ? kZoneDead : all ? kZonePass : kZoneCheck;
}

// skip[b] = zone_verdict(Z, Z.zone, b); counter (null: none) += number of dead blocks.
__global__ void __launch_bounds__(256)
zone_verdict_kernel(const ZoneVerdictParams Z, uint8_t* __restrict__ skip, unsigned long long* __restrict__ counter) {
  unsigned long long mine = 0;
  for (uint64_t b = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; b < Z.n_blocks; b += uint64_t(gridDim.x) * blockDim.x) {
    const uint8_t v = zone_verdict(Z, Z.zone, b);
    skip[b] = v;
    mine += v == kZoneDead ? 1ull : 0ull;
  }
  if (counter == nullptr) return;
  mine = warp_sum64(mine);
  if ((threadIdx.x & 31u) == 0u && mine) atomicAdd(counter, mine);
}

// The pushed predicate chain of a full-text entry (SDBG_OP_AND_NEXT) over one segment; ps.n == 0: no filter. zone, when
// set: the chain's verdict per kZoneRows rows of the segment (zone_verdict_kernel), n_zones of them.
struct ChainDev {
  PredSet ps;
  const uint8_t* zone;
  uint32_t n_zones;
  uint32_t pad;
};

// Doc `doc` (row doc - 1) against a chain: its zone's verdict when the zone is decided, else every predicate.
__device__ __forceinline__ bool chain_pass(const ChainDev& f, uint32_t doc) {
  const uint64_t r = uint64_t(doc) - 1u;
  if (f.zone != nullptr) {
    const uint8_t v = __ldg(f.zone + r / kZoneRows);
    if (v != kZoneCheck) return v == kZonePass;
  }
  return preds_row(f.ps, r);
}

// ------------------------------------------------------------------------------------------
// Hash-table GROUP BY for key ranges too wide for the dense table (DuckDB's regular hash aggregate).
// Open addressing with linear probing in global memory; a slot is claimed by CAS on its key, the
// aggregates are then updated with the same RED atomics as the dense path. Capacity is a power of two
// >= 2x the group-count hint; if the table fills up the kernel raises `overflow` and the host retries
// with a larger table. The reserved key value INT64_MIN lives in an extra slot at index `capacity`.
// ------------------------------------------------------------------------------------------
struct HashSlot {              // 48 bytes
  long long key;               // kEmptyKey = unclaimed
  unsigned long long count;
  long long sum_lo, sum_hi;    // SUM(int) limbs (wide form: v & 0xFFFFFFFF, v >> 32)
  double sum_f;
  unsigned long long cnt_f;
};
constexpr long long kEmptyKey = static_cast<long long>(0x8000000000000000ull);

struct HashGroupByParams {
  PredSet ps;
  ColDev key, sum_i, sum_f;
  int32_t has_sum_i, has_sum_f;
  uint64_t rows;
  HashSlot* table;             // capacity + 1 slots
  uint64_t capacity;           // power of two
  unsigned int* overflow;      // set when a probe sequence wraps the whole table
};

__device__ __forceinline__ uint64_t hash_key(long long k) {
  unsigned long long z = static_cast<unsigned long long>(k) * 0x9E3779B97F4A7C15ull;
  z ^= z >> 32;
  return z;
}

__device__ __forceinline__ void hash_update(const HashGroupByParams& P, long long key, long long v, bool v_ok, double w, bool w_ok) {
  HashSlot* g = nullptr;
  if (key == kEmptyKey) {
    g = P.table + P.capacity;  // dedicated slot for the reserved value
    g->key = key;              // benign race: every writer stores the same value
  } else {
    uint64_t h = hash_key(key) & (P.capacity - 1);
    for (uint64_t probes = 0; probes < P.capacity; ++probes) {
      long long cur = *reinterpret_cast<volatile long long*>(&P.table[h].key);
      if (cur == kEmptyKey) cur = static_cast<long long>(atomicCAS(reinterpret_cast<unsigned long long*>(&P.table[h].key),
                                                                   static_cast<unsigned long long>(kEmptyKey), static_cast<unsigned long long>(key)));
      if (cur == kEmptyKey || cur == key) { g = P.table + h; break; }
      h = (h + 1) & (P.capacity - 1);
    }
    if (!g) { atomicExch(P.overflow, 1u); return; }
  }
  atomicAdd(&g->count, 1ull);
  if (P.has_sum_i && v_ok) {
    atomicAdd(reinterpret_cast<unsigned long long*>(&g->sum_lo), static_cast<unsigned long long>(v) & 0xFFFFFFFFull);
    atomicAdd(reinterpret_cast<unsigned long long*>(&g->sum_hi), static_cast<unsigned long long>(v >> 32));
  }
  if (P.has_sum_f && w_ok) { atomicAdd(&g->sum_f, w); atomicAdd(&g->cnt_f, 1ull); }
}

__global__ void __launch_bounds__(256)
hash_init_kernel(HashSlot* table, uint64_t n) {
  for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += uint64_t(gridDim.x) * blockDim.x) {
    HashSlot s; s.key = kEmptyKey; s.count = 0; s.sum_lo = 0; s.sum_hi = 0; s.sum_f = 0.0; s.cnt_f = 0;
    table[i] = s;
  }
}

__global__ void __launch_bounds__(256)
filter_groupby_hash_kernel(const HashGroupByParams P) {
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x * 2ull;
  for (uint64_t r = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) * 2ull; r < P.rows; r += stride) {
    const uint32_t m = preds2(P.ps, r, P.rows);
    if (!m) continue;
    long long k0, k1, v0 = 0, v1 = 0;
    double w0 = 0, w1 = 0;
    load2_i64(P.key, r, k0, k1);
    if (P.has_sum_i) load2_i64(P.sum_i, r, v0, v1);
    if (P.has_sum_f) load2_f64(P.sum_f, r, w0, w1);
    bool vi0 = true, vi1 = true, wf0 = true, wf1 = true;
    if (P.has_sum_i && P.sum_i.validity) { vi0 = col_valid(P.sum_i, r); vi1 = r + 1 < P.rows && col_valid(P.sum_i, r + 1); }
    if (P.has_sum_f && P.sum_f.validity) { wf0 = col_valid(P.sum_f, r); wf1 = r + 1 < P.rows && col_valid(P.sum_f, r + 1); }
    if (m & 1u) hash_update(P, k0, v0, vi0, w0, wf0);
    if (m & 2u) hash_update(P, k1, v1, vi1, w1, wf1);
  }
}

// Dense table -> flat partial buffers for a SUM all-reduce:
// d_i64 = [count | sum_lo | sum_hi | cnt_f64] (4*span int64), d_f64 = [sum_f] (span float64).
__global__ void __launch_bounds__(256)
groupby_pack_kernel(const GroupSlot* __restrict__ table, const unsigned long long* __restrict__ cnt_f,
                    uint64_t span, long long* __restrict__ d_i64, double* __restrict__ d_f64,
                    int pack_shift, int pack_tables, long long pack_bias) {
  for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < span; i += uint64_t(gridDim.x) * blockDim.x) {
    GroupSlot g = table[i];
    if (pack_tables) {  // packed accumulators: split count << shift | sum(v - bias) back into the plain fields
      const unsigned long long w[3] = {g.count, static_cast<unsigned long long>(g.sum_lo), static_cast<unsigned long long>(g.sum_hi)};
      const unsigned long long mask = (1ull << pack_shift) - 1ull;
      unsigned long long cnt = 0, sum = 0;
      for (int t = 0; t < pack_tables; ++t) { cnt += w[t] >> pack_shift; sum += w[t] & mask; }
      g.count = cnt;
      g.sum_lo = static_cast<long long>(sum + static_cast<unsigned long long>(pack_bias) * cnt);   // two's complement: exact, |SUM| < 2^62 here
      g.sum_hi = 0;
    }
    d_i64[i] = static_cast<long long>(g.count);
    d_i64[span + i] = g.sum_lo;
    d_i64[2 * span + i] = g.sum_hi;
    d_i64[3 * span + i] = cnt_f ? static_cast<long long>(cnt_f[i]) : static_cast<long long>(g.count);
    d_f64[i] = g.sum_f;
  }
}

// min/max of an integer column (statistics gathered at staging: the reference keeps them per
// column block in ColumnBlockMeta::statistics, column_reader.hpp:90-96).
__global__ void __launch_bounds__(256)
minmax_i64_kernel(const ColDev col, uint64_t rows, long long* __restrict__ out /* [2] = {min, max} */) {
  long long mn = 0x7FFFFFFFFFFFFFFFll, mx = -0x7FFFFFFFFFFFFFFFll - 1;
  for (uint64_t r = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; r < rows; r += uint64_t(gridDim.x) * blockDim.x) {
    if (!col_valid(col, r)) continue;
    const long long v = col.type == 2 ? static_cast<long long>(static_cast<const int*>(col.values)[r])
                                      : static_cast<const long long*>(col.values)[r];
    mn = min(mn, v); mx = max(mx, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { mn = min(mn, __shfl_xor_sync(kFull, mn, o)); mx = max(mx, __shfl_xor_sync(kFull, mx, o)); }
  if ((threadIdx.x & 31u) == 0) { atomicMin(out, mn); atomicMax(out + 1, mx); }
}

// ------------------------------------------------------------------------------------------
// Synthetic column generator (SURVEY §8d): splitmix64 finaliser over seed ^ (stream << 48) ^ index.
// ------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ unsigned long long synth_hash(unsigned long long stream, unsigned long long index) {
  unsigned long long z = (0x5EDB2026ull ^ (stream << 48) ^ index) + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__global__ void __launch_bounds__(256)
synth_column_kernel(unsigned long long stream, int kind, uint64_t row0, uint64_t rows, void* __restrict__ out) {
  for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < rows; i += uint64_t(gridDim.x) * blockDim.x) {
    const unsigned long long h = synth_hash(stream, row0 + i);
    switch (kind) {
      case 0: static_cast<long long*>(out)[i] = static_cast<long long>(h % 100000ull); break;
      case 1: static_cast<long long*>(out)[i] = static_cast<long long>(h % 1000000ull); break;
      case 2: static_cast<double*>(out)[i] = static_cast<double>(h >> 11) * 0x1.0p-53; break;
      case 3: static_cast<long long*>(out)[i] = static_cast<long long>(h % 2001ull) - 1000ll; break;
      case 4: static_cast<double*>(out)[i] = static_cast<double>(h >> 11) * 0x1.0p-53 * 1000.0; break;
      case 6: static_cast<int*>(out)[i] = static_cast<int>(h % 1000000ull); break;
      case 7: static_cast<long long*>(out)[i] = static_cast<long long>((row0 + i) / 100ull); break;   // clustered (an insertion timestamp)
      default: static_cast<long long*>(out)[i] = static_cast<long long>(h); break;
    }
  }
}

// Late materialisation of hit rows (HitBatcher::MaterializeColumn, index/hit_batcher.hpp: the projected columns are fetched
// for the surviving doc ids only): out[i] = column[docs[i] - 1], validity bit i when the column is nullable.
template <typename T>
__global__ void __launch_bounds__(256)
gather_rows_kernel(const T* __restrict__ values, const unsigned long long* __restrict__ validity, const uint32_t* __restrict__ docs,
                   uint64_t n, uint64_t rows, T* __restrict__ out, unsigned char* __restrict__ out_valid) {
  for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += uint64_t(gridDim.x) * blockDim.x) {
    const uint64_t r = uint64_t(docs[i]) - 1ull;              // doc ids start at 1
    const bool inside = r < rows;
    const bool ok = inside && (validity == nullptr || ((validity[r >> 6] >> (r & 63ull)) & 1ull));
    out[i] = ok ? values[r] : T(0);
    if (out_valid != nullptr) out_valid[i] = ok ? 1u : 0u;
  }
}

// Frame-of-reference bit-packed int64 column (ForBlockDev above) -> raw values: the raw view of a packed column, and the
// decode of a caller's stream whose groups are not 16-byte aligned. One warp per 2048-row group.
__device__ __forceinline__ long long for_value(const ForBlockDev& h, const unsigned long long* w, uint32_t i) {
  unsigned long long v = 0ull;
  if (h.bits != 0u) {
    const unsigned long long mask = h.bits >= 64u ? ~0ull : ((1ull << h.bits) - 1ull);
    const uint64_t bit = uint64_t(i) * h.bits;
    const uint32_t sh = uint32_t(bit & 63ull);
    const unsigned long long lo = w[bit >> 6] >> sh;
    const unsigned long long hi = (sh != 0u && sh + h.bits > 64u) ? (w[(bit >> 6) + 1ull] << (64u - sh)) : 0ull;
    v = (lo | hi) & mask;
  }
  return h.base + static_cast<long long>(v);   // two's complement wrap-around = the encoder's subtraction undone
}

__global__ void __launch_bounds__(256)
for_unpack_kernel(const ForBlockDev* __restrict__ headers, const unsigned long long* __restrict__ words, uint64_t rows,
                  long long* __restrict__ out) {
  const uint64_t n_groups = (rows + kForGroupRows - 1) / kForGroupRows;
  const uint32_t lane = threadIdx.x & 31u;
  for (uint64_t g = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; g < n_groups; g += (uint64_t(gridDim.x) * blockDim.x) >> 5) {
    const ForBlockDev h = headers[g];
    const uint64_t row0 = g * kForGroupRows;
    const uint32_t n = (rows - row0 < kForGroupRows) ? uint32_t(rows - row0) : kForGroupRows;
    for (uint32_t i = lane; i < n; i += 32u) out[row0 + i] = for_value(h, words + h.off8, i);   // coalesced stores
  }
}

// Device packer, pass 1: per 2048-row group min / max of raw int64 values (or of an already packed stream when
// `words` is given: only the zonemap is written then). Writes the zonemap {min, max} per group (the predicate key space
// of an integer column is the value itself), and for raw input the header {base = min, bits = width of max - min} and
// the group's word count. One warp per group.
__global__ void __launch_bounds__(256)
for_stats_kernel(const long long* __restrict__ values, const ForBlockDev* __restrict__ packed_hdr,
                 const unsigned long long* __restrict__ words, uint64_t rows, long long* __restrict__ zone,
                 ForBlockDev* __restrict__ hdr, unsigned long long* __restrict__ n_words) {
  const uint64_t n_groups = (rows + kForGroupRows - 1) / kForGroupRows;
  const uint32_t lane = threadIdx.x & 31u;
  for (uint64_t g = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; g < n_groups; g += (uint64_t(gridDim.x) * blockDim.x) >> 5) {
    const uint64_t row0 = g * kForGroupRows;
    const uint32_t n = (rows - row0 < kForGroupRows) ? uint32_t(rows - row0) : kForGroupRows;
    long long mn = 0x7FFFFFFFFFFFFFFFll, mx = -0x7FFFFFFFFFFFFFFFll - 1;
    for (uint32_t i = lane; i < n; i += 32u) {
      const long long v = words ? for_value(packed_hdr[g], words + packed_hdr[g].off8, i) : values[row0 + i];
      mn = min(mn, v); mx = max(mx, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { mn = min(mn, __shfl_xor_sync(kFull, mn, o)); mx = max(mx, __shfl_xor_sync(kFull, mx, o)); }
    if (lane == 0) {
      zone[2 * g] = mn; zone[2 * g + 1] = mx;
      if (!words) {
        const unsigned long long span = static_cast<unsigned long long>(mx) - static_cast<unsigned long long>(mn);
        const uint32_t bits = span == 0ull ? 0u : uint32_t(64 - __clzll(static_cast<long long>(span)));
        ForBlockDev h; h.base = mn; h.bits = bits; h.off8 = 0u;
        hdr[g] = h;
        n_words[g] = (uint64_t(n) * bits + 63u) / 64u;
      }
    }
  }
}

// Device packer, pass 2: the word stream in sdbg_pack_for's layout (same bytes for the same values). Each lane builds
// whole 64-bit words from the values that overlap them, so no atomics are needed; off8 is the exclusive scan of the word
// counts. One warp per group; the last word of the stream (offsets[n_groups]) is the writer's zero slack word.
__global__ void __launch_bounds__(256)
for_pack_kernel(const long long* __restrict__ values, const ForBlockDev* __restrict__ stats_hdr,
                const unsigned long long* __restrict__ offsets, uint64_t rows, ForBlockDev* __restrict__ hdr,
                unsigned long long* __restrict__ words) {
  const uint64_t n_groups = (rows + kForGroupRows - 1) / kForGroupRows;
  const uint32_t lane = threadIdx.x & 31u;
  for (uint64_t g = (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; g < n_groups; g += (uint64_t(gridDim.x) * blockDim.x) >> 5) {
    ForBlockDev h = stats_hdr[g];
    h.off8 = uint32_t(offsets[g]);
    const uint64_t row0 = g * kForGroupRows;
    const uint32_t n = (rows - row0 < kForGroupRows) ? uint32_t(rows - row0) : kForGroupRows;
    if (lane == 0) hdr[g] = h;
    const uint32_t nw = uint32_t(offsets[g + 1] - offsets[g]);
    for (uint32_t wi = lane; wi < nw; wi += 32u) {
      const uint64_t b0 = uint64_t(wi) * 64u;
      const uint32_t i0 = uint32_t(b0 / h.bits), i1 = min(n - 1u, uint32_t((b0 + 63u) / h.bits));
      unsigned long long word = 0ull;
      for (uint32_t i = i0; i <= i1; ++i) {
        const unsigned long long d = static_cast<unsigned long long>(values[row0 + i]) - static_cast<unsigned long long>(h.base);
        const uint64_t p = uint64_t(i) * h.bits;
        word |= p >= b0 ? d << (p - b0) : d >> (b0 - p);
      }
      words[h.off8 + wi] = word;
    }
    if (g + 1 == n_groups && lane == 0) words[offsets[n_groups]] = 0ull;
  }
}

}  // namespace sdbg
