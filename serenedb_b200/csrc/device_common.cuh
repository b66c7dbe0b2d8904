// device_common.cuh -- small device helpers shared by the sm_90a kernels.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace sdbg {

constexpr uint32_t kWarp = 32;
constexpr unsigned kFull = 0xFFFFFFFFu;

// Streaming 16-byte load that does not allocate in L1 (column scans touch every byte once).
__device__ __forceinline__ uint4 ld_stream_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
// Read-only 16-byte load that stays cacheable (posting payloads and descriptors are re-read by
// neighbouring windows and by other queries of a batch).
__device__ __forceinline__ uint4 ld_ro_v4(const uint4* p) { return __ldg(p); }

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v, uint32_t lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(kFull, v, o);
    if (lane >= uint32_t(o)) v += t;
  }
  return v;
}
__device__ __forceinline__ uint32_t warp_sum(uint32_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}
__device__ __forceinline__ unsigned long long warp_sum64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

// ---- mbarrier + 1-D bulk async copy (TMA engine; SASS: SYNCS / UBLKCP) ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// Sortable top-k key: positive fp32 scores order like their bit patterns; the low half holds the
// complemented global doc ordinal so that, among equal scores, the smaller ordinal wins a
// "larger key" comparison. Canonical order = (score desc, segment asc, doc asc).
__device__ __host__ __forceinline__ unsigned long long make_key(float score, uint32_t ordinal) {
#ifdef __CUDA_ARCH__
  const uint32_t bits = __float_as_uint(score);
#else
  uint32_t bits; memcpy(&bits, &score, 4);
#endif
  return (static_cast<unsigned long long>(bits) << 32) | static_cast<unsigned long long>(~ordinal);
}

// In-place bitonic sort (descending) of n = power-of-two 64-bit keys in shared memory by the
// whole CTA. Ends with a barrier.
__device__ __forceinline__ void block_sort_desc(unsigned long long* s, uint32_t n) {
  for (uint32_t k = 2; k <= n; k <<= 1) {
    for (uint32_t j = k >> 1; j > 0; j >>= 1) {
      for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t p = i ^ j;
        if (p > i) {
          const unsigned long long a = s[i], b = s[p];
          const bool desc = (i & k) == 0;
          if ((a < b) == desc) { s[i] = b; s[p] = a; }
        }
      }
      __syncthreads();
    }
  }
}


// Exact top-k selection of 64-bit keys in shared memory, O(n): MSB-first radix select finds the k-th
// largest key (keys are unique: the doc ordinal is part of the key), then the keys >= it are compacted
// to the front in place (order not preserved) and the rest of the buffer is zeroed. Zero = empty slot.
// `hist` = 258 u32 of shared scratch; n_slots is a multiple of blockDim.x. All threads call it; ends
// with a barrier. Returns the k-th largest key, or 0 (nothing dropped) when fewer than k keys exist.
__device__ __forceinline__ unsigned long long block_select_topk(unsigned long long* keys, uint32_t n_slots, uint32_t k,
                                                                uint32_t* hist) {
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5, nwarps = blockDim.x >> 5;
  unsigned long long prefix = 0ull, mask = 0ull;
  uint32_t need = k;
  for (int shift = 56; shift >= 0; shift -= 8) {
    if (tid < 256) hist[tid] = 0u;
    __syncthreads();
    for (uint32_t i = tid; i < n_slots; i += blockDim.x) {
      const unsigned long long v = keys[i];
      if (v != 0ull && (v & mask) == prefix) atomicAdd(&hist[(v >> shift) & 255ull], 1u);
    }
    __syncthreads();
    if (warp == 0) {
      // lane l owns digits 255-8l .. 248-8l (descending); find the digit where the running count reaches `need`
      uint32_t c[8], sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) { c[j] = hist[255 - 8 * int(lane) - j]; sum += c[j]; }
      uint32_t run = warp_incl_scan(sum, lane) - sum;  // keys in higher digits (lower lanes)
      uint32_t found = 0xFFFFFFFFu, need_in = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (found == 0xFFFFFFFFu && run < need && run + c[j] >= need) { found = 255u - 8u * lane - uint32_t(j); need_in = need - run; }
        run += c[j];
      }
      const uint32_t who = __ballot_sync(kFull, found != 0xFFFFFFFFu);
      if (who == 0u) { if (lane == 0) { hist[256] = 0xFFFFFFFFu; hist[257] = 0u; } }   // fewer than `need` keys in total
      else if (lane == uint32_t(__ffs(who) - 1)) { hist[256] = found; hist[257] = need_in; }
    }
    __syncthreads();
    const uint32_t digit = hist[256];
    need = hist[257];
    __syncthreads();
    if (digit == 0xFFFFFFFFu) return 0ull;   // uniform: fewer than k keys, keep everything
    prefix |= static_cast<unsigned long long>(digit) << shift;
    mask |= 0xFFull << shift;
  }
  const unsigned long long kth = prefix;
  // In-place compaction, one tile of blockDim.x*4 slots at a time: survivors of a tile are written to
  // positions that only cover slots of tiles already read, so no unread key is overwritten.
  uint32_t written = 0;  // survivors placed so far (uniform)
  for (uint32_t t0 = 0; t0 < n_slots; t0 += blockDim.x * 4u) {
    unsigned long long v[4];
    uint32_t keep = 0;
#pragma unroll
    for (uint32_t i = 0; i < 4; ++i) {
      const uint32_t idx = t0 + tid * 4u + i;
      v[i] = idx < n_slots ? keys[idx] : 0ull;
      keep += (v[i] != 0ull && v[i] >= kth) ? 1u : 0u;
    }
    const uint32_t incl = warp_incl_scan(keep, lane);
    if (lane == 31) hist[warp] = incl;
    __syncthreads();   // all reads of this tile are done; warp totals visible
    uint32_t base = written + incl - keep, total = 0;
    for (uint32_t w = 0; w < nwarps; ++w) { if (w < warp) base += hist[w]; total += hist[w]; }
#pragma unroll
    for (uint32_t i = 0; i < 4; ++i) if (v[i] != 0ull && v[i] >= kth) keys[base++] = v[i];
    written += total;
    __syncthreads();
  }
  for (uint32_t i = written + tid; i < n_slots; i += blockDim.x) keys[i] = 0ull;
  __syncthreads();
  return kth;
}

}  // namespace sdbg
