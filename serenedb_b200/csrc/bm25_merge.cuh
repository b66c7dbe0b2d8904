// bm25_merge.cuh -- the exhaustive form of the warp-autonomous scan (bm25_stream.cuh): every list of a 1..4-term
// disjunction is streamed and merged, nothing is pruned or probed. Per-term stream state lives in registers (the term
// count is a template parameter) and there is no probe / block-max code in the loop, which keeps it at the size the
// instruction cache and the 80-register budget allow. Used when block-max pruning is off or cannot apply yet (the threshold of a query
// is still below the bound of its densest list); bm25_stream_kernel takes over once it can (lead list + probes).
// Helpers (StreamCtl, unpack4s, decode_block_global, warp_first_block, stream_compact / stream_rendezvous) are shared.
#pragma once

#include "bm25_stream.cuh"

namespace sdbg {

// A block is prefetched into its slot unless it is a StreamVByte tail (decoded from the arena by the scalar-ish svb
// path) or larger than a slot. Its size is exact: payloads are contiguous in the arena in block order, so
// units = off16 of the next block - off16 of this one (the block table ends with a sentinel).
__device__ __forceinline__ bool merge_block_is_svb(uint32_t packed) {
  const uint32_t de = desc_doc_enc(packed);
  return de == 5u || de == 7u || desc_freq_enc(packed) == 4u;
}

// Doc ids and frequencies of one prefetched block; `pd` / `pf` point at the doc / freq payload in SHARED memory.
// `stage` = 128 u32 of per-warp shared scratch (bitset rank scatter). Lane l gets postings 4l .. 4l+3.
__device__ __forceinline__ void merge_decode_block_smem(const uint4* pd, const uint4* pf, const uint4& d, uint32_t lane,
                                                  uint32_t* stage, uint32_t doc[4], uint32_t f[4]) {
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
  } else {                                          // de_values
    uint4 x = make_uint4(0, 0, 0, 0);
    if (4u * lane < len) x = pd[lane];
    doc[0] = x.x; doc[1] = x.y; doc[2] = x.z; doc[3] = x.w;
  }
  const uint32_t fenc = desc_freq_enc(d.w);
  if (fenc >= 5u) {
    unpack4s(pf, fenc - 4u, lane, f);
  } else if (fenc >= 1u && fenc <= 3u) {
    const uint32_t raw = *reinterpret_cast<const uint32_t*>(pf);
    f[0] = f[1] = f[2] = f[3] = fenc == 1u ? (raw & 0xFFu) : fenc == 2u ? (raw & 0xFFFFu) : raw;
  } else {
    uint4 x = make_uint4(0, 0, 0, 0);
    if (4u * lane < len) x = pf[lane];
    f[0] = x.x; f[1] = x.y; f[2] = x.z; f[3] = x.w;
  }
}

// per warp and term: docs[128] u32 | scores[128] f32 | slots[2][32] uint4 | descriptor window[16] uint4. The window is
// half the stream kernel's: with the 16 KB candidate buffer that is 52 KB per 2-term CTA, so four CTAs fit an SM.
constexpr uint32_t kMergeWin = 16u;
constexpr uint32_t kMergeTermBytes = 512u + 512u + 1024u + kMergeWin * 16u;

// Dynamic shared memory: cand[cap] u64 | per warp: T x kMergeTermBytes.
// Terms are in ascending-cost order (the host sorts them); T-1 is the "top" term.
template <uint32_t T>
__global__ void __launch_bounds__(kTopkThreads, kStreamMinBlocks)
bm25_merge_kernel(const TopkParams P) {
  static_assert(T >= 1 && T <= kStreamMaxTerms, "1..4 terms");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* cand = reinterpret_cast<unsigned long long*>(smem_raw);
  unsigned char* warp_area = reinterpret_cast<unsigned char*>(cand + P.cap);

  __shared__ __align__(16) StreamCtl ctl;
  __shared__ uint64_t s_bar[kTopkWarps][kStreamMaxTerms][2];
  __shared__ QTermDev s_qt[kStreamMaxTerms];

  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  unsigned char* mine = warp_area + warp * (T * kMergeTermBytes);
  auto live_docs = [&](uint32_t t) { return reinterpret_cast<uint32_t*>(mine + t * kMergeTermBytes); };
  auto live_scores = [&](uint32_t t) { return reinterpret_cast<float*>(mine + t * kMergeTermBytes + 512u); };
  auto slot_of = [&](uint32_t t, uint32_t s) { return reinterpret_cast<uint4*>(mine + t * kMergeTermBytes + 1024u + s * 512u); };
  auto desc_win = [&](uint32_t t) { return reinterpret_cast<uint4*>(mine + t * kMergeTermBytes + 2048u); };

  const uint4 work = P.work[blockIdx.x];
  const uint32_t q = work.x, chunk = work.z;   // work item = {query, first doc, docs, candidate list}
  const uint32_t t0 = P.qterm_off[q];
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
  if (tid < T) s_qt[tid] = P.qterms[t0 + tid];
  if (tid == 0) { ctl.ncand = 0u; ctl.matched = 0u; ctl.full = 0u; ctl.active = kTopkWarps; ctl.theta = 0ull; }
  if (lane == 0) {
#pragma unroll
    for (uint32_t t = 0; t < T; ++t) { mbar_init(&s_bar[warp][t][0], 1u); mbar_init(&s_bar[warp][t][1], 1u); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (P.claim != nullptr) {
    // This item may instead be run as lead list + probes by bm25_stream_kernel (lead mode), which is valid once the
    // query's threshold exceeds the summed list-wide bounds of every list but the shortest. First arrival decides.
    if (tid == 0) {
      float sfx1 = 0.f;
      for (uint32_t t = T; t-- > 1u;) {
        const uint32_t rf = s_qt[t].root_freq & 0x7FFFFFFFu;
        const float ub = (P.seg.blk_max != nullptr && rf != 0u) ? pair_bound(rf, s_qt[t].root_norm, s_qt[t])
                                                                 : __int_as_float(0x7f800000);
        sfx1 = __fadd_rn(sfx1, ub);
      }
      const float th = __uint_as_float(uint32_t(*reinterpret_cast<volatile unsigned long long*>(P.theta + q) >> 32));
      const uint32_t mine_mode = (__fmul_rn(sfx1, 1.000001f) < th) ? 2u : 1u;
      const uint32_t old = atomicCAS(P.claim + blockIdx.x, 0u, mine_mode);
      ctl.full = (old ? old : mine_mode) == 1u ? 0u : 0xFFFFFFFFu;
    }
    __syncthreads();
    if (ctl.full == 0xFFFFFFFFu) return;                 // the lead-mode kernel owns this item
  }
  unsigned long long* const theta_global = P.theta + q;
  const uint8_t* const norms_m1 = P.seg.norms ? P.seg.norms - 1 : nullptr;   // row = doc - 1 (full blocks, 1-byte norms)

  if (!warp_empty) {
    // ---- per-term stream state: registers (every loop over t is unrolled) ----
    uint32_t cur[T] = {};     // next block to load (index within the term)
    uint32_t wb[T] = {};      // first block of the descriptor window
    uint32_t start[T] = {};   // first block of this warp (slot / parity bookkeeping)
    uint32_t fr[T] = {};      // last doc of the live block (kNoDoc: list exhausted for this warp)
    uint32_t a0[T] = {};      // first pending entry of the live block (lower terms)
    uint32_t matched = 0;     // per lane; summed at the end
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
        if (want && pos < P.cap) { cand[pos] = key; want = false; }
        if (!__any_sync(kFull, want)) break;
        if (lane == 0) *reinterpret_cast<volatile uint32_t*>(&ctl.full) = 1u;
        stream_rendezvous(&ctl, cand, P.cap, P.k, theta_global);
        want = want && key > *reinterpret_cast<volatile unsigned long long*>(&ctl.theta);
      }
    };

    // Issues the bulk copy of block b of term t into its slot (b - start) & 1; every block gets exactly one arrival
    // on its slot's barrier, in block order (a block that is not prefetched arrives with 0 bytes). The window holds
    // the descriptors of b and b + 1 (refilled before it runs out), b + 1 possibly being the table's sentinel.
    auto prefetch = [&](const uint32_t t, uint32_t b) {
      if (b >= s_qt[t].nblk) return;
      if (lane == 0) {
        const uint4* w = desc_win(t);
        const uint4 d = w[b - wb[t]];
        uint32_t units = w[b - wb[t] + 1u].x - d.x;
        if (units > kSlotUnits || merge_block_is_svb(d.w)) units = 0u;
        const uint32_t r = b - start[t];
        uint64_t* bar = &s_bar[warp][t][r & 1u];
        mbar_arrive_expect_tx(bar, units * 16u);
        if (units) bulk_g2s(slot_of(t, r & 1u), P.seg.arena + d.x, units * 16u, bar);
      }
    };
    // Window = descriptors [wb, wb + 32) of the term (zeros past the sentinel).
    auto load_window = [&](const uint32_t t, uint32_t first) {
      __syncwarp();
      wb[t] = first;
      if (lane < kMergeWin)
        desc_win(t)[lane] = (first + lane <= s_qt[t].nblk) ? __ldg(P.seg.blocks + s_qt[t].blk_begin + first + lane) : make_uint4(0, 0, 0, 0);
      __syncwarp();
    };

    // Makes block cur[t] the live block of term t: wait for its payload, decode, gather norms, score, publish.
    auto advance = [&](const uint32_t t, uint32_t plo) {
      __syncwarp();                                                // every lane is done reading the block being replaced
      uint32_t* ld = live_docs(t);
      float* ls = live_scores(t);
      bool have = cur[t] < s_qt[t].nblk;
      uint4 d = make_uint4(0, 0, 0, 0);
      if (have) {
        if (cur[t] - wb[t] >= kMergeWin - 4u) load_window(t, cur[t]);   // keeps cur .. cur + 3 inside the window
        d = desc_win(t)[cur[t] - wb[t]];
        have = d.z < hi_w;                                         // first doc of the block (prev_last + 1) inside the sub-range
      }
      if (!have) {
        reinterpret_cast<uint4*>(ld)[lane] = make_uint4(kNoDoc, kNoDoc, kNoDoc, kNoDoc);
        fr[t] = kNoDoc; a0[t] = 0u;
        return;
      }
      const uint32_t r = cur[t] - start[t];
      mbar_wait(&s_bar[warp][t][r & 1u], (r >> 1) & 1u);
      uint32_t doc[4], f[4];
      const uint32_t units = desc_win(t)[cur[t] - wb[t] + 1u].x - d.x;
      if (units <= kSlotUnits && !merge_block_is_svb(d.w)) {
        const uint4* p = slot_of(t, r & 1u);
        merge_decode_block_smem(p, p + desc_fdelta(d.w), d, lane, ld, doc, f);
      } else {
        decode_block_global(P.seg.arena, d, lane, ld, reinterpret_cast<uint32_t*>(ls));
        const uint4 x = reinterpret_cast<const uint4*>(ld)[lane], y = reinterpret_cast<const uint4*>(ls)[lane];
        doc[0] = x.x; doc[1] = x.y; doc[2] = x.z; doc[3] = x.w;
        f[0] = y.x; f[1] = y.y; f[2] = y.z; f[3] = y.w;
      }
      __syncwarp();                                                // every lane is done with the slot
      prefetch(t, cur[t] + 2u);
      const uint32_t len = desc_len(d.w);
      uint32_t nrm[4];
      if (len == 128u && norms_m1 != nullptr && P.seg.norm_width == 1u) {   // uniform: full block, byte norms -- no pads, no width switch
#pragma unroll
        for (int j = 0; j < 4; ++j) nrm[j] = __ldg(norms_m1 + doc[j]);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const bool valid = 4u * lane + j < len;
          if (!valid) { doc[j] = kNoDoc; f[j] = 1u; }
          nrm[j] = valid ? load_norm(P.seg.norms, P.seg.norm_width, doc[j]) : 1u;
        }
      }
      float s[4];
      const float c0 = s_qt[t].c0, nc = s_qt[t].norm_const, nl = s_qt[t].norm_length;
#pragma unroll
      for (int j = 0; j < 4; ++j) s[j] = bm25_plain(f[j], nrm[j], c0, nc, nl);
      reinterpret_cast<uint4*>(ld)[lane] = make_uint4(doc[0], doc[1], doc[2], doc[3]);
      reinterpret_cast<float4*>(ls)[lane] = make_float4(s[0], s[1], s[2], s[3]);
      a0[t] = 0u;
      if (cur[t] == start[t]) {
        // the first block of a warp may hold docs below its sub-range: they are not pending
        a0[t] = __popc(__ballot_sync(kFull, doc[0] <= plo)) + __popc(__ballot_sync(kFull, doc[1] <= plo)) +
                __popc(__ballot_sync(kFull, doc[2] <= plo)) + __popc(__ballot_sync(kFull, doc[3] <= plo));
      }
      fr[t] = d.y;
      ++cur[t];
    };

    // Final entries (nobody absorbs them any more): count, threshold test, append.
    auto emit = [&](bool alive, uint32_t dv, float sv) {
      matched += alive ? 1u : 0u;
      bool want = alive && __float_as_uint(sv) >= theta_hi;
      if (__any_sync(kFull, want)) {
        unsigned long long key = 0ull;
        if (want) { key = make_key(sv, P.seg.ordinal_base + dv); want = key > theta; }
        append(want, key);
      }
    };

#pragma unroll
    for (uint32_t t = 0; t < T; ++t) {
      const uint32_t st = warp_first_block(P.seg.blocks + s_qt[t].blk_begin, s_qt[t].nblk, lo_w, lane);
      start[t] = st; cur[t] = st;
      load_window(t, st);
      fr[t] = lo_w - 1u;
    }
#pragma unroll
    for (uint32_t t = 0; t < T; ++t) { prefetch(t, start[t]); prefetch(t, start[t] + 1u); }

    uint32_t plo = lo_w - 1u;   // docs <= plo are final
    for (uint32_t step = 0;; ++step) {
      // ---- replace the live blocks that ended at plo (first step: every term) ----
#pragma unroll
      for (uint32_t t = 0; t < T; ++t)
        if (fr[t] == plo) advance(t, plo);
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

      // ---- lower terms: pending entries [a0, a1) with doc <= phi, 32 at a time, one entry per lane ----
#pragma unroll
      for (uint32_t t = 0; t + 1u < T; ++t) {
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
            // absorbed by a later term's live block? (a pending doc can only sit in live blocks: everything a list
            // holds before its live block is <= plo)
            if (fr[u] == kNoDoc) continue;                         // uniform: nothing live in term u
            const uint32_t* a = live_docs(u);
            uint32_t pos = 0;
#pragma unroll
            for (uint32_t stp = 64u; stp; stp >>= 1) pos += (a[pos + stp - 1u] < dv) ? stp : 0u;
            if (alive && a[pos] == dv) {
              float* as = live_scores(u);
              as[pos] = __fadd_rn(sv, as[pos]);                    // unique writer: docs are unique within term t
              alive = false;
            }
          }
          emit(alive, dv, sv);                                     // whatever is still alive is final
        }
        a0[t] = a1;
        __syncwarp();   // folds into later terms are visible before those terms are read
      }
      // ---- top term: its block is finalised as a whole when it retires (every lower term has been folded in up to
      // its last doc by then); lane l holds entries 4l .. 4l+3 ----
      if (fr[T - 1u] <= phi || phi >= hi_w) {
        const uint4 dd = reinterpret_cast<const uint4*>(live_docs(T - 1u))[lane];
        const float4 ss = reinterpret_cast<const float4*>(live_scores(T - 1u))[lane];
        const uint32_t dv[4] = {dd.x, dd.y, dd.z, dd.w};
        const float sv[4] = {ss.x, ss.y, ss.z, ss.w};
        const uint32_t first = 4u * lane;
        bool want_any = false;
        bool alive[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          alive[j] = first + j >= a0[T - 1u] && dv[j] <= phi;      // pads are kNoDoc > phi
          matched += alive[j] ? 1u : 0u;
          want_any |= alive[j] && __float_as_uint(sv[j]) >= theta_hi;
        }
        if (__any_sync(kFull, want_any)) {
#pragma unroll 1
          for (int j = 0; j < 4; ++j) {
            const uint32_t d1 = j == 0 ? dv[0] : j == 1 ? dv[1] : j == 2 ? dv[2] : dv[3];
            const float s1 = j == 0 ? sv[0] : j == 1 ? sv[1] : j == 2 ? sv[2] : sv[3];
            const bool al = j == 0 ? alive[0] : j == 1 ? alive[1] : j == 2 ? alive[2] : alive[3];
            bool want = al && __float_as_uint(s1) >= theta_hi;
            unsigned long long key = 0ull;
            if (want) { key = make_key(s1, P.seg.ordinal_base + d1); want = key > theta; }
            append(want, key);
          }
        }
        // on the last step of a warp (phi == hi_w) the block may still hold docs beyond the sub-range: they belong
        // to the next warp; a0 keeps what has been emitted if the same block is looked at again
        a0[T - 1u] = 128u;
      }
      plo = phi;
      if (phi >= hi_w) break;
      if (*reinterpret_cast<volatile uint32_t*>(&ctl.full)) stream_rendezvous(&ctl, cand, P.cap, P.k, theta_global);
    }
    // drain bulk copies that were issued but never consumed (they must not outlive the CTA's shared memory)
#pragma unroll
    for (uint32_t t = 0; t < T; ++t) {
      for (uint32_t b = cur[t]; b < min(s_qt[t].nblk, cur[t] + 2u); ++b) {   // issued: every block below cur + 2
        const uint32_t r = b - start[t];
        mbar_wait(&s_bar[warp][t][r & 1u], (r >> 1) & 1u);
      }
    }
    matched = warp_sum(matched);
    if (lane == 0 && matched) atomicAdd(&ctl.matched, matched);
  }
  __syncwarp();
  if (lane == 0) atomicSub(&ctl.active, 1u);
  // finished warps keep serving compactions until every warp of the CTA is done
  while (!stream_rendezvous(&ctl, cand, P.cap, P.k, theta_global)) {}

  // ---- chain epilogue: best k, sorted descending ----
  stream_compact(&ctl, cand, P.cap, P.k, theta_global);
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
