// sdbg_abi.cu -- the C ABI of libsdbg.so (include/sdbg.h): contexts, staging into HBM, query
// preparation and kernel launches. Host code only orchestrates; all per-posting / per-row work is
// in bm25_kernels.cuh and column_kernels.cuh. There is no CPU fallback anywhere in this file.
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <dlfcn.h>
#include <nccl.h>   // types only: the library is resolved at run time (sdbg_dist_init)

#include <algorithm>
#include <array>
#include <atomic>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <limits>
#include <thread>
#include <vector>

#include "../../include/sdbg.h"
#include "bm25_kernels.cuh"
#include "bm25_stream.cuh"
#include "bm25_merge.cuh"
#include "bm25_count.cuh"
#include "bm25_sort.cuh"
#include "column_kernels.cuh"
#include "posting_format.hpp"

using namespace sdbg;

// ------------------------------------------------------------------------------------------
// context / segment objects
// ------------------------------------------------------------------------------------------
namespace {

struct DevBuf {  // grow-only device scratch
  void* p = nullptr;
  size_t cap = 0;
};

struct ColumnObj {
  // Raw values. For a packed column this is the raw view, decoded on first use by raw_values() and kept until the column
  // is restaged or freed.
  void* d_values = nullptr;
  // Owned NOT NULL int64 columns whose frame-of-reference bit-packed form is smaller than the raw one stay packed:
  // ForBlockDev headers (packed_hdr_bytes, 256-aligned) | word stream (every group 16-byte aligned) | 64 B of slack.
  // The TMA GROUP BY reads this directly; every other reader goes through raw_values().
  void* d_packed = nullptr;
  size_t packed_bytes = 0;
  uint64_t* d_validity = nullptr;
  int type = 0;
  uint64_t rows = 0;
  bool owned = true;
  bool has_minmax = false;
  int64_t mn = 0, mx = 0;
  long long* d_zone = nullptr;  // zonemap: {min, max} per 2048-row block in predicate key space (NOT NULL columns, built on first use)
  bool zone_ok = false;         // d_zone holds the current values' zonemap (a restage of the same shape keeps the allocation)
  std::vector<long long> h_zone;  // host copy of the current zonemap, fetched on first use by the filter chains (empty: none)
};

}  // namespace

struct sdbg_ctx {
  int device = 0;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  cudaStream_t stream2 = nullptr;          // second lane for the top-k launch pair (driver-mode / plain chains)
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  std::string err;
  uint64_t launches = 0;
  DevBuf scratch[16];
  // the full-text top-k, count, facet, aggregate and sorted passes: [0] the call's region (a dist rank's buffer), [1] the
  // gathered buffers, [2] per-shape rows of a mixed-shape batch, [3] count scratch and the merged cells
  DevBuf pass[4];
  DevBuf stage_raw;          // raw int64 values of a column being packed at staging (reused: restaging allocates nothing)
  void* h_pinned = nullptr;  // pinned host staging for small transfers
  size_t h_pinned_cap = 0;
  void* flush = nullptr;
  size_t flush_bytes = 0;
  cudaEvent_t ev_copy[16] = {};   // one per host conversion thread of a top-k copy back (topk_to_host)
  bool topk_attr_set = false;   // topk_smem_attrs has run
  void* nccl_comm = nullptr;   // ncclComm_t once sdbg_dist_init ran
  // pinned [2]: out-of-range key count of the last deferred GROUP BY partial, and the number of SUM(double) partials
  // beyond abs_bound of the last sdbg_dist_groupby_merge (over all ranks)
  unsigned long long* h_oor = nullptr;
  void* h_result = nullptr;     // mapped pinned memory the point-query kernels write their result into (no D2H copy)
  void* d_result = nullptr;     // its device address
  unsigned long long result_seq = 0;   // completion word value of the last point query
  size_t h_result_cap = 0;
  bool counter_zeroed = false;  // scratch[10] starts at zero; every kernel that uses it leaves it at zero
  bool oor_pending = false;
  bool fix_over_pending = false;
  uint64_t zone_blocks_total = 0;   // last GROUP BY scan: 2048-row blocks seen / proven dead by their zonemaps
  unsigned long long* d_zone_skipped = nullptr;
  int dist_rank = 0, dist_world = 1;
  // optional per-kernel timing: CUDA events recorded on `stream` around the hot kernels
  int wand = 1;       // block-max pruning level: 0 off (exact total_matches), 1 planner-level block/window skips, 2 + exact-partial-score skips of the largest term
  bool profiling = false;
  struct ProfSpan { int id; cudaEvent_t a, b; };
  std::vector<ProfSpan> spans;
  std::vector<cudaEvent_t> event_pool;
};

struct sdbg_segment {
  sdbg_ctx* ctx = nullptr;
  uint32_t n_docs = 0;
  // postings
  void* d_arena = nullptr;
  void* d_blocks = nullptr;
  void* d_anchor = nullptr;
  void* d_blkmax = nullptr;
  // positions (sdbg_stage_positions, bm25_phrase.cuh): per block + sentinel a u64 base into d_pos; null: not staged
  void* d_pos_base = nullptr;
  void* d_pos = nullptr;
  std::vector<uint32_t> term_blk_begin, term_docs;
  std::vector<MaxPair> term_max;
  std::vector<uint8_t> term_probe;
  std::vector<uint64_t> term_bytes;
  uint64_t arena_bytes = 0, n_blocks = 0, n_postings = 0;
  bool has_wand = false;
  float wand_b = 0.75f;   // the b the block-max (freq, norm) pairs were chosen for (BM25 default unless told otherwise)
  // the average field length the pairs were chosen with (PostingWriter::feed); 0 = none: without norms every doc scores
  // with norm 1, so a pair's order cannot depend on the average length
  float wand_avg_dl = 0.f;
  // norms
  void* d_norms = nullptr;
  uint32_t norm_width = 0;
  // deleted docs (DocumentMask) as a bitmap over doc ids 0..n_docs
  void* d_deleted = nullptr;
  uint64_t n_deleted = 0;
  // columns
  std::map<uint64_t, ColumnObj> cols;
  // zone verdicts of the last full-text call's filter chain over this segment (chain_verdicts)
  DevBuf verdict;
};

struct sdbg_writer {
  std::unique_ptr<PostingWriter> w;
  std::vector<sdbg_term_meta> metas;
};

namespace {

int fail(sdbg_ctx* c, int code, const std::string& msg) {
  if (c) c->err = msg;
  return code;
}
#define CU(ctx, expr)                                                                                   \
  do {                                                                                                  \
    cudaError_t e_ = (expr);                                                                            \
    if (e_ != cudaSuccess)                                                                              \
      return fail((ctx), SDBG_ECUDA, std::string(#expr) + ": " + cudaGetErrorString(e_));              \
  } while (0)

int ensure(sdbg_ctx* c, DevBuf& b, size_t bytes) {
  if (b.cap >= bytes) return SDBG_OK;
  if (b.p) { cudaStreamSynchronize(c->stream); cudaFree(b.p); b.p = nullptr; b.cap = 0; }
  const size_t want = std::max(bytes, size_t(1) << 20);
  CU(c, cudaMalloc(&b.p, want));
  b.cap = want;
  return SDBG_OK;
}
int ensure_pinned(sdbg_ctx* c, size_t bytes) {
  if (c->h_pinned_cap >= bytes) return SDBG_OK;
  if (c->h_pinned) { cudaStreamSynchronize(c->stream); cudaFreeHost(c->h_pinned); c->h_pinned = nullptr; c->h_pinned_cap = 0; }
  const size_t want = std::max(bytes, size_t(1) << 20);
  CU(c, cudaMallocHost(&c->h_pinned, want));
  c->h_pinned_cap = want;
  return SDBG_OK;
}

__global__ void fill_u64_kernel(unsigned long long* p, size_t n, unsigned long long v) {
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += size_t(gridDim.x) * blockDim.x) p[i] = v;
}
__global__ void flush_kernel(uint4* p, size_t n, uint32_t v) {
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += size_t(gridDim.x) * blockDim.x)
    p[i] = make_uint4(v, v, v, v);
}

// Kernel ids for sdbg_profile_*: the kernels a roofline is reported for.
enum { kProfGroupBy = 0, kProfTopk = 1, kProfMerge = 2, kProfCountSum = 3, kProfBitmap = 4, kProfIds = 5 };

struct ProfScope {  // records an event pair around a launch when profiling is on
  sdbg_ctx* c; int idx = -1;
  ProfScope(sdbg_ctx* ctx, int id) : c(ctx) {
    if (!c->profiling) return;
    auto get = [&]() { cudaEvent_t e; if (!c->event_pool.empty()) { e = c->event_pool.back(); c->event_pool.pop_back(); } else cudaEventCreate(&e); return e; };
    sdbg_ctx::ProfSpan sp{id, get(), get()};
    cudaEventRecord(sp.a, c->stream);
    c->spans.push_back(sp);
    idx = int(c->spans.size()) - 1;
  }
  ~ProfScope() { if (idx >= 0) cudaEventRecord(c->spans[size_t(idx)].b, c->stream); }
};

uint32_t next_pow2(uint32_t v) { uint32_t p = 1; while (p < v) p <<= 1; return p; }

int env_int(const char* name, int dflt) {
  const char* s = std::getenv(name);
  return s && *s ? std::atoi(s) : dflt;
}

// The GROUP BY errors found on the device after an asynchronous call returned (h_oor); the stream has been synchronised.
int deferred_groupby_errors(sdbg_ctx* c) {
  const bool oor = c->oor_pending && c->h_oor[0], over = c->fix_over_pending && c->h_oor[1];
  c->oor_pending = c->fix_over_pending = false;
  if (oor) return fail(c, SDBG_EINVAL, "GROUP BY key outside [key_min, key_min + span)");
  if (over) return fail(c, SDBG_EINVAL, "a SUM(double) partial exceeds the abs_bound of sdbg_dist_groupby_merge");
  return SDBG_OK;
}

}  // namespace

// ------------------------------------------------------------------------------------------
// lifecycle
// ------------------------------------------------------------------------------------------
extern "C" const char* sdbg_version(void) { return "serenedb-b200 0.1 (sm_90a)"; }

extern "C" int sdbg_init(int device, sdbg_ctx** out) {
  if (!out) return SDBG_EINVAL;
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) return SDBG_ENODEVICE;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return SDBG_ENODEVICE;
  if (prop.major != 9 || prop.minor != 0) return SDBG_ENODEVICE;  // kernels are built for sm_90a only
  auto* c = new sdbg_ctx;
  c->device = device;
  c->sm_count = prop.multiProcessorCount;
  c->wand = std::max(0, std::min(2, env_int("SDBG_WAND", 2)));
  if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&c->stream2, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreate(&c->ev0) != cudaSuccess || cudaEventCreate(&c->ev1) != cudaSuccess) {
    delete c;
    return SDBG_ECUDA;
  }
  *out = c;
  return SDBG_OK;
}

extern "C" int sdbg_dist_destroy(sdbg_ctx* c);
extern "C" void sdbg_destroy(sdbg_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  for (auto& b : c->scratch) if (b.p) cudaFree(b.p);
  for (auto& b : c->pass) if (b.p) cudaFree(b.p);
  if (c->stage_raw.p) cudaFree(c->stage_raw.p);
  if (c->h_pinned) cudaFreeHost(c->h_pinned);
  if (c->h_oor) cudaFreeHost(c->h_oor);
  if (c->d_zone_skipped) cudaFree(c->d_zone_skipped);
  if (c->h_result) cudaFreeHost(c->h_result);
  if (c->flush) cudaFree(c->flush);
  cudaStreamSynchronize(c->stream2);
  sdbg_dist_destroy(c);
  cudaEventDestroy(c->ev0); cudaEventDestroy(c->ev1);
  cudaEventDestroy(c->ev_fork); cudaEventDestroy(c->ev_join);
  for (cudaEvent_t e : c->ev_copy) if (e) cudaEventDestroy(e);
  cudaStreamDestroy(c->stream2);
  cudaStreamDestroy(c->stream);
  delete c;
}
extern "C" const char* sdbg_last_error(const sdbg_ctx* c) { return c ? c->err.c_str() : "null context"; }
extern "C" int sdbg_timer_start(sdbg_ctx* c) { CU(c, cudaSetDevice(c->device)); CU(c, cudaEventRecord(c->ev0, c->stream)); return SDBG_OK; }
extern "C" int sdbg_timer_stop(sdbg_ctx* c, float* ms) {
  CU(c, cudaEventRecord(c->ev1, c->stream));
  CU(c, cudaEventSynchronize(c->ev1));
  CU(c, cudaEventElapsedTime(ms, c->ev0, c->ev1));
  return SDBG_OK;
}
extern "C" int sdbg_sync(sdbg_ctx* c) {
  CU(c, cudaStreamSynchronize(c->stream));
  return deferred_groupby_errors(c);
}
extern "C" uint64_t sdbg_launch_count(const sdbg_ctx* c) { return c ? c->launches : 0; }
extern "C" int sdbg_flush_l2(sdbg_ctx* c) {
  CU(c, cudaSetDevice(c->device));
  if (!c->flush) { c->flush_bytes = size_t(256) << 20; CU(c, cudaMalloc(&c->flush, c->flush_bytes)); }
  static uint32_t tick = 0;
  flush_kernel<<<c->sm_count * 4, 256, 0, c->stream>>>(static_cast<uint4*>(c->flush), c->flush_bytes / 16, ++tick);
  CU(c, cudaGetLastError());
  return SDBG_OK;
}

extern "C" int sdbg_set_wand(sdbg_ctx* c, int enabled) {
  if (!c) return SDBG_EINVAL;
  c->wand = enabled < 0 ? 0 : enabled > 2 ? 2 : enabled;
  return SDBG_OK;
}
extern "C" int sdbg_profile_enable(sdbg_ctx* c, int on) {
  if (!c) return SDBG_EINVAL;
  CU(c, cudaStreamSynchronize(c->stream));
  for (auto& sp : c->spans) { c->event_pool.push_back(sp.a); c->event_pool.push_back(sp.b); }
  c->spans.clear();
  c->profiling = on != 0;
  return SDBG_OK;
}
extern "C" int sdbg_profile_read(sdbg_ctx* c, int kernel_id, double* total_ms, uint64_t* launches) {
  if (!c || !total_ms || !launches || kernel_id < 0 || kernel_id >= kProfIds) return SDBG_EINVAL;
  CU(c, cudaStreamSynchronize(c->stream));
  double ms = 0; uint64_t n = 0;
  for (auto& sp : c->spans) {
    if (sp.id != kernel_id) continue;
    float t = 0;
    CU(c, cudaEventElapsedTime(&t, sp.a, sp.b));
    ms += t; ++n;
  }
  *total_ms = ms; *launches = n;
  return SDBG_OK;
}

// ------------------------------------------------------------------------------------------
// staging
// ------------------------------------------------------------------------------------------
extern "C" int sdbg_segment_create(sdbg_ctx* c, uint32_t docs_count, sdbg_segment** out) {
  if (!c || !out) return SDBG_EINVAL;
  if (docs_count > kMaxDocId) return fail(c, SDBG_EINVAL, "docs_count > 2^32-2 (2^32-1 is doc_limits::eof)");
  auto* s = new sdbg_segment;
  s->ctx = c; s->n_docs = docs_count;
  *out = s;
  return SDBG_OK;
}

namespace {
void free_positions(sdbg_segment* s) {   // they index the posting blocks: restaging the postings drops them
  if (s->d_pos_base) cudaFree(s->d_pos_base);
  if (s->d_pos) cudaFree(s->d_pos);
  s->d_pos_base = s->d_pos = nullptr;
}
void free_postings(sdbg_segment* s) {
  if (s->d_arena) cudaFree(s->d_arena);
  if (s->d_blocks) cudaFree(s->d_blocks);
  if (s->d_anchor) cudaFree(s->d_anchor);
  s->d_anchor = nullptr;
  if (s->d_blkmax) cudaFree(s->d_blkmax);
  s->d_arena = s->d_blocks = s->d_blkmax = nullptr;
  free_positions(s);
}
void free_column(ColumnObj& c) {
  if (c.d_zone) { cudaFree(c.d_zone); c.d_zone = nullptr; }
  if (c.owned && c.d_values) cudaFree(c.d_values);
  if (c.d_packed) cudaFree(c.d_packed);
  if (c.d_validity) cudaFree(c.d_validity);
  c.d_values = nullptr; c.d_validity = nullptr; c.d_packed = nullptr;
}
}  // namespace

extern "C" void sdbg_segment_destroy(sdbg_segment* s) {
  if (!s) return;
  cudaSetDevice(s->ctx->device);
  cudaStreamSynchronize(s->ctx->stream);
  free_postings(s);
  if (s->d_norms) cudaFree(s->d_norms);
  if (s->d_deleted) cudaFree(s->d_deleted);
  for (auto& kv : s->cols) free_column(kv.second);
  if (s->verdict.p) cudaFree(s->verdict.p);
  delete s;
}

extern "C" sdbg_ctx* sdbg_segment_context(const sdbg_segment* s) { return s ? s->ctx : nullptr; }

// Zonemap effect of the last GROUP BY scan on this context: 2048-row blocks looked at by the verdict pass and how many
// of them were proven dead (never copied, never evaluated). Synchronises the stream.
extern "C" int sdbg_scan_stats(sdbg_ctx* c, uint64_t* blocks_total, uint64_t* blocks_skipped) {
  if (!c) return SDBG_EINVAL;
  unsigned long long skipped = 0;
  if (c->d_zone_skipped) {
    CU(c, cudaMemcpyAsync(&skipped, c->d_zone_skipped, 8, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
  }
  if (blocks_total) *blocks_total = c->zone_blocks_total;
  if (blocks_skipped) *blocks_skipped = skipped;
  return SDBG_OK;
}

extern "C" int sdbg_segment_set_wand_b(sdbg_segment* s, float wand_b) {
  if (!s) return SDBG_EINVAL;
  s->wand_b = wand_b;
  return SDBG_OK;
}

extern "C" int sdbg_segment_set_wand_avg_dl(sdbg_segment* s, float avg_dl) {
  if (!s || !(avg_dl >= 0.f) || avg_dl == std::numeric_limits<float>::infinity()) return SDBG_EINVAL;
  s->wand_avg_dl = avg_dl;
  return SDBG_OK;
}

extern "C" int sdbg_stage_docs_mask(sdbg_segment* s, const uint32_t* deleted_docs, size_t n) {
  if (!s || (!deleted_docs && n)) return SDBG_EINVAL;
  sdbg_ctx* c = s->ctx;
  CU(c, cudaSetDevice(c->device));
  CU(c, cudaStreamSynchronize(c->stream));
  if (s->d_deleted) { CU(c, cudaFree(s->d_deleted)); s->d_deleted = nullptr; }
  s->n_deleted = 0;
  if (!n) return SDBG_OK;
  std::vector<uint32_t> bits((size_t(s->n_docs) + 32) / 32 + 1, 0u);
  for (size_t i = 0; i < n; ++i) {
    const uint32_t d = deleted_docs[i];
    if (d == 0 || d > s->n_docs) return fail(c, SDBG_EINVAL, "deleted doc id outside 1..docs_count");
    if (!((bits[d >> 5] >> (d & 31u)) & 1u)) ++s->n_deleted;
    bits[d >> 5] |= 1u << (d & 31u);
  }
  CU(c, cudaMalloc(&s->d_deleted, bits.size() * 4));
  CU(c, cudaMemcpyAsync(s->d_deleted, bits.data(), bits.size() * 4, cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  return SDBG_OK;
}

namespace {
int upload_postings(sdbg_segment* s, const StagedPostings& sp) {
  sdbg_ctx* c = s->ctx;
  CU(c, cudaSetDevice(c->device));
  free_postings(s);
  CU(c, cudaMalloc(&s->d_arena, std::max<size_t>(sp.arena.size(), 16)));
  // one sentinel descriptor behind the last block: off16 = end of the payloads, so that "next offset - own offset" is
  // the payload size of every block (the stream kernel's prefetch size)
  CU(c, cudaMalloc(&s->d_blocks, (sp.blocks.size() + 1) * sizeof(BlockDesc)));
  {
    BlockDesc sentinel;
    sentinel.off16 = uint32_t((sp.arena.size() >= 1024 ? sp.arena.size() - 1024 : 0) / 16);
    sentinel.last_doc = 0xFFFFFFFFu; sentinel.prev_last = 0xFFFFFFFFu; sentinel.packed = 0;
    CU(c, cudaMemcpyAsync(static_cast<BlockDesc*>(s->d_blocks) + sp.blocks.size(), &sentinel, sizeof sentinel, cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
  }
  CU(c, cudaMalloc(&s->d_blkmax, std::max<size_t>(sp.blk_max.size() * sizeof(MaxPair), 16)));
  CU(c, cudaMalloc(&s->d_anchor, std::max<size_t>(sp.blk_anchor.size() * 4, 16)));
  CU(c, cudaMemcpyAsync(s->d_anchor, sp.blk_anchor.data(), sp.blk_anchor.size() * 4, cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaMemcpyAsync(s->d_arena, sp.arena.data(), sp.arena.size(), cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaMemcpyAsync(s->d_blocks, sp.blocks.data(), sp.blocks.size() * sizeof(BlockDesc), cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaMemcpyAsync(s->d_blkmax, sp.blk_max.data(), sp.blk_max.size() * sizeof(MaxPair), cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  s->term_blk_begin = sp.term_blk_begin;
  s->term_docs = sp.term_docs;
  s->term_max = sp.term_max;
  s->term_probe = sp.term_probe;
  s->term_bytes = sp.term_bytes;
  s->arena_bytes = sp.arena.size();
  s->n_blocks = sp.blocks.size();
  s->n_postings = sp.n_postings;
  s->has_wand = sp.has_wand;
  return SDBG_OK;
}
}  // namespace

extern "C" int sdbg_stage_postings(sdbg_segment* s, const uint8_t* doc_file, size_t n, const sdbg_term_meta* terms,
                                   size_t n_terms, int has_wand) {
  if (!s || (!doc_file && n) || (!terms && n_terms)) return SDBG_EINVAL;
  static_assert(sizeof(sdbg_term_meta) == sizeof(TermMeta), "ABI term meta mirrors the host struct");
  StagedPostings sp;
  const std::string e = stage_postings(doc_file, n, reinterpret_cast<const TermMeta*>(terms), n_terms, has_wand != 0, &sp);
  if (!e.empty()) return fail(s->ctx, SDBG_EFORMAT, e);
  for (size_t t = 0; t < n_terms; ++t)
    if (terms[t].docs_count && sp.blocks[sp.term_blk_begin[t + 1] - 1].last_doc > s->n_docs)
      return fail(s->ctx, SDBG_EFORMAT, "doc id beyond segment size");
  return upload_postings(s, sp);
}

extern "C" int sdbg_stage_positions(sdbg_segment* s, const uint32_t* positions, const uint64_t* term_pos_off, size_t n_terms) {
  if (!s) return SDBG_EINVAL;
  sdbg_ctx* c = s->ctx;
  if (!s->d_blocks) return fail(c, SDBG_EINVAL, "stage the postings before the positions");
  if (!term_pos_off || n_terms + 1 != s->term_blk_begin.size()) return fail(c, SDBG_EINVAL, "n_terms differs from the staged term count");
  for (size_t t = 0; t < n_terms; ++t)
    if (term_pos_off[t + 1] < term_pos_off[t]) return fail(c, SDBG_EINVAL, "term_pos_off must be non-decreasing");
  const uint64_t n_pos = term_pos_off[n_terms] - term_pos_off[0];
  if (n_pos && !positions) return fail(c, SDBG_EINVAL, "positions is NULL");
  CU(c, cudaSetDevice(c->device));
  const uint64_t nb = s->n_blocks;
  const unsigned grid = unsigned(std::max<uint64_t>(1, (nb * 32 + 255) / 256));
  // per block its frequency sum (device) and its length (descriptors)
  std::vector<unsigned long long> fsum(nb);
  std::vector<BlockDesc> desc(nb);
  DevBuf& b_sum = c->scratch[0];
  if (int rc = ensure(c, b_sum, std::max<uint64_t>(nb, 1) * 8)) return rc;
  if (nb) {
    phrase_freq_sums_kernel<<<grid, 256, 0, c->stream>>>(static_cast<const uint4*>(s->d_arena), static_cast<const uint4*>(s->d_blocks), nb,
                                                         static_cast<unsigned long long*>(b_sum.p));
    ++c->launches;
    CU(c, cudaGetLastError());
    CU(c, cudaMemcpyAsync(fsum.data(), b_sum.p, nb * 8, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaMemcpyAsync(desc.data(), s->d_blocks, nb * sizeof(BlockDesc), cudaMemcpyDeviceToHost, c->stream));
  }
  CU(c, cudaStreamSynchronize(c->stream));
  // src_off: each block's first position in `positions`; base: its region in the arena (prefixes, then positions)
  std::vector<unsigned long long> src_off(std::max<uint64_t>(nb, 1)), base(nb + 1);
  unsigned long long at = 0;
  for (size_t t = 0; t < n_terms; ++t) {
    unsigned long long got = 0;
    for (uint32_t g = s->term_blk_begin[t]; g < s->term_blk_begin[t + 1]; ++g) {
      if (fsum[g] > 0xFFFFFFFFull) return fail(c, SDBG_EFORMAT, "more than 2^32 - 1 positions in one posting block");
      src_off[g] = term_pos_off[t] - term_pos_off[0] + got;
      got += fsum[g];
      base[g] = at;
      at += ((desc[g].packed >> 12) & 127u) + 1u + fsum[g];
    }
    if (got != term_pos_off[t + 1] - term_pos_off[t])
      return fail(c, SDBG_EFORMAT, "a term's position count differs from the sum of its postings' frequencies");
  }
  base[nb] = at;
  void* d_base = nullptr; void* d_pos = nullptr; void* d_src = nullptr; void* d_src_off = nullptr;
  auto cleanup = [&]() { for (void* p : {d_base, d_pos, d_src, d_src_off}) if (p) cudaFree(p); };
  auto run = [&]() -> int {
    CU(c, cudaMalloc(&d_base, (nb + 1) * 8));
    CU(c, cudaMalloc(&d_pos, std::max<unsigned long long>(at, 1) * 4));
    CU(c, cudaMalloc(&d_src, std::max<uint64_t>(n_pos, 1) * 4));
    CU(c, cudaMalloc(&d_src_off, src_off.size() * 8));
    CU(c, cudaMemcpyAsync(d_base, base.data(), (nb + 1) * 8, cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemcpyAsync(d_src_off, src_off.data(), src_off.size() * 8, cudaMemcpyHostToDevice, c->stream));
    if (n_pos) CU(c, cudaMemcpyAsync(d_src, positions + term_pos_off[0], n_pos * 4, cudaMemcpyHostToDevice, c->stream));
    unsigned int* d_bad = static_cast<unsigned int*>(b_sum.p);
    CU(c, cudaMemsetAsync(d_bad, 0, 4, c->stream));
    if (nb) {
      phrase_fill_kernel<<<grid, 256, 0, c->stream>>>(static_cast<const uint4*>(s->d_arena), static_cast<const uint4*>(s->d_blocks), nb,
                                                      static_cast<const unsigned long long*>(d_base),
                                                      static_cast<const unsigned long long*>(d_src_off), static_cast<const uint32_t*>(d_src),
                                                      static_cast<uint32_t*>(d_pos), d_bad);
      ++c->launches;
      CU(c, cudaGetLastError());
    }
    unsigned int bad = 0;
    CU(c, cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    if (bad) return fail(c, SDBG_EFORMAT, "positions do not ascend strictly within a posting");
    return SDBG_OK;
  };
  const int rc = run();
  cudaFree(d_src); cudaFree(d_src_off);
  d_src = d_src_off = nullptr;
  if (rc) { cleanup(); return rc; }
  free_positions(s);
  s->d_pos_base = d_base;
  s->d_pos = d_pos;
  return SDBG_OK;
}

extern "C" int sdbg_stage_norms(sdbg_segment* s, const uint8_t* bytes, size_t n, const sdbg_norm_rg* rgs, size_t n_rg) {
  if (!s || !bytes || !rgs || !n_rg) return SDBG_EINVAL;
  sdbg_ctx* c = s->ctx;
  // Row groups may differ in width (norm_column_reader.hpp:43-48); HBM holds one uniform width per
  // segment (the widest) so a gather is a single indexed load.
  uint32_t width = 1; uint64_t rows = 0;
  for (size_t i = 0; i < n_rg; ++i) {
    if (rgs[i].byte_size != 1 && rgs[i].byte_size != 2 && rgs[i].byte_size != 4) return fail(c, SDBG_EINVAL, "norm width must be 1, 2 or 4");
    if (rgs[i].file_offset + uint64_t(rgs[i].row_count) * rgs[i].byte_size > n) return fail(c, SDBG_EINVAL, "norm row group beyond buffer");
    width = std::max<uint32_t>(width, rgs[i].byte_size);
    rows += rgs[i].row_count;
  }
  if (rows != s->n_docs) return fail(c, SDBG_EINVAL, "norm rows != segment docs");
  std::vector<uint8_t> flat;
  const uint8_t* src = bytes + rgs[0].file_offset;
  if (!(n_rg == 1 && rgs[0].byte_size == width)) {
    flat.resize(rows * width);
    uint64_t r = 0;
    for (size_t i = 0; i < n_rg; ++i)
      for (uint32_t j = 0; j < rgs[i].row_count; ++j, ++r) {
        uint32_t v = 0;
        std::memcpy(&v, bytes + rgs[i].file_offset + size_t(j) * rgs[i].byte_size, rgs[i].byte_size);
        std::memcpy(flat.data() + r * width, &v, width);
      }
    src = flat.data();
  }
  // The average length the writer chose the block-max pairs with: NormReader::GetAvg (norm_reader_impl.hpp:83-88), as
  // PostingWriter computes it. A writer that used another average overrides it with sdbg_segment_set_wand_avg_dl.
  uint64_t sum = 0, nonzero = 0;
  for (uint64_t r = 0; r < rows; ++r) {
    uint32_t v = 0;
    std::memcpy(&v, src + r * width, width);
    sum += v; nonzero += v != 0;
  }
  CU(c, cudaSetDevice(c->device));
  if (s->d_norms) { cudaFree(s->d_norms); s->d_norms = nullptr; }
  CU(c, cudaMalloc(&s->d_norms, rows * width + 16));
  CU(c, cudaMemcpyAsync(s->d_norms, src, rows * width, cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  s->norm_width = width;
  s->wand_avg_dl = nonzero ? float(double(sum) / double(nonzero)) : 0.f;
  return SDBG_OK;
}

namespace {
size_t type_width(int t) { return t == SDBG_I32 ? 4 : 8; }

// ---- bit-packed storage of int64 columns (ColumnObj::d_packed) ----
uint64_t for_groups(uint64_t rows) { return (rows + kForGroupRows - 1) / kForGroupRows; }
size_t for_hdr_bytes(uint64_t rows) { return (for_groups(rows) * sizeof(ForBlockDev) + 255) & ~size_t(255); }
const ForBlockDev* for_headers(const ColumnObj& col) { return static_cast<const ForBlockDev*>(col.d_packed); }
const unsigned long long* for_words(const ColumnObj& col) {
  return reinterpret_cast<const unsigned long long*>(static_cast<const char*>(col.d_packed) + for_hdr_bytes(col.rows));
}
unsigned grid_per_group_warp(sdbg_ctx* c, uint64_t n_groups) {
  return unsigned(std::max<uint64_t>(1, std::min<uint64_t>((n_groups * 32 + 255) / 256, uint64_t(c->sm_count) * 16)));
}
int ensure_zone(sdbg_ctx* c, ColumnObj& col) {
  if (!col.d_zone) CU(c, cudaMalloc(reinterpret_cast<void**>(&col.d_zone), for_groups(col.rows) * 16));
  return SDBG_OK;
}

// Raw values of a column for every reader that does not decode the packed form: a packed column is decoded once and the
// raw view kept until the column is restaged or freed.
int raw_values(sdbg_ctx* c, ColumnObj& col, void** out) {
  if (!col.d_values && col.d_packed) {
    CU(c, cudaMalloc(&col.d_values, col.rows * 8 + 64));
    CU(c, cudaMemsetAsync(static_cast<char*>(col.d_values) + col.rows * 8, 0, 64, c->stream));
    for_unpack_kernel<<<grid_per_group_warp(c, for_groups(col.rows)), 256, 0, c->stream>>>(for_headers(col), for_words(col), col.rows,
                                                                                           static_cast<long long*>(col.d_values));
    ++c->launches;
    CU(c, cudaGetLastError());
  }
  *out = col.d_values;
  return SDBG_OK;
}

// Staging of an owned NOT NULL int64 column: its raw values are in c->stage_raw (rows * 8 bytes + 64 zeroed). Fills the
// zonemap (one pass over the values), then bit-packs the column on the device when that is smaller, else copies the raw
// values into the column. Synchronises the stream once (the packed size decides the layout). A column restaged with the
// same packed size keeps its allocation.
int pack_column(sdbg_ctx* c, ColumnObj& col) {
  const uint64_t rows = col.rows, n_groups = for_groups(rows);
  int rc;
  auto keep_raw = [&]() -> int {
    if (col.d_packed) { cudaFree(col.d_packed); col.d_packed = nullptr; col.packed_bytes = 0; }
    CU(c, cudaMalloc(&col.d_values, rows * 8 + 64));
    CU(c, cudaMemcpyAsync(col.d_values, c->stage_raw.p, rows * 8 + 64, cudaMemcpyDeviceToDevice, c->stream));
    return SDBG_OK;
  };
  if (rows >= (1ull << 32)) return keep_raw();                   // 32-bit word offsets: such a column stays raw
  if ((rc = ensure_zone(c, col))) return rc;
  // scratch: stats headers | word counts [n_groups + 1] | offsets [n_groups + 1] | scan temp
  const size_t h_bytes = (n_groups * sizeof(ForBlockDev) + 255) & ~size_t(255), n_bytes = ((n_groups + 1) * 8 + 255) & ~size_t(255);
  size_t scan_bytes = 0;
  CU(c, cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, static_cast<const unsigned long long*>(nullptr),
                                      static_cast<unsigned long long*>(nullptr), int(n_groups + 1), c->stream));
  if ((rc = ensure(c, c->scratch[12], h_bytes + 2 * n_bytes + scan_bytes))) return rc;
  char* base = static_cast<char*>(c->scratch[12].p);
  auto* s_hdr = reinterpret_cast<ForBlockDev*>(base);
  auto* s_nw = reinterpret_cast<unsigned long long*>(base + h_bytes);
  auto* s_off = reinterpret_cast<unsigned long long*>(base + h_bytes + n_bytes);
  CU(c, cudaMemsetAsync(s_nw + n_groups, 0, 8, c->stream));
  const auto* raw = static_cast<const long long*>(c->stage_raw.p);
  const unsigned grid = grid_per_group_warp(c, n_groups);
  for_stats_kernel<<<grid, 256, 0, c->stream>>>(raw, nullptr, nullptr, rows, col.d_zone, s_hdr, s_nw);
  col.zone_ok = true; col.h_zone.clear();
  ++c->launches;
  CU(c, cudaGetLastError());
  CU(c, cub::DeviceScan::ExclusiveSum(base + h_bytes + 2 * n_bytes, scan_bytes, s_nw, s_off, int(n_groups + 1), c->stream));
  unsigned long long total = 0;
  CU(c, cudaMemcpyAsync(&total, s_off + n_groups, 8, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  const size_t packed_bytes = for_hdr_bytes(rows) + (total + 1) * 8 + 64;   // + the writer's slack word + 64 B of slack
  if (packed_bytes >= rows * 8) return keep_raw();               // not smaller (e.g. full 64-bit hashes): stays raw
  if (col.d_packed && col.packed_bytes != packed_bytes) { cudaFree(col.d_packed); col.d_packed = nullptr; }
  if (!col.d_packed) CU(c, cudaMalloc(&col.d_packed, packed_bytes));
  col.packed_bytes = packed_bytes;
  CU(c, cudaMemsetAsync(static_cast<char*>(col.d_packed) + packed_bytes - 64, 0, 64, c->stream));
  for_pack_kernel<<<grid, 256, 0, c->stream>>>(raw, s_hdr, s_off, rows, static_cast<ForBlockDev*>(col.d_packed),
                                               const_cast<unsigned long long*>(for_words(col)));
  ++c->launches;
  CU(c, cudaGetLastError());
  return SDBG_OK;
}

// Resets `col` for a restaged owned int64 column of `rows` rows. A column of the same length keeps its packed and zonemap
// allocations for pack_column to reuse, so restaging allocates and frees nothing (a cudaFree would wait for the device).
void reset_for_packing(ColumnObj& col, uint64_t rows) {
  void* keep = nullptr;
  long long* zone = nullptr;
  size_t keep_bytes = 0;
  if (col.owned && col.rows == rows) {
    keep = col.d_packed; keep_bytes = col.packed_bytes; zone = col.d_zone;
    col.d_packed = nullptr; col.d_zone = nullptr;
  }
  free_column(col);
  col = ColumnObj{};
  col.type = SDBG_I64; col.rows = rows; col.owned = true;
  col.d_packed = keep; col.packed_bytes = keep_bytes; col.d_zone = zone;
}
}  // namespace

extern "C" int sdbg_stage_column(sdbg_segment* s, uint64_t field, sdbg_type t, const void* values,
                                 const uint64_t* validity, uint64_t rows) {
  if (!s || !values || t < 0 || t > 2) return SDBG_EINVAL;
  sdbg_ctx* c = s->ctx;
  CU(c, cudaSetDevice(c->device));
  ColumnObj& col = s->cols[field];
  const size_t bytes = rows * type_width(t);
  if (t == SDBG_I64 && !validity && rows) {   // NOT NULL int64: packed on the device when that is smaller
    int rc;
    if ((rc = ensure(c, c->stage_raw, bytes + 64))) return rc;
    reset_for_packing(col, rows);
    CU(c, cudaMemsetAsync(static_cast<char*>(c->stage_raw.p) + bytes, 0, 64, c->stream));
    CU(c, cudaMemcpyAsync(c->stage_raw.p, values, bytes, cudaMemcpyHostToDevice, c->stream));
    return pack_column(c, col);
  }
  if (col.d_packed || !(col.owned && col.d_values && col.rows == rows && col.type == t)) {
    free_column(col);
    col = ColumnObj{};
    CU(c, cudaMalloc(&col.d_values, bytes + 64));  // slack: row pairs are loaded as one 16-byte vector
    CU(c, cudaMemsetAsync(static_cast<char*>(col.d_values) + bytes, 0, 64, c->stream));
  }
  col.zone_ok = false; col.h_zone.clear();   // new values: the zonemap is built again on first use (into the same allocation)
  col.type = t; col.rows = rows; col.owned = true; col.has_minmax = false;
  CU(c, cudaMemcpyAsync(col.d_values, values, bytes, cudaMemcpyHostToDevice, c->stream));
  if (validity) {
    const size_t vb = ((rows + 63) / 64) * 8;
    if (!col.d_validity) CU(c, cudaMalloc(reinterpret_cast<void**>(&col.d_validity), vb + 16));
    CU(c, cudaMemcpyAsync(col.d_validity, validity, vb, cudaMemcpyHostToDevice, c->stream));
  } else if (col.d_validity) {
    cudaFree(col.d_validity); col.d_validity = nullptr;
  }
  return SDBG_OK;  // asynchronous on the context stream; consumers run on the same stream
}

// ---- frame-of-reference bit-packed int64 columns (DuckDB's bitpacking codec in FOR mode is this algorithm: per group
// of 2048 values a base and a bit width, formats/column/column_reader.hpp:90-96 ColumnBlockMeta::codec; DuckDB itself is
// not vendored in the reference tree, so the byte layout below is this library's own) ----
static_assert(sizeof(sdbg_for_block) == sizeof(ForBlockDev), "header layout");

extern "C" int sdbg_pack_for(const int64_t* values, uint64_t rows, sdbg_for_block* headers, uint64_t* words, uint64_t cap_words,
                             uint64_t* n_words) {
  if (!values || !headers || !n_words || (cap_words && !words)) return SDBG_EINVAL;
  const uint64_t n_groups = (rows + kForGroupRows - 1) / kForGroupRows;
  // pass 1 (threaded): base = min, bits = width of max - min, word count per group
  const size_t n_thr = std::max<size_t>(1, std::min<size_t>(size_t(env_int("SDBG_HOST_THREADS", 16)), n_groups / 64 + 1));
  auto stats = [&](uint64_t g0, uint64_t g1) {
    for (uint64_t g = g0; g < g1; ++g) {
      const uint64_t r0 = g * kForGroupRows, r1 = std::min<uint64_t>(rows, r0 + kForGroupRows);
      int64_t mn = values[r0], mx = values[r0];
      for (uint64_t r = r0 + 1; r < r1; ++r) { mn = std::min(mn, values[r]); mx = std::max(mx, values[r]); }
      const uint64_t span = uint64_t(mx) - uint64_t(mn);
      headers[g].base = mn;
      headers[g].bits = span == 0 ? 0u : uint32_t(64 - __builtin_clzll(span));
    }
  };
  {
    std::vector<std::thread> pool;
    for (size_t t = 0; t < n_thr; ++t) pool.emplace_back(stats, n_groups * t / n_thr, n_groups * (t + 1) / n_thr);
    for (auto& th : pool) th.join();
  }
  uint64_t off = 0;
  for (uint64_t g = 0; g < n_groups; ++g) {
    const uint64_t n = std::min<uint64_t>(kForGroupRows, rows - g * kForGroupRows);
    if (off > 0xFFFFFFFFull) return SDBG_EUNSUPPORTED;            // 32-bit word offsets: 32 GiB of packed data per column
    headers[g].off8 = uint32_t(off);
    off += (n * headers[g].bits + 63) / 64;
  }
  *n_words = off + 1;                                             // one word of slack: the decoder may read one past a value
  if (*n_words > cap_words) return SDBG_ECAPACITY;
  auto pack = [&](uint64_t g0, uint64_t g1) {
    for (uint64_t g = g0; g < g1; ++g) {
      const uint32_t bits = headers[g].bits;
      if (!bits) continue;
      const uint64_t r0 = g * kForGroupRows, n = std::min<uint64_t>(kForGroupRows, rows - r0);
      uint64_t* w = words + headers[g].off8;
      const uint64_t nw = (n * bits + 63) / 64;
      std::fill(w, w + nw, 0ull);
      const uint64_t base = uint64_t(headers[g].base);
      for (uint64_t i = 0; i < n; ++i) {
        const uint64_t v = uint64_t(values[r0 + i]) - base, bit = i * bits;
        w[bit >> 6] |= v << (bit & 63);
        if ((bit & 63) + bits > 64) w[(bit >> 6) + 1] |= v >> (64 - (bit & 63));
      }
    }
  };
  {
    std::vector<std::thread> pool;
    for (size_t t = 0; t < n_thr; ++t) pool.emplace_back(pack, n_groups * t / n_thr, n_groups * (t + 1) / n_thr);
    for (auto& th : pool) th.join();
  }
  words[off] = 0;
  return SDBG_OK;
}

extern "C" int sdbg_stage_column_for(sdbg_segment* s, uint64_t field, const sdbg_for_block* headers, const uint64_t* words,
                                     uint64_t n_words, uint64_t rows) {
  if (!s || !headers || !words || !rows || !n_words) return SDBG_EINVAL;
  sdbg_ctx* c = s->ctx;
  CU(c, cudaSetDevice(c->device));
  const uint64_t n_groups = (rows + kForGroupRows - 1) / kForGroupRows;
  for (uint64_t g = 0; g < n_groups; ++g) {                       // the stream is untrusted input: every group must lie inside it
    const uint64_t n = std::min<uint64_t>(kForGroupRows, rows - g * kForGroupRows);
    if (headers[g].bits > 64u || uint64_t(headers[g].off8) + (n * headers[g].bits + 63) / 64 + 1 > n_words)
      return fail(c, SDBG_EFORMAT, "bit-packed column: group outside the word stream");
  }
  ColumnObj& col = s->cols[field];
  const size_t bytes = rows * 8;
  // The caller's stream is kept as the column's storage when every group starts 16-byte aligned (what sdbg_pack_for
  // writes) and it is smaller than the raw column; otherwise it is decoded to raw values.
  bool aligned = rows < (1ull << 32);
  for (uint64_t g = 0; g < n_groups && aligned; ++g) aligned = (headers[g].off8 & 1u) == 0u;
  const size_t packed_bytes = for_hdr_bytes(rows) + n_words * 8 + 64;
  if (aligned && packed_bytes < bytes) {
    if (!(col.d_packed && col.packed_bytes == packed_bytes && col.rows == rows && !col.d_values && col.d_zone)) {   // else: same shape, reused
      free_column(col);
      col = ColumnObj{};
      col.rows = rows; col.packed_bytes = packed_bytes;
      CU(c, cudaMalloc(&col.d_packed, packed_bytes));
    }
    col.type = SDBG_I64; col.rows = rows; col.owned = true; col.has_minmax = false;
    CU(c, cudaMemcpyAsync(col.d_packed, headers, n_groups * sizeof(ForBlockDev), cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemcpyAsync(const_cast<unsigned long long*>(for_words(col)), words, n_words * 8, cudaMemcpyHostToDevice, c->stream));
    CU(c, cudaMemsetAsync(static_cast<char*>(col.d_packed) + packed_bytes - 64, 0, 64, c->stream));
    { int rc = ensure_zone(c, col); if (rc) return rc; }
    col.zone_ok = true; col.h_zone.clear();
    for_stats_kernel<<<grid_per_group_warp(c, n_groups), 256, 0, c->stream>>>(nullptr, for_headers(col), for_words(col), rows, col.d_zone,
                                                                              nullptr, nullptr);
    ++c->launches;
    CU(c, cudaGetLastError());
    return SDBG_OK;   // asynchronous on the context stream, like sdbg_stage_column
  }
  if (col.d_packed || !(col.owned && col.d_values && col.rows == rows && col.type == SDBG_I64)) {
    free_column(col);
    col = ColumnObj{};
    CU(c, cudaMalloc(&col.d_values, bytes + 64));
    CU(c, cudaMemsetAsync(static_cast<char*>(col.d_values) + bytes, 0, 64, c->stream));
  }
  if (col.d_validity) { cudaFree(col.d_validity); col.d_validity = nullptr; }
  col.type = SDBG_I64; col.rows = rows; col.owned = true; col.has_minmax = false;
  col.zone_ok = false; col.h_zone.clear();
  DevBuf& buf = c->scratch[12];
  const size_t hdr_bytes = (n_groups * sizeof(ForBlockDev) + 255) & ~size_t(255);
  int rc = ensure(c, buf, hdr_bytes + n_words * 8);
  if (rc) return rc;
  char* base = static_cast<char*>(buf.p);
  CU(c, cudaMemcpyAsync(base, headers, n_groups * sizeof(ForBlockDev), cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaMemcpyAsync(base + hdr_bytes, words, n_words * 8, cudaMemcpyHostToDevice, c->stream));
  const unsigned grid = unsigned(std::min<uint64_t>((n_groups * 32 + 255) / 256, uint64_t(c->sm_count) * 16));
  for_unpack_kernel<<<std::max(grid, 1u), 256, 0, c->stream>>>(reinterpret_cast<const ForBlockDev*>(base),
                                                               reinterpret_cast<const unsigned long long*>(base + hdr_bytes), rows,
                                                               static_cast<long long*>(col.d_values));
  ++c->launches;
  CU(c, cudaGetLastError());
  return SDBG_OK;   // asynchronous on the context stream, like sdbg_stage_column
}

extern "C" int sdbg_stage_column_device(sdbg_segment* s, uint64_t field, sdbg_type t, const void* d_values, uint64_t rows) {
  if (!s || !d_values || t < 0 || t > 2) return SDBG_EINVAL;
  if (rows & 1) return fail(s->ctx, SDBG_EINVAL, "borrowed device columns need an even row count (16-byte row pairs)");
  ColumnObj& col = s->cols[field];
  free_column(col);
  col = ColumnObj{};
  col.d_values = const_cast<void*>(d_values); col.type = t; col.rows = rows; col.owned = false;
  return SDBG_OK;
}

extern "C" int sdbg_column_device_ptr(sdbg_segment* s, uint64_t field, void** d_values, uint64_t* rows) {
  if (!s) return SDBG_EINVAL;
  auto it = s->cols.find(field);
  if (it == s->cols.end()) return fail(s->ctx, SDBG_ENOTFOUND, "unknown column");
  CU(s->ctx, cudaSetDevice(s->ctx->device));
  ColumnObj& col = it->second;
  void* p = nullptr;
  const int rc = raw_values(s->ctx, col, &p);
  if (rc) return rc;
  // The caller is about to write the values: every statistic of the old ones is dropped, and a packed column becomes
  // its raw view (the packed words would keep the old values) until it is restaged.
  if (col.d_packed) {
    CU(s->ctx, cudaStreamSynchronize(s->ctx->stream));   // queued readers of the packed words finish first
    cudaFree(col.d_packed);
    col.d_packed = nullptr; col.packed_bytes = 0;
  }
  col.has_minmax = false; col.zone_ok = false; col.h_zone.clear();
  if (d_values) *d_values = p;
  if (rows) *rows = it->second.rows;
  return SDBG_OK;
}

extern "C" int sdbg_column_for_to_host(sdbg_segment* s, uint64_t field, sdbg_for_block* headers, uint64_t* words, uint64_t cap_words,
                                       uint64_t* n_words) {
  if (!s || !n_words) return SDBG_EINVAL;
  auto it = s->cols.find(field);
  if (it == s->cols.end()) return fail(s->ctx, SDBG_ENOTFOUND, "unknown column");
  const ColumnObj& col = it->second;
  *n_words = 0;
  if (!col.d_packed) return SDBG_OK;                             // held raw
  const uint64_t n = (col.packed_bytes - for_hdr_bytes(col.rows) - 64) / 8;
  *n_words = n;
  if (n > cap_words || !headers || !words) return SDBG_ECAPACITY;
  sdbg_ctx* c = s->ctx;
  CU(c, cudaSetDevice(c->device));
  CU(c, cudaMemcpyAsync(headers, col.d_packed, for_groups(col.rows) * sizeof(ForBlockDev), cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaMemcpyAsync(words, for_words(col), n * 8, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  return SDBG_OK;
}

extern "C" int sdbg_column_to_host(sdbg_segment* s, uint64_t field, void* host_dst, uint64_t rows) {
  if (!s || !host_dst) return SDBG_EINVAL;
  auto it = s->cols.find(field);
  if (it == s->cols.end()) return fail(s->ctx, SDBG_ENOTFOUND, "unknown column");
  if (rows > it->second.rows) return fail(s->ctx, SDBG_EINVAL, "more rows requested than staged");
  sdbg_ctx* c = s->ctx;
  CU(c, cudaSetDevice(c->device));
  void* src = nullptr;
  const int rc = raw_values(c, it->second, &src);
  if (rc) return rc;
  CU(c, cudaMemcpyAsync(host_dst, src, rows * type_width(it->second.type), cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  return SDBG_OK;
}

// Values of one column for a set of hit docs (late materialisation: HitBatcher::MaterializeColumn, hit_batcher.hpp:39;
// FinalizeBatch in duckdb_search_full_scan.cpp fetches the projected columns for the emitted doc ids only).
extern "C" int sdbg_gather_column(sdbg_segment* s, uint64_t field, const uint32_t* docs, size_t n, void* out_values, uint8_t* out_valid) {
  if (!s || (n && (!docs || !out_values))) return SDBG_EINVAL;
  sdbg_ctx* c = s->ctx;
  auto it = s->cols.find(field);
  if (it == s->cols.end()) return fail(c, SDBG_ENOTFOUND, "unknown column");
  if (!n) return SDBG_OK;
  CU(c, cudaSetDevice(c->device));
  ColumnObj& co = it->second;
  void* raw = nullptr;
  int rc = raw_values(c, co, &raw);
  if (rc) return rc;
  const size_t w = type_width(co.type);
  const size_t docs_bytes = (n * 4 + 255) & ~size_t(255), val_bytes = (n * w + 255) & ~size_t(255);
  DevBuf& buf = c->scratch[12];
  if ((rc = ensure(c, buf, docs_bytes + val_bytes + n))) return rc;
  char* base = static_cast<char*>(buf.p);
  auto* d_docs = reinterpret_cast<uint32_t*>(base);
  void* d_out = base + docs_bytes;
  auto* d_valid = reinterpret_cast<unsigned char*>(base + docs_bytes + val_bytes);
  CU(c, cudaMemcpyAsync(d_docs, docs, n * 4, cudaMemcpyHostToDevice, c->stream));
  const unsigned grid = unsigned(std::min<size_t>((n + 255) / 256, size_t(c->sm_count) * 8));
  const auto* valid = reinterpret_cast<const unsigned long long*>(co.d_validity);
  if (w == 4) gather_rows_kernel<uint32_t><<<grid, 256, 0, c->stream>>>(static_cast<const uint32_t*>(raw), valid, d_docs, n, co.rows, static_cast<uint32_t*>(d_out), out_valid ? d_valid : nullptr);
  else gather_rows_kernel<unsigned long long><<<grid, 256, 0, c->stream>>>(static_cast<const unsigned long long*>(raw), valid, d_docs, n, co.rows, static_cast<unsigned long long*>(d_out), out_valid ? d_valid : nullptr);
  ++c->launches;
  CU(c, cudaGetLastError());
  CU(c, cudaMemcpyAsync(out_values, d_out, n * w, cudaMemcpyDeviceToHost, c->stream));
  if (out_valid) CU(c, cudaMemcpyAsync(out_valid, d_valid, n, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  return SDBG_OK;
}

extern "C" int sdbg_segment_posting_stats(const sdbg_segment* s, uint64_t* payload_bytes, uint64_t* table_bytes,
                                          uint64_t* n_blocks, uint64_t* n_postings) {
  if (!s) return SDBG_EINVAL;
  if (payload_bytes) *payload_bytes = s->arena_bytes;
  if (table_bytes) *table_bytes = s->n_blocks * (sizeof(BlockDesc) + sizeof(MaxPair));
  if (n_blocks) *n_blocks = s->n_blocks;
  if (n_postings) *n_postings = s->n_postings;
  return SDBG_OK;
}

extern "C" int sdbg_segment_term_bytes(const sdbg_segment* s, uint64_t* bytes_out, size_t n_terms) {
  if (!s || !bytes_out || n_terms > s->term_bytes.size()) return SDBG_EINVAL;
  std::copy(s->term_bytes.begin(), s->term_bytes.begin() + long(n_terms), bytes_out);
  return SDBG_OK;
}

// ------------------------------------------------------------------------------------------
// Pushed predicates: the constant resolved against the column's type before any kernel sees it
// ------------------------------------------------------------------------------------------
namespace {

constexpr double kTwo63 = 9223372036854775808.0;   // 2^63, the first double above INT64_MAX

// Smallest int64 v with v >= x (strict: v > x); false when no int64 qualifies (x NaN or beyond INT64_MAX).
bool int_lower_bound(double x, bool strict, int64_t* v) {
  if (std::isnan(x)) return false;
  const double c = strict ? std::floor(x) : std::ceil(x);
  if (c >= kTwo63) return false;
  if (c < -kTwo63) { *v = INT64_MIN; return true; }
  *v = static_cast<int64_t>(c) + (strict ? 1 : 0);   // c <= 2^63 - 1024 here (doubles below 2^63 step by 1024): no overflow
  return true;
}
// Largest int64 v with v <= x (strict: v < x); false when no int64 qualifies (x NaN or below INT64_MIN).
bool int_upper_bound(double x, bool strict, int64_t* v) {
  if (std::isnan(x)) return false;
  const double c = strict ? std::ceil(x) : std::floor(x);
  if (strict ? c <= -kTwo63 : c < -kTwo63) return false;
  if (c >= kTwo63) { *v = INT64_MAX; return true; }
  *v = static_cast<int64_t>(c) - (strict ? 1 : 0);
  return true;
}

}  // namespace

extern "C" int sdbg_col_pred_resolve(const sdbg_col_pred* in, int type, sdbg_col_pred* out) {
  if (!in || !out || in->op < SDBG_OP_LT || in->op > SDBG_OP_IS_NOT_NULL || type < SDBG_I64 || type > SDBG_I32) return SDBG_EINVAL;
  sdbg_col_pred p = *in;
  const bool compares = p.op < SDBG_OP_IS_NULL;
  if (compares && type == SDBG_F64 && !p.is_float) {
    p.lo_f = static_cast<double>(p.lo_i); p.hi_f = static_cast<double>(p.hi_i); p.is_float = 1;   // rounded to nearest
  } else if (compares && type != SDBG_F64 && p.is_float) {
    int64_t lo = INT64_MIN, hi = INT64_MAX;
    bool some = true;
    const double x = p.lo_f;
    switch (p.op) {
      case SDBG_OP_LT: some = int_upper_bound(x, true, &hi); break;
      case SDBG_OP_LE: some = int_upper_bound(x, false, &hi); break;
      case SDBG_OP_GT: some = int_lower_bound(x, true, &lo); break;
      case SDBG_OP_GE: some = int_lower_bound(x, false, &lo); break;
      case SDBG_OP_EQ: some = int_lower_bound(x, false, &lo) && int_upper_bound(x, false, &hi); break;
      case SDBG_OP_NE:
        if (int_lower_bound(x, false, &lo) && int_upper_bound(x, false, &hi) && lo == hi) {   // an int64 value: stays <>
          p.lo_i = lo; p.is_float = 0;
          *out = p;
          return SDBG_OK;
        }
        lo = INT64_MIN; hi = INT64_MAX;   // NaN, fractional or outside int64: every non-NULL row
        break;
      default: some = int_lower_bound(x, false, &lo) && int_upper_bound(p.hi_f, false, &hi); break;
    }
    if (!some) { lo = INT64_MAX; hi = INT64_MIN; }
    p.op = SDBG_OP_BETWEEN; p.is_float = 0; p.lo_i = lo; p.hi_i = hi;
  }
  *out = p;
  return SDBG_OK;
}

// ------------------------------------------------------------------------------------------
// BM25 top-k
// ------------------------------------------------------------------------------------------
namespace {

PostingsDev postings_view(const sdbg_segment* s, uint32_t ordinal_base) {
  PostingsDev p;
  p.arena = static_cast<const uint4*>(s->d_arena);
  p.blocks = static_cast<const uint4*>(s->d_blocks);
  p.blk_max = static_cast<const uint2*>(s->d_blkmax);
  p.anchors = static_cast<const uint4*>(s->d_anchor);
  p.norms = static_cast<const uint8_t*>(s->d_norms);
  p.norm_width = s->norm_width;
  p.deleted = static_cast<const uint32_t*>(s->d_deleted);
  p.n_docs = s->n_docs;
  p.ordinal_base = ordinal_base;
  return p;
}

// packed_ok: a packed column is described as {values = its d_packed block, type = kTypeFor} (for the TMA GROUP BY);
// otherwise every column is described by its raw values.
int col_view(sdbg_segment* s, uint64_t field, ColDev* out, uint64_t* rows, bool packed_ok = false) {
  auto it = s->cols.find(field);
  if (it == s->cols.end()) return fail(s->ctx, SDBG_ENOTFOUND, "column " + std::to_string(field) + " not staged");
  ColumnObj& col = it->second;
  out->validity = col.d_validity; out->type = col.type; out->pad = 0;
  if (packed_ok && col.d_packed) { out->values = col.d_packed; out->type = kTypeFor; }
  else { const int rc = raw_values(s->ctx, col, const_cast<void**>(&out->values)); if (rc) return rc; }
  if (rows) *rows = col.rows;
  return SDBG_OK;
}

// One pushed predicate on segment s: its column's view (col_view) and its constants resolved against the column's type.
// *rows: the column's length.
int pred_dev(sdbg_segment* s, const sdbg_col_pred& in, PredDev* out, uint64_t* rows, bool packed_ok = false) {
  if (int rc = col_view(s, in.field, &out->col, rows, packed_ok)) return rc;
  sdbg_col_pred p;
  const int type = out->col.type == kTypeFor ? SDBG_I64 : out->col.type;   // a packed column holds int64
  if (sdbg_col_pred_resolve(&in, type, &p)) return fail(s->ctx, SDBG_EINVAL, "bad predicate op");
  out->op = p.op; out->pad = 0;
  out->lo_i = p.lo_i; out->hi_i = p.hi_i;
  out->lo_f = p.lo_f; out->hi_f = p.hi_f;
  return SDBG_OK;
}

// Rewrites a resolved comparison as the per-doc test of the full-text kernels takes it (pred1): `lo <= v <= hi`
// (SDBG_OP_BETWEEN; lo > hi: no row), or its negation for SQL <> (SDBG_OP_NE, lo == hi). Exact: integers step by 1 and
// doubles by one ulp; NaN bounds hold for no row, so `<> NaN` holds for every non-NULL row. Keeps the per-doc code one
// range test whatever the op.
void between_form(PredDev& p) {
  if (p.op == SDBG_OP_BETWEEN || p.op >= SDBG_OP_IS_NULL) return;
  if (p.col.type == SDBG_F64) {
    const double x = p.lo_f;
    double lo = -HUGE_VAL, hi = HUGE_VAL;
    switch (p.op) {
      case SDBG_OP_LT: if (x == -HUGE_VAL) lo = 1.0, hi = 0.0; else hi = std::nextafter(x, -HUGE_VAL); break;
      case SDBG_OP_LE: hi = x; break;
      case SDBG_OP_GT: if (x == HUGE_VAL) lo = 1.0, hi = 0.0; else lo = std::nextafter(x, HUGE_VAL); break;
      case SDBG_OP_GE: lo = x; break;
      default: lo = hi = x; break;   // = and <>
    }
    p.lo_f = lo; p.hi_f = hi;
  } else {
    const int64_t x = p.lo_i;
    int64_t lo = INT64_MIN, hi = INT64_MAX;
    switch (p.op) {
      case SDBG_OP_LT: if (x == INT64_MIN) lo = 1, hi = 0; else hi = x - 1; break;
      case SDBG_OP_LE: hi = x; break;
      case SDBG_OP_GT: if (x == INT64_MAX) lo = 1, hi = 0; else lo = x + 1; break;
      case SDBG_OP_GE: lo = x; break;
      default: lo = hi = x; break;
    }
    p.lo_i = lo; p.hi_i = hi;
  }
  if (p.op != SDBG_OP_NE) p.op = SDBG_OP_BETWEEN;
}

// The filter chain `f` of a full-text entry over segment s (sdbg.h, SDBG_OP_AND_NEXT): at most kMaxPreds predicates,
// each on a column of at least n_docs rows. Only reads and checks; the zone verdicts come from chain_verdicts.
int filter_view(sdbg_segment* s, const sdbg_col_pred* f, ChainDev* out) {
  std::memset(out, 0, sizeof *out);
  if (!f) return SDBG_OK;
  int n = 1;
  while (f[n - 1].op & SDBG_OP_AND_NEXT) {
    if (n == kMaxPreds) return fail(s->ctx, SDBG_EUNSUPPORTED, "a filter chain holds at most 4 predicates");
    ++n;
  }
  out->ps.n = n;
  for (int i = 0; i < n; ++i) {
    sdbg_col_pred p = f[i];
    p.op &= ~SDBG_OP_AND_NEXT;
    uint64_t rows = 0;
    if (int rc = pred_dev(s, p, &out->ps.p[i], &rows)) return rc;
    if (rows < s->n_docs) return fail(s->ctx, SDBG_EINVAL, "filter column shorter than segment");
    between_form(out->ps.p[i]);
  }
  return SDBG_OK;
}

// The zonemap of a NOT NULL column ({min, max} per kZoneRows rows in predicate key space), built on first use and kept
// until the values change (restaging, sdbg_column_device_ptr).
int column_zonemap(sdbg_ctx* c, ColumnObj& col, const long long** out) {
  if (!col.zone_ok) {
    void* raw = nullptr;
    if (int rc = raw_values(c, col, &raw)) return rc;
    if (int rc = ensure_zone(c, col)) return rc;
    const uint64_t n_zones = (col.rows + kZoneRows - 1) / kZoneRows;
    const unsigned zg = unsigned(std::min<uint64_t>((n_zones + 7) / 8, uint64_t(c->sm_count) * 8));
    const auto* vals = static_cast<const unsigned char*>(raw);
    if (col.type == SDBG_F64) zonemap_kernel<1><<<zg, 256, 0, c->stream>>>(vals, col.rows, col.d_zone);
    else if (col.type == SDBG_I32) zonemap_kernel<2><<<zg, 256, 0, c->stream>>>(vals, col.rows, col.d_zone);
    else zonemap_kernel<0><<<zg, 256, 0, c->stream>>>(vals, col.rows, col.d_zone);
    ++c->launches;
    CU(c, cudaGetLastError());
    col.zone_ok = true; col.h_zone.clear();
  }
  *out = col.d_zone;
  return SDBG_OK;
}

// Host copy of a NOT NULL column's zonemap (column_zonemap), fetched once per version of the values: one wait for the
// stream, on first use only.
int column_zonemap_host(sdbg_ctx* c, ColumnObj& col, const std::vector<long long>** out) {
  if (col.h_zone.empty()) {
    const long long* d = nullptr;
    if (int rc = column_zonemap(c, col, &d)) return rc;
    std::vector<long long> h(2 * ((col.rows + kZoneRows - 1) / kZoneRows));
    CU(c, cudaMemcpyAsync(h.data(), d, h.size() * 8, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    col.h_zone = std::move(h);
  }
  *out = &col.h_zone;
  return SDBG_OK;
}

// A resolved comparison (op < SDBG_OP_IS_NULL) as a closed range [*lo, *lo + *span] in the int64 key space of the
// zonemaps (integers as they are, doubles through fkey()), from its between_form. *neg = 1 for SQL <>, which holds
// outside the range. kKeyAll: the comparison holds for every non-NULL row; kKeyNone: for none.
enum KeyRange { kKeyRange, kKeyAll, kKeyNone };
KeyRange key_range(const PredDev& in, int64_t* lo, uint64_t* span, int* neg) {
  PredDev pd = in;
  between_form(pd);
  *neg = pd.op == SDBG_OP_NE ? 1 : 0;
  int64_t l, h;
  if (pd.col.type == SDBG_F64) {
    double lf = pd.lo_f, hf = pd.hi_f;
    if (std::isnan(lf) || std::isnan(hf) || lf > hf) return *neg ? kKeyAll : kKeyNone;   // comparisons with NaN are false
    if (lf == 0.0) lf = -0.0;                                      // -0.0 == +0.0: the range must cover both keys
    if (hf == 0.0) hf = 0.0;
    int64_t bl, bh; std::memcpy(&bl, &lf, 8); std::memcpy(&bh, &hf, 8);
    l = fkey(bl); h = fkey(bh);
  } else {
    l = pd.lo_i; h = pd.hi_i;
    if (l > h) return *neg ? kKeyAll : kKeyNone;
  }
  *lo = l; *span = static_cast<uint64_t>(h) - static_cast<uint64_t>(l);
  return kKeyRange;
}

// Queues the zone verdicts of segment s's chain f (filter_view of `filt`): one verdict byte per kZoneRows-row zone, in
// s->verdict. A predicate on a nullable column decides no zone; IS NULL / IS NOT NULL on a NOT NULL column holds for no
// row / every row. Whether any zone is decided is known on the host from the zonemaps' host copies: when none is,
// f->zone stays null and nothing is queued, so the per-doc kernels (top-k, scan) test nothing but the chain.
int chain_verdicts(sdbg_segment* s, const sdbg_col_pred* filt, ChainDev* f) {
  sdbg_ctx* c = s->ctx;
  const uint64_t n_zones = (uint64_t(s->n_docs) + kZoneRows - 1) / kZoneRows;
  if (!f->ps.n || !n_zones) return SDBG_OK;
  ZoneVerdictParams Z;
  std::memset(&Z, 0, sizeof Z);
  Z.n_blocks = n_zones;
  Z.pass = 1;
  const long long* hz[kMaxPreds] = {};
  bool never = false;
  for (int i = 0; i < f->ps.n && !never; ++i) {
    const PredDev& pd = f->ps.p[i];
    ColumnObj& col = s->cols.find(filt[i].field)->second;
    if (col.d_validity) { Z.pass = 0; continue; }
    if (pd.op == SDBG_OP_IS_NULL) { never = true; continue; }
    if (pd.op == SDBG_OP_IS_NOT_NULL) continue;
    int64_t lo = 0; uint64_t span = 0; int neg = 0;
    const KeyRange kr = key_range(pd, &lo, &span, &neg);
    if (kr == kKeyAll) continue;
    if (kr == kKeyNone) { never = true; continue; }
    const int k = Z.n_preds++;
    if (int rc = column_zonemap(c, col, &Z.zone[k])) return rc;
    const std::vector<long long>* h = nullptr;
    if (int rc = column_zonemap_host(c, col, &h)) return rc;
    hz[k] = h->data();
    Z.lo[k] = lo; Z.span[k] = span; Z.negate[k] = neg;
  }
  bool decided = never || (Z.pass && !Z.n_preds);   // some predicate holds for no row, or every one for every row
  for (uint64_t z = 0; z < n_zones && !decided; ++z) decided = zone_verdict(Z, hz, z) != kZoneCheck;
  if (!decided) return SDBG_OK;
  if (int rc = ensure(c, s->verdict, n_zones)) return rc;
  auto* v = static_cast<uint8_t*>(s->verdict.p);
  f->zone = v; f->n_zones = uint32_t(n_zones);
  if (never || !Z.n_preds) {
    CU(c, cudaMemsetAsync(v, never ? kZoneDead : kZonePass, n_zones, c->stream));
    return SDBG_OK;
  }
  const unsigned vg = unsigned(std::min<uint64_t>((n_zones + 255) / 256, uint64_t(c->sm_count) * 4));
  zone_verdict_kernel<<<vg, 256, 0, c->stream>>>(Z, v, nullptr);
  ++c->launches;
  CU(c, cudaGetLastError());
  return SDBG_OK;
}

// The filter chains of a call's segments with their zone verdicts (out[n_segs]).
int filter_chains(sdbg_segment* const* segs, size_t n_segs, const sdbg_col_pred* filt, ChainDev* out) {
  for (size_t si = 0; si < n_segs; ++si) {
    if (int rc = filter_view(segs[si], filt, &out[si])) return rc;
    if (int rc = chain_verdicts(segs[si], filt, &out[si])) return rc;
  }
  return SDBG_OK;
}

constexpr int kMaxCopyEvents = 16;
constexpr float kTfidfK1 = -1.f;   // internal selector of the TFIDF scorer (it has no k / b): see sdbg_tfidf_topk_batch

// norm_const / norm_length that turn the segment's block-max pairs into upper bounds for a query whose BM25 constants
// are nc = k - k*b and nl = k*b / A_q (A_q: the corpus-wide average length). The writer kept the pair (f*, n*) with the
// largest f / ((1-b) A_s + b n) under the segment's own average A_s. With M = max(A_q, A_s), every posting of the block
// scores at most the BM25 form at (f*, n*) with nc_b = k (1-b) A_s / M and nl_b = k b / M. In terms of nl and
// nl_s = k b / A_s: nl_b = min(nl, nl_s) and nc_b = nc * min(1, nl / nl_s). When A_s == A_q these are the query's own
// constants, bit for bit; only BM25-form queries prune, so only they use the result.
void bound_consts(const sdbg_segment* s, float k1, float b, float nc, float nl, float& bnc, float& bnl) {
  bnc = nc; bnl = nl;
  if (!(s->wand_avg_dl > 0.f)) return;        // no norms: every norm is 1 and the pair order cannot depend on A_s
  const float nl_s = (k1 * b) / s->wand_avg_dl;
  if (nl < nl_s) bnc = nc * (nl / nl_s);       // A_q > A_s
  else bnl = nl_s;                             // A_q <= A_s
}

// Device-side descriptor of one query term over one segment (the caller has checked the term id).
void fill_qterm(const sdbg_segment* s, const sdbg_bm25_term& t, float k1, float b, QTermDev& d) {
  d.blk_begin = s->term_blk_begin[t.term];
  d.nblk = s->term_blk_begin[t.term + 1] - d.blk_begin;
  d.c0 = t.boost * (k1 + 1) * t.idf;  // bm25.cpp:224
  d.norm_const = t.norm_const; d.norm_length = t.norm_length;
  if (k1 == kTfidfK1) {                                                  // TFIDF (tfidf.cpp:59-80, 101): c0 = boost * idf
    d.c0 = t.boost * t.idf;
    d.norm_const = std::numeric_limits<float>::quiet_NaN();               // device-side marker, see bm25()
    d.norm_length = b != 0.f ? 1.f : 0.f;                                 // normalised by sqrt(doc length) or not
  }
  else if (k1 == 0.f) d.c0 = 0.f;                                       // BM1: Bm1Score without a filter boost scores 0 (bm25.cpp:118-126)
  else if (b == 0.f) d.norm_length = std::numeric_limits<float>::quiet_NaN();   // BM15 form (device-side marker, see bm25())
  d.bound_const = d.norm_const; d.bound_length = d.norm_length;
  if (k1 != kTfidfK1 && k1 != 0.f && b != 0.f) bound_consts(s, k1, b, d.norm_const, d.norm_length, d.bound_const, d.bound_length);
  d.docs_count = s->term_docs[t.term];
  d.root_freq = s->term_max[t.term].freq & 0x7FFFFFFFu; d.root_norm = s->term_max[t.term].norm;
  if (t.term < s->term_probe.size() && s->term_probe[t.term]) d.root_freq |= 0x80000000u;   // probe-friendly list (driver mode)
}

// Device-side {first BlockDesc, blocks} of an excluded term in a segment: a term id the segment does not hold is an empty
// list, which excludes nothing.
uint2 excl_list(const sdbg_segment* s, uint32_t term) {
  if (size_t(term) + 1 >= s->term_blk_begin.size()) return make_uint2(0u, 0u);
  return make_uint2(s->term_blk_begin[term], s->term_blk_begin[term + 1] - s->term_blk_begin[term]);
}

// The instantiation of a top-k kernel family for a run-time term count T = 1..4. Conjunctions and lead mode stream one
// list (T = 1) and probe the others.
using TopkKernel = void (*)(TopkParams);
TopkKernel merge_kernel(uint32_t T) {
  switch (T) {
    case 1: return bm25_merge_kernel<1>;
    case 2: return bm25_merge_kernel<2>;
    case 3: return bm25_merge_kernel<3>;
    default: return bm25_merge_kernel<4>;
  }
}
template <int kMode, bool kExcl = false, bool kGroups = false>
TopkKernel stream_kernel(uint32_t T) {
  if constexpr (kMode != kModeOr) {
    return bm25_stream_kernel<1, kMode, kExcl>;
  } else {
    switch (T) {
      case 1: return bm25_stream_kernel<1, kModeOr, kExcl, kGroups>;
      case 2: return bm25_stream_kernel<2, kModeOr, kExcl, kGroups>;
      case 3: return bm25_stream_kernel<3, kModeOr, kExcl, kGroups>;
      default: return bm25_stream_kernel<4, kModeOr, kExcl, kGroups>;
    }
  }
}

// Dynamic shared memory of bm25_stream_kernel: candidates | per warp T live blocks with their prefetch slots, plus the
// probe ring when lists are probed (conjunctions, lead mode).
size_t stream_smem(uint32_t cap, uint32_t T, bool probe_rest) {
  return size_t(cap) * 8 + size_t(kTopkWarps) * (T * kStreamTermBytes + (probe_rest ? 1024 : 0));
}

// Lets every top-k kernel use 200 KB of dynamic shared memory; once per context.
int topk_smem_attrs(sdbg_ctx* c) {
  if (c->topk_attr_set) return SDBG_OK;
  auto set = [](TopkKernel k) { return cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); };
  for (uint32_t T = 1; T <= kStreamMaxTerms; ++T) {
    CU(c, set(merge_kernel(T)));
    CU(c, set(stream_kernel<kModeOr>(T)));
    CU(c, set(stream_kernel<kModeOr, true>(T)));
    CU(c, set(stream_kernel<kModeOr, true, true>(T)));
  }
  CU(c, set(stream_kernel<kModeAnd>(1)));
  CU(c, set(stream_kernel<kModeAnd, true>(1)));
  CU(c, set(stream_kernel<kModeLead>(1)));
  CU(c, set(bm25_topk_kernel<false>));
  CU(c, set(bm25_topk_kernel<true>));
  CU(c, set(bm25_topk_kernel<false, true>));
  CU(c, set(bm25_topk_kernel<true, true>));
  CU(c, set(bm25_topk_kernel<false, true, true>));
  CU(c, set(bm25_topk_kernel<true, true, true>));
  CU(c, cudaFuncSetAttribute(topk_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  c->topk_attr_set = true;
  return SDBG_OK;
}

struct TopkPlan {
  uint32_t G, cap, k;
  size_t smem;
};

// Device-side result of a batch: keys_out[Q][k] (sorted desc, 0 = empty), n_out[Q], total[Q].
struct TopkDevOut { unsigned long long* keys; uint32_t* n_out; unsigned long long* total; };

uint32_t term_id(const sdbg_bm25_term& t) { return t.term; }
uint32_t term_id(uint32_t t) { return t; }

// A batch of queries as the flat entries take it (the caller's arrays, not copied). Query q has the positive terms
// terms[term_off[q] .. term_off[q + 1]) and excludes the term ids excl_terms[excl_off[q] .. excl_off[q + 1]) (NULL
// excl_off: none). term_grp (kind OR only; NULL: none): query q is an AND of OR groups, positive term i belongs to group
// term_grp[i] & 15 of its query, which needs (term_grp[i] >> 4) + 1 of its lists. Term: sdbg_bm25_term for top-k, the
// bare term id for the unscored passes.
template <class Term>
struct QueryBatch {
  int kind;
  const Term* terms;
  const uint32_t* term_off;
  size_t nq;
  const uint32_t* excl_terms;
  const uint32_t* excl_off;
  const uint8_t* term_grp;
};

// Checks of a query batch shared by the top-k and count entries: 1..16 positive terms and at most 16 excluded ones per
// query, a non-decreasing excl_off, segments of one context with staged postings, positive term ids every segment
// holds, and a staged filter column. Sets *total_excl to excl_off[nq] when some query excludes terms, else 0.
template <class Term>
int check_query_batch(sdbg_segment* const* segs, size_t n_segs, const QueryBatch<Term>& Q, const sdbg_col_pred* filt,
                      uint32_t* total_excl) {
  const auto& [kind, terms, term_off, nq, excl_terms, excl_off, term_grp] = Q;
  sdbg_ctx* c = segs[0]->ctx;
  for (size_t q = 0; q < nq; ++q) {
    const uint32_t nt = term_off[q + 1] - term_off[q];
    if (nt == 0 || nt > kMaxQueryTerms) return fail(c, SDBG_EUNSUPPORTED, "a query needs 1..16 terms");
  }
  *total_excl = 0;
  if (excl_off) {
    for (size_t q = 0; q < nq; ++q) {
      if (excl_off[q + 1] < excl_off[q]) return fail(c, SDBG_EINVAL, "excl_off must be non-decreasing");
      if (excl_off[q + 1] - excl_off[q] > kMaxQueryTerms) return fail(c, SDBG_EUNSUPPORTED, "a query excludes at most 16 terms");
    }
    if (excl_off[nq] > excl_off[0]) {
      if (!excl_terms) return fail(c, SDBG_EINVAL, "excl_terms is NULL");
      *total_excl = excl_off[nq];
    }
  }
  for (size_t si = 0; si < n_segs; ++si) {
    if (segs[si]->ctx != c) return fail(c, SDBG_EINVAL, "segments of one call must share a context");
    if (!segs[si]->d_blocks) return fail(c, SDBG_EINVAL, "segment has no staged postings");
  }
  for (size_t si = 0; si < n_segs; ++si)
    for (uint32_t i = term_off[0]; i < term_off[nq]; ++i)
      if (size_t(term_id(terms[i])) + 1 >= segs[si]->term_blk_begin.size()) return fail(c, SDBG_EINVAL, "term id out of range");
  ChainDev fv;
  for (size_t si = 0; si < n_segs; ++si)
    if (int rc = filter_view(segs[si], filt, &fv)) return rc;
  return SDBG_OK;
}

int topk_limits(sdbg_ctx* c, size_t nq, uint32_t k) {
  if (k > 8192) return fail(c, SDBG_EUNSUPPORTED, "k > 8192");
  if (nq > 65535) return fail(c, SDBG_EUNSUPPORTED, "more than 65535 queries per batch");
  return SDBG_OK;
}

// A batch of group queries split by shape. Shape 0: one group, run as the flat OR of its terms; 1: every group one term,
// run as the AND; 2: a true nested query, run with its groups (term_grp). Each shape becomes a batch of the existing
// entry points' form: terms / term_off / excl_terms / excl_off over its queries, in batch order.
template <class Term>
struct GroupSplit {
  std::vector<uint32_t> qs[3];   // the batch positions of each shape's queries
  std::vector<Term> terms[3];
  std::vector<uint32_t> term_off[3], excl_terms[3], excl_off[3];
  std::vector<uint8_t> term_grp[3];
  uint32_t total_excl[3] = {};   // per shape, as check_query_batch sets it
  int whole = -1;                 // the shape of a batch of one shape; -1: several

  QueryBatch<Term> view(int sh) const {
    return {sh == 1 ? SDBG_QUERY_AND : SDBG_QUERY_OR, terms[sh].data(), term_off[sh].data(), qs[sh].size(),
            excl_terms[sh].empty() ? nullptr : excl_terms[sh].data(), excl_off[sh].data(),
            sh == 2 ? term_grp[sh].data() : nullptr};
  }
};

// check_query_batch on every shape of a split batch of nq queries; sets S.whole.
template <class Term>
int check_shapes(sdbg_segment* const* segs, size_t n_segs, size_t nq, const sdbg_col_pred* filt, GroupSplit<Term>& S) {
  for (int sh = 0; sh < 3; ++sh) {
    if (S.qs[sh].empty()) continue;
    if (int rc = check_query_batch(segs, n_segs, S.view(sh), filt, &S.total_excl[sh])) return rc;
    if (S.qs[sh].size() == nq) S.whole = sh;
  }
  return SDBG_OK;
}

// Splits a batch of sdbg_*_batch_groups(_min) by shape and checks it, every shape included, before anything is queued:
// non-decreasing query_group_off / group_off / excl_off, 1..16 groups, 1..16 positive terms and at most 16 excluded ones
// per query, no empty group, no positive term id twice in a query, 1 <= group_min[g] <= the group's size; then
// check_query_batch on every shape.
// group_min (NULL: every group 1) is normalised first: a group that needs all its s terms is s single-term groups, so
// that a query whose groups then all need 1 term takes the shapes above with exactly their results. The remaining queries
// (some group needs 2 <= m < s terms, so m <= 15) run with their groups, and each term's tag carries m - 1 in its high
// nibble (kCheckExcl's comment).
template <class Term>
int split_groups(sdbg_segment* const* segs, size_t n_segs, const Term* terms, const uint32_t* group_off,
                 const uint32_t* query_group_off, const uint32_t* group_min, size_t nq, const uint32_t* excl_terms,
                 const uint32_t* excl_off, const sdbg_col_pred* filt, GroupSplit<Term>& S) {
  sdbg_ctx* c = segs[0]->ctx;
  for (size_t q = 0; q < nq; ++q) {
    if (query_group_off[q + 1] < query_group_off[q]) return fail(c, SDBG_EINVAL, "query_group_off must be non-decreasing");
    for (uint32_t g = query_group_off[q]; g < query_group_off[q + 1]; ++g)
      if (group_off[g + 1] < group_off[g]) return fail(c, SDBG_EINVAL, "group_off must be non-decreasing");
    if (excl_off && excl_off[q + 1] < excl_off[q]) return fail(c, SDBG_EINVAL, "excl_off must be non-decreasing");
  }
  for (size_t q = 0; q < nq; ++q) {
    const uint32_t ng = query_group_off[q + 1] - query_group_off[q];
    if (ng == 0 || ng > kMaxQueryTerms) return fail(c, SDBG_EUNSUPPORTED, "a query needs 1..16 groups");
    const uint32_t t0 = group_off[query_group_off[q]], t1 = group_off[query_group_off[q + 1]];
    if (t1 - t0 > kMaxQueryTerms) return fail(c, SDBG_EUNSUPPORTED, "a query needs 1..16 terms");
    if (excl_off && excl_off[q + 1] - excl_off[q] > kMaxQueryTerms) return fail(c, SDBG_EUNSUPPORTED, "a query excludes at most 16 terms");
  }
  for (size_t q = 0; q < nq; ++q) {
    for (uint32_t g = query_group_off[q]; g < query_group_off[q + 1]; ++g) {
      if (group_off[g + 1] == group_off[g]) return fail(c, SDBG_EINVAL, "empty OR group");
      if (group_min && (group_min[g] == 0 || group_min[g] > group_off[g + 1] - group_off[g]))
        return fail(c, SDBG_EINVAL, "a group's minimum match count must be 1..its number of terms");
    }
    const uint32_t t0 = group_off[query_group_off[q]], t1 = group_off[query_group_off[q + 1]];
    if (!terms) return fail(c, SDBG_EINVAL, "terms is NULL");
    if (excl_off && excl_off[q + 1] > excl_off[q] && !excl_terms) return fail(c, SDBG_EINVAL, "excl_terms is NULL");
    std::array<uint32_t, kMaxQueryTerms> ids;
    for (uint32_t i = t0; i < t1; ++i) ids[i - t0] = term_id(terms[i]);
    std::sort(ids.begin(), ids.begin() + (t1 - t0));
    if (std::adjacent_find(ids.begin(), ids.begin() + (t1 - t0)) != ids.begin() + (t1 - t0))
      return fail(c, SDBG_EINVAL, "a positive term id occurs twice in a query");
  }
  for (int sh = 0; sh < 3; ++sh) { S.term_off[sh].assign(1, 0u); S.excl_off[sh].assign(1, 0u); }
  for (size_t q = 0; q < nq; ++q) {
    const uint32_t g0 = query_group_off[q], g1 = query_group_off[q + 1];
    const uint32_t t0 = group_off[g0], t1 = group_off[g1];
    // normalised groups: m == s becomes s single-term groups; a group of 2 <= m < s keeps its m
    uint32_t n_groups = 0;
    bool min_group = false;
    for (uint32_t g = g0; g < g1; ++g) {
      const uint32_t s = group_off[g + 1] - group_off[g], m = group_min ? group_min[g] : 1u;
      if (m == s) n_groups += s;
      else { ++n_groups; min_group |= m > 1u; }
    }
    const int sh = min_group ? 2 : n_groups == 1 ? 0 : (t1 - t0 == n_groups ? 1 : 2);
    S.qs[sh].push_back(uint32_t(q));
    uint32_t gi = 0;
    for (uint32_t g = g0; g < g1; ++g) {
      const uint32_t s = group_off[g + 1] - group_off[g], m = group_min ? group_min[g] : 1u;
      for (uint32_t i = group_off[g]; i < group_off[g + 1]; ++i) {
        S.terms[sh].push_back(terms[i]);
        if (sh == 2) S.term_grp[sh].push_back(m == s ? uint8_t(gi++) : uint8_t(gi | ((m - 1u) << 4)));
      }
      if (m != s) ++gi;
    }
    S.term_off[sh].push_back(uint32_t(S.terms[sh].size()));
    if (excl_off)
      for (uint32_t i = excl_off[q]; i < excl_off[q + 1]; ++i) S.excl_terms[sh].push_back(excl_terms[i]);
    S.excl_off[sh].push_back(uint32_t(S.excl_terms[sh].size()));
  }
  return check_shapes(segs, n_segs, nq, filt, S);
}

// The queries of one call, checked before anything is queued (rc: the checks' result): a batch that runs whole (a flat
// batch, or a group batch of one shape), or a group batch of several shapes (S; whole.nq == 0). Term: sdbg_bm25_term for
// the top-k, the bare term id for the count, facet, aggregate and sorted passes.
template <class Term>
struct PassBatch {
  int rc;
  size_t nq;
  QueryBatch<Term> whole{};
  uint32_t total_excl = 0;   // whole's, as check_query_batch sets it
  GroupSplit<Term> S;

  PassBatch(sdbg_segment* const* segs, size_t n_segs, const QueryBatch<Term>& Q, const sdbg_col_pred* filt) : nq(Q.nq), whole(Q) {
    rc = !segs || !n_segs || !Q.terms || !Q.term_off || !Q.nq ? SDBG_EINVAL : check_query_batch(segs, n_segs, Q, filt, &total_excl);
  }
  PassBatch(sdbg_segment* const* segs, size_t n_segs, const Term* terms, const uint32_t* group_off, const uint32_t* query_group_off,
            const uint32_t* group_min, size_t nq, const uint32_t* excl_terms, const uint32_t* excl_off, const sdbg_col_pred* filt)
      : nq(nq) {
    rc = split_groups(segs, n_segs, terms, group_off, query_group_off, group_min, nq, excl_terms, excl_off, filt, S);
    if (S.whole >= 0) { whole = S.view(S.whole); total_excl = S.total_excl[S.whole]; }
  }
  // A batch its caller has split (S_: every query in one shape, no term twice in a query; PhraseBatch::candidates).
  PassBatch(sdbg_segment* const* segs, size_t n_segs, GroupSplit<Term>&& S_, size_t nq, const sdbg_col_pred* filt)
      : nq(nq), S(std::move(S_)) {
    rc = check_shapes(segs, n_segs, nq, filt, S);
    if (S.whole >= 0) { whole = S.view(S.whole); total_excl = S.total_excl[S.whole]; }
  }
  PassBatch(const PassBatch&) = delete;   // whole may point into S
};

// dst row to[j] = src row j, rows of row_words words.
template <class Word>
__global__ void __launch_bounds__(256) scatter_rows_kernel(const Word* __restrict__ src, Word* __restrict__ dst,
                                                           const uint32_t* __restrict__ to, size_t n_rows, size_t row_words) {
  const size_t n = n_rows * row_words;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += size_t(gridDim.x) * blockDim.x) {
    const size_t j = i / row_words;
    dst[size_t(to[j]) * row_words + (i - j * row_words)] = src[i];
  }
}

// Runs the shapes of a mixed-shape batch S one after another, each into zeroed rows of its own (c->pass[2]):
// run(sh, part) fills shape sh's rows part[i], row[i] bytes per query (0: no such array), and scatter_rows_kernel moves
// them to the caller's query positions in dst[i] on the stream (rows of u32 words when row[i] is not a multiple of 8,
// else of u64 words). Nothing waits.
template <class Term, class Run>
int shapes_run(sdbg_ctx* c, const GroupSplit<Term>& S, const std::array<size_t, 3>& row, void* const (&dst)[3], Run run) {
  const auto pad = [](size_t b) { return (b + 7) & ~size_t(7); };
  // per shape: its query positions (u32), then its rows of each array, every part 8-byte aligned
  size_t pos[3] = {}, bytes = 0;
  for (int sh = 0; sh < 3; ++sh) {
    const size_t n = S.qs[sh].size();
    pos[sh] = bytes;
    bytes += pad(n * 4);
    for (size_t r : row) bytes += pad(n * r);
  }
  if (int rc = ensure(c, c->pass[2], bytes)) return rc;
  char* d = static_cast<char*>(c->pass[2].p);
  CU(c, cudaMemsetAsync(d, 0, bytes, c->stream));
  for (int sh = 0; sh < 3; ++sh)   // pageable: consumed on return
    if (!S.qs[sh].empty()) CU(c, cudaMemcpyAsync(d + pos[sh], S.qs[sh].data(), S.qs[sh].size() * 4, cudaMemcpyHostToDevice, c->stream));
  for (int sh = 0; sh < 3; ++sh) {
    const size_t n = S.qs[sh].size();
    if (!n) continue;
    const auto* to = reinterpret_cast<const uint32_t*>(d + pos[sh]);
    void* part[3];
    char* p = d + pos[sh] + pad(n * 4);
    for (int i = 0; i < 3; ++i) { part[i] = p; p += pad(n * row[i]); }
    if (int rc = run(sh, part)) return rc;
    for (int i = 0; i < 3; ++i) {
      if (!row[i]) continue;
      const size_t words = row[i] % 8 ? row[i] / 4 : row[i] / 8;
      const unsigned grid = unsigned(std::min<size_t>((n * words + 255) / 256, size_t(c->sm_count) * 8));
      if (row[i] % 8)
        scatter_rows_kernel<<<grid, 256, 0, c->stream>>>(static_cast<const uint32_t*>(part[i]), static_cast<uint32_t*>(dst[i]),
                                                         to, n, words);
      else
        scatter_rows_kernel<<<grid, 256, 0, c->stream>>>(static_cast<const unsigned long long*>(part[i]),
                                                         static_cast<unsigned long long*>(dst[i]), to, n, words);
      ++c->launches;
    }
    CU(c, cudaGetLastError());
  }
  return SDBG_OK;
}

// The top-k entries' checks of their scalar arguments, before their batch's (PassBatch).
int topk_args(sdbg_segment* const* segs, size_t n_segs, size_t nq, uint32_t k) {
  if (!segs || !n_segs || !segs[0] || !nq || !k) return SDBG_EINVAL;
  sdbg_ctx* c = segs[0]->ctx;
  if (int rc = topk_limits(c, nq, k)) return rc;
  CU(c, cudaSetDevice(c->device));
  return SDBG_OK;
}

// The top-k entries' checks after topk_args and their batch's: at most 2^32 - 2 docs per call (the kernels' ordinals).
int topk_checked(sdbg_segment* const* segs, size_t n_segs, const PassBatch<sdbg_bm25_term>& B) {
  if (B.rc) return B.rc;
  uint64_t ord = 0;
  for (size_t si = 0; si < n_segs; ++si) ord += segs[si]->n_docs;
  if (ord > kMaxDocId) return fail(segs[0]->ctx, SDBG_EUNSUPPORTED, "more than 2^32-2 docs per call");
  return SDBG_OK;
}

// Each query's terms over each segment as QTermDev, dst[segment][term], by ascending docs_count in that segment (stable,
// conjunction.hpp:520-523): the order in which the top-k kernels sum a doc's term scores.
void qterms_by_cost(sdbg_segment* const* segs, size_t n_segs, const QueryBatch<sdbg_bm25_term>& Q, float k1, float b, QTermDev* qt) {
  const size_t nq = Q.nq, n_terms = Q.term_off[nq];
  for (size_t si = 0; si < n_segs; ++si) {
    QTermDev* dst = qt + si * n_terms;
    for (size_t q = 0; q < nq; ++q) {
      const uint32_t t_begin = Q.term_off[q], t_end = Q.term_off[q + 1];
      for (uint32_t i = t_begin; i < t_end; ++i) fill_qterm(segs[si], Q.terms[i], k1, b, dst[i]);
      std::stable_sort(dst + t_begin, dst + t_end, [](const QTermDev& x, const QTermDev& y) { return x.docs_count < y.docs_count; });
    }
  }
}

// The descriptor block of the top-k kernels (TopkParams, MergeParams::list_off), staged in pageable memory for one copy:
// [QTermDev [segment][term_off[nq]], each query's terms by ascending docs_count (conjunction.hpp:520-523) | term_off
// [nq + 1] | from 16 B on, the work items {query, first doc, docs, candidate list} | list_off [nq + 1] | when some query
// has per-doc checks, from 16 B on: {first block, blocks} [segment][check] | chk_off [nq + 1] | with Q.term_grp, each
// check's group tag].
struct TopkDesc {
  std::vector<char> h;
  size_t n_segs, n_terms, n_chk, off_pos, work_pos, list_pos, x_pos, chk_off_pos, grp_pos;
  bool grp;

  // Points segment si's launch parameters at the block's device copy d, its work items from `first` on.
  void params(const char* d, size_t si, size_t first, TopkParams& P) const {
    P.qterms = reinterpret_cast<const QTermDev*>(d) + si * n_terms;
    P.qterm_off = reinterpret_cast<const uint32_t*>(d + off_pos);
    P.work = reinterpret_cast<const uint4*>(d + work_pos) + first;
    if (!n_chk) return;
    P.excl = reinterpret_cast<const uint2*>(d + x_pos) + si * n_chk;
    P.excl_off = reinterpret_cast<const uint32_t*>(d + chk_off_pos);
    if (grp) P.excl_grp = reinterpret_cast<const uint8_t*>(d + grp_pos);
  }
};

// Writes the descriptor block of queries Q over segs (term ids checked): work items `work`, list_off, and the per-doc
// check lists chk_terms[chk_off[q] .. chk_off[q + 1]) of query q with their group tags chk_grp (Q.term_grp).
TopkDesc topk_desc(sdbg_segment* const* segs, size_t n_segs, const QueryBatch<sdbg_bm25_term>& Q, float k1, float b,
                   const std::vector<uint4>& work, const std::vector<uint32_t>& list_off, const std::vector<uint32_t>& chk_terms,
                   const std::vector<uint32_t>& chk_off, const std::vector<uint8_t>& chk_grp) {
  const size_t nq = Q.nq, n_terms = Q.term_off[nq], n_chk = chk_terms.size(), off_bytes = (nq + 1) * sizeof(uint32_t);
  TopkDesc D{{}, n_segs, n_terms, n_chk, 0, 0, 0, 0, 0, 0, Q.term_grp != nullptr};
  D.off_pos = n_terms * sizeof(QTermDev) * n_segs;
  D.work_pos = (D.off_pos + off_bytes + 15) & ~size_t(15);   // work items are 16-byte loads
  D.list_pos = D.work_pos + work.size() * sizeof(uint4);
  D.x_pos = (D.list_pos + off_bytes + 15) & ~size_t(15);
  D.chk_off_pos = D.x_pos + n_chk * n_segs * sizeof(uint2);
  D.grp_pos = D.chk_off_pos + off_bytes;
  D.h.resize(n_chk ? D.grp_pos + (D.grp ? n_chk : 0) : D.list_pos + off_bytes);
  char* h = D.h.data();
  qterms_by_cost(segs, n_segs, Q, k1, b, reinterpret_cast<QTermDev*>(h));
  std::memcpy(h + D.off_pos, Q.term_off, off_bytes);
  std::memcpy(h + D.work_pos, work.data(), work.size() * sizeof(uint4));
  std::memcpy(h + D.list_pos, list_off.data(), off_bytes);
  if (n_chk) {
    auto* x = reinterpret_cast<uint2*>(h + D.x_pos);
    for (size_t si = 0; si < n_segs; ++si)
      for (size_t i = 0; i < n_chk; ++i) x[si * n_chk + i] = excl_list(segs[si], chk_terms[i]);
    std::memcpy(h + D.chk_off_pos, chk_off.data(), off_bytes);
    if (D.grp) std::memcpy(h + D.grp_pos, chk_grp.data(), n_chk);
  }
  return D;
}

// Queues a batch that passed topk_args and topk_checked (total_excl: as check_query_batch set it) into the device arrays
// out: keys [nq][k] (sorted descending, then zeros), n_out [nq] and total [nq] (NULL: not wanted). The descriptors are
// staged from pageable memory, which the copy has consumed when it returns, so the shapes of a mixed batch follow one
// another without a wait. A query of OR groups (Q.term_grp) runs as the OR of all its terms, and a doc must also occur in
// as many lists of every group as the group needs.
int topk_run(sdbg_segment* const* segs, size_t n_segs, const QueryBatch<sdbg_bm25_term>& Q, uint32_t total_excl, float k1,
             const float b, const sdbg_col_pred* filt, uint32_t k, float threshold_in, const TopkDevOut& out) {
  const auto& [kind, terms, term_off, nq, excl_terms, excl_off, term_grp] = Q;
  sdbg_ctx* c = segs[0]->ctx;
  const uint32_t total_terms = term_off[nq];
  // Per-doc check lists of each query: its excluded terms (tag kCheckExcl), then, for a query of OR groups, each positive
  // term tagged with its group. chk_off[q] .. chk_off[q + 1] index chk_terms / chk_grp.
  std::vector<uint32_t> chk_off, chk_terms;
  std::vector<uint8_t> chk_grp;
  if (total_excl || term_grp) {
    chk_off.assign(nq + 1, 0u);
    for (size_t q = 0; q < nq; ++q) {
      if (total_excl)
        for (uint32_t i = excl_off[q]; i < excl_off[q + 1]; ++i) { chk_terms.push_back(excl_terms[i]); chk_grp.push_back(kCheckExcl); }
      if (term_grp)
        for (uint32_t i = term_off[q]; i < term_off[q + 1]; ++i) { chk_terms.push_back(terms[i].term); chk_grp.push_back(uint8_t(term_grp[i])); }
      chk_off[q + 1] = uint32_t(chk_terms.size());
    }
  }
  const uint32_t total_chk = uint32_t(chk_terms.size());   // > 0: some query has per-doc checks

  TopkPlan pl;
  pl.k = k;
  const uint32_t entries = kTopkBudget * 128u;
  pl.cap = std::max(next_pow2(k + 1024), 2048u);  // selection is O(n): buffer size trades shared memory (occupancy) against selection count
  // Enough CTAs to fill the machine a few times over; a query is split into chains (contiguous doc
  // ranges) only when the batch alone cannot do that.
  const uint32_t target_ctas = uint32_t(c->sm_count) * 8u;
  pl.G = uint32_t(std::max<size_t>(1, (target_ctas + nq - 1) / nq));
  const uint32_t max_chains = 2u * uint32_t(c->sm_count);
  // Work list: (segment, query) pairs get max(G, postings / target) chains, so that a query over a 5 M-doc
  // list is not one CTA-long critical path next to thousands of short ones; largest chains are issued first.
  uint64_t batch_postings = 0;
  for (size_t si = 0; si < n_segs; ++si)
    for (uint32_t i = 0; i < total_terms; ++i)
      if (terms[i].term < segs[si]->term_docs.size()) batch_postings += segs[si]->term_docs[terms[i].term];
  const uint64_t chain_target = std::max<uint64_t>(65536, batch_postings / (uint64_t(c->sm_count) * 4u));
  // Work classes (one launch each):
  //   0 / 1        legacy window kernel (driver mode / plain): > 4-term disjunctions, BM15 / BM1 forms
  //   2 + (T-1)    exhaustive warp-autonomous merge of T = 1..4 lists (bm25_merge.cuh): pruning off or not applicable
  //   6 + (T-1)    stream kernel, disjunction with MaxScore demotion / single-list block-max skip (bm25_stream.cuh)
  //   10           conjunctions: lead list + probes (stream kernel, kModeAnd), hybrid filter and deleted docs included
  //   11           first slice of a two-term disjunction whose long list is worth probing instead of scanning: merged
  //                exhaustively FIRST so that the query has a threshold when the rest of its range starts
  //   12           the rest of such a query: launched into BOTH the merge kernel and the stream kernel in lead mode
  //                (short list streamed, long list probed per candidate); the first CTA to arrive decides from the
  //                threshold which of the two runs the item (TopkParams::claim)
  //   kClasses + c class c (0 / 1, 6 .. 10 only) for queries that exclude terms: the kExcl instantiations of the same
  //                kernels. Never the merge kernel, slices or lead mode, which have no per-doc checks.
  //   2 kClasses + c  the same for queries of OR groups (term_grp; classes 0 / 1, 6 .. 9): the kGroups instantiations.
  struct WorkItem { uint32_t q, lo, len, list; uint64_t weight; uint32_t cls; };
  constexpr uint32_t kClsMerge = 2, kClsStream = 2 + kStreamMaxTerms, kClsAnd = 2 + 2 * kStreamMaxTerms, kClsSlice = kClsAnd + 1,
                     kClsLead = kClsAnd + 2, kClasses = kClsAnd + 3, kAllClasses = 3 * kClasses;
  const bool level2 = c->wand >= 2 && kind != SDBG_QUERY_AND && k1 != 0.f && k1 != kTfidfK1 && b != 0.f;
  const bool stream_ok = env_int("SDBG_STREAM", 1) != 0 && k1 != 0.f && b != 0.f && k1 != kTfidfK1 &&
                         stream_smem(pl.cap, kStreamMaxTerms, false) <= 200 * 1024;
  const bool lead_ok = env_int("SDBG_STREAM_LEAD", 1) != 0;
  // The staged block-max pairs are maximisers for BM25 with the index-time b only (FreqNormProducer::CmpBm25,
  // wand_writer.hpp:142-175; the order of two pairs does not depend on k); the reference enables WAND only when
  // Scorer::equals matches (PostingsReaderImpl::WandIterator, reader.hpp:457-501). Any other b: exhaustive.
  auto seg_wand = [&](const sdbg_segment* s) { return (c->wand && s->has_wand && k1 != 0.f && k1 != kTfidfK1 && b != 0.f && b == s->wand_b) ? c->wand : 0; };
  std::vector<std::array<size_t, kAllClasses>> n_cls(n_segs);
  for (auto& a : n_cls) a.fill(0);
  std::vector<std::vector<WorkItem>> seg_work(n_segs);
  std::vector<uint32_t> list_off(nq + 1, 0);
  for (size_t q = 0; q < nq; ++q) {          // lists of one query are contiguous: [segment 0 chains | segment 1 chains | ...]
    uint32_t lists = 0;
    for (size_t si = 0; si < n_segs; ++si) {
      const sdbg_segment* s = segs[si];
      uint64_t postings = 0;
      uint32_t largest = 0, largest_term = UINT32_MAX, smallest = UINT32_MAX;
      for (uint32_t i = term_off[q]; i < term_off[q + 1]; ++i)
        if (terms[i].term < s->term_docs.size()) {
          const uint32_t dc = s->term_docs[terms[i].term];
          postings += dc;
          smallest = std::min(smallest, dc);
          if (dc >= largest) { largest = dc; largest_term = terms[i].term; }
        }
      const uint32_t nt = term_off[q + 1] - term_off[q];
      const int wand = seg_wand(s);
      // Driver mode (pruning level 2) pays only when the largest list can be probed without decoding blocks; the
      // other queries run the plain kernel, which is lighter (fewer registers, no probe buffers, level-1 planner).
      const bool drive_q = level2 && wand && nt >= 2 && largest_term < s->term_probe.size() && s->term_probe[largest_term] != 0;
      const bool excludes = total_chk && chk_off[q + 1] > chk_off[q];
      uint32_t cls = drive_q ? 0u : 1u;
      uint32_t slice_docs = 0;    // > 0: lead candidate
      if (stream_ok && kind == SDBG_QUERY_AND) cls = kClsAnd;
      else if (stream_ok && kind != SDBG_QUERY_AND && nt <= kStreamMaxTerms) {
        const bool plain = !filt && !s->d_deleted && !excludes;     // the merge kernel has no per-doc checks
        cls = (!plain || (wand && (nt != 2 || !lead_ok))) ? kClsStream + (nt - 1u) : kClsMerge + (nt - 1u);
        if (wand && nt == 2 && lead_ok && plain && uint64_t(largest) >= 4ull * smallest && smallest >= 3u * k) {
          // Lead mode needs the threshold above the long list's bound. That happens when a typical posting of the short
          // list (freq 1, average length) already outscores the best posting of the long one; then about k docs of the
          // short list, i.e. the first 1.5 k / |short| of the doc range, are enough to get there.
          const sdbg_bm25_term* ta = &terms[term_off[q]];
          const sdbg_bm25_term* tb = ta + 1;
          if (s->term_docs[ta->term] > s->term_docs[tb->term]) std::swap(ta, tb);       // ta = short list
          const MaxPair root = tb->term < s->term_max.size() ? s->term_max[tb->term] : MaxPair{0, 0};
          if (root.freq != 0) {
            float bnc, bnl;
            bound_consts(s, k1, b, tb->norm_const, tb->norm_length, bnc, bnl);
            const float c0b = tb->boost * (k1 + 1) * tb->idf, c1b = bnc + bnl * float(root.norm);
            const float ub_b = c0b - c0b * c1b / (c1b + float(root.freq));
            const float c0a = ta->boost * (k1 + 1) * ta->idf, c1a = ta->norm_const + ta->norm_length * (ta->norm_length > 0.f ? (k1 * b) / ta->norm_length : 1.f);
            const float typ_a = c0a - c0a * c1a / (c1a + 1.f);                           // freq 1 at the average length
            if (ub_b * 1.05f < typ_a) {
              const double frac = 1.5 * double(k) / double(smallest);
              slice_docs = uint32_t(std::min<double>(double(s->n_docs), std::max(4096.0, std::ceil(double(s->n_docs) * frac))));
              if (slice_docs > s->n_docs / 2) slice_docs = 0;
            }
          }
        }
      }
      const uint32_t first = slice_docs ? slice_docs + 1u : 1u;             // first doc of the chained range
      const uint32_t rest_docs = s->n_docs - (first - 1u);
      const uint64_t rest_postings = slice_docs ? uint64_t(double(postings) * double(rest_docs) / double(s->n_docs)) : postings;
      if (slice_docs) {
        seg_work[si].push_back({uint32_t(q), 1u, slice_docs, list_off[q] + lists, postings - rest_postings, kClsSlice});
        ++n_cls[si][kClsSlice];
        ++lists;
        cls = kClsLead;
      }
      if (excludes) cls += term_grp ? 2 * kClasses : kClasses;
      uint32_t g = uint32_t(std::max<uint64_t>(pl.G, (rest_postings + chain_target - 1) / chain_target));
      // lead mode is latency-bound (dependent loads per probe), not throughput-bound: more, shorter chains
      if (slice_docs) g = std::max(g, std::min(16u, std::max(1u, smallest / 8192u)));
      g = std::min(g, max_chains);
      g = std::min(g, std::max(1u, rest_docs / 4096u));
      const uint32_t chunk = uint32_t((uint64_t(rest_docs) + g - 1) / g);   // 64-bit: rest_docs reaches 2^32 - 2
      for (uint32_t j = 0; j < g; ++j)
        seg_work[si].push_back({uint32_t(q), first + j * chunk, chunk, list_off[q] + lists + j, rest_postings / g, cls});
      n_cls[si][cls] += g;
      lists += g;
    }
    list_off[q + 1] = list_off[q] + lists;
  }
  const uint32_t total_lists = list_off[nq];
  size_t total_work = 0;
  for (auto& w : seg_work) {
    std::stable_sort(w.begin(), w.end(), [](const WorkItem& x, const WorkItem& y) { return x.cls != y.cls ? x.cls < y.cls : x.weight > y.weight; });
    total_work += w.size();
  }
  pl.smem = size_t(entries) * 8 + (kind == SDBG_QUERY_AND ? entries : 0) + size_t(pl.cap) * 8;
  const size_t smem_drive = pl.smem + size_t(entries) * 4;   // probe list | decode-fallback list
  if (smem_drive > 200 * 1024) return fail(c, SDBG_EUNSUPPORTED, "hash window + candidate buffer exceed shared memory");

  std::vector<uint4> work;
  work.reserve(total_work);
  for (auto& w : seg_work) for (const WorkItem& it : w) work.push_back(make_uint4(it.q, it.lo, it.len, it.list));
  const TopkDesc D = topk_desc(segs, n_segs, Q, k1, b, work, list_off, chk_terms, chk_off, chk_grp);
  DevBuf& b_qt = c->scratch[0]; DevBuf& b_theta = c->scratch[1]; DevBuf& b_cand = c->scratch[2]; DevBuf& b_candn = c->scratch[3];
  int rc;
  if ((rc = ensure(c, b_qt, D.h.size()))) return rc;
  if ((rc = ensure(c, b_theta, nq * 16))) return rc;  // theta[nq] | total[nq] when out.total is NULL
  if ((rc = ensure(c, b_cand, size_t(total_lists) * pl.cap * 8))) return rc;
  if ((rc = ensure(c, b_candn, size_t(total_lists) * 4))) return rc;
  CU(c, cudaMemcpyAsync(b_qt.p, D.h.data(), D.h.size(), cudaMemcpyHostToDevice, c->stream));
  const char* d_desc = static_cast<const char*>(b_qt.p);
  auto* d_theta = static_cast<unsigned long long*>(b_theta.p);
  auto* d_total = out.total ? out.total : d_theta + nq;
  uint32_t thr_bits; std::memcpy(&thr_bits, &threshold_in, 4);
  if (!(threshold_in >= 0.f)) thr_bits = 0;  // negative / NaN seeds accept every positive score
  fill_u64_kernel<<<64, 256, 0, c->stream>>>(d_theta, nq, (static_cast<unsigned long long>(thr_bits) << 32) | 0xFFFFFFFFull);
  ++c->launches;
  CU(c, cudaMemsetAsync(d_total, 0, nq * 8, c->stream));

  if ((rc = topk_smem_attrs(c))) return rc;
  // one claim word per work item of class kClsLead (zeroed per call)
  size_t n_lead_total = 0;
  for (size_t si = 0; si < n_segs; ++si) n_lead_total += n_cls[si][kClsLead];
  DevBuf& b_claim = c->scratch[11];
  if (n_lead_total) {
    if ((rc = ensure(c, b_claim, n_lead_total * 4))) return rc;
    CU(c, cudaMemsetAsync(b_claim.p, 0, n_lead_total * 4, c->stream));
  }
  uint32_t base = 0;
  size_t work_done = 0, lead_done = 0;
  // Work classes are separate launches; with more than one present they alternate between two streams (forked from
  // and joined back into the context's stream) so that no class waits for another's tail. First slices (class 11) go
  // first, and everything that depends on their thresholds is ordered behind them.
  uint64_t classes_present = 0;
  for (size_t si = 0; si < n_segs; ++si) for (uint32_t k2 = 0; k2 < kAllClasses; ++k2) if (n_cls[si][k2]) classes_present |= 1ull << k2;
  const bool two_lanes = (classes_present & (classes_present - 1u)) != 0u;
  std::vector<ChainDev> chains(n_segs);
  if ((rc = filter_chains(segs, n_segs, filt, chains.data()))) return rc;
  {
    ProfScope ps_(c, kProfTopk);   // one span for all top-k launches of the call
    uint32_t lane_no = 0;
    for (size_t si = 0; si < n_segs; ++si) {
      sdbg_segment* s = segs[si];
      TopkParams P;
      P.seg = postings_view(s, base);
      P.filt = chains[si];
      D.params(d_desc, si, work_done, P);
      const uint4* const work0 = P.work;
      work_done += seg_work[si].size();
      P.theta = d_theta; P.total = d_total;
      P.cand = static_cast<unsigned long long*>(b_cand.p);
      P.cand_n = static_cast<uint32_t*>(b_candn.p);
      P.k = k; P.cap = pl.cap; P.conjunction = kind == SDBG_QUERY_AND ? 1 : 0;
      P.claim = nullptr;
      const int wand = seg_wand(s);
      std::array<size_t, kAllClasses> cls_off{};
      { size_t o = 0; for (uint32_t cls = 0; cls < kAllClasses; ++cls) { cls_off[cls] = o; o += n_cls[si][cls]; } }
      auto launch_merge = [&](uint32_t T, size_t n, cudaStream_t st) {
        const size_t sm = size_t(pl.cap) * 8 + size_t(kTopkWarps) * T * kMergeTermBytes;
        merge_kernel(T)<<<unsigned(n), kTopkThreads, sm, st>>>(P);
        ++c->launches;
      };
      // first slices: before everything else of this segment, on the main stream
      if (n_cls[si][kClsSlice]) {
        P.work = work0 + cls_off[kClsSlice]; P.wand = 0;
        launch_merge(2, n_cls[si][kClsSlice], c->stream);
      }
      if (two_lanes) {
        CU(c, cudaEventRecord(c->ev_fork, c->stream));
        CU(c, cudaStreamWaitEvent(c->stream2, c->ev_fork, 0));
      }
      for (uint32_t cls = 0; cls < kAllClasses; ++cls) {
        const size_t n = n_cls[si][cls];
        if (!n || cls == kClsSlice) continue;
        cudaStream_t st = (two_lanes && (lane_no++ & 1u)) ? c->stream2 : c->stream;
        P.work = work0 + cls_off[cls];
        P.claim = nullptr;
        // queries with excluded terms / OR groups: the kExcl / kGroups instantiations of the same kernels
        const bool grp = cls >= 2 * kClasses;
        const bool excl = cls >= kClasses && !grp;
        const uint32_t cb = cls % kClasses;
        TopkKernel kern;
        size_t sm;
        if (cb == 0) {
          P.wand = wand;
          kern = grp ? bm25_topk_kernel<true, true, true> : excl ? bm25_topk_kernel<true, true> : bm25_topk_kernel<true>;
          sm = smem_drive;
        } else if (cb == 1) {
          P.wand = std::min(wand, 1);
          kern = grp ? bm25_topk_kernel<false, true, true> : excl ? bm25_topk_kernel<false, true> : bm25_topk_kernel<false>;
          sm = pl.smem;
        } else if (cb == kClsAnd) {
          P.wand = 0;                                  // conjunctions are exact: every candidate of the lead list is probed
          kern = excl ? stream_kernel<kModeAnd, true>(1) : stream_kernel<kModeAnd>(1);
          sm = stream_smem(pl.cap, 1, true);
        } else if (cb == kClsLead) {
          // both kernels over the same items; each item is run by exactly one of them (claim word)
          P.claim = static_cast<uint32_t*>(b_claim.p) + lead_done;
          lead_done += n;
          P.wand = 0;
          launch_merge(2, n, c->stream);
          P.wand = wand;
          kern = stream_kernel<kModeLead>(1);
          sm = stream_smem(pl.cap, 1, true);
          st = two_lanes ? c->stream2 : c->stream;
        } else if (cb >= kClsStream) {
          const uint32_t T = cb - kClsStream + 1u;
          P.wand = wand;
          kern = grp ? stream_kernel<kModeOr, true, true>(T) : excl ? stream_kernel<kModeOr, true>(T) : stream_kernel<kModeOr>(T);
          sm = stream_smem(pl.cap, T, false);
        } else {
          P.wand = 0;
          launch_merge(cb - kClsMerge + 1u, n, st);
          continue;
        }
        kern<<<unsigned(n), kTopkThreads, sm, st>>>(P);
        ++c->launches;
      }
      CU(c, cudaGetLastError());
      base += s->n_docs;
      if (two_lanes) {
        CU(c, cudaEventRecord(c->ev_join, c->stream2));
        CU(c, cudaStreamWaitEvent(c->stream, c->ev_join, 0));
      }
    }
  }
  MergeParams M;
  M.cand = static_cast<const unsigned long long*>(b_cand.p);
  M.cand_n = static_cast<const uint32_t*>(b_candn.p);
  M.list_off = reinterpret_cast<const uint32_t*>(d_desc + D.list_pos);
  M.G = 0; M.stride = pl.cap; M.k = k; M.cap = pl.cap;
  M.keys_out = out.keys;
  M.n_out = out.n_out;
  { ProfScope ps_(c, kProfMerge);
    topk_merge_kernel<<<unsigned(nq), kTopkThreads, size_t(pl.cap) * 8, c->stream>>>(M); }
  ++c->launches;
  CU(c, cudaGetLastError());
  return SDBG_OK;
}

// Copies a top-k result d back through the pinned staging, [keys | total (when d.total) | n_out], and converts it into
// the caller's arrays: hit i of query q is keys[q][i] as {score bits, decode(ordinal)}, with total_matches[q] (NULL: not
// wanted) when d has totals. Turning keys into hits is a few ns per hit; a large batch (millions of hits) is cut into
// per-thread query ranges whose keys are copied back one after the other, each followed by an event: a thread converts
// its range as soon as it has landed, while the later ranges are still on the wire. One wait at the end.
template <class Decode>
int topk_to_host(sdbg_ctx* c, const TopkDevOut& d, size_t nq, uint32_t k, Decode decode, sdbg_hit* out, uint32_t* n_out,
                 uint64_t* total_matches) {
  const size_t kb = nq * size_t(k) * 8, tb = d.total ? nq * 8 : 0, nb = nq * 4;
  if (int rc = ensure_pinned(c, kb + tb + nb)) return rc;
  char* h = static_cast<char*>(c->h_pinned);
  const size_t n_thr = std::max<size_t>(1, std::min<size_t>({size_t(env_int("SDBG_HOST_THREADS", 16)), (nq * size_t(k)) / 65536, size_t(kMaxCopyEvents)}));
  if (tb) CU(c, cudaMemcpyAsync(h + kb, d.total, tb, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaMemcpyAsync(h + kb + tb, d.n_out, nb, cudaMemcpyDeviceToHost, c->stream));
  for (size_t t = 0; t < n_thr; ++t) {
    const size_t q0 = nq * t / n_thr, q1 = nq * (t + 1) / n_thr;
    CU(c, cudaMemcpyAsync(h + q0 * k * 8, d.keys + q0 * k, (q1 - q0) * k * 8, cudaMemcpyDeviceToHost, c->stream));
    if (n_thr > 1) {
      if (!c->ev_copy[t]) CU(c, cudaEventCreateWithFlags(&c->ev_copy[t], cudaEventDisableTiming));
      CU(c, cudaEventRecord(c->ev_copy[t], c->stream));
    }
  }
  const auto* keys = reinterpret_cast<const unsigned long long*>(h);
  const auto* tot = reinterpret_cast<const unsigned long long*>(h + kb);
  const auto* cnt = reinterpret_cast<const uint32_t*>(h + kb + tb);
  auto convert = [&](size_t q0, size_t q1) {
    for (size_t q = q0; q < q1; ++q) {
      n_out[q] = cnt[q];
      for (uint32_t i = 0; i < cnt[q]; ++i) {
        const unsigned long long key = keys[q * k + i];
        const uint32_t bits = uint32_t(key >> 32);
        sdbg_hit& hit = out[q * k + i];
        std::memcpy(&hit.score, &bits, 4);
        const uint2 sd = decode(~uint32_t(key));
        hit.seg = sd.x;
        hit.doc = sd.y;
      }
      if (tb && total_matches) total_matches[q] = tot[q];
    }
  };
  if (n_thr <= 1) {
    CU(c, cudaStreamSynchronize(c->stream));
    convert(0, nq);
  } else {
    std::atomic<int> err{0};
    std::vector<std::thread> pool;
    for (size_t t = 0; t < n_thr; ++t)
      pool.emplace_back([&, t] {
        if (cudaSetDevice(c->device) != cudaSuccess || cudaEventSynchronize(c->ev_copy[t]) != cudaSuccess) { err = 1; return; }
        convert(nq * t / n_thr, nq * (t + 1) / n_thr);
      });
    for (auto& th : pool) th.join();
    CU(c, cudaStreamSynchronize(c->stream));
    if (err) return fail(c, SDBG_ECUDA, "copying the hits back failed");
  }
  return SDBG_OK;
}

// The top-k entries' region at d: [keys [nq][k] | total [nq] | n_out [nq]], nq * (8k + 12) bytes.
TopkDevOut topk_region(void* d, size_t nq, uint32_t k) {
  char* p = static_cast<char*>(d);
  const size_t kb = nq * size_t(k) * 8;
  return {reinterpret_cast<unsigned long long*>(p), reinterpret_cast<uint32_t*>(p + kb + nq * 8),
          reinterpret_cast<unsigned long long*>(p + kb)};
}

// Queues a batch that passed topk_args and topk_checked into the region dev: topk_run for a whole batch, else shape by
// shape through shapes_run. Nothing waits.
int topk_batch_run(sdbg_segment* const* segs, size_t n_segs, const PassBatch<sdbg_bm25_term>& B, float k1, float b,
                   const sdbg_col_pred* filt, uint32_t k, float threshold_in, const TopkDevOut& dev) {
  if (B.whole.nq) return topk_run(segs, n_segs, B.whole, B.total_excl, k1, b, filt, k, threshold_in, dev);
  return shapes_run(segs[0]->ctx, B.S, {size_t(k) * 8, 8, 4}, {dev.keys, dev.total, dev.n_out}, [&](int sh, void* const* part) {
    const TopkDevOut o{static_cast<unsigned long long*>(part[0]), static_cast<uint32_t*>(part[2]),
                       static_cast<unsigned long long*>(part[1])};
    return topk_run(segs, n_segs, B.S.view(sh), B.S.total_excl[sh], k1, b, filt, k, threshold_in, o);
  });
}

int topk_hits_to_host(sdbg_segment* const* segs, size_t n_segs, const TopkDevOut& dev, size_t nq, uint32_t k, sdbg_hit* out,
                      uint32_t* n_out, uint64_t* total_matches);

// The host top-k entries after topk_args and their batch (B): runs it into the call's region in c->pass[0]
// (topk_region, topk_batch_run), and copies it back (topk_to_host) with each ordinal decoded into {segment, doc}.
int topk_batch_host(sdbg_segment* const* segs, size_t n_segs, const PassBatch<sdbg_bm25_term>& B, float k1, float b,
                    const sdbg_col_pred* filt, uint32_t k, float threshold_in, sdbg_hit* out, uint32_t* n_out,
                    uint64_t* total_matches) {
  if (int rc = topk_checked(segs, n_segs, B)) return rc;
  sdbg_ctx* c = segs[0]->ctx;
  const size_t nq = B.nq;
  if (int rc = ensure(c, c->pass[0], nq * (size_t(k) * 8 + 12))) return rc;
  const TopkDevOut dev = topk_region(c->pass[0].p, nq, k);
  if (int rc = topk_batch_run(segs, n_segs, B, k1, b, filt, k, threshold_in, dev)) return rc;
  return topk_hits_to_host(segs, n_segs, dev, nq, k, out, n_out, total_matches);
}

// topk_to_host for the local entries: each ordinal decoded into {segment, doc}.
int topk_hits_to_host(sdbg_segment* const* segs, size_t n_segs, const TopkDevOut& dev, size_t nq, uint32_t k, sdbg_hit* out,
                      uint32_t* n_out, uint64_t* total_matches) {
  sdbg_ctx* c = segs[0]->ctx;
  std::vector<uint64_t> bases(n_segs);   // the first ordinal of each segment
  uint64_t ord0 = 0;
  for (size_t si = 0; si < n_segs; ++si) { bases[si] = ord0; ord0 += segs[si]->n_docs; }
  return topk_to_host(c, dev, nq, k, [&](uint32_t ordinal) {
    if (n_segs == 1) return make_uint2(0u, ordinal);   // one segment: no search for the owner of an ordinal
    const size_t seg = std::upper_bound(bases.begin(), bases.end(), uint64_t(ordinal) - 1) - bases.begin() - 1;
    return make_uint2(uint32_t(seg), uint32_t(ordinal - bases[seg]));
  }, out, n_out, total_matches);
}

}  // namespace

extern "C" int sdbg_bm25_collect(uint64_t docs_with_field, uint64_t total_term_freq, uint64_t docs_with_term, float k, float b,
                                 sdbg_bm25_term* out) {
  if (!out || docs_with_term > docs_with_field) return SDBG_EINVAL;
  // bm25.cpp:288-309, operation for operation (host code is built with -ffp-contract=off)
  out->idf = float(std::log1p((double(docs_with_field - docs_with_term) + 0.5) / (double(docs_with_term) + 0.5)));
  const float kb = k * b;
  out->norm_const = k - kb;
  if (total_term_freq && docs_with_field) {
    const float avg_dl = float(total_term_freq) / float(docs_with_field);
    out->norm_length = kb / avg_dl;
  } else {
    out->norm_length = kb;
  }
  out->boost = 1.f;
  return SDBG_OK;
}

// TFIDF (search/tfidf.cpp): idf = (float) log1p((docs_with_field + 1.0) / (docs_with_term + 1.0)), :149-150.
extern "C" int sdbg_tfidf_collect(uint64_t docs_with_field, uint64_t docs_with_term, sdbg_bm25_term* out) {
  if (!out) return SDBG_EINVAL;
  out->idf = float(std::log1p((double(docs_with_field) + 1.0) / (double(docs_with_term) + 1.0)));
  out->norm_const = 0.f; out->norm_length = 0.f; out->boost = 1.f;
  return SDBG_OK;
}

extern "C" int sdbg_bm25_topk_batch(sdbg_segment* const* segs, size_t n_segs, int kind, const sdbg_bm25_term* terms,
                                    const uint32_t* term_off, size_t nq, float k1, float b, const sdbg_col_pred* filt,
                                    uint32_t k, float threshold_in, sdbg_hit* out, uint32_t* n_out, uint64_t* total_matches);
// Same scan, scored with TFIDF: sqrt(freq) * boost * idf, divided by sqrt(doc length) when `normalize` (tfidf.cpp:59-80).
// Exhaustive (the segment's block-max entries belong to BM25).
extern "C" int sdbg_tfidf_topk_batch(sdbg_segment* const* segs, size_t n_segs, int kind, const sdbg_bm25_term* terms,
                                     const uint32_t* term_off, size_t nq, int normalize, const sdbg_col_pred* filt, uint32_t k,
                                     float threshold_in, sdbg_hit* out, uint32_t* n_out, uint64_t* total_matches) {
  return sdbg_bm25_topk_batch(segs, n_segs, kind, terms, term_off, nq, kTfidfK1, normalize ? 1.f : 0.f, filt, k, threshold_in, out, n_out,
                              total_matches);
}

extern "C" int sdbg_bm25_topk_batch(sdbg_segment* const* segs, size_t n_segs, int kind, const sdbg_bm25_term* terms,
                                    const uint32_t* term_off, size_t nq, float k1, float b, const sdbg_col_pred* filt,
                                    uint32_t k, float threshold_in, sdbg_hit* out, uint32_t* n_out,
                                    uint64_t* total_matches) {
  if (!out || !n_out) return SDBG_EINVAL;
  if (int rc = topk_args(segs, n_segs, nq, k)) return rc;
  const PassBatch<sdbg_bm25_term> B(segs, n_segs, {kind, terms, term_off, nq, nullptr, nullptr, nullptr}, filt);
  return topk_batch_host(segs, n_segs, B, k1, b, filt, k, threshold_in, out, n_out, total_matches);
}

extern "C" int sdbg_bm25_topk_batch_excl(sdbg_segment* const* segs, size_t n_segs, int kind, const sdbg_bm25_term* terms,
                                         const uint32_t* term_off, size_t nq, const uint32_t* excl_terms, const uint32_t* excl_off,
                                         float k1, float b, const sdbg_col_pred* filt, uint32_t k, float threshold_in, sdbg_hit* out,
                                         uint32_t* n_out, uint64_t* total_matches) {
  if (!excl_off || !out || !n_out) return SDBG_EINVAL;
  if (int rc = topk_args(segs, n_segs, nq, k)) return rc;
  const PassBatch<sdbg_bm25_term> B(segs, n_segs, {kind, terms, term_off, nq, excl_terms, excl_off, nullptr}, filt);
  return topk_batch_host(segs, n_segs, B, k1, b, filt, k, threshold_in, out, n_out, total_matches);
}

extern "C" int sdbg_bm25_topk_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const sdbg_bm25_term* terms,
                                               const uint32_t* group_off, const uint32_t* query_group_off, const uint32_t* group_min,
                                               size_t nq, const uint32_t* excl_terms, const uint32_t* excl_off, float k1, float b,
                                               const sdbg_col_pred* filt, uint32_t k, float threshold_in, sdbg_hit* out,
                                               uint32_t* n_out, uint64_t* total_matches) {
  if (!group_off || !query_group_off || !out || !n_out) return SDBG_EINVAL;
  if (int rc = topk_args(segs, n_segs, nq, k)) return rc;
  const PassBatch<sdbg_bm25_term> B(segs, n_segs, terms, group_off, query_group_off, group_min, nq, excl_terms, excl_off, filt);
  return topk_batch_host(segs, n_segs, B, k1, b, filt, k, threshold_in, out, n_out, total_matches);
}

extern "C" int sdbg_bm25_topk_batch_groups(sdbg_segment* const* segs, size_t n_segs, const sdbg_bm25_term* terms,
                                           const uint32_t* group_off, const uint32_t* query_group_off, size_t nq,
                                           const uint32_t* excl_terms, const uint32_t* excl_off, float k1, float b,
                                           const sdbg_col_pred* filt, uint32_t k, float threshold_in, sdbg_hit* out,
                                           uint32_t* n_out, uint64_t* total_matches) {
  return sdbg_bm25_topk_batch_groups_min(segs, n_segs, terms, group_off, query_group_off, nullptr, nq, excl_terms, excl_off, k1, b,
                                         filt, k, threshold_in, out, n_out, total_matches);
}

// Count mode (duckdb_search_full_scan RunCountScan): bm25_count_kernel over work items {query, first window, windows} of
// kCountWindow-doc windows, planned per segment from posting counts and issued largest first. A single-term query over a
// segment without filter, deleted docs or an excluded list holding blocks there is answered from the term's docs_count.
// Queries of OR groups (Q.term_grp; groups 0 .. n - 1 of a query all present) run the kGroups instantiations
// (CountPlan::kernel).
// The same plan serves three more passes (CountJob), without the single-term shortcut: the sorted scan of
// sdbg_match_topk_by_column_batch (sort_prepare), the facet pass of sdbg_match_facet_counts_batch
// (facet_prepare) and the aggregate pass of sdbg_match_aggregate_batch (agg_prepare).
namespace {

// The facet pass's part of a count_run call.
struct FacetJob {
  uint64_t field;
  int64_t key_min;
  uint32_t span;
  std::vector<FacetSink> sink;   // per segment, filled by facet_prepare (output pointers set at launch)
};

int facet_check_range(sdbg_ctx* c, int64_t key_min, uint32_t span, uint32_t max_span = kFacetMaxSpan) {
  if (span == 0) return fail(c, SDBG_EINVAL, "key_span is 0");
  if (key_min > INT64_MAX - int64_t(span - 1)) return fail(c, SDBG_EINVAL, "key_min + key_span - 1 overflows int64");
  if (span > max_span)
    return fail(c, SDBG_EUNSUPPORTED, "key_span > " + std::to_string(max_span) + " (the bins are shared memory)");
  return SDBG_OK;
}

// Checks the key range and the key column of every segment, then fills the per-segment sinks. Every check runs before
// anything is queued (a packed column's raw view is decoded on first use).
int facet_prepare(sdbg_ctx* c, sdbg_segment* const* segs, size_t n_segs, FacetJob& J) {
  if (int rc = facet_check_range(c, J.key_min, J.span)) return rc;
  for (size_t si = 0; si < n_segs; ++si) {
    auto it = segs[si]->cols.find(J.field);
    if (it == segs[si]->cols.end()) return fail(c, SDBG_ENOTFOUND, "key column not staged in every segment");
    if (it->second.type != segs[0]->cols.find(J.field)->second.type)
      return fail(c, SDBG_EINVAL, "key column type differs between segments");
  }
  if (segs[0]->cols.find(J.field)->second.type == SDBG_F64) return fail(c, SDBG_EUNSUPPORTED, "float64 key column");
  J.sink.assign(n_segs, FacetSink{});
  for (size_t si = 0; si < n_segs; ++si) {
    ColumnObj& col = segs[si]->cols.find(J.field)->second;
    FacetSink& F = J.sink[si];
    void* raw = nullptr;
    if (int rc = raw_values(c, col, &raw)) return rc;
    F.values = raw; F.validity = reinterpret_cast<const unsigned long long*>(col.d_validity); F.rows = col.rows;
    F.type = uint32_t(col.type); F.span = J.span; F.key_min = J.key_min;
  }
  return SDBG_OK;
}

// The aggregate pass's part of a count_run call.
struct AggJob {
  FacetJob key;               // key column and range (key.field UINT64_MAX: one group)
  uint64_t field;             // value column
  std::vector<AggSink> sink;  // per segment, filled by agg_prepare (output pointers set at launch)
};

// The key range of an aggregate call: a key column's range as for the facet pass (at most kAggMaxSpan keys); no key
// column: exactly (0, 1).
int agg_check_range(sdbg_ctx* c, uint64_t key_field, int64_t key_min, uint32_t span) {
  if (key_field == UINT64_MAX)
    return key_min == 0 && span == 1 ? SDBG_OK : fail(c, SDBG_EINVAL, "an ungrouped aggregate needs key_min 0 and key_span 1");
  return facet_check_range(c, key_min, span, kAggMaxSpan);
}

// Checks the key range, the key column (facet_prepare) and the value column of every segment, then fills the
// per-segment sinks. Every check runs before anything is queued.
int agg_prepare(sdbg_ctx* c, sdbg_segment* const* segs, size_t n_segs, AggJob& J) {
  if (int rc = agg_check_range(c, J.key.field, J.key.key_min, J.key.span)) return rc;
  for (size_t si = 0; si < n_segs; ++si) {
    auto it = segs[si]->cols.find(J.field);
    if (it == segs[si]->cols.end()) return fail(c, SDBG_ENOTFOUND, "value column not staged in every segment");
    if (it->second.type != segs[0]->cols.find(J.field)->second.type)
      return fail(c, SDBG_EINVAL, "value column type differs between segments");
  }
  if (J.key.field != UINT64_MAX)
    if (int rc = facet_prepare(c, segs, n_segs, J.key)) return rc;
  J.sink.assign(n_segs, AggSink{});
  for (size_t si = 0; si < n_segs; ++si) {
    ColumnObj& col = segs[si]->cols.find(J.field)->second;
    AggSink& A = J.sink[si];
    if (J.key.field != UINT64_MAX) A.key = J.key.sink[si];
    else A.key.span = 1;
    void* raw = nullptr;
    if (int rc = raw_values(c, col, &raw)) return rc;
    A.values = raw; A.validity = reinterpret_cast<const unsigned long long*>(col.d_validity); A.rows = col.rows;
    A.type = uint32_t(col.type);
  }
  return SDBG_OK;
}

// One output cell as the caller sees it: the limbs and order keys of AggCell turned into values; zeros when no value.
sdbg_match_agg agg_result(const AggCell& g, uint32_t type) {
  sdbg_match_agg a{};
  a.count = g.count;
  a.count_value = g.count_value;
  if (!g.count_value) return a;
  if (type == SDBG_F64) std::memcpy(&a.sum_f64, &g.sum_lo, 8);
  else { a.sum_i128[0] = int64_t(g.sum_lo); a.sum_i128[1] = int64_t(g.sum_hi); }
  a.min = int64_t(sort_order_value(~g.nmin, type));
  a.max = int64_t(sort_order_value(g.max, type));
  return a;
}

// The caller's cells from the device's: out [nq][span] from g [nq][span], null_out [nq] from the NULL cells after them.
void agg_results(const AggCell* g, size_t nq, uint32_t span, uint32_t type, sdbg_match_agg* out, sdbg_match_agg* null_out) {
  for (size_t i = 0; i < nq * span; ++i) out[i] = agg_result(g[i], type);
  for (size_t q = 0; q < nq; ++q) null_out[q] = agg_result(g[nq * span + q], type);
}

// The sorted scan's part of a count_run call.
struct SortJob {
  uint64_t field;
  int desc, nulls_first;
  uint32_t k;
  // filled by sort_prepare
  std::vector<SortSink> sink;                 // per segment (pointers to outputs set at launch)
  std::vector<std::vector<long long>> zone;   // per segment: host copy of the zonemap (empty: no zone pruning there)
};
static_assert(sizeof(sdbg_sort_hit) == sizeof(SortHitDev), "sdbg_sort_hit layout");

// Checks the sort column of every segment and fills the per-segment sinks. With pruning, NOT NULL columns get their
// zonemap (built on first use, as the GROUP BY scan builds it), and a host copy of it for planning.
int sort_prepare(sdbg_ctx* c, sdbg_segment* const* segs, size_t n_segs, SortJob& J) {
  J.sink.assign(n_segs, SortSink{});
  J.zone.assign(n_segs, {});
  // all checks first: nothing is queued before a call can fail
  uint64_t total_docs = 0;
  for (size_t si = 0; si < n_segs; ++si) {
    auto it = segs[si]->cols.find(J.field);
    if (it == segs[si]->cols.end()) return fail(c, SDBG_ENOTFOUND, "sort column not staged in every segment");
    if (it->second.type != segs[0]->cols.find(J.field)->second.type)
      return fail(c, SDBG_EINVAL, "sort column type differs between segments");
    total_docs += segs[si]->n_docs;
  }
  // ordinals reach total_docs - 1 <= 2^32 - 3, so ~ordinal (the key's lo) stays non-zero
  if (total_docs > kMaxDocId) return fail(c, SDBG_EUNSUPPORTED, "more than 2^32-2 docs per call");
  uint32_t base = 0;   // ordinals of the earlier segments (the total fits in 32 bits)
  for (size_t si = 0; si < n_segs; ++si) {
    ColumnObj& col = segs[si]->cols.find(J.field)->second;
    SortSink& S = J.sink[si];
    void* raw = nullptr;
    if (int rc = raw_values(c, col, &raw)) return rc;
    S.values = raw; S.validity = reinterpret_cast<const unsigned long long*>(col.d_validity); S.rows = col.rows; S.type = uint32_t(col.type);
    S.desc = J.desc ? 1u : 0u; S.nulls_first = J.nulls_first ? 1u : 0u;
    S.ordinal_base = base; S.k = J.k;
    uint32_t kp = 1;
    while (kp < J.k) kp <<= 1;
    S.cap = std::max(256u, 2u * kp);
    base += segs[si]->n_docs;
    if (!c->wand || col.d_validity || !col.rows) continue;
    const uint64_t n_zones = (col.rows + kZoneRows - 1) / kZoneRows;
    if (int rc = column_zonemap(c, col, &S.zone)) return rc;
    S.n_zones = uint32_t(n_zones);
  }
  // host copies of the zonemaps last, and always waited for: J.zone must outlive every queued copy
  cudaError_t e = cudaSuccess;
  for (size_t si = 0; si < n_segs; ++si) {
    if (!J.sink[si].zone) continue;
    J.zone[si].resize(size_t(J.sink[si].n_zones) * 2);
    if (e == cudaSuccess)
      e = cudaMemcpyAsync(J.zone[si].data(), J.sink[si].zone, size_t(J.sink[si].n_zones) * 16, cudaMemcpyDeviceToHost, c->stream);
  }
  const cudaError_t e2 = cudaStreamSynchronize(c->stream);
  CU(c, e);
  CU(c, e2);
  return SDBG_OK;
}

// Best zonemap bound (sort_zone_bound) of window w of segment si's sink, over a host copy of the zonemap.
unsigned long long sort_window_bound(const SortJob& J, size_t si, uint32_t w) {
  SortSink S = J.sink[si];
  S.zone = J.zone[si].data();
  const uint32_t ws = w << kCountWindowLog, zb = ws == 0u ? 0u : (ws >> 11) - 1u, nz = ws == 0u ? 32u : 33u;
  unsigned long long b = 0;
  for (uint32_t z = zb; z < zb + nz; ++z) b = std::max(b, sort_zone_bound(S, z));
  return b;
}

struct CountItem { uint32_t q, w0, nw; uint64_t weight; bool seed = false; };

// Raises `kernel`'s dynamic shared memory limit to `bytes` when a launch with them needs it: by default a launch may
// take 48 KB minus the kernel's static shared memory (9.1 / 17.4 KB for the count kernels).
template <class Kernel>
cudaError_t fit_dynamic_smem(Kernel* kernel, size_t bytes) {
  cudaFuncAttributes a;
  cudaError_t e = cudaFuncGetAttributes(&a, kernel);
  if (e == cudaSuccess && bytes + a.sharedSizeBytes > 48 * 1024)
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(bytes));
  return e;
}

// Planes of the bit-sliced counter for groups that need up to max_min of their lists: bits(max_min), none for 1.
uint32_t count_planes(uint32_t max_min) {
  uint32_t planes = 0;
  if (max_min > 1u)
    while ((max_min >> planes) != 0u) ++planes;
  return planes;
}

using CountKernel = void (*)(CountParams);
enum class CountMode { count, sort, facet, agg, emit, phrase };

// The match scan's part of a count_run call: the page of each query of the plan's batch.
struct EmitJob {
  uint32_t limit;
  const unsigned long long* offset;   // host [nq]: the first ordinal of each query's page
};

// The phrase pass's part of a count_run call (the plan's batch is the candidate batch of PhraseBatch::candidates): batch
// query b's alternatives are [query_off[b] .. query_off[b + 1]), alternative j's slots slot_term / slot_rel
// [clause_off[j] .. clause_off[j + 1]), with flags[j] = kAltNegated | group << 1 | kAltGuaranteed | (m - 1) <<
// kAltMinShift (bm25_phrase.cuh); write adds each entry's need.
// The job's queries are the batch's at positions qpos (null: all of them), so a
// shape of a mixed batch runs the job of its own queries. k == 0: count only; else the top-k, scored with consts[j] =
// {c0, norm_const, norm_length} per alternative and seeded with the key of threshold_in.
struct PhraseJob {
  const uint32_t* slot_term = nullptr;
  const uint32_t* slot_rel = nullptr;
  const uint32_t* clause_off = nullptr;
  const uint32_t* flags = nullptr;
  const uint32_t* query_off = nullptr;
  const uint32_t* qpos = nullptr;
  size_t nq = 0;        // the job's queries
  uint32_t n_alts = 0;  // the batch's alternatives, query_off[its nq]
  std::vector<float4> consts;
  uint32_t k = 0;
  unsigned long long seed = 0;

  uint32_t n_clauses() const { return n_alts; }
  uint32_t n_slots() const { return clause_off[n_alts]; }
  uint32_t batch_query(size_t q) const { return qpos ? qpos[q] : uint32_t(q); }

  // The job for the batch's queries at positions qs.
  PhraseJob on(const std::vector<uint32_t>& qs) const {
    PhraseJob J = *this;
    J.qpos = qs.data();
    J.nq = qs.size();
    return J;
  }

  // The job's device tables, staged as [per query its table offsets | per segment the alternative tables | per segment
  // the slots' lists | per alternative consts], from a 16-B aligned offset.
  size_t clauses_pos() const { return ((nq + 1) * 4 + 15) & ~size_t(15); }
  size_t lists_pos(size_t n_segs) const { return clauses_pos() + n_segs * n_clauses() * sizeof(uint4); }
  size_t consts_pos(size_t n_segs) const { return lists_pos(n_segs) + n_segs * n_slots() * sizeof(uint4); }
  size_t bytes(size_t n_segs) const { return consts_pos(n_segs) + (consts.empty() ? 0 : n_clauses() * sizeof(float4)); }
  void write(sdbg_segment* const* segs, size_t n_segs, char* h, bool conj) const;

  // Segment si's view of the tables staged at d for the kernels' PhraseSink.
  void sink(sdbg_segment* const* segs, size_t n_segs, size_t si, const char* d, PhraseSink& F) const {
    F.pos_base = static_cast<const unsigned long long*>(segs[si]->d_pos_base);
    F.pos = static_cast<const uint32_t*>(segs[si]->d_pos);
    F.clause_off = reinterpret_cast<const uint32_t*>(d);
    F.clauses = reinterpret_cast<const uint4*>(d + clauses_pos()) + si * n_clauses();
    F.slots = reinterpret_cast<const uint4*>(d + lists_pos(n_segs)) + si * n_slots();
    F.consts = consts.empty() ? nullptr : reinterpret_cast<const float4*>(d + consts_pos(n_segs));
  }
};

// One pass of count_run: its mode and that mode's parameters. job_prepare checks them and fills the sinks, once per call.
struct CountJob {
  CountMode mode;
  SortJob sort;     // CountMode::sort
  FacetJob facet;   // CountMode::facet
  AggJob agg;       // CountMode::agg
  EmitJob emit;     // CountMode::emit
  PhraseJob phrase; // CountMode::phrase

  // Bytes per query of count_run's per-query arrays {counts, bins, nulls} (CountOut); rank: the sorted scan's rank form.
  std::array<size_t, 3> rows(bool rank) const {
    switch (mode) {
      case CountMode::sort: return {rank ? 8u : 4u, size_t(sort.k) * (rank ? sizeof(SortDistRow) : sizeof(SortHitDev)), 0};
      case CountMode::facet: return {8, size_t(facet.span) * 8, 8};
      case CountMode::agg: return {8, size_t(agg.key.span) * sizeof(AggCell), sizeof(AggCell)};
      case CountMode::emit: return {8, size_t(emit.limit) * sizeof(EmitHit), 4};
      case CountMode::phrase: return {8, size_t(phrase.k) * 8, phrase.k ? 4u : 0u};
      default: return {8, 0, 0};
    }
  }
};

int job_prepare(sdbg_ctx* c, sdbg_segment* const* segs, size_t n_segs, CountJob& job) {
  switch (job.mode) {
    case CountMode::sort: return sort_prepare(c, segs, n_segs, job.sort);
    case CountMode::facet: return facet_prepare(c, segs, n_segs, job.facet);
    case CountMode::agg: return agg_prepare(c, segs, n_segs, job.agg);
    default: return SDBG_OK;
  }
}

// Where count_run leaves a pass's results: device arrays the caller has zeroed, which the pass adds to. Nothing is copied
// back and nothing waits (the sorted scan's zonemap planning in sort_prepare excepted), so a collective can follow.
struct CountOut {
  void* counts;                // [nq]: count u64 counts; facet / aggregate u64 scratch; sorted scan u32 n_out (rank < 0) or
                               // u64 row counts; match scan u64 totals
  void* bins;                  // facet u64 [nq][span], aggregate AggCell [nq][span]; sorted scan SortHitDev [nq][k] (rank < 0)
                               // or SortDistRow [nq][k]; match scan EmitHit [nq][limit]
  void* nulls;                 // facet u64 [nq], aggregate AggCell [nq]; match scan u32 n_out [nq]
  unsigned int* oor;           // facet / aggregate: set to 1 when a matching doc's key lies outside the range
  unsigned long long* stats;   // sorted scan: windows judged / skipped by the zonemaps
  int64_t rank;                // sorted scan: < 0 hits, else this rank's rows (sort_dist_rows_kernel)
};

// A count_run plan: per segment each query's lists and the work items; with OR groups (Q.term_grp), each segment's group
// ends. Its host staging, which every mode shares: [term_off | excl_off | lists per segment | work items {query, first
// window, windows, 0} | grp_off | group ends per segment]; the sorted scan appends its own arrays.
struct CountPlan {
  QueryBatch<uint32_t> Q;
  uint32_t n_pos, total_excl;
  uint32_t planes;                               // of the bit-sliced counter, for the batch's largest group minimum
  std::vector<uint2> lists;                      // per segment: positive lists | excluded lists
  std::vector<std::vector<CountItem>> seg_work;  // per segment
  std::vector<uint32_t> grp_off, grp_end;        // grp_off[q] .. grp_off[q + 1] index each segment's group ends
  std::vector<uint64_t> host;                    // per query: the counts of the single-term shortcut
  size_t items = 0;                              // work items over all segments
  size_t off_bytes = 0, lists_pos = 0, work_pos = 0, grp_pos = 0, staged = 0;   // the staging's layout; staged: its bytes

  size_t n_lists() const { return size_t(n_pos) + total_excl; }

  void layout() {
    size_t items = 0;
    for (const auto& w : seg_work) items += w.size();
    off_bytes = (Q.nq + 1) * 4;
    lists_pos = (2 * off_bytes + 7) & ~size_t(7);
    work_pos = (lists_pos + lists.size() * sizeof(uint2) + 15) & ~size_t(15);
    grp_pos = work_pos + items * sizeof(uint4);
    staged = grp_pos + (Q.term_grp ? off_bytes + grp_end.size() * 4 : 0);
  }

  void write(char* h) const {
    std::memcpy(h, Q.term_off, off_bytes);
    if (total_excl) std::memcpy(h + off_bytes, Q.excl_off, off_bytes);
    std::memcpy(h + lists_pos, lists.data(), lists.size() * sizeof(uint2));
    auto* hw = reinterpret_cast<uint4*>(h + work_pos);
    for (const auto& w : seg_work) for (const CountItem& it : w) *hw++ = make_uint4(it.q, it.w0, it.nw, 0u);
    if (Q.term_grp) {
      std::memcpy(h + grp_pos, grp_off.data(), off_bytes);
      std::memcpy(h + grp_pos + off_bytes, grp_end.data(), grp_end.size() * 4);
    }
  }

  // The parameters of segment si's launch over its work items from `first` on, d the device copy of the staging.
  void params(const char* d, sdbg_segment* s, size_t si, size_t first, const ChainDev& filt, CountParams* P) const {
    P->seg = postings_view(s, 0);
    P->filt = filt;
    P->lists = reinterpret_cast<const uint2*>(d + lists_pos) + si * n_lists();
    P->term_off = reinterpret_cast<const uint32_t*>(d);
    P->excl_off = total_excl ? reinterpret_cast<const uint32_t*>(d + off_bytes) : nullptr;
    P->n_pos = n_pos;
    P->work = reinterpret_cast<const uint4*>(d + work_pos) + first;
    if (Q.term_grp) {
      P->grp_off = reinterpret_cast<const uint32_t*>(d + grp_pos);
      P->grp_end = reinterpret_cast<const uint32_t*>(d + grp_pos + off_bytes) + si * grp_off[Q.nq];
    }
  }

  // The bm25_count_kernel instantiation of this plan's launches in `mode`, with its dynamic shared memory: the mode's
  // own bytes (facet bins, sorted keys, aggregate cells, the phrase sink's keys; none for a count), then the counter
  // planes. phrased: the plan's batch is the candidates of phrase alternatives, checked by the phrase sink
  // (CountMode::phrase) or before / in another sink.
  std::pair<CountKernel, size_t> kernel(CountMode mode, size_t mode_bytes, bool phrased = false) const {
    static const CountKernel kernels[3][5] = {   // [OR | AND | OR groups][count | sort | facet | agg | emit]
        {bm25_count_kernel<false>, bm25_count_kernel<false, false, true>, bm25_count_kernel<false, false, false, true>,
         bm25_count_kernel<false, false, false, false, true>, bm25_count_kernel<false, false, false, false, false, true>},
        {bm25_count_kernel<true>, bm25_count_kernel<true, false, true>, bm25_count_kernel<true, false, false, true>,
         bm25_count_kernel<true, false, false, false, true>, bm25_count_kernel<true, false, false, false, false, true>},
        {bm25_count_kernel<false, true>, bm25_count_kernel<false, true, true>, bm25_count_kernel<false, true, false, true>,
         bm25_count_kernel<false, true, false, false, true>, bm25_count_kernel<false, true, false, false, false, true>}};
    // [OR | AND | OR groups][phrase sink | sort | facet | agg | emit] of phrase alternatives' candidates
    static const CountKernel phrase_kernels[3][5] = {
        {bm25_count_kernel<false, false, false, false, false, false, true>, bm25_count_kernel<false, false, true, false, false, false, true>,
         bm25_count_kernel<false, false, false, true, false, false, true>, bm25_count_kernel<false, false, false, false, true, false, true>,
         bm25_count_kernel<false, false, false, false, false, true, true>},
        {bm25_count_kernel<true, false, false, false, false, false, true>, bm25_count_kernel<true, false, true, false, false, false, true>,
         bm25_count_kernel<true, false, false, true, false, false, true>, bm25_count_kernel<true, false, false, false, true, false, true>,
         bm25_count_kernel<true, false, false, false, false, true, true>},
        {bm25_count_kernel<false, true, false, false, false, false, true>, bm25_count_kernel<false, true, true, false, false, false, true>,
         bm25_count_kernel<false, true, false, true, false, false, true>, bm25_count_kernel<false, true, false, false, true, false, true>,
         bm25_count_kernel<false, true, false, false, false, true, true>}};
    const int shape = Q.term_grp ? 2 : Q.kind == SDBG_QUERY_AND ? 1 : 0;
    const CountKernel k = mode == CountMode::phrase ? phrase_kernels[shape][0] : phrased ? phrase_kernels[shape][int(mode)]
                                                                                          : kernels[shape][int(mode)];
    return {k, mode_bytes + size_t(planes) * kCountWords * 4u};
  }
};

// The plan of a batch checked by check_query_batch (total_excl: what it set) for a prepared job (job_prepare), on the
// host: queues nothing.
CountPlan count_plan(sdbg_segment* const* segs, size_t n_segs, const QueryBatch<uint32_t>& Q, uint32_t total_excl,
                     const sdbg_col_pred* filt, const CountJob& job) {
  const auto& [kind, terms, term_off, nq, excl_terms, excl_off, term_grp] = Q;
  sdbg_ctx* c = segs[0]->ctx;
  const SortJob* sort = job.mode == CountMode::sort ? &job.sort : nullptr;
  const bool conj = kind == SDBG_QUERY_AND;
  const uint32_t n_pos = term_off[nq];
  const size_t n_lists = size_t(n_pos) + total_excl;   // per segment: positive lists | excluded lists

  std::vector<uint64_t> host(nq, 0);                    // shortcut counts
  using Item = CountItem;
  // Sorted scan with zonemaps: one seed window per call, the one whose zones can hold the best value (first segment,
  // then first window, on ties), split off every query's item that holds it. Seed items run first, so each query's
  // threshold is known before its other windows are judged: a sort that prefers the last rows ("newest first") would
  // otherwise only find its best values at the end of the scan (measured: 196 against 94 ms per step, DESIGN §4.9).
  std::vector<uint32_t> best_win(n_segs, UINT32_MAX);
  size_t seed_seg = SIZE_MAX;
  if (sort) {
    unsigned long long best = 0;
    for (size_t si = 0; si < n_segs; ++si) {
      if (sort->zone[si].empty()) continue;
      const uint32_t n_win = (segs[si]->n_docs >> kCountWindowLog) + 1u;
      unsigned long long sb = 0;
      for (uint32_t w = 0; w < n_win; ++w) {
        const unsigned long long b = sort_window_bound(*sort, si, w);
        if (best_win[si] == UINT32_MAX || b > sb) { sb = b; best_win[si] = w; }
      }
      if (seed_seg == SIZE_MAX || sb > best) { best = sb; seed_seg = si; }
    }
  }
  std::vector<std::vector<Item>> seg_work(n_segs);
  std::vector<uint2> lists(n_lists * n_segs);
  // OR groups: grp_off[q] .. grp_off[q + 1] index each segment's group ends (relative to term_off[q]), lead group first
  std::vector<uint32_t> grp_off, grp_end;
  uint32_t max_min = 1;   // largest group minimum of the batch: sizes the count kernel's bit-sliced counter
  if (term_grp) {
    grp_off.assign(nq + 1, 0u);
    for (size_t q = 0; q < nq; ++q) {
      uint32_t ng = 0;
      for (uint32_t i = term_off[q]; i < term_off[q + 1]; ++i) {
        ng = std::max(ng, uint32_t(term_grp[i] & 15u) + 1u);
        max_min = std::max(max_min, uint32_t(term_grp[i] >> 4) + 1u);
      }
      grp_off[q + 1] = grp_off[q] + ng;
    }
    grp_end.assign(size_t(grp_off[nq]) * n_segs, 0u);
  }
  uint64_t batch_postings = 0;
  for (size_t si = 0; si < n_segs; ++si)
    for (uint32_t i = term_off[0]; i < n_pos; ++i) batch_postings += segs[si]->term_docs[terms[i]];
  const uint64_t chain_target = std::max<uint64_t>(65536, batch_postings / (uint64_t(c->sm_count) * 4u));
  const uint32_t G = uint32_t(std::max<size_t>(1, (size_t(c->sm_count) * 8u + nq - 1) / nq));
  size_t total_items = 0;
  for (size_t si = 0; si < n_segs; ++si) {
    const sdbg_segment* s = segs[si];
    uint2* L = lists.data() + si * n_lists;
    for (uint32_t i = 0; i < total_excl; ++i) L[n_pos + i] = excl_list(s, excl_terms[i]);
    const uint32_t n_win = (s->n_docs >> kCountWindowLog) + 1u;
    for (size_t q = 0; q < nq; ++q) {
      const uint32_t t0 = term_off[q], t1 = term_off[q + 1];
      uint64_t sum = 0;
      uint32_t smallest = UINT32_MAX;
      std::array<std::pair<uint32_t, uint2>, kMaxQueryTerms> by_docs;
      for (uint32_t i = t0; i < t1; ++i) {
        const uint32_t dc = s->term_docs[terms[i]];
        by_docs[i - t0] = {dc, excl_list(s, terms[i])};
        sum += dc;
        smallest = std::min(smallest, dc);
      }
      uint64_t weight;
      if (term_grp) {
        // Each group's lists by ascending docs_count; a group of s lists that needs m of them costs its s - m + 1
        // shortest lists (all of them for m = 1), which is what it leads with. Groups by ascending cost: the lead group
        // (the cheapest) fills the window bitmap and the most selective groups narrow it first.
        const uint32_t ng = grp_off[q + 1] - grp_off[q];
        std::array<uint64_t, kMaxQueryTerms> gsum{};
        std::array<uint32_t, kMaxQueryTerms> order{}, gsize{}, gmin{}, gnz{}, seen{};
        std::array<uint32_t, kMaxQueryTerms> by_cost{};   // positions i - t0, ascending docs_count
        for (uint32_t i = t0; i < t1; ++i) {
          const uint32_t g = term_grp[i] & 15u;
          by_cost[i - t0] = i - t0;
          gmin[g] = (term_grp[i] >> 4) + 1u;
          ++gsize[g];
          gnz[g] += by_docs[i - t0].first != 0u;
        }
        std::stable_sort(by_cost.begin(), by_cost.begin() + (t1 - t0), [&](uint32_t a, uint32_t b) { return by_docs[a].first < by_docs[b].first; });
        for (uint32_t j = 0; j < t1 - t0; ++j) {
          const uint32_t g = term_grp[t0 + by_cost[j]] & 15u;
          if (seen[g]++ < gsize[g] - gmin[g] + 1u) gsum[g] += by_docs[by_cost[j]].first;
        }
        bool short_group = false;
        for (uint32_t g = 0; g < ng; ++g) short_group |= gnz[g] < gmin[g];
        for (uint32_t g = 0; g < ng; ++g) order[g] = g;
        std::stable_sort(order.begin(), order.begin() + ng, [&](uint32_t a, uint32_t b) { return gsum[a] < gsum[b]; });
        uint32_t* gend = grp_end.data() + si * grp_off[nq] + grp_off[q];
        uint32_t o = 0;
        for (uint32_t j = 0; j < ng; ++j) {
          for (uint32_t x = 0; x < t1 - t0; ++x)
            if ((term_grp[t0 + by_cost[x]] & 15u) == order[j]) L[t0 + o++] = by_docs[by_cost[x]].second;
          gend[j] = o | ((gmin[order[j]] - 1u) << 8);
        }
        if (short_group) continue;                       // a group with fewer than m non-empty lists here: no match
        weight = gsum[order[0]] * ng;
      } else {
        // ascending docs_count: the shortest list of a conjunction fills the window bitmap
        std::stable_sort(by_docs.begin(), by_docs.begin() + (t1 - t0), [](const auto& a, const auto& b) { return a.first < b.first; });
        for (uint32_t i = t0; i < t1; ++i) L[i] = by_docs[i - t0].second;
        if (conj ? smallest == 0 : sum == 0) continue;
        bool excl_blocks = false;
        if (total_excl)
          for (uint32_t i = excl_off[q]; i < excl_off[q + 1]; ++i) excl_blocks |= L[n_pos + i].y != 0;
        if (t1 - t0 == 1 && !filt && !s->d_deleted && !excl_blocks && job.mode == CountMode::count) { host[q] += sum; continue; }
        weight = conj ? uint64_t(smallest) * (t1 - t0) : sum;
      }
      uint32_t g = uint32_t(std::max<uint64_t>(G, (weight + chain_target - 1) / chain_target));
      g = std::min({g, n_win, 2u * uint32_t(c->sm_count)});
      const uint32_t per = (n_win + g - 1) / g;
      for (uint32_t w0 = 0; w0 < n_win; w0 += per) {
        const uint32_t nw = std::min(per, n_win - w0), sw = best_win[si];
        // A query with one item in one segment that starts at the seed visits it first anyway: splitting would only
        // add an item and a launch.
        const bool first_anyway = n_segs == 1 && g == 1 && sw == w0;
        if (si != seed_seg || sw < w0 || sw >= w0 + nw || first_anyway) {
          seg_work[si].push_back({uint32_t(q), w0, nw, weight / g});
          continue;
        }
        // the item holding the seed window: [w0, sw) | seed | (sw, w0 + nw)
        if (sw > w0) seg_work[si].push_back({uint32_t(q), w0, sw - w0, weight / g});
        seg_work[si].push_back({uint32_t(q), sw, 1u, weight / g, true});
        if (sw + 1u < w0 + nw) seg_work[si].push_back({uint32_t(q), sw + 1u, w0 + nw - sw - 1u, weight / g});
      }
    }
    std::stable_sort(seg_work[si].begin(), seg_work[si].end(), [](const Item& x, const Item& y) { return x.weight > y.weight; });
    std::stable_partition(seg_work[si].begin(), seg_work[si].end(), [](const Item& x) { return x.seed; });
    total_items += seg_work[si].size();
  }
  CountPlan pl{Q, n_pos, total_excl, count_planes(max_min), std::move(lists), std::move(seg_work), std::move(grp_off),
               std::move(grp_end), std::move(host), total_items};
  pl.layout();
  return pl;
}

// The item slots of the plan's staging h: each work item's output slot is its index (work item .w), and query q's items
// are slots[slot_off[q] .. slot_off[q + 1]) in work order, i.e. by segment, then first window.
void item_slots(const CountPlan& pl, char* h, size_t slot_off_pos, size_t slots_pos) {
  const size_t nq = pl.Q.nq, total = pl.items;
  auto* hw = reinterpret_cast<uint4*>(h + pl.work_pos);
  auto* h_slot_off = reinterpret_cast<uint32_t*>(h + slot_off_pos);
  auto* h_slots = reinterpret_cast<uint32_t*>(h + slots_pos);
  std::fill(h_slot_off, h_slot_off + nq + 1, 0u);
  for (uint32_t i = 0; i < total; ++i) { hw[i].w = i; ++h_slot_off[hw[i].x + 1]; }
  for (size_t q = 0; q < nq; ++q) h_slot_off[q + 1] += h_slot_off[q];
  std::vector<uint32_t> fillq(h_slot_off, h_slot_off + nq);
  for (uint32_t i = 0; i < total; ++i) h_slots[fillq[hw[i].x]++] = i;
}

// The tables of PhraseJob::bytes at h. Per query of the job its table offsets. Per segment: each
// slot's list {first BlockDesc, blocks, rel_pos, 0}, and each query's alternatives {first slot, slots, flags, alternative
// index} in that segment's cost order, the smallest docs_count of the alternative's terms (a term the segment does not
// hold costs 0), ascending, ties in query order: the order of a conjunction of the terms' lists
// (conjunction.hpp:185-195), in which the scores of the matching positive alternatives are summed; each positive entry
// gets its `need` (kAltNeedShift) from the positive entries of its group after it. conj: the job's candidates are the AND
// (every positive group one alternative), whose
// walk (phrase_clauses<false>) reads the flags as the negated bit alone. Slots before the batch's first query's are left
// as they are.
void PhraseJob::write(sdbg_segment* const* segs, size_t n_segs, char* h, bool conj) const {
  const uint32_t nc = n_clauses(), ns = n_slots(), c0 = query_off[0];
  auto* off = reinterpret_cast<uint32_t*>(h);
  off[0] = 0;
  for (size_t q = 0; q < nq; ++q) {
    const uint32_t b = batch_query(q);
    off[q + 1] = off[q] + (query_off[b + 1] - query_off[b]);
  }
  auto* lists = reinterpret_cast<uint4*>(h + lists_pos(n_segs));
  auto* tables = reinterpret_cast<uint4*>(h + clauses_pos());
  std::vector<uint32_t> cost(nc);
  for (size_t si = 0; si < n_segs; ++si) {
    const sdbg_segment* sg = segs[si];
    for (uint32_t i = clause_off[c0]; i < ns; ++i) {
      const uint2 l = excl_list(sg, slot_term[i]);
      lists[si * ns + i] = make_uint4(l.x, l.y, slot_rel[i], 0u);
    }
    for (uint32_t j = c0; j < nc; ++j) {
      uint32_t m = 0xFFFFFFFFu;
      for (uint32_t i = clause_off[j]; i < clause_off[j + 1]; ++i)
        m = std::min(m, slot_term[i] < sg->term_docs.size() ? sg->term_docs[slot_term[i]] : 0u);
      cost[j] = m;
    }
    uint4* T = tables + si * nc;
    for (size_t q = 0; q < nq; ++q) {
      const uint32_t b = batch_query(q);
      uint4* E = T + off[q];
      const uint32_t n = off[q + 1] - off[q];
      for (uint32_t i = 0; i < n; ++i) {
        const uint32_t j = query_off[b] + i;
        E[i] = make_uint4(clause_off[j], clause_off[j + 1] - clause_off[j], conj ? flags[j] & kAltNegated : flags[j], j);
      }
      std::stable_sort(E, E + n, [&](const uint4& x, const uint4& y) { return cost[x.w] < cost[y.w]; });
      if (conj) continue;
      std::array<uint32_t, kMaxQueryTerms> after{};   // per group: its positive entries after entry i
      for (uint32_t i = n; i-- > 0;) {
        if (E[i].z & kAltNegated) continue;
        const uint32_t g = (E[i].z >> 1) & 15u, m = ((E[i].z >> kAltMinShift) & 15u) + 1u;
        E[i].z |= (m > after[g] ? m - after[g] : 0u) << kAltNeedShift;
        ++after[g];
      }
    }
  }
  if (!consts.empty()) std::memcpy(h + consts_pos(n_segs), consts.data(), nc * sizeof(float4));
}

// The phrase pass of count_run (CountMode::phrase) over a plan with work items: bm25_count_kernel<kAnd, .., kPhrase> per
// segment, the count into out.counts; with a top-k (job.k) each item writes its k best keys to its own slot, then
// phrase_merge_kernel keeps each query's k best in out.bins (u64 keys [nq][k]) with their number in out.nulls (u32 [nq]).
// Host staging: the plan's, then [slot_off | slots | the job's tables (PhraseJob::bytes)].
int phrase_run(sdbg_segment* const* segs, size_t n_segs, const CountPlan& pl, const sdbg_col_pred* filt, const PhraseJob& job,
               const CountOut& out) {
  sdbg_ctx* c = segs[0]->ctx;
  const size_t nq = pl.Q.nq, total = pl.items;
  const uint32_t k = job.k;
  uint32_t cap = 0;
  if (k) { uint32_t kp = 1; while (kp < k) kp <<= 1; cap = std::max(256u, 2u * kp); }
  const size_t slot_off_pos = pl.staged;
  const size_t slots_pos = slot_off_pos + pl.off_bytes;
  const size_t tables_pos = (slots_pos + total * 4 + 15) & ~size_t(15);
  const size_t bytes = tables_pos + job.bytes(n_segs);
  std::vector<char> staging(bytes);
  char* h = staging.data();
  pl.write(h);
  item_slots(pl, h, slot_off_pos, slots_pos);
  job.write(segs, n_segs, h + tables_pos, pl.Q.kind == SDBG_QUERY_AND);
  // device scratch: [item keys [items][k] | item key counts | thresholds [nq]]
  const size_t keys_n_pos = total * size_t(k) * 8;
  const size_t thr_pos = (keys_n_pos + total * 4 + 15) & ~size_t(15);
  DevBuf& b_desc = c->scratch[0]; DevBuf& b_out = c->scratch[1];
  if (int rc = ensure(c, b_desc, bytes)) return rc;
  if (int rc = k ? ensure(c, b_out, thr_pos + nq * 8) : SDBG_OK) return rc;
  char* d = static_cast<char*>(b_desc.p);
  char* o = static_cast<char*>(b_out.p);
  auto* thr = reinterpret_cast<unsigned long long*>(o + thr_pos);
  CU(c, cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, c->stream));
  if (k) {
    fill_u64_kernel<<<64, 256, 0, c->stream>>>(thr, nq, job.seed);
    ++c->launches;
  }
  const auto [kernel, smem] = pl.kernel(CountMode::phrase, size_t(cap) * 16);
  CU(c, fit_dynamic_smem(kernel, smem));
  std::vector<ChainDev> chains(n_segs);
  if (int rc = filter_chains(segs, n_segs, filt, chains.data())) return rc;
  size_t first = 0;
  uint64_t base = 0;   // ordinals of the earlier segments (at most 2^32 - 2 docs per call)
  for (size_t si = 0; si < n_segs; ++si) {
    const size_t n = pl.seg_work[si].size();
    CountParams P;
    pl.params(d, segs[si], si, first, chains[si], &P);
    P.counts = static_cast<unsigned long long*>(out.counts);
    PhraseSink& F = P.phrase;
    job.sink(segs, n_segs, si, d + tables_pos, F);
    F.ordinal_base = uint32_t(base);
    F.k = k; F.cap = cap; F.thr = thr;
    F.out = reinterpret_cast<unsigned long long*>(o);
    F.out_n = reinterpret_cast<uint32_t*>(o + keys_n_pos);
    base += segs[si]->n_docs;
    first += n;
    if (!n) continue;
    kernel<<<unsigned(n), kCountThreads, smem, c->stream>>>(P);
    ++c->launches;
  }
  CU(c, cudaGetLastError());
  if (!k) return SDBG_OK;
  CU(c, fit_dynamic_smem(phrase_merge_kernel, size_t(cap) * 16));
  phrase_merge_kernel<<<unsigned(nq), 256, size_t(cap) * 16, c->stream>>>(
      reinterpret_cast<const unsigned long long*>(o), reinterpret_cast<const uint32_t*>(o + keys_n_pos),
      reinterpret_cast<const uint32_t*>(d + slot_off_pos), reinterpret_cast<const uint32_t*>(d + slots_pos), k, cap,
      static_cast<unsigned long long*>(out.bins), static_cast<uint32_t*>(out.nulls));
  ++c->launches;
  CU(c, cudaGetLastError());
  return SDBG_OK;
}

// Queues a pass over its plan into out. A count pass first sets out.counts to the single-term shortcut's counts. The
// sorted scan launches per segment its seed items first (all segments), then the rest, each item writing its k best to
// its own slot (its index in the work array); then sort_merge_kernel per query, and for a rank sort_dist_rows_kernel.
// The match scan launches its items twice (bm25_emit.cuh): pass A, emit_bases_kernel over each query's items in
// (segment, first window) order, pass B. A job with phrase clauses (job.phrase.query_off; the plan's batch is the AND of
// the positive clauses' terms) runs the phrase instantiations of its mode and stages the phrase tables.
// The plan is staged from pageable memory, which the copy has consumed when it returns, so calls can follow one another
// without a wait (a host group entry queues its shapes back to back).
int count_run(sdbg_segment* const* segs, size_t n_segs, const CountPlan& pl, const sdbg_col_pred* filt, const CountJob& job,
              const CountOut& out) {
  sdbg_ctx* c = segs[0]->ctx;
  const size_t nq = pl.Q.nq, total = pl.items;
  const bool sort = job.mode == CountMode::sort, emit = job.mode == CountMode::emit, phrase = job.mode == CountMode::phrase;
  if (std::any_of(pl.host.begin(), pl.host.end(), [](uint64_t v) { return v != 0; }))   // else out.counts is zero already
    CU(c, cudaMemcpyAsync(out.counts, pl.host.data(), nq * 8, cudaMemcpyHostToDevice, c->stream));
  if (!total && !sort) return SDBG_OK;
  if (phrase) return phrase_run(segs, n_segs, pl, filt, job.phrase, out);
  const SortJob& J = job.sort;
  const uint32_t k = J.k, cap = sort ? J.sink[0].cap : 0u;
  const bool phrased = job.phrase.query_off != nullptr;
  // host staging: the plan's, then for the sorted scan [slot_off | slots | segments], for the match scan [slot_off |
  // slots | offsets]; then for a phrase its tables (PhraseJob::bytes)
  const size_t slot_off_pos = pl.staged;
  const size_t slots_pos = slot_off_pos + pl.off_bytes;
  const size_t segs_pos = (slots_pos + total * 4 + 15) & ~size_t(15);
  const size_t mode_end = sort ? segs_pos + n_segs * sizeof(SortSegDev) : emit ? segs_pos + nq * 8 : pl.staged;
  const size_t tables_pos = (mode_end + 15) & ~size_t(15);
  const size_t bytes = phrased ? tables_pos + job.phrase.bytes(n_segs) : mode_end;
  std::vector<char> staging(bytes);
  char* h = staging.data();
  pl.write(h);
  if (sort || emit) item_slots(pl, h, slot_off_pos, slots_pos);
  if (emit) std::memcpy(h + segs_pos, job.emit.offset, nq * 8);
  if (phrased) job.phrase.write(segs, n_segs, h + tables_pos, pl.Q.kind == SDBG_QUERY_AND);
  if (sort) {
    auto* h_segs = reinterpret_cast<SortSegDev*>(h + segs_pos);
    for (size_t si = 0; si < n_segs; ++si) {
      const SortSink& S = J.sink[si];
      h_segs[si] = SortSegDev{S.values, S.validity, S.rows, S.ordinal_base, 0u};
    }
  }
  // the sorted scan's device scratch: [item keys | item key counts | thresholds | a rank's hits | its n_out]
  const size_t keys_n_pos = std::max<size_t>(total, 1) * k * sizeof(ulonglong2);
  const size_t thr_pos = (keys_n_pos + std::max<size_t>(total, 1) * 4 + 15) & ~size_t(15);
  const size_t hits_pos = (thr_pos + nq * 8 + 15) & ~size_t(15);
  const size_t n_out_pos = hits_pos + nq * k * sizeof(SortHitDev);
  DevBuf& b_desc = c->scratch[0]; DevBuf& b_out = c->scratch[1];
  if (int rc = ensure(c, b_desc, bytes)) return rc;
  if (int rc = sort ? ensure(c, b_out, out.rank < 0 ? hits_pos : n_out_pos + nq * 4) : SDBG_OK) return rc;
  // the match scan's device scratch: [item bases u64 | item counts u32]
  if (int rc = emit ? ensure(c, b_out, total * 12) : SDBG_OK) return rc;
  char* d = static_cast<char*>(b_desc.p);
  char* o = static_cast<char*>(b_out.p);
  auto* thr = reinterpret_cast<unsigned long long*>(o + thr_pos);
  CU(c, cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, c->stream));
  if (sort) CU(c, cudaMemsetAsync(thr, 0, nq * 8, c->stream));
  // the sorted keys, facet bins or aggregate cells, then for groups that need m >= 2 of their lists a bit-sliced counter
  // of bits(m) planes for the batch's largest m (at most 128 + 32 KB)
  const size_t mode_bytes = sort ? size_t(cap) * 16
                            : job.mode == CountMode::facet ? (size_t(job.facet.span) * 4 + 15) & ~size_t(15)
                            : job.mode == CountMode::agg   ? agg_cells_bytes(job.agg.key.span)
                                                           : 0;
  const auto [kernel, smem] = pl.kernel(job.mode, mode_bytes, phrased);
  CU(c, fit_dynamic_smem(kernel, smem));
  std::vector<ChainDev> chains(n_segs);
  if (int rc = filter_chains(segs, n_segs, filt, chains.data())) return rc;
  auto* e_base = reinterpret_cast<unsigned long long*>(o);
  auto* e_n = reinterpret_cast<uint32_t*>(o + total * 8);
  const auto* e_off = reinterpret_cast<const unsigned long long*>(d + segs_pos);
  for (int pass = 0; pass < (emit ? 2 : 1); ++pass) {   // the match scan: pass A, the bases, pass B
    if (pass) {
      emit_bases_kernel<<<unsigned(nq), 32, 0, c->stream>>>(e_n, reinterpret_cast<const uint32_t*>(d + slot_off_pos),
                                                            reinterpret_cast<const uint32_t*>(d + slots_pos), e_off, job.emit.limit,
                                                            e_base, static_cast<unsigned long long*>(out.counts),
                                                            static_cast<uint32_t*>(out.nulls));
      ++c->launches;
    }
    for (int phase = 0; phase < 2; ++phase) {   // seeds (sorted scan only), then the rest
      size_t begin = 0;
      for (size_t si = 0; si < n_segs; ++si) {
        const auto& w = pl.seg_work[si];
        const size_t n_seed = size_t(std::count_if(w.begin(), w.end(), [](const CountItem& x) { return x.seed; }));
        const size_t first = begin + (phase ? n_seed : 0), n = phase ? w.size() - n_seed : n_seed;
        begin += w.size();
        if (!n) continue;
        CountParams P;
        pl.params(d, segs[si], si, first, chains[si], &P);
        P.counts = static_cast<unsigned long long*>(out.counts);
        if (phrased) job.phrase.sink(segs, n_segs, si, d + tables_pos, P.phrase);
        if (sort) {
          P.counts = nullptr;
          P.sort = J.sink[si];
          P.sort.thr = c->wand ? thr : nullptr;
          P.sort.out = reinterpret_cast<ulonglong2*>(o);
          P.sort.out_n = reinterpret_cast<uint32_t*>(o + keys_n_pos);
          P.sort.stats = out.stats;
        }
        if (job.mode == CountMode::facet) {
          P.facet = job.facet.sink[si];
          P.facet.counts = static_cast<unsigned long long*>(out.bins);
          P.facet.nulls = static_cast<unsigned long long*>(out.nulls);
          P.facet.out_of_range = out.oor;
        }
        if (job.mode == CountMode::agg) {
          P.agg = job.agg.sink[si];
          P.agg.cells = static_cast<AggCell*>(out.bins);
          P.agg.nulls = static_cast<AggCell*>(out.nulls);
          P.agg.out_of_range = out.oor;
        }
        if (emit) {
          P.counts = nullptr;
          P.emit = EmitSink{e_n, pass ? e_base : nullptr, e_off, static_cast<EmitHit*>(out.bins), job.emit.limit, uint32_t(si)};
        }
        kernel<<<unsigned(n), kCountThreads, smem, c->stream>>>(P);
        ++c->launches;
      }
    }
  }
  CU(c, cudaGetLastError());
  if (!sort) return SDBG_OK;
  SortMergeParams M;
  M.keys = reinterpret_cast<const ulonglong2*>(o);
  M.keys_n = reinterpret_cast<const uint32_t*>(o + keys_n_pos);
  M.slot_off = reinterpret_cast<const uint32_t*>(d + slot_off_pos);
  M.slots = reinterpret_cast<const uint32_t*>(d + slots_pos);
  M.segs = reinterpret_cast<const SortSegDev*>(d + segs_pos);
  M.n_segs = uint32_t(n_segs); M.type = J.sink[0].type; M.nulls_first = J.sink[0].nulls_first; M.k = k; M.cap = cap;
  const bool rank = out.rank >= 0;   // a rank's hits stay in the scratch and become its rows below
  M.out = rank ? reinterpret_cast<SortHitDev*>(o + hits_pos) : static_cast<SortHitDev*>(out.bins);
  M.n_out = rank ? reinterpret_cast<uint32_t*>(o + n_out_pos) : static_cast<uint32_t*>(out.counts);
  CU(c, fit_dynamic_smem(sort_merge_kernel, size_t(cap) * 16));
  sort_merge_kernel<<<unsigned(nq), 256, size_t(cap) * 16, c->stream>>>(M);
  ++c->launches;
  CU(c, cudaGetLastError());
  if (!rank) return SDBG_OK;
  sort_dist_rows_kernel<<<unsigned(nq), 256, 0, c->stream>>>(M.out, M.n_out, M.segs, k, M.type, J.sink[0].desc, M.nulls_first,
                                                             uint32_t(out.rank), static_cast<unsigned long long*>(out.counts),
                                                             static_cast<SortDistRow*>(out.bins));
  ++c->launches;
  CU(c, cudaGetLastError());
  return SDBG_OK;
}

// Runs a prepared pass over B into out: count_run for a whole batch, else shape by shape through shapes_run. Nothing waits.
int pass_run(sdbg_segment* const* segs, size_t n_segs, const PassBatch<uint32_t>& B, const sdbg_col_pred* filt, const CountJob& job,
             const CountOut& out) {
  if (B.whole.nq) return count_run(segs, n_segs, count_plan(segs, n_segs, B.whole, B.total_excl, filt, job), filt, job, out);
  const GroupSplit<uint32_t>& S = B.S;
  return shapes_run(segs[0]->ctx, S, job.rows(out.rank >= 0), {out.counts, out.bins, out.nulls}, [&](int sh, void* const* part) {
    const CountOut o{part[0], part[1], part[2], out.oor, out.stats, out.rank};
    if (!job.phrase.query_off)
      return count_run(segs, n_segs, count_plan(segs, n_segs, S.view(sh), S.total_excl[sh], filt, job), filt, job, o);
    CountJob js = job;   // the phrase tables of this shape's queries
    js.phrase = job.phrase.on(S.qs[sh]);
    return count_run(segs, n_segs, count_plan(segs, n_segs, S.view(sh), S.total_excl[sh], filt, js), filt, js, o);
  });
}

// The aggregate device form's buffer: this header, then AggCell [nq][span], then AggCell [nq] for the NULL key.
struct AggDistHeader {
  unsigned long long type;           // the value column's sdbg_type (UINT64_MAX: not found)
  unsigned long long span, nq;
  unsigned long long failed;         // non-zero: this rank's local pass failed
  unsigned long long out_of_range;   // non-zero: a matching doc's key lay outside the range
  unsigned long long pad[3];
};
static_assert(sizeof(AggDistHeader) == 64, "the cells stay 16-byte aligned");

size_t agg_dist_bytes(size_t nq, uint32_t span) { return sizeof(AggDistHeader) + nq * (size_t(span) + 1) * sizeof(AggCell); }
size_t sort_dist_bytes(size_t nq, uint32_t k) { return sizeof(SortDistHeader) + nq * 8 + nq * size_t(k) * sizeof(SortDistRow); }

// Where count_run's arrays lie in one device buffer, the region of a call: byte offsets (kNone: not in the region) and
// its size. One layout per pass, the same for the host entries and a rank's buffer.
constexpr size_t kNone = SIZE_MAX;
struct PassRegion {
  size_t counts, bins, nulls, oor, stats, bytes;

  CountOut at(void* base, int64_t rank = -1) const {
    const auto in = [&](size_t o) -> void* { return o == kNone ? nullptr : static_cast<char*>(base) + o; };
    return {in(counts), in(bins), in(nulls), static_cast<unsigned int*>(in(oor)), static_cast<unsigned long long*>(in(stats)), rank};
  }
};

// The count and facet passes: u64 words [counts [nq] | facet: counts [nq][span], NULL counts [nq] | out-of-range |
// failed], which one all-reduce of int64 merges across ranks (dist_reduce_to_host: the failure word last).
PassRegion words_region(size_t nq, uint32_t span /* 0: the count pass */) {
  const size_t w = nq + (span ? nq * (size_t(span) + 1) : 0);
  return {0, span ? nq * 8 : kNone, span ? (w - nq) * 8 : kNone, w * 8, kNone, (w + 2) * 8};
}

// The aggregate pass: its device form's buffer (AggDistHeader, cells, NULL cells); the counts are scratch.
PassRegion agg_region(size_t nq, uint32_t span) {
  return {kNone, sizeof(AggDistHeader), sizeof(AggDistHeader) + nq * span * sizeof(AggCell), offsetof(AggDistHeader, out_of_range),
          kNone, agg_dist_bytes(nq, span)};
}

// The sorted scan of the local entries: [n_out u32 [nq] | windows judged, skipped | hits SortHitDev [nq][k]].
PassRegion sort_region(size_t nq, uint32_t k) {
  const size_t stats = (nq * 4 + 15) & ~size_t(15);
  return {0, stats + 16, kNone, kNone, stats, stats + 16 + nq * k * sizeof(SortHitDev)};
}

// A rank's sorted scan: its device form's buffer (SortDistHeader, row counts, rows); the windows are scratch.
PassRegion sort_rank_region(size_t nq, uint32_t k) {
  return {sizeof(SortDistHeader), sizeof(SortDistHeader) + nq * 8, kNone, kNone, kNone, sort_dist_bytes(nq, k)};
}

// The host copy h of a call's region: fails on its out-of-range word, else fills the caller's arrays (fill(h)).
template <class Fill>
int pass_finish(sdbg_ctx* c, const PassRegion& L, const char* h, Fill fill) {
  unsigned int oor = 0;
  if (L.oor != kNone) std::memcpy(&oor, h + L.oor, 4);
  if (oor) return fail(c, SDBG_EINVAL, "a matching doc's key lies outside [key_min, key_min + key_span)");
  fill(h);
  return SDBG_OK;
}

void facet_fill(const char* h, size_t nq, uint32_t span, uint64_t* counts, uint64_t* null_counts) {
  const PassRegion L = words_region(nq, span);
  std::memcpy(counts, h + L.bins, nq * size_t(span) * 8);
  std::memcpy(null_counts, h + L.nulls, nq * 8);
}

// The host entries' one path, after their checks (B): prepares the job, then lays out its region L in c->pass[0], zeroes
// it, runs the pass into it, copies it back through the pinned staging with one copy and one wait, and finishes
// (pass_finish). The sorted scan's windows go to sdbg_scan_stats. A count batch that the plan answers entirely from
// docs_count queues nothing: fill gets the plan's counts, which is where the count region starts.
template <class Fill>
int pass_to_host(sdbg_segment* const* segs, size_t n_segs, const PassBatch<uint32_t>& B, const sdbg_col_pred* filt, CountJob& job,
                 const PassRegion& L, Fill fill) {
  if (B.rc) return B.rc;
  sdbg_ctx* c = segs[0]->ctx;
  CU(c, cudaSetDevice(c->device));
  if (int rc = job_prepare(c, segs, n_segs, job)) return rc;
  CountPlan pl;
  if (B.whole.nq) {
    pl = count_plan(segs, n_segs, B.whole, B.total_excl, filt, job);
    if (job.mode == CountMode::count && !pl.items) {
      fill(reinterpret_cast<const char*>(pl.host.data()));
      return SDBG_OK;
    }
  }
  if (int rc = ensure(c, c->pass[0], L.bytes + B.nq * 8)) return rc;   // then the aggregate pass's count scratch
  if (int rc = ensure_pinned(c, L.bytes)) return rc;
  CountOut out = L.at(c->pass[0].p);
  if (!out.counts) out.counts = static_cast<char*>(c->pass[0].p) + L.bytes;
  CU(c, cudaMemsetAsync(c->pass[0].p, 0, L.bytes + B.nq * 8, c->stream));
  if (int rc = B.whole.nq ? count_run(segs, n_segs, pl, filt, job, out) : pass_run(segs, n_segs, B, filt, job, out)) return rc;
  if (out.stats) {   // windows skipped: a device word, as the GROUP BY scan leaves it
    if (!c->d_zone_skipped) CU(c, cudaMalloc(reinterpret_cast<void**>(&c->d_zone_skipped), 8));
    CU(c, cudaMemcpyAsync(c->d_zone_skipped, out.stats + 1, 8, cudaMemcpyDeviceToDevice, c->stream));
  }
  CU(c, cudaMemcpyAsync(c->h_pinned, c->pass[0].p, L.bytes, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  const char* h = static_cast<const char*>(c->h_pinned);
  if (out.stats) std::memcpy(&c->zone_blocks_total, h + L.stats, 8);   // windows judged (only where a zonemap is)
  return pass_finish(c, L, h, fill);
}

// phrase: the job's phrase slots (PhraseBatch::job) when B is the AND of phrases' terms.
int sort_to_host(sdbg_segment* const* segs, size_t n_segs, const PassBatch<uint32_t>& B, const sdbg_col_pred* filt, uint64_t field,
                 int descending, int nulls_first, uint32_t k, sdbg_sort_hit* out, uint32_t* n_out, const PhraseJob& phrase = {}) {
  CountJob job{CountMode::sort, {field, descending, nulls_first, k, {}, {}}, {}, {}};
  job.phrase = phrase;
  const PassRegion L = sort_region(B.nq, k);
  return pass_to_host(segs, n_segs, B, filt, job, L, [&](const char* h) {
    std::memcpy(n_out, h + L.counts, B.nq * 4);
    std::memcpy(out, h + L.bins, B.nq * k * sizeof(SortHitDev));
  });
}

int agg_to_host(sdbg_segment* const* segs, size_t n_segs, const PassBatch<uint32_t>& B, const sdbg_col_pred* filt, uint64_t key_field,
                int64_t key_min, uint32_t key_span, uint64_t value_field, sdbg_match_agg* out, sdbg_match_agg* null_out,
                const PhraseJob& phrase = {}) {
  CountJob job{CountMode::agg, {}, {}, {{key_field, key_min, key_span, {}}, value_field, {}}};
  job.phrase = phrase;
  const PassRegion L = agg_region(B.nq, key_span);
  return pass_to_host(segs, n_segs, B, filt, job, L, [&](const char* h) {
    agg_results(reinterpret_cast<const AggCell*>(h + L.bins), B.nq, key_span, job.agg.sink[0].type, out, null_out);
  });
}
}  // namespace

extern "C" int sdbg_match_count_batch(sdbg_segment* const* segs, size_t n_segs, int kind, const uint32_t* terms,
                                      const uint32_t* term_off, size_t nq, const uint32_t* excl_terms,
                                      const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t* counts) {
  if (!counts) return SDBG_EINVAL;
  const PassBatch<uint32_t> B(segs, n_segs, QueryBatch<uint32_t>{kind, terms, term_off, nq, excl_terms, excl_off, nullptr}, filt);
  CountJob job{CountMode::count, {}, {}, {}};
  return pass_to_host(segs, n_segs, B, filt, job, words_region(nq, 0), [&](const char* h) { std::memcpy(counts, h, nq * 8); });
}

namespace {
// The phrase entries' queries as their callers pass them. Query q is an AND of the groups [query_group_off[q] ..
// query_group_off[q + 1]) (null: group q), group g an OR of the alternatives [group_off[g] .. group_off[g + 1]) (null:
// alternative g), negated when group_neg[g] (null: none), alternative j the phrase of slots terms / rel_pos [clause_off[j]
// .. clause_off[j + 1]) (rel_pos null: adjacent); excl_terms / excl_off as the flat entries take them. Positive group g
// needs group_min[g] of its alternatives (null: 1).
struct PhraseQueries {
  const uint32_t* terms;
  const uint32_t* rel_pos;
  const uint32_t* clause_off;
  const uint32_t* group_off;
  const uint8_t* group_neg;
  const uint32_t* query_group_off;
  size_t nq;
  const uint32_t* excl_terms;
  const uint32_t* excl_off;
  const uint32_t* group_min = nullptr;
};

// A batch of phrase queries (PhraseQueries), checked before anything is queued, with its candidate batch S: per query
// a superset of its matches that the existing candidate scans find, which the alternative check then narrows exactly.
// The groups are normalised first, as split_groups does for terms: a positive group that needs all its s alternatives is
// s groups of one (qoff / goff / gneg / gmin hold the normalised groups, alternatives in the caller's order).
//   every positive group has one alternative: the AND of the distinct terms of the positive groups (shape 1);
//   else, exactly one group kept, needing one of its lists: the flat OR of its proxies (shape 0); otherwise OR groups of
//   proxies (shape 2).
// A positive group of one alternative contributes each of its distinct terms as a one-list group. A group of several
// alternatives contributes, per one-slot alternative, its term, and per phrase alternative one of its terms, the cheapest
// by docs_count summed over the call's segments among those the query has not used yet (none when the group holds one of
// its terms already, which then stands for it). With c_l alternatives standing on list l, the group needs the least
// number m' of its lists whose c_l, largest first, sum to its minimum m: a doc in which m alternatives occur is in all
// their lists, and fewer than m' lists cannot carry m alternatives. A term stays in one group of a query, so a group that
// cannot avoid a repeat is left out and only checked per doc. The one-alternative groups are always kept, and so is the
// first group of several when there are none, so the candidate batch always holds a group. A group is guaranteed
// (kAltGuaranteed) when it is kept, all its alternatives are one slot and, for m >= 2, no two of them share a term
// (m' == m).
// Per alternative j: flags[j] (PhraseJob); per query: its alternatives [aoff[q] .. aoff[q + 1]).
struct PhraseBatch {
  int rc = SDBG_OK;
  size_t nq;
  std::vector<uint32_t> rel, qoff, goff, aoff, flags, gmin;
  std::vector<uint8_t> gneg;
  const uint32_t* terms;
  const uint32_t* clause_off;
  GroupSplit<uint32_t> S;

  PhraseBatch(sdbg_segment* const* segs, size_t n_segs, const PhraseQueries& A)
      : nq(A.nq), terms(A.terms), clause_off(A.clause_off) {
    if (!segs || !n_segs || !segs[0] || !nq || !clause_off) { rc = SDBG_EINVAL; return; }
    sdbg_ctx* c = segs[0]->ctx;
    qoff.resize(nq + 1);
    for (size_t q = 0; q <= nq; ++q) qoff[q] = A.query_group_off ? A.query_group_off[q] : uint32_t(q);
    for (size_t q = 0; q < nq && !rc; ++q) {
      if (qoff[q + 1] < qoff[q]) rc = fail(c, SDBG_EINVAL, "query offsets must be non-decreasing");
      else if (qoff[q + 1] == qoff[q]) rc = fail(c, SDBG_EINVAL, "a query without a clause");
      else if (qoff[q + 1] - qoff[q] > kMaxQueryTerms) rc = fail(c, SDBG_EUNSUPPORTED, "a query holds 1..16 groups");
    }
    if (rc) return;
    goff.assign(size_t(qoff[nq]) + 1, 0u);
    for (uint32_t g = qoff[0]; g <= qoff[nq]; ++g) goff[g] = A.group_off ? A.group_off[g] : g;
    for (uint32_t g = qoff[0]; g < qoff[nq] && !rc; ++g) {
      const uint32_t m = A.group_min ? A.group_min[g] : 1u;
      if (goff[g + 1] < goff[g]) rc = fail(c, SDBG_EINVAL, "group_off must be non-decreasing");
      else if (goff[g + 1] == goff[g]) rc = fail(c, SDBG_EINVAL, "empty OR group");
      else if (m == 0u || m > goff[g + 1] - goff[g])
        rc = fail(c, SDBG_EINVAL, "a group's minimum match count must be 1..its number of alternatives");
      else if (m != 1u && A.group_neg && A.group_neg[g])
        rc = fail(c, SDBG_EUNSUPPORTED, "a negated group with a minimum match count other than 1");
    }
    if (rc) return;
    normalise(A);
    for (uint32_t j = goff[qoff[0]]; j < goff[qoff[nq]] && !rc; ++j) {
      if (clause_off[j + 1] < clause_off[j]) rc = fail(c, SDBG_EINVAL, "clause_off must be non-decreasing");
      else if (clause_off[j + 1] == clause_off[j]) rc = fail(c, SDBG_EINVAL, "empty clause");
    }
    for (size_t q = 0; q < nq && !rc; ++q) {
      bool pos = false;
      for (uint32_t g = qoff[q]; g < qoff[q + 1]; ++g) pos |= !gneg[g];
      if (!pos) rc = fail(c, SDBG_EINVAL, "a query without a positive clause");
    }
    for (size_t q = 0; q < nq && !rc; ++q)
      if (clause_off[goff[qoff[q + 1]]] - clause_off[goff[qoff[q]]] > kMaxPhraseSlots) rc = fail(c, SDBG_EUNSUPPORTED, "a query holds 1..16 slots");
    if (!rc && !terms) rc = fail(c, SDBG_EINVAL, "terms is NULL");
    if (rc) return;
    aoff.resize(nq + 1);
    flags.assign(goff[qoff[nq]], 0u);
    rel.resize(clause_off[goff[qoff[nq]]]);
    for (size_t q = 0; q <= nq; ++q) aoff[q] = goff[qoff[q]];
    for (size_t q = 0; q < nq; ++q) {
      for (uint32_t g = qoff[q]; g < qoff[q + 1]; ++g) {
        const bool neg = gneg[g];
        for (uint32_t j = goff[g]; j < goff[g + 1]; ++j) {
          flags[j] = (neg ? kAltNegated : 0u) | ((g - qoff[q]) << 1) | ((gmin[g] - 1u) << kAltMinShift);
          const uint32_t s0 = clause_off[j], s1 = clause_off[j + 1];
          for (uint32_t i = s0; i < s1; ++i) {
            rel[i] = A.rel_pos ? A.rel_pos[i] : i - s0;
            if (i == s0 ? rel[i] != 0u : rel[i] <= rel[i - 1]) {
              rc = fail(c, SDBG_EINVAL, "rel_pos must start at 0 and increase");
              return;
            }
            if (!neg)
              for (size_t si = 0; si < n_segs; ++si)
                if (size_t(terms[i]) + 1 >= segs[si]->term_blk_begin.size()) {
                  rc = fail(c, SDBG_EINVAL, "term id out of range");
                  return;
                }
          }
        }
      }
    }
    if (A.excl_off)
      for (size_t q = 0; q < nq && !rc; ++q) {
        if (A.excl_off[q + 1] < A.excl_off[q]) rc = fail(c, SDBG_EINVAL, "excl_off must be non-decreasing");
        else if (A.excl_off[q + 1] - A.excl_off[q] > kMaxQueryTerms) rc = fail(c, SDBG_EUNSUPPORTED, "a query excludes at most 16 terms");
        else if (A.excl_off[q + 1] > A.excl_off[q] && !A.excl_terms) rc = fail(c, SDBG_EINVAL, "excl_terms is NULL");
      }
    if (!rc) candidates(segs, n_segs, A);
  }

  uint32_t slots(uint32_t j) const { return clause_off[j + 1] - clause_off[j]; }

  // Replaces the caller's groups (checked) with the normalised ones: a positive group of s >= 2 alternatives with
  // minimum s becomes s groups of one.
  void normalise(const PhraseQueries& A) {
    std::vector<uint32_t> q2{0u}, g2;
    gneg.clear();
    gmin.clear();
    for (size_t q = 0; q < nq; ++q) {
      for (uint32_t g = qoff[q]; g < qoff[q + 1]; ++g) {
        const uint32_t s = goff[g + 1] - goff[g], m = A.group_min ? A.group_min[g] : 1u;
        const bool neg = A.group_neg && A.group_neg[g];
        const bool split = !neg && m == s;
        for (uint32_t j = goff[g]; j < goff[g + 1]; j += split ? 1u : s) {
          g2.push_back(j);
          gneg.push_back(neg);
          gmin.push_back(split ? 1u : m);
        }
      }
      q2.push_back(uint32_t(g2.size()));
    }
    g2.push_back(goff[qoff[nq]]);
    qoff = std::move(q2);
    goff = std::move(g2);
  }

  void candidates(sdbg_segment* const* segs, size_t n_segs, const PhraseQueries& A) {
    const auto docs = [&](uint32_t t) {
      uint64_t n = 0;
      for (size_t si = 0; si < n_segs; ++si) n += segs[si]->term_docs[t];
      return n;
    };
    for (int sh = 0; sh < 3; ++sh) { S.term_off[sh].assign(1, 0u); S.excl_off[sh].assign(1, 0u); }
    std::vector<std::vector<uint32_t>> groups;
    std::vector<uint32_t> used;
    const auto in = [](const std::vector<uint32_t>& v, uint32_t t) { return std::find(v.begin(), v.end(), t) != v.end(); };
    std::vector<uint32_t> need;   // per kept group: its minimum number of lists m'
    for (size_t q = 0; q < nq; ++q) {
      groups.clear();
      used.clear();
      need.clear();
      bool single = true;
      for (uint32_t g = qoff[q]; g < qoff[q + 1]; ++g)
        if (!gneg[g]) single &= goff[g + 1] - goff[g] == 1u;
      for (uint32_t g = qoff[q]; g < qoff[q + 1]; ++g) {
        if (gneg[g] || goff[g + 1] - goff[g] != 1u) continue;
        const uint32_t j = goff[g];
        for (uint32_t i = clause_off[j]; i < clause_off[j + 1]; ++i)
          if (!in(used, terms[i])) { used.push_back(terms[i]); groups.push_back({terms[i]}); need.push_back(1u); }
        if (slots(j) == 1u) flags[j] |= kAltGuaranteed;
      }
      for (uint32_t g = qoff[q]; g < qoff[q + 1]; ++g) {
        if (gneg[g] || goff[g + 1] - goff[g] == 1u) continue;
        std::vector<uint32_t> G, cnt;   // the group's lists and the alternatives standing on each
        bool ok = true, terms_only = true;
        const auto stand = [&](uint32_t t) {
          const size_t l = std::find(G.begin(), G.end(), t) - G.begin();
          if (l == G.size()) { G.push_back(t); cnt.push_back(0u); }
          ++cnt[l];
        };
        for (uint32_t j = goff[g]; j < goff[g + 1] && ok; ++j) {
          if (slots(j) != 1u) { terms_only = false; continue; }
          const uint32_t t = terms[clause_off[j]];
          ok = in(G, t) || !in(used, t);
          stand(t);
        }
        for (uint32_t j = goff[g]; j < goff[g + 1] && ok; ++j) {
          if (slots(j) == 1u) continue;
          uint32_t best = 0, cover = 0;
          bool covered = false;
          uint64_t best_docs = UINT64_MAX;
          for (uint32_t i = clause_off[j]; i < clause_off[j + 1]; ++i) {
            if (!covered && in(G, terms[i])) { covered = true; cover = terms[i]; }
            if (in(used, terms[i])) continue;
            const uint64_t n = docs(terms[i]);
            if (n < best_docs) { best_docs = n; best = terms[i]; }
          }
          ok = covered || best_docs != UINT64_MAX;
          if (ok) stand(covered ? cover : best);
        }
        if (!ok) continue;
        std::sort(cnt.begin(), cnt.end(), std::greater<uint32_t>());
        uint32_t m2 = 0;
        for (uint32_t sum = 0; sum < gmin[g]; sum += cnt[m2++]) {}
        used.insert(used.end(), G.begin(), G.end());
        groups.push_back(std::move(G));
        need.push_back(m2);
        if (terms_only && (gmin[g] == 1u || m2 == gmin[g]))
          for (uint32_t j = goff[g]; j < goff[g + 1]; ++j) flags[j] |= kAltGuaranteed;
      }
      const int sh = single ? 1 : groups.size() == 1 && need[0] == 1u ? 0 : 2;
      S.qs[sh].push_back(uint32_t(q));
      for (size_t gi = 0; gi < groups.size(); ++gi)
        for (uint32_t t : groups[gi]) {
          S.terms[sh].push_back(t);
          if (sh == 2) S.term_grp[sh].push_back(uint8_t(gi | ((need[gi] - 1u) << 4)));
        }
      S.term_off[sh].push_back(uint32_t(S.terms[sh].size()));
      if (A.excl_off)
        for (uint32_t i = A.excl_off[q]; i < A.excl_off[q + 1]; ++i) S.excl_terms[sh].push_back(A.excl_terms[i]);
      S.excl_off[sh].push_back(uint32_t(S.excl_terms[sh].size()));
    }
  }

  // The alternatives of a count_run job over the candidate batch: count only until k or consts are set.
  PhraseJob job() const {
    PhraseJob J;
    J.slot_term = terms; J.slot_rel = rel.data(); J.clause_off = clause_off; J.flags = flags.data();
    J.query_off = aoff.data(); J.nq = nq; J.n_alts = aoff[nq];
    return J;
  }

  // consts[j] = {c0, norm_const, norm_length, 0} of positive alternative j's statistics clause_stats[j] (negated ones: 0):
  // the scorer form of fill_qterm, as the phrase top-k and the scored phrase scan score a match.
  std::vector<float4> consts(sdbg_segment* const* segs, const sdbg_bm25_term* clause_stats, float k1, float b) const {
    std::vector<float4> out(aoff[nq], make_float4(0.f, 0.f, 0.f, 0.f));
    for (uint32_t j = aoff[0]; j < aoff[nq]; ++j) {
      if (flags[j] & kAltNegated) continue;
      sdbg_bm25_term t = clause_stats[j];
      t.term = terms[clause_off[j]];
      QTermDev d;
      fill_qterm(segs[0], t, k1, b, d);
      out[j] = make_float4(d.c0, d.norm_const, d.norm_length, 0.f);
    }
    return out;
  }
};

// Every segment holds positions (sdbg_stage_positions).
int phrase_positions_staged(sdbg_segment* const* segs, size_t n_segs) {
  for (size_t si = 0; si < n_segs; ++si)
    if (!segs[si]->d_pos) return fail(segs[0]->ctx, SDBG_ENOTFOUND, "segment has no staged positions");
  return SDBG_OK;
}

// The count, top-k, sorted scan, facet counts and aggregates of a batch of phrase queries (PhraseQueries): PhraseBatch's
// checks, its candidate batch, staged positions, then the flat entry's pass with the alternatives on its job.
int phrase_count(sdbg_segment* const* segs, size_t n_segs, const PhraseQueries& A, const sdbg_col_pred* filt, uint64_t* counts) {
  if (!counts) return SDBG_EINVAL;
  PhraseBatch PB(segs, n_segs, A);
  if (PB.rc) return PB.rc;
  const PassBatch<uint32_t> B(segs, n_segs, std::move(PB.S), A.nq, filt);
  if (B.rc) return B.rc;
  if (int rc = phrase_positions_staged(segs, n_segs)) return rc;
  CountJob job{CountMode::count, {}, {}, {}};
  job.mode = CountMode::phrase;
  job.phrase = PB.job();
  return pass_to_host(segs, n_segs, B, filt, job, words_region(A.nq, 0), [&](const char* h) { std::memcpy(counts, h, A.nq * 8); });
}

int phrase_topk(sdbg_segment* const* segs, size_t n_segs, const PhraseQueries& A, const sdbg_bm25_term* clause_stats, float k1,
                float b, const sdbg_col_pred* filt, uint32_t k, float threshold_in, sdbg_hit* out, uint32_t* n_out,
                uint64_t* total_matches) {
  if (!out || !n_out || !clause_stats) return SDBG_EINVAL;
  const size_t nq = A.nq;
  if (int rc = topk_args(segs, n_segs, nq, k)) return rc;
  sdbg_ctx* c = segs[0]->ctx;
  if (k > kSortMaxK) return fail(c, SDBG_EUNSUPPORTED, "k > 4096");
  PhraseBatch PB(segs, n_segs, A);
  if (PB.rc) return PB.rc;
  const PassBatch<uint32_t> B(segs, n_segs, std::move(PB.S), nq, filt);
  if (B.rc) return B.rc;
  uint64_t ord = 0;
  for (size_t si = 0; si < n_segs; ++si) ord += segs[si]->n_docs;
  if (ord > kMaxDocId) return fail(c, SDBG_EUNSUPPORTED, "more than 2^32-2 docs per call");
  if (int rc = phrase_positions_staged(segs, n_segs)) return rc;
  CountJob job{CountMode::count, {}, {}, {}};
  job.mode = CountMode::phrase;
  PhraseJob& J = job.phrase;
  J = PB.job();
  J.k = k;
  J.consts = PB.consts(segs, clause_stats, k1, b);
  uint32_t thr_bits; std::memcpy(&thr_bits, &threshold_in, 4);
  if (!(threshold_in >= 0.f)) thr_bits = 0;  // negative / NaN seeds accept every positive score, as the top-k entries
  J.seed = (static_cast<unsigned long long>(thr_bits) << 32) | 0xFFFFFFFFull;
  if (int rc = job_prepare(c, segs, n_segs, job)) return rc;
  if (int rc = ensure(c, c->pass[0], nq * (size_t(k) * 8 + 12))) return rc;
  const TopkDevOut dev = topk_region(c->pass[0].p, nq, k);
  CU(c, cudaMemsetAsync(c->pass[0].p, 0, nq * (size_t(k) * 8 + 12), c->stream));
  const CountOut o{dev.total, dev.keys, dev.n_out, nullptr, nullptr, -1};
  if (int rc = pass_run(segs, n_segs, B, filt, job, o)) return rc;
  return topk_hits_to_host(segs, n_segs, dev, nq, k, out, n_out, total_matches);
}

int phrase_topk_by_column(sdbg_segment* const* segs, size_t n_segs, const PhraseQueries& A, const sdbg_col_pred* filt,
                          uint64_t sort_field, int descending, int nulls_first, uint32_t k, sdbg_sort_hit* out, uint32_t* n_out) {
  if (!segs || !n_segs || !segs[0] || !k || !out || !n_out) return SDBG_EINVAL;
  if (k > kSortMaxK) return fail(segs[0]->ctx, SDBG_EUNSUPPORTED, "k > 4096");
  PhraseBatch PB(segs, n_segs, A);
  if (PB.rc) return PB.rc;
  const PassBatch<uint32_t> B(segs, n_segs, std::move(PB.S), A.nq, filt);
  if (B.rc) return B.rc;
  if (int rc = phrase_positions_staged(segs, n_segs)) return rc;
  return sort_to_host(segs, n_segs, B, filt, sort_field, descending, nulls_first, k, out, n_out, PB.job());
}

int phrase_facet_counts(sdbg_segment* const* segs, size_t n_segs, const PhraseQueries& A, const sdbg_col_pred* filt, uint64_t key_field,
                        int64_t key_min, uint32_t key_span, uint64_t* counts, uint64_t* null_counts) {
  if (!counts || !null_counts) return SDBG_EINVAL;
  PhraseBatch PB(segs, n_segs, A);
  if (PB.rc) return PB.rc;
  const PassBatch<uint32_t> B(segs, n_segs, std::move(PB.S), A.nq, filt);
  if (B.rc) return B.rc;
  if (int rc = phrase_positions_staged(segs, n_segs)) return rc;
  CountJob job{CountMode::facet, {}, {key_field, key_min, key_span, {}}, {}};
  job.phrase = PB.job();
  return pass_to_host(segs, n_segs, B, filt, job, words_region(A.nq, key_span),
                      [&](const char* h) { facet_fill(h, A.nq, key_span, counts, null_counts); });
}

int phrase_aggregate(sdbg_segment* const* segs, size_t n_segs, const PhraseQueries& A, const sdbg_col_pred* filt, uint64_t key_field,
                     int64_t key_min, uint32_t key_span, uint64_t value_field, sdbg_match_agg* out, sdbg_match_agg* null_out) {
  if (!out || !null_out) return SDBG_EINVAL;
  PhraseBatch PB(segs, n_segs, A);
  if (PB.rc) return PB.rc;
  const PassBatch<uint32_t> B(segs, n_segs, std::move(PB.S), A.nq, filt);
  if (B.rc) return B.rc;
  if (int rc = phrase_positions_staged(segs, n_segs)) return rc;
  return agg_to_host(segs, n_segs, B, filt, key_field, key_min, key_span, value_field, out, null_out, PB.job());
}
}  // namespace

namespace {
// The queries of the sdbg_phrase_* entries: each one positive group of one alternative.
PhraseQueries phrase_one(const uint32_t* terms, const uint32_t* rel_pos, const uint32_t* phrase_off, size_t nq,
                         const uint32_t* excl_terms, const uint32_t* excl_off) {
  return {terms, rel_pos, phrase_off, nullptr, nullptr, nullptr, nq, excl_terms, excl_off};
}
}  // namespace

extern "C" int sdbg_phrase_count_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms, const uint32_t* rel_pos,
                                       const uint32_t* phrase_off, size_t nq, const uint32_t* excl_terms, const uint32_t* excl_off,
                                       const sdbg_col_pred* filt, uint64_t* counts) {
  return phrase_count(segs, n_segs, phrase_one(terms, rel_pos, phrase_off, nq, excl_terms, excl_off), filt, counts);
}

extern "C" int sdbg_phrase_and_count_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms, const uint32_t* rel_pos,
                                           const uint32_t* clause_off, const uint8_t* clause_negated, const uint32_t* query_clause_off,
                                           size_t nq, const uint32_t* excl_terms, const uint32_t* excl_off, const sdbg_col_pred* filt,
                                           uint64_t* counts) {
  if (!query_clause_off) return SDBG_EINVAL;
  return phrase_count(segs, n_segs, {terms, rel_pos, clause_off, nullptr, clause_negated, query_clause_off, nq, excl_terms, excl_off},
                      filt, counts);
}

extern "C" int sdbg_phrase_groups_count_batch_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                  const uint32_t* rel_pos, const uint32_t* clause_off, const uint32_t* group_off,
                                                  const uint8_t* group_negated, const uint32_t* group_min,
                                                  const uint32_t* query_group_off, size_t nq, const uint32_t* excl_terms,
                                                  const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t* counts) {
  if (!group_off || !query_group_off) return SDBG_EINVAL;
  return phrase_count(segs, n_segs,
                      {terms, rel_pos, clause_off, group_off, group_negated, query_group_off, nq, excl_terms, excl_off, group_min},
                      filt, counts);
}

extern "C" int sdbg_phrase_groups_count_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                              const uint32_t* rel_pos, const uint32_t* clause_off, const uint32_t* group_off,
                                              const uint8_t* group_negated, const uint32_t* query_group_off, size_t nq,
                                              const uint32_t* excl_terms, const uint32_t* excl_off, const sdbg_col_pred* filt,
                                              uint64_t* counts) {
  return sdbg_phrase_groups_count_batch_min(segs, n_segs, terms, rel_pos, clause_off, group_off, group_negated, nullptr,
                                            query_group_off, nq, excl_terms, excl_off, filt, counts);
}

extern "C" int sdbg_phrase_topk_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms, const uint32_t* rel_pos,
                                      const uint32_t* phrase_off, size_t nq, const uint32_t* excl_terms, const uint32_t* excl_off,
                                      const sdbg_bm25_term* phrase_stats, float k1, float b, const sdbg_col_pred* filt, uint32_t k,
                                      float threshold_in, sdbg_hit* out, uint32_t* n_out, uint64_t* total_matches) {
  return phrase_topk(segs, n_segs, phrase_one(terms, rel_pos, phrase_off, nq, excl_terms, excl_off), phrase_stats, k1, b, filt, k,
                     threshold_in, out, n_out, total_matches);
}

extern "C" int sdbg_phrase_and_topk_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms, const uint32_t* rel_pos,
                                          const uint32_t* clause_off, const uint8_t* clause_negated, const uint32_t* query_clause_off,
                                          size_t nq, const uint32_t* excl_terms, const uint32_t* excl_off,
                                          const sdbg_bm25_term* clause_stats, float k1, float b, const sdbg_col_pred* filt, uint32_t k,
                                          float threshold_in, sdbg_hit* out, uint32_t* n_out, uint64_t* total_matches) {
  if (!query_clause_off) return SDBG_EINVAL;
  return phrase_topk(segs, n_segs, {terms, rel_pos, clause_off, nullptr, clause_negated, query_clause_off, nq, excl_terms, excl_off},
                     clause_stats, k1, b, filt, k, threshold_in, out, n_out, total_matches);
}

extern "C" int sdbg_phrase_groups_topk_batch_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                 const uint32_t* rel_pos, const uint32_t* clause_off, const uint32_t* group_off,
                                                 const uint8_t* group_negated, const uint32_t* group_min,
                                                 const uint32_t* query_group_off, size_t nq, const uint32_t* excl_terms,
                                                 const uint32_t* excl_off, const sdbg_bm25_term* clause_stats, float k1, float b,
                                                 const sdbg_col_pred* filt, uint32_t k, float threshold_in, sdbg_hit* out,
                                                 uint32_t* n_out, uint64_t* total_matches) {
  if (!group_off || !query_group_off) return SDBG_EINVAL;
  return phrase_topk(segs, n_segs,
                     {terms, rel_pos, clause_off, group_off, group_negated, query_group_off, nq, excl_terms, excl_off, group_min},
                     clause_stats, k1, b, filt, k, threshold_in, out, n_out, total_matches);
}

extern "C" int sdbg_phrase_groups_topk_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                             const uint32_t* rel_pos, const uint32_t* clause_off, const uint32_t* group_off,
                                             const uint8_t* group_negated, const uint32_t* query_group_off, size_t nq,
                                             const uint32_t* excl_terms, const uint32_t* excl_off,
                                             const sdbg_bm25_term* clause_stats, float k1, float b, const sdbg_col_pred* filt,
                                             uint32_t k, float threshold_in, sdbg_hit* out, uint32_t* n_out,
                                             uint64_t* total_matches) {
  return sdbg_phrase_groups_topk_batch_min(segs, n_segs, terms, rel_pos, clause_off, group_off, group_negated, nullptr,
                                           query_group_off, nq, excl_terms, excl_off, clause_stats, k1, b, filt, k, threshold_in,
                                           out, n_out, total_matches);
}

extern "C" int sdbg_phrase_topk_by_column_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms, const uint32_t* rel_pos,
                                                const uint32_t* phrase_off, size_t nq, const uint32_t* excl_terms,
                                                const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t sort_field,
                                                int descending, int nulls_first, uint32_t k, sdbg_sort_hit* out, uint32_t* n_out) {
  return phrase_topk_by_column(segs, n_segs, phrase_one(terms, rel_pos, phrase_off, nq, excl_terms, excl_off), filt, sort_field,
                               descending, nulls_first, k, out, n_out);
}

extern "C" int sdbg_phrase_and_topk_by_column_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                    const uint32_t* rel_pos, const uint32_t* clause_off, const uint8_t* clause_negated,
                                                    const uint32_t* query_clause_off, size_t nq, const uint32_t* excl_terms,
                                                    const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t sort_field,
                                                    int descending, int nulls_first, uint32_t k, sdbg_sort_hit* out, uint32_t* n_out) {
  if (!query_clause_off) return SDBG_EINVAL;
  return phrase_topk_by_column(segs, n_segs, {terms, rel_pos, clause_off, nullptr, clause_negated, query_clause_off, nq, excl_terms,
                                              excl_off}, filt, sort_field, descending, nulls_first, k, out, n_out);
}

extern "C" int sdbg_phrase_groups_topk_by_column_batch_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                           const uint32_t* rel_pos, const uint32_t* clause_off,
                                                           const uint32_t* group_off, const uint8_t* group_negated,
                                                           const uint32_t* group_min, const uint32_t* query_group_off, size_t nq,
                                                           const uint32_t* excl_terms, const uint32_t* excl_off,
                                                           const sdbg_col_pred* filt, uint64_t sort_field, int descending,
                                                           int nulls_first, uint32_t k, sdbg_sort_hit* out, uint32_t* n_out) {
  if (!group_off || !query_group_off) return SDBG_EINVAL;
  return phrase_topk_by_column(segs, n_segs,
                               {terms, rel_pos, clause_off, group_off, group_negated, query_group_off, nq, excl_terms, excl_off, group_min},
                               filt, sort_field, descending, nulls_first, k, out, n_out);
}

extern "C" int sdbg_phrase_groups_topk_by_column_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                       const uint32_t* rel_pos, const uint32_t* clause_off,
                                                       const uint32_t* group_off, const uint8_t* group_negated,
                                                       const uint32_t* query_group_off, size_t nq, const uint32_t* excl_terms,
                                                       const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t sort_field,
                                                       int descending, int nulls_first, uint32_t k, sdbg_sort_hit* out,
                                                       uint32_t* n_out) {
  return sdbg_phrase_groups_topk_by_column_batch_min(segs, n_segs, terms, rel_pos, clause_off, group_off, group_negated, nullptr,
                                                     query_group_off, nq, excl_terms, excl_off, filt, sort_field, descending,
                                                     nulls_first, k, out, n_out);
}

extern "C" int sdbg_phrase_facet_counts_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms, const uint32_t* rel_pos,
                                              const uint32_t* phrase_off, size_t nq, const uint32_t* excl_terms,
                                              const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t key_field,
                                              int64_t key_min, uint32_t key_span, uint64_t* counts, uint64_t* null_counts) {
  return phrase_facet_counts(segs, n_segs, phrase_one(terms, rel_pos, phrase_off, nq, excl_terms, excl_off), filt, key_field, key_min,
                             key_span, counts, null_counts);
}

extern "C" int sdbg_phrase_and_facet_counts_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms, const uint32_t* rel_pos,
                                                  const uint32_t* clause_off, const uint8_t* clause_negated,
                                                  const uint32_t* query_clause_off, size_t nq, const uint32_t* excl_terms,
                                                  const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t key_field,
                                                  int64_t key_min, uint32_t key_span, uint64_t* counts, uint64_t* null_counts) {
  if (!query_clause_off) return SDBG_EINVAL;
  return phrase_facet_counts(segs, n_segs, {terms, rel_pos, clause_off, nullptr, clause_negated, query_clause_off, nq, excl_terms,
                                            excl_off}, filt, key_field, key_min, key_span, counts, null_counts);
}

extern "C" int sdbg_phrase_groups_facet_counts_batch_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                         const uint32_t* rel_pos, const uint32_t* clause_off,
                                                         const uint32_t* group_off, const uint8_t* group_negated,
                                                         const uint32_t* group_min, const uint32_t* query_group_off, size_t nq,
                                                         const uint32_t* excl_terms, const uint32_t* excl_off,
                                                         const sdbg_col_pred* filt, uint64_t key_field, int64_t key_min,
                                                         uint32_t key_span, uint64_t* counts, uint64_t* null_counts) {
  if (!group_off || !query_group_off) return SDBG_EINVAL;
  return phrase_facet_counts(segs, n_segs,
                             {terms, rel_pos, clause_off, group_off, group_negated, query_group_off, nq, excl_terms, excl_off, group_min},
                             filt, key_field, key_min, key_span, counts, null_counts);
}

extern "C" int sdbg_phrase_groups_facet_counts_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                     const uint32_t* rel_pos, const uint32_t* clause_off,
                                                     const uint32_t* group_off, const uint8_t* group_negated,
                                                     const uint32_t* query_group_off, size_t nq, const uint32_t* excl_terms,
                                                     const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t key_field,
                                                     int64_t key_min, uint32_t key_span, uint64_t* counts,
                                                     uint64_t* null_counts) {
  return sdbg_phrase_groups_facet_counts_batch_min(segs, n_segs, terms, rel_pos, clause_off, group_off, group_negated, nullptr,
                                                   query_group_off, nq, excl_terms, excl_off, filt, key_field, key_min, key_span,
                                                   counts, null_counts);
}

extern "C" int sdbg_phrase_aggregate_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms, const uint32_t* rel_pos,
                                           const uint32_t* phrase_off, size_t nq, const uint32_t* excl_terms,
                                           const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t key_field,
                                           int64_t key_min, uint32_t key_span, uint64_t value_field, sdbg_match_agg* out,
                                           sdbg_match_agg* null_out) {
  return phrase_aggregate(segs, n_segs, phrase_one(terms, rel_pos, phrase_off, nq, excl_terms, excl_off), filt, key_field, key_min,
                          key_span, value_field, out, null_out);
}

extern "C" int sdbg_phrase_and_aggregate_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms, const uint32_t* rel_pos,
                                               const uint32_t* clause_off, const uint8_t* clause_negated,
                                               const uint32_t* query_clause_off, size_t nq, const uint32_t* excl_terms,
                                               const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t key_field,
                                               int64_t key_min, uint32_t key_span, uint64_t value_field, sdbg_match_agg* out,
                                               sdbg_match_agg* null_out) {
  if (!query_clause_off) return SDBG_EINVAL;
  return phrase_aggregate(segs, n_segs, {terms, rel_pos, clause_off, nullptr, clause_negated, query_clause_off, nq, excl_terms, excl_off},
                          filt, key_field, key_min, key_span, value_field, out, null_out);
}

extern "C" int sdbg_phrase_groups_aggregate_batch_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                      const uint32_t* rel_pos, const uint32_t* clause_off,
                                                      const uint32_t* group_off, const uint8_t* group_negated,
                                                      const uint32_t* group_min, const uint32_t* query_group_off, size_t nq,
                                                      const uint32_t* excl_terms, const uint32_t* excl_off,
                                                      const sdbg_col_pred* filt, uint64_t key_field, int64_t key_min,
                                                      uint32_t key_span, uint64_t value_field, sdbg_match_agg* out,
                                                      sdbg_match_agg* null_out) {
  if (!group_off || !query_group_off) return SDBG_EINVAL;
  return phrase_aggregate(segs, n_segs,
                          {terms, rel_pos, clause_off, group_off, group_negated, query_group_off, nq, excl_terms, excl_off, group_min},
                          filt, key_field, key_min, key_span, value_field, out, null_out);
}

extern "C" int sdbg_phrase_groups_aggregate_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                  const uint32_t* rel_pos, const uint32_t* clause_off, const uint32_t* group_off,
                                                  const uint8_t* group_negated, const uint32_t* query_group_off, size_t nq,
                                                  const uint32_t* excl_terms, const uint32_t* excl_off, const sdbg_col_pred* filt,
                                                  uint64_t key_field, int64_t key_min, uint32_t key_span, uint64_t value_field,
                                                  sdbg_match_agg* out, sdbg_match_agg* null_out) {
  return sdbg_phrase_groups_aggregate_batch_min(segs, n_segs, terms, rel_pos, clause_off, group_off, group_negated, nullptr,
                                                query_group_off, nq, excl_terms, excl_off, filt, key_field, key_min, key_span,
                                                value_field, out, null_out);
}

extern "C" int sdbg_match_topk_by_column_batch(sdbg_segment* const* segs, size_t n_segs, int kind, const uint32_t* terms,
                                               const uint32_t* term_off, size_t nq, const uint32_t* excl_terms,
                                               const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t sort_field,
                                               int descending, int nulls_first, uint32_t k, sdbg_sort_hit* out, uint32_t* n_out) {
  if (!segs || !n_segs || !segs[0] || !k || !out || !n_out) return SDBG_EINVAL;
  if (k > kSortMaxK) return fail(segs[0]->ctx, SDBG_EUNSUPPORTED, "k > 4096");
  const PassBatch<uint32_t> B(segs, n_segs, QueryBatch<uint32_t>{kind, terms, term_off, nq, excl_terms, excl_off, nullptr}, filt);
  return sort_to_host(segs, n_segs, B, filt, sort_field, descending, nulls_first, k, out, n_out);
}

extern "C" int sdbg_match_facet_counts_batch(sdbg_segment* const* segs, size_t n_segs, int kind, const uint32_t* terms,
                                             const uint32_t* term_off, size_t nq, const uint32_t* excl_terms,
                                             const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t key_field,
                                             int64_t key_min, uint32_t key_span, uint64_t* counts, uint64_t* null_counts) {
  if (!counts || !null_counts) return SDBG_EINVAL;
  const PassBatch<uint32_t> B(segs, n_segs, QueryBatch<uint32_t>{kind, terms, term_off, nq, excl_terms, excl_off, nullptr}, filt);
  CountJob job{CountMode::facet, {}, {key_field, key_min, key_span, {}}, {}};
  return pass_to_host(segs, n_segs, B, filt, job, words_region(nq, key_span),
                      [&](const char* h) { facet_fill(h, nq, key_span, counts, null_counts); });
}

extern "C" int sdbg_match_aggregate_batch(sdbg_segment* const* segs, size_t n_segs, int kind, const uint32_t* terms,
                                          const uint32_t* term_off, size_t nq, const uint32_t* excl_terms,
                                          const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t key_field,
                                          int64_t key_min, uint32_t key_span, uint64_t value_field, sdbg_match_agg* out,
                                          sdbg_match_agg* null_out) {
  if (!out || !null_out) return SDBG_EINVAL;
  const PassBatch<uint32_t> B(segs, n_segs, QueryBatch<uint32_t>{kind, terms, term_off, nq, excl_terms, excl_off, nullptr}, filt);
  return agg_to_host(segs, n_segs, B, filt, key_field, key_min, key_span, value_field, out, null_out);
}

extern "C" int sdbg_match_count_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                 const uint32_t* group_off, const uint32_t* query_group_off,
                                                 const uint32_t* group_min, size_t nq, const uint32_t* excl_terms,
                                                 const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t* counts) {
  if (!segs || !n_segs || !segs[0] || !group_off || !query_group_off || !nq || !counts) return SDBG_EINVAL;
  const PassBatch<uint32_t> B(segs, n_segs, terms, group_off, query_group_off, group_min, nq, excl_terms, excl_off, filt);
  CountJob job{CountMode::count, {}, {}, {}};
  return pass_to_host(segs, n_segs, B, filt, job, words_region(nq, 0), [&](const char* h) { std::memcpy(counts, h, nq * 8); });
}

extern "C" int sdbg_match_count_batch_groups(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                             const uint32_t* group_off, const uint32_t* query_group_off, size_t nq,
                                             const uint32_t* excl_terms, const uint32_t* excl_off, const sdbg_col_pred* filt,
                                             uint64_t* counts) {
  return sdbg_match_count_batch_groups_min(segs, n_segs, terms, group_off, query_group_off, nullptr, nq, excl_terms, excl_off,
                                           filt, counts);
}

extern "C" int sdbg_match_topk_by_column_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                          const uint32_t* group_off, const uint32_t* query_group_off,
                                                          const uint32_t* group_min, size_t nq, const uint32_t* excl_terms,
                                                          const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t sort_field,
                                                          int descending, int nulls_first, uint32_t k, sdbg_sort_hit* out,
                                                          uint32_t* n_out) {
  if (!segs || !n_segs || !segs[0] || !group_off || !query_group_off || !nq || !k || !out || !n_out) return SDBG_EINVAL;
  if (k > kSortMaxK) return fail(segs[0]->ctx, SDBG_EUNSUPPORTED, "k > 4096");
  const PassBatch<uint32_t> B(segs, n_segs, terms, group_off, query_group_off, group_min, nq, excl_terms, excl_off, filt);
  return sort_to_host(segs, n_segs, B, filt, sort_field, descending, nulls_first, k, out, n_out);
}

extern "C" int sdbg_match_facet_counts_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                        const uint32_t* group_off, const uint32_t* query_group_off,
                                                        const uint32_t* group_min, size_t nq, const uint32_t* excl_terms,
                                                        const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t key_field,
                                                        int64_t key_min, uint32_t key_span, uint64_t* counts,
                                                        uint64_t* null_counts) {
  if (!segs || !n_segs || !segs[0] || !group_off || !query_group_off || !nq || !counts || !null_counts) return SDBG_EINVAL;
  if (int rc = facet_check_range(segs[0]->ctx, key_min, key_span)) return rc;   // before the rows are sized
  const PassBatch<uint32_t> B(segs, n_segs, terms, group_off, query_group_off, group_min, nq, excl_terms, excl_off, filt);
  CountJob job{CountMode::facet, {}, {key_field, key_min, key_span, {}}, {}};
  return pass_to_host(segs, n_segs, B, filt, job, words_region(nq, key_span),
                      [&](const char* h) { facet_fill(h, nq, key_span, counts, null_counts); });
}

extern "C" int sdbg_match_aggregate_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                     const uint32_t* group_off, const uint32_t* query_group_off,
                                                     const uint32_t* group_min, size_t nq, const uint32_t* excl_terms,
                                                     const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t key_field,
                                                     int64_t key_min, uint32_t key_span, uint64_t value_field,
                                                     sdbg_match_agg* out, sdbg_match_agg* null_out) {
  if (!segs || !n_segs || !segs[0] || !group_off || !query_group_off || !nq || !out || !null_out) return SDBG_EINVAL;
  if (int rc = agg_check_range(segs[0]->ctx, key_field, key_min, key_span)) return rc;   // before the rows are sized
  const PassBatch<uint32_t> B(segs, n_segs, terms, group_off, query_group_off, group_min, nq, excl_terms, excl_off, filt);
  return agg_to_host(segs, n_segs, B, filt, key_field, key_min, key_span, value_field, out, null_out);
}

// ---- the match scan (Stream mode) ----
namespace {
static_assert(sizeof(sdbg_hit) == sizeof(EmitHit), "sdbg_hit layout");

struct ScanArgs {
  const uint64_t* offset;   // per query of the call (NULL: all 0)
  uint32_t limit;
  int scored;
  float k1, b;
};

// The match scan's region: [totals u64 [nq] | hits EmitHit [nq][limit] | n_out u32 [nq]].
PassRegion scan_region(size_t nq, uint32_t limit) {
  const size_t n_out = nq * 8 + nq * size_t(limit) * sizeof(EmitHit);
  return {0, nq * 8, n_out, kNone, kNone, n_out + nq * 4};
}

// Queues the match scan of a batch of one shape (checked; total_excl as check_query_batch set it) into out, zeroed:
// the emit pass over its count plan, then, when scored, emit_score_kernel over the pages. qpos: the call's position of
// each query (NULL: the same), which picks its offset.
int scan_run(sdbg_segment* const* segs, size_t n_segs, const QueryBatch<sdbg_bm25_term>& Q, uint32_t total_excl, const uint32_t* qpos,
             const sdbg_col_pred* filt, const ScanArgs& A, const CountOut& out) {
  sdbg_ctx* c = segs[0]->ctx;
  const size_t nq = Q.nq, n_terms = Q.term_off[nq];
  std::vector<uint32_t> ids(n_terms);
  for (size_t i = 0; i < n_terms; ++i) ids[i] = Q.terms[i].term;
  std::vector<unsigned long long> offs(nq, 0ull);
  if (A.offset)
    for (size_t q = 0; q < nq; ++q) offs[q] = A.offset[qpos ? qpos[q] : q];
  const QueryBatch<uint32_t> Qi{Q.kind, ids.data(), Q.term_off, nq, Q.excl_terms, Q.excl_off, Q.term_grp};
  CountJob job{CountMode::emit, {}, {}, {}, {A.limit, offs.data()}};
  if (int rc = count_run(segs, n_segs, count_plan(segs, n_segs, Qi, total_excl, filt, job), filt, job, out)) return rc;
  if (!A.scored) return SDBG_OK;
  // the scorer's staging: [PostingsDev [n_segs] | QTermDev [n_segs][n_terms] | qterm_off [nq + 1]]
  const size_t qt_pos = (n_segs * sizeof(PostingsDev) + 15) & ~size_t(15);
  const size_t off_pos = qt_pos + n_segs * n_terms * sizeof(QTermDev);
  std::vector<char> h(off_pos + (nq + 1) * 4);
  for (size_t si = 0; si < n_segs; ++si) {
    const PostingsDev p = postings_view(segs[si], 0);
    std::memcpy(h.data() + si * sizeof(PostingsDev), &p, sizeof(p));
  }
  qterms_by_cost(segs, n_segs, Q, A.k1, A.b, reinterpret_cast<QTermDev*>(h.data() + qt_pos));
  std::memcpy(h.data() + off_pos, Q.term_off, (nq + 1) * 4);
  DevBuf& b_sc = c->scratch[4];
  if (int rc = ensure(c, b_sc, h.size())) return rc;
  CU(c, cudaMemcpyAsync(b_sc.p, h.data(), h.size(), cudaMemcpyHostToDevice, c->stream));   // pageable: consumed on return
  const char* d = static_cast<const char*>(b_sc.p);
  EmitScoreParams P;
  P.segs = reinterpret_cast<const PostingsDev*>(d);
  P.qterms = reinterpret_cast<const QTermDev*>(d + qt_pos);
  P.qterm_off = reinterpret_cast<const uint32_t*>(d + off_pos);
  P.n_terms = uint32_t(n_terms);
  P.blocks_per_query = (A.limit + kEmitScoreHits - 1) / kEmitScoreHits;
  P.limit = A.limit;
  P.out = static_cast<EmitHit*>(out.bins);
  P.n_out = static_cast<const uint32_t*>(out.nulls);
  emit_score_kernel<<<unsigned(nq * P.blocks_per_query), kEmitScoreThreads, 0, c->stream>>>(P);
  ++c->launches;
  CU(c, cudaGetLastError());
  return SDBG_OK;
}

// The match scan of a checked batch of nq queries: run(o) queues it into the call's region in c->pass[0], zeroed; then
// one copy back through the pinned staging, one wait, and pass_finish.
template <class Run>
int scan_to_host(sdbg_ctx* c, size_t nq, uint32_t limit, Run run, sdbg_hit* out, uint32_t* n_out, uint64_t* total) {
  CU(c, cudaSetDevice(c->device));
  const PassRegion L = scan_region(nq, limit);
  if (int rc = ensure(c, c->pass[0], L.bytes)) return rc;
  if (int rc = ensure_pinned(c, L.bytes)) return rc;
  CU(c, cudaMemsetAsync(c->pass[0].p, 0, L.bytes, c->stream));
  if (int rc = run(L.at(c->pass[0].p))) return rc;
  CU(c, cudaMemcpyAsync(c->h_pinned, c->pass[0].p, L.bytes, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  return pass_finish(c, L, static_cast<const char*>(c->h_pinned), [&](const char* h) {
    std::memcpy(total, h + L.counts, nq * 8);
    std::memcpy(out, h + L.bins, nq * size_t(limit) * sizeof(sdbg_hit));
    std::memcpy(n_out, h + L.nulls, nq * 4);
  });
}

// The match scan of a checked batch B: scan_run for a whole batch, else shape by shape through shapes_run.
int scan_batch_to_host(sdbg_segment* const* segs, size_t n_segs, const PassBatch<sdbg_bm25_term>& B, const sdbg_col_pred* filt,
                       const ScanArgs& A, sdbg_hit* out, uint32_t* n_out, uint64_t* total) {
  if (B.rc) return B.rc;
  sdbg_ctx* c = segs[0]->ctx;
  return scan_to_host(c, B.nq, A.limit, [&](const CountOut& o) {
    if (B.whole.nq) return scan_run(segs, n_segs, B.whole, B.total_excl, nullptr, filt, A, o);
    const CountJob job{CountMode::emit, {}, {}, {}, {A.limit, nullptr}};
    return shapes_run(c, B.S, job.rows(false), {o.counts, o.bins, o.nulls}, [&](int sh, void* const* part) {
      return scan_run(segs, n_segs, B.S.view(sh), B.S.total_excl[sh], B.S.qs[sh].data(), filt, A,
                      CountOut{part[0], part[1], part[2], nullptr, nullptr, -1});
    });
  }, out, n_out, total);
}

// Queues the match scan of one shape Q of a checked phrase batch (total_excl as check_query_batch set it; J: the job of
// its queries) into out, zeroed: the emit pass with the alternatives, then, when scored (J.consts set),
// phrase_score_kernel over the pages. qpos: the call's position of each query (NULL: the same), which picks its offset.
// The scorer's staging: [PostingsDev [n_segs] | PhraseSink [n_segs] | the job's tables (PhraseJob::bytes)].
int phrase_scan_run(sdbg_segment* const* segs, size_t n_segs, const QueryBatch<uint32_t>& Q, uint32_t total_excl, const uint32_t* qpos,
                    const sdbg_col_pred* filt, const PhraseJob& J, const uint64_t* offset, uint32_t limit, const CountOut& out) {
  sdbg_ctx* c = segs[0]->ctx;
  const size_t nq = Q.nq;
  std::vector<unsigned long long> offs(nq, 0ull);
  if (offset)
    for (size_t q = 0; q < nq; ++q) offs[q] = offset[qpos ? qpos[q] : q];
  CountJob job{CountMode::emit, {}, {}, {}, {limit, offs.data()}};
  job.phrase = J;
  if (int rc = count_run(segs, n_segs, count_plan(segs, n_segs, Q, total_excl, filt, job), filt, job, out)) return rc;
  if (J.consts.empty()) return SDBG_OK;
  const size_t sinks_pos = (n_segs * sizeof(PostingsDev) + 15) & ~size_t(15);
  const size_t tables_pos = (sinks_pos + n_segs * sizeof(PhraseSink) + 15) & ~size_t(15);
  std::vector<char> h(tables_pos + J.bytes(n_segs));
  DevBuf& b_sc = c->scratch[4];
  if (int rc = ensure(c, b_sc, h.size())) return rc;
  const char* d = static_cast<const char*>(b_sc.p);
  for (size_t si = 0; si < n_segs; ++si) {
    const PostingsDev p = postings_view(segs[si], 0);
    std::memcpy(h.data() + si * sizeof(PostingsDev), &p, sizeof(p));
    PhraseSink F;
    J.sink(segs, n_segs, si, d + tables_pos, F);
    std::memcpy(h.data() + sinks_pos + si * sizeof(PhraseSink), &F, sizeof(F));
  }
  J.write(segs, n_segs, h.data() + tables_pos, Q.kind == SDBG_QUERY_AND);
  CU(c, cudaMemcpyAsync(b_sc.p, h.data(), h.size(), cudaMemcpyHostToDevice, c->stream));   // pageable: consumed on return
  PhraseScoreParams P;
  P.segs = reinterpret_cast<const PostingsDev*>(d);
  P.sinks = reinterpret_cast<const PhraseSink*>(d + sinks_pos);
  P.blocks_per_query = (limit + kEmitScoreThreads - 1) / kEmitScoreThreads;
  P.limit = limit;
  P.out = static_cast<EmitHit*>(out.bins);
  P.n_out = static_cast<const uint32_t*>(out.nulls);
  phrase_score_kernel<<<unsigned(nq * P.blocks_per_query), kEmitScoreThreads, 0, c->stream>>>(P);
  ++c->launches;
  CU(c, cudaGetLastError());
  return SDBG_OK;
}
}  // namespace

extern "C" int sdbg_match_scan_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const sdbg_bm25_term* terms,
                                                const uint32_t* group_off, const uint32_t* query_group_off,
                                                const uint32_t* group_min, size_t nq, const uint32_t* excl_terms,
                                                const uint32_t* excl_off, float k1, float b, const sdbg_col_pred* filt,
                                                const uint64_t* offset, uint32_t limit, int scored, sdbg_hit* out,
                                                uint32_t* n_out, uint64_t* total) {
  if (!segs || !n_segs || !segs[0] || !group_off || !query_group_off || !nq) return SDBG_EINVAL;
  if (!limit || !out || !n_out || !total) return SDBG_EINVAL;
  if (scored)
    if (int rc = topk_limits(segs[0]->ctx, nq, 1)) return rc;
  const PassBatch<sdbg_bm25_term> B(segs, n_segs, terms, group_off, query_group_off, group_min, nq, excl_terms, excl_off, filt);
  if (scored)
    if (int rc = topk_checked(segs, n_segs, B)) return rc;
  return scan_batch_to_host(segs, n_segs, B, filt, {offset, limit, scored, k1, b}, out, n_out, total);
}

namespace {
int phrase_scan(sdbg_segment* const* segs, size_t n_segs, const PhraseQueries& A, const sdbg_col_pred* filt,
                const sdbg_bm25_term* clause_stats, float k1, float b, const uint64_t* offset, uint32_t limit, int scored, sdbg_hit* out,
                uint32_t* n_out, uint64_t* total) {
  if (!limit || !out || !n_out || !total || (scored && !clause_stats)) return SDBG_EINVAL;
  const size_t nq = A.nq;
  PhraseBatch PB(segs, n_segs, A);
  if (PB.rc) return PB.rc;
  sdbg_ctx* c = segs[0]->ctx;
  if (scored)
    if (int rc = topk_limits(c, nq, 1)) return rc;
  const PassBatch<uint32_t> B(segs, n_segs, std::move(PB.S), nq, filt);
  if (B.rc) return B.rc;
  if (scored) {
    uint64_t ord = 0;
    for (size_t si = 0; si < n_segs; ++si) ord += segs[si]->n_docs;
    if (ord > kMaxDocId) return fail(c, SDBG_EUNSUPPORTED, "more than 2^32-2 docs per call");
  }
  if (int rc = phrase_positions_staged(segs, n_segs)) return rc;
  PhraseJob J = PB.job();
  if (scored) J.consts = PB.consts(segs, clause_stats, k1, b);
  return scan_to_host(c, nq, limit, [&](const CountOut& o) {
    if (B.whole.nq) return phrase_scan_run(segs, n_segs, B.whole, B.total_excl, nullptr, filt, J, offset, limit, o);
    const CountJob job{CountMode::emit, {}, {}, {}, {limit, nullptr}};
    return shapes_run(c, B.S, job.rows(false), {o.counts, o.bins, o.nulls}, [&](int sh, void* const* part) {
      return phrase_scan_run(segs, n_segs, B.S.view(sh), B.S.total_excl[sh], B.S.qs[sh].data(), filt, J.on(B.S.qs[sh]), offset, limit,
                             CountOut{part[0], part[1], part[2], nullptr, nullptr, -1});
    });
  }, out, n_out, total);
}
}  // namespace

extern "C" int sdbg_phrase_scan_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms, const uint32_t* rel_pos,
                                      const uint32_t* phrase_off, size_t nq, const uint32_t* excl_terms, const uint32_t* excl_off,
                                      const sdbg_col_pred* filt, const sdbg_bm25_term* phrase_stats, float k1, float b,
                                      const uint64_t* offset, uint32_t limit, int scored, sdbg_hit* out, uint32_t* n_out,
                                      uint64_t* total) {
  return phrase_scan(segs, n_segs, phrase_one(terms, rel_pos, phrase_off, nq, excl_terms, excl_off), filt, phrase_stats, k1, b, offset,
                     limit, scored, out, n_out, total);
}

extern "C" int sdbg_phrase_and_scan_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms, const uint32_t* rel_pos,
                                          const uint32_t* clause_off, const uint8_t* clause_negated, const uint32_t* query_clause_off,
                                          size_t nq, const uint32_t* excl_terms, const uint32_t* excl_off, const sdbg_col_pred* filt,
                                          const sdbg_bm25_term* clause_stats, float k1, float b, const uint64_t* offset,
                                          uint32_t limit, int scored, sdbg_hit* out, uint32_t* n_out, uint64_t* total) {
  if (!query_clause_off) return SDBG_EINVAL;
  return phrase_scan(segs, n_segs, {terms, rel_pos, clause_off, nullptr, clause_negated, query_clause_off, nq, excl_terms, excl_off},
                     filt, clause_stats, k1, b, offset, limit, scored, out, n_out, total);
}

extern "C" int sdbg_phrase_groups_scan_batch_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                 const uint32_t* rel_pos, const uint32_t* clause_off, const uint32_t* group_off,
                                                 const uint8_t* group_negated, const uint32_t* group_min,
                                                 const uint32_t* query_group_off, size_t nq, const uint32_t* excl_terms,
                                                 const uint32_t* excl_off, const sdbg_col_pred* filt,
                                                 const sdbg_bm25_term* clause_stats, float k1, float b, const uint64_t* offset,
                                                 uint32_t limit, int scored, sdbg_hit* out, uint32_t* n_out, uint64_t* total) {
  if (!group_off || !query_group_off) return SDBG_EINVAL;
  return phrase_scan(segs, n_segs,
                     {terms, rel_pos, clause_off, group_off, group_negated, query_group_off, nq, excl_terms, excl_off, group_min},
                     filt, clause_stats, k1, b, offset, limit, scored, out, n_out, total);
}

extern "C" int sdbg_phrase_groups_scan_batch(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                             const uint32_t* rel_pos, const uint32_t* clause_off, const uint32_t* group_off,
                                             const uint8_t* group_negated, const uint32_t* query_group_off, size_t nq,
                                             const uint32_t* excl_terms, const uint32_t* excl_off, const sdbg_col_pred* filt,
                                             const sdbg_bm25_term* clause_stats, float k1, float b, const uint64_t* offset,
                                             uint32_t limit, int scored, sdbg_hit* out, uint32_t* n_out, uint64_t* total) {
  return sdbg_phrase_groups_scan_batch_min(segs, n_segs, terms, rel_pos, clause_off, group_off, group_negated, nullptr,
                                           query_group_off, nq, excl_terms, excl_off, filt, clause_stats, k1, b, offset, limit,
                                           scored, out, n_out, total);
}

// ---- the count, facet, aggregate and sorted passes across GPUs ----
namespace {
// The dist entries' checks of the call's scalar arguments, which fail alike on every rank: before anything is queued.
int dist_check(sdbg_segment* const* segs, size_t n_segs, const uint32_t* group_off, const uint32_t* query_group_off, size_t nq) {
  if (!segs || !n_segs || !segs[0] || !group_off || !query_group_off || !nq) return SDBG_EINVAL;
  sdbg_ctx* c = segs[0]->ctx;
  if (c->dist_world > 1 && !c->nccl_comm) return fail(c, SDBG_EINVAL, "sdbg_dist_init has not run");
  return SDBG_OK;
}

// All-reduces `words` int64 words of this rank's buffer, whose last word is its failure flag, and copies them to the
// pinned staging: the call's one wait. rc_local: this rank's local pass. A flag set on any rank fails the call on every
// rank: the failing rank returns its own code, the others SDBG_EINVAL.
int dist_reduce_to_host(sdbg_ctx* c, int rc_local, unsigned long long* d, size_t words) {
  if (rc_local) CU(c, cudaMemsetAsync(d + words - 1, 1, 1, c->stream));
  if (int rc = sdbg_dist_allreduce_i64(c, d, words)) return rc_local ? rc_local : rc;
  if (int rc = ensure_pinned(c, words * 8)) return rc;
  CU(c, cudaMemcpyAsync(c->h_pinned, d, words * 8, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  if (rc_local) return rc_local;
  if (static_cast<const unsigned long long*>(c->h_pinned)[words - 1]) return fail(c, SDBG_EINVAL, "the call failed on another rank");
  return SDBG_OK;
}

// One thread per (query, key) cell: the cells of ranks 0 .. n_ranks - 1 in rank order. Counts are u64 sums, the integer
// sum a 128-bit add with its carry, the float64 sum the ranks' partials added in rank order (so every rank computes the
// same bits), MIN / MAX the maxima of the order keys. Block 0 also checks the headers: status = {headers disagree, some
// rank failed, some key out of range, the value type}.
__global__ void __launch_bounds__(256) agg_merge_gathered_kernel(const char* __restrict__ all, size_t rank_bytes, uint32_t n_ranks,
                                                                 unsigned long long nq, unsigned long long span,
                                                                 unsigned long long* __restrict__ status, AggCell* __restrict__ out) {
  const auto* h0 = reinterpret_cast<const AggDistHeader*>(all);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    unsigned long long bad = 0, failed = 0, oor = 0;
    for (uint32_t r = 0; r < n_ranks; ++r) {
      const auto* h = reinterpret_cast<const AggDistHeader*>(all + r * rank_bytes);
      bad |= h->type != h0->type || h->span != span || h->nq != nq;
      failed |= h->failed;
      oor |= h->out_of_range;
    }
    status[0] = bad; status[1] = failed; status[2] = oor; status[3] = h0->type;
  }
  const bool is_f64 = h0->type == SDBG_F64;
  const unsigned long long n = nq * (span + 1);
  for (unsigned long long i = blockIdx.x * 256ull + threadIdx.x; i < n; i += gridDim.x * 256ull) {
    AggCell a = reinterpret_cast<const AggCell*>(all + sizeof(AggDistHeader))[i];
    for (uint32_t r = 1; r < n_ranks; ++r) {
      const AggCell b = reinterpret_cast<const AggCell*>(all + r * rank_bytes + sizeof(AggDistHeader))[i];
      a.count += b.count;
      if (!b.count_value) continue;
      a.count_value += b.count_value;
      if (is_f64) {
        a.sum_lo = __double_as_longlong(__longlong_as_double(a.sum_lo) + __longlong_as_double(b.sum_lo));
      } else {
        const unsigned long long lo = a.sum_lo + b.sum_lo;
        a.sum_hi += b.sum_hi + (lo < a.sum_lo ? 1ull : 0ull);
        a.sum_lo = lo;
      }
      a.nmin = a.nmin > b.nmin ? a.nmin : b.nmin;
      a.max = a.max > b.max ? a.max : b.max;
    }
    out[i] = a;
  }
}

// The dist count and facet entries after their checks (B): this rank's region (words_region) in c->pass[0], zeroed, the
// pass run into it, one all-reduce of int64 over it, then the host entries' finish (pass_finish). A rank whose checks or
// pass fail still joins the collective, with its failure word set.
template <class Fill>
int dist_words(sdbg_segment* const* segs, size_t n_segs, const PassBatch<uint32_t>& B, const sdbg_col_pred* filt, CountJob& job, Fill fill) {
  sdbg_ctx* c = segs[0]->ctx;
  CU(c, cudaSetDevice(c->device));
  const PassRegion L = words_region(B.nq, job.mode == CountMode::facet ? job.facet.span : 0);
  if (int rc = ensure(c, c->pass[0], L.bytes)) return rc;
  int rc_local = B.rc ? B.rc : job_prepare(c, segs, n_segs, job);
  CU(c, cudaMemsetAsync(c->pass[0].p, 0, L.bytes, c->stream));
  if (!rc_local) rc_local = pass_run(segs, n_segs, B, filt, job, L.at(c->pass[0].p));
  if (int rc = dist_reduce_to_host(c, rc_local, static_cast<unsigned long long*>(c->pass[0].p), L.bytes / 8)) return rc;
  return pass_finish(c, L, static_cast<const char*>(c->h_pinned), fill);
}

// The aggregate and sorted device forms after their checks (B): zeroes the buffer (region L), writes its 64-byte header
// hdr, prepares the job and runs the pass into the buffer, with c->pass[3] zeroed for what the device forms do not
// report (the aggregate pass's counts, the sorted scan's windows). When the checks or the pass fail, sets the header's
// failure word (at byte `failed`), so that the rank still joins the collective and the merge fails.
int rank_device(sdbg_segment* const* segs, size_t n_segs, const PassBatch<uint32_t>& B, const sdbg_col_pred* filt, CountJob& job,
                const void* hdr, size_t failed, const PassRegion& L, int64_t rank, void* d_buf) {
  sdbg_ctx* c = segs[0]->ctx;
  CU(c, cudaSetDevice(c->device));
  int rc = B.rc ? B.rc : job_prepare(c, segs, n_segs, job);
  CU(c, cudaMemsetAsync(d_buf, 0, L.bytes, c->stream));
  CU(c, cudaMemcpyAsync(d_buf, hdr, 64, cudaMemcpyHostToDevice, c->stream));   // pageable: consumed on return
  CountOut out = L.at(d_buf, rank);
  if (!rc) rc = ensure(c, c->pass[3], B.nq * 8 + 16);
  if (!rc) {
    auto* scratch = static_cast<unsigned long long*>(c->pass[3].p);
    CU(c, cudaMemsetAsync(scratch, 0, B.nq * 8 + 16, c->stream));
    if (!out.counts) out.counts = scratch + 2;
    if (!out.stats) out.stats = scratch;
    rc = pass_run(segs, n_segs, B, filt, job, out);
  }
  if (rc) CU(c, cudaMemsetAsync(static_cast<char*>(d_buf) + failed, 1, 1, c->stream));
  return rc;
}
}  // namespace

extern "C" int sdbg_dist_match_count_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                      const uint32_t* group_off, const uint32_t* query_group_off,
                                                      const uint32_t* group_min, size_t nq, const uint32_t* excl_terms,
                                                      const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t* counts) {
  if (int rc = dist_check(segs, n_segs, group_off, query_group_off, nq)) return rc;
  if (!counts) return SDBG_EINVAL;
  CountJob job{CountMode::count, {}, {}, {}};
  const PassBatch<uint32_t> B(segs, n_segs, terms, group_off, query_group_off, group_min, nq, excl_terms, excl_off, filt);
  return dist_words(segs, n_segs, B, filt, job, [&](const char* h) { std::memcpy(counts, h, nq * 8); });
}

extern "C" int sdbg_dist_match_facet_counts_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                             const uint32_t* group_off, const uint32_t* query_group_off,
                                                             const uint32_t* group_min, size_t nq, const uint32_t* excl_terms,
                                                             const uint32_t* excl_off, const sdbg_col_pred* filt,
                                                             uint64_t key_field, int64_t key_min, uint32_t key_span,
                                                             uint64_t* counts, uint64_t* null_counts) {
  if (int rc = dist_check(segs, n_segs, group_off, query_group_off, nq)) return rc;
  if (!counts || !null_counts) return SDBG_EINVAL;
  if (int rc = facet_check_range(segs[0]->ctx, key_min, key_span)) return rc;
  CountJob job{CountMode::facet, {}, {key_field, key_min, key_span, {}}, {}};
  const PassBatch<uint32_t> B(segs, n_segs, terms, group_off, query_group_off, group_min, nq, excl_terms, excl_off, filt);
  return dist_words(segs, n_segs, B, filt, job, [&](const char* h) { facet_fill(h, nq, key_span, counts, null_counts); });
}

extern "C" int sdbg_match_aggregate_batch_groups_min_device(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                            const uint32_t* group_off, const uint32_t* query_group_off,
                                                            const uint32_t* group_min, size_t nq, const uint32_t* excl_terms,
                                                            const uint32_t* excl_off, const sdbg_col_pred* filt,
                                                            uint64_t key_field, int64_t key_min, uint32_t key_span,
                                                            uint64_t value_field, void* d_cells) {
  if (!segs || !n_segs || !segs[0] || !group_off || !query_group_off || !nq || !d_cells) return SDBG_EINVAL;
  if (int rc = agg_check_range(segs[0]->ctx, key_field, key_min, key_span)) return rc;
  CountJob job{CountMode::agg, {}, {}, {{key_field, key_min, key_span, {}}, value_field, {}}};
  const auto it = segs[0]->cols.find(value_field);   // the header's type: UINT64_MAX when not staged
  const AggDistHeader h{it == segs[0]->cols.end() ? UINT64_MAX : uint64_t(it->second.type), key_span, nq, 0, 0, {}};
  const PassBatch<uint32_t> B(segs, n_segs, terms, group_off, query_group_off, group_min, nq, excl_terms, excl_off, filt);
  return rank_device(segs, n_segs, B, filt, job, &h, offsetof(AggDistHeader, failed), agg_region(nq, key_span), -1, d_cells);
}

extern "C" int sdbg_match_aggregate_merge_gathered(sdbg_ctx* c, const void* d_all, uint32_t n_ranks, size_t nq, uint32_t key_span,
                                                   sdbg_match_agg* out, sdbg_match_agg* null_out) {
  if (!c || !d_all || !n_ranks || !nq || !key_span || !out || !null_out) return SDBG_EINVAL;
  if (key_span > kAggMaxSpan) return fail(c, SDBG_EUNSUPPORTED, "key_span > 4096");
  CU(c, cudaSetDevice(c->device));
  const size_t n = nq * (size_t(key_span) + 1), bytes = 64 + n * sizeof(AggCell);
  if (int rc = ensure(c, c->pass[3], bytes)) return rc;
  char* m = static_cast<char*>(c->pass[3].p);
  const unsigned grid = unsigned(std::max<size_t>(1, std::min<size_t>((n + 255) / 256, size_t(c->sm_count) * 16)));
  agg_merge_gathered_kernel<<<grid, 256, 0, c->stream>>>(static_cast<const char*>(d_all), agg_dist_bytes(nq, key_span), n_ranks, nq,
                                                        key_span, reinterpret_cast<unsigned long long*>(m),
                                                        reinterpret_cast<AggCell*>(m + 64));
  ++c->launches;
  CU(c, cudaGetLastError());
  if (int rc = ensure_pinned(c, bytes)) return rc;
  CU(c, cudaMemcpyAsync(c->h_pinned, m, bytes, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  const auto* st = static_cast<const unsigned long long*>(c->h_pinned);
  if (st[0]) return fail(c, SDBG_EINVAL, "the ranks' aggregate headers disagree (value type, key_span or n_queries)");
  if (st[1]) return fail(c, SDBG_EINVAL, "the aggregate pass failed on a rank");
  if (st[2]) return fail(c, SDBG_EINVAL, "a matching doc's key lies outside [key_min, key_min + key_span)");
  agg_results(reinterpret_cast<const AggCell*>(static_cast<const char*>(c->h_pinned) + 64), nq, key_span, uint32_t(st[3]), out,
              null_out);
  return SDBG_OK;
}

extern "C" int sdbg_dist_match_aggregate_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                          const uint32_t* group_off, const uint32_t* query_group_off,
                                                          const uint32_t* group_min, size_t nq, const uint32_t* excl_terms,
                                                          const uint32_t* excl_off, const sdbg_col_pred* filt, uint64_t key_field,
                                                          int64_t key_min, uint32_t key_span, uint64_t value_field,
                                                          sdbg_match_agg* out, sdbg_match_agg* null_out) {
  if (int rc = dist_check(segs, n_segs, group_off, query_group_off, nq)) return rc;
  if (!out || !null_out) return SDBG_EINVAL;
  sdbg_ctx* c = segs[0]->ctx;
  if (int rc = agg_check_range(c, key_field, key_min, key_span)) return rc;
  const uint32_t world = uint32_t(c->dist_world);
  const size_t bytes = agg_dist_bytes(nq, key_span);
  if (int rc = ensure(c, c->pass[0], bytes)) return rc;
  if (int rc = ensure(c, c->pass[1], bytes * world)) return rc;
  const int rc_local = sdbg_match_aggregate_batch_groups_min_device(segs, n_segs, terms, group_off, query_group_off, group_min, nq,
                                                                    excl_terms, excl_off, filt, key_field, key_min, key_span,
                                                                    value_field, c->pass[0].p);
  if (int rc = sdbg_dist_allgather(c, c->pass[0].p, c->pass[1].p, bytes)) return rc_local ? rc_local : rc;
  const int rc = sdbg_match_aggregate_merge_gathered(c, c->pass[1].p, world, nq, key_span, out, null_out);
  return rc_local ? rc_local : rc;
}

extern "C" int sdbg_match_topk_by_column_batch_groups_min_device(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                                 const uint32_t* group_off, const uint32_t* query_group_off,
                                                                 const uint32_t* group_min, size_t nq, const uint32_t* excl_terms,
                                                                 const uint32_t* excl_off, const sdbg_col_pred* filt,
                                                                 uint64_t sort_field, int descending, int nulls_first, uint32_t k,
                                                                 uint32_t rank, void* d_rows) {
  if (!segs || !n_segs || !segs[0] || !group_off || !query_group_off || !nq || !k || !d_rows) return SDBG_EINVAL;
  if (k > kSortMaxK) return fail(segs[0]->ctx, SDBG_EUNSUPPORTED, "k > 4096");
  if (rank > 0x7FFFFFFFu) return fail(segs[0]->ctx, SDBG_EUNSUPPORTED, "rank >= 2^31");
  CountJob job{CountMode::sort, {sort_field, descending, nulls_first, k, {}, {}}, {}, {}};
  const auto it = segs[0]->cols.find(sort_field);   // the header's type: UINT64_MAX when not staged
  const SortDistHeader h{it == segs[0]->cols.end() ? UINT64_MAX : uint64_t(it->second.type), descending ? 1u : 0u,
                         nulls_first ? 1u : 0u, k, nq, 0, {}};
  const PassBatch<uint32_t> B(segs, n_segs, terms, group_off, query_group_off, group_min, nq, excl_terms, excl_off, filt);
  return rank_device(segs, n_segs, B, filt, job, &h, offsetof(SortDistHeader, failed), sort_rank_region(nq, k), rank, d_rows);
}

extern "C" int sdbg_match_topk_by_column_merge_gathered(sdbg_ctx* c, const void* d_all, uint32_t n_ranks, size_t nq, uint32_t k,
                                                        sdbg_sort_hit* out, uint32_t* n_out) {
  if (!c || !d_all || !n_ranks || !nq || !k || !out || !n_out) return SDBG_EINVAL;
  if (k > kSortMaxK) return fail(c, SDBG_EUNSUPPORTED, "k > 4096");
  if (nq > 0x7FFFFFFFu) return fail(c, SDBG_EUNSUPPORTED, "more than 2^31 queries");
  CU(c, cudaSetDevice(c->device));
  const size_t hits_bytes = nq * size_t(k) * sizeof(SortHitDev), bytes = 64 + hits_bytes + nq * 4;
  if (int rc = ensure(c, c->pass[3], bytes)) return rc;
  char* m = static_cast<char*>(c->pass[3].p);
  const uint32_t cap = std::max(256u, 2u * next_pow2(k));
  CU(c, fit_dynamic_smem(sort_merge_gathered_kernel, size_t(cap) * 16));
  sort_merge_gathered_kernel<<<unsigned(nq), 256, size_t(cap) * 16, c->stream>>>(
      static_cast<const char*>(d_all), sort_dist_bytes(nq, k), n_ranks, uint32_t(nq), k, cap,
      reinterpret_cast<unsigned long long*>(m), reinterpret_cast<SortHitDev*>(m + 64), reinterpret_cast<uint32_t*>(m + 64 + hits_bytes));
  ++c->launches;
  CU(c, cudaGetLastError());
  if (int rc = ensure_pinned(c, bytes)) return rc;
  CU(c, cudaMemcpyAsync(c->h_pinned, m, bytes, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  const auto* st = static_cast<const unsigned long long*>(c->h_pinned);
  if (st[0]) return fail(c, SDBG_EINVAL, "the ranks' sorted-scan headers disagree (sort type, order, k or n_queries)");
  if (st[1]) return fail(c, SDBG_EINVAL, "the sorted scan failed on a rank");
  std::memcpy(out, static_cast<const char*>(c->h_pinned) + 64, hits_bytes);
  std::memcpy(n_out, static_cast<const char*>(c->h_pinned) + 64 + hits_bytes, nq * 4);
  return SDBG_OK;
}

extern "C" int sdbg_dist_match_topk_by_column_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const uint32_t* terms,
                                                               const uint32_t* group_off, const uint32_t* query_group_off,
                                                               const uint32_t* group_min, size_t nq, const uint32_t* excl_terms,
                                                               const uint32_t* excl_off, const sdbg_col_pred* filt,
                                                               uint64_t sort_field, int descending, int nulls_first, uint32_t k,
                                                               sdbg_sort_hit* out, uint32_t* n_out) {
  if (int rc = dist_check(segs, n_segs, group_off, query_group_off, nq)) return rc;
  if (!k || !out || !n_out) return SDBG_EINVAL;
  sdbg_ctx* c = segs[0]->ctx;
  if (k > kSortMaxK) return fail(c, SDBG_EUNSUPPORTED, "k > 4096");
  const uint32_t world = uint32_t(c->dist_world);
  const size_t bytes = sort_dist_bytes(nq, k);
  if (int rc = ensure(c, c->pass[0], bytes)) return rc;
  if (int rc = ensure(c, c->pass[1], bytes * world)) return rc;
  const int rc_local = sdbg_match_topk_by_column_batch_groups_min_device(segs, n_segs, terms, group_off, query_group_off, group_min,
                                                                         nq, excl_terms, excl_off, filt, sort_field, descending,
                                                                         nulls_first, k, uint32_t(c->dist_rank), c->pass[0].p);
  if (int rc = sdbg_dist_allgather(c, c->pass[0].p, c->pass[1].p, bytes)) return rc_local ? rc_local : rc;
  const int rc = sdbg_match_topk_by_column_merge_gathered(c, c->pass[1].p, world, nq, k, out, n_out);
  return rc_local ? rc_local : rc;
}

// Streaming mode (duckdb_search_full_scan.cpp RunStreamingScan :2370-2403; DocIterator::EmitScoredDocs,
// iterators.hpp:202-204): every match of one query in docs [doc_min, doc_max) of one segment with its score, ascending
// by doc. Same stream kernel as the top-k scan with pruning off; its sink writes through a global cursor and the
// pairs are then radix-sorted by doc id on the device.
namespace {
int scan_run(sdbg_segment* s, int kind, const sdbg_bm25_term* terms, size_t n_terms, const uint32_t* excl_terms, size_t n_excl,
             float k1, float b, const sdbg_col_pred* filt, uint32_t doc_min, uint32_t doc_max, uint32_t* out_docs, float* out_scores,
             uint64_t cap, uint64_t* n_out) {
  if (!s || !terms || !n_terms || !n_out || (cap && (!out_docs || !out_scores))) return SDBG_EINVAL;
  sdbg_ctx* c = s->ctx;
  CU(c, cudaSetDevice(c->device));
  if (!s->d_blocks) return fail(c, SDBG_EINVAL, "segment has no staged postings");
  if (n_excl > kMaxQueryTerms) return fail(c, SDBG_EUNSUPPORTED, "a query excludes at most 16 terms");
  if (n_excl && !excl_terms) return fail(c, SDBG_EINVAL, "excl_terms is NULL");
  const bool conj = kind == SDBG_QUERY_AND;
  if (n_terms > (conj ? size_t(kMaxQueryTerms) : size_t(kStreamMaxTerms)))
    return fail(c, SDBG_EUNSUPPORTED, "scored scan: disjunctions take 1..4 terms, conjunctions 1..16");
  if (k1 == 0.f || b == 0.f || k1 == kTfidfK1) return fail(c, SDBG_EUNSUPPORTED, "scored scan: BM25 form only");
  *n_out = 0;
  doc_min = std::max(doc_min, 1u);                                   // doc ids start at doc_limits::min()
  doc_max = uint32_t(std::min<uint64_t>(doc_max, uint64_t(s->n_docs) + 1u));
  if (doc_min >= doc_max) return SDBG_OK;
  const uint32_t range = doc_max - doc_min;
  const uint32_t T = uint32_t(n_terms);
  const uint32_t scan_cap = 1024;                                    // candidate buffer of the kernel: unused here, kept minimal
  const uint32_t g = std::max(1u, std::min(uint32_t(c->sm_count) * 3u, range / 4096u));
  const uint32_t chunk = uint32_t((uint64_t(range) + g - 1) / g);   // 64-bit: range reaches 2^32 - 2
  for (uint32_t i = 0; i < T; ++i)
    if (terms[i].term + 1 >= s->term_blk_begin.size()) return fail(c, SDBG_EINVAL, "term id out of range");
  ChainDev chain;
  if (int rc = filter_chains(&s, 1, filt, &chain)) return rc;
  // one query, one candidate list per chain, its excluded terms as its check lists
  std::vector<uint4> work(g);
  for (uint32_t j = 0; j < g; ++j) {
    const uint32_t lo = doc_min + j * chunk;
    work[j] = make_uint4(0u, lo, lo < doc_max ? std::min(chunk, doc_max - lo) : 0u, j);
    if (lo >= doc_max) work[j].y = s->n_docs + 1u;               // empty chain
  }
  const uint32_t term_off[2] = {0, T};
  const TopkDesc D = topk_desc(&s, 1, {kind, terms, term_off, 1, nullptr, nullptr, nullptr}, k1, b, work, {0, g},
                               std::vector<uint32_t>(excl_terms, excl_terms + n_excl), {0, uint32_t(n_excl)}, {});
  int rc;
  DevBuf& b_qt = c->scratch[0]; DevBuf& b_theta = c->scratch[1]; DevBuf& b_cand = c->scratch[2]; DevBuf& b_candn = c->scratch[3];
  DevBuf& b_emit = c->scratch[12];
  const uint64_t room = std::max<uint64_t>(cap, 1);
  size_t sort_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, static_cast<const uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr),
                                  static_cast<const float*>(nullptr), static_cast<float*>(nullptr), room, 0, 32, c->stream);
  const size_t pair_bytes = (size_t(room) * 4 + 255) & ~size_t(255);
  if ((rc = ensure(c, b_qt, D.h.size()))) return rc;
  if ((rc = ensure(c, b_theta, 32))) return rc;                      // theta | total | cursor
  if ((rc = ensure(c, b_cand, size_t(g) * scan_cap * 8))) return rc;
  if ((rc = ensure(c, b_candn, size_t(g) * 4))) return rc;
  if ((rc = ensure(c, b_emit, 4 * pair_bytes + sort_bytes))) return rc;
  CU(c, cudaMemcpyAsync(b_qt.p, D.h.data(), D.h.size(), cudaMemcpyHostToDevice, c->stream));
  CU(c, cudaMemsetAsync(b_theta.p, 0, 32, c->stream));
  TopkParams P;
  P.seg = postings_view(s, 0);
  P.filt = chain;
  D.params(static_cast<const char*>(b_qt.p), 0, 0, P);
  P.theta = static_cast<unsigned long long*>(b_theta.p);
  P.total = P.theta + 1;
  P.emit_count = P.theta + 2;
  P.cand = static_cast<unsigned long long*>(b_cand.p);
  P.cand_n = static_cast<uint32_t*>(b_candn.p);
  P.claim = nullptr;
  P.k = 1; P.cap = scan_cap; P.conjunction = conj ? 1 : 0; P.wand = 0;
  char* e = static_cast<char*>(b_emit.p);
  P.emit_docs = reinterpret_cast<uint32_t*>(e);
  P.emit_scores = reinterpret_cast<float*>(e + pair_bytes);
  P.emit_cap = cap;
  auto* sorted_docs = reinterpret_cast<uint32_t*>(e + 2 * pair_bytes);
  auto* sorted_scores = reinterpret_cast<float*>(e + 3 * pair_bytes);
  if ((rc = topk_smem_attrs(c))) return rc;
  TopkKernel kern;
  if (n_excl) kern = conj ? stream_kernel<kModeAnd, true>(1) : stream_kernel<kModeOr, true>(T);   // as in topk_run
  else kern = conj ? stream_kernel<kModeAnd>(1) : stream_kernel<kModeOr>(T);
  {
    ProfScope ps_(c, kProfTopk);
    kern<<<g, kTopkThreads, stream_smem(scan_cap, conj ? 1u : T, conj), c->stream>>>(P);
  }
  ++c->launches;
  CU(c, cudaGetLastError());
  unsigned long long found = 0;
  CU(c, cudaMemcpyAsync(&found, P.emit_count, 8, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  *n_out = found;
  if (found > cap) return fail(c, SDBG_ECAPACITY, "scored scan: more matches than the output has room for (*n_out = needed)");
  if (!found) return SDBG_OK;
  cub::DeviceRadixSort::SortPairs(e + 4 * pair_bytes, sort_bytes, P.emit_docs, sorted_docs, P.emit_scores, sorted_scores, found, 0, 32,
                                  c->stream);
  ++c->launches;
  CU(c, cudaGetLastError());
  CU(c, cudaMemcpyAsync(out_docs, sorted_docs, size_t(found) * 4, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaMemcpyAsync(out_scores, sorted_scores, size_t(found) * 4, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  return SDBG_OK;
}
}  // namespace

extern "C" int sdbg_bm25_scan(sdbg_segment* s, int kind, const sdbg_bm25_term* terms, size_t n_terms, float k1, float b,
                              const sdbg_col_pred* filt, uint32_t doc_min, uint32_t doc_max, uint32_t* out_docs, float* out_scores,
                              uint64_t cap, uint64_t* n_out) {
  return scan_run(s, kind, terms, n_terms, nullptr, 0, k1, b, filt, doc_min, doc_max, out_docs, out_scores, cap, n_out);
}

extern "C" int sdbg_bm25_scan_excl(sdbg_segment* s, int kind, const sdbg_bm25_term* terms, size_t n_terms, const uint32_t* excl_terms,
                                   size_t n_excl, float k1, float b, const sdbg_col_pred* filt, uint32_t doc_min, uint32_t doc_max,
                                   uint32_t* out_docs, float* out_scores, uint64_t cap, uint64_t* n_out) {
  return scan_run(s, kind, terms, n_terms, excl_terms, n_excl, k1, b, filt, doc_min, doc_max, out_docs, out_scores, cap, n_out);
}

extern "C" int sdbg_bm25_topk(sdbg_segment* const* segs, size_t n_segs, int kind, const sdbg_bm25_term* terms,
                              size_t n_terms, float k1, float b, const sdbg_col_pred* filt, uint32_t k, float threshold_in,
                              sdbg_hit* out, uint32_t* n_out, uint64_t* total_matches, float* threshold_out) {
  const uint32_t off[2] = {0, uint32_t(n_terms)};
  uint64_t tot = 0;
  const int rc = sdbg_bm25_topk_batch(segs, n_segs, kind, terms, off, 1, k1, b, filt, k, threshold_in, out, n_out, &tot);
  if (rc) return rc;
  if (total_matches) *total_matches = tot;
  if (threshold_out) *threshold_out = (*n_out == k) ? out[k - 1].score : threshold_in;
  return SDBG_OK;
}

namespace {
__global__ void shift_keys_kernel(unsigned long long* __restrict__ keys, size_t n, uint32_t add) {
  // Re-bases ordinals for a cross-rank gather: ordinal' = ordinal + add (keys keep their order within a rank).
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += size_t(gridDim.x) * blockDim.x) {
    const unsigned long long k = keys[i];
    keys[i] = k ? ((k & 0xFFFFFFFF00000000ull) | static_cast<unsigned long long>(~(~uint32_t(k) + add))) : 0ull;
  }
}

// The device form: the batch's keys straight into d_keys, its ordinals shifted into the rank's slot there, and its
// totals into d_totals (NULL: not wanted). sync: wait for the stream before returning.
int topk_batch_device(sdbg_segment* const* segs, size_t n_segs, int kind, const sdbg_bm25_term* terms, const uint32_t* term_off,
                      size_t nq, float k1, float b, const sdbg_col_pred* filt, uint32_t k, float threshold_in, uint32_t rank,
                      void* d_keys, void* d_totals, bool sync) {
  if (!d_keys || !segs || !n_segs) return SDBG_EINVAL;
  for (size_t si = 0; si < n_segs; ++si) if (!segs[si]) return SDBG_EINVAL;
  sdbg_ctx* c = segs[0]->ctx;
  // Each rank owns a 2^28-ordinal slot in the merged key space: rank r's docs sort after rank r-1's on ties. Checked
  // before the scan is queued, so a rejected call does no work.
  uint64_t docs = 0;
  for (size_t si = 0; si < n_segs; ++si) docs += segs[si]->n_docs;
  if (rank >= 15) return fail(c, SDBG_EUNSUPPORTED, "rank slot overflow (rank >= 15)");
  if (docs >= (1ull << 28)) return fail(c, SDBG_EUNSUPPORTED, "rank slot overflow (>= 2^28 docs per rank)");
  if (int rc = topk_args(segs, n_segs, nq, k)) return rc;
  const PassBatch<sdbg_bm25_term> B(segs, n_segs, {kind, terms, term_off, nq, nullptr, nullptr, nullptr}, filt);
  if (int rc = topk_checked(segs, n_segs, B)) return rc;
  DevBuf& b_n_out = c->scratch[5];   // the hit counts, which the device form does not report
  if (int rc = ensure(c, b_n_out, nq * 4)) return rc;
  auto* keys = static_cast<unsigned long long*>(d_keys);
  if (int rc = topk_run(segs, n_segs, B.whole, B.total_excl, k1, b, filt, k, threshold_in,
                        {keys, static_cast<uint32_t*>(b_n_out.p), static_cast<unsigned long long*>(d_totals)}))
    return rc;
  shift_keys_kernel<<<256, 256, 0, c->stream>>>(keys, nq * size_t(k), rank << 28);
  ++c->launches;
  CU(c, cudaGetLastError());
  if (sync) CU(c, cudaStreamSynchronize(c->stream));
  return SDBG_OK;
}
}  // namespace

extern "C" int sdbg_bm25_topk_batch_device(sdbg_segment* const* segs, size_t n_segs, int kind, const sdbg_bm25_term* terms,
                                           const uint32_t* term_off, size_t nq, float k1, float b, const sdbg_col_pred* filt,
                                           uint32_t k, float threshold_in, uint32_t rank, void* d_keys, void* d_totals) {
  return topk_batch_device(segs, n_segs, kind, terms, term_off, nq, k1, b, filt, k, threshold_in, rank, d_keys, d_totals, true);
}

extern "C" int sdbg_topk_merge_gathered(sdbg_ctx* c, const void* d_keys_all, uint32_t n_ranks, size_t nq, uint32_t k,
                                        sdbg_hit* out, uint32_t* n_out) {
  if (!c || !d_keys_all || !n_ranks || !nq || !k || (out && !n_out)) return SDBG_EINVAL;   // out == NULL: n_out != NULL asks for a sync
  if (int rc = topk_limits(c, nq, k)) return rc;   // the keys come from top-k entries, which produce no larger lists
  CU(c, cudaSetDevice(c->device));
  // gathered layout [rank][query][k]; the merge kernel wants [query][list][stride] -> stride trick:
  // treat each rank's block as a list with a rank-major base pointer. Re-pack with a tiny kernel-free
  // copy: n_ranks strided memcpy2D calls.
  DevBuf& b_in = c->scratch[6]; DevBuf& b_keys = c->scratch[7]; DevBuf& b_small = c->scratch[8];
  int rc;
  if ((rc = ensure(c, b_in, nq * size_t(n_ranks) * k * 8))) return rc;
  if ((rc = ensure(c, b_keys, nq * size_t(k) * 8))) return rc;
  if ((rc = ensure(c, b_small, nq * 4))) return rc;
  for (uint32_t r = 0; r < n_ranks; ++r)
    CU(c, cudaMemcpy2DAsync(static_cast<char*>(b_in.p) + size_t(r) * k * 8, size_t(n_ranks) * k * 8,
                            static_cast<const char*>(d_keys_all) + size_t(r) * nq * k * 8, size_t(k) * 8, size_t(k) * 8, nq,
                            cudaMemcpyDeviceToDevice, c->stream));
  const uint32_t cap = std::max(next_pow2(k + 1024), 4096u);
  if ((rc = topk_smem_attrs(c))) return rc;
  MergeParams M;
  M.cand = static_cast<const unsigned long long*>(b_in.p); M.cand_n = nullptr; M.list_off = nullptr;
  M.G = n_ranks; M.stride = k; M.k = k; M.cap = cap;
  M.keys_out = static_cast<unsigned long long*>(b_keys.p); M.n_out = static_cast<uint32_t*>(b_small.p);
  topk_merge_kernel<<<unsigned(nq), kTopkThreads, size_t(cap) * 8, c->stream>>>(M);
  ++c->launches;
  CU(c, cudaGetLastError());
  if (!out && !n_out) return SDBG_OK;                                       // enqueue only: results stay in HBM, nothing waits
  if (!out) { CU(c, cudaStreamSynchronize(c->stream)); return SDBG_OK; }   // results stay in HBM (scratch of this context)
  // an ordinal is its rank's slot (ordinal >> 28) and the ordinal within the rank (segment base + doc)
  return topk_to_host(c, {M.keys_out, M.n_out, nullptr}, nq, k,
                      [](uint32_t ordinal) { return make_uint2(ordinal >> 28, ordinal & ((1u << 28) - 1)); }, out, n_out, nullptr);
}

// ---- the BM25 top-k of group queries across GPUs: no rank slots (TopkDistHeader, bm25_kernels.cuh) ----
extern "C" int sdbg_bm25_topk_batch_groups_min_device(sdbg_segment* const* segs, size_t n_segs, const sdbg_bm25_term* terms,
                                                      const uint32_t* group_off, const uint32_t* query_group_off,
                                                      const uint32_t* group_min, size_t nq, const uint32_t* excl_terms,
                                                      const uint32_t* excl_off, float k1, float b, const sdbg_col_pred* filt,
                                                      uint32_t k, float threshold_in, void* d_buf) {
  if (!group_off || !query_group_off || !d_buf) return SDBG_EINVAL;
  if (int rc = topk_args(segs, n_segs, nq, k)) return rc;
  sdbg_ctx* c = segs[0]->ctx;
  const PassBatch<sdbg_bm25_term> B(segs, n_segs, terms, group_off, query_group_off, group_min, nq, excl_terms, excl_off, filt);
  const TopkDistHeader h{k, nq, 0, {}};
  CU(c, cudaMemsetAsync(d_buf, 0, topk_dist_bytes(nq, k), c->stream));
  CU(c, cudaMemcpyAsync(d_buf, &h, sizeof(h), cudaMemcpyHostToDevice, c->stream));   // pageable: consumed on return
  int rc = topk_checked(segs, n_segs, B);
  if (!rc) rc = topk_batch_run(segs, n_segs, B, k1, b, filt, k, threshold_in,
                               topk_region(static_cast<char*>(d_buf) + sizeof(TopkDistHeader), nq, k));
  if (rc) CU(c, cudaMemsetAsync(static_cast<char*>(d_buf) + offsetof(TopkDistHeader, failed), 1, 1, c->stream));
  return rc;
}

// Checks the n_ranks headers on the host (one small copy and a wait) so that a bad gather queues no kernel, then re-keys
// the lists by position (topk_rekey_gathered_kernel), selects each query's k best with topk_merge_kernel and maps them back
// to hits (topk_hits_gathered_kernel); one copy back of [totals | hits | n_out] through the pinned staging.
extern "C" int sdbg_bm25_topk_merge_gathered(sdbg_ctx* c, const void* d_all, uint32_t n_ranks, size_t nq, uint32_t k,
                                             sdbg_hit* out, uint32_t* n_out, uint64_t* total_matches) {
  if (!c || !d_all || !n_ranks || !nq || !k || !out || !n_out) return SDBG_EINVAL;
  if (int rc = topk_limits(c, nq, k)) return rc;
  if (uint64_t(n_ranks) * k >= (1ull << 32)) return fail(c, SDBG_EUNSUPPORTED, "n_ranks * k >= 2^32");
  CU(c, cudaSetDevice(c->device));
  static_assert(sizeof(sdbg_hit) == sizeof(uint3), "topk_hits_gathered_kernel writes sdbg_hit as uint3");
  const size_t rank_bytes = topk_dist_bytes(nq, k), hits_bytes = nq * size_t(k) * sizeof(sdbg_hit);
  const size_t out_bytes = nq * 8 + hits_bytes + nq * 4;
  if (int rc = ensure_pinned(c, std::max(size_t(n_ranks) * sizeof(TopkDistHeader), out_bytes))) return rc;
  CU(c, cudaMemcpy2DAsync(c->h_pinned, sizeof(TopkDistHeader), d_all, rank_bytes, sizeof(TopkDistHeader), n_ranks,
                          cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  const auto* hdr = static_cast<const TopkDistHeader*>(c->h_pinned);
  for (uint32_t r = 0; r < n_ranks; ++r) {
    if (hdr[r].k != k || hdr[r].nq != nq) return fail(c, SDBG_EINVAL, "the ranks' top-k headers disagree (k or n_queries)");
    if (hdr[r].failed) return fail(c, SDBG_EINVAL, "the top-k pass failed on a rank");
  }
  const size_t rows = nq * n_ranks;
  DevBuf& b_in = c->scratch[6]; DevBuf& b_keys = c->scratch[7];
  int rc;
  if ((rc = ensure(c, b_in, rows * size_t(k) * 8 + rows * 4))) return rc;
  if ((rc = ensure(c, b_keys, nq * size_t(k) * 8))) return rc;
  if ((rc = ensure(c, c->pass[3], out_bytes))) return rc;
  if ((rc = topk_smem_attrs(c))) return rc;
  auto* pos_keys = static_cast<unsigned long long*>(b_in.p);
  auto* cand_n = reinterpret_cast<uint32_t*>(pos_keys + rows * k);
  char* m = static_cast<char*>(c->pass[3].p);   // [totals u64 [nq] | hits [nq][k] | n_out u32 [nq]]
  auto* d_totals = reinterpret_cast<unsigned long long*>(m);
  auto* d_hits = reinterpret_cast<uint3*>(m + nq * 8);
  auto* d_n_out = reinterpret_cast<uint32_t*>(m + nq * 8 + hits_bytes);
  const char* all = static_cast<const char*>(d_all);
  const unsigned grid = unsigned(std::min<size_t>(rows, size_t(c->sm_count) * 16));
  topk_rekey_gathered_kernel<<<grid, 256, 0, c->stream>>>(all, rank_bytes, n_ranks, uint32_t(nq), k, pos_keys, cand_n);
  ++c->launches;
  const uint32_t cap = std::max(next_pow2(k + 1024), 4096u);   // as sdbg_topk_merge_gathered
  MergeParams M;
  M.cand = pos_keys; M.cand_n = cand_n; M.list_off = nullptr;
  M.G = n_ranks; M.stride = k; M.k = k; M.cap = cap;
  M.keys_out = static_cast<unsigned long long*>(b_keys.p); M.n_out = d_n_out;
  topk_merge_kernel<<<unsigned(nq), kTopkThreads, size_t(cap) * 8, c->stream>>>(M);
  ++c->launches;
  topk_hits_gathered_kernel<<<unsigned(nq), 256, 0, c->stream>>>(all, rank_bytes, n_ranks, uint32_t(nq), k, M.keys_out, d_n_out,
                                                                 d_hits, d_totals);
  ++c->launches;
  CU(c, cudaGetLastError());
  CU(c, cudaMemcpyAsync(c->h_pinned, m, out_bytes, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  const char* h = static_cast<const char*>(c->h_pinned);
  std::memcpy(n_out, h + nq * 8 + hits_bytes, nq * 4);
  if (total_matches) std::memcpy(total_matches, h, nq * 8);
  const auto* hits = reinterpret_cast<const sdbg_hit*>(h + nq * 8);
  for (size_t q = 0; q < nq; ++q) std::memcpy(out + q * k, hits + q * k, n_out[q] * sizeof(sdbg_hit));
  return SDBG_OK;
}

extern "C" int sdbg_dist_bm25_topk_batch_groups_min(sdbg_segment* const* segs, size_t n_segs, const sdbg_bm25_term* terms,
                                                    const uint32_t* group_off, const uint32_t* query_group_off,
                                                    const uint32_t* group_min, size_t nq, const uint32_t* excl_terms,
                                                    const uint32_t* excl_off, float k1, float b, const sdbg_col_pred* filt,
                                                    uint32_t k, float threshold_in, sdbg_hit* out, uint32_t* n_out,
                                                    uint64_t* total_matches) {
  if (int rc = dist_check(segs, n_segs, group_off, query_group_off, nq)) return rc;
  if (!k || !out || !n_out) return SDBG_EINVAL;
  sdbg_ctx* c = segs[0]->ctx;
  if (int rc = topk_limits(c, nq, k)) return rc;
  const uint32_t world = uint32_t(c->dist_world);
  if (uint64_t(world) * k >= (1ull << 32)) return fail(c, SDBG_EUNSUPPORTED, "n_ranks * k >= 2^32");
  const size_t bytes = topk_dist_bytes(nq, k);
  if (int rc = ensure(c, c->pass[0], bytes)) return rc;
  if (int rc = ensure(c, c->pass[1], bytes * world)) return rc;
  const int rc_local = sdbg_bm25_topk_batch_groups_min_device(segs, n_segs, terms, group_off, query_group_off, group_min, nq,
                                                              excl_terms, excl_off, k1, b, filt, k, threshold_in, c->pass[0].p);
  if (int rc = sdbg_dist_allgather(c, c->pass[0].p, c->pass[1].p, bytes)) return rc_local ? rc_local : rc;
  const int rc = sdbg_bm25_topk_merge_gathered(c, c->pass[1].p, world, nq, k, out, n_out, total_matches);
  return rc_local ? rc_local : rc;
}

extern "C" int sdbg_decode_score_term(sdbg_segment* s, uint32_t term, float c0, float nc, float nl, uint32_t* docs,
                                      uint32_t* freqs, float* scores) {
  if (!s || !docs || !freqs || !scores) return SDBG_EINVAL;
  sdbg_ctx* c = s->ctx;
  if (term + 1 >= s->term_blk_begin.size()) return fail(c, SDBG_EINVAL, "term id out of range");
  CU(c, cudaSetDevice(c->device));
  const uint32_t b0 = s->term_blk_begin[term], nblk = s->term_blk_begin[term + 1] - b0;
  const uint32_t n = s->term_docs[term];
  if (!n) return SDBG_OK;
  const size_t slots = size_t(nblk) * 128;
  int rc;
  if ((rc = ensure(c, c->scratch[9], slots * 12))) return rc;
  auto* d_docs = static_cast<uint32_t*>(c->scratch[9].p);
  auto* d_freqs = d_docs + slots;
  auto* d_scores = reinterpret_cast<float*>(d_freqs + slots);
  const unsigned grid = unsigned(std::min<uint32_t>((nblk + kTopkWarps - 1) / kTopkWarps, uint32_t(c->sm_count) * 8u));
  decode_score_kernel<<<grid, kTopkThreads, 0, c->stream>>>(postings_view(s, 0), b0, nblk, c0, nc, nl, d_docs, d_freqs, d_scores);
  ++c->launches;
  CU(c, cudaGetLastError());
  CU(c, cudaMemcpyAsync(docs, d_docs, size_t(n) * 4, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaMemcpyAsync(freqs, d_freqs, size_t(n) * 4, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaMemcpyAsync(scores, d_scores, size_t(n) * 4, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  return SDBG_OK;
}

// ------------------------------------------------------------------------------------------
// columnar
// ------------------------------------------------------------------------------------------
namespace {

int pred_set(sdbg_segment* s, const sdbg_col_pred* preds, size_t n, PredSet* ps, uint64_t* rows, bool packed_ok = false) {
  if (n > size_t(kMaxPreds)) return fail(s->ctx, SDBG_EUNSUPPORTED, "more than 4 pushed predicates");
  std::memset(ps, 0, sizeof *ps);
  ps->n = int(n);
  for (size_t i = 0; i < n; ++i) {
    uint64_t r = 0;
    if (int rc = pred_dev(s, preds[i], &ps->p[i], &r, packed_ok)) return rc;
    if (*rows == 0) *rows = r;
    if (r != *rows) return fail(s->ctx, SDBG_EINVAL, "columns of one segment differ in length");
  }
  return SDBG_OK;
}

int column_minmax(sdbg_segment* s, uint64_t field, int64_t* mn, int64_t* mx) {
  sdbg_ctx* c = s->ctx;
  auto it = s->cols.find(field);
  if (it == s->cols.end()) return fail(c, SDBG_ENOTFOUND, "column not staged");
  ColumnObj& col = it->second;
  if (col.type == SDBG_F64) return fail(c, SDBG_EINVAL, "min/max statistics are kept for integer columns");
  if (!col.has_minmax) {
    int rc;
    if ((rc = ensure(c, c->scratch[10], 16))) return rc;
    const long long init[2] = {INT64_MAX, INT64_MIN};
    CU(c, cudaMemcpyAsync(c->scratch[10].p, init, 16, cudaMemcpyHostToDevice, c->stream));
    // a packed column's min / max are those of its zonemap entries (filled at staging): no raw view needed
    ColDev cd; cd.validity = col.d_validity; cd.type = col.type; cd.pad = 0;
    uint64_t n = col.rows;
    if (col.d_packed) { cd.values = col.d_zone; n = 2 * for_groups(col.rows); }
    else cd.values = col.d_values;
    minmax_i64_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(cd, n, static_cast<long long*>(c->scratch[10].p));
    ++c->launches;
    CU(c, cudaGetLastError());
    long long res[2];
    CU(c, cudaMemcpyAsync(res, c->scratch[10].p, 16, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    col.mn = res[0]; col.mx = res[1]; col.has_minmax = true;
  }
  *mn = col.mn; *mx = col.mx;
  return SDBG_OK;
}

}  // namespace

extern "C" int sdbg_column_minmax_i64(sdbg_segment* s, uint64_t field, int64_t* mn, int64_t* mx) {
  if (!s || !mn || !mx) return SDBG_EINVAL;
  CU(s->ctx, cudaSetDevice(s->ctx->device));
  return column_minmax(s, field, mn, mx);
}

extern "C" int sdbg_filter_bitmap(sdbg_segment* s, const sdbg_col_pred* preds, size_t n_preds, uint64_t* mask_out) {
  if (!s || !mask_out || (!preds && n_preds)) return SDBG_EINVAL;
  sdbg_ctx* c = s->ctx;
  CU(c, cudaSetDevice(c->device));
  PredSet ps; uint64_t rows = 0;
  int rc = pred_set(s, preds, n_preds, &ps, &rows);
  if (rc) return rc;
  if (!rows) rows = s->n_docs;
  if (rows > s->n_docs) return fail(c, SDBG_EINVAL, "filter column longer than the segment: mask_out holds (docs_count + 63) / 64 words");
  const size_t words = (rows + 63) / 64;
  if ((rc = ensure(c, c->scratch[9], words * 8))) return rc;
  const unsigned grid = unsigned(std::min<size_t>((words * 32 + 255) / 256, size_t(c->sm_count) * 8));
  filter_bitmap_kernel<<<std::max(grid, 1u), 256, 0, c->stream>>>(ps, rows, static_cast<unsigned long long*>(c->scratch[9].p));
  ++c->launches;
  CU(c, cudaGetLastError());
  CU(c, cudaMemcpyAsync(mask_out, c->scratch[9].p, words * 8, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  return SDBG_OK;
}

extern "C" int sdbg_filter_count_sum(sdbg_segment* const* segs, size_t n_segs, const sdbg_col_pred* preds, size_t n_preds,
                                     uint64_t sum_field, uint64_t* count, int64_t sum_i128[2], double* sum_f64) {
  if (!segs || !n_segs || !count || (!preds && n_preds)) return SDBG_EINVAL;
  sdbg_ctx* c = segs[0]->ctx;
  CU(c, cudaSetDevice(c->device));
  const unsigned grid = unsigned(c->sm_count) * 4u;
  int rc;
  if ((rc = ensure(c, c->scratch[9], (size_t(grid) + 1) * sizeof(CountSumOut) * n_segs + 64))) return rc;
  // Point-query latency: ONE launch per segment and one stream synchronisation. The completion counter is zeroed once
  // (the kernel leaves it at zero), and the final partial is written by the kernel straight into mapped pinned memory.
  if (!c->counter_zeroed || c->scratch[15].cap < 16) {
    if ((rc = ensure(c, c->scratch[15], 16))) return rc;
    CU(c, cudaMemsetAsync(c->scratch[15].p, 0, 16, c->stream));
    c->counter_zeroed = true;
  }
  const size_t seq_off = (n_segs * sizeof(CountSumOut) + 63) & ~size_t(63);   // [results | completion words]
  if (c->h_result_cap < seq_off + n_segs * 8) {
    if (c->h_result) { cudaStreamSynchronize(c->stream); cudaFreeHost(c->h_result); c->h_result = nullptr; }
    const size_t want = std::max<size_t>(seq_off + n_segs * 8, 4096);
    CU(c, cudaHostAlloc(&c->h_result, want, cudaHostAllocMapped));
    CU(c, cudaHostGetDevicePointer(&c->d_result, c->h_result, 0));
    std::memset(c->h_result, 0, want);
    c->h_result_cap = want;
  }
  const unsigned long long seq = ++c->result_seq;
  auto* h_seq = reinterpret_cast<volatile unsigned long long*>(static_cast<char*>(c->h_result) + seq_off);
  auto* d_seq = reinterpret_cast<unsigned long long*>(static_cast<char*>(c->d_result) + seq_off);
  for (size_t si = 0; si < n_segs; ++si) {
    sdbg_segment* s = segs[si];
    PredSet ps; uint64_t rows = 0;
    if ((rc = pred_set(s, preds, n_preds, &ps, &rows))) return rc;
    ColDev sc{}; int has_sum = 0;
    if (sum_field != UINT64_MAX) {
      uint64_t r = 0;
      if ((rc = col_view(s, sum_field, &sc, &r))) return rc;
      if (!rows) rows = r;
      if (r != rows) return fail(c, SDBG_EINVAL, "columns of one segment differ in length");
      has_sum = 1;
    }
    if (!rows) rows = s->n_docs;
    auto* part = static_cast<CountSumOut*>(c->scratch[9].p) + si * (size_t(grid) + 1);
    const unsigned g2 = unsigned(std::max<uint64_t>(1, std::min<uint64_t>(grid, (rows + 2047) / 2048)));   // 8 rows per thread at least
    { ProfScope ps_(c, kProfCountSum);
      filter_count_sum_kernel<<<g2, 256, 0, c->stream>>>(ps, sc, has_sum, rows, part, static_cast<unsigned int*>(c->scratch[15].p),
                                                         static_cast<CountSumOut*>(c->d_result) + si, d_seq + si, seq); }
    ++c->launches;
    CU(c, cudaGetLastError());
  }
  // Wait on the completion words the kernels write into mapped host memory after their result (a PCIe write, ~1 us
  // after the last block finishes) instead of synchronising the stream; the stream is only queried now and then so
  // that a failed launch cannot spin forever.
  for (size_t si = 0; si < n_segs; ++si) {
    uint32_t spins = 0;
    while (__atomic_load_n(const_cast<const unsigned long long*>(&h_seq[si]), __ATOMIC_ACQUIRE) != seq) {
      if ((++spins & 0x3FFFu) == 0u) {
        const cudaError_t q = cudaStreamQuery(c->stream);
        if (q != cudaErrorNotReady && q != cudaSuccess) { CU(c, q); }
        if (q == cudaSuccess && __atomic_load_n(const_cast<const unsigned long long*>(&h_seq[si]), __ATOMIC_ACQUIRE) != seq) {
          CU(c, cudaStreamSynchronize(c->stream));   // finished without the word (cannot happen unless the write was lost)
          break;
        }
      }
#if defined(__x86_64__)
      __builtin_ia32_pause();
#endif
    }
  }
  unsigned __int128 tot = 0; uint64_t cnt = 0; double sf = 0;
  for (size_t si = 0; si < n_segs; ++si) {
    const CountSumOut& o = static_cast<const CountSumOut*>(c->h_result)[si];
    cnt += o.count; sf += o.sum_f;
    tot += (static_cast<unsigned __int128>(static_cast<uint64_t>(o.sum_hi)) << 64) | o.sum_lo;
  }
  *count = cnt;
  if (sum_i128) { sum_i128[0] = int64_t(uint64_t(tot)); sum_i128[1] = int64_t(uint64_t(tot >> 64)); }
  if (sum_f64) *sum_f64 = sf;
  return SDBG_OK;
}

namespace {

struct GroupPlan { int wide_int = 0; int count_f = 0; int pack_shift = 0; int pack_tables = 0; int64_t pack_bias = 0; };

int groupby_launch(sdbg_segment* const* segs, size_t n_segs, const sdbg_col_pred* preds, size_t n_preds, uint64_t key_field,
                   int64_t key_min, uint64_t span, uint64_t sum_int_field, uint64_t avg_f64_field, void* d_i64, void* d_f64,
                   bool defer_check = false) {
  sdbg_ctx* c = segs[0]->ctx;
  int rc;
  // table | cnt_f | out_of_range
  const size_t table_bytes = span * sizeof(GroupSlot);
  if ((rc = ensure(c, c->scratch[11], table_bytes + span * 8 + 64))) return rc;
  auto* table = static_cast<GroupSlot*>(c->scratch[11].p);
  auto* cnt_f = reinterpret_cast<unsigned long long*>(static_cast<char*>(c->scratch[11].p) + table_bytes);
  auto* oor = cnt_f + span;
  CU(c, cudaMemsetAsync(c->scratch[11].p, 0, table_bytes + span * 8 + 64, c->stream));
  GroupPlan plan;
  uint64_t total_rows = 0;
  int64_t sum_mn = INT64_MAX, sum_mx = INT64_MIN;
  bool all_tma = env_int("SDBG_GROUPBY_TMA", 1) != 0;
  for (size_t si = 0; si < n_segs; ++si) {  // statistics decide the accumulator shape
    sdbg_segment* s = segs[si];
    if (sum_int_field != UINT64_MAX) {
      int64_t mn, mx;
      if ((rc = column_minmax(s, sum_int_field, &mn, &mx))) return rc;
      if (mn < INT32_MIN || mx > INT32_MAX) plan.wide_int = 1;
      sum_mn = std::min(sum_mn, mn); sum_mx = std::max(sum_mx, mx);
      auto sit = s->cols.find(sum_int_field);
      if (sit != s->cols.end() && sit->second.d_validity) all_tma = false;
    }
    for (size_t i = 0; i < n_preds; ++i) {
      auto pit = s->cols.find(preds[i].field);
      if (preds[i].op >= 7 || (pit != s->cols.end() && pit->second.d_validity)) all_tma = false;
    }
    if (avg_f64_field != UINT64_MAX) {
      auto it = s->cols.find(avg_f64_field);
      if (it == s->cols.end()) return fail(c, SDBG_ENOTFOUND, "avg column not staged");
      if (it->second.d_validity) { plan.count_f = 1; all_tma = false; }
    }
    auto kit = s->cols.find(key_field);
    if (kit == s->cols.end()) return fail(c, SDBG_ENOTFOUND, "key column not staged");
    if (kit->second.d_validity) return fail(c, SDBG_EUNSUPPORTED, "nullable GROUP BY key");
    if (kit->second.type == SDBG_F64) return fail(c, SDBG_EUNSUPPORTED, "float GROUP BY key");
    total_rows += kit->second.rows;
  }
  if (total_rows >= (1ull << 31)) return fail(c, SDBG_EUNSUPPORTED, ">= 2^31 rows per GPU in one GROUP BY (limb overflow guard)");
  // Packed accumulators: one RED carries COUNT and SUM(int) when the column statistics prove that
  // count << shift | sum(v - min) cannot overflow either field (the RED issue rate, not HBM, is what the
  // consumer warps run into). Rows are dealt to 1..3 words of the slot by tile index.
  if (sum_int_field != UINT64_MAX && !plan.wide_int && all_tma && total_rows && sum_mx >= sum_mn && env_int("SDBG_GROUPBY_PACKED", 1)) {
    const unsigned __int128 range = static_cast<unsigned __int128>(static_cast<uint64_t>(sum_mx) - static_cast<uint64_t>(sum_mn));
    const int max_tables = avg_f64_field != UINT64_MAX ? 2 : 3;   // with a SUM(double) at most two words: a third is free, but that plan has not been measured
    for (int nt = std::max(1, env_int("SDBG_GROUPBY_PACK_TABLES_MIN", 1)); nt <= max_tables && !plan.pack_tables; ++nt) {   // env: test hook
      uint64_t cap_rows = 0;   // most rows any one word can receive: its share of every segment's tiles
      for (size_t si = 0; si < n_segs; ++si) {
        const uint64_t tiles = (segs[si]->cols.find(key_field)->second.rows + kGroupByTileRows - 1) / kGroupByTileRows;
        cap_rows += (tiles + nt - 1) / nt * kGroupByTileRows;
      }
      const unsigned __int128 max_sum = range * cap_rows;
      int shift = 1;
      while (shift < 63 && (static_cast<unsigned __int128>(1) << shift) <= max_sum) ++shift;
      if (shift < 63 && cap_rows < (1ull << (64 - shift))) { plan.pack_tables = nt; plan.pack_shift = shift; plan.pack_bias = sum_mn; }
    }
  }
  for (size_t si = 0; si < n_segs; ++si) {
    sdbg_segment* s = segs[si];
    // Packed columns are read packed by the TMA kernel, which takes segments without nullable columns; every other
    // path reads their raw view.
    auto nullable = [&](uint64_t f) { auto it = s->cols.find(f); return it != s->cols.end() && it->second.d_validity != nullptr; };
    bool packed_ok = env_int("SDBG_GROUPBY_TMA", 1) != 0 && !nullable(key_field) &&
                     (sum_int_field == UINT64_MAX || !nullable(sum_int_field)) && (avg_f64_field == UINT64_MAX || !nullable(avg_f64_field));
    for (size_t i = 0; i < n_preds; ++i) packed_ok = packed_ok && preds[i].op < 7 && !nullable(preds[i].field);
    GroupByParams P;
    std::memset(&P, 0, sizeof P);
    uint64_t rows = 0;
    if ((rc = pred_set(s, preds, n_preds, &P.ps, &rows, packed_ok))) return rc;
    uint64_t r = 0;
    if ((rc = col_view(s, key_field, &P.key, &r, packed_ok))) return rc;
    if (!rows) rows = r;
    if (r != rows) return fail(c, SDBG_EINVAL, "key column length differs");
    if (sum_int_field != UINT64_MAX) {
      if ((rc = col_view(s, sum_int_field, &P.sum_i, &r, packed_ok))) return rc;
      if (r != rows) return fail(c, SDBG_EINVAL, "sum_int column length differs");
      if (P.sum_i.type == SDBG_F64) return fail(c, SDBG_EINVAL, "sum_int_field is a float column");
      P.has_sum_i = 1;
    }
    if (avg_f64_field != UINT64_MAX) {
      if ((rc = col_view(s, avg_f64_field, &P.sum_f, &r))) return rc;
      if (r != rows) return fail(c, SDBG_EINVAL, "avg_f64 column length differs");
      if (P.sum_f.type != SDBG_F64) return fail(c, SDBG_EINVAL, "avg_f64_field is not a float column");
      P.has_sum_f = 1;
    }
    P.wide_int = plan.wide_int; P.count_f = plan.count_f;
    P.key_min = key_min; P.key_span = span; P.rows = rows;
    P.table = table; P.cnt_f = cnt_f; P.out_of_range = oor;
    // NOT NULL columns (the common analytic case) go through the TMA-pipelined kernel; nullable
    // columns need their validity words next to the values and keep the register-staged kernel.
    bool any_nullable = P.key.validity || (P.has_sum_i && P.sum_i.validity) || (P.has_sum_f && P.sum_f.validity);
    for (int i = 0; i < P.ps.n; ++i) any_nullable |= P.ps.p[i].col.validity != nullptr || P.ps.p[i].op >= 7;
    if (plan.pack_tables && any_nullable) return fail(c, SDBG_EINVAL, "internal: packed accumulators planned for a nullable segment");
    if (!any_nullable && env_int("SDBG_GROUPBY_TMA", 1)) {
      TmaGroupByParams T;
      std::memset(&T, 0, sizeof T);
      // the column a stream comes from: its raw values or, for kTypeFor, its packed block
      auto column_of = [&](const void* id) -> ColumnObj* {
        for (auto& kv : s->cols) if (kv.second.d_values == id || (id && kv.second.d_packed == id)) return &kv.second;
        return nullptr;
      };
      const void* stream_id[kMaxStreams] = {};
      auto stream_of = [&](const ColDev& col) {
        for (int i = 0; i < T.n_streams; ++i) if (stream_id[i] == col.values) return i;
        const int n = T.n_streams++;
        stream_id[n] = col.values;
        T.elem[n] = col.type == SDBG_I32 ? 4 : 8;
        if (col.type == kTypeFor) {
          T.hdr[n] = static_cast<const ForBlockDev*>(col.values);
          T.src[n] = static_cast<const char*>(col.values) + for_hdr_bytes(rows);
        } else {
          T.src[n] = col.values;
        }
        return n;
      };
      // Every comparison becomes a closed range of the zonemaps' key space (key_range). Predicates that hold for every
      // row are dropped; one that holds for none makes the segment contribute nothing.
      bool never = false;
      int stream_idx[kMaxPreds];
      T.n_preds = 0;
      for (int i = 0; i < P.ps.n; ++i) {
        const PredDev& pd = P.ps.p[i];
        int64_t lo = 0; uint64_t span = 0; int neg = 0;
        const KeyRange kr = key_range(pd, &lo, &span, &neg);
        if (kr == kKeyAll) continue;
        if (kr == kKeyNone) { never = true; break; }
        const int k = T.n_preds++;
        stream_idx[k] = stream_of(pd.col);
        T.pred_type[k] = pd.col.type; T.pred_negate[k] = neg;
        T.pred_lo[k] = lo; T.pred_span[k] = span;
      }
      if (never) continue;   // WHERE is false for every row of this segment
      // Zonemap verdicts: blocks whose min / max miss a predicate's range are skipped by producer and consumers alike.
      T.skip = nullptr;
      if (T.n_preds && env_int("SDBG_ZONEMAP", 1) != 0) {
        ZoneVerdictParams Z;
        std::memset(&Z, 0, sizeof Z);
        Z.n_preds = T.n_preds;
        Z.n_blocks = (rows + kZoneRows - 1) / kZoneRows;
        bool any_zone = false;
        for (int k2 = 0; k2 < T.n_preds; ++k2) {
          Z.lo[k2] = T.pred_lo[k2]; Z.span[k2] = T.pred_span[k2]; Z.negate[k2] = T.pred_negate[k2];
          ColumnObj* co = column_of(stream_id[stream_idx[k2]]);
          if (!co || co->d_validity) continue;
          if ((rc = column_zonemap(c, *co, &Z.zone[k2]))) return rc;
          any_zone = true;
        }
        if (any_zone) {
          DevBuf& b_skip = c->scratch[13];
          if ((rc = ensure(c, b_skip, Z.n_blocks + 16))) return rc;
          if (!c->d_zone_skipped) CU(c, cudaMalloc(reinterpret_cast<void**>(&c->d_zone_skipped), 8));
          if (si == 0) { CU(c, cudaMemsetAsync(c->d_zone_skipped, 0, 8, c->stream)); c->zone_blocks_total = 0; }
          const unsigned vg = unsigned(std::min<uint64_t>((Z.n_blocks + 255) / 256, uint64_t(c->sm_count) * 4));
          zone_verdict_kernel<<<vg, 256, 0, c->stream>>>(Z, static_cast<uint8_t*>(b_skip.p), c->d_zone_skipped);
          ++c->launches;
          c->zone_blocks_total += Z.n_blocks;
          T.skip = static_cast<const uint8_t*>(b_skip.p);
        }
      }
      const int key_s = stream_of(P.key);
      const int sum_i_s = P.has_sum_i ? stream_of(P.sum_i) : -1;
      const int sum_f_s = P.has_sum_f ? stream_of(P.sum_f) : -1;
      T.key_type = P.key.type; T.sum_i_type = P.has_sum_i ? P.sum_i.type : 0;
      T.has_sum_i = P.has_sum_i; T.has_sum_f = P.has_sum_f;
      T.debug_skip = env_int("SDBG_GROUPBY_DEBUG", 0);
      T.wide_int = plan.wide_int; T.key_min = key_min; T.key_span = span; T.rows = rows; T.table = table; T.out_of_range = oor;
      T.pack_shift = plan.pack_shift; T.pack_tables = plan.pack_tables; T.pack_bias = plan.pack_bias;
      for (int i = 0; i < T.n_preds; ++i) T.pred_stream[i] = stream_idx[i];
      T.key_stream = key_s; T.sum_i_stream = sum_i_s >= 0 ? sum_i_s : 0;
      bool any_for = false;
      for (int i = 0; i < T.n_streams; ++i) any_for |= T.hdr[i] != nullptr;
      // A packed stream keeps its raw slot size, so the shared-memory footprint and CTAs per SM are those of the raw scan.
      uint32_t o = 0;
      for (int i = 0; i < T.n_streams; ++i) { T.off[i] = o; o += uint32_t(T.elem[i]) * uint32_t(kGroupByTileRows); }
      T.off[T.n_streams] = o;
      for (int i = 0; i < T.n_preds; ++i) T.pred_off[i] = T.off[stream_idx[i]];
      T.key_off = T.off[key_s];
      T.sum_i_off = sum_i_s >= 0 ? T.off[sum_i_s] : 0;
      T.sum_f_off = sum_f_s >= 0 ? T.off[sum_f_s] : 0;
      constexpr int threads = (kGroupByConsumerWarps + 1) * 32;
      const size_t smem = size_t(kGroupByStages) * size_t(T.off[T.n_streams]) + (any_for ? size_t(kGroupByStages) * kMaxStreams * 16 : 0);
      auto launch = [&](auto kern) -> int {
        CU(c, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
        const size_t fit = std::max<size_t>(1, (220 * 1024) / (smem + 2048));
        int resident = 0;   // persistent CTAs: never more per SM than can be resident at once (registers included)
        CU(c, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, kern, threads, smem));
        const unsigned per_sm = unsigned(std::max<size_t>(1, std::min<size_t>({fit, size_t(2048 / threads), size_t(resident)})));
        ProfScope ps_(c, kProfGroupBy);
        kern<<<unsigned(c->sm_count) * per_sm, threads, smem, c->stream>>>(T);
        return SDBG_OK;
      };
      const int lrc = plan.pack_tables ? (any_for ? launch(filter_groupby_tma_kernel<true, true>) : launch(filter_groupby_tma_kernel<true, false>))
                                       : (any_for ? launch(filter_groupby_tma_kernel<false, true>) : launch(filter_groupby_tma_kernel<false, false>));
      if (lrc) return lrc;
    } else {
      const unsigned grid = unsigned(c->sm_count) * 8u;
      ProfScope ps_(c, kProfGroupBy);
      filter_groupby_kernel<2><<<grid, 256, 0, c->stream>>>(P);
    }
    ++c->launches;
    CU(c, cudaGetLastError());
  }
  groupby_pack_kernel<<<c->sm_count * 2, 256, 0, c->stream>>>(table, plan.count_f ? cnt_f : nullptr, span,
                                                               static_cast<long long*>(d_i64), static_cast<double*>(d_f64),
                                                               plan.pack_shift, plan.pack_tables, plan.pack_bias);
  ++c->launches;
  CU(c, cudaGetLastError());
  if (defer_check) {
    // the partial path stays asynchronous (a collective usually follows on the same stream): the out-of-range count
    // lands in pinned memory and is looked at by the next call that synchronises (finalize / sdbg_sync)
    if (!c->h_oor) CU(c, cudaHostAlloc(reinterpret_cast<void**>(&c->h_oor), 16, cudaHostAllocDefault));
    CU(c, cudaMemcpyAsync(c->h_oor, oor, 8, cudaMemcpyDeviceToHost, c->stream));
    c->oor_pending = true;
  } else {
    unsigned long long h_oor = 0;
    CU(c, cudaMemcpyAsync(&h_oor, oor, 8, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    if (h_oor) return fail(c, SDBG_EINVAL, "GROUP BY key outside [key_min, key_min + span)");
  }
  return SDBG_OK;
}

}  // namespace

namespace {

int groupby_hash(sdbg_segment* const* segs, size_t n_segs, const sdbg_col_pred* preds, size_t n_preds, uint64_t key_field,
                 uint32_t n_groups_hint, uint64_t sum_int_field, uint64_t avg_f64_field, sdbg_group_row* out, uint64_t cap,
                 uint64_t* n_out) {
  sdbg_ctx* c = segs[0]->ctx;
  // the SUM(int) lo limb adds up to 2^32 - 1 per row as a signed 64-bit value: the dense path's row limit holds here too
  uint64_t total_rows = 0;
  for (size_t si = 0; si < n_segs; ++si) {
    auto it = segs[si]->cols.find(key_field);
    if (it != segs[si]->cols.end()) total_rows += it->second.rows;
  }
  if (total_rows >= (1ull << 31)) return fail(c, SDBG_EUNSUPPORTED, ">= 2^31 rows per GPU in one GROUP BY (limb overflow guard)");
  uint64_t capacity = 1 << 16;
  while (capacity < 2ull * std::max<uint64_t>(n_groups_hint, cap)) capacity <<= 1;
  int rc;
  for (int attempt = 0; attempt < 8; ++attempt, capacity <<= 2) {
    const size_t bytes = (capacity + 1) * sizeof(HashSlot);
    if (bytes > (size_t(8) << 30)) return fail(c, SDBG_ECAPACITY, "hash aggregate table would exceed 8 GiB");
    if ((rc = ensure(c, c->scratch[11], bytes + 64))) return rc;
    auto* table = static_cast<HashSlot*>(c->scratch[11].p);
    auto* overflow = reinterpret_cast<unsigned int*>(static_cast<char*>(c->scratch[11].p) + bytes);
    hash_init_kernel<<<c->sm_count * 4, 256, 0, c->stream>>>(table, capacity + 1);
    ++c->launches;
    CU(c, cudaMemsetAsync(overflow, 0, 64, c->stream));
    for (size_t si = 0; si < n_segs; ++si) {
      sdbg_segment* s = segs[si];
      HashGroupByParams P;
      std::memset(&P, 0, sizeof P);
      uint64_t rows = 0, r = 0;
      if ((rc = pred_set(s, preds, n_preds, &P.ps, &rows))) return rc;
      if ((rc = col_view(s, key_field, &P.key, &r))) return rc;
      if (P.key.validity) return fail(c, SDBG_EUNSUPPORTED, "nullable GROUP BY key");
      if (P.key.type == SDBG_F64) return fail(c, SDBG_EUNSUPPORTED, "float GROUP BY key");
      if (!rows) rows = r;
      if (r != rows) return fail(c, SDBG_EINVAL, "key column length differs");
      if (sum_int_field != UINT64_MAX) {
        if ((rc = col_view(s, sum_int_field, &P.sum_i, &r))) return rc;
        if (r != rows) return fail(c, SDBG_EINVAL, "sum_int column length differs");
        if (P.sum_i.type == SDBG_F64) return fail(c, SDBG_EINVAL, "sum_int_field is a float column");
        P.has_sum_i = 1;
      }
      if (avg_f64_field != UINT64_MAX) {
        if ((rc = col_view(s, avg_f64_field, &P.sum_f, &r))) return rc;
        if (r != rows) return fail(c, SDBG_EINVAL, "avg_f64 column length differs");
        if (P.sum_f.type != SDBG_F64) return fail(c, SDBG_EINVAL, "avg_f64_field is not a float column");
        P.has_sum_f = 1;
      }
      P.rows = rows; P.table = table; P.capacity = capacity; P.overflow = overflow;
      { ProfScope ps_(c, kProfGroupBy);
        filter_groupby_hash_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(P); }
      ++c->launches;
      CU(c, cudaGetLastError());
    }
    unsigned int h_over = 0;
    CU(c, cudaMemcpyAsync(&h_over, overflow, 4, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    if (h_over) continue;  // table filled up: retry with 4x the capacity
    std::vector<HashSlot> h(capacity + 1);
    CU(c, cudaMemcpyAsync(h.data(), table, bytes, cudaMemcpyDeviceToHost, c->stream));
    CU(c, cudaStreamSynchronize(c->stream));
    std::vector<const HashSlot*> live;
    for (const HashSlot& sl : h) if (sl.count) live.push_back(&sl);
    std::sort(live.begin(), live.end(), [](const HashSlot* a, const HashSlot* b) { return a->key < b->key; });
    *n_out = live.size();
    if (live.size() > cap) return fail(c, SDBG_ECAPACITY, "group output buffer too small");
    for (size_t i = 0; i < live.size(); ++i) {
      const HashSlot& sl = *live[i];
      sdbg_group_row& g = out[i];
      g.key = sl.key; g.count = sl.count;
      const __int128 tot = (static_cast<__int128>(sl.sum_hi) << 32) + static_cast<__int128>(sl.sum_lo);
      g.sum_i128[0] = int64_t(uint64_t(static_cast<unsigned __int128>(tot)));
      g.sum_i128[1] = int64_t(uint64_t(static_cast<unsigned __int128>(tot) >> 64));
      g.sum_f64 = sl.sum_f;
      g.cnt_f64 = avg_f64_field != UINT64_MAX ? sl.cnt_f : sl.count;
    }
    return SDBG_OK;
  }
  return fail(c, SDBG_ECAPACITY, "hash aggregate: too many groups");
}

}  // namespace

extern "C" int sdbg_filter_groupby_partial(sdbg_segment* const* segs, size_t n_segs, const sdbg_col_pred* preds, size_t n_preds,
                                           uint64_t key_field, int64_t key_min, uint64_t key_span, uint64_t sum_int_field,
                                           uint64_t avg_f64_field, void* d_i64, void* d_f64) {
  if (!segs || !n_segs || !d_i64 || !d_f64 || !key_span || (!preds && n_preds)) return SDBG_EINVAL;
  CU(segs[0]->ctx, cudaSetDevice(segs[0]->ctx->device));
  // asynchronous: nothing here waits for the GPU (SUM(int) leaves as two limbs, total = hi * 2^32 + lo; a narrow sum
  // keeps the whole value in lo -- sdbg_dist_groupby_merge normalises the limbs before they are all-reduced)
  return groupby_launch(segs, n_segs, preds, n_preds, key_field, key_min, key_span, sum_int_field, avg_f64_field, d_i64, d_f64, true);
}

extern "C" int sdbg_groupby_finalize(sdbg_ctx* c, int64_t key_min, uint64_t span, const void* d_i64, const void* d_f64,
                                     sdbg_group_row* out, uint64_t cap, uint64_t* n_out) {
  if (!c || !d_i64 || !d_f64 || !out || !n_out || !span) return SDBG_EINVAL;
  CU(c, cudaSetDevice(c->device));
  // The dense partials are exactly as large as the answer (40 B per key), so they cross PCIe once
  // into pinned memory and the ascending-key compaction of non-empty groups is a host loop -- one
  // stream synchronisation per call instead of a compaction kernel plus three.
  int rc;
  if ((rc = ensure_pinned(c, span * 40))) return rc;
  auto* h_i = static_cast<long long*>(c->h_pinned);
  auto* h_f = reinterpret_cast<double*>(h_i + 4 * span);
  CU(c, cudaMemcpyAsync(h_i, d_i64, span * 32, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaMemcpyAsync(h_f, d_f64, span * 8, cudaMemcpyDeviceToHost, c->stream));
  CU(c, cudaStreamSynchronize(c->stream));
  if ((rc = deferred_groupby_errors(c))) return rc;
  uint64_t n = 0;
  for (uint64_t i = 0; i < span; ++i) {
    if (h_i[i] == 0) continue;
    if (n < cap) {
      sdbg_group_row& r = out[n];
      r.key = key_min + int64_t(i);
      r.count = uint64_t(h_i[i]);
      // SUM(int) limbs: total = hi * 2^32 + lo (a narrow sum has hi == 0); exact in 128 bits.
      const __int128 tot = (static_cast<__int128>(h_i[2 * span + i]) << 32) + static_cast<__int128>(h_i[span + i]);
      r.sum_i128[0] = int64_t(uint64_t(static_cast<unsigned __int128>(tot)));
      r.sum_i128[1] = int64_t(uint64_t(static_cast<unsigned __int128>(tot) >> 64));
      r.sum_f64 = h_f[i];
      r.cnt_f64 = uint64_t(h_i[3 * span + i]);
    }
    ++n;
  }
  *n_out = n;
  if (n > cap) return fail(c, SDBG_ECAPACITY, "group output buffer too small");
  return SDBG_OK;
}

extern "C" int sdbg_filter_groupby(sdbg_segment* const* segs, size_t n_segs, const sdbg_col_pred* preds, size_t n_preds,
                                   uint64_t key_field, uint32_t n_groups_hint, uint64_t sum_int_field, uint64_t avg_f64_field,
                                   sdbg_group_row* out, uint64_t cap, uint64_t* n_out) {
  if (!segs || !n_segs || !out || !n_out || (!preds && n_preds)) return SDBG_EINVAL;
  sdbg_ctx* c = segs[0]->ctx;
  CU(c, cudaSetDevice(c->device));
  int64_t kmin = INT64_MAX, kmax = INT64_MIN;
  for (size_t si = 0; si < n_segs; ++si) {
    int64_t mn, mx;
    const int rc = column_minmax(segs[si], key_field, &mn, &mx);
    if (rc) return rc;
    kmin = std::min(kmin, mn); kmax = std::max(kmax, mx);
  }
  if (kmin > kmax) { *n_out = 0; return SDBG_OK; }
  const unsigned __int128 span128 = static_cast<unsigned __int128>(static_cast<__int128>(kmax) - kmin) + 1;
  // Dense ("perfect hash") table when statistics bound the key range to something table-sized,
  // otherwise a real hash table sized from the group-count hint.
  const unsigned __int128 dense_limit = std::max<unsigned __int128>(static_cast<unsigned __int128>(1) << 20,
                                                                    static_cast<unsigned __int128>(n_groups_hint) * 8);
  if (span128 > (static_cast<unsigned __int128>(1) << 26) || span128 > dense_limit || env_int("SDBG_GROUPBY_FORCE_HASH", 0))
    return groupby_hash(segs, n_segs, preds, n_preds, key_field, n_groups_hint, sum_int_field, avg_f64_field, out, cap, n_out);
  const uint64_t span = uint64_t(span128);
  int rc;
  if ((rc = ensure(c, c->scratch[8], span * 40 + 64))) return rc;
  void* d_i64 = c->scratch[8].p;
  void* d_f64 = static_cast<char*>(c->scratch[8].p) + span * 32;
  if ((rc = groupby_launch(segs, n_segs, preds, n_preds, key_field, kmin, span, sum_int_field, avg_f64_field, d_i64, d_f64))) return rc;
  return sdbg_groupby_finalize(c, kmin, span, d_i64, d_f64, out, cap, n_out);
}

// ------------------------------------------------------------------------------------------
// Collectives over NVLink for a C++ host (no torch): NCCL resolved lazily with dlopen, so libsdbg.so itself does not
// link it and a process that already carries an NCCL (e.g. PyTorch's bundled one: same SONAME) shares that copy.
// Everything below is enqueued on the context's stream: a partial aggregate or a top-k batch flows kernel ->
// collective -> kernel without a host synchronisation in between.
// ------------------------------------------------------------------------------------------
namespace {
struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok() const { return lib && GetUniqueId && CommInitRank && CommDestroy && AllReduce && AllGather && GetErrorString; }
};
NcclApi& nccl_api() {
  static NcclApi api = [] {
    NcclApi a;
    for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
      a.lib = dlopen(name, RTLD_NOW | RTLD_LOCAL);
      if (a.lib) break;
    }
    if (a.lib) {
      a.GetUniqueId = reinterpret_cast<decltype(a.GetUniqueId)>(dlsym(a.lib, "ncclGetUniqueId"));
      a.CommInitRank = reinterpret_cast<decltype(a.CommInitRank)>(dlsym(a.lib, "ncclCommInitRank"));
      a.CommDestroy = reinterpret_cast<decltype(a.CommDestroy)>(dlsym(a.lib, "ncclCommDestroy"));
      a.AllReduce = reinterpret_cast<decltype(a.AllReduce)>(dlsym(a.lib, "ncclAllReduce"));
      a.AllGather = reinterpret_cast<decltype(a.AllGather)>(dlsym(a.lib, "ncclAllGather"));
      a.GetErrorString = reinterpret_cast<decltype(a.GetErrorString)>(dlsym(a.lib, "ncclGetErrorString"));
    }
    return a;
  }();
  return api;
}
#define NC(c, call)                                                                          \
  do {                                                                                       \
    const ncclResult_t r_ = (call);                                                          \
    if (r_ != ncclSuccess) return fail((c), SDBG_ECUDA, std::string("NCCL: ") + nccl_api().GetErrorString(r_)); \
  } while (0)

// SUM(double) partials as fixed point: x / 2^eunit truncated to a 120-bit integer, two signed 60-bit limbs in int64 --
// sums of up to 8 ranks cannot overflow a limb, the integer all-reduce is exact and independent of the rank order,
// and the only roundings left are the truncation below 2^eunit and the final conversion back to double.
// A NaN or infinite partial has no fixed-point form: it adds one to its key's count of NaN, +inf or -inf partials
// (one 16-bit field each of one more word per key, summed by the same all-reduce) and the unpack rebuilds the IEEE sum
// from the counts. A finite partial beyond abs_bound adds one to the last word of the wire instead; the next
// synchronising call reports it.
constexpr long long kWireNan = 1ll, kWirePosInf = 1ll << 16, kWireNegInf = 1ll << 32;
__global__ void __launch_bounds__(256)
dist_pack_kernel(const long long* __restrict__ part_i64, const double* __restrict__ part_f64, uint64_t span, int eunit,
                 double abs_bound, long long* __restrict__ wire /* [7 * span + 1], the last word zeroed */) {
  for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < span; i += uint64_t(gridDim.x) * blockDim.x) {
    wire[i] = part_i64[i];
    // SUM(int) limbs normalised so that lo is in [0, 2^32): the all-reduce of up to 2^31 ranks' lo limbs cannot wrap
    const long long lo = part_i64[span + i], hi = part_i64[2 * span + i];
    const long long carry = lo >> 32;                         // arithmetic shift: floor(lo / 2^32)
    wire[span + i] = lo - (carry << 32);
    wire[2 * span + i] = hi + carry;
    wire[3 * span + i] = part_i64[3 * span + i];
    const double w = part_f64[i];
    long long l0 = 0, l1 = 0, special = 0;
    if (isnan(w)) special = kWireNan;
    else if (isinf(w)) special = w > 0.0 ? kWirePosInf : kWireNegInf;
    else if (fabs(w) <= abs_bound) fix_limbs(w, 60, eunit, l0, l1);
    else atomicAdd(reinterpret_cast<unsigned long long*>(wire + 7 * span), 1ull);
    wire[4 * span + i] = l0;
    wire[5 * span + i] = l1;
    wire[6 * span + i] = special;
  }
}
__global__ void __launch_bounds__(256)
dist_unpack_kernel(const long long* __restrict__ wire, uint64_t span, int eunit, long long* __restrict__ part_i64,
                   double* __restrict__ part_f64) {
  for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < span; i += uint64_t(gridDim.x) * blockDim.x) {
    part_i64[i] = wire[i];
    part_i64[span + i] = wire[span + i];
    part_i64[2 * span + i] = wire[2 * span + i];
    part_i64[3 * span + i] = wire[3 * span + i];
    // IEEE sum semantics: NaN if any partial is NaN or both infinities occur, else the infinity that occurs
    const long long special = wire[6 * span + i];
    const bool nan = (special & 0xFFFF) != 0, pinf = ((special >> 16) & 0xFFFF) != 0, ninf = ((special >> 32) & 0xFFFF) != 0;
    part_f64[i] = nan || (pinf && ninf) ? __longlong_as_double(0x7FF8000000000000ll)
                : pinf                  ? __longlong_as_double(0x7FF0000000000000ll)
                : ninf                  ? __longlong_as_double(static_cast<long long>(0xFFF0000000000000ull))
                                        : fix_total(wire[4 * span + i], wire[5 * span + i], 60, eunit);
  }
}
}  // namespace

extern "C" int sdbg_dist_unique_id(uint8_t* id128) {
  if (!id128) return SDBG_EINVAL;
  if (!nccl_api().ok()) return SDBG_EUNSUPPORTED;
  ncclUniqueId id;
  if (nccl_api().GetUniqueId(&id) != ncclSuccess) return SDBG_ECUDA;
  std::memcpy(id128, id.internal, NCCL_UNIQUE_ID_BYTES);
  return SDBG_OK;
}

extern "C" int sdbg_dist_init(sdbg_ctx* c, const uint8_t* id128, int rank, int world) {
  if (!c || !id128 || world < 1 || rank < 0 || rank >= world) return SDBG_EINVAL;
  if (!nccl_api().ok()) return fail(c, SDBG_EUNSUPPORTED, "libnccl.so.2 not found");
  if (c->nccl_comm) return fail(c, SDBG_EINVAL, "context already has a communicator");
  CU(c, cudaSetDevice(c->device));
  ncclUniqueId id;
  std::memcpy(id.internal, id128, NCCL_UNIQUE_ID_BYTES);
  ncclComm_t comm = nullptr;
  NC(c, nccl_api().CommInitRank(&comm, world, id, rank));
  c->nccl_comm = comm; c->dist_rank = rank; c->dist_world = world;
  return SDBG_OK;
}

extern "C" int sdbg_dist_destroy(sdbg_ctx* c) {
  if (!c) return SDBG_EINVAL;
  if (c->nccl_comm) { nccl_api().CommDestroy(static_cast<ncclComm_t>(c->nccl_comm)); c->nccl_comm = nullptr; }
  c->dist_rank = 0; c->dist_world = 1;
  return SDBG_OK;
}

extern "C" int sdbg_dist_allreduce_i64(sdbg_ctx* c, void* d_buf, size_t n) {
  if (!c || !d_buf) return SDBG_EINVAL;
  if (!c->nccl_comm) return c->dist_world == 1 ? SDBG_OK : fail(c, SDBG_EINVAL, "sdbg_dist_init has not run");
  NC(c, nccl_api().AllReduce(d_buf, d_buf, n, ncclInt64, ncclSum, static_cast<ncclComm_t>(c->nccl_comm), c->stream));
  return SDBG_OK;
}

extern "C" int sdbg_dist_allgather(sdbg_ctx* c, const void* d_send, void* d_recv, size_t bytes_per_rank) {
  if (!c || !d_send || !d_recv) return SDBG_EINVAL;
  if (!c->nccl_comm) {
    if (c->dist_world != 1) return fail(c, SDBG_EINVAL, "sdbg_dist_init has not run");
    CU(c, cudaMemcpyAsync(d_recv, d_send, bytes_per_rank, cudaMemcpyDeviceToDevice, c->stream));
    return SDBG_OK;
  }
  NC(c, nccl_api().AllGather(d_send, d_recv, bytes_per_rank, ncclInt8, static_cast<ncclComm_t>(c->nccl_comm), c->stream));
  return SDBG_OK;
}

// Dense GROUP BY partials of every rank -> the global partials on every rank, in ONE all-reduce: counts, the SUM(int)
// limbs and SUM(double) as fixed-point limbs travel in one int64 buffer. abs_bound >= every rank's |partial| fixes the
// fixed-point unit (identical on every rank: derive it from the column statistics and the total row count, which are
// known when the shards are built; the sum of |w| over all passing rows bounds every partial).
// Distributed top-k in one call: local scan of this rank's segments, ONE all-gather of every rank's k best keys per query
// over NVLink, local selection of the global top-k -- enqueued back to back on the context's stream, one host
// synchronisation at the very end (none when out == NULL: the keys stay in HBM, see sdbg_topk_merge_gathered).
extern "C" int sdbg_dist_bm25_topk_batch(sdbg_segment* const* segs, size_t n_segs, int kind, const sdbg_bm25_term* terms,
                                         const uint32_t* term_off, size_t nq, float k1, float b, const sdbg_col_pred* filt, uint32_t k,
                                         float threshold_in, sdbg_hit* out, uint32_t* n_out) {
  if (!segs || !n_segs) return SDBG_EINVAL;
  sdbg_ctx* c = segs[0]->ctx;
  const uint32_t world = uint32_t(c->dist_world), rank = uint32_t(c->dist_rank);
  if (world > 1 && !c->nccl_comm) return fail(c, SDBG_EINVAL, "sdbg_dist_init has not run");
  DevBuf& mine = c->pass[0];   // this rank's keys
  DevBuf& all = c->pass[1];    // every rank's, gathered
  int rc;
  const size_t bytes = nq * size_t(k) * 8;
  if ((rc = ensure(c, mine, bytes))) return rc;
  if ((rc = ensure(c, all, bytes * world))) return rc;
  if ((rc = topk_batch_device(segs, n_segs, kind, terms, term_off, nq, k1, b, filt, k, threshold_in, rank, mine.p, nullptr, false))) return rc;
  if ((rc = sdbg_dist_allgather(c, mine.p, all.p, bytes))) return rc;
  return sdbg_topk_merge_gathered(c, all.p, world, nq, k, out, out ? n_out : nullptr);
}

extern "C" int sdbg_dist_groupby_merge(sdbg_ctx* c, void* d_i64, void* d_f64, uint64_t span, double abs_bound) {
  if (!c || !d_i64 || !d_f64 || !span || !(abs_bound >= 0.0) || std::isinf(abs_bound)) return SDBG_EINVAL;
  if (!c->nccl_comm) return c->dist_world == 1 ? SDBG_OK : fail(c, SDBG_EINVAL, "sdbg_dist_init has not run");
  if (c->dist_world > 8) return fail(c, SDBG_EUNSUPPORTED, "fixed-point limbs are sized for up to 8 ranks");
  CU(c, cudaSetDevice(c->device));
  int ex = 0;
  std::frexp(abs_bound > 0.0 ? abs_bound : 1.0, &ex);        // abs_bound < 2^ex
  const int eunit = ex + 1 - 117;                              // 120-bit fixed point with 3 bits of headroom for 8 ranks
  DevBuf& wire = c->scratch[14];
  int rc;
  if ((rc = ensure(c, wire, (span * 7 + 1) * sizeof(long long)))) return rc;
  if (!c->h_oor) CU(c, cudaHostAlloc(reinterpret_cast<void**>(&c->h_oor), 16, cudaHostAllocDefault));
  long long* over = static_cast<long long*>(wire.p) + span * 7;
  CU(c, cudaMemsetAsync(over, 0, sizeof(long long), c->stream));
  const unsigned grid = unsigned(std::min<uint64_t>((span + 255) / 256, uint64_t(c->sm_count) * 8));
  dist_pack_kernel<<<grid, 256, 0, c->stream>>>(static_cast<const long long*>(d_i64), static_cast<const double*>(d_f64), span, eunit,
                                               abs_bound, static_cast<long long*>(wire.p));
  ++c->launches;
  // the overflow word travels with the partials, so every rank sees a bound broken on any rank
  NC(c, nccl_api().AllReduce(wire.p, wire.p, span * 7 + 1, ncclInt64, ncclSum, static_cast<ncclComm_t>(c->nccl_comm), c->stream));
  dist_unpack_kernel<<<grid, 256, 0, c->stream>>>(static_cast<const long long*>(wire.p), span, eunit, static_cast<long long*>(d_i64),
                                                 static_cast<double*>(d_f64));
  ++c->launches;
  CU(c, cudaGetLastError());
  CU(c, cudaMemcpyAsync(c->h_oor + 1, over, 8, cudaMemcpyDeviceToHost, c->stream));
  c->fix_over_pending = true;
  return SDBG_OK;
}

// ------------------------------------------------------------------------------------------
// host-side writer mirror + synthetic inputs
// ------------------------------------------------------------------------------------------
extern "C" int sdbg_writer_create(uint32_t segment_docs, int has_wand, float wand_b, const uint32_t* norms, sdbg_writer** out) {
  if (!out || segment_docs > kMaxDocId) return SDBG_EINVAL;
  auto* w = new sdbg_writer;
  w->w.reset(new PostingWriter(segment_docs, has_wand != 0, wand_b, norms));
  *out = w;
  return SDBG_OK;
}
extern "C" void sdbg_writer_destroy(sdbg_writer* w) { delete w; }
extern "C" int sdbg_writer_add_term(sdbg_writer* w, const uint32_t* docs, const uint32_t* freqs, uint32_t n) {
  if (!w || (n && (!docs || !freqs))) return SDBG_EINVAL;
  for (uint32_t i = 1; i < n; ++i) if (docs[i] <= docs[i - 1]) return SDBG_EINVAL;
  if (n && docs[0] == 0) return SDBG_EINVAL;
  w->w->add_term(docs, freqs, n);
  return SDBG_OK;
}
extern "C" int sdbg_writer_finish(sdbg_writer* w, const uint8_t** doc_file, size_t* n, const sdbg_term_meta** terms, size_t* n_terms) {
  if (!w) return SDBG_EINVAL;
  w->metas.clear();
  for (const TermMeta& m : w->w->terms()) w->metas.push_back(sdbg_term_meta{m.docs_count, m.freq, m.doc_start, m.e_skip_start});
  if (doc_file) *doc_file = w->w->bytes().data();
  if (n) *n = w->w->bytes().size();
  if (terms) *terms = w->metas.data();
  if (n_terms) *n_terms = w->metas.size();
  return SDBG_OK;
}

extern "C" uint64_t sdbg_synth_hash(uint64_t stream, uint64_t index) { return synth_hash(stream, index); }

extern "C" int sdbg_synth_corpus_ex(sdbg_segment* seg, uint64_t doc0, uint32_t n_docs, uint32_t t0, uint32_t nt, int threads,
                                    double p_floor, uint32_t* docs_count_out, uint64_t* sum_dl_out);
extern "C" int sdbg_synth_corpus(sdbg_segment* seg, uint64_t doc0, uint32_t n_docs, uint32_t t0, uint32_t nt, int threads,
                                 uint32_t* docs_count_out, uint64_t* sum_dl_out) {
  return sdbg_synth_corpus_ex(seg, doc0, n_docs, t0, nt, threads, 0.0, docs_count_out, sum_dl_out);
}
// p_floor > 0: inclusion probability max(p_floor, min(0.5, 0.6 / (t + 1))) -- a flat tail of equally sized lists, used to
// build an index much larger than L2 (the HBM-resident bench workload).
extern "C" int sdbg_synth_corpus_ex(sdbg_segment* seg, uint64_t doc0, uint32_t n_docs, uint32_t t0, uint32_t nt, int threads,
                                    double p_floor, uint32_t* docs_count_out, uint64_t* sum_dl_out) {
  if (!seg || !n_docs || !nt || n_docs != seg->n_docs || !(p_floor >= 0.0 && p_floor <= 0.5)) return SDBG_EINVAL;
  threads = std::max(1, threads);
  std::vector<uint32_t> dl(n_docs);
  uint64_t sum_dl = 0;
  for (uint32_t i = 0; i < n_docs; ++i) { dl[i] = 16 + uint32_t(synth_hash(1, doc0 + 1 + i) % 240); sum_dl += dl[i]; }
  // one writer per term (terms are independent streams), built by a pool of threads, then
  // concatenated in term order -- byte-identical to a single sequential writer.
  std::vector<std::unique_ptr<PostingWriter>> per_term(nt);
  std::atomic<uint32_t> next{0};
  const float avg = float(double(sum_dl) / double(n_docs));
  auto work = [&]() {
    std::vector<uint32_t> docs, freqs;
    for (;;) {
      const uint32_t i = next.fetch_add(1);
      if (i >= nt) break;
      const uint32_t t = t0 + i;
      // terms 1000000 .. 1000004: BASELINE configs[3]'s conjunction terms, p = 0.50, 0.40, 0.30, 0.25, 0.20 (SURVEY §8d)
      static const double kCfg4P[5] = {0.50, 0.40, 0.30, 0.25, 0.20};
      const double p = (t >= 1000000u && t < 1000005u) ? kCfg4P[t - 1000000u] : std::max(p_floor, std::min(0.5, 0.6 / double(t + 1)));
      const uint64_t thr = uint64_t(std::ldexp(p, 64));
      docs.clear(); freqs.clear();
      for (uint32_t d = 0; d < n_docs; ++d) {
        const uint64_t g = doc0 + 1 + d;
        if (synth_hash(100 + t, g) >= thr) continue;
        const uint64_t h2 = synth_hash(1000 + t, g);
        uint32_t f = 1 + (h2 ? uint32_t(__builtin_ctzll(h2)) : 64);
        f = std::min(f, dl[d]);
        docs.push_back(d + 1); freqs.push_back(f);
      }
      per_term[i].reset(new PostingWriter(n_docs, true, 0.75f, dl.data(), avg));
      per_term[i]->add_term(docs.data(), freqs.data(), uint32_t(docs.size()));
    }
  };
  std::vector<std::thread> pool;
  for (int i = 0; i < threads; ++i) pool.emplace_back(work);
  for (auto& th : pool) th.join();
  PostingWriter all(n_docs, true, 0.75f, dl.data(), avg);
  for (uint32_t i = 0; i < nt; ++i) {
    all.append(*per_term[i]);
    if (docs_count_out) docs_count_out[i] = per_term[i]->terms()[0].docs_count;
    per_term[i].reset();
  }
  if (sum_dl_out) *sum_dl_out = sum_dl;
  int rc = sdbg_stage_postings(seg, all.bytes().data(), all.bytes().size(),
                               reinterpret_cast<const sdbg_term_meta*>(all.terms().data()), all.terms().size(), 1);
  if (rc) return rc;
  std::vector<uint8_t> nb(n_docs);
  for (uint32_t i = 0; i < n_docs; ++i) nb[i] = uint8_t(dl[i]);
  const sdbg_norm_rg rg{1, n_docs, 0};
  return sdbg_stage_norms(seg, nb.data(), nb.size(), &rg, 1);
}

extern "C" int sdbg_synth_column(sdbg_segment* seg, uint64_t field, uint64_t stream, int kind, uint64_t row0, uint64_t rows) {
  if (!seg || !rows) return SDBG_EINVAL;
  sdbg_ctx* c = seg->ctx;
  CU(c, cudaSetDevice(c->device));
  const int type = (kind == 2 || kind == 4) ? SDBG_F64 : (kind == 6 ? SDBG_I32 : SDBG_I64);
  ColumnObj& col = seg->cols[field];
  const size_t bytes = rows * type_width(type);
  if (type == SDBG_I64) {   // generated into the staging buffer, then packed when that is smaller
    int rc;
    if ((rc = ensure(c, c->stage_raw, bytes + 64))) return rc;
    reset_for_packing(col, rows);
    CU(c, cudaMemsetAsync(static_cast<char*>(c->stage_raw.p) + bytes, 0, 64, c->stream));
    synth_column_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(stream, kind, row0, rows, c->stage_raw.p);
    ++c->launches;
    CU(c, cudaGetLastError());
    return pack_column(c, col);
  }
  free_column(col);
  col = ColumnObj{};
  CU(c, cudaMalloc(&col.d_values, bytes + 64));
  CU(c, cudaMemsetAsync(static_cast<char*>(col.d_values) + bytes, 0, 64, c->stream));
  col.type = type; col.rows = rows; col.owned = true;
  synth_column_kernel<<<c->sm_count * 8, 256, 0, c->stream>>>(stream, kind, row0, rows, col.d_values);
  ++c->launches;
  CU(c, cudaGetLastError());
  return SDBG_OK;
}

// ------------------------------------------------------------------------------------------
// Host-only probe of the staging parser (no device needed): lets CPU tests compare the block table
// built from a ".doc" stream with the oracle's reading of the same bytes.
// ------------------------------------------------------------------------------------------
extern "C" int sdbg_debug_stage_host(const uint8_t* doc_file, size_t n, const sdbg_term_meta* terms, size_t n_terms, int has_wand,
                                     uint32_t cap, uint32_t* n_blocks, uint32_t* term_blk_begin /* n_terms+1 */,
                                     uint32_t* last_doc, uint32_t* prev_last, uint32_t* packed, uint32_t* max_freq,
                                     uint32_t* max_norm, uint64_t* arena_bytes) {
  StagedPostings sp;
  const std::string e = stage_postings(doc_file, n, reinterpret_cast<const TermMeta*>(terms), n_terms, has_wand != 0, &sp);
  if (!e.empty()) { std::fprintf(stderr, "sdbg_debug_stage_host: %s\n", e.c_str()); return SDBG_EFORMAT; }
  if (n_blocks) *n_blocks = uint32_t(sp.blocks.size());
  if (arena_bytes) *arena_bytes = sp.arena.size();
  if (term_blk_begin) std::copy(sp.term_blk_begin.begin(), sp.term_blk_begin.end(), term_blk_begin);
  if (sp.blocks.size() > cap) return SDBG_ECAPACITY;
  for (size_t i = 0; i < sp.blocks.size(); ++i) {
    if (last_doc) last_doc[i] = sp.blocks[i].last_doc;
    if (prev_last) prev_last[i] = sp.blocks[i].prev_last;
    if (packed) packed[i] = sp.blocks[i].packed;
    if (max_freq) max_freq[i] = sp.blk_max[i].freq;
    if (max_norm) max_norm[i] = sp.blk_max[i].norm;
  }
  return SDBG_OK;
}
