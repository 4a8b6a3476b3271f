// CUDA backend for sm_90a: device memory management, uploads and launches around the tile kernel
// (tile_kernel.cuh).  Host <-> device transfers are staged through pinned memory on a private stream; the
// kernel itself can also be launched on a caller-provided stream into caller-owned device buffers (multi-GPU
// gather path, where torch.distributed owns the buffers).
#include <cuda_runtime.h>

#include <cub/cub.cuh>

#include <algorithm>
#include <chrono>
#include <functional>
#include <memory>
#include <cstdio>
#include <cstring>
#include <mutex>

#include <dlfcn.h>

#include <list>
#include <sstream>
#include <tuple>

#include "backend.hpp"
#include "ingest_kernels.cuh"
#include "spec_codegen.hpp"
#include "tile_kernel.cuh"

namespace gk {

#define CK(x)                                                                                         \
  do {                                                                                                \
    cudaError_t e_ = (x);                                                                             \
    if (e_ != cudaSuccess) throw BackendError{std::string("CUDA error: ") + cudaGetErrorString(e_) + " at " #x}; \
  } while (0)

// The host evaluates a missed lookup from its argument spans in the page.  Without the caller's page (reextract), the spans are
// gathered from the device copy of it into one compact buffer: fills `spans` with a (page offset, buffer offset, length) triple per
// span, points the records at the buffer and returns its size.
inline size_t gk_compact_miss_spans(GkMiss* m, size_t n, std::vector<unsigned long long>& spans) {
  spans.clear();
  size_t total = 0;
  for (size_t i = 0; i < n; ++i)
    for (GkMissArg& a : m[i].args) {
      if ((a.kind != GK_ARG_JSON && a.kind != GK_ARG_SYNSTR) || a.len == 0) continue;
      spans.insert(spans.end(), {a.off, (unsigned long long)total, (unsigned long long)a.len});
      a.off = total;
      total += a.len;
    }
  return total;
}

struct DevBatch {
  uint8_t* arena = nullptr;
  size_t bytes = 0;
  GkBatch hdr{};
  uint32_t n = 0;
  // per-batch output buffers (reused by every eval of a resident batch)
  uint32_t* viol = nullptr;
  uint32_t* err = nullptr;
  uint32_t words = 0;
  // tiling (depends on the batch's row distribution and on the program's slot table)
  uint32_t* d_tile_lo = nullptr;
  uint32_t* d_units = nullptr;       // [2 * n] object ranges the specialised kernel hands to the interpreter (GkKParams::units): never more than objects
  uint32_t* d_whole = nullptr;       // [ntiles + 1] the tiles handed over whole (GkKParams::whole), then the count of d_units
  uint64_t planned = 0;              // the constraint-set version whose hand-over plan d_units / d_whole hold (0: none yet)
  uint32_t nunits = 0;               // the plan's unit count
  uint32_t multi = 0;                // of those, units of more than one object (a whole tile's wide objects)
  uint64_t handed = 0;               // the objects those units cover
  // the offset image the plan writes beside it (SpecSource::image_stride): img_stride values per tile, grown (never shrunk)
  uint16_t* d_img = nullptr;
  size_t img_bytes = 0;
  uint32_t img_stride = 0;
  // the netlist with every slot id replaced by the slot's word offset in this batch's shared-memory slot area
  GkOp* d_ops = nullptr;
  uint32_t* d_pool = nullptr;
  GkOutEnt* d_outs = nullptr;
  uint32_t ntiles = 0, slot_words = 0, tile = 0;
  uint64_t prog_version = 0;
  bool gvk_uniform = false;   // every object that was not skipped has the same apiVersion and kind
  unsigned long long* gvk = nullptr;   // [n] hash of (apiVersion, kind) per object, 0 for a skipped one (audit_candidates)
  std::vector<uint32_t> cap;  // rows of the largest tile per scope (sizes the slot area of any netlist over this batch)
  std::vector<uint32_t> rows; // rows per scope in the batch, rows[0] = objects (sizes the generated kernel's export arrays)
  // the type words (program.h): pointer table and every packed scope's words, laid out by `tw` (pack_type_words); a fork's are its
  // batch's
  uint8_t* d_tw = nullptr;
  size_t tw_bytes = 0;
  GkTwLayout tw;
  bool fork = false;          // a view made by fork_batch: arena and tiling belong to the batch it was forked from
  // a resultant batch of an expanded batch (set_parents): its parents as a CSR, and the totals its own evaluations write
  uint32_t* fold_par = nullptr;
  uint32_t* fold_off = nullptr;
  uint32_t fold_m = 0;
  unsigned long long* fold_tot = nullptr;   // [2 * words * 32]
};

// ---- audit candidates (Backend::audit_candidates): rank the batch's identities, then select per constraint
// (group, version, kind) arrive as one rank per object (gr, from the page's few distinct apiVersion / kind pairs ranked on the host by
// their decoded bytes); namespace and name are the decoded bytes of the batch header, read as IdView reads them (audit.cpp).
struct GkIdLess {
  const uint32_t* gr;
  const uint32_t* flags;
  const uint32_t* ns_off;
  const uint8_t* ns;
  const uint32_t* nm_off;
  const uint8_t* nm;
  static __device__ int bytes(const uint8_t* a, uint32_t al, const uint8_t* b, uint32_t bl) {
    const uint32_t m = al < bl ? al : bl;
    for (uint32_t i = 0; i < m; ++i)
      if (a[i] != b[i]) return a[i] < b[i] ? -1 : 1;
    return al < bl ? -1 : al > bl ? 1 : 0;
  }
  __device__ uint32_t ns_len(uint32_t o) const {
    const uint32_t fl = flags[o];
    return ((fl & GK_F_IS_NS) || !(fl & GK_F_NSNAME)) ? 0u : ns_off[o + 1] - ns_off[o];
  }
  __device__ int cmp(uint32_t a, uint32_t b) const {
    if (gr[a] != gr[b]) return gr[a] < gr[b] ? -1 : 1;
    const int r = bytes(ns + ns_off[a], ns_len(a), ns + ns_off[b], ns_len(b));
    return r ? r : bytes(nm + nm_off[a], nm_off[a + 1] - nm_off[a], nm + nm_off[b], nm_off[b + 1] - nm_off[b]);
  }
  __device__ bool operator()(uint32_t a, uint32_t b) const { return cmp(a, b) < 0; }
};

__device__ __forceinline__ uint32_t gk_gvk_slot(unsigned long long k, uint32_t mask) { return (uint32_t)((k * 0x9E3779B97F4A7C15ull) >> 40) & mask; }

// distinct apiVersion / kind hashes of the page into an open-addressing table (keys 0 = empty), with the smallest object of each
__global__ void gk_gvk_insert_kernel(const unsigned long long* gvk, uint32_t n, unsigned long long* keys, uint32_t* rep, uint32_t mask) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned long long k = gvk[i];
    if (!k) continue;
    for (uint32_t s = gk_gvk_slot(k, mask);; s = (s + 1) & mask) {
      const unsigned long long prev = atomicCAS(&keys[s], 0ull, k);
      if (prev == 0ull || prev == k) {
        atomicMin(&rep[s], i);
        break;
      }
    }
  }
}
__global__ void gk_gvk_collect_kernel(const unsigned long long* keys, const uint32_t* rep, uint32_t cap, uint32_t* cnt, uint32_t* out) {
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < cap; s += gridDim.x * blockDim.x)
    if (keys[s]) {
      const uint32_t j = atomicAdd(cnt, 1u);
      out[2 * j] = s;
      out[2 * j + 1] = rep[s];
    }
}
// rank of each table entry (slot, rank pairs from the host) into rep, then one rank per object
__global__ void gk_gvk_assign_kernel(const uint32_t* pairs, uint32_t m, uint32_t* rep) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < m) rep[pairs[2 * j]] = pairs[2 * j + 1];
}
__global__ void gk_gvk_map_kernel(const unsigned long long* gvk, uint32_t n, const unsigned long long* keys, const uint32_t* rank, uint32_t mask,
                                  uint32_t* gr, uint32_t* perm) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned long long k = gvk[i];
    uint32_t r = 0;
    if (k)
      for (uint32_t s = gk_gvk_slot(k, mask);; s = (s + 1) & mask)
        if (keys[s] == k) {
          r = rank[s];
          break;
        }
    gr[i] = r;
    perm[i] = i;
  }
}
// after the sort: 1 where a sorted position starts a new identity (then scanned into the identity's rank)
__global__ void gk_id_heads_kernel(const uint32_t* perm, uint32_t n, GkIdLess id, uint32_t* head) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) head[p] = p && id.cmp(perm[p - 1], perm[p]) != 0;
}
__global__ void gk_id_scatter_kernel(const uint32_t* perm, const uint32_t* grp, uint32_t n, uint32_t* rank) {
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) rank[perm[p]] = grp[p];
}
constexpr uint32_t kSelChunk = 1024;   // sorted positions per block of the per-constraint counts
// cnt[b * C + c]: objects with bit c among the sorted positions [b * kSelChunk, (b + 1) * kSelChunk)
__global__ void __launch_bounds__(256) gk_sel_count_kernel(const uint32_t* perm, const uint32_t* viol, uint32_t n, uint32_t words, uint32_t C, uint32_t* cnt) {
  extern __shared__ uint32_t sh[];
  for (uint32_t c = threadIdx.x; c < C; c += blockDim.x) sh[c] = 0;
  __syncthreads();
  const uint32_t lo = blockIdx.x * kSelChunk, hi = min(n, lo + kSelChunk);
  for (uint32_t p = lo + threadIdx.x; p < hi; p += blockDim.x) {
    const uint32_t* row = viol + (size_t)perm[p] * words;
    for (uint32_t w = 0; w < words; ++w)
      for (uint32_t v = row[w]; v; v &= v - 1) {
        const uint32_t c = w * 32 + (uint32_t)__ffs(v) - 1;
        if (c < C) atomicAdd(&sh[c], 1u);
      }
  }
  __syncthreads();
  for (uint32_t c = threadIdx.x; c < C; c += blockDim.x) cnt[(size_t)blockIdx.x * C + c] = sh[c];
}
// one warp per constraint: the sorted position of its limit-th flagged object -> thr[c] = that object's rank (all ones: fewer than limit)
__global__ void gk_sel_thresh_kernel(const uint32_t* perm, const uint32_t* viol, const uint32_t* cnt, const uint32_t* rank, uint32_t n, uint32_t words,
                                     uint32_t C, uint32_t nb, uint32_t limit, uint32_t* thr) {
  const uint32_t c = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x & 31u;
  if (c >= C) return;
  uint32_t acc = 0, need = 0, blk = ~0u;
  for (uint32_t base = 0; base < nb && blk == ~0u; base += 32) {
    const uint32_t v = base + lane < nb ? cnt[(size_t)(base + lane) * C + c] : 0u;
    uint32_t s = v;
    for (uint32_t d = 1; d < 32; d <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += t;
    }
    const uint32_t hit = __ballot_sync(0xffffffffu, acc + s >= limit);
    if (hit) {
      const uint32_t f = (uint32_t)__ffs(hit) - 1;
      need = limit - (acc + __shfl_sync(0xffffffffu, s - v, f));   // 1-based among the block's flagged positions
      blk = base + f;
    }
    acc += __shfl_sync(0xffffffffu, s, 31);
  }
  if (blk == ~0u) {
    if (!lane) thr[c] = ~0u;
    return;
  }
  const uint32_t lo = blk * kSelChunk, hi = min(n, lo + kSelChunk);
  for (uint32_t p = lo; p < hi; p += 32) {
    const uint32_t q = p + lane;
    const bool b = q < hi && (viol[(size_t)perm[q] * words + (c >> 5)] >> (c & 31u) & 1u);
    const uint32_t bal = __ballot_sync(0xffffffffu, b);
    const uint32_t k = (uint32_t)__popc(bal);
    if (need <= k) {
      uint32_t m = bal;
      for (uint32_t j = 1; j < need; ++j) m &= m - 1;
      if (!lane) thr[c] = rank[perm[p + (uint32_t)__ffs(m) - 1]];
      return;
    }
    need -= k;
  }
}
__global__ void gk_sel_emit_kernel(const uint32_t* viol, const uint32_t* rank, const uint32_t* thr, uint32_t n, uint32_t words, uint32_t C, uint32_t* cand) {
  const size_t total = (size_t)n * words;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const uint32_t o = (uint32_t)(i / words), w = (uint32_t)(i % words), r = rank[o];
    uint32_t out = 0;
    for (uint32_t v = viol[i]; v; v &= v - 1) {
      const uint32_t k = (uint32_t)__ffs(v) - 1, c = w * 32 + k;
      if (c < C && r <= thr[c]) out |= 1u << k;
    }
    cand[i] = out;
  }
}

// the type words of one scope (program.h), one thread per row
__global__ void gk_tw_pack_kernel(const GkColumn* cols, const uint32_t* vtcols, uint32_t nvt, uint32_t W, uint32_t rows, uint32_t* dst) {
  for (size_t row = (size_t)blockIdx.x * blockDim.x + threadIdx.x; row < rows; row += (size_t)gridDim.x * blockDim.x) gk_tw_pack_row(cols, vtcols, nvt, W, row, dst);
}

// ---- expanded batches (Backend::select_generators, eval_expanded, fold_into)
// 1 for every object whose apiVersion / kind hash was selected on the host (pick[slot] != 0), and for every object with hash 0
__global__ void gk_gen_mark_kernel(const unsigned long long* gvk, uint32_t n, const unsigned long long* keys, const uint32_t* pick, uint32_t mask,
                                   uint8_t* mark, uint32_t* idx) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned long long k = gvk[i];
    uint8_t m = 1;
    if (k)
      for (uint32_t s = gk_gvk_slot(k, mask);; s = (s + 1) & mask)
        if (keys[s] == k) {
          m = pick[s] != 0;
          break;
        }
    mark[i] = m;
    idx[i] = i;
  }
}
// one thread per parent with resultants (fold_core.h), the newly set bits counted per CTA in shared memory [2 * C], then one atomic per
// CTA and constraint
__global__ void __launch_bounds__(256) gk_fold_kernel(GkFoldArgs a) {
  extern __shared__ uint32_t sh[];
  const uint32_t C = a.nconstraints;
  for (uint32_t c = threadIdx.x; c < 2 * C; c += blockDim.x) sh[c] = 0;
  __syncthreads();
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < a.m; j += gridDim.x * blockDim.x)
    gk_fold_parent(a, j, [&](uint32_t c, uint32_t plane) {
      if (c < C) atomicAdd(&sh[plane * C + c], 1u);
    });
  __syncthreads();
  for (uint32_t c = threadIdx.x; c < C; c += blockDim.x) {
    if (sh[c]) atomicAdd(a.totals + c, (unsigned long long)sh[c]);
    if (sh[C + c]) atomicAdd(a.err_totals + c, (unsigned long long)sh[C + c]);
  }
}
// ---- the audit of an expanded batch's resultants (Backend::audit_resultants)
struct GkResAuditArgs {
  GkResClassArgs a;
  const uint32_t* par;             // the resident CSR of set_parents: parent par[j] has resultants off[j] .. off[j + 1] - 1
  const uint32_t* off;
  uint32_t m, nres;                // parents in the CSR, resultants
  const uint32_t* rank;            // [parents] the parents' ranking (audit_candidates), and per constraint its threshold rank
  const uint32_t* thr;
  const uint8_t* cls;              // [nres] action class
  const uint8_t* dead;             // [parents] or null
  uint32_t classes;
  unsigned long long* counted;     // [classes * nconstraints]
  uint32_t* list;                  // [2 * cap] (resultant, constraint | is_err << 31)
  uint32_t* nlist;
  uint32_t cap;
};
// One thread per resultant row (fold_core.h gk_classify_resultant): a row is a few words, and a thread per row keeps the lanes busy
// whatever the parents' fan-out -- a thread per parent would leave a warp waiting on its one parent with many resultants.  The parent
// comes from a binary search of the resident CSR.  Counts go through shared memory [classes * C], one atomic per CTA and counter; each
// warp reserves its pairs to render with one atomic (a first pass counts them, a second writes them).
__global__ void __launch_bounds__(256) gk_res_classify_kernel(GkResAuditArgs x) {
  extern __shared__ uint32_t sh[];
  const uint32_t C = x.a.nconstraints, NC = x.classes * C, lane = threadIdx.x & 31u;
  for (uint32_t i = threadIdx.x; i < NC; i += blockDim.x) sh[i] = 0;
  __syncthreads();
  for (uint32_t base = blockIdx.x * blockDim.x; base < x.nres; base += gridDim.x * blockDim.x) {   // (uniform per warp: the shuffles see all lanes)
    const uint32_t r = base + threadIdx.x;
    bool on = false;
    uint32_t rk = 0;
    if (r < x.nres) {
      uint32_t lo = 0, hi = x.m;   // off[lo] <= r < off[hi]
      while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (x.off[mid] <= r) lo = mid;
        else hi = mid;
      }
      const uint32_t p = x.par[lo];
      on = !(x.dead && x.dead[p]);
      rk = x.rank[p];
    }
    auto cand = [&](uint32_t c) { return rk <= x.thr[c]; };
    uint32_t ne = 0;
    if (on) gk_classify_resultant(x.a, r, cand, [](uint32_t) {}, [&](uint32_t, uint32_t) { ++ne; });
    uint32_t incl = ne;
    for (uint32_t d = 1; d < 32; d <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += t;
    }
    const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
    uint32_t at = 0;
    if (lane == 31 && total) at = atomicAdd(x.nlist, total);
    at = __shfl_sync(0xffffffffu, at, 31) + incl - ne;
    if (on)
      gk_classify_resultant(
          x.a, r, cand, [&](uint32_t c) { atomicAdd(&sh[x.cls[r] * C + c], 1u); },
          [&](uint32_t c, uint32_t is_err) {
            if (at < x.cap) {
              x.list[2 * (size_t)at] = r;
              x.list[2 * (size_t)at + 1] = c | is_err << 31;
            }
            ++at;
          });
  }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < NC; i += blockDim.x)
    if (sh[i]) atomicAdd(x.counted + i, (unsigned long long)sh[i]);
}

// the fused exchange: the folded totals replace the ones the evaluation published to every peer
__global__ void gk_fold_publish_kernel(GkFoldArgs a) {
  for (uint32_t c = threadIdx.x; c < a.nconstraints; c += blockDim.x)
    for (uint32_t q = 0; q < a.npeers; ++q) {
      a.peer_tot[q][c] = a.totals[c];
      a.peer_tot[q][a.tot_stride + c] = a.err_totals[c];
    }
  __threadfence_system();
}

class CudaBackend : public Backend {
 public:
  explicit CudaBackend(int device) : device_(device) {
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
      throw BackendError{"no CUDA device: gatekeeper_b200 has no CPU fallback; the evaluation path requires an H100 (sm_90a) GPU"};
    if (device_ >= ndev) throw BackendError{"CUDA device index out of range"};
    CK(cudaSetDevice(device_));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device_));
    sms_ = prop.multiProcessorCount;
    max_smem_ = optin_smem_ = (size_t)prop.sharedMemPerBlockOptin;
    sm_smem_ = (size_t)prop.sharedMemPerMultiprocessor;
    CK(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&copy_stream_, cudaStreamNonBlocking));
    {
      // The tokeniser of the NEXT page runs on a high-priority stream: its launches are small (a few hundred CTAs per 32 MB
      // chunk) and would otherwise only start in the tails of the current page's extraction kernels, whose grids keep the
      // block scheduler busy -- the two pages then run fully serialised.
      int lo = 0, hi = 0;
      CK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
      const bool prio = !getenv("GK_NO_STREAM_PRIORITY");
      CK(cudaStreamCreateWithPriority(&front_stream_, cudaStreamNonBlocking, prio ? hi : lo));
    }
    // result bitmaps are copied back into page-locked blocks (backend.hpp HostBlockAlloc)
    host_block_hooks().alloc = [](size_t bytes) -> void* {
      void* p = nullptr;
      return cudaHostAlloc(&p, bytes, cudaHostAllocPortable) == cudaSuccess ? p : nullptr;
    };
    host_block_hooks().release = [](void* p) { cudaFreeHost(p); };
    {
      // per-batch device memory comes from the stream-ordered pool and goes back to it: with the release threshold lifted a
      // resident-batch-sized arena is reused by the next batch instead of being mapped / unmapped by the driver every time
      cudaMemPool_t pool;
      CK(cudaDeviceGetDefaultMemPool(&pool, device_));
      unsigned long long keep = ~0ull;
      CK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
    }
    CK(cudaEventCreate(&ev0_));
    CK(cudaEventCreate(&ev1_));
    {
      int lo = 0, hi = 0;
      CK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
      CK(cudaStreamCreateWithPriority(&side_stream_, cudaStreamNonBlocking, hi));   // fire(): the interpreter's units
    }
    CK(cudaEventCreateWithFlags(&ev_fork_, cudaEventDisableTiming));
    cudaFuncAttributes fa;
    CK(cudaFuncGetAttributes(&fa, gk_eval_kernel));
    max_smem_ -= fa.sharedSizeBytes;   // the kernel's few static shared bytes come out of the same per-CTA budget
    CK(cudaFuncSetAttribute(gk_eval_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_smem_));
    CK(cudaMalloc(&d_scalars_, 4096));
  }
  ~CudaBackend() override {
    cudaSetDevice(device_);
    free_tables();
    if (d_dict_off_) cudaFree(d_dict_off_);
    if (d_dict_bytes_) cudaFree(d_dict_bytes_);
    if (d_scalars_) cudaFree(d_scalars_);
    if (d_totals_) cudaFree(d_totals_);
    if (d_errlist_) cudaFree(d_errlist_);
    if (d_spec_x_) cudaFree(d_spec_x_);
    if (d_active_) cudaFree(d_active_);
    if (pinned_) cudaFreeHost(pinned_);
    cudaEventDestroy(ev0_);
    cudaEventDestroy(ev1_);
    cudaEventDestroy(ev_fork_);
    cudaStreamDestroy(side_stream_);
    cudaStreamDestroy(stream_);
  }
  const char* name() const override { return "cuda-sm90a"; }
  const char* last_kernel() const override { return last_kernel_; }

  void set_program(const Compiled& c) override {
    std::lock_guard<std::mutex> l(mu_);
    if (version_ == c.version) return;
    CK(cudaSetDevice(device_));
    free_tables();
    prog_ = GkProgram{};
    prog_.nconstraints = (uint32_t)c.cons_match.size();
    prog_.nmatch = (uint32_t)c.match.size();
    prog_.nops = (uint32_t)c.ops.size();
    prog_.nslots = (uint32_t)c.slot_level.size();
    prog_.npool = (uint32_t)c.pool.size();
    prog_.ncbytes = (uint32_t)c.cbytes.size();
    prog_.nphases = (uint32_t)c.phase_off.size() - 1;
    prog_.nitems = (uint32_t)c.items.size();
    if (prog_.nphases > kMaxPhases) throw BackendError{"netlist has more dependency phases than the kernel supports"};
    auto up = [&](const void* src, size_t bytes, void** dst) {
      size_t padded = (bytes + 63) / 64 * 64 + 64;
      CK(cudaMalloc(dst, padded));
      CK(cudaMemset(*dst, 0, padded));
      if (bytes) CK(cudaMemcpy(*dst, src, bytes, cudaMemcpyHostToDevice));
    };
    up(c.ops.data(), c.ops.size() * sizeof(GkOp), (void**)&d_ops_);
    up(c.items.data(), c.items.size() * 4, (void**)&d_items_);
    up(c.outs.data(), c.outs.size() * sizeof(GkOutEnt), (void**)&d_outs_);
    up(c.phase_off.data(), c.phase_off.size() * 4, (void**)&d_phase_off_);
    up(c.match.data(), c.match.size() * sizeof(GkMatch), (void**)&d_match_);
    up(c.pool.data(), c.pool.size() * 4, (void**)&d_pool_);
    up(c.cbytes.data(), c.cbytes.size(), (void**)&d_cbytes_);
    prog_.ops = d_ops_;
    prog_.items = d_items_;
    prog_.outs = d_outs_;
    prog_.phase_off = d_phase_off_;
    prog_.match = d_match_;
    prog_.pool = d_pool_;
    prog_.cbytes = d_cbytes_;
    const uint32_t C = prog_.nconstraints;
    if (d_totals_) cudaFree(d_totals_);
    CK(cudaMalloc(&d_totals_, (size_t)(2 * std::max(C, 1u)) * sizeof(unsigned long long)));
    if (d_active_) cudaFree(d_active_);
    CK(cudaMalloc(&d_active_, (size_t)std::max(C, 1u) * 4));
    if (!d_errlist_) CK(cudaMalloc(&d_errlist_, (size_t)err_cap_ * 3 * 4));
    last_active_.clear();
    version_ = c.version;
    spec_select(c);
  }

  void sync_strings(const StringTable& st) override {
    std::lock_guard<std::mutex> l(mu_);
    uint32_t n = st.size();
    if (n == dict_n_) return;
    CK(cudaSetDevice(device_));
    std::vector<uint32_t> off;
    std::vector<uint8_t> bytes;
    st.snapshot(off, bytes);
    if (d_dict_off_) cudaFree(d_dict_off_);
    if (d_dict_bytes_) cudaFree(d_dict_bytes_);
    CK(cudaMalloc(&d_dict_off_, off.size() * 4 + 64));
    CK(cudaMalloc(&d_dict_bytes_, bytes.size() + 64));
    CK(cudaMemcpy(d_dict_off_, off.data(), off.size() * 4, cudaMemcpyHostToDevice));
    if (!bytes.empty()) CK(cudaMemcpy(d_dict_bytes_, bytes.data(), bytes.size(), cudaMemcpyHostToDevice));
    dict_n_ = (uint32_t)off.size() - 1;
  }

  void* upload(const HostBatch& hb, const Compiled& c, double* h2d_ms, uint64_t* h2d_bytes) override {
    CK(cudaSetDevice(device_));
    PackedBatch pb;
    PackPlan plan;
    pack_layout(hb, c, pb, plan);   // offsets only: the bytes are copied once, below, straight into pinned memory
    // ---- tiling: first row of every scope for every tile, slot offsets from the per-scope tile capacities
    const uint32_t NS = (uint32_t)c.schema.scopes.size();
    // Tile size: kTile objects unless the page needs smaller tiles.  (Shrinking tiles so that the tile count fills whole waves of
    // resident CTAs -- 480 instead of 512 objects for 1M -- measured slower: the per-tile fixed cost outweighs the fuller last wave.)
    uint32_t ntiles = 0;
    std::vector<uint32_t> tile_lo, cap;
    const uint32_t tile = gk_choose_tile(kTile, net_sizes(c), max_smem_, [&](uint32_t per_tile) -> const std::vector<uint32_t>& {
      ntiles = (hb.n + per_tile - 1) / per_tile;
      tile_lo.assign((size_t)(ntiles + 1) * NS, 0);
      cap.assign(NS, 0);
      for (uint32_t t = 0; t <= ntiles; ++t) {
        uint32_t* lo = &tile_lo[(size_t)t * NS];
        lo[0] = std::min<uint32_t>(t * per_tile, hb.n);
        for (uint32_t s = 1; s < NS; ++s) lo[s] = hb.scope_off[s][lo[c.schema.scopes[s].parent]];
        if (t)
          for (uint32_t s = 0; s < NS; ++s) cap[s] = std::max(cap[s], lo[s] - tile_lo[(size_t)(t - 1) * NS + s]);
      }
      return cap;
    });
    auto* db = new DevBatch();
    db->bytes = gk_align(plan.total);
    db->n = hb.n;
    db->ntiles = ntiles;
    db->tile = tile;
    db->prog_version = c.version;
    db->gvk_uniform = hb.gvk_hi == 0 || hb.gvk_lo == hb.gvk_hi;
    db->rows = hb.scope_rows;
    db->rows.resize(NS, 0);
    db->rows[0] = hb.n;
    dmalloc(&db->arena, db->bytes);
    dmalloc(&db->d_tile_lo, tile_lo.size() * 4 + 64);
    if (hb.n) dmalloc(&db->gvk, (size_t)hb.n * 8);
    finish_batch(db, c, cap);
    const size_t tables_bytes = c.ops.size() * sizeof(GkOp) + c.pool.size() * 4 + c.outs.size() * sizeof(GkOutEnt);
    Event a, b;
    {
      std::lock_guard<std::mutex> l(mu_);
      // the arena image is assembled by all host threads directly in pinned memory (one copy of every byte), its
      // in-arena pointer tables are rebased to the device address, and one DMA moves it
      if (pinned_bytes_ < plan.total) {
        if (pinned_) cudaFreeHost(pinned_);
        pinned_bytes_ = plan.total + (plan.total >> 2);
        CK(cudaMallocHost(&pinned_, pinned_bytes_));
      }
      uint8_t* image = static_cast<uint8_t*>(pinned_);
      pack_copy(plan, image, host_threads_);
      db->hdr = rebase_batch(pb, image, db->arena);
      CK(cudaEventRecord(a, stream_));
      CK(cudaMemcpyAsync(db->arena, image, plan.total, cudaMemcpyHostToDevice, stream_));
      CK(cudaMemcpyAsync(db->d_tile_lo, tile_lo.data(), tile_lo.size() * 4, cudaMemcpyHostToDevice, stream_));
      if (hb.n) CK(cudaMemcpyAsync(db->gvk, hb.gvk.data(), (size_t)hb.n * 8, cudaMemcpyHostToDevice, stream_));
      CK(cudaEventRecord(b, stream_));
      pack_type_words(db, c);
      CK(cudaStreamSynchronize(stream_));
    }
    float ms = 0;
    cudaEventElapsedTime(&ms, a, b);
    if (h2d_ms) *h2d_ms = ms;
    if (h2d_bytes) *h2d_bytes = plan.total + tile_lo.size() * 4 + tables_bytes;
    return db;
  }

  // what the decision netlist and, for the audit, the ambiguity netlist of `c` need in shared memory (eval_layout.h)
  static std::vector<GkNetSize> net_sizes(const Compiled& c) {
    std::vector<GkNetSize> nets;
    for (const Compiled* k : {&c, c.amb.get()})
      if (k)
        nets.push_back({(uint32_t)k->cons_match.size(), (uint32_t)k->schema.scopes.size(), (uint32_t)k->phase_off.size() - 1, (uint32_t)k->ops.size(),
                        (uint32_t)k->items.size(), (uint32_t)k->match.size(), (uint32_t)k->schema.cols.size(), (uint32_t)k->pool.size(),
                        (uint32_t)k->cbytes.size(), k->slot_level});
    return nets;
  }

  // The type words of a batch whose columns are resident, or are being copied there on stream_ (program.h): derived on the device from
  // the VT byte columns, which stay (the interpreter reads them), one pass per scope that has them.  upload() and extract(), every
  // path by which a batch's columns become resident, end here; the caller synchronises stream_ before the batch is evaluated.
  void pack_type_words(DevBatch* db, const Compiled& c) {
    const size_t NS = c.schema.scopes.size();
    db->tw = gk_tw_layout(c.schema.cols, NS);
    if (!db->tw.any()) return;
    std::vector<size_t> at;
    db->tw_bytes = db->tw.bytes(db->rows, &at);
    std::vector<uint32_t> vc;   // every scope's VT columns, back to back
    std::vector<size_t> vc_at(NS, 0);
    for (size_t s = 0; s < NS; ++s) {
      vc_at[s] = vc.size();
      vc.insert(vc.end(), db->tw.vtcols[s].begin(), db->tw.vtcols[s].end());
    }
    // the layout's allocation (pointer table, words), then the column lists the pack pass reads
    dmalloc(&db->d_tw, db->tw_bytes + vc.size() * 4);
    std::vector<uint64_t> ptr(NS, 0);
    for (size_t s = 0; s < NS; ++s)
      if (db->tw.words[s]) ptr[s] = reinterpret_cast<uint64_t>(db->d_tw + at[s]);
    push_small(db->d_tw, ptr.data(), NS * 8);
    uint32_t* d_vc = reinterpret_cast<uint32_t*>(db->d_tw + db->tw_bytes);
    push_small(d_vc, vc.data(), vc.size() * 4);
    for (size_t s = 0; s < NS; ++s) {
      const uint32_t rows = s < db->rows.size() ? db->rows[s] : 0u;
      if (!db->tw.words[s] || !rows) continue;
      gk_tw_pack_kernel<<<std::min<uint32_t>((rows + 255u) / 256u, (uint32_t)sms_ * 16u), 256, 0, stream_>>>(
          db->hdr.cols, d_vc + vc_at[s], (uint32_t)db->tw.vtcols[s].size(), db->tw.words[s], rows, reinterpret_cast<uint32_t*>(db->d_tw + at[s]));
      CK(cudaGetLastError());
      ++launches_;
    }
    db->hdr.tw = reinterpret_cast<const uint32_t* const*>(db->d_tw);
    if (getenv("GK_TRACE_LAUNCH")) {
      std::string line = "[launch] type words:";
      for (size_t s = 0; s < NS; ++s)
        if (db->tw.words[s]) line += " scope " + std::to_string(s) + ": " + std::to_string(db->tw.vtcols[s].size()) + " vt columns in " + std::to_string(db->tw.words[s]) + " words;";
      fprintf(stderr, "%s %zu bytes for %u objects\n", line.c_str(), db->tw_bytes, db->n);
    }
  }

  // slot area of a tile from the per-scope tile capacities; the netlist with slot ids resolved to word offsets; output planes
  void finish_batch(DevBatch* db, const Compiled& c, std::vector<uint32_t> cap) {
    cap[0] = db->tile;
    db->cap = cap;
    std::vector<uint32_t> slot_off;
    const uint64_t slot_words = gk_slot_layout(c.slot_level, cap, &slot_off);
    if (slot_words > 0xffffu) throw BackendError{"slot area exceeds 16-bit word offsets"};
    db->slot_words = (uint32_t)slot_words;
    // resolve slot ids -> word offsets once per batch: the kernel then addresses slots without a table lookup
    std::vector<GkOp> ops_r = c.ops;
    std::vector<uint32_t> pool_r = c.pool;
    std::vector<GkOutEnt> outs_r = c.outs;
    {
      std::vector<uint8_t> done(pool_r.size(), 0);
      auto so = [&](uint32_t slot) { return slot < slot_off.size() ? slot_off[slot] : 0u; };
      for (auto& op : ops_r) {
        const uint32_t kind = op.w0 & 0xffu;
        op.w0 = (op.w0 & 0xffffu) | (so(op.w0 >> 16) << 16);
        if (kind == GK_N_GATE) {
          for (uint32_t j = 0; j < op.w3; ++j) {
            uint32_t& e = pool_r[op.w1 + j];
            if (done[op.w1 + j]++) continue;
            e = (e & 0x80000000u) | so(e & 0xffffu);
          }
        } else if (kind == GK_N_BCAST || kind == GK_N_ACC || kind == GK_N_ACC2) {
          for (uint32_t j = 0; j < op.w3; ++j) {
            uint32_t& e = pool_r[op.w1 + j];
            if (done[op.w1 + j]++) continue;
            e = so(e & 0xffffu) | (so(e >> 16) << 16);
          }
        } else if (kind == GK_N_MATCH) {
          op.w1 = so(op.w1 & 0xffffu);
        } else if (kind == GK_N_ATOMS) {
          for (uint32_t j = 0; j < op.w3; ++j) {
            uint32_t& e = pool_r[op.w2 + j * GK_ATOMS_ENT];
            if (done[op.w2 + j * GK_ATOMS_ENT]++) continue;
            e = (e & 0xffffu) | (so(e >> 16) << 16);
          }
        }
      }
      for (auto& oe : outs_r) {
        oe.prog_slot = (uint16_t)so(oe.prog_slot);
        oe.match_slot = (uint16_t)so(oe.match_slot);
        oe.err_slot = (uint16_t)so(oe.err_slot);
      }
    }
    auto r64 = [](size_t b) { return (b + 63) / 64 * 64 + 64; };
    dmalloc(&db->d_ops, r64(ops_r.size() * sizeof(GkOp)));
    dmalloc(&db->d_pool, r64(pool_r.size() * 4));
    dmalloc(&db->d_outs, r64(outs_r.size() * sizeof(GkOutEnt)));
    CK(cudaMemsetAsync(db->d_ops, 0, r64(ops_r.size() * sizeof(GkOp)), stream_));
    CK(cudaMemsetAsync(db->d_pool, 0, r64(pool_r.size() * 4), stream_));
    CK(cudaMemsetAsync(db->d_outs, 0, r64(outs_r.size() * sizeof(GkOutEnt)), stream_));
    push_small(db->d_ops, ops_r.data(), ops_r.size() * sizeof(GkOp));
    push_small(db->d_pool, pool_r.data(), pool_r.size() * 4);
    push_small(db->d_outs, outs_r.data(), outs_r.size() * sizeof(GkOutEnt));
    db->words = std::max<uint32_t>(1, (uint32_t)((c.cons_match.size() + 31) / 32));
    dmalloc(&db->d_units, (size_t)db->n * 2 * 4);
    dmalloc(&db->d_whole, ((size_t)db->ntiles + 1) * 4);
    dmalloc(&db->viol, (size_t)std::max(db->n, 1u) * db->words * 4);
    dmalloc(&db->err, (size_t)std::max(db->n, 1u) * db->words * 4);
    CK(cudaStreamSynchronize(stream_));
  }

  // ---- small uploads through the SMs (gk_push_kernel): staged in a ring of mapped page-locked memory.  The caller's buffer is free
  // to go as soon as the call returns.
  void push_small(void* dst, const void* src, size_t bytes) {
    if (!bytes) return;
    std::lock_guard<std::mutex> sl(stage_mu_);   // (uploads and forks of different batches run concurrently: one ring, one writer)
    if (bytes > (4u << 20) || getenv("GK_NO_PUSH_KERNEL")) {   // (big: the copy engine is the right tool)
      CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream_));
      CK(cudaStreamSynchronize(stream_));
      return;
    }
    const size_t need = (bytes + 15) & ~(size_t)15;
    if (!stage_host_) {
      stage_cap_ = 16u << 20;
      CK(cudaHostAlloc(reinterpret_cast<void**>(&stage_host_), stage_cap_, cudaHostAllocMapped | cudaHostAllocPortable));
      CK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&stage_dev_), stage_host_, 0));
      stage_off_ = 0;
    }
    if (stage_off_ + need > stage_cap_) {   // wrap: everything staged so far must have been read
      CK(cudaStreamSynchronize(stream_));
      stage_off_ = 0;
    }
    memcpy(stage_host_ + stage_off_, src, bytes);
    const uint32_t grid = (uint32_t)std::min<size_t>(64, (bytes + 4095) / 4096);
    gk_push_kernel<<<grid, 256, 0, stream_>>>(static_cast<uint8_t*>(dst), stage_dev_ + stage_off_, bytes);
    CK(cudaGetLastError());
    stage_off_ += need;
  }
  uint8_t *stage_host_ = nullptr, *stage_dev_ = nullptr;
  size_t stage_cap_ = 0, stage_off_ = 0;
  std::mutex stage_mu_;

  template <class T>
  void dmalloc(T** p, size_t bytes) { CK(cudaMallocAsync(reinterpret_cast<void**>(p), std::max<size_t>(bytes, 256), stream_)); }
  void dfree(void* p) {
    if (p) cudaFreeAsync(p, stream_);
  }
  // stream-ordered scratch of one call: every take() is freed on stream_ when the call returns or throws
  struct Temps {
    CudaBackend* be;
    std::vector<void*> held;
    explicit Temps(CudaBackend* b) : be(b) {}
    Temps(const Temps&) = delete;
    Temps& operator=(const Temps&) = delete;
    ~Temps() {
      for (void* p : held) be->dfree(p);
    }
    template <class T = void>
    T* take(size_t bytes) {
      T* p = nullptr;
      be->dmalloc(&p, bytes);
      held.push_back(p);
      return p;
    }
  };
  // a timing event of one call, destroyed when the call returns or throws (those of a call are locals, so a failed create destroys
  // the ones already made)
  struct Event {
    cudaEvent_t e = nullptr;
    Event() { CK(cudaEventCreate(&e)); }
    Event(const Event&) = delete;
    Event& operator=(const Event&) = delete;
    ~Event() { cudaEventDestroy(e); }
    operator cudaEvent_t() const { return e; }
  };
  void release(void* b) override {
    auto* db = static_cast<DevBatch*>(b);
    if (!db) return;
    cudaSetDevice(device_);
    if (!db->fork) dfree(db->arena);
    dfree(db->viol);
    dfree(db->err);
    if (!db->fork) dfree(db->d_tile_lo);
    if (!db->fork) dfree(db->gvk);
    dfree(db->fold_par);
    dfree(db->fold_off);
    dfree(db->fold_tot);
    dfree(db->d_units);
    dfree(db->d_whole);
    dfree(db->d_img);
    dfree(db->d_ops);
    dfree(db->d_pool);
    dfree(db->d_outs);
    dfree(db->d_tw);
    delete db;
  }

  // One evaluation as prepare() decides it and fire() carries it out: the interpreter's parameters and, when the kernel generated
  // for the constraint set runs, that kernel and its sizes.
  struct SpecEntry;
  struct Launch {
    KParams p;
    size_t smem = 0;             // the interpreter's dynamic shared memory per CTA
    cudaStream_t st = nullptr;
    SpecEntry* spec = nullptr;   // the generated kernel, or null: the interpreter alone
    uint32_t* x = nullptr;       // its export arrays
    const uint16_t* img = nullptr;   // the batch's offset image, img_stride values per tile
    uint32_t img_stride = 0;
    size_t spec_smem = 0;        // its dynamic shared memory per CTA
    int spec_per_sm = 1;         // its resident CTAs per SM at that size
    uint32_t rows_grid = 0;      // blocks of the rows kernel
    uint32_t units = 0;          // units the interpreter evaluates beside it (the batch's hand-over plan)
    uint32_t multi = 0;          // of those, units of more than one object
    uint64_t handed = 0;         // the objects they cover
  };

  // the fused exchange's peer addressing, from the caller's DevOutPtrs into GkKParams or GkFoldArgs.  Called before anything is zeroed
  // or launched (first in prepare(), and in fold_into() before the resultants' evaluation): bad addressing leaves the caller's buffers
  // untouched.
  template <class A>
  static void set_peers(A& a, const DevOutPtrs& dst) {
    if (dst.npeers > GK_MAX_PEERS || (dst.npeers && dst.rank >= dst.npeers)) throw BackendError{"bad peer addressing for the fused exchange"};
    a.npeers = dst.npeers;
    a.tot_stride = dst.tot_stride;
    for (uint32_t q = 0; q < GK_MAX_PEERS; ++q) {
      a.peer_viol[q] = q < dst.npeers ? reinterpret_cast<uint32_t*>(dst.peer_viol[q]) : nullptr;
      a.peer_tot[q] = q < dst.npeers ? reinterpret_cast<unsigned long long*>(dst.peer_tot[q]) : nullptr;
    }
  }

  // everything a launch needs besides the kernels themselves (kept outside the timed region); `peers`: eval_into()'s fused exchange
  Launch prepare(DevBatch* db, const std::vector<uint32_t>& active, uint32_t* viol, uint32_t* err, unsigned long long* totals,
                 unsigned long long* err_totals, cudaStream_t st, const DevOutPtrs& peers = DevOutPtrs{}) {
    const uint32_t C = prog_.nconstraints;
    if (db->prog_version != version_) throw BackendError{"batch was uploaded for another constraint set"};
    Launch l;
    l.st = st;
    KParams& p = l.p;
    set_peers(p, peers);
    p.batch = db->hdr;
    p.batch.dict_off = d_dict_off_;
    p.batch.dict_bytes = d_dict_bytes_;
    p.batch.dict_n = dict_n_;
    p.prog = prog_;
    p.out.viol = viol;
    p.out.err = err;
    p.out.totals = totals;
    p.out.err_totals = err_totals;
    p.out.errlist = d_errlist_;
    p.out.errcount = reinterpret_cast<uint32_t*>(d_scalars_);
    p.out.errcap = err_cap_;
    p.out.words = db->words;
    p.active = d_active_;
    p.prog.ops = db->d_ops;      // slot ids resolved for this batch
    p.prog.pool = db->d_pool;
    p.prog.outs = db->d_outs;
    p.tile_lo = db->d_tile_lo;
    p.ntiles = db->ntiles;
    p.tile = db->tile;
    p.slot_words = db->slot_words;
    p.done_ctr = reinterpret_cast<uint32_t*>(d_scalars_) + 4;   // zeroed with the error counter before every launch
    p.done_target = 0;   // (set by fire())
    p.timing = nullptr;
    p.units = db->d_units;
    p.whole = db->d_whole;
    p.unit_count = db->d_whole + db->ntiles;
    p.list_mode = 0;
    if (spec_ready(db->n)) {   // (an NVRTC run the first time: here, outside the timed region)
      SpecEntry& se = *spec_cur_;
      // The generated kernel stages the largest tile's rows in shared memory: one bit per row per export plane of a scope that has
      // atoms, where the interpreter holds one bit per row per live slot.  A scope with many rows in a tile can therefore need more
      // than the device allows while the interpreter fits: that batch is interpreted.  So is a batch with a tile of more rows in a
      // nested scope than the offset image's 16-bit values hold.
      // (the rows read the batch's type words as the text lays them out: both come from gk_tw_layout over the same columns)
      if (!(se.src.tw == db->tw)) throw BackendError{"batch type words are laid out for another column table"};
      l.spec_smem = se.src.smem + se.src.stage_bytes(db->cap);
      bool run = l.spec_smem <= se.max_smem && se.src.image_fits(db->cap);
      l.spec_per_sm = 0;   // resident CTAs per SM: the persistent grid of fire()
      if (run && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&l.spec_per_sm, reinterpret_cast<const void*>(se.kern), se.threads, l.spec_smem) != cudaSuccess) {
        cudaGetLastError();
        l.spec_per_sm = spec_minb_;
      }
      l.spec_per_sm = std::max(1, l.spec_per_sm);
      // The hand-over plan depends on the batch's CSR offsets, which never change, and on the generated text: made by the first
      // evaluation of the batch with this constraint set, here, and kept, with its unit counts and the objects they cover on the host.
      // (It reads every offset array the netlist uses: at config 2 about as long as the interpreter's units take, so planning on
      // every evaluation would give back most of the overlap.)  The same pass writes the batch's offset image, which the tile kernel
      // stages instead of reading those arrays again.
      if (run && db->planned != se.version && p.ntiles) {
        db->img_stride = se.src.image_stride(db->cap);
        const size_t ib = (size_t)p.ntiles * db->img_stride * 2;
        if (ib > db->img_bytes) {
          CK(cudaStreamSynchronize(st));   // (an evaluation still in flight may be reading the old image)
          dfree(db->d_img);
          db->d_img = nullptr;
          db->img_bytes = 0;
          dmalloc(&db->d_img, ib);
          CK(cudaStreamSynchronize(stream_));
          db->img_bytes = ib;
        }
        if (getenv("GK_TRACE_LAUNCH"))
          fprintf(stderr, "[spec] offset image: %zu bytes, %u bytes per tile x %u tiles\n", ib, db->img_stride * 2, p.ntiles);
        CK(cudaMemsetAsync(p.unit_count, 0, 4, st));
        void* args[] = {&p, &db->d_img, &db->img_stride};
        CK(cudaLaunchKernel(reinterpret_cast<const void*>(se.plan_kern), dim3(p.ntiles), dim3(256), args, 0, st));
        ++launches_;
        CK(cudaMemcpyAsync(&db->nunits, p.unit_count, 4, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        std::vector<uint32_t> u((size_t)db->nunits * 2);
        if (db->nunits) CK(cudaMemcpy(u.data(), p.units, u.size() * 4, cudaMemcpyDeviceToHost));
        db->multi = 0;
        db->handed = 0;
        for (uint32_t i = 0; i < db->nunits; ++i) {
          db->multi += u[2 * i + 1] > 1u;
          db->handed += u[2 * i + 1];
        }
        db->planned = se.version;
      }
      // A batch the plan hands over whole (every tile has more wide objects than GK_HANDOVER_MAX) is the interpreter's alone: the
      // rows and tile kernels would evaluate every row for nothing.
      if (run && p.ntiles && db->handed >= db->n) run = false;
      // the export planes: scratch rewritten by every evaluation, grown (never shrunk) outside the timed region
      const size_t xb = se.src.export_bytes(db->rows);
      if (run && xb > spec_x_bytes_) {
        if (d_spec_x_) CK(cudaFree(d_spec_x_));
        d_spec_x_ = nullptr;
        spec_x_bytes_ = 0;
        CK(cudaMalloc(&d_spec_x_, xb));
        spec_x_bytes_ = xb;
        if (getenv("GK_TRACE_LAUNCH")) fprintf(stderr, "[spec] export arrays: %zu bytes for %u objects\n", xb, db->n);
      }
      if (run) {
        l.spec = &se;
        l.x = d_spec_x_;
        l.img = db->d_img;
        l.img_stride = db->img_stride;
        l.rows_grid = se.src.rows_blocks(db->rows, (uint32_t)se.rows_threads);
        l.units = db->nunits;
        l.multi = db->multi;
        l.handed = db->handed;
      }
    }
#ifdef GK_PHASE_TIMING
    if (!d_timing_) CK(cudaMalloc(&d_timing_, (kMaxPhases + 2 + 16) * 16));
    CK(cudaMemsetAsync(d_timing_, 0, (kMaxPhases + 2 + 16) * 16, st));
    p.timing = d_timing_;
#endif
    if (active.size() != C) throw BackendError{"active mask size mismatch"};
    if (db->words == 2 && ((reinterpret_cast<uintptr_t>(viol) | reinterpret_cast<uintptr_t>(err)) & 7u))
      throw BackendError{"result bitmaps must be 8-byte aligned (two-word rows are stored as one 64-bit word)"};
    if (C && active != last_active_) {
      CK(cudaMemcpyAsync(d_active_, active.data(), (size_t)C * 4, cudaMemcpyHostToDevice, st));
      CK(cudaStreamSynchronize(st));   // `active` is a caller temporary
      last_active_ = active;
    }
    if (C) CK(cudaMemsetAsync(totals, 0, (size_t)C * sizeof(unsigned long long), st));
    if (C) CK(cudaMemsetAsync(err_totals, 0, (size_t)C * sizeof(unsigned long long), st));
    CK(cudaMemsetAsync(d_scalars_, 0, 64, st));
    // the kernel carves its shared memory with the same call on the same parameters
    l.smem = gk_eval_layout(p.prog.nconstraints, p.batch.nscopes, p.prog.nphases, p.slot_words, p.prog.nops, p.prog.nitems, p.prog.nmatch,
                            p.batch.ncols, p.prog.npool, p.prog.ncbytes).total;
    if (l.smem > max_smem_)
      throw BackendError{"constraint set needs " + std::to_string(l.smem) + " bytes of shared memory per CTA (limit " + std::to_string(max_smem_) +
                         "): too many live netlist columns for one launch"};
    return l;
  }

  void fire(Launch l) {
    KParams& p = l.p;
    const size_t smem = l.smem;
    cudaStream_t st = l.st;
    if (p.ntiles == 0) return;
    // persistent CTAs: as many as fit per SM (shared-memory bound), each walks tiles with a grid stride
    int per_sm = 1;   // resident CTAs per SM for this launch configuration (registers and shared memory)
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gk_eval_kernel, kThreads, smem));
    per_sm = std::max(1, per_sm);
    if (getenv("GK_TRACE_LAUNCH")) fprintf(stderr, "[launch] %d CTAs/SM x %d threads, %zu B smem/CTA, %u tiles of %u objects\n", per_sm, kThreads, smem, p.ntiles, p.tile);
    uint32_t grid = std::max(1u, std::min<uint32_t>(p.ntiles, (uint32_t)(sms_ * per_sm)));
    last_kernel_ = "gk_eval_kernel";
    if (!l.spec) {
      p.done_target = grid;
      gk_eval_kernel<<<grid, kThreads, smem, st>>>(p);
      CK(cudaGetLastError());
      ++launches_;
      return;
    }
    // The kernel generated for this constraint set does the objects that fit its mask registers (all of them, normally); the
    // interpreter does the object ranges the plan lists (prepare()), on a side stream while the rows kernel streams the batch:
    //   st:    (memsets) fork -- rows kernel -- tile kernel -- wait(join)
    //   side:         wait(fork) -- interpreter, list mode -- join
    // The side stream has the higher priority, so that the interpreter's CTAs are placed at once instead of behind the rows
    // kernel's pending blocks.  Neither grid waits for the other on the device: the two write disjoint words, add into the same
    // totals, and in the fused exchange the last CTA of either publishes (done_target).  A batch without units launches no
    // interpreter at all.
    SpecEntry& se = *l.spec;
    const uint32_t spec_grid = std::max(1u, std::min<uint32_t>(p.ntiles, (uint32_t)(sms_ * l.spec_per_sm)));
    // the interpreter's persistent grid, each CTA striding over the list
    grid = std::max(1u, std::min<uint32_t>(p.batch.n, (uint32_t)(sms_ * per_sm)));
    p.list_mode = 1;
    p.done_target = spec_grid + (l.units ? grid : 0u);
    if (l.units) {
      CK(cudaEventRecord(ev_fork_, st));
      CK(cudaStreamWaitEvent(side_stream_, ev_fork_, 0));
      gk_eval_kernel<<<grid, kThreads, smem, side_stream_>>>(p);
      CK(cudaGetLastError());
      ++launches_;
      CK(cudaEventRecord(ev_fork_, side_stream_));   // (re-recorded as the join: the wait above already holds the fork)
    }
    void* args[] = {&p, &l.x, &l.img, &l.img_stride};
    // the rows kernel evaluates every row of the batch into the export arrays, one thread per row (its parameters: the first two)
    if (l.rows_grid) {
      void* rows_args[] = {&p, &l.x};
      CK(cudaLaunchKernel(reinterpret_cast<const void*>(se.rows_kern), dim3(l.rows_grid), dim3((unsigned)se.rows_threads), rows_args, 0, st));
      ++launches_;
    }
    // persistent CTAs, as many as are resident at once, walk the tiles with a grid stride: the per-CTA set-up (tables, enforcement
    // mask) is paid once per CTA, and where two or more are resident one CTA's copy overlaps another's object walk.  (Launched as the
    // rows kernel's programmatic dependent, so that this set-up overlaps the rows kernel's last blocks, it measured no faster.)
    CK(cudaLaunchKernel(reinterpret_cast<const void*>(se.kern), dim3(spec_grid), dim3((unsigned)se.threads), args, l.spec_smem, st));
    ++launches_;
    if (l.units) CK(cudaStreamWaitEvent(st, ev_fork_, 0));
    last_kernel_ = "gk_spec_kernel";
    if (getenv("GK_TRACE_LAUNCH"))
      fprintf(stderr, "[spec] handed to the interpreter: %u units (%llu of more than one object), %llu objects, on %u CTAs\n", l.units,
              (unsigned long long)l.multi, (unsigned long long)l.handed, grid);
  }

  // ---- the specialised kernel: source per constraint-set version (spec_codegen.cpp), compiled by NVRTC when first needed
  struct SpecEntry {
    uint64_t version = 0;
    SpecSource src;
    int state = 0;            // 0 = not compiled yet, 1 = ready, -1 = failed (the interpreter runs; reported once on stderr)
    cudaLibrary_t lib = nullptr;
    cudaKernel_t kern = nullptr;        // gk_spec_kernel
    cudaKernel_t rows_kern = nullptr;   // gk_spec_rows_kernel
    cudaKernel_t plan_kern = nullptr;   // gk_spec_plan_kernel
    int threads = 128, rows_threads = 256;
    size_t max_smem = 0;      // dynamic shared memory the kernel may be launched with (fixed part + the tile's staging area)
    double compile_ms = 0;
  };
  void spec_select(const Compiled& c) {
    spec_cur_ = nullptr;
    if (!spec_on_) return;
    for (auto it = spec_cache_.begin(); it != spec_cache_.end(); ++it)
      if (it->version == c.version) {
        spec_cache_.splice(spec_cache_.begin(), spec_cache_, it);
        spec_cur_ = &spec_cache_.front();
        return;
      }
    spec_cache_.emplace_front();
    spec_cache_.front().version = c.version;
    spec_cache_.front().src = spec_codegen(c);
    spec_cur_ = &spec_cache_.front();
    while (spec_cache_.size() > 8) {
      if (spec_cache_.back().lib) cudaLibraryUnload(spec_cache_.back().lib);
      spec_cache_.pop_back();
    }
  }
  bool spec_ready(uint32_t n) {
    if (!spec_cur_ || n < spec_min_objects_) return false;
    if (spec_cur_->state == 0) spec_compile(*spec_cur_);
    return spec_cur_->state == 1;
  }
  void spec_compile(SpecEntry& se) {
    se.state = -1;
    const auto t0 = std::chrono::steady_clock::now();
    try {
      // NVRTC is loaded at run time: the library itself links only the CUDA runtime (and loads in a container without a driver)
      typedef void* Prog;
      typedef int (*CreateFn)(Prog*, const char*, const char*, int, const char* const*, const char* const*);
      typedef int (*CompileFn)(Prog, int, const char* const*);
      typedef int (*SizeFn)(Prog, size_t*);
      typedef int (*GetFn)(Prog, char*);
      typedef int (*DestroyFn)(Prog*);
      static void* h = nullptr;
      if (!h) {
        for (const char* name : {"libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so"}) {
          h = dlopen(name, RTLD_NOW | RTLD_LOCAL);
          if (h) break;
        }
      }
      if (!h) throw BackendError{"libnvrtc.so.12 not found"};
      auto create = reinterpret_cast<CreateFn>(dlsym(h, "nvrtcCreateProgram"));
      auto compile = reinterpret_cast<CompileFn>(dlsym(h, "nvrtcCompileProgram"));
      auto log_size = reinterpret_cast<SizeFn>(dlsym(h, "nvrtcGetProgramLogSize"));
      auto get_log = reinterpret_cast<GetFn>(dlsym(h, "nvrtcGetProgramLog"));
      auto bin_size = reinterpret_cast<SizeFn>(dlsym(h, "nvrtcGetCUBINSize"));
      auto get_bin = reinterpret_cast<GetFn>(dlsym(h, "nvrtcGetCUBIN"));
      auto destroy = reinterpret_cast<DestroyFn>(dlsym(h, "nvrtcDestroyProgram"));
      if (!create || !compile || !log_size || !get_log || !bin_size || !get_bin || !destroy) throw BackendError{"NVRTC entry points missing"};
      Prog prog = nullptr;
      if (create(&prog, se.src.src.c_str(), "gk_spec_kernel.cu", 0, nullptr, nullptr) != 0) throw BackendError{"nvrtcCreateProgram failed"};
      const std::string threads = "-DGK_SPEC_THREADS=" + std::to_string(spec_threads_), minb = "-DGK_SPEC_MINB=" + std::to_string(spec_minb_),
                        rthreads = "-DGK_SPEC_ROWS_THREADS=" + std::to_string(spec_rows_threads_), rminb = "-DGK_SPEC_ROWS_MINB=" + std::to_string(spec_rows_minb_);
      std::vector<std::string> extra;   // GK_SPEC_DEFS="-DX -DY": measurement switches of the generated text
      if (const char* d = getenv("GK_SPEC_DEFS")) {
        std::istringstream in(d);
        std::string tok;
        while (in >> tok) extra.push_back(tok);
      }
      std::vector<const char*> opts = {"--gpu-architecture=sm_90a", "-std=c++17", "-lineinfo", "-default-device", threads.c_str(), minb.c_str(), rthreads.c_str(), rminb.c_str()};
      for (auto& x : extra) opts.push_back(x.c_str());
      const int rc = compile(prog, (int)opts.size(), opts.data());
      if (rc != 0) {
        size_t ls = 0;
        log_size(prog, &ls);
        std::string log(ls + 1, 0);
        if (ls) get_log(prog, &log[0]);
        destroy(&prog);
        throw BackendError{"NVRTC: " + log.substr(0, 2000)};
      }
      size_t bs = 0;
      bin_size(prog, &bs);
      std::vector<char> cubin(bs);
      get_bin(prog, cubin.data());
      destroy(&prog);
      CK(cudaLibraryLoadData(&se.lib, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0));
      CK(cudaLibraryGetKernel(&se.kern, se.lib, "gk_spec_kernel"));
      CK(cudaLibraryGetKernel(&se.rows_kern, se.lib, "gk_spec_rows_kernel"));
      CK(cudaLibraryGetKernel(&se.plan_kern, se.lib, "gk_spec_plan_kernel"));
      se.threads = spec_threads_;
      se.rows_threads = spec_rows_threads_;
      cudaFuncAttributes fa;
      CK(cudaFuncGetAttributes(&fa, reinterpret_cast<const void*>(se.kern)));
      se.max_smem = optin_smem_ - fa.sharedSizeBytes;
      CK(cudaFuncSetAttribute(reinterpret_cast<const void*>(se.kern), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)se.max_smem));
      se.state = 1;
    } catch (const BackendError& e) {
      fprintf(stderr, "[gatekeeper_b200] the kernel generated for constraint set %llu could not be built (%s): the netlist interpreter runs instead\n",
              (unsigned long long)se.version, e.msg.c_str());
    }
    se.compile_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (getenv("GK_TRACE_LAUNCH"))
      fprintf(stderr, "[spec] constraint set %llu: %zu bytes of source, %zu atoms as immediates / %zu generic, NVRTC %.0f ms, state %d; %s\n", (unsigned long long)se.version,
              se.src.src.size(), se.src.n_fast, se.src.n_generic, se.compile_ms, se.state, se.src.fold_text().c_str());
  }

  void eval(void* b, const std::vector<uint32_t>& active, EvalOut& out, bool copy_back) override {
    auto* db = static_cast<DevBatch*>(b);
    std::lock_guard<std::mutex> l(mu_);
    CK(cudaSetDevice(device_));
    const uint32_t C = prog_.nconstraints;
    out.n = db->n;
    out.nconstraints = C;
    out.words = db->words;
    unsigned long long* totals = d_totals_;
    unsigned long long* err_totals = d_totals_ + std::max(C, 1u);
    uint32_t nerr = 0;
    for (;;) {
      const Launch l = prepare(db, active, db->viol, db->err, totals, err_totals, stream_);
      CK(cudaStreamSynchronize(stream_));
      // the event pair brackets exactly the evaluation kernel
      CK(cudaEventRecord(ev0_, stream_));
      fire(l);
      CK(cudaEventRecord(ev1_, stream_));
      CK(cudaStreamSynchronize(stream_));
      CK(cudaMemcpy(&nerr, d_scalars_, 4, cudaMemcpyDeviceToHost));
      if (nerr <= err_cap_) break;
      // The kernels count every matcher error but store only the first err_cap_ (object, match block, code) triples.  The code of a
      // dropped one would be lost -- its autoreject message would carry no reason -- so the list grows to the count and the page is
      // evaluated again.  Rare (a namespaceSelector over ~a million objects without a cached Namespace), so it costs a normal
      // evaluation nothing.  eval_into() returns no list and needs no second pass.
      CK(cudaFree(d_errlist_));
      d_errlist_ = nullptr;
      err_cap_ = 0;   // (should the allocation fail, the kernels store nothing until a later evaluation grows the list)
      CK(cudaMalloc(&d_errlist_, (size_t)nerr * 3 * 4));
      err_cap_ = nerr;
    }
    CK(cudaEventElapsedTime(&out.kernel_ms, ev0_, ev1_));
#ifdef GK_PHASE_TIMING
    {
      std::vector<unsigned long long> t((kMaxPhases + 2 + 16) * 2);
      CK(cudaMemcpy(t.data(), d_timing_, t.size() * 8, cudaMemcpyDeviceToHost));
      unsigned long long tot = 0;
      for (uint32_t ph = 0; ph <= prog_.nphases; ++ph) tot += t[2 * ph];
      fprintf(stderr, "[phase timing] kernel %.3f ms, %u tiles\n", out.kernel_ms, db->ntiles);
      for (uint32_t ph = 0; ph <= prog_.nphases; ++ph)
        fprintf(stderr, "  %s %2u: %5.1f%% of CTA time, %7.0f cycles/tile, warp utilisation %4.1f%%\n", ph == prog_.nphases ? "gather" : "phase ", ph,
                100.0 * t[2 * ph] / std::max(1ull, tot), (double)t[2 * ph] / std::max(1u, db->ntiles),
                100.0 * t[2 * ph + 1] / std::max(1.0, (double)t[2 * ph] * kWarps));
      const char* kn[] = {"", "", "atom", "gate", "const", "bcast", "acc", "match", "atoms", "atoms(head)"};
      for (uint32_t k = 2; k < 10; ++k) {
        const unsigned long long cyc = t[2 * (kMaxPhases + 2) + 2 * k], cnt = t[2 * (kMaxPhases + 2) + 2 * k + 1];
        if (cnt) fprintf(stderr, "  items %-11s: %6.1f per tile, %7.0f cycles each, %8.0f warp-cycles per tile\n", kn[k], (double)cnt / db->ntiles,
                         (double)cyc / cnt, (double)cyc / db->ntiles);
      }
    }
#endif
    out.launches = launches_;
    out.totals.assign(C, 0);
    out.err_totals.assign(C, 0);
    if (C) {
      std::vector<unsigned long long> t(2 * (size_t)std::max(C, 1u));
      CK(cudaMemcpy(t.data(), d_totals_, t.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
      for (uint32_t c = 0; c < C; ++c) {
        out.totals[c] = t[c];
        out.err_totals[c] = t[std::max(C, 1u) + c];
      }
    }
    out.errlist.resize((size_t)nerr * 3);
    if (nerr) CK(cudaMemcpy(out.errlist.data(), d_errlist_, (size_t)nerr * 12, cudaMemcpyDeviceToHost));
    if (copy_back) copy_planes(*db, out);
  }

  // a batch's result planes into `out`
  void copy_planes(const DevBatch& db, EvalOut& out) {
    out.viol.resize((size_t)db.n * db.words);
    out.err.resize((size_t)db.n * db.words);
    if (!db.n) return;
    CK(cudaMemcpyAsync(out.viol.data(), db.viol, out.viol.size() * 4, cudaMemcpyDeviceToHost, stream_));
    CK(cudaMemcpyAsync(out.err.data(), db.err, out.err.size() * 4, cudaMemcpyDeviceToHost, stream_));
    CK(cudaStreamSynchronize(stream_));
  }

  // ---- device ingest (ingest_core.h / ingest_kernels.cuh): raw JSON blob -> resident columnar batch
  struct Scratch {   // grow-only device buffer
    uint8_t* p = nullptr;
    size_t cap = 0;
    uint8_t* need(size_t bytes) {
      if (bytes > cap) {
        if (p) cudaFree(p);
        p = nullptr;
        cap = bytes + (bytes >> 3) + 4096;
        cudaError_t e = cudaMalloc(&p, cap);
        if (e != cudaSuccess) {
          cap = 0;
          throw BackendError{std::string("CUDA error: ") + cudaGetErrorString(e) + " allocating ingest scratch"};
        }
      }
      return p;
    }
  };
  struct Carver {   // 256-byte aligned sub-allocations of one buffer
    size_t off = 0;
    size_t take(size_t bytes) {
      size_t o = gk_align(off);
      off = o + std::max<size_t>(bytes, 16);
      return o;
    }
  };

  void upload_htab(const HashTabHost& h, unsigned long long** dk, uint32_t** dv, size_t* dcap) {
    const size_t cap = (size_t)h.mask + 1;
    if (*dcap != cap) {
      if (*dk) cudaFree(*dk);
      if (*dv) cudaFree(*dv);
      CK(cudaMalloc(dk, cap * 8));
      CK(cudaMalloc(dv, cap * 4));
      *dcap = cap;
    }
    CK(cudaMemcpyAsync(*dk, h.keys.data(), cap * 8, cudaMemcpyHostToDevice, stream_));
    CK(cudaMemcpyAsync(*dv, h.vals.data(), cap * 4, cudaMemcpyHostToDevice, stream_));
    CK(cudaStreamSynchronize(stream_));
  }

  // A page's device JSON, offsets and token tape, kept for reextract(): the allocation of the front buffer the page was ingested
  // from, which start_front never hands out again (the front allocates a new one).
  struct KeptSource {
    uint8_t* buf = nullptr;
    GkIngestIn in{};                 // blob / ooff / tape / ntape / status pointers into buf, n
    unsigned long long bytes = 0;    // the page's JSON bytes
    ~KeptSource() {
      if (buf) cudaFree(buf);
    }
  };

  void* ingest(const IngestReq& rq, IngestStats* st, std::vector<uint32_t>* status) override { return ingest_page(rq, st, status, nullptr); }
  void* ingest_keep(const IngestReq& rq, IngestStats* st, std::vector<uint32_t>* status, void** keep) override { return ingest_page(rq, st, status, keep); }

  // copy (or take the prefetched copy) and tokenise, then extract; with `keep`, the batch's caller receives the front buffer
  void* ingest_page(const IngestReq& rq, IngestStats* st, std::vector<uint32_t>* status, void** keep) {
    std::lock_guard<std::mutex> l(ingest_mu_);
    CK(cudaSetDevice(device_));
    std::unique_ptr<KeptSource> ks;
    // the front buffer (blob, offsets, tape): the prefetched copy of this page, or copy + tokenise now
    auto acquire = [&]() {
      Front* fr = nullptr;
      {
        std::lock_guard<std::mutex> fl(front_mu_);
        for (auto& f : fronts_)
          if (f.pending && f.host_blob == rq.blob && f.n == rq.n) fr = &f;   // (prefetched)
        if (!fr) fr = &start_front(rq.blob, rq.ooff, rq.n);
        fr->pending = false;
        if (keep) {
          ks.reset(new KeptSource());
          ks->buf = fr->buf.p;
          ks->in = fr->in;
          ks->bytes = rq.ooff[rq.n];
          fr->buf = Scratch{};
        }
      }
      CK(cudaStreamWaitEvent(stream_, fr->done, 0));
      return fr->in;
    };
    void* db = extract(rq, acquire, rq.ooff[rq.n], true, st, status);
    if (keep) *keep = ks.release();
    return db;
  }

  void* reextract(void* source, const IngestReq& rq, IngestStats* st, std::vector<uint32_t>* status) override {
    std::lock_guard<std::mutex> l(ingest_mu_);
    CK(cudaSetDevice(device_));
    auto* ks = static_cast<KeptSource*>(source);
    if (!ks || ks->in.n != rq.n) throw BackendError{"device ingest: the kept source is of another page"};
    if (getenv("GK_TRACE_LAUNCH")) fprintf(stderr, "[launch] extraction of %u objects from the kept source: no copy, no tokeniser\n", ks->in.n);
    return extract(rq, [ks]() { return ks->in; }, ks->bytes, false, st, status);
  }

  // A new page from a kept one (gk_batch_patch): the staying objects' offsets by one scan over their lengths, their JSON, tape,
  // tape lengths and status words moved by gk_splice_kernel, then the added documents copied and tokenised into the tail by the
  // front buffer's code.  Nothing of the old page is changed; it is freed by its owner.
  void* patch_source(void* source, const std::vector<uint32_t>& keep, const uint8_t* blob, const unsigned long long* ooff, size_t n_add,
                     IngestStats* st) override {
    std::lock_guard<std::mutex> l(ingest_mu_);
    CK(cudaSetDevice(device_));
    auto* old = static_cast<KeptSource*>(source);
    if (!old) throw BackendError{"kept source: none"};
    const uint32_t nk = (uint32_t)keep.size();
    if ((uint64_t)nk + n_add > 0x7fffff00ull) throw BackendError{"device ingest: more than 2^31 objects in one batch"};
    const uint32_t n = nk + (uint32_t)n_add;
    const unsigned long long add_bytes = n_add ? ooff[n_add] - ooff[0] : 0ull;
    Event e0, e1;
    CK(cudaEventRecord(e0, stream_));
    // ---- the staying objects' new offsets, and their bytes' total
    Temps temps(this);
    auto* d_keep = temps.take<uint32_t>((size_t)nk * 4 + 4);
    auto* d_len = temps.take<unsigned long long>(((size_t)nk + 1) * 8);
    auto* d_off = temps.take<unsigned long long>(((size_t)nk + 1) * 8);
    if (nk) CK(cudaMemcpyAsync(d_keep, keep.data(), (size_t)nk * 4, cudaMemcpyHostToDevice, stream_));
    gk_keep_len_kernel<<<(nk + 1 + 255) / 256, 256, 0, stream_>>>(old->in.ooff, d_keep, nk, d_len);
    size_t scan_bytes = 0;
    CK(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, d_len, d_off, (int64_t)nk + 1, stream_));
    CK(cub::DeviceScan::ExclusiveSum(temps.take(scan_bytes), scan_bytes, d_len, d_off, (int64_t)nk + 1, stream_));
    launches_ += 2;
    unsigned long long kept_bytes = 0;
    CK(cudaMemcpyAsync(&kept_bytes, d_off + nk, 8, cudaMemcpyDeviceToHost, stream_));
    CK(cudaStreamSynchronize(stream_));
    CK(cudaGetLastError());
    // ---- the new page: staying objects first, then the added ones
    const unsigned long long B = kept_bytes + add_bytes;
    const PageLayout lay(B, n);
    auto ks = std::make_unique<KeptSource>();
    CK(cudaMalloc(&ks->buf, lay.total));
    ks->in = lay.at(ks->buf);
    ks->bytes = B;
    uint8_t* d_ooff = ks->buf + lay.o_ooff;
    CK(cudaMemcpyAsync(d_ooff, d_off, ((size_t)nk + 1) * 8, cudaMemcpyDeviceToDevice, stream_));
    if (n_add) {
      std::vector<unsigned long long> tail(n_add);
      for (size_t k = 0; k < n_add; ++k) tail[k] = kept_bytes + (ooff[k + 1] - ooff[0]);
      CK(cudaMemcpyAsync(d_ooff + ((size_t)nk + 1) * 8, tail.data(), n_add * 8, cudaMemcpyHostToDevice, stream_));
    }
    CK(cudaMemsetAsync(ks->buf + lay.o_blob + B, 0, 16, stream_));
    if (nk) {
      gk_splice_kernel<<<std::min<uint32_t>((nk + 7) / 8, (uint32_t)sms_ * 16), 256, 0, stream_>>>(ks->in, ks->buf + lay.o_blob, old->in, d_keep, nk);
      ++launches_;
    }
    if (getenv("GK_TRACE_LAUNCH")) fprintf(stderr, "[launch] gk_splice_kernel over %u staying objects, %llu bytes\n", nk, kept_bytes);
    Event spliced;
    CK(cudaEventRecord(spliced, stream_));
    {
      std::lock_guard<std::mutex> fl(front_mu_);
      CK(cudaStreamWaitEvent(copy_stream_, spliced, 0));   // (the tail's offsets are in place)
      copy_and_tokenise(ks->in, ks->buf + lay.o_blob + kept_bytes, nk, blob, ooff, (uint32_t)n_add);
      cudaEvent_t done = chunk_event(0);
      CK(cudaEventRecord(done, front_stream_));
      CK(cudaStreamWaitEvent(stream_, done, 0));
    }
    CK(cudaEventRecord(e1, stream_));
    CK(cudaStreamSynchronize(stream_));   // (the temporaries are freed on stream_ and the caller's page may change once this returns)
    CK(cudaGetLastError());
    if (st) {
      float ms = 0;
      cudaEventElapsedTime(&ms, e0, e1);
      st->h2d_ms = ms;   // splice, copy and tokeniser
      st->h2d_bytes = add_bytes + (n_add + (size_t)nk) * 8;
      st->launches = launches_;
    }
    return ks.release();
  }

  void source_bytes(void* source, const std::vector<uint32_t>& idx, std::string& bytes, std::vector<uint64_t>& off) override {
    std::lock_guard<std::mutex> l(ingest_mu_);
    CK(cudaSetDevice(device_));
    auto* ks = static_cast<KeptSource*>(source);
    if (!ks) throw BackendError{"kept source: none"};
    std::vector<unsigned long long> ooff((size_t)ks->in.n + 1);
    CK(cudaMemcpy(ooff.data(), ks->in.ooff, ooff.size() * 8, cudaMemcpyDeviceToHost));
    std::vector<unsigned long long> spans;
    off.assign(1, 0);
    for (uint32_t i : idx) {
      if (i >= ks->in.n) throw BackendError{"kept source: object index out of range"};
      const unsigned long long len = ooff[i + 1] - ooff[i];
      spans.insert(spans.end(), {ooff[i], (unsigned long long)off.back(), len});
      off.push_back(off.back() + len);
    }
    bytes.assign((size_t)off.back(), '\0');
    const uint32_t nspans = (uint32_t)(spans.size() / 3);
    if (!nspans || bytes.empty()) return;
    Temps temps(this);
    auto* d_spans = temps.take<unsigned long long>(spans.size() * 8);
    auto* d_out = temps.take<uint8_t>(bytes.size());
    CK(cudaMemcpyAsync(d_spans, spans.data(), spans.size() * 8, cudaMemcpyHostToDevice, stream_));
    gk_gather_kernel<<<std::min<uint32_t>(nspans, 4096u), 128, 0, stream_>>>(d_out, ks->in.blob, d_spans, nspans);
    ++launches_;
    CK(cudaMemcpyAsync(&bytes[0], d_out, bytes.size(), cudaMemcpyDeviceToHost, stream_));
    CK(cudaStreamSynchronize(stream_));
    CK(cudaGetLastError());
  }

  void release_source(void* source) override {
    if (!source) return;
    cudaSetDevice(device_);
    delete static_cast<KeptSource*>(source);
  }

  // The extraction half of the device ingest: header, scope, column, byte-column and tile passes over the front buffer `acquire`
  // makes ready on stream_ (its tokeniser finished).  `B`: the page's JSON bytes; `copied`: this call moved the page to the device.
  void* extract(const IngestReq& rq, const std::function<GkIngestIn()>& acquire, unsigned long long B, bool copied, IngestStats* st,
                std::vector<uint32_t>* status) {
    const auto T0 = std::chrono::steady_clock::now();
    const XProgHost& xh = *rq.xprog;
    const Compiled& c = *rq.c;
    const uint32_t n = (uint32_t)rq.n, NS = (uint32_t)xh.scopes.size(), NK = xh.ncounters(), NC = (uint32_t)xh.cols.size();
    if (rq.n > 0x7fffff00ull) throw BackendError{"device ingest: more than 2^31 objects in one batch"};
    // ---- lookup tables
    if (sid_.nstrings != rq.strings->size()) {
      build_sid_table(*rq.strings, sid_);
      upload_htab(sid_.tab, &d_sid_keys_, &d_sid_vals_, &d_sid_cap_);
    }
    if (lut_.mask == 0) {
      lut_.init(1u << 20);
      upload_htab(lut_, &d_lut_keys_, &d_lut_vals_, &d_lut_cap_);
    }
    // ---- extraction program + namespace cache tables: one host image, one copy
    std::vector<uint32_t> xkeys = xh.xkeys;
    std::vector<uint8_t> xbytes = xh.xbytes;
    const uint32_t excl_off = (uint32_t)xkeys.size();
    uint32_t excl_n = 0;
    for (auto& pat : rq.excluded) {
      const bool pre = !pat.empty() && pat.front() == '*', suf = pat.size() > (pre ? 1u : 0u) && pat.back() == '*';
      const std::string core = pat.substr(pre ? 1 : 0, pat.size() - (pre ? 1 : 0) - (suf ? 1 : 0));
      xkeys.push_back(pre && suf ? GK_W_CONTAINS : pre ? GK_W_SUFFIX : suf ? GK_W_PREFIX : GK_W_EXACT);
      xkeys.push_back((uint32_t)xbytes.size());
      xkeys.push_back((uint32_t)core.size());
      xbytes.insert(xbytes.end(), core.begin(), core.end());
      ++excl_n;
    }
    const NsTableHost& ns = *rq.ns;
    Carver tc;
    const size_t o_cl = tc.take(xh.cl.size() * sizeof(GkXClosure)), o_cols = tc.take(xh.cols.size() * sizeof(GkXCol)),
                 o_scopes = tc.take(xh.scopes.size() * sizeof(GkXScope)), o_order = tc.take(xh.col_order.size() * 4), o_xkeys = tc.take(xkeys.size() * 4),
                 o_xargs = tc.take(xh.xargs.size() * 4), o_xbytes = tc.take(xbytes.size()), o_nskeys = tc.take(ns.tab.keys.size() * 8),
                 o_nsvals = tc.take(ns.tab.vals.size() * 4), o_nsnoff = tc.take(ns.nsn_off.size() * 4), o_nsnbytes = tc.take(ns.nsn_bytes.size());
    const size_t tab_bytes = gk_align(tc.off);
    std::vector<uint8_t> timg(tab_bytes, 0);
    auto putv = [&](size_t off, const void* src, size_t bytes) {
      if (bytes) memcpy(timg.data() + off, src, bytes);
    };
    putv(o_cl, xh.cl.data(), xh.cl.size() * sizeof(GkXClosure));
    putv(o_cols, xh.cols.data(), xh.cols.size() * sizeof(GkXCol));
    putv(o_scopes, xh.scopes.data(), xh.scopes.size() * sizeof(GkXScope));
    putv(o_order, xh.col_order.data(), xh.col_order.size() * 4);
    putv(o_xkeys, xkeys.data(), xkeys.size() * 4);
    putv(o_xargs, xh.xargs.data(), xh.xargs.size() * 4);
    putv(o_xbytes, xbytes.data(), xbytes.size());
    putv(o_nskeys, ns.tab.keys.data(), ns.tab.keys.size() * 8);
    putv(o_nsvals, ns.tab.vals.data(), ns.tab.vals.size() * 4);
    putv(o_nsnoff, ns.nsn_off.data(), ns.nsn_off.size() * 4);
    putv(o_nsnbytes, ns.nsn_bytes.data(), ns.nsn_bytes.size());
    uint8_t* d_tab = tabs_.need(tab_bytes);
    push_small(d_tab, timg.data(), tab_bytes);
    GkXProg xp;
    memset(&xp, 0, sizeof xp);
    xp.cl = reinterpret_cast<const GkXClosure*>(d_tab + o_cl);
    xp.cols = reinterpret_cast<const GkXCol*>(d_tab + o_cols);
    xp.scopes = reinterpret_cast<const GkXScope*>(d_tab + o_scopes);
    xp.col_order = reinterpret_cast<const uint32_t*>(d_tab + o_order);
    xp.xkeys = reinterpret_cast<const uint32_t*>(d_tab + o_xkeys);
    xp.xargs = reinterpret_cast<const uint32_t*>(d_tab + o_xargs);
    xp.xbytes = d_tab + o_xbytes;
    xp.ncl = (uint32_t)xh.cl.size();
    xp.ncols = NC;
    xp.nscopes = NS;
    xp.nbytecols = xh.nbytecols;
    xp.sid_tab.keys = d_sid_keys_;
    xp.sid_tab.vals = d_sid_vals_;
    xp.sid_tab.mask = sid_.tab.mask;
    xp.sid_true = sid_.sid_true;
    xp.sid_false = sid_.sid_false;
    xp.sid_null = sid_.sid_null;
    xp.ns_tab.keys = reinterpret_cast<unsigned long long*>(d_tab + o_nskeys);
    xp.ns_tab.vals = reinterpret_cast<uint32_t*>(d_tab + o_nsvals);
    xp.ns_tab.mask = ns.tab.mask;
    xp.nsn_off = reinterpret_cast<const uint32_t*>(d_tab + o_nsnoff);
    xp.nsn_bytes = d_tab + o_nsnbytes;
    xp.excl_off = excl_off;
    xp.excl_n = excl_n;
    uint32_t clanes = 1;
    if (const char* ev = getenv("GK_INGEST_COL_LANES")) clanes = std::max(1, std::min(32, atoi(ev)));
    while (clanes & (clanes - 1)) --clanes;
    Event e0, e1, e2, e3;
    CK(cudaEventRecord(e0, stream_));
    const GkIngestIn src = acquire();
    // ---- back scratch: header counters + scratch flags, totals, scan block sums, miss list, the pointer tables of the count phase
    const uint32_t miss_cap = 1u << 17;
    const uint32_t NT = GK_CNT_EXTRA + NS + xh.nbytecols + 4;          // totals: header counters, scopes, byte columns
    Carver sc;
    const size_t o_counts = sc.take((size_t)GK_CNT_EXTRA * n * 4 + 16), o_flags = sc.take((size_t)n * 4 + 16), o_totals = sc.take((size_t)(NT + NS + 4) * 4),
                 o_sums = sc.take((size_t)NT * 4096 * 4), o_miss = sc.take((size_t)miss_cap * sizeof(GkMiss)), o_fill = sc.take((size_t)miss_cap * 8),
                 o_prec = sc.take((size_t)NS * 8);
    uint8_t* d_s = scratch_.need(gk_align(sc.off));
    GkIngestIn in = src;
    in.source = rq.source;
    in.counts = reinterpret_cast<uint32_t*>(d_s + o_counts);
    in.misses = reinterpret_cast<GkMiss*>(d_s + o_miss);
    uint32_t* d_totals = reinterpret_cast<uint32_t*>(d_s + o_totals);   // [0,4) header, [4, 4+NS) scopes, then byte columns
    uint32_t* d_cap = d_totals + NT;
    in.nmiss = d_cap + NS;
    in.miss_cap = miss_cap;
    uint32_t* d_fill = reinterpret_cast<uint32_t*>(d_s + o_fill);
    uint32_t* d_sums = reinterpret_cast<uint32_t*>(d_s + o_sums);
    // exclusive scan of a[0..len) in place (+ a[len] = total when `tail`), total also at d_totals[slot]
    auto scan = [&](uint32_t* a, uint32_t len, uint32_t slot, bool tail) {
      const uint32_t nb = (len + kScanBlock - 1) / kScanBlock;
      if (nb > 4096) throw BackendError{"device ingest: more than 16M rows in one scope of one batch"};
      uint32_t* sums = d_sums + (size_t)slot * 4096;
      if (nb) gk_scan_sums_kernel<<<nb, kScanThreads, 0, stream_>>>(a, len, sums);
      gk_scan_top_kernel<<<1, kScanThreads, 0, stream_>>>(sums, nb, d_totals + slot);
      if (nb) gk_scan_apply_kernel<<<nb, kScanThreads, 0, stream_>>>(a, len, sums, d_totals + slot, tail ? 1u : 0u);
      else if (tail) CK(cudaMemsetAsync(a, 0, 4, stream_));
      launches_ += nb ? 3 : 1;
    };
    auto blocks = [](uint32_t rows) { return (rows + kIngestThreads - 1) / kIngestThreads; };
    // the count phase works on scratch: flags, CSR offsets (= scanned member counts), generator nodes, row handles, byte lengths
    GkIngestOut outc;
    memset(&outc, 0, sizeof outc);
    outc.flags = reinterpret_cast<uint32_t*>(d_s + o_flags);
    outc.row_rec = reinterpret_cast<GkRowRec* const*>(d_s + o_prec);
    std::vector<uint64_t> h_prec(NS, 0);
    std::vector<uint32_t*> d_cnt(NS, nullptr), d_coll(NS, nullptr), d_blen(xh.nbytecols, nullptr);
    Temps temps(this);
    CK(cudaEventRecord(e1, stream_));
    std::vector<uint32_t> total(NS, 0), htot(GK_CNT_EXTRA, 0), btot(xh.nbytecols, 0);
    total[0] = n;
    if (n) {
      gk_hcount_kernel<<<blocks(n), kIngestThreads, 0, stream_>>>(xp, in, outc);
      ++launches_;
      for (uint32_t k = 0; k < GK_CNT_EXTRA; ++k) scan(in.counts + (size_t)k * n, n, k, false);
      // scopes, one depth level at a time (the rows of a level size the kernels of the next)
      uint32_t maxd = 0;
      std::vector<uint32_t> depth(NS, 0);
      for (uint32_t s2 = 1; s2 < NS; ++s2) depth[s2] = depth[xh.scopes[s2].parent] + 1, maxd = std::max(maxd, depth[s2]);
      std::vector<uint32_t> hbuf(NT, 0);
      for (uint32_t d = 1; d <= maxd; ++d) {
        for (uint32_t t = 1; t < NS; ++t) {
          if (depth[t] != d) continue;
          const uint32_t prows = total[xh.scopes[t].parent];
          d_cnt[t] = temps.take<uint32_t>(((size_t)prows + 1) * 4);
          d_coll[t] = temps.take<uint32_t>(((size_t)prows + 1) * 4);
          if (prows) {
            gk_scope_count_kernel<<<blocks(prows), kIngestThreads, 0, stream_>>>(xp, in, outc, t, prows, d_cnt[t], d_coll[t]);
            ++launches_;
          }
          scan(d_cnt[t], prows, GK_CNT_EXTRA + t, true);
        }
        CK(cudaMemcpyAsync(hbuf.data(), d_totals, (size_t)NT * 4, cudaMemcpyDeviceToHost, stream_));
        CK(cudaStreamSynchronize(stream_));
        CK(cudaGetLastError());
        bool any = false;
        for (uint32_t t = 1; t < NS; ++t) {
          if (depth[t] != d) continue;
          total[t] = hbuf[GK_CNT_EXTRA + t];
          h_prec[t] = reinterpret_cast<uint64_t>(temps.take(((size_t)total[t] + 1) * sizeof(GkRowRec)));
          any = true;
        }
        if (!any) continue;
        push_small(d_s + o_prec, h_prec.data(), (size_t)NS * 8);
        for (uint32_t t = 1; t < NS; ++t) {
          if (depth[t] != d) continue;
          const uint32_t prows = total[xh.scopes[t].parent];
          if (!prows || !total[t]) continue;
          gk_scope_fill_kernel<<<blocks(prows), kIngestThreads, 0, stream_>>>(xp, in, outc, t, prows, d_cnt[t], d_coll[t]);
          ++launches_;
        }
      }
      // byte-encoded columns: decoded length per row -> offsets
      for (uint32_t ci = 0; ci < NC; ++ci) {
        const GkXCol& xc = xh.cols[ci];
        if (!(xc.enc & GK_ENC_BYTES)) continue;
        const uint32_t rows = total[xc.scope];
        d_blen[xc.bytes_slot] = temps.take<uint32_t>(((size_t)rows + 1) * 4);
        if (rows) {
          gk_bcol_len_kernel<<<blocks(rows), kIngestThreads, 0, stream_>>>(xp, in, outc, ci, rows, d_blen[xc.bytes_slot]);
          ++launches_;
        }
        scan(d_blen[xc.bytes_slot], rows, GK_CNT_EXTRA + NS + xc.bytes_slot, true);
      }
      CK(cudaMemcpyAsync(hbuf.data(), d_totals, (size_t)NT * 4, cudaMemcpyDeviceToHost, stream_));
      CK(cudaStreamSynchronize(stream_));
      CK(cudaGetLastError());
      for (uint32_t k = 0; k < GK_CNT_EXTRA; ++k) htot[k] = hbuf[k];
      for (uint32_t k = 0; k < xh.nbytecols; ++k) btot[k] = hbuf[GK_CNT_EXTRA + NS + k];
    }
    // ---- destination arena (exact sizes) + the pointer tables of the write pass
    Carver ac;
    GkBatch h;
    memset(&h, 0, sizeof h);
    h.n = n;
    h.has_old = 0;
    uint64_t alg = 0;
    auto arr = [&](size_t bytes) {
      alg += bytes;
      return ac.take(bytes);
    };
    const size_t a_flags = arr((size_t)n * 4), a_kind = arr((size_t)n * 4), a_group = arr((size_t)n * 4), a_nsnoff = arr(((size_t)n + 1) * 4),
                 a_nsnb = arr(htot[3]), a_nameoff = arr(((size_t)n + 1) * 4), a_nameb = arr(htot[0]), a_genoff = arr(((size_t)n + 1) * 4),
                 a_genb = arr(htot[1]), a_lbloff = arr(((size_t)n + 1) * 4), a_lblkv = arr((size_t)htot[2] * 8), a_nsrow = arr((size_t)n * 4),
                 a_nsloff = arr(ns.nsl_off.size() * 4), a_nslkv = arr(ns.nsl_kv.size() * 4);
    std::vector<size_t> a_scope(NS, 0);
    for (uint32_t s2 = 1; s2 < NS; ++s2) a_scope[s2] = arr(((size_t)total[xh.scopes[s2].parent] + 1) * 4);
    struct ColOff {
      size_t vt = 0, sid = 0, num = 0, boff = 0, bytes = 0, head = 0;
    };
    std::vector<ColOff> a_col(NC);
    for (uint32_t ci = 0; ci < NC; ++ci) {
      const GkXCol& xc = xh.cols[ci];
      const size_t rows = total[xc.scope];
      if (xc.enc & GK_ENC_VT) a_col[ci].vt = arr(rows);
      if (xc.enc & GK_ENC_SID) a_col[ci].sid = arr(rows * 4);
      if (xc.enc & GK_ENC_NUM) a_col[ci].num = arr(rows * 8);
      if (xc.enc & GK_ENC_HEAD) a_col[ci].head = arr(rows * 32);
      if (xc.enc & GK_ENC_BYTES) {
        a_col[ci].boff = arr((rows + 1) * 4);
        a_col[ci].bytes = arr(btot[xc.bytes_slot]);
      }
    }
    // in-arena tables: GkColumn[], GkScope[], and the pointer arrays of GkIngestOut
    const size_t a_cols = ac.take((size_t)NC * sizeof(GkColumn)), a_scopes = ac.take((size_t)NS * sizeof(GkScope)), a_pscope = ac.take((size_t)NS * 8),
                 a_pvt = ac.take((size_t)NC * 8), a_psid = ac.take((size_t)NC * 8), a_pnum = ac.take((size_t)NC * 8), a_pboff = ac.take((size_t)NC * 8),
                 a_pbytes = ac.take((size_t)NC * 8), a_phead = ac.take((size_t)NC * 8);
    const size_t tables_lo = gk_align(a_cols) == a_cols ? a_cols : a_cols;
    auto* db = new DevBatch();
    std::unique_ptr<DevBatch, std::function<void(DevBatch*)>> guard(db, [this](DevBatch* x) { release(x); });
    db->bytes = gk_align(ac.off);
    db->n = n;
    db->rows = total;
    db->rows[0] = n;
    db->prog_version = c.version;
    dmalloc(&db->arena, db->bytes);
    uint8_t* A = db->arena;
    std::vector<uint8_t> aimg(db->bytes - tables_lo, 0);   // host image of the table tail of the arena
    auto tail = [&](size_t off) { return aimg.data() + (off - tables_lo); };
    GkColumn* hc = reinterpret_cast<GkColumn*>(tail(a_cols));
    GkScope* hs = reinterpret_cast<GkScope*>(tail(a_scopes));
    auto dptr = [&](size_t off) { return reinterpret_cast<uint64_t>(A + off); };
    for (uint32_t ci = 0; ci < NC; ++ci) {
      const GkXCol& xc = xh.cols[ci];
      GkColumn& g = hc[ci];
      g.scope = (int32_t)xc.scope;
      g.enc = xc.enc;
      g.vt = (xc.enc & GK_ENC_VT) ? A + a_col[ci].vt : nullptr;
      g.sid = (xc.enc & GK_ENC_SID) ? reinterpret_cast<const uint32_t*>(A + a_col[ci].sid) : nullptr;
      g.num = (xc.enc & GK_ENC_NUM) ? reinterpret_cast<const int64_t*>(A + a_col[ci].num) : nullptr;
      g.boff = (xc.enc & GK_ENC_BYTES) ? reinterpret_cast<const uint32_t*>(A + a_col[ci].boff) : nullptr;
      g.bytes = (xc.enc & GK_ENC_BYTES) ? A + a_col[ci].bytes : nullptr;
      g.head = (xc.enc & GK_ENC_HEAD) ? reinterpret_cast<const uint32_t*>(A + a_col[ci].head) : nullptr;
      reinterpret_cast<uint64_t*>(tail(a_pvt))[ci] = g.vt ? dptr(a_col[ci].vt) : 0;
      reinterpret_cast<uint64_t*>(tail(a_psid))[ci] = g.sid ? dptr(a_col[ci].sid) : 0;
      reinterpret_cast<uint64_t*>(tail(a_pnum))[ci] = g.num ? dptr(a_col[ci].num) : 0;
      reinterpret_cast<uint64_t*>(tail(a_pboff))[ci] = g.boff ? dptr(a_col[ci].boff) : 0;
      reinterpret_cast<uint64_t*>(tail(a_pbytes))[ci] = g.bytes ? dptr(a_col[ci].bytes) : 0;
      reinterpret_cast<uint64_t*>(tail(a_phead))[ci] = g.head ? dptr(a_col[ci].head) : 0;
    }
    for (uint32_t s2 = 0; s2 < NS; ++s2) {
      hs[s2].parent = s2 ? xh.scopes[s2].parent : 0;
      hs[s2].rows = s2 ? total[s2] : n;
      hs[s2].off = s2 ? reinterpret_cast<const uint32_t*>(A + a_scope[s2]) : nullptr;
      reinterpret_cast<uint64_t*>(tail(a_pscope))[s2] = s2 ? dptr(a_scope[s2]) : 0;
    }
    push_small(A + tables_lo, aimg.data(), aimg.size());
    push_small(A + a_nsloff, ns.nsl_off.data(), ns.nsl_off.size() * 4);
    push_small(A + a_nslkv, ns.nsl_kv.data(), ns.nsl_kv.size() * 4);
    h.flags = reinterpret_cast<const uint32_t*>(A + a_flags);
    h.kind_sid = reinterpret_cast<const uint32_t*>(A + a_kind);
    h.group_sid = reinterpret_cast<const uint32_t*>(A + a_group);
    h.nsn_off = reinterpret_cast<const uint32_t*>(A + a_nsnoff);
    h.nsn_bytes = A + a_nsnb;
    h.name_off = reinterpret_cast<const uint32_t*>(A + a_nameoff);
    h.name_bytes = A + a_nameb;
    h.gen_off = reinterpret_cast<const uint32_t*>(A + a_genoff);
    h.gen_bytes = A + a_genb;
    h.lbl_off = reinterpret_cast<const uint32_t*>(A + a_lbloff);
    h.lbl_kv = reinterpret_cast<const uint32_t*>(A + a_lblkv);
    h.nsrow = reinterpret_cast<const uint32_t*>(A + a_nsrow);
    h.nsl_off = reinterpret_cast<const uint32_t*>(A + a_nsloff);
    h.nsl_kv = reinterpret_cast<const uint32_t*>(A + a_nslkv);
    h.cols = reinterpret_cast<const GkColumn*>(A + a_cols);
    h.scopes = reinterpret_cast<const GkScope*>(A + a_scopes);
    h.ncols = NC;
    h.nscopes = NS;
    db->hdr = h;
    GkIngestOut out;
    memset(&out, 0, sizeof out);
    out.flags = reinterpret_cast<uint32_t*>(A + a_flags);
    out.kind_sid = reinterpret_cast<uint32_t*>(A + a_kind);
    out.group_sid = reinterpret_cast<uint32_t*>(A + a_group);
    out.name_off = reinterpret_cast<uint32_t*>(A + a_nameoff);
    out.name_bytes = A + a_nameb;
    out.gen_off = reinterpret_cast<uint32_t*>(A + a_genoff);
    out.gen_bytes = A + a_genb;
    out.lbl_off = reinterpret_cast<uint32_t*>(A + a_lbloff);
    out.lbl_kv = reinterpret_cast<uint32_t*>(A + a_lblkv);
    out.nsrow = reinterpret_cast<uint32_t*>(A + a_nsrow);
    out.nsn_off = reinterpret_cast<uint32_t*>(A + a_nsnoff);
    out.nsn_bytes = A + a_nsnb;
    out.scope_off = reinterpret_cast<uint32_t* const*>(A + a_pscope);
    out.vt = reinterpret_cast<uint8_t* const*>(A + a_pvt);
    out.sid = reinterpret_cast<uint32_t* const*>(A + a_psid);
    out.num = reinterpret_cast<long long* const*>(A + a_pnum);
    out.boff = reinterpret_cast<uint32_t* const*>(A + a_pboff);
    out.bytes = reinterpret_cast<uint8_t* const*>(A + a_pbytes);
    out.head = reinterpret_cast<uint32_t* const*>(A + a_phead);
    out.row_rec = outc.row_rec;   // (the row handles of the count phase)
    unsigned long long* d_mm = temps.take<unsigned long long>(64);
    {
      const unsigned long long init[2] = {~0ull, 0ull};
      push_small(d_mm, init, 16);
      if (n) dmalloc(&db->gvk, (size_t)n * 8);
      out.gvk = db->gvk;
    }
    if (!n) CK(cudaMemsetAsync(A, 0, db->bytes, stream_));   // (no kernel writes the closing CSR entries of an empty batch)
    // the CSR offsets of the scopes and of the byte columns are the scanned counts of the count phase
    for (uint32_t s2 = 1; s2 < NS; ++s2)
      if (d_cnt[s2]) CK(cudaMemcpyAsync(A + a_scope[s2], d_cnt[s2], ((size_t)total[xh.scopes[s2].parent] + 1) * 4, cudaMemcpyDeviceToDevice, stream_));
    for (uint32_t ci = 0; ci < NC; ++ci) {
      const GkXCol& xc = xh.cols[ci];
      if ((xc.enc & GK_ENC_BYTES) && d_blen[xc.bytes_slot])
        CK(cudaMemcpyAsync(A + a_col[ci].boff, d_blen[xc.bytes_slot], ((size_t)total[xc.scope] + 1) * 4, cudaMemcpyDeviceToDevice, stream_));
    }
    // ---- write passes, repeated while lookups are missing (the host evaluates each distinct argument tuple once)
    CK(cudaEventRecord(e2, stream_));
    uint64_t total_miss = 0;
    double lut_ms = 0;
    std::vector<GkMiss> hmiss;
    for (int round = 0; n && round < 4096; ++round) {
      xp.lut_tab.keys = d_lut_keys_;
      xp.lut_tab.vals = d_lut_vals_;
      xp.lut_tab.mask = lut_.mask;
      xp.lut_vals = d_lutv_;
      CK(cudaMemsetAsync(in.nmiss, 0, 4, stream_));
      if (round == 0 || xh.nbytecols) {   // (the header does not depend on the lookups; a byte column's sid may)
        gk_header_kernel<<<blocks(n), kIngestThreads, 0, stream_>>>(xp, in, out);
        ++launches_;
        for (uint32_t ci = 0; ci < NC; ++ci) {
          const GkXCol& xc = xh.cols[ci];
          if (!(xc.enc & GK_ENC_BYTES) || !total[xc.scope]) continue;
          gk_bcol_write_kernel<<<blocks(total[xc.scope]), kIngestThreads, 0, stream_>>>(xp, in, out, ci, total[xc.scope]);
          ++launches_;
        }
      }
      for (uint32_t s2 = 0; s2 < NS; ++s2) {
        const uint32_t rows = total[s2];
        if (!rows || !xh.scopes[s2].ncols) continue;
        gk_cols_kernel<<<(uint32_t)(((uint64_t)rows * clanes + kIngestThreads - 1) / kIngestThreads), kIngestThreads, 0, stream_>>>(xp, in, out, s2, rows, clanes);
        ++launches_;
      }
      uint32_t nm = 0;
      CK(cudaMemcpyAsync(&nm, in.nmiss, 4, cudaMemcpyDeviceToHost, stream_));
      CK(cudaStreamSynchronize(stream_));
      CK(cudaGetLastError());
      if (nm == 0) break;
      const auto L0 = std::chrono::steady_clock::now();
      const uint32_t m = std::min(nm, miss_cap);
      hmiss.resize(m);
      CK(cudaMemcpy(hmiss.data(), in.misses, (size_t)m * sizeof(GkMiss), cudaMemcpyDeviceToHost));
      std::vector<GkLutVal> vals;
      if (rq.blob) {
        rq.lut_fill(hmiss.data(), m, vals);
      } else {   // (reextract: the argument bytes come from the device copy of the page)
        std::vector<unsigned long long> spans;
        std::vector<uint8_t> args(gk_compact_miss_spans(hmiss.data(), m, spans) + 1);
        const uint32_t nspans = (uint32_t)(spans.size() / 3);
        if (nspans) {
          auto* d_spans = temps.take<unsigned long long>(spans.size() * 8);
          auto* d_args = temps.take<uint8_t>(args.size());
          CK(cudaMemcpyAsync(d_spans, spans.data(), spans.size() * 8, cudaMemcpyHostToDevice, stream_));
          gk_gather_kernel<<<std::min<uint32_t>(nspans, 4096u), 128, 0, stream_>>>(d_args, in.blob, d_spans, nspans);
          ++launches_;
          CK(cudaMemcpyAsync(args.data(), d_args, args.size() - 1, cudaMemcpyDeviceToHost, stream_));
          CK(cudaStreamSynchronize(stream_));
          CK(cudaGetLastError());
        }
        rq.lut_fill_from(args.data(), hmiss.data(), m, vals);
      }
      // append the results, point the claimed slots at them
      const uint32_t base = (uint32_t)lutv_.size();
      lutv_.insert(lutv_.end(), vals.begin(), vals.end());
      if (lutv_.size() > d_lutv_cap_) {
        GkLutVal* nv = nullptr;
        const size_t ncap = lutv_.size() * 2 + 1024;
        CK(cudaMalloc(&nv, ncap * sizeof(GkLutVal)));
        if (base) CK(cudaMemcpy(nv, d_lutv_, (size_t)base * sizeof(GkLutVal), cudaMemcpyDeviceToDevice));
        if (d_lutv_) cudaFree(d_lutv_);
        d_lutv_ = nv;
        d_lutv_cap_ = ncap;
      }
      CK(cudaMemcpy(d_lutv_ + base, vals.data(), (size_t)m * sizeof(GkLutVal), cudaMemcpyHostToDevice));
      std::vector<uint32_t> pairs((size_t)m * 2);
      for (uint32_t j = 0; j < m; ++j) {
        pairs[2 * j] = hmiss[j].slot;
        pairs[2 * j + 1] = base + j;
        lut_filled_.emplace_back(hmiss[j].key, base + j);
      }
      CK(cudaMemcpy(d_fill, pairs.data(), pairs.size() * 4, cudaMemcpyHostToDevice));
      gk_fill_kernel<<<(m + 255) / 256, 256, 0, stream_>>>(d_lut_vals_, d_fill, m);
      ++launches_;
      total_miss += m;
      if ((lut_filled_.size() + (nm - m)) * 2 > (size_t)lut_.mask) {   // grow: filled entries re-inserted, pending claims dropped
        CK(cudaStreamSynchronize(stream_));
        uint32_t cap = (lut_.mask + 1) * 4;
        while ((size_t)cap < lut_filled_.size() * 4) cap <<= 1;
        lut_.init(cap);
        for (auto& kv : lut_filled_) lut_.put(kv.first, kv.second);
        upload_htab(lut_, &d_lut_keys_, &d_lut_vals_, &d_lut_cap_);
      }
      lut_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - L0).count();
      if (round == 4095) throw BackendError{"device ingest: lookups did not converge"};
    }
    CK(cudaEventRecord(e3, stream_));
    // ---- status of every object, tiling of the evaluation kernel
    if (status) {
      status->assign(n, 0);
      if (n) CK(cudaMemcpyAsync(status->data(), in.status, (size_t)n * 4, cudaMemcpyDeviceToHost, stream_));
    }
    unsigned long long mm[2] = {~0ull, 0ull};
    if (n) {
      gk_gvk_minmax_kernel<<<std::min<uint32_t>(1024u, (n + 255u) / 256u), 256, 0, stream_>>>(out.gvk, n, d_mm);
      ++launches_;
      CK(cudaMemcpyAsync(mm, d_mm, 16, cudaMemcpyDeviceToHost, stream_));
    }
    std::vector<uint32_t> cap(NS, 0);
    uint32_t ntiles = 0;
    const uint32_t tile = gk_choose_tile(kTile, net_sizes(c), max_smem_, [&](uint32_t per_tile) -> const std::vector<uint32_t>& {
      ntiles = (n + per_tile - 1) / per_tile;
      if (db->d_tile_lo) dfree(db->d_tile_lo), db->d_tile_lo = nullptr;
      dmalloc(&db->d_tile_lo, ((size_t)(ntiles + 1) * NS) * 4 + 64);
      CK(cudaMemsetAsync(d_cap, 0, (size_t)NS * 4, stream_));
      gk_tiles_kernel<<<(ntiles + 1 + 127) / 128, 128, 0, stream_>>>(xp, out, n, NS, per_tile, ntiles, db->d_tile_lo, d_cap);
      ++launches_;
      CK(cudaMemcpyAsync(cap.data(), d_cap, (size_t)NS * 4, cudaMemcpyDeviceToHost, stream_));
      CK(cudaStreamSynchronize(stream_));
      CK(cudaGetLastError());
      return cap;
    });
    db->tile = tile;
    db->ntiles = ntiles;
    db->gvk_uniform = mm[1] == 0 || mm[0] == mm[1];
    pack_type_words(db, c);
    finish_batch(db, c, cap);
    if (st) {
      float ms = 0;
      cudaEventElapsedTime(&ms, e0, e1);
      st->h2d_ms = ms;   // copy + tokenise, overlapped chunk by chunk
      st->tape_ms = ms;
      cudaEventElapsedTime(&ms, e1, e3);
      st->extract_ms = ms - lut_ms;
      st->lut_ms = lut_ms;
      st->h2d_bytes = (copied ? B + ((size_t)n + 1) * 8 : 0) + tab_bytes + aimg.size();
      st->lut_misses = total_miss;
      st->alg_bytes = alg;
      st->launches = launches_;
      st->total_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - T0).count();
    }
    if (getenv("GK_TRACE_INGEST")) {
      float a = 0, b = 0, d = 0;
      cudaEventElapsedTime(&a, e0, e1);
      cudaEventElapsedTime(&b, e1, e2);
      cudaEventElapsedTime(&d, e2, e3);
      fprintf(stderr, "[ingest] n=%u blob %.1f MB: copy+tokenise %.2f ms, count+scan(+alloc) %.2f ms, write(+lookups: %llu missed, %.1f ms host) %.2f ms, total wall %.2f ms, arena %.1f MB\n",
              n, B / 1e6, a, b, (unsigned long long)total_miss, lut_ms, d,
              std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - T0).count(), db->bytes / 1e6);
    }
    guard.release();
    return db;
  }
  void* fork_batch(void* b, const Compiled& other) override {
    auto* db = static_cast<DevBatch*>(b);
    CK(cudaSetDevice(device_));
    auto* f = new DevBatch();
    f->arena = db->arena;
    f->bytes = db->bytes;
    f->hdr = db->hdr;
    f->n = db->n;
    f->d_tile_lo = db->d_tile_lo;
    f->ntiles = db->ntiles;
    f->tile = db->tile;
    f->gvk_uniform = db->gvk_uniform;
    f->gvk = db->gvk;
    f->rows = db->rows;
    f->tw = db->tw;   // (f->hdr.tw: the batch's type words, which it keeps)
    f->tw_bytes = db->tw_bytes;
    f->fork = true;
    f->prog_version = other.version;
    std::unique_ptr<DevBatch, std::function<void(DevBatch*)>> guard(f, [this](DevBatch* x) { release(x); });
    finish_batch(f, other, db->cap);
    guard.release();
    return f;
  }

  void identity(void* b, BatchIdentity& out) override {
    auto* db = static_cast<DevBatch*>(b);
    std::lock_guard<std::mutex> l(mu_);
    CK(cudaSetDevice(device_));
    const uint32_t n = db->n;
    out.uniform_gvk = db->gvk_uniform;
    out.flags.resize(n);
    out.ns_off.resize((size_t)n + 1);
    out.name_off.resize((size_t)n + 1);
    if (!n) {
      out.ns_off[0] = out.name_off[0] = 0;
      return;
    }
    CK(cudaMemcpyAsync(out.flags.data(), db->hdr.flags, (size_t)n * 4, cudaMemcpyDeviceToHost, stream_));
    CK(cudaMemcpyAsync(out.ns_off.data(), db->hdr.nsn_off, ((size_t)n + 1) * 4, cudaMemcpyDeviceToHost, stream_));
    CK(cudaMemcpyAsync(out.name_off.data(), db->hdr.name_off, ((size_t)n + 1) * 4, cudaMemcpyDeviceToHost, stream_));
    CK(cudaStreamSynchronize(stream_));
    out.ns_bytes.resize(out.ns_off[n]);
    out.name_bytes.resize(out.name_off[n]);
    if (!out.ns_bytes.empty()) CK(cudaMemcpyAsync(out.ns_bytes.data(), db->hdr.nsn_bytes, out.ns_bytes.size(), cudaMemcpyDeviceToHost, stream_));
    if (!out.name_bytes.empty()) CK(cudaMemcpyAsync(out.name_bytes.data(), db->hdr.name_bytes, out.name_bytes.size(), cudaMemcpyDeviceToHost, stream_));
    CK(cudaStreamSynchronize(stream_));
  }

  // Ranking: the page's distinct apiVersion / kind hashes (a device hash table) are decoded on the host from one object each and ranked
  // by (group, version, kind); every object gets its triple's rank; the objects are merge-sorted by (that rank, namespace, name) and the
  // heads of equal runs scanned into one rank per identity.  Selection: per block of sorted positions and per constraint, the count of
  // flagged objects; per constraint (one warp), the rank of its limit-th flagged object; then every flagged bit at or below it.
  // `keep`: the ranks and thresholds stay on the device, in a DevRanks, until the last copy of keep->dev is dropped.
  struct DevRanks {
    uint32_t* rank = nullptr;
    uint32_t* thr = nullptr;
  };
  void audit_candidates(void* b, const uint32_t* viol, uint32_t words, uint32_t C, uint32_t limit, const GvkOf& gvk_of, std::vector<uint32_t>& cand,
                        float* device_ms, AuditRanks* keep) override {
    auto* db = static_cast<DevBatch*>(b);
    std::lock_guard<std::mutex> l(mu_);
    CK(cudaSetDevice(device_));
    const uint32_t n = db->n;
    cand.assign((size_t)n * words, 0u);
    if (device_ms) *device_ms = 0.f;
    if (!n || !C || !words) return;
    if (!db->gvk) throw BackendError{"audit candidates: the batch holds no apiVersion / kind hashes"};
    Temps temps(this);
    uint32_t cap = 1024;
    while (cap < 2 * n) cap <<= 1;
    const uint32_t mask = cap - 1, T = 256, grid = std::min<uint32_t>((n + T - 1) / T, (uint32_t)sms_ * 16);
    auto* keys = temps.take<unsigned long long>((size_t)cap * 8);
    auto* rep = temps.take<uint32_t>((size_t)cap * 4);
    auto* d_cnt = temps.take<uint32_t>(64);
    auto* d_list = temps.take<uint32_t>((size_t)2 * n * 4);
    auto* d_viol = temps.take<uint32_t>((size_t)n * words * 4);
    Event e0, e1, e2, e3;
    CK(cudaMemcpyAsync(d_viol, viol, (size_t)n * words * 4, cudaMemcpyHostToDevice, stream_));
    CK(cudaEventRecord(e0, stream_));
    CK(cudaMemsetAsync(keys, 0, (size_t)cap * 8, stream_));
    CK(cudaMemsetAsync(rep, 0xff, (size_t)cap * 4, stream_));
    CK(cudaMemsetAsync(d_cnt, 0, 4, stream_));
    gk_gvk_insert_kernel<<<grid, T, 0, stream_>>>(db->gvk, n, keys, rep, mask);
    gk_gvk_collect_kernel<<<std::min<uint32_t>((cap + T - 1) / T, (uint32_t)sms_ * 16), T, 0, stream_>>>(keys, rep, cap, d_cnt, d_list);
    CK(cudaEventRecord(e1, stream_));
    uint32_t m = 0;
    CK(cudaMemcpyAsync(&m, d_cnt, 4, cudaMemcpyDeviceToHost, stream_));
    CK(cudaStreamSynchronize(stream_));
    CK(cudaGetLastError());
    std::vector<uint32_t> list((size_t)2 * m);
    if (m) CK(cudaMemcpy(list.data(), d_list, list.size() * 4, cudaMemcpyDeviceToHost));
    // (group, version, kind) of one object per distinct hash, ranked; equal triples (differently escaped JSON) share a rank
    struct Gvk {
      std::string g, v, k;
      uint32_t j;
    };
    std::vector<Gvk> tri(m);
    for (uint32_t j = 0; j < m; ++j) {
      tri[j].j = j;
      gvk_of(list[2 * j + 1], tri[j].g, tri[j].v, tri[j].k);
    }
    auto key = [](const Gvk& x) { return std::tie(x.g, x.v, x.k); };
    std::sort(tri.begin(), tri.end(), [&](const Gvk& a, const Gvk& c2) { return key(a) < key(c2); });
    std::vector<uint32_t> pairs((size_t)2 * m);
    for (uint32_t r = 0, i = 0; i < m; ++i) {
      if (i && key(tri[i - 1]) != key(tri[i])) ++r;
      pairs[2 * i] = list[2 * tri[i].j];
      pairs[2 * i + 1] = r;
    }
    auto* gr = temps.take<uint32_t>((size_t)n * 4);
    auto* perm = temps.take<uint32_t>((size_t)n * 4);
    auto* head = temps.take<uint32_t>((size_t)n * 4);
    uint32_t* rank = nullptr;
    uint32_t* thr = nullptr;
    if (keep) {
      auto* kept = new DevRanks();
      keep->dev = std::shared_ptr<void>(kept, [this](void* p) {
        auto* k = static_cast<DevRanks*>(p);
        cudaSetDevice(device_);
        dfree(k->rank);
        dfree(k->thr);
        delete k;
      });
      dmalloc(&kept->rank, (size_t)n * 4);
      dmalloc(&kept->thr, (size_t)C * 4);
      rank = kept->rank;
      thr = kept->thr;
    } else {
      rank = temps.take<uint32_t>((size_t)n * 4);
      thr = temps.take<uint32_t>((size_t)C * 4);
    }
    CK(cudaEventRecord(e2, stream_));
    if (m) {
      CK(cudaMemcpyAsync(d_list, pairs.data(), pairs.size() * 4, cudaMemcpyHostToDevice, stream_));
      gk_gvk_assign_kernel<<<(m + T - 1) / T, T, 0, stream_>>>(d_list, m, rep);
    }
    gk_gvk_map_kernel<<<grid, T, 0, stream_>>>(db->gvk, n, keys, rep, mask, gr, perm);
    const GkIdLess less{gr, db->hdr.flags, db->hdr.nsn_off, db->hdr.nsn_bytes, db->hdr.name_off, db->hdr.name_bytes};
    size_t sort_bytes = 0, scan_bytes = 0;
    CK(cub::DeviceMergeSort::SortKeys(nullptr, sort_bytes, perm, (int64_t)n, less, stream_));
    CK(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, head, rank, (int64_t)n, stream_));
    void* cub_tmp = temps.take(std::max(sort_bytes, scan_bytes));
    CK(cub::DeviceMergeSort::SortKeys(cub_tmp, sort_bytes, perm, (int64_t)n, less, stream_));
    gk_id_heads_kernel<<<grid, T, 0, stream_>>>(perm, n, less, head);
    CK(cub::DeviceScan::InclusiveSum(cub_tmp, scan_bytes, head, gr, (int64_t)n, stream_));   // (gr is free again: the sort is done)
    gk_id_scatter_kernel<<<grid, T, 0, stream_>>>(perm, gr, n, rank);
    const uint32_t nb = (n + kSelChunk - 1) / kSelChunk;
    auto* cnt = temps.take<uint32_t>((size_t)nb * C * 4);
    auto* d_cand = temps.take<uint32_t>((size_t)n * words * 4);
    if ((size_t)C * 4 > max_smem_) throw BackendError{"audit candidates: too many constraints for one block's counters"};
    if ((size_t)C * 4 > 48 * 1024) CK(cudaFuncSetAttribute(gk_sel_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(C * 4)));
    gk_sel_count_kernel<<<nb, 256, (size_t)C * 4, stream_>>>(perm, d_viol, n, words, C, cnt);
    gk_sel_thresh_kernel<<<(C * 32 + 255) / 256, 256, 0, stream_>>>(perm, d_viol, cnt, rank, n, words, C, nb, limit, thr);
    gk_sel_emit_kernel<<<std::min<uint32_t>((uint32_t)(((size_t)n * words + T - 1) / T), (uint32_t)sms_ * 16), T, 0, stream_>>>(d_viol, rank, thr, n, words, C, d_cand);
    CK(cudaEventRecord(e3, stream_));
    CK(cudaMemcpyAsync(cand.data(), d_cand, (size_t)n * words * 4, cudaMemcpyDeviceToHost, stream_));
    CK(cudaStreamSynchronize(stream_));
    CK(cudaGetLastError());
    launches_ += 8 + (m ? 1 : 0);
    float a = 0.f, c2 = 0.f;
    cudaEventElapsedTime(&a, e0, e1);
    cudaEventElapsedTime(&c2, e2, e3);
    if (device_ms) *device_ms = a + c2;
  }

  // ---- front buffers: a page's JSON, offsets and tape.  Two of them, so that page k+1 streams in (copy stream + front stream)
  // while page k is extracted and evaluated on the main stream.
  struct Front {
    Scratch buf;
    GkIngestIn in{};            // blob / ooff / tape / ntape / status pointers into buf, n
    const uint8_t* host_blob = nullptr;
    size_t n = 0;
    bool pending = false;       // prefetched, not yet consumed
    cudaEvent_t done = nullptr; // copy + tokenise finished
  };
  // The layout of a page's front buffer for B bytes of JSON and n objects: the JSON (16 bytes over, for the tokeniser's word
  // reads), the offsets, the tape (object i's at gk_tape_off), the tape lengths and the status words.  bytes(): the whole buffer.
  struct PageLayout {
    size_t o_blob, o_ooff, o_tape, o_ntape, o_status, total;
    uint32_t n;
    PageLayout(unsigned long long B, uint32_t nn) : n(nn) {
      Carver sc;
      o_blob = sc.take((size_t)B + 16), o_ooff = sc.take(((size_t)n + 1) * 8), o_tape = sc.take(((size_t)(B / 2) + 4ull * n + 64) * 8),
      o_ntape = sc.take((size_t)n * 4), o_status = sc.take((size_t)n * 4);
      total = gk_align(sc.off);
    }
    GkIngestIn at(uint8_t* d) const {
      GkIngestIn in;
      memset(&in, 0, sizeof in);
      in.blob = d + o_blob;
      in.ooff = reinterpret_cast<const unsigned long long*>(d + o_ooff);
      in.tape = reinterpret_cast<unsigned long long*>(d + o_tape);
      in.ntape = reinterpret_cast<uint32_t*>(d + o_ntape);
      in.status = reinterpret_cast<uint32_t*>(d + o_status);
      in.n = n;
      return in;
    }
  };

  Front& start_front(const uint8_t* blob, const unsigned long long* ooff, size_t nn) {   // (front_mu_ held)
    Front& f = fronts_[next_front_];
    next_front_ ^= 1;
    const uint32_t n = (uint32_t)nn;
    const PageLayout lay(ooff[n], n);
    if (!f.done) CK(cudaEventCreateWithFlags(&f.done, cudaEventDisableTiming));
    // the buffer may still be read by the kernels of the page that used it last: they ran on the main stream
    CK(cudaStreamSynchronize(stream_));
    uint8_t* d = f.buf.need(lay.total);
    f.in = lay.at(d);
    f.host_blob = blob;
    f.n = nn;
    CK(cudaMemcpyAsync(d + lay.o_ooff, ooff, ((size_t)n + 1) * 8, cudaMemcpyHostToDevice, copy_stream_));
    copy_and_tokenise(f.in, d + lay.o_blob + ooff[0], 0, blob, ooff, n);
    CK(cudaEventRecord(f.done, front_stream_));
    f.pending = true;
    return f;
  }
  // Objects [0, cnt) of a host page (JSON at blob + ooff[k]) become objects first .. first + cnt - 1 of the device page `in`, their
  // bytes at dst + (ooff[k] - ooff[0]), where in.ooff already places them: the JSON goes over in chunks on the copy stream, and the
  // tokeniser of a chunk starts on the front stream as soon as its bytes have landed.  (front_mu_ held)
  void copy_and_tokenise(const GkIngestIn& in, uint8_t* dst, uint32_t first, const uint8_t* blob, const unsigned long long* ooff, uint32_t cnt) {
    // Chunk size: a tokeniser launch of a 32 MB chunk (50k Pods) fills a small share of the warp slots and takes about the same
    // time whatever its size (one thread walks one object); bigger chunks mean fewer, fuller launches at the price of a later
    // start, much smaller ones multiply the page time.  GK_INGEST_CHUNK_MB overrides.
    static const size_t kChunk = []() {
      size_t mb = 32;
      if (const char* ev = getenv("GK_INGEST_CHUNK_MB")) mb = (size_t)std::max(1, atoi(ev));
      return mb << 20;
    }();
    uint32_t k = 0;
    while (k < cnt) {
      uint32_t last = k;
      const unsigned long long lo = ooff[k];
      while (last < cnt && ooff[last + 1] - lo <= kChunk) ++last;
      if (last == k) ++last;   // one object larger than a chunk
      const unsigned long long hi = ooff[last];
      CK(cudaMemcpyAsync(dst + (lo - ooff[0]), blob + lo, (size_t)(hi - lo), cudaMemcpyHostToDevice, copy_stream_));
      cudaEvent_t ev = chunk_event(k);
      CK(cudaEventRecord(ev, copy_stream_));
      CK(cudaStreamWaitEvent(front_stream_, ev, 0));
      const uint32_t m = last - k;
      gk_tape_kernel<<<(m + kIngestThreads - 1) / kIngestThreads, kIngestThreads, 0, front_stream_>>>(in, first + k, m);
      ++launches_;
      k = last;
    }
    if (getenv("GK_TRACE_LAUNCH"))
      fprintf(stderr, "[launch] gk_tape_kernel over %u objects, after a host->device copy of %llu bytes\n", cnt, cnt ? ooff[cnt] - ooff[0] : 0ull);
    if (cnt == 0) CK(cudaStreamWaitEvent(front_stream_, chunk_event_after_copy(), 0));
  }
  cudaEvent_t chunk_event_after_copy() {
    cudaEvent_t ev = chunk_event(0);
    CK(cudaEventRecord(ev, copy_stream_));
    return ev;
  }
  void prefetch(const uint8_t* blob, const unsigned long long* ooff, size_t n) override {
    std::lock_guard<std::mutex> fl(front_mu_);
    CK(cudaSetDevice(device_));
    start_front(blob, ooff, n);
  }

  void pin_host(const void* p, size_t bytes, bool pin) override {
    CK(cudaSetDevice(device_));
    if (pin) CK(cudaHostRegister(const_cast<void*>(p), bytes, cudaHostRegisterDefault));
    else CK(cudaHostUnregister(const_cast<void*>(p)));
  }
  cudaEvent_t chunk_event(uint32_t k) {
    (void)k;
    if (chunk_ev_next_ >= chunk_evs_.size()) {
      cudaEvent_t e;
      CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      chunk_evs_.push_back(e);
    }
    cudaEvent_t e = chunk_evs_[chunk_ev_next_];
    chunk_ev_next_ = (chunk_ev_next_ + 1) % 64 == 0 ? 0 : chunk_ev_next_ + 1;
    return e;
  }

  void eval_into(void* b, const std::vector<uint32_t>& active, const DevOutPtrs& dst) override {
    auto* db = static_cast<DevBatch*>(b);
    std::lock_guard<std::mutex> l(mu_);
    CK(cudaSetDevice(device_));
    fire(prepare(db, active, static_cast<uint32_t*>(dst.viol), static_cast<uint32_t*>(dst.err), static_cast<unsigned long long*>(dst.totals),
                 static_cast<unsigned long long*>(dst.err_totals), static_cast<cudaStream_t>(dst.stream), dst));
  }

  // Generator selection: the page's distinct apiVersion / kind hashes into a device table (as audit_candidates finds them), decided on
  // the host from one object each, then every object marked and the marks compacted, in object order, into the index list.
  void select_generators(void* b, const GvkOf& gvk_of, const GvkWanted& wanted, std::vector<uint32_t>& sel, uint32_t* kinds, float* device_ms) override {
    auto* db = static_cast<DevBatch*>(b);
    std::lock_guard<std::mutex> l(mu_);
    CK(cudaSetDevice(device_));
    const uint32_t n = db->n;
    sel.clear();
    if (kinds) *kinds = 0;
    if (device_ms) *device_ms = 0.f;
    if (!n) return;
    if (!db->gvk) throw BackendError{"select generators: the batch holds no apiVersion / kind hashes"};
    Temps temps(this);
    uint32_t cap = 1024;
    while (cap < 2 * n) cap <<= 1;
    const uint32_t mask = cap - 1, T = 256, grid = std::min<uint32_t>((n + T - 1) / T, (uint32_t)sms_ * 16);
    auto* keys = temps.take<unsigned long long>((size_t)cap * 8);
    auto* rep = temps.take<uint32_t>((size_t)cap * 4);
    auto* d_cnt = temps.take<uint32_t>(64);
    auto* d_list = temps.take<uint32_t>((size_t)2 * n * 4);
    Event e0, e1, e2, e3;
    CK(cudaEventRecord(e0, stream_));
    CK(cudaMemsetAsync(keys, 0, (size_t)cap * 8, stream_));
    CK(cudaMemsetAsync(rep, 0xff, (size_t)cap * 4, stream_));
    CK(cudaMemsetAsync(d_cnt, 0, 4, stream_));
    gk_gvk_insert_kernel<<<grid, T, 0, stream_>>>(db->gvk, n, keys, rep, mask);
    gk_gvk_collect_kernel<<<std::min<uint32_t>((cap + T - 1) / T, (uint32_t)sms_ * 16), T, 0, stream_>>>(keys, rep, cap, d_cnt, d_list);
    CK(cudaEventRecord(e1, stream_));
    uint32_t m = 0;
    CK(cudaMemcpyAsync(&m, d_cnt, 4, cudaMemcpyDeviceToHost, stream_));
    CK(cudaStreamSynchronize(stream_));
    CK(cudaGetLastError());
    std::vector<uint32_t> list((size_t)2 * m);
    if (m) CK(cudaMemcpy(list.data(), d_list, list.size() * 4, cudaMemcpyDeviceToHost));
    std::vector<uint32_t> pairs;   // (slot, 1) of every selected hash
    for (uint32_t j = 0; j < m; ++j) {
      std::string g, v, k;
      gvk_of(list[2 * j + 1], g, v, k);
      if (wanted(g, v, k)) pairs.insert(pairs.end(), {list[2 * j], 1u});
    }
    const uint32_t np = (uint32_t)(pairs.size() / 2);
    auto* mark = temps.take<uint8_t>(n);
    auto* idx = temps.take<uint32_t>((size_t)n * 4);
    auto* d_sel = temps.take<uint32_t>((size_t)n * 4);
    CK(cudaEventRecord(e2, stream_));
    CK(cudaMemsetAsync(rep, 0, (size_t)cap * 4, stream_));   // (rep is free again: now the pick flag per slot)
    if (np) {
      CK(cudaMemcpyAsync(d_list, pairs.data(), pairs.size() * 4, cudaMemcpyHostToDevice, stream_));
      gk_gvk_assign_kernel<<<(np + T - 1) / T, T, 0, stream_>>>(d_list, np, rep);
    }
    gk_gen_mark_kernel<<<grid, T, 0, stream_>>>(db->gvk, n, keys, rep, mask, mark, idx);
    size_t sel_bytes = 0;
    CK(cub::DeviceSelect::Flagged(nullptr, sel_bytes, idx, mark, d_sel, d_cnt, (int64_t)n, stream_));
    CK(cub::DeviceSelect::Flagged(temps.take(sel_bytes), sel_bytes, idx, mark, d_sel, d_cnt, (int64_t)n, stream_));
    CK(cudaEventRecord(e3, stream_));
    uint32_t g = 0;
    CK(cudaMemcpyAsync(&g, d_cnt, 4, cudaMemcpyDeviceToHost, stream_));
    CK(cudaStreamSynchronize(stream_));
    CK(cudaGetLastError());
    sel.resize(g);
    if (g) CK(cudaMemcpy(sel.data(), d_sel, (size_t)g * 4, cudaMemcpyDeviceToHost));
    launches_ += 4 + (np ? 1 : 0);
    if (kinds) *kinds = m;
    float a = 0.f, c2 = 0.f;
    cudaEventElapsedTime(&a, e0, e1);
    cudaEventElapsedTime(&c2, e2, e3);
    if (device_ms) *device_ms = a + c2;
  }

  void set_parents(void* res, const std::vector<uint32_t>& par, const std::vector<uint32_t>& off) override {
    auto* r = static_cast<DevBatch*>(res);
    std::lock_guard<std::mutex> l(mu_);
    CK(cudaSetDevice(device_));
    if (off.size() != par.size() + 1) throw BackendError{"set_parents: the offsets must have one entry more than the parents"};
    dfree(r->fold_par);
    dfree(r->fold_off);
    dfree(r->fold_tot);
    r->fold_par = r->fold_off = nullptr;
    r->fold_tot = nullptr;
    r->fold_m = 0;
    dmalloc(&r->fold_par, par.size() * 4);
    dmalloc(&r->fold_off, off.size() * 4);
    dmalloc(&r->fold_tot, (size_t)2 * r->words * 32 * 8);
    if (!par.empty()) CK(cudaMemcpyAsync(r->fold_par, par.data(), par.size() * 4, cudaMemcpyHostToDevice, stream_));
    CK(cudaMemcpyAsync(r->fold_off, off.data(), off.size() * 4, cudaMemcpyHostToDevice, stream_));
    CK(cudaStreamSynchronize(stream_));   // (the host vectors are the caller's)
    r->fold_m = (uint32_t)par.size();
  }

  GkFoldArgs fold_args(const DevBatch& r) const {
    GkFoldArgs a{};
    a.par = r.fold_par;
    a.off = r.fold_off;
    a.m = r.fold_m;
    a.words = r.words;
    a.nconstraints = prog_.nconstraints;
    a.cviol = r.viol;
    a.cerr = r.err;
    return a;
  }
  void launch_fold(const GkFoldArgs& a, cudaStream_t st) {
    const uint32_t C = a.nconstraints;
    if (!a.m || !C) return;
    const size_t smem = (size_t)2 * C * 4;
    if (smem > max_smem_) throw BackendError{"fold: too many constraints for one block's counters"};
    if (smem > 48 * 1024) CK(cudaFuncSetAttribute(gk_fold_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const uint32_t T = 256, grid = std::max(1u, std::min<uint32_t>((a.m + T - 1) / T, (uint32_t)sms_ * 8));
    gk_fold_kernel<<<grid, T, smem, st>>>(a);
    CK(cudaGetLastError());
    ++launches_;
    if (a.npeers) {
      gk_fold_publish_kernel<<<1, 256, 0, st>>>(a);
      CK(cudaGetLastError());
      ++launches_;
    }
  }

  // eval() of the parents (their unfolded planes copied back into `own` when asked), eval() of the resultants into their own planes,
  // then the fold into the parents' own planes (the device copy of the CSR, set_parents)
  void eval_expanded(void* b, void* res, const std::vector<uint32_t>& par, const std::vector<uint32_t>& off, const std::vector<uint32_t>& active,
                     EvalOut& out, bool copy_back, EvalOut* own, EvalOut* rout) override {
    (void)par, (void)off;
    eval(b, active, out, own != nullptr);
    if (own) {
      own->viol = std::move(out.viol);
      own->err = std::move(out.err);
      out.viol = BitPlane();
      out.err = BitPlane();
    }
    EvalOut tmp;
    EvalOut& r = rout ? *rout : tmp;
    eval(res, active, r, rout != nullptr);
    out.kernel_ms += r.kernel_ms;
    fold_planes(b, res, out, copy_back);
  }

  // the fold into `b`'s own planes after eval() of both; the newly set bits added to out's totals, the folded planes copied back
  void fold_planes(void* b, void* res, EvalOut& out, bool copy_back) {
    auto* db = static_cast<DevBatch*>(b);
    auto* r = static_cast<DevBatch*>(res);
    std::lock_guard<std::mutex> l(mu_);
    CK(cudaSetDevice(device_));
    const uint32_t C = prog_.nconstraints;
    GkFoldArgs a = fold_args(*r);
    a.sviol = a.dviol = db->viol;
    a.serr = a.derr = db->err;
    a.totals = r->fold_tot;
    a.err_totals = r->fold_tot + C;
    if (C) CK(cudaMemsetAsync(r->fold_tot, 0, (size_t)2 * C * 8, stream_));
    CK(cudaEventRecord(ev0_, stream_));
    launch_fold(a, stream_);
    CK(cudaEventRecord(ev1_, stream_));
    std::vector<unsigned long long> t(2 * (size_t)C);
    if (C) CK(cudaMemcpyAsync(t.data(), r->fold_tot, t.size() * 8, cudaMemcpyDeviceToHost, stream_));
    CK(cudaStreamSynchronize(stream_));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, ev0_, ev1_));
    out.kernel_ms += ms;
    out.launches = launches_;
    for (uint32_t c = 0; c < C && c < out.totals.size(); ++c) {
      out.totals[c] += t[c];
      out.err_totals[c] += t[C + c];
    }
    if (copy_back) copy_planes(*db, out);
  }

  void fold_into(void* res, const std::vector<uint32_t>& par, const std::vector<uint32_t>& off, const std::vector<uint32_t>& active,
                 const DevOutPtrs& dst) override {
    (void)par, (void)off;   // (the device copy of set_parents)
    auto* r = static_cast<DevBatch*>(res);
    std::lock_guard<std::mutex> l(mu_);
    CK(cudaSetDevice(device_));
    GkFoldArgs a = fold_args(*r);
    set_peers(a, dst);
    const uint32_t C = prog_.nconstraints;
    cudaStream_t st = static_cast<cudaStream_t>(dst.stream);
    // the resultants into their own planes (their totals are not the caller's)
    fire(prepare(r, active, r->viol, r->err, r->fold_tot, r->fold_tot + std::max(C, 1u), st));
    a.sviol = dst.npeers ? reinterpret_cast<const uint32_t*>(dst.peer_viol[dst.rank]) : static_cast<const uint32_t*>(dst.viol);
    a.serr = a.derr = static_cast<uint32_t*>(dst.err);
    a.dviol = dst.npeers ? nullptr : static_cast<uint32_t*>(dst.viol);
    a.totals = static_cast<unsigned long long*>(dst.totals);
    a.err_totals = static_cast<unsigned long long*>(dst.err_totals);
    launch_fold(a, st);
  }

  // The resultants' planes as eval() left them in `res` (and the ambiguity fork's in `amb`), the parents' CSR as set_parents() left it,
  // the ranking audit_candidates() kept: gk_res_classify_kernel, then the counters and the listed pairs back to the host.  The list
  // holds at most the resultants' flagged pairs, which their totals bound.
  void audit_resultants(void* res, void* amb, const EvalOut& rev, const EvalOut* ramb, const std::vector<uint32_t>& par, const std::vector<uint32_t>& off,
                        const AuditRanks& ranks, const ResultantClasses& cls, ResultantSplit& out, float* device_ms) override {
    (void)ramb, (void)par, (void)off;   // (the planes and the CSR are read where they are resident)
    auto* r = static_cast<DevBatch*>(res);
    std::lock_guard<std::mutex> l(mu_);
    CK(cudaSetDevice(device_));
    const uint32_t C = cls.nconstraints, NC = cls.classes * C, m = r->n;
    out.counted.assign(NC, 0);
    out.render.clear();
    if (device_ms) *device_ms = 0.f;
    if (!m || !C) return;
    auto* dr = static_cast<DevRanks*>(ranks.dev.get());
    if (!dr) throw BackendError{"audit resultants: the parents' ranking was not kept on the device"};
    if (r->fold_m + 1 != off.size() || (off.size() && off.back() != m)) throw BackendError{"audit resultants: the batch's parents are not the CSR given"};
    if ((size_t)NC * 4 > max_smem_) throw BackendError{"audit resultants: too many constraints and action classes for one block's counters"};
    uint64_t flagged = 0;
    for (uint32_t c = 0; c < C && c < rev.totals.size(); ++c) flagged += rev.totals[c] + rev.err_totals[c];
    if (flagged > 0x7fffffffull) throw BackendError{"audit resultants: more than 2^31 flagged pairs"};
    Temps temps(this);
    GkResAuditArgs x{};
    x.a.viol = r->viol;
    x.a.err = r->err;
    x.a.amb = amb ? static_cast<DevBatch*>(amb)->viol : nullptr;
    x.a.words = r->words;
    x.a.nconstraints = C;
    x.par = r->fold_par;
    x.off = r->fold_off;
    x.m = r->fold_m;
    x.nres = m;
    x.rank = dr->rank;
    x.thr = dr->thr;
    x.classes = cls.classes;
    x.cap = (uint32_t)std::max<uint64_t>(flagged, 1);
    auto* d_single = temps.take<uint8_t>(C);
    auto* d_cls = temps.take<uint8_t>(m);
    x.counted = temps.take<unsigned long long>((size_t)NC * 8);
    x.list = temps.take<uint32_t>((size_t)x.cap * 8);
    x.nlist = temps.take<uint32_t>(4);
    CK(cudaMemcpyAsync(d_single, cls.single, C, cudaMemcpyHostToDevice, stream_));
    CK(cudaMemcpyAsync(d_cls, cls.cls, m, cudaMemcpyHostToDevice, stream_));
    if (cls.dead) {
      auto* d_dead = temps.take<uint8_t>(cls.parents);
      CK(cudaMemcpyAsync(d_dead, cls.dead, cls.parents, cudaMemcpyHostToDevice, stream_));
      x.dead = d_dead;
    }
    x.a.single = d_single;
    x.cls = d_cls;
    CK(cudaMemsetAsync(x.counted, 0, (size_t)NC * 8, stream_));
    CK(cudaMemsetAsync(x.nlist, 0, 4, stream_));
    const size_t smem = (size_t)NC * 4;
    if (smem > 48 * 1024) CK(cudaFuncSetAttribute(gk_res_classify_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const uint32_t T = 256, grid = std::max(1u, std::min<uint32_t>((m + T - 1) / T, (uint32_t)sms_ * 8));
    Event e0, e1;
    CK(cudaEventRecord(e0, stream_));
    gk_res_classify_kernel<<<grid, T, smem, stream_>>>(x);
    CK(cudaGetLastError());
    CK(cudaEventRecord(e1, stream_));
    ++launches_;
    uint32_t nl = 0;
    CK(cudaMemcpyAsync(out.counted.data(), x.counted, (size_t)NC * 8, cudaMemcpyDeviceToHost, stream_));
    CK(cudaMemcpyAsync(&nl, x.nlist, 4, cudaMemcpyDeviceToHost, stream_));
    CK(cudaStreamSynchronize(stream_));
    if (nl > x.cap) throw BackendError{"audit resultants: more pairs to render than the resultants' totals"};
    out.render.resize((size_t)nl * 2);
    if (nl) CK(cudaMemcpy(out.render.data(), x.list, (size_t)nl * 8, cudaMemcpyDeviceToHost));
    if (device_ms) CK(cudaEventElapsedTime(device_ms, e0, e1));
  }

 private:
  void free_tables() {
    void** ptrs[] = {(void**)&d_outs_, (void**)&d_ops_, (void**)&d_items_, (void**)&d_phase_off_, (void**)&d_match_, (void**)&d_pool_, (void**)&d_cbytes_};
    for (auto pp : ptrs) {
      if (*pp) cudaFree(*pp);
      *pp = nullptr;
    }
  }
  std::mutex ingest_mu_;
  Scratch scratch_, tabs_, rows_;
  SidTable sid_;
  unsigned long long* d_sid_keys_ = nullptr;
  uint32_t* d_sid_vals_ = nullptr;
  size_t d_sid_cap_ = 0;
  HashTabHost lut_;                                               // geometry of the device table (the device copy is authoritative)
  std::vector<std::pair<unsigned long long, uint32_t>> lut_filled_;   // every answered lookup (key, result index): re-inserted on growth
  unsigned long long* d_lut_keys_ = nullptr;
  uint32_t* d_lut_vals_ = nullptr;
  size_t d_lut_cap_ = 0;
  std::vector<GkLutVal> lutv_;
  GkLutVal* d_lutv_ = nullptr;
  size_t d_lutv_cap_ = 0;
  cudaStream_t copy_stream_ = nullptr, front_stream_ = nullptr;
  std::mutex front_mu_;
  Front fronts_[2];
  int next_front_ = 0;
  std::vector<cudaEvent_t> chunk_evs_;
  size_t chunk_ev_next_ = 0;
  int device_;
  int sms_ = 132;
  size_t max_smem_ = 0, sm_smem_ = 0;
  cudaStream_t stream_ = nullptr;
  cudaEvent_t ev0_ = nullptr, ev1_ = nullptr;
  cudaStream_t side_stream_ = nullptr;   // fire(): the interpreter's units, beside the generated kernel
  cudaEvent_t ev_fork_ = nullptr;
  std::mutex mu_;
  uint64_t version_ = 0, launches_ = 0;
  GkProgram prog_{};
  std::vector<uint32_t> last_active_;
  GkOp* d_ops_ = nullptr;
  uint32_t* d_items_ = nullptr;
  GkOutEnt* d_outs_ = nullptr;
  uint32_t* d_phase_off_ = nullptr;
  GkMatch* d_match_ = nullptr;
  uint32_t* d_pool_ = nullptr;
  uint8_t* d_cbytes_ = nullptr;
  uint32_t* d_dict_off_ = nullptr;
  uint8_t* d_dict_bytes_ = nullptr;
  uint32_t dict_n_ = 0;
  void* d_scalars_ = nullptr;
  unsigned long long* d_totals_ = nullptr;
  uint32_t* d_errlist_ = nullptr;
  uint32_t err_cap_ = 1u << 20;   // triples d_errlist_ holds; eval() grows it when a page has more matcher errors
  uint32_t* d_active_ = nullptr;
  unsigned long long* d_timing_ = nullptr;
  int host_threads_ = effective_cpus();
  std::list<SpecEntry> spec_cache_;
  SpecEntry* spec_cur_ = nullptr;
  bool spec_on_ = !(getenv("GK_SPEC") && atoi(getenv("GK_SPEC")) == 0);
  uint32_t spec_min_objects_ = getenv("GK_SPEC_MIN_OBJECTS") ? (uint32_t)atoll(getenv("GK_SPEC_MIN_OBJECTS")) : 8192u;   // below: not worth a ~2 s NVRTC run
  // 256 threads walk a 512-object tile (two objects each), at least two CTAs per SM (<= 128 registers) so that one CTA's staging
  // overlaps another's object walk: the fastest of 512 x 1, 256 x 2 and 256 x 3 over configs 2, 4 and 5 (256 x 3 spills at config 2)
  int spec_threads_ = getenv("GK_SPEC_THREADS") ? std::min(1024, std::max(32, atoi(getenv("GK_SPEC_THREADS")) / 32 * 32)) : 256;
  int spec_minb_ = getenv("GK_SPEC_MINB") ? std::max(1, atoi(getenv("GK_SPEC_MINB"))) : 3;   // 256 x 3: an 80-register cap, measured best or level at configs 2, 4 and 5 (DESIGN 5a)
  const char* last_kernel_ = "gk_eval_kernel";
  // gk_spec_rows_kernel: one thread per row, no shared memory
  int spec_rows_threads_ = getenv("GK_SPEC_ROWS_THREADS") ? std::min(1024, std::max(32, atoi(getenv("GK_SPEC_ROWS_THREADS")) / 32 * 32)) : 256;
  int spec_rows_minb_ = getenv("GK_SPEC_ROWS_MINB") ? std::max(1, atoi(getenv("GK_SPEC_ROWS_MINB"))) : 6;   // 256 x 6: a 40-register cap, no spill at config 2 (DESIGN 5a)
  uint32_t* d_spec_x_ = nullptr;   // the export arrays (SpecSource::export_bytes), grow-only
  size_t spec_x_bytes_ = 0;
  size_t optin_smem_ = 0;     // the device's per-CTA shared-memory limit
  void* pinned_ = nullptr;
  size_t pinned_bytes_ = 0;
};

Backend* make_backend(int device) { return new CudaBackend(device); }

}  // namespace gk
