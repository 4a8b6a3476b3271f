// CUDA kernels of the device ingest path (the shared per-object / per-row code is ingest_core.h).
//   gk_tape_kernel        per object: raw JSON -> tape (+ review-level status)
//   gk_hcount_kernel      per object: byte / label counts of the header arrays, flags word (skip bit)
//   gk_header_kernel      per object: flags, kind / group sids, names, labels, namespace row
//   gk_scope_count_kernel per row of the PARENT scope: members of the generator collection of scope t
//   gk_scope_fill_kernel  per row of the parent scope: the 16-byte row handles of its members
//   gk_bcol_len_kernel    per row: decoded length of a byte-encoded column    gk_bcol_write_kernel: its encodings + bytes
//   gk_cols_kernel        per row of one scope: every other column encoding; lookups through the device hash tables
//   gk_scan_*             exclusive prefix sums (counts -> CSR offsets), three small kernels for any length
//   gk_fill_kernel        the host's answers to the miss list -> table slots
//   gk_gather_kernel      the argument bytes of the miss list, when the host's copy of the page is not at hand (a kept source)
//   gk_keep_len_kernel    gk_batch_patch: byte lengths of a kept page's staying objects (scanned into their new offsets)
//   gk_splice_kernel      gk_batch_patch: one warp per staying object moves its JSON, tape, tape length and status to the new page
//   gk_tiles_kernel       first row of every scope for every evaluation tile + the largest tile of each scope
// Level-synchronous: every kernel after the tokeniser runs ONE step for all rows of ONE scope, so the threads of a warp follow
// the same path (the per-object walk of the whole scope tree it replaces ran at 1.7 active threads per warp instruction).
// HBM-bound byte work (no tensor cores).
#pragma once
#include <cuda_runtime.h>

#include "ingest_core.h"

namespace gk {

constexpr int kIngestThreads = 128;
#ifndef GK_INGEST_MIN_BLOCKS
#define GK_INGEST_MIN_BLOCKS 8   /* 64 registers per thread: these passes are latency-bound, resident warps are what hides it */
#endif

__global__ void __launch_bounds__(kIngestThreads) gk_tape_kernel(const GkIngestIn in, uint32_t first, uint32_t count) {
  const uint32_t i = first + blockIdx.x * blockDim.x + threadIdx.x;
  if (i < first + count) gk_tape_obj(in, i);
}

__global__ void __launch_bounds__(kIngestThreads) gk_hcount_kernel(const GkXProg xp, const GkIngestIn in, const GkIngestOut out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= in.n) return;
  uint32_t cur[GK_CNT_EXTRA];
  gk_ingest_obj<GK_PASS_COUNT>(xp, in, out, i, GkCur{cur, 1}, 0u, 1u);
}

__global__ void __launch_bounds__(kIngestThreads) gk_header_kernel(const GkXProg xp, const GkIngestIn in, const GkIngestOut out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= in.n) return;
  uint32_t cur[GK_CNT_EXTRA];
  gk_ingest_obj<GK_PASS_HEADER>(xp, in, out, i, GkCur{cur, 1}, 0u, 1u);
}

// the per-row column pass of one scope: a thread (or `lanes` threads) per row
__global__ void __launch_bounds__(kIngestThreads, GK_INGEST_MIN_BLOCKS) gk_cols_kernel(const GkXProg xp, const GkIngestIn in, const GkIngestOut out, uint32_t scope, uint32_t rows,
                                                                 uint32_t lanes) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x, r = t / lanes, lane = t % lanes;
  if (r >= rows) return;
  gk_ingest_row(xp, in, out, scope, r, lane, lanes);
}

// scope t: cnt[r] = members of the generator under parent row r, coll[r] = its tape index
__global__ void __launch_bounds__(kIngestThreads, GK_INGEST_MIN_BLOCKS) gk_scope_count_kernel(const GkXProg xp, const GkIngestIn in, const GkIngestOut out, uint32_t t,
                                                                                        uint32_t prows, uint32_t* cnt, uint32_t* coll) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= prows) return;
  uint32_t node;
  cnt[r] = gk_scope_count(xp, in, out, t, r, &node);
  coll[r] = node;
}
__global__ void __launch_bounds__(kIngestThreads, GK_INGEST_MIN_BLOCKS) gk_scope_fill_kernel(const GkXProg xp, const GkIngestIn in, const GkIngestOut out, uint32_t t,
                                                                                       uint32_t prows, const uint32_t* off, const uint32_t* coll) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= prows) return;
  gk_scope_fill(xp, in, out, t, r, coll[r], off[r]);
}
__global__ void __launch_bounds__(kIngestThreads, GK_INGEST_MIN_BLOCKS) gk_bcol_len_kernel(const GkXProg xp, const GkIngestIn in, const GkIngestOut out, uint32_t ci,
                                                                                     uint32_t rows, uint32_t* len) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < rows) len[r] = gk_bcol_len(xp, in, out, ci, r);
}
__global__ void __launch_bounds__(kIngestThreads, GK_INGEST_MIN_BLOCKS) gk_bcol_write_kernel(const GkXProg xp, const GkIngestIn in, const GkIngestOut out, uint32_t ci,
                                                                                       uint32_t rows) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < rows) gk_bcol_write(xp, in, out, ci, r);
}

// ---- exclusive prefix sums of a[0 .. n) in place, a[n] = the total (also stored at *total): block sums, scan of the block
// sums (one CTA), per-block scan.  kScanBlock elements per CTA.
constexpr uint32_t kScanThreads = 512, kScanPer = 8, kScanBlock = kScanThreads * kScanPer;
__device__ __forceinline__ uint32_t gk_block_scan_incl(uint32_t x, uint32_t* warp_sum) {   // inclusive scan over the CTA; warp_sum[16]
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
    if ((int)lane >= d) x += y;
  }
  if (lane == 31) warp_sum[warp] = x;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = lane < kScanThreads / 32 ? warp_sum[lane] : 0u;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, w, d);
      if ((int)lane >= d) w += y;
    }
    if (lane < kScanThreads / 32) warp_sum[lane] = w;
  }
  __syncthreads();
  const uint32_t r = x + (warp ? warp_sum[warp - 1] : 0u);
  __syncthreads();
  return r;
}
__global__ void __launch_bounds__(kScanThreads) gk_scan_sums_kernel(const uint32_t* a, uint32_t n, uint32_t* sums) {
  __shared__ uint32_t ws[kScanThreads / 32];
  const uint32_t base = blockIdx.x * kScanBlock + threadIdx.x * kScanPer;
  uint32_t s = 0;
#pragma unroll
  for (uint32_t u = 0; u < kScanPer; ++u) s += base + u < n ? a[base + u] : 0u;
  const uint32_t incl = gk_block_scan_incl(s, ws);
  if (threadIdx.x == kScanThreads - 1) sums[blockIdx.x] = incl;
}
__global__ void __launch_bounds__(kScanThreads) gk_scan_top_kernel(uint32_t* sums, uint32_t nb, uint32_t* total) {   // one CTA
  __shared__ uint32_t ws[kScanThreads / 32];
  __shared__ uint32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (uint32_t base = 0; base < nb; base += kScanThreads) {
    const uint32_t ix = base + threadIdx.x;
    const uint32_t v = ix < nb ? sums[ix] : 0u;
    const uint32_t incl = gk_block_scan_incl(v, ws);
    if (ix < nb) sums[ix] = carry + incl - v;
    __syncthreads();
    if (threadIdx.x == kScanThreads - 1) carry += incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry;
}
__global__ void __launch_bounds__(kScanThreads) gk_scan_apply_kernel(uint32_t* a, uint32_t n, const uint32_t* sums, const uint32_t* total, uint32_t tail) {
  __shared__ uint32_t ws[kScanThreads / 32];
  const uint32_t base = blockIdx.x * kScanBlock + threadIdx.x * kScanPer;
  uint32_t v[kScanPer];
  uint32_t s = 0;
#pragma unroll
  for (uint32_t u = 0; u < kScanPer; ++u) {
    v[u] = base + u < n ? a[base + u] : 0u;
    s += v[u];
  }
  const uint32_t incl = gk_block_scan_incl(s, ws);
  uint32_t excl = sums[blockIdx.x] + incl - s;
#pragma unroll
  for (uint32_t u = 0; u < kScanPer; ++u) {
    if (base + u < n) a[base + u] = excl;
    excl += v[u];
  }
  if (tail && blockIdx.x == 0 && threadIdx.x == 0) a[n] = *total;
}

// mm[0] = min, mm[1] = max of the non-zero entries of g (mm preset to ~0 / 0): is the batch of one (apiVersion, kind)?
__global__ void __launch_bounds__(256) gk_gvk_minmax_kernel(const unsigned long long* g, uint32_t n, unsigned long long* mm) {
  unsigned long long lo = ~0ull, hi = 0ull;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned long long v = g[i];
    if (v) lo = min(lo, v), hi = max(hi, v);
  }
#pragma unroll
  for (int d = 16; d; d >>= 1) {
    lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, d));
    hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, d));
  }
  if ((threadIdx.x & 31u) == 0u && hi) {
    atomicMin(&mm[0], lo);
    atomicMax(&mm[1], hi);
  }
}

// small host -> device transfers done by the SMs from mapped page-locked memory: they do not queue behind the next page's 32 MB
// chunks on the copy engine (a 100 KB table upload waited behind them there)
__global__ void __launch_bounds__(256) gk_push_kernel(uint8_t* dst, const uint8_t* src, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x * 16u;
  const bool vec = (reinterpret_cast<size_t>(dst) & 15u) == 0u;
  for (size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 16u; i < n; i += stride) {
    if (vec && i + 16u <= n) {
      *reinterpret_cast<uint4*>(dst + i) = *reinterpret_cast<const uint4*>(src + i);
    } else {
      for (size_t k = i; k < n && k < i + 16u; ++k) dst[k] = src[k];
    }
  }
}

// the page's bytes that missed lookups take as arguments, packed for the host (gk_compact_miss_spans): span k = (page offset,
// destination offset, length)
__global__ void gk_gather_kernel(uint8_t* dst, const uint8_t* blob, const unsigned long long* spans, uint32_t nspans) {
  for (uint32_t k = blockIdx.x; k < nspans; k += gridDim.x) {
    const unsigned long long src = spans[3 * k], to = spans[3 * k + 1], len = spans[3 * k + 2];
    for (unsigned long long i = threadIdx.x; i < len; i += blockDim.x) dst[to + i] = blob[src + i];
  }
}

// ---- gk_batch_patch: a kept page's staying objects moved into a new page
// len[j] = byte length of staying object keep[j] of the old page; len[n_keep] = 0, so that an exclusive scan over n_keep + 1
// entries gives the staying objects' offsets in the new page and, last, their total
__global__ void gk_keep_len_kernel(const unsigned long long* ooff, const uint32_t* keep, uint32_t n_keep, unsigned long long* len) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n_keep) len[j] = ooff[keep[j] + 1] - ooff[keep[j]];
  else if (j == n_keep) len[j] = 0;
}

// one warp copies len bytes in words of W, with byte copies before the first aligned destination word and after the last one
// (src and dst agree modulo sizeof(W))
template <class W>
__device__ void gk_warp_copy_words(uint8_t* dst, const uint8_t* src, unsigned long long len, uint32_t lane) {
  const unsigned long long head = min((unsigned long long)((sizeof(W) - (reinterpret_cast<size_t>(dst) & (sizeof(W) - 1))) & (sizeof(W) - 1)), len);
  for (unsigned long long k = lane; k < head; k += 32) dst[k] = src[k];
  const unsigned long long words = (len - head) / sizeof(W);
  W* d = reinterpret_cast<W*>(dst + head);
  const W* s = reinterpret_cast<const W*>(src + head);
  for (unsigned long long k = lane; k < words; k += 32) d[k] = s[k];
  for (unsigned long long k = head + words * sizeof(W) + lane; k < len; k += 32) dst[k] = src[k];
}
__device__ void gk_warp_copy(uint8_t* dst, const uint8_t* src, unsigned long long len, uint32_t lane) {
  const uint32_t mis = (uint32_t)((reinterpret_cast<size_t>(dst) ^ reinterpret_cast<size_t>(src)) & 15u);
  if (mis == 0u) gk_warp_copy_words<uint4>(dst, src, len, lane);
  else if ((mis & 7u) == 0u) gk_warp_copy_words<unsigned long long>(dst, src, len, lane);
  else if ((mis & 3u) == 0u) gk_warp_copy_words<uint32_t>(dst, src, len, lane);
  else gk_warp_copy_words<uint8_t>(dst, src, len, lane);
}

// One warp per staying object j (= old object keep[j]): its JSON bytes, its tape entries and its tape length and status word.
// Tape entries hold positions relative to the object's own first byte (gk_tape_obj tokenises in.blob + ooff[i] as a text of its
// own), so they move as they are; only where the tape starts, gk_tape_off of the object's offset, changes.  `blob`: to.blob, writable.
__global__ void __launch_bounds__(256) gk_splice_kernel(const GkIngestIn to, uint8_t* blob, const GkIngestIn from, const uint32_t* keep, uint32_t n_keep) {
  const uint32_t lane = threadIdx.x & 31u, warps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n_keep; j += warps) {
    const uint32_t i = keep[j];
    const unsigned long long a = from.ooff[i];
    gk_warp_copy(blob + to.ooff[j], from.blob + a, from.ooff[i + 1] - a, lane);
    const uint32_t nt = from.ntape[i];
    gk_warp_copy(reinterpret_cast<uint8_t*>(to.tape + gk_tape_off(to.ooff, j)), reinterpret_cast<const uint8_t*>(from.tape + gk_tape_off(from.ooff, i)),
                 (unsigned long long)nt * 8u, lane);
    if (lane == 0) {
      to.ntape[j] = nt;
      to.status[j] = from.status[i];
    }
  }
}

__global__ void gk_fill_kernel(uint32_t* vals, const uint32_t* pairs, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) vals[pairs[2 * i]] = pairs[2 * i + 1];
}

// tile_lo[t * NS + s] = first row of scope s in tile t (t = ntiles: the totals); cap[s] = rows of the largest tile.  The first row
// of a scope at an object boundary is found through the CSR offsets of the scope chain (scopes are numbered parents first).
__global__ void gk_tiles_kernel(const GkXProg xp, const GkIngestOut out, uint32_t n, uint32_t NS, uint32_t tile, uint32_t ntiles, uint32_t* tile_lo, uint32_t* cap) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t > ntiles) return;
  uint32_t* lo = tile_lo + (size_t)t * NS;
  lo[0] = min(t * tile, n);
  for (uint32_t s = 1; s < NS; ++s) lo[s] = out.scope_off[s][lo[xp.scopes[s].parent]];
  if (t < ntiles) {
    uint32_t prev = min((t + 1u) * tile, n);
    atomicMax(&cap[0], prev - lo[0]);
    // the tile's end rows: the same chain from the next boundary (recomputed: tile t + 1 may not have written yet)
    uint32_t hi[GK_MAX_SCOPES];
    hi[0] = prev;
    for (uint32_t s = 1; s < NS; ++s) {
      hi[s] = out.scope_off[s][hi[xp.scopes[s].parent]];
      atomicMax(&cap[s], hi[s] - lo[s]);
    }
  }
}

}  // namespace gk
