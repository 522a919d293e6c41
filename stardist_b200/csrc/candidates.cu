// candidates.cu -- prob threshold + border mask + compaction, score sort, candidate gather.
//
// Reference: stardist/nms.py:6-17 (_ind_prob_thresh), stardist/models/base.py:553-557,606-621
// (prob > thresh minus b-pixel border, gather prob/dist rows, points = index*grid, drop points in
// the padded region, StarDistPadAndCropResizer.filter_points base.py:1204-1211) and
// stardist/nms.py:167,313 (np.argsort(prob)[::-1]).
//
// The reference's argsort is unstable (tie order is machine dependent, SURVEY H5).  This
// implementation defines the order as  np.argsort(prob, kind='stable')[::-1]  == (prob desc,
// flat index desc); the oracle restatement uses the same definition.  It is realised by sorting
// unique 64-bit keys (order_bits(prob) << 32 | flat_index) ascending with a bitonic network and
// reading the result back to front -- no stability requirement, fully deterministic.
#include <vector>
#include <algorithm>
#include "common.cuh"
#include "bitonic.cuh"
#include "../../include/stardist_b200.h"

namespace {

using sdb::cdiv;
using sdb::bitonic::BTILE;
typedef unsigned long long u64;

struct ShapeDesc {
  int ndim;
  int shape[3];
  int valid[3];
  int blo[3], bhi[3];
};

__global__ void k_threshold(const float* __restrict__ prob, long long npix, ShapeDesc S, float thr,
                            u64* __restrict__ keys, unsigned int* __restrict__ count, unsigned int capacity) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += (long long)gridDim.x * blockDim.x) {
    const float v = prob[p];
    if (!(v > thr)) continue;
    long long r = p;
    bool ok = true;
    for (int a = S.ndim - 1; a >= 0; --a) {
      const int c = (int)(r % S.shape[a]); r /= S.shape[a];
      ok = ok && (c >= S.blo[a]) && (c < S.shape[a] - S.bhi[a]) && (c < S.valid[a]);
    }
    if (!ok) continue;
    const unsigned int pos = atomicAdd(count, 1u);
    if (pos < capacity) keys[pos] = ((u64)sdb::float_order_key(v) << 32) | (u64)(unsigned int)p;
  }
}

__global__ void k_emit_sorted(const u64* __restrict__ keys, unsigned int n, const float* __restrict__ prob,
                              int* __restrict__ out_index, float* __restrict__ out_prob) {
  unsigned int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const unsigned int idx = (unsigned int)(keys[n - 1 - r] & 0xffffffffull);
  out_index[r] = (int)idx;
  out_prob[r] = prob[idx];
}

__global__ void k_gather(const float* __restrict__ dist, const int* __restrict__ index, int n, int R,
                         ShapeDesc S, int g0, int g1, int g2, float* __restrict__ out_dist,
                         float* __restrict__ out_points, const int* __restrict__ slot) {
  // one warp per candidate row: coalesced 4*R byte row copy
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= n) return;
  const long long idx = index[row];
  const long long src = slot ? (long long)slot[idx] : idx;      // dense map row, or the row of the sparse candidate store
  for (int k = lane; k < R; k += 32) {
    const float d = dist[src * R + k];
    out_dist[(size_t)row * R + k] = fmaxf(1e-3f, d);     // np.maximum(1e-3, dist), base.py:556
  }
  if (lane == 0) {
    long long r = idx;
    int c[3] = {0, 0, 0};
    for (int a = S.ndim - 1; a >= 0; --a) { c[a] = (int)(r % S.shape[a]); r /= S.shape[a]; }
    const int g[3] = {g0, g1, g2};
    for (int a = 0; a < S.ndim; ++a) out_points[(size_t)row * S.ndim + a] = (float)(c[a] * g[a]);
  }
}

}  // namespace

extern "C" int sdb_threshold_sort(const float* d_prob, int ndim, const int* shape, const int* valid_shape,
                                  const int* b_lo, const int* b_hi, float prob_thresh,
                                  int* d_sorted_index, float* d_sorted_prob, int capacity, int* h_count,
                                  sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (ndim < 1 || ndim > 3) { sdb::set_error("threshold_sort: ndim must be 1..3"); return 1; }
  ShapeDesc S; S.ndim = ndim;
  long long npix = 1;
  for (int a = 0; a < 3; ++a) {
    S.shape[a] = a < ndim ? shape[a] : 1; S.valid[a] = a < ndim ? valid_shape[a] : 1;
    S.blo[a] = a < ndim ? b_lo[a] : 0; S.bhi[a] = a < ndim ? b_hi[a] : 0;
    npix *= S.shape[a];
  }
  if (npix >= (1ll << 32)) { sdb::set_error("threshold_sort: more than 2^32 pixels"); return 1; }
  *h_count = 0;
  if (npix == 0 || capacity <= 0) return 0;
  // keys buffer sized to the next power of two of capacity
  const unsigned int cap_pad = sdb::bitonic::padded_length((unsigned int)capacity);
  sdb::DevBuf b_keys, b_count;
  SDB_CUDA(b_keys.alloc((size_t)cap_pad * sizeof(u64), st));
  SDB_CUDA(b_count.alloc(sizeof(unsigned int), st));
  SDB_CUDA(cudaMemsetAsync(b_count.p, 0, sizeof(unsigned int), st));
  const int blocks = (int)std::min<long long>(cdiv(npix, 256), 132 * 16);
  SDB_LAUNCH(k_threshold, blocks, 256, 0, st, d_prob, npix, S, prob_thresh, b_keys.as<u64>(), b_count.as<unsigned int>(), (unsigned int)capacity);
  unsigned int n = 0;
  SDB_CUDA(cudaMemcpyAsync(&n, b_count.p, sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  if (n > (unsigned int)capacity) { sdb::set_error("threshold_sort: candidate capacity exceeded"); return 1; }
  *h_count = (int)n;
  if (n == 0) return 0;
  if (sdb::bitonic::sort(b_keys.as<u64>(), n, sdb::bitonic::padded_length(n), st)) return 1;
  SDB_LAUNCH(k_emit_sorted, cdiv(n, 256), 256, 0, st, b_keys.as<u64>(), n, d_prob, d_sorted_index, d_sorted_prob);
  return 0;
}

extern "C" int sdb_gather_candidates(const float* d_dist, const int* d_index, int n, int n_rays, int ndim,
                                     const int* shape, const int* grid, float* d_out_dist,
                                     float* d_out_points, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n <= 0) return 0;
  ShapeDesc S; S.ndim = ndim;
  int g[3] = {1, 1, 1};
  for (int a = 0; a < 3; ++a) { S.shape[a] = a < ndim ? shape[a] : 1; S.valid[a] = S.shape[a]; S.blo[a] = S.bhi[a] = 0; if (a < ndim) g[a] = grid[a]; }
  SDB_LAUNCH(k_gather, cdiv((long long)n * 32, 256), 256, 0, st, d_dist, d_index, n, n_rays, S, g[0], g[1], g[2], d_out_dist, d_out_points, (const int*)nullptr);
  return 0;
}

// ---- sparse candidate store (SURVEY H7; the reference's per-tile sparse gather, base.py:580-593): the dense dist map of a
// large volume is never materialised -- the heads run slab by slab and only the rows of voxels with prob > thresh are kept.
namespace {
__global__ void __launch_bounds__(256) k_count_above(const float* __restrict__ prob, long long n, float thr, unsigned int* __restrict__ count) {
  unsigned int c = 0;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (long long)gridDim.x * blockDim.x) c += prob[p] > thr ? 1u : 0u;
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, c);
}
// warp per 32 voxels: the voxels above the threshold get a row (atomic counter), the warp copies their dist rows
__global__ void __launch_bounds__(256) k_store_rows(const float* __restrict__ prob, const float* __restrict__ dist, long long n, int R, float thr,
                                                    long long flat0, unsigned int row0, unsigned int capacity, unsigned int* __restrict__ counter,
                                                    float* __restrict__ store, int* __restrict__ slot) {
  const int lane = threadIdx.x & 31;
  const long long warps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long base = (((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 32; base < n; base += warps * 32) {
    const long long p = base + lane;
    const bool hit = p < n && prob[p] > thr;
    unsigned int m = __ballot_sync(0xffffffffu, hit);
    while (m) {
      const int src = __ffs(m) - 1; m &= m - 1;
      unsigned int r = 0;
      if (lane == 0) r = atomicAdd(counter, 1u);
      r = __shfl_sync(0xffffffffu, r, 0);
      if (r >= capacity) continue;
      const long long q = base + src;
      for (int k = lane; k < R; k += 32) store[(size_t)r * R + k] = dist[q * R + k];
      if (lane == 0) slot[flat0 + q] = (int)(row0 + r);
    }
  }
}
}  // namespace

// number of entries of d_prob[n] above thresh (one 4-byte read-back, stream synchronised)
extern "C" int sdb_count_above(const float* d_prob, long long n, float thresh, int* h_count, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  sdb::DevBuf b; SDB_CUDA(b.alloc(4, st)); SDB_CUDA(cudaMemsetAsync(b.p, 0, 4, st));
  if (n > 0) SDB_LAUNCH(k_count_above, (int)std::min<long long>(cdiv(n, 1024), 132 * 8), 256, 0, st, d_prob, n, thresh, b.as<unsigned int>());
  unsigned int h = 0;
  SDB_CUDA(cudaMemcpyAsync(&h, b.p, 4, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  *h_count = (int)h;
  return 0;
}
// rows of d_dist[n, n_rays] whose d_prob[i] > thresh -> d_store[capacity, n_rays] (row order arbitrary), d_slot[flat0 + i] =
// row0 + row.  capacity must be >= sdb_count_above of the same slab.
extern "C" int sdb_store_rows_above(const float* d_prob, const float* d_dist, long long n, int n_rays, float thresh, long long flat0,
                                    int row0, int capacity, float* d_store, int* d_slot, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n <= 0 || capacity <= 0) return 0;
  sdb::DevBuf b; SDB_CUDA(b.alloc(4, st)); SDB_CUDA(cudaMemsetAsync(b.p, 0, 4, st));
  SDB_LAUNCH(k_store_rows, (int)std::min<long long>(cdiv(n, 256), 132 * 16), 256, 0, st, d_prob, d_dist, n, n_rays, thresh, flat0, (unsigned int)row0,
             (unsigned int)capacity, b.as<unsigned int>(), d_store, d_slot);
  return 0;
}
// sdb_gather_candidates from the sparse store: out_dist[r,:] = max(1e-3, store[slot[idx[r]],:])
extern "C" int sdb_gather_candidates_slots(const float* d_store, const int* d_slot, const int* d_index, int n, int n_rays, int ndim,
                                           const int* shape, const int* grid, float* d_out_dist, float* d_out_points, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n <= 0) return 0;
  ShapeDesc S; S.ndim = ndim;
  int g[3] = {1, 1, 1};
  for (int a = 0; a < 3; ++a) { S.shape[a] = a < ndim ? shape[a] : 1; S.valid[a] = S.shape[a]; S.blo[a] = S.bhi[a] = 0; if (a < ndim) g[a] = grid[a]; }
  SDB_LAUNCH(k_gather, cdiv((long long)n * 32, 256), 256, 0, st, d_store, d_index, n, n_rays, S, g[0], g[1], g[2], d_out_dist, d_out_points, d_slot);
  return 0;
}
