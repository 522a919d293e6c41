// blocks.cu -- device side of predict_instances_big's per-block bookkeeping (integer work, bit-exact).
//
// Reference: stardist/big.py:340-413 (BlockND.filter_objects: regionprops bounding box of every label ->
// is_responsible -> labels of the other objects zeroed), stardist/models/base.py:959 (relabel_sequential with the
// running label offset) and stardist/big.py:319-326 (BlockND.write: entries > 0 overwrite the write region, later
// blocks win).  Here the label tile never leaves HBM:
//   k_label_bbox        one pass over the context-cropped tile, per-label bounding box by warp-aggregated atomics
//   (host)              vectorised is_responsible on the [n, 2*nd] box table (a few thousand rows) -> lookup table
//   k_label_remap       tile[v] = lut[v]           (drops foreign objects, compacts ids to 1..n_kept)
//   k_label_write       dst[origin + idx] = tile[idx] + add   where tile[idx] > 0   (ordered by the caller's stream)
#include <algorithm>
#include "common.cuh"
#include "../../include/stardist_b200.h"

namespace {
using sdb::cdiv;

struct Dims { int nd; int shape[3]; };

// bbox[l] = {min0, min1, min2, max0, max1, max2} (inclusive), initialised to {INT_MAX.., -1..} by the caller's fill
__global__ void __launch_bounds__(256) k_label_bbox(const int* __restrict__ lab, Dims D, long long n, int max_label,
                                                    int* __restrict__ bbox, int* __restrict__ bad) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const int s1 = D.shape[1], s2 = D.shape[2], lane = threadIdx.x & 31;
  // warp-uniform trip count: every lane takes part in the match / reduce of each round
  for (long long base = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31); base < n; base += stride) {
    const long long i = base + lane;
    int v = i < n ? lab[i] : 0;
    if (v < 0 || v > max_label) { *bad = 1; v = 0; }
    const int c2 = (int)(i % s2); const long long q = i / s2;
    const int c1 = (int)(q % s1); const int c0 = (int)(q / s1);
    // lanes that hold the same label (runs along a row) share one set of atomics
    const unsigned m = __match_any_sync(0xffffffffu, v);
    const int lo0 = __reduce_min_sync(m, c0), lo1 = __reduce_min_sync(m, c1), lo2 = __reduce_min_sync(m, c2);
    const int hi0 = __reduce_max_sync(m, c0), hi1 = __reduce_max_sync(m, c1), hi2 = __reduce_max_sync(m, c2);
    if (v != 0 && lane == __ffs(m) - 1) {
      int* b = bbox + 6ll * v;
      if (lo0 < b[0]) atomicMin(b + 0, lo0);
      if (lo1 < b[1]) atomicMin(b + 1, lo1);
      if (lo2 < b[2]) atomicMin(b + 2, lo2);
      if (hi0 > b[3]) atomicMax(b + 3, hi0);
      if (hi1 > b[4]) atomicMax(b + 4, hi1);
      if (hi2 > b[5]) atomicMax(b + 5, hi2);
    }
  }
}

__global__ void k_bbox_init(int* bbox, int n_labels) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 6 * n_labels) bbox[i] = (i % 6) < 3 ? 0x7fffffff : -1;
}

__global__ void __launch_bounds__(256) k_label_remap(int* __restrict__ lab, long long n, const int* __restrict__ lut) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int v = lab[i];
    if (v) lab[i] = __ldg(lut + v);
  }
}

__global__ void __launch_bounds__(256) k_label_write(const int* __restrict__ tile, Dims T, long long n, int add,
                                                     int* __restrict__ dst, Dims G, int o0, int o1, int o2) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const int s1 = T.shape[1], s2 = T.shape[2];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int v = tile[i];
    if (v <= 0) continue;
    const int c2 = (int)(i % s2); const long long q = i / s2;
    const int c1 = (int)(q % s1); const int c0 = (int)(q / s1);
    dst[((long long)(o0 + c0) * G.shape[1] + (o1 + c1)) * G.shape[2] + (o2 + c2)] = v + add;
  }
}

static bool dims_from(int nd, const int* shape, Dims* D, long long* n) {
  if (nd < 1 || nd > 3) return false;
  D->nd = nd; D->shape[0] = D->shape[1] = D->shape[2] = 1;
  for (int i = 0; i < nd; ++i) { if (shape[i] < 0) return false; D->shape[3 - nd + i] = shape[i]; }
  *n = (long long)D->shape[0] * D->shape[1] * D->shape[2];
  return true;
}
}  // namespace

// Bounding boxes of the labels 1..max_label of a C-contiguous label tile.  d_bbox: int32[(max_label+1) * 6] =
// {min0,min1,min2,max0,max1,max2} per label over the LAST nd axes padded in front with a unit axis (2-D tiles use
// columns 1,2 and 4,5); labels that do not occur keep {INT_MAX.., -1..}.  d_bad[0] is set when a value lies outside
// [0, max_label].  big.py:367-373 (regionprops bbox) on the device.
extern "C" int sdb_label_bbox(const int* d_labels, int ndim, const int* shape, int max_label, int* d_bbox, int* d_bad,
                              sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  Dims D; long long n;
  if (!dims_from(ndim, shape, &D, &n) || max_label < 0) { sdb::set_error("label_bbox: bad shape"); return 1; }
  SDB_LAUNCH(k_bbox_init, cdiv(6ll * (max_label + 1), 256), 256, 0, st, d_bbox, max_label + 1);
  SDB_CUDA(cudaMemsetAsync(d_bad, 0, sizeof(int), st));
  if (n > 0) SDB_LAUNCH(k_label_bbox, (int)std::min<long long>(cdiv(n, 256), 132 * 16), 256, 0, st, d_labels, D, n, max_label, d_bbox, d_bad);
  return 0;
}

// In-place lookup: labels[i] = lut[labels[i]] for labels[i] != 0 (lut has max_label+1 entries, lut[0] ignored).
extern "C" int sdb_label_remap(int* d_labels, long long n, const int* d_lut, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n < 0) { sdb::set_error("label_remap: negative size"); return 1; }
  if (n > 0) SDB_LAUNCH(k_label_remap, (int)std::min<long long>(cdiv(n, 256), 132 * 16), 256, 0, st, d_labels, n, d_lut);
  return 0;
}

// BlockND.write (big.py:319-326) with the label offset of base.py:959 folded in: for every entry > 0 of the
// C-contiguous tile, dst[origin + index] = entry + add.  Calls on one stream execute in order, so later blocks win.
extern "C" int sdb_label_write(const int* d_tile, int ndim, const int* tile_shape, int add, int* d_dst, const int* dst_shape,
                               const int* origin, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  Dims T, G; long long n, ng;
  if (!dims_from(ndim, tile_shape, &T, &n) || !dims_from(ndim, dst_shape, &G, &ng)) { sdb::set_error("label_write: bad shape"); return 1; }
  int o[3] = {0, 0, 0};
  for (int i = 0; i < ndim; ++i) {
    o[3 - ndim + i] = origin[i];
    if (origin[i] < 0 || origin[i] + tile_shape[i] > dst_shape[i]) { sdb::set_error("label_write: tile outside the destination"); return 1; }
  }
  if (n > 0) SDB_LAUNCH(k_label_write, (int)std::min<long long>(cdiv(n, 256), 132 * 16), 256, 0, st, d_tile, T, n, add, d_dst, G, o[0], o[1], o[2]);
  return 0;
}
