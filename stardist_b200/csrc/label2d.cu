// label2d.cu -- dist_to_coord and polygon label painting for the 2D path.
//
// Reference: stardist/geometry/geom2d.py:130-146 (dist_to_coord), :149-166
// (polygons_to_label_coord: for each polygon, skimage.draw.polygon(r, c, shape) -> lbl[rr,cc]=id,
// later polygons overwrite earlier ones) and :169-197 (polygons_to_label: painted in ascending
// stable prob order, id = original index + 1).
//
// skimage is an un-vendored third-party dependency of the reference (setup.py:141, unpinned);
// the rule restated here is skimage >= 0.18 (skimage/draw/_draw.pyx::_polygon and
// skimage/_shared/geometry.pyx::point_in_polygon), see SURVEY A.4 / DESIGN.md:
//   minr = int(max(0, r.min())), maxr = int(ceil(r.max())) clipped to shape-1 (same for c);
//   pixel (r_i,c_i) is painted iff point_in_polygon(c, r, c_i, r_i) != OUTSIDE, in float64:
//   vertex hit (|dx|,|dy| < 1e-12), right/left crossing counts with the quotient test,
//   different parity -> on an edge (painted), else painted iff r_cross is odd.
// "Later overwrites earlier" is realised as a per-pixel atomicMax over the paint rank.
//
// Must be compiled with -fmad=false (the reference arithmetic is unfused float64).
#include <vector>
#include <algorithm>
#include "common.cuh"
#include "../../include/stardist_b200.h"

namespace {

using sdb::cdiv;

__global__ void k_dist_to_coord(const float* __restrict__ dist, const double* __restrict__ points, int n, int R,
                                const double* __restrict__ sincos, double sy, double sx,
                                float* __restrict__ coord) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)n * R) return;
  const int i = (int)(t / R), k = (int)(t % R);
  const double d = (double)dist[t];
  float cy = (float)(d * sincos[k]);          // (dist * sin(phi)).astype(float32)
  float cx = (float)(d * sincos[R + k]);
  // coord *= scale_dist  (float32 array times int64/float64 array: computed in float64, cast back)
  cy = (float)((double)cy * sy);
  cx = (float)((double)cx * sx);
  // coord += points[..., None]  (points: int64 -> exact in float64, or float64 after rescale)
  cy = (float)((double)cy + points[2 * i]);
  cx = (float)((double)cx + points[2 * i + 1]);
  coord[((size_t)i * 2 + 0) * R + k] = cy;
  coord[((size_t)i * 2 + 1) * R + k] = cx;
}

constexpr int MAXR = 512;

// one block per polygon; threads stride over the pixels of its clipped bounding box
__global__ void k_paint(const float* __restrict__ coord, const int* __restrict__ rank, int n, int R,
                        int ny, int nx, int* __restrict__ img) {
  __shared__ double sr[MAXR], sc[MAXR];
  __shared__ float red[4][32];
  __shared__ int box[4];
  const int p = blockIdx.x;
  const float* cr = coord + (size_t)p * 2 * R;
  const float* cc = cr + R;
  float rmin = INFINITY, rmax = -INFINITY, cmin = INFINITY, cmax = -INFINITY;
  for (int k = threadIdx.x; k < R; k += blockDim.x) {
    const float r = cr[k], c = cc[k];
    sr[k] = (double)r; sc[k] = (double)c;
    rmin = fminf(rmin, r); rmax = fmaxf(rmax, r); cmin = fminf(cmin, c); cmax = fmaxf(cmax, c);
  }
  for (int o = 16; o > 0; o >>= 1) {
    rmin = fminf(rmin, __shfl_xor_sync(0xffffffffu, rmin, o)); rmax = fmaxf(rmax, __shfl_xor_sync(0xffffffffu, rmax, o));
    cmin = fminf(cmin, __shfl_xor_sync(0xffffffffu, cmin, o)); cmax = fmaxf(cmax, __shfl_xor_sync(0xffffffffu, cmax, o));
  }
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { red[0][w] = rmin; red[1][w] = rmax; red[2][w] = cmin; red[3][w] = cmax; }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int nw = blockDim.x >> 5;
    for (int i = 1; i < nw; ++i) {
      rmin = fminf(rmin, red[0][i]); rmax = fmaxf(rmax, red[1][i]); cmin = fminf(cmin, red[2][i]); cmax = fmaxf(cmax, red[3][i]);
    }
    // int(max(0, r.min())), int(ceil(r.max())); maxr = min(shape-1, maxr)
    long long r0 = (rmin > 0.f) ? (long long)rmin : 0, r1 = (long long)ceil((double)rmax);
    long long c0 = (cmin > 0.f) ? (long long)cmin : 0, c1 = (long long)ceil((double)cmax);
    if (r1 > ny - 1) r1 = ny - 1;
    if (c1 > nx - 1) c1 = nx - 1;
    if (r0 > r1 || c0 > c1) { r0 = 0; r1 = -1; c0 = 0; c1 = -1; }
    box[0] = (int)r0; box[1] = (int)r1; box[2] = (int)c0; box[3] = (int)c1;
  }
  __syncthreads();
  const int r0 = box[0], r1 = box[1], c0 = box[2], c1 = box[3];
  if (r1 < r0) return;
  const int bw = c1 - c0 + 1;
  const long long npx = (long long)(r1 - r0 + 1) * bw;
  const int val = rank[p] + 1;
  for (long long q = threadIdx.x; q < npx; q += blockDim.x) {
    const int ri = r0 + (int)(q / bw), ci = c0 + (int)(q % bw);
    const double y = (double)ri, x = (double)ci;
    // point_in_polygon(xp = c, yp = r, x = c_i, y = r_i)
    unsigned int lcross = 0, rcross = 0;
    bool vertex = false;
    double x1 = sc[R - 1] - x, y1 = sr[R - 1] - y;
    for (int k = 0; k < R; ++k) {
      const double x0 = sc[k] - x, y0 = sr[k] - y;
      if ((-1e-12 < x0 && x0 < 1e-12) && (-1e-12 < y0 && y0 < 1e-12)) { vertex = true; break; }
      if ((y0 > 0) != (y1 > 0)) { if (((x0 * y1 - x1 * y0) / (y1 - y0)) > 0) rcross++; }
      if ((y0 < 0) != (y1 < 0)) { if (((x0 * y1 - x1 * y0) / (y1 - y0)) < 0) lcross++; }
      x1 = x0; y1 = y0;
    }
    bool inside;
    if (vertex) inside = true;
    else if ((rcross & 1u) != (lcross & 1u)) inside = true;      // on an edge
    else inside = (rcross & 1u) != 0;
    if (inside) atomicMax(&img[(size_t)ri * nx + ci], val);
  }
}

__global__ void k_rank_to_label(int* __restrict__ img, long long npix, const int* __restrict__ id_by_rank) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < npix; p += (long long)gridDim.x * blockDim.x) {
    const int v = img[p];
    if (v > 0) img[p] = id_by_rank[v - 1];
  }
}

}  // namespace

extern "C" int sdb_dist_to_coord_2d(const float* d_dist, const double* d_points, int n_polys, int n_rays,
                                    const double* d_sincos, double scale_y, double scale_x,
                                    float* d_coord, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n_polys <= 0) return 0;
  SDB_LAUNCH(k_dist_to_coord, cdiv((long long)n_polys * n_rays, 256), 256, 0, st, d_dist, d_points, n_polys, n_rays,
             d_sincos, scale_y, scale_x, d_coord);
  return 0;
}

extern "C" int sdb_polygons_to_label_2d(const float* d_coord, const int* d_rank, const int* d_id_by_rank,
                                        int n_polys, int n_rays, int ny, int nx, int* d_out,
                                        sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n_rays > MAXR) { sdb::set_error("polygons_to_label_2d: n_rays > 512"); return 1; }
  SDB_CUDA(cudaMemsetAsync(d_out, 0, (size_t)ny * nx * sizeof(int), st));
  if (n_polys <= 0) return 0;
  SDB_LAUNCH(k_paint, n_polys, 128, 0, st, d_coord, d_rank, n_polys, n_rays, ny, nx, d_out);
  const long long npix = (long long)ny * nx;
  SDB_LAUNCH(k_rank_to_label, (int)std::min<long long>(cdiv(npix, 256), 132 * 8), 256, 0, st, d_out, npix, d_id_by_rank);
  return 0;
}

// host ABI: paint in the given order, value labels[i]+1 (polygons_to_label_coord semantics)
extern "C" int _LIB_polygons_to_label_2d(const float* coord, const int* labels, const int n_polys,
                                         const int n_rays, const int ny, const int nx, int* result) {
  cudaStream_t st = 0;
  sdb::DevBuf d_coord, d_rank, d_ids, d_out;
  const size_t nc = (size_t)n_polys * 2 * n_rays;
  SDB_CUDA(d_coord.alloc(nc * sizeof(float), st));
  SDB_CUDA(d_rank.alloc((size_t)n_polys * sizeof(int), st));
  SDB_CUDA(d_ids.alloc((size_t)n_polys * sizeof(int), st));
  SDB_CUDA(d_out.alloc((size_t)ny * nx * sizeof(int), st));
  std::vector<int> rank(n_polys), ids(n_polys);
  for (int i = 0; i < n_polys; ++i) { rank[i] = i; ids[i] = labels[i] + 1; }
  if (n_polys > 0) {
    SDB_CUDA(cudaMemcpyAsync(d_coord.p, coord, nc * sizeof(float), cudaMemcpyHostToDevice, st));
    SDB_CUDA(cudaMemcpyAsync(d_rank.p, rank.data(), (size_t)n_polys * sizeof(int), cudaMemcpyHostToDevice, st));
    SDB_CUDA(cudaMemcpyAsync(d_ids.p, ids.data(), (size_t)n_polys * sizeof(int), cudaMemcpyHostToDevice, st));
  }
  int rc = sdb_polygons_to_label_2d(d_coord.as<float>(), d_rank.as<int>(), d_ids.as<int>(), n_polys, n_rays, ny, nx,
                                    d_out.as<int>(), (sdb_stream_t)st);
  if (rc) return rc;
  SDB_CUDA(cudaMemcpyAsync(result, d_out.p, (size_t)ny * nx * sizeof(int), cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  return 0;
}
