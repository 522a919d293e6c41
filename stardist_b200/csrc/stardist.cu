// stardist.cu -- star distances of a label map (star_dist / star_dist3D) and per-label region statistics.
//
// Reference: stardist/lib/stardist2d.cpp:55-125 (c_star_dist) and stardist3d.cpp:245-345 (c_star_dist3d).  For every
// output pixel (the label map subsampled by the grid) and every ray, walk from the pixel in unit steps of the ray
// direction until the rounded position leaves the image or reaches a different label; labels are compared as uint16
// (the reference reads the map after `astype(np.uint16)`).  Every float operation is the reference's, one float32 op
// at a time in its order (this unit is compiled with -fmad=false and uses the _rn intrinsics where a contraction could
// otherwise happen), so the distances are bit-identical to the reference's C++.
//
// One warp per output pixel, lanes over the rays: a pixel's R floats are written as one coalesced run and a background
// pixel exits uniformly per warp.  The walk is bounded: sdb_star_dist_walk_bound (host) rejects ray sets that could
// stall for the given shape and returns the step count after which every walk has left the image; the kernels use it
// as a hard cap (unreachable for accepted inputs; reaching it would write NaN).  sdb_star_dist_batch walks a batch of maps
// laid end to end, each on its own, and writes every pixel's R floats at a stride (the dist_and_mask layout of training).
#include <algorithm>
#include <climits>
#include <cmath>
#include "common.cuh"
#include "../../include/stardist_b200.h"

namespace {

using sdb::cdiv;

constexpr int SD_WARPS = 8;                 // output pixels per CTA
constexpr int SD_THREADS = SD_WARPS * 32;

template <typename T>
__device__ __forceinline__ unsigned short lbl16(const T* __restrict__ p, long long i) {
  return (unsigned short)__ldg(p + i);      // low 16 bits: the reference's astype(np.uint16)
}

// 2-D: dirs = [dy | dx] (dy = cosf(phi_k) pairs with the column, dx = sinf(phi_k) with the row, stardist2d.cpp:92-104)
template <typename T>
__global__ void __launch_bounds__(SD_THREADS) k_star_dist_2d(const T* __restrict__ lbl, int H, int W, int gy, int gx, int Ho, int Wo,
                                                             const float* __restrict__ dirs, int R, const int* __restrict__ points,
                                                             long long n_out, long long n_item, int ostride, long long cap,
                                                             float* __restrict__ out) {
  const long long p = (long long)blockIdx.x * SD_WARPS + (threadIdx.x >> 5);
  if (p >= n_out) return;
  const int lane = threadIdx.x & 31;
  const long long b = p / n_item, q = p - b * n_item;       // batch item, output pixel within it
  lbl += b * H * W;
  float* o = out + p * ostride;
  int i, j;
  if (points) {
    i = points[2 * q]; j = points[2 * q + 1];
    if (i < 0 || i >= Ho || j < 0 || j >= Wo) {           // the callers validate; never read outside the map
      for (int k = lane; k < R; k += 32) o[k] = __int_as_float(0x7fc00000);
      return;
    }
  } else {
    i = (int)(q / Wo); j = (int)(q - (long long)i * Wo);
  }
  const int pi = i * gy, pj = j * gx;
  const unsigned short value = lbl16(lbl, (long long)pi * W + pj);
  if (value == 0) {
    for (int k = lane; k < R; k += 32) o[k] = 0.f;
    return;
  }
  const float fi = __int2float_rn(pi), fj = __int2float_rn(pj);
  for (int k = lane; k < R; k += 32) {
    const float dy = dirs[k], dx = dirs[R + k];
    float x = 0.f, y = 0.f, d = __int_as_float(0x7fc00000);
    for (long long s = 0; s < cap; ++s) {
      x = __fadd_rn(x, dx);
      y = __fadd_rn(y, dy);
      const int ii = __float2int_rn(__fadd_rn(fi, x)), jj = __float2int_rn(__fadd_rn(fj, y));
      if (ii < 0 || ii >= H || jj < 0 || jj >= W || value != lbl16(lbl, (long long)ii * W + jj)) {
        // half-step correction for the overshoot: t_corr = .5f/fmax(|dx|,|dy|); x += (t_corr-1)*dx; sqrt(x*x+y*y)
        const float t1 = __fsub_rn(__fdiv_rn(0.5f, fmaxf(fabsf(dx), fabsf(dy))), 1.f);
        x = __fadd_rn(x, __fmul_rn(t1, dx));
        y = __fadd_rn(y, __fmul_rn(t1, dy));
        d = __fsqrt_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)));
        break;
      }
    }
    o[k] = d;
  }
}

// 3-D: rays = [dz | dy | dx]; the exit distance is sqrt(double(x2*x2 + y2*y2 + z2*z2)) of the rounded offsets, no correction
template <typename T>
__global__ void __launch_bounds__(SD_THREADS) k_star_dist_3d(const T* __restrict__ lbl, int D, int H, int W, int gz, int gy, int gx,
                                                             int Do, int Ho, int Wo, const float* __restrict__ rays, int R,
                                                             const int* __restrict__ points, long long n_out, long long n_item,
                                                             int ostride, long long cap, float* __restrict__ out) {
  const long long p = (long long)blockIdx.x * SD_WARPS + (threadIdx.x >> 5);
  if (p >= n_out) return;
  const int lane = threadIdx.x & 31;
  const long long b = p / n_item, q = p - b * n_item;
  lbl += b * D * H * W;
  float* o = out + p * ostride;
  int i, j, l;
  if (points) {
    i = points[3 * q]; j = points[3 * q + 1]; l = points[3 * q + 2];
    if (i < 0 || i >= Do || j < 0 || j >= Ho || l < 0 || l >= Wo) {
      for (int k = lane; k < R; k += 32) o[k] = __int_as_float(0x7fc00000);
      return;
    }
  } else {
    const long long plane = (long long)Ho * Wo;
    i = (int)(q / plane);
    const long long r = q - (long long)i * plane;
    j = (int)(r / Wo); l = (int)(r - (long long)j * Wo);
  }
  const int pi = i * gz, pj = j * gy, pl = l * gx;
  const unsigned short value = lbl16(lbl, ((long long)pi * H + pj) * W + pl);
  if (value == 0) {
    for (int k = lane; k < R; k += 32) o[k] = 0.f;
    return;
  }
  const float fi = __int2float_rn(pi), fj = __int2float_rn(pj), fl = __int2float_rn(pl);
  for (int k = lane; k < R; k += 32) {
    const float dz = rays[k], dy = rays[R + k], dx = rays[2 * R + k];
    float x = 0.f, y = 0.f, z = 0.f, d = __int_as_float(0x7fc00000);
    for (long long s = 0; s < cap; ++s) {
      x = __fadd_rn(x, dx);
      y = __fadd_rn(y, dy);
      z = __fadd_rn(z, dz);
      const int ii = __float2int_rn(__fadd_rn(fi, z)), jj = __float2int_rn(__fadd_rn(fj, y)), kk = __float2int_rn(__fadd_rn(fl, x));
      if (ii < 0 || ii >= D || jj < 0 || jj >= H || kk < 0 || kk >= W || value != lbl16(lbl, ((long long)ii * H + jj) * W + kk)) {
        const int x2 = __float2int_rn(x), y2 = __float2int_rn(y), z2 = __float2int_rn(z);
        d = __double2float_rn(__dsqrt_rn((double)(x2 * x2 + y2 * y2 + z2 * z2)));
        break;
      }
    }
    o[k] = d;
  }
}

// region statistics: every thread takes a run of RS_SEG pixels of one row (last axis) and flushes each run of equal labels
// with one set of atomics (label maps are spatially coherent, so runs are long)
constexpr int RS_SEG = 32;

__global__ void k_region_stats(const int* __restrict__ lbl, int ndim, int ny, int nx, int nseg, long long n_work, int n_labels,
                               unsigned long long* __restrict__ count, unsigned long long* __restrict__ sum, int* __restrict__ bmin,
                               int* __restrict__ bmax, unsigned int* __restrict__ bad) {
  for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < n_work; w += (long long)gridDim.x * blockDim.x) {
    const long long row = w / nseg;
    const int seg = (int)(w - row * nseg);
    const int z = (int)(row / ny), y = (int)(row - (long long)z * ny);
    const int x0 = seg * RS_SEG, x1 = min(x0 + RS_SEG, nx);
    const int* r = lbl + row * nx;
    int cur = 0, start = x0;
    for (int x = x0; x <= x1; ++x) {
      const int v = x < x1 ? __ldg(r + x) : 0;                         // 0 at the end flushes the last run
      if (v == cur) continue;
      if (cur > 0) {
        if (cur > n_labels) {
          atomicOr(bad, 2u);
        } else {
          const int b = cur - 1;
          const unsigned long long c = (unsigned long long)(x - start);
          const unsigned long long sx = (unsigned long long)(start + x - 1) * c / 2;   // start + ... + (x - 1)
          atomicAdd(count + b, c);
          const int coord[3] = {z, y, 0};
          const int* c0 = coord + (3 - ndim);                          // 2-D: (y, x), 3-D: (z, y, x)
          for (int a = 0; a < ndim - 1; ++a) {
            atomicAdd(sum + (long long)b * ndim + a, c * (unsigned long long)c0[a]);
            atomicMin(bmin + (long long)b * ndim + a, c0[a]);
            atomicMax(bmax + (long long)b * ndim + a, c0[a]);
          }
          atomicAdd(sum + (long long)b * ndim + ndim - 1, sx);
          atomicMin(bmin + (long long)b * ndim + ndim - 1, start);
          atomicMax(bmax + (long long)b * ndim + ndim - 1, x - 1);
        }
      }
      if (v < 0) atomicOr(bad, 1u);
      cur = v; start = x;
    }
  }
}

}  // namespace

extern "C" int sdb_star_dist_walk_bound(const float* h_dirs, int ndim, int n_rays, const int* shape, long long* h_cap) {
  if ((ndim != 2 && ndim != 3) || n_rays < 1) { sdb::set_error("star_dist: ndim must be 2 or 3 and n_rays >= 1"); return 1; }
  int ext = 0;
  for (int a = 0; a < ndim; ++a) {
    if (shape[a] < 1 || shape[a] > (1 << 22)) { sdb::set_error("star_dist: every image extent must lie in [1, 2^22]"); return 1; }
    ext = std::max(ext, shape[a]);
  }
  // a walk has left the image once the offset along any axis reaches S = max extent + 1 in magnitude.  Positions stay below
  // M = S + max|component| in magnitude, where float32 rounding moves a sum by at most u/2, u = ulp(M); along the ray's
  // largest component m the offset thus grows by at least m - u/2 per step.  Requiring m >= 2^-8 and m >= 2u bounds the
  // walk by S / (m - u/2) steps.
  float dmax = 0.f;
  for (long long k = 0; k < (long long)ndim * n_rays; ++k) dmax = std::max(dmax, std::fabs(h_dirs[k]));
  if (!(dmax <= 1e6f)) { sdb::set_error("star_dist: ray components must be finite"); return 1; }
  const double S = (double)ext + 1.0, M = S + (double)dmax;
  const double u = std::ldexp(1.0, std::ilogb(M) - 23);
  long long cap = 0;
  for (int k = 0; k < n_rays; ++k) {
    float m = 0.f;
    for (int a = 0; a < ndim; ++a) m = std::max(m, std::fabs(h_dirs[(long long)a * n_rays + k]));
    if (!(m >= 1.0f / 256.0f) || !((double)m >= 2.0 * u)) {
      char b[256];
      snprintf(b, sizeof(b), "star_dist: ray %d has largest component %g; every ray needs one >= max(2^-8, %g) for an image "
               "extent of %d, or its walk is not bounded", k, (double)m, 2.0 * u, ext);
      sdb::set_error(b);
      return 1;
    }
    cap = std::max(cap, (long long)std::ceil(S / ((double)m - 0.5 * u)) + 2);
  }
  *h_cap = cap;
  return 0;
}

namespace {

// shared by the 2-D and 3-D entry points: bound, table upload, launch
// batch maps of `shape` laid end to end (dense mode only for batch > 1); output pixel p of the whole batch is written at
// d_out + p * ostride (ostride = n_rays for a plain [..., n_rays] map)
int star_dist_launch(int ndim, const void* d_labels, int label_bytes, int batch, const int* shape, const int* grid, int n_rays,
                     const float* h_dirs, const int* d_points, long long n_points, int ostride, float* d_out, cudaStream_t st) {
  if (label_bytes != 2 && label_bytes != 4) { sdb::set_error("star_dist: labels must be uint16 (2 bytes) or int32 (4 bytes)"); return 1; }
  if (batch < 1 || (batch > 1 && d_points) || ostride < n_rays) {
    sdb::set_error("star_dist: batch must be >= 1 (1 in point mode) and the output stride >= n_rays"); return 1;
  }
  int oshape[3];
  for (int a = 0; a < ndim; ++a) {
    if (grid[a] < 1) { sdb::set_error("star_dist: grid values must be >= 1"); return 1; }
    oshape[a] = (shape[a] - 1) / grid[a] + 1;
  }
  long long cap = 0;
  if (sdb_star_dist_walk_bound(h_dirs, ndim, n_rays, shape, &cap)) return 1;
  if (n_points < 0) { sdb::set_error("star_dist: n_points must be >= 0"); return 1; }
  long long n_item = n_points;
  if (!d_points) { n_item = 1; for (int a = 0; a < ndim; ++a) n_item *= oshape[a]; }
  if (n_item == 0) return 0;
  const long long n_out = n_item * batch;
  sdb::DevBuf d_dirs;
  SDB_CUDA(d_dirs.alloc((size_t)ndim * n_rays * sizeof(float), st));
  SDB_CUDA(cudaMemcpyAsync(d_dirs.p, h_dirs, (size_t)ndim * n_rays * sizeof(float), cudaMemcpyHostToDevice, st));
  const long long blocks = (n_out + SD_WARPS - 1) / SD_WARPS;
  if (blocks > INT_MAX) { sdb::set_error("star_dist: too many output pixels"); return 1; }
  if (ndim == 2) {
    if (label_bytes == 2)
      SDB_LAUNCH(k_star_dist_2d<unsigned short>, (int)blocks, SD_THREADS, 0, st, (const unsigned short*)d_labels, shape[0], shape[1],
                 grid[0], grid[1], oshape[0], oshape[1], d_dirs.as<float>(), n_rays, d_points, n_out, n_item, ostride, cap, d_out);
    else
      SDB_LAUNCH(k_star_dist_2d<int>, (int)blocks, SD_THREADS, 0, st, (const int*)d_labels, shape[0], shape[1],
                 grid[0], grid[1], oshape[0], oshape[1], d_dirs.as<float>(), n_rays, d_points, n_out, n_item, ostride, cap, d_out);
  } else {
    if (label_bytes == 2)
      SDB_LAUNCH(k_star_dist_3d<unsigned short>, (int)blocks, SD_THREADS, 0, st, (const unsigned short*)d_labels, shape[0], shape[1],
                 shape[2], grid[0], grid[1], grid[2], oshape[0], oshape[1], oshape[2], d_dirs.as<float>(), n_rays, d_points, n_out,
                 n_item, ostride, cap, d_out);
    else
      SDB_LAUNCH(k_star_dist_3d<int>, (int)blocks, SD_THREADS, 0, st, (const int*)d_labels, shape[0], shape[1],
                 shape[2], grid[0], grid[1], grid[2], oshape[0], oshape[1], oshape[2], d_dirs.as<float>(), n_rays, d_points, n_out,
                 n_item, ostride, cap, d_out);
  }
  return 0;
}

// host-pointer entry points: void like the reference's C functions; on failure the result is zeroed and the message is
// left in sdb_last_error(), on success it is cleared
void star_dist_host(int ndim, const unsigned short* src, const int* shape, const int* grid, int n_rays, const float* dirs,
                    float* dst) {
  cudaStream_t st = 0;
  long long n_in = 1, n_out = n_rays;
  for (int a = 0; a < ndim; ++a) { n_in *= shape[a]; n_out *= (shape[a] - 1) / std::max(grid[a], 1) + 1; }
  auto run = [&]() -> int {
    sdb::DevBuf d_src, d_dst;
    SDB_CUDA(d_src.alloc((size_t)n_in * 2, st));
    SDB_CUDA(d_dst.alloc((size_t)n_out * 4, st));
    SDB_CUDA(cudaMemcpyAsync(d_src.p, src, (size_t)n_in * 2, cudaMemcpyHostToDevice, st));
    if (star_dist_launch(ndim, d_src.p, 2, 1, shape, grid, n_rays, dirs, nullptr, 0, n_rays, d_dst.as<float>(), st)) return 1;
    SDB_CUDA(cudaMemcpyAsync(dst, d_dst.p, (size_t)n_out * 4, cudaMemcpyDeviceToHost, st));
    SDB_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  if (run()) {
    for (long long i = 0; i < n_out; ++i) dst[i] = 0.f;
    cudaGetLastError();
    return;
  }
  sdb::set_error("");
}

}  // namespace

extern "C" int sdb_star_dist_2d(const void* d_labels, int label_bytes, int H, int W, int grid_y, int grid_x, int n_rays,
                                const float* h_dirs, const int* d_points, long long n_points, float* d_out, sdb_stream_t stream) {
  const int shape[2] = {H, W}, grid[2] = {grid_y, grid_x};
  return star_dist_launch(2, d_labels, label_bytes, 1, shape, grid, n_rays, h_dirs, d_points, n_points, n_rays, d_out, (cudaStream_t)stream);
}

extern "C" int sdb_star_dist_3d(const void* d_labels, int label_bytes, int D, int H, int W, int grid_z, int grid_y, int grid_x,
                                int n_rays, const float* h_rays, const int* d_points, long long n_points, float* d_out,
                                sdb_stream_t stream) {
  const int shape[3] = {D, H, W}, grid[3] = {grid_z, grid_y, grid_x};
  return star_dist_launch(3, d_labels, label_bytes, 1, shape, grid, n_rays, h_rays, d_points, n_points, n_rays, d_out, (cudaStream_t)stream);
}

extern "C" int sdb_star_dist_batch(const int* d_labels, int ndim, int batch, const int* shape, const int* grid, int n_rays,
                                   const float* h_dirs, int out_stride, float* d_out, sdb_stream_t stream) {
  if (ndim != 2 && ndim != 3) { sdb::set_error("star_dist: ndim must be 2 or 3"); return 1; }
  return star_dist_launch(ndim, d_labels, 4, batch, shape, grid, n_rays, h_dirs, nullptr, 0, out_stride, d_out, (cudaStream_t)stream);
}

extern "C" void _LIB_star_dist_2d(const unsigned short* src, int H, int W, int n_rays, int grid_y, int grid_x, const float* dirs,
                                  float* dst) {
  const int shape[2] = {H, W}, grid[2] = {grid_y, grid_x};
  star_dist_host(2, src, shape, grid, n_rays, dirs, dst);
}

extern "C" void _LIB_star_dist_3d(const unsigned short* src, int D, int H, int W, int n_rays, int grid_z, int grid_y, int grid_x,
                                  const float* rays, float* dst) {
  const int shape[3] = {D, H, W}, grid[3] = {grid_z, grid_y, grid_x};
  star_dist_host(3, src, shape, grid, n_rays, rays, dst);
}

extern "C" int sdb_region_stats(const int* d_labels, int ndim, const int* shape, int n_labels, long long* d_count, long long* d_sum,
                                int* d_bbox_min, int* d_bbox_max, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if ((ndim != 2 && ndim != 3) || n_labels < 0) { sdb::set_error("region_stats: ndim must be 2 or 3 and n_labels >= 0"); return 1; }
  long long rows = 1;
  for (int a = 0; a < ndim; ++a) {
    if (shape[a] < 0) { sdb::set_error("region_stats: negative extent"); return 1; }
    if (a < ndim - 1) rows *= shape[a];
  }
  const int ny = ndim == 3 ? shape[1] : shape[0], nx = shape[ndim - 1];
  if (n_labels > 0) {
    SDB_CUDA(cudaMemsetAsync(d_count, 0, (size_t)n_labels * 8, st));
    SDB_CUDA(cudaMemsetAsync(d_sum, 0, (size_t)n_labels * ndim * 8, st));
    SDB_CUDA(cudaMemsetAsync(d_bbox_min, 0x7f, (size_t)n_labels * ndim * 4, st));     // 0x7f7f7f7f > any coordinate
    SDB_CUDA(cudaMemsetAsync(d_bbox_max, 0xff, (size_t)n_labels * ndim * 4, st));     // -1
  }
  if (rows == 0 || nx == 0) return 0;
  const int nseg = cdiv(nx, RS_SEG);
  const long long n_work = rows * nseg;
  sdb::DevBuf b_bad;
  SDB_CUDA(b_bad.alloc(sizeof(unsigned int), st));
  SDB_CUDA(cudaMemsetAsync(b_bad.p, 0, sizeof(unsigned int), st));
  SDB_LAUNCH(k_region_stats, (int)std::min<long long>(cdiv(n_work, 256), 132 * 16), 256, 0, st, d_labels, ndim, ny, nx, nseg, n_work,
             n_labels, (unsigned long long*)d_count, (unsigned long long*)d_sum, d_bbox_min, d_bbox_max, b_bad.as<unsigned int>());
  unsigned int* h_bad = sdb::pinned_scratch();
  SDB_CUDA(cudaMemcpyAsync(h_bad, b_bad.p, sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  if (*h_bad & 1u) { sdb::set_error("region_stats: negative label"); return 1; }
  if (*h_bad & 2u) { sdb::set_error("region_stats: label above n_labels (relabel the map sequentially first)"); return 1; }
  return 0;
}
