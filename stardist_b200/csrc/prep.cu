// prep.cu -- the two steps in front of the network: percentile normalisation and the `scale=` zoom (SURVEY 8 f3).
//
// Reference call sites: stardist/scripts/predict2d.py:77 / predict3d.py (csbdeep.utils.normalize(x, pmin, pmax):
// mi, ma = np.percentile(x, [pmin, pmax]);  x = (x - mi) / (ma - mi + eps) in float32), csbdeep.data.PercentileNormalizer
// passed as `normalizer=` (stardist/models/base.py:398-404), and stardist/models/base.py:725-735
// (`img = ndi.zoom(img, scale, order=1)`).  csbdeep / scipy are third-party code that is not under /root/reference; the
// arithmetic restated here is numpy's percentile (method 'linear') and scipy.ndimage.zoom(order=1, mode='constant').
//
//   sdb_select_ranks     exact order statistics (k-th smallest of the un-padded region) by a 4-pass, 8-bit MSD radix
//                        select on order-preserving keys; several ranks share every pass; the linear interpolation between
//                        the two neighbouring order statistics is done by the caller with numpy itself (two scalars), so
//                        mi / ma are the bits numpy produces.
//   sdb_normalize_mi_ma  x = (x - mi) / den   (IEEE float32 sub + div == numpy / numexpr on float32 arrays), optional clip
//   sdb_zoom_linear      scipy's NI_ZoomShift for order 1: cc = j * (in-1)/(out-1) in double, weights (1-y, y), the 2^d
//                        corners accumulated in double in C order with the per-axis weights multiplied in axis order, and
//                        scipy's edge rule (cc > len-1 by rounding -> cval 0).  Compile with -fmad=false.
#include <algorithm>
#include <cstring>
#include "common.cuh"
#include "../../include/stardist_b200.h"

namespace {
using sdb::cdiv;
constexpr int MAXQ = 8;

struct Region { int nd; int shape[3]; int valid[3]; };

struct SelState {
  unsigned int prefix[MAXQ];        // key bits decided so far (high bits)
  unsigned long long rank[MAXQ];    // remaining rank inside the bucket
  unsigned int hist[MAXQ][256];
};

__device__ __forceinline__ bool in_region(long long p, const Region& R) {
  bool ok = true;
#pragma unroll
  for (int a = 2; a >= 0; --a) { const int c = (int)(p % R.shape[a]); p /= R.shape[a]; ok = ok && c < R.valid[a]; }
  return ok;
}

// pass over the data: histogram of the current 8-bit digit of the keys whose higher digits equal each query's prefix
__global__ void __launch_bounds__(256) k_select_hist(const float* __restrict__ x, long long n, Region R, int pass, int nq, SelState* __restrict__ S) {
  __shared__ unsigned int h[MAXQ][256];
  __shared__ unsigned int pre[MAXQ];
  for (int i = threadIdx.x; i < nq * 256; i += blockDim.x) h[i >> 8][i & 255] = 0;
  if (threadIdx.x < nq) pre[threadIdx.x] = S->prefix[threadIdx.x];
  __syncthreads();
  const int shift = 24 - 8 * pass;
  const unsigned int himask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (long long)gridDim.x * blockDim.x) {
    if (!in_region(p, R)) continue;
    const unsigned int k = sdb::float_order_key(x[p]);
    const unsigned int d = (k >> shift) & 255u;
    for (int q = 0; q < nq; ++q)
      if ((k & himask) == pre[q]) atomicAdd(&h[q][d], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nq * 256; i += blockDim.x) { const unsigned int v = h[i >> 8][i & 255]; if (v) atomicAdd(&S->hist[i >> 8][i & 255], v); }
}

// one block: pick the digit bucket that holds each query's rank, extend the prefix, clear the histograms
__global__ void __launch_bounds__(256) k_select_step(int pass, int nq, SelState* __restrict__ S, float* __restrict__ out) {
  const int shift = 24 - 8 * pass;
  if (threadIdx.x < nq) {
    const int q = threadIdx.x;
    unsigned long long r = S->rank[q], acc = 0;
    unsigned int d = 255;
    for (unsigned int b = 0; b < 256; ++b) {
      const unsigned long long c = S->hist[q][b];
      if (r < acc + c) { d = b; break; }
      acc += c;
    }
    S->rank[q] = r - acc;
    S->prefix[q] |= d << shift;
    if (pass == 3) {
      const unsigned int k = S->prefix[q];
      const unsigned int u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;      // inverse of float_order_key
      out[q] = __uint_as_float(u);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nq * 256; i += blockDim.x) S->hist[i >> 8][i & 255] = 0;
}

__global__ void __launch_bounds__(256) k_normalize(float* __restrict__ x, long long n, float mi, float den, int clip) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (long long)gridDim.x * blockDim.x) {
    float v = __fdiv_rn(__fsub_rn(x[p], mi), den);
    if (clip) v = fminf(fmaxf(v, 0.f), 1.f);
    x[p] = v;
  }
}

struct ZoomArgs { int nd; int in[3]; int out[3]; double z[3]; int round_int; double lo, hi; };

__global__ void __launch_bounds__(256) k_zoom_linear(const float* __restrict__ src, float* __restrict__ dst, ZoomArgs Z, long long n_out) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n_out; p += (long long)gridDim.x * blockDim.x) {
    int j[3]; long long r = p;
#pragma unroll
    for (int a = 2; a >= 0; --a) { j[a] = (int)(r % Z.out[a]); r /= Z.out[a]; }
    int i0[3], i1[3]; double w0[3], w1[3]; bool zero = false;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double cc = (double)j[a] * Z.z[a];
      if (cc > (double)(Z.in[a] - 1)) zero = true;                 // scipy: outside the input in mode 'constant' -> cval
      const double f = floor(cc), y = cc - f;
      const int b = (int)f;
      i0[a] = min(max(b, 0), Z.in[a] - 1); i1[a] = min(max(b + 1, 0), Z.in[a] - 1);
      w0[a] = 1.0 - y; w1[a] = y;
    }
    double t = 0.0;
    if (!zero) {
      for (int c0 = 0; c0 < (Z.nd == 3 ? 2 : 1); ++c0)
        for (int c1 = 0; c1 < 2; ++c1)
          for (int c2 = 0; c2 < 2; ++c2) {
            const int a0 = c0 ? i1[0] : i0[0], a1 = c1 ? i1[1] : i0[1], a2 = c2 ? i1[2] : i0[2];
            double c = (double)src[((long long)a0 * Z.in[1] + a1) * Z.in[2] + a2];
            if (Z.nd == 3) c = c * (c0 ? w1[0] : w0[0]);
            c = c * (c1 ? w1[1] : w0[1]);
            c = c * (c2 ? w1[2] : w0[2]);
            t = t + c;
          }
    }
    if (Z.round_int) {
      // scipy writes an integer output array (the dtype of the input image): unsigned: t > 0 ? t + 0.5 : 0, signed: t +- 0.5,
      // clipped to the type's range, truncated (ni_interpolation.c CASE_INTERP_OUT_UINT / _INT)
      if (Z.lo >= 0) t = t > 0 ? t + 0.5 : 0.0; else t = t > 0 ? t + 0.5 : t - 0.5;
      t = t > Z.hi ? Z.hi : (t < Z.lo ? Z.lo : t);
      t = trunc(t);
    }
    dst[p] = (float)t;
  }
}
}  // namespace

// k-th smallest values (0-based ranks) of the region [0,valid) of a C-contiguous float32 array of `shape` (ndim <= 3):
// h_out[q] = sorted(valid elements)[ranks[q]].  n_ranks <= 8.  One 32-byte read-back (stream synchronised on return).
extern "C" int sdb_select_ranks(const float* d_x, int ndim, const int* shape, const int* valid, const long long* ranks, int n_ranks,
                                float* h_out, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (ndim < 1 || ndim > 3 || n_ranks < 1 || n_ranks > MAXQ) { sdb::set_error("select_ranks: ndim <= 3, 1..8 ranks"); return 1; }
  Region R; R.nd = ndim;
  long long n = 1, nv = 1;
  for (int a = 0; a < 3; ++a) { R.shape[a] = 1; R.valid[a] = 1; }
  for (int a = 0; a < ndim; ++a) {
    R.shape[3 - ndim + a] = shape[a]; R.valid[3 - ndim + a] = valid[a]; n *= shape[a]; nv *= valid[a];
    if (valid[a] < 1 || valid[a] > shape[a]) { sdb::set_error("select_ranks: bad region"); return 1; }
  }
  SelState hs; memset(&hs, 0, sizeof(hs));
  for (int q = 0; q < n_ranks; ++q) {
    if (ranks[q] < 0 || ranks[q] >= nv) { sdb::set_error("select_ranks: rank outside the region"); return 1; }
    hs.rank[q] = (unsigned long long)ranks[q];
  }
  sdb::DevBuf b_state, b_out;
  SDB_CUDA(b_state.alloc(sizeof(SelState), st)); SDB_CUDA(b_out.alloc(MAXQ * sizeof(float), st));
  SDB_CUDA(cudaMemcpyAsync(b_state.p, &hs, sizeof(hs), cudaMemcpyHostToDevice, st));
  const int grid = (int)std::min<long long>(cdiv(n, 256 * 8), 132 * 8);
  for (int pass = 0; pass < 4; ++pass) {
    SDB_LAUNCH(k_select_hist, std::max(grid, 1), 256, 0, st, d_x, n, R, pass, n_ranks, b_state.as<SelState>());
    SDB_LAUNCH(k_select_step, 1, 256, 0, st, pass, n_ranks, b_state.as<SelState>(), b_out.as<float>());
  }
  float tmp[MAXQ];
  SDB_CUDA(cudaMemcpyAsync(tmp, b_out.p, MAXQ * sizeof(float), cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  for (int q = 0; q < n_ranks; ++q) h_out[q] = tmp[q];
  return 0;
}

// in place x = (x - mi) / den (float32, round to nearest) [+ clip to [0,1]] -- csbdeep normalize_mi_ma with den = ma - mi + eps
extern "C" int sdb_normalize_mi_ma(float* d_x, long long n, float mi, float den, int clip, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n > 0) SDB_LAUNCH(k_normalize, (int)std::min<long long>(cdiv(n, 256 * 4), 132 * 16), 256, 0, st, d_x, n, mi, den, clip);
  return 0;
}

// scipy.ndimage.zoom(x, zoom, order=1) for a C-contiguous float32 array (ndim 2 or 3): out_shape given by the caller
// (round(in * zoom)); per axis the sample position is j * (in-1)/(out-1).
// round_int != 0: the result is rounded and clipped to [int_lo, int_hi] like scipy does for an integer input array.
extern "C" int sdb_zoom_linear(const float* d_in, int ndim, const int* in_shape, const int* out_shape, float* d_out, int round_int,
                               double int_lo, double int_hi, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (ndim < 2 || ndim > 3) { sdb::set_error("zoom_linear: ndim 2 or 3"); return 1; }
  ZoomArgs Z; Z.nd = ndim; Z.round_int = round_int; Z.lo = int_lo; Z.hi = int_hi;
  long long n_out = 1;
  for (int a = 0; a < 3; ++a) { Z.in[a] = 1; Z.out[a] = 1; Z.z[a] = 1.0; }
  for (int a = 0; a < ndim; ++a) {
    const int k = 3 - ndim + a;
    Z.in[k] = in_shape[a]; Z.out[k] = out_shape[a];
    if (in_shape[a] < 1 || out_shape[a] < 1) { sdb::set_error("zoom_linear: empty axis"); return 1; }
    Z.z[k] = out_shape[a] > 1 ? (double)(in_shape[a] - 1) / (double)(out_shape[a] - 1) : 1.0;
    n_out *= out_shape[a];
  }
  SDB_LAUNCH(k_zoom_linear, (int)std::min<long long>(cdiv(n_out, 256), 132 * 16), 256, 0, st, d_in, d_out, Z, n_out);
  return 0;
}

namespace {
struct PadArgs { int in[3]; int out[3]; };
// numpy.pad(mode='reflect') at the END of each axis (StarDistPadAndCropResizer, base.py:1162-1211): out index i >= n maps
// to the reflection without repeating the edge, period 2(n-1)
__global__ void __launch_bounds__(256) k_pad_reflect_end(const float* __restrict__ src, float* __restrict__ dst, PadArgs P, int ch, long long n_out) {
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < n_out; p += (long long)gridDim.x * blockDim.x) {
    long long r = p / ch; const int c = (int)(p % ch);
    int j[3];
#pragma unroll
    for (int a = 2; a >= 0; --a) { j[a] = (int)(r % P.out[a]); r /= P.out[a]; }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const int n = P.in[a];
      if (j[a] >= n) {
        if (n == 1) j[a] = 0;
        else { const int per = 2 * (n - 1); int m = j[a] % per; j[a] = m < n ? m : per - m; }
      }
    }
    dst[p] = src[(((long long)j[0] * P.in[1] + j[1]) * P.in[2] + j[2]) * ch + c];
  }
}
}  // namespace

// reflect-pad a channels-last float32 array [*in_shape, ch] at the end of each spatial axis to [*out_shape, ch]
extern "C" int sdb_pad_reflect_end(const float* d_in, int ndim, const int* in_shape, const int* out_shape, int channels, float* d_out,
                                   sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (ndim < 1 || ndim > 3 || channels < 1) { sdb::set_error("pad_reflect_end: ndim <= 3"); return 1; }
  PadArgs P; long long n_out = channels;
  for (int a = 0; a < 3; ++a) { P.in[a] = 1; P.out[a] = 1; }
  for (int a = 0; a < ndim; ++a) {
    P.in[3 - ndim + a] = in_shape[a]; P.out[3 - ndim + a] = out_shape[a]; n_out *= out_shape[a];
    if (out_shape[a] < in_shape[a] || in_shape[a] < 1) { sdb::set_error("pad_reflect_end: bad shapes"); return 1; }
  }
  SDB_LAUNCH(k_pad_reflect_end, (int)std::min<long long>(cdiv(n_out, 256), 132 * 16), 256, 0, st, d_in, d_out, P, channels, n_out);
  return 0;
}
