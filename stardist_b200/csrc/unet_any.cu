// unet_any.cu -- fp32 CUDA-core network kernels for any layer shape of a U-Net / ResNet model (NHWC / NDHWC).
//
// The kernels of unet_simt.cu cover the default architecture family (3^d kernels, ReLU, channel counts that are multiples
// of 8 / 32, 128 feature channels).  These cover what a model folder of the reference may hold beyond that: kernel extents
// 1..7 per axis (odd or even), strides 1 / 2 under TensorFlow's padding='same' rule, any channel count, any feature width,
// and the Keras activations of the table below.  The executors (models/unet_device.py) use them only for the layers the
// unet_simt.cu kernels do not accept.  For training the same layers, the tiled convolution also serves as the input
// gradient (sdb_conv_dgrad_any_nd), and sdb_act_any / sdb_act_backward split the activation off the convolution.
//
// Activation ids (the `act` argument; 0 and 1 match the `relu` flag of the older kernels):
//   0 linear, 1 relu, 2 elu, 3 selu, 4 tanh, 5 sigmoid, 6 softplus, 7 softsign, 8 exponential, 9 swish, 10 gelu
#include <cmath>
#include <algorithm>
#include <string>
#include "common.cuh"
#include "../../include/stardist_b200.h"

namespace {

using sdb::cdiv;

constexpr int kNumActs = 11;

// Keras / TensorFlow definitions.  elu and selu use expm1 for x <= 0; softplus is TF's stable form (x above
// -log(eps) - 2, exp(x) below log(eps) + 2, log1p(exp(x)) between, eps = float32 epsilon); gelu is the exact
// (approximate=False) 0.5 x (1 + erf(x / sqrt 2)), evaluated as 0.5 x erfc(-x / sqrt 2), which is the same function
// without the cancellation of 1 + erf for x << 0.
__device__ __forceinline__ float act_apply(int act, float x) {
  switch (act) {
    case 0: return x;
    case 1: return fmaxf(x, 0.f);
    case 2: return x > 0.f ? x : expm1f(x);
    case 3: return x > 0.f ? 1.05070098735548049342f * x : 1.75809934084737685994f * expm1f(x);
    case 4: return tanhf(x);
    case 5: return 1.f / (1.f + expf(-x));
    case 6: {
      const float thr = -13.9423847f;              // log(FLT_EPSILON) + 2
      if (x > -thr) return x;
      if (x < thr) return expf(x);
      return log1pf(expf(x));
    }
    case 7: return x / (1.f + fabsf(x));
    case 8: return expf(x);
    case 9: return x / (1.f + expf(-x));
    default: return 0.5f * x * erfcf(x * -0.707106781186547524f);
  }
}

// act'(z) of the table above in float32 forms without cancellation at either end: elu / selu use exp(z) for z <= 0 (which
// expm1(z) + 1 would lose to cancellation once expm1(z) rounds to -1), tanh' = 4u / (1 + u)^2 with u = exp(-2|z|) and
// sigmoid' = u / (1 + u)^2 with u = exp(-|z|) (no 1 - t^2 or s(1 - s) near saturation), softplus' = sigmoid(z) from the
// same u (the derivative of log(1 + e^z); the thresholds of act_apply only choose how that function is evaluated, and
// their pieces differ from it by less than one float32 rounding), swish' = s (1 + z (1 - s)) with s and 1 - s both from
// u, gelu' = 0.5 erfc(-z / sqrt 2) + z exp(-z^2 / 2) / sqrt(2 pi).  relu' is 1 for z > 0 and 0 otherwise (TensorFlow's
// ReluGrad).
__device__ __forceinline__ float act_grad(int act, float z) {
  switch (act) {
    case 0: return 1.f;
    case 1: return z > 0.f ? 1.f : 0.f;
    case 2: return z > 0.f ? 1.f : expf(z);
    case 3: return z > 0.f ? 1.05070098735548049342f : 1.75809934084737685994f * expf(z);
    case 4: { const float u = expf(-2.f * fabsf(z)), q = 1.f + u; return 4.f * u / (q * q); }
    case 5: { const float u = expf(-fabsf(z)), q = 1.f + u; return u / (q * q); }
    case 6: { const float u = expf(-fabsf(z)); return (z >= 0.f ? 1.f : u) / (1.f + u); }
    case 7: { const float q = 1.f + fabsf(z); return 1.f / (q * q); }
    case 8: return expf(z);
    case 9: {
      const float u = expf(-fabsf(z)), r = 1.f / (1.f + u);
      const float s = z >= 0.f ? r : u * r, sc = z >= 0.f ? u * r : r;      // sigmoid(z), 1 - sigmoid(z)
      return s * (1.f + z * sc);
    }
    default: return 0.5f * erfcf(z * -0.707106781186547524f) + z * 0.398942280401432678f * expf(-0.5f * z * z);
  }
}

// ------------------------------------------------------------------------------------------ tiled convolution
// CTA tile: 16 x 16 output pixels of one output plane x COUT_T output channels.  Thread = 8 consecutive output pixels of
// one row x 8 consecutive output channels.  For every chunk of CK input channels and every z tap, the input halo of the
// tile ((16-1)*sy + ky rows x (16-1)*sx + kx columns) and the chunk's weights of all ky*kx taps are staged in shared
// memory.  Per output, the sum runs over channel chunks, then z, y and x taps, then the channels of the chunk, each term an
// fmaf; the bias is added at the end and the activation applied.  The decoder input [upsample(x_lo), skip] is read through
// address math (x_lo channels first, nearest up-sampling by (uz,uy,ux)).
struct ConvAny {
  int d, h, w, c_skip, c_lo, uz, uy, ux;
  int cout, kz, ky, kx, sz, sy, sx;
  int od, oh, ow, pz, py, px;
  int act, rows, cols, plane, tiles_x;
};

constexpr int kCK = 8, kTH = 16, kTW = 16;

template <int COUT_T, int SX>
__global__ void __launch_bounds__(COUT_T * 4)
k_conv_any(const float* __restrict__ in_skip, const float* __restrict__ in_lo, const float* __restrict__ wgt,
           const float* __restrict__ bias, ConvAny P, float* __restrict__ out) {
  constexpr int CG = COUT_T / 8, NT = COUT_T * 4;
  extern __shared__ __align__(16) float sm[];
  float* sA = sm;                                   // [CK][plane]: halo, channel-major
  float* sB = sm + kCK * P.plane;                   // [ky*kx][CK][COUT_T]
  const int cin = P.c_skip + P.c_lo;
  const int taps = P.ky * P.kx;
  const int n0 = blockIdx.y * COUT_T;
  const int zo = blockIdx.z % P.od, img = blockIdx.z / P.od;
  const int ty0 = (blockIdx.x / P.tiles_x) * kTH, tx0 = (blockIdx.x % P.tiles_x) * kTW;
  const int t = threadIdx.x, cg = t % CG, pg = t / CG, prow = pg >> 1, pcol = (pg & 1) * 8;
  const int iy0 = ty0 * P.sy - P.py, ix0 = tx0 * SX - P.px;
  const int Dlo = P.d / P.uz, Hlo = P.h / P.uy, Wlo = P.w / P.ux;

  float acc[8][8];
#pragma unroll
  for (int p = 0; p < 8; ++p)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[p][j] = 0.f;

  for (int c0 = 0; c0 < cin; c0 += kCK)
  for (int dz = 0; dz < P.kz; ++dz) {
    const int iz = zo * P.sz - P.pz + dz;
    if (iz < 0 || iz >= P.d) continue;                       // zero padding along z (block-uniform)
    const float* skip_pl = in_skip + ((size_t)img * P.d + iz) * P.h * P.w * P.c_skip;
    const float* lo_pl = in_lo ? in_lo + ((size_t)img * Dlo + iz / P.uz) * Hlo * Wlo * P.c_lo : nullptr;
    for (int e = t; e < P.rows * P.cols * kCK; e += NT) {
      const int ci = e % kCK, q = e / kCK;
      const int r = q / P.cols, c = q % P.cols;
      const int gy = iy0 + r, gx = ix0 + c, ch = c0 + ci;
      float v = 0.f;
      if (gy >= 0 && gy < P.h && gx >= 0 && gx < P.w && ch < cin) {
        if (ch < P.c_lo) v = lo_pl[((size_t)(gy / P.uy) * Wlo + gx / P.ux) * P.c_lo + ch];
        else v = skip_pl[((size_t)gy * P.w + gx) * P.c_skip + (ch - P.c_lo)];
      }
      sA[ci * P.plane + q] = v;
    }
    for (int e = t; e < taps * kCK * COUT_T; e += NT) {
      const int co = e % COUT_T, r = e / COUT_T;
      const int ci = r % kCK, tap = r / kCK;
      float v = 0.f;
      if (c0 + ci < cin && n0 + co < P.cout) v = wgt[((size_t)(dz * taps + tap) * cin + c0 + ci) * P.cout + n0 + co];
      sB[e] = v;
    }
    __syncthreads();
    for (int dy = 0; dy < P.ky; ++dy)
    for (int dx = 0; dx < P.kx; ++dx) {
      const float* arow = sA + (prow * P.sy + dy) * P.cols + pcol * SX + dx;
      const float* brow = sB + (dy * P.kx + dx) * kCK * COUT_T + 8 * cg;
#pragma unroll
      for (int ci = 0; ci < kCK; ++ci) {
        const float4 b0 = *reinterpret_cast<const float4*>(brow + ci * COUT_T);
        const float4 b1 = *reinterpret_cast<const float4*>(brow + ci * COUT_T + 4);
        const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
        const float* ap = arow + ci * P.plane;
#pragma unroll
        for (int p = 0; p < 8; ++p) {
          const float a = ap[p * SX];
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[p][j] = fmaf(a, b[j], acc[p][j]);
        }
      }
    }
    __syncthreads();
  }
  const int oy = ty0 + prow;
  const int co0 = n0 + 8 * cg;
  if (oy >= P.oh || co0 >= P.cout) return;
  float bb[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) bb[j] = (bias != nullptr && co0 + j < P.cout) ? bias[co0 + j] : 0.f;
  const bool vec = (P.cout % 4 == 0) && (co0 + 8 <= P.cout);
  float* orow = out + ((((size_t)img * P.od + zo) * P.oh + oy) * (size_t)P.ow) * P.cout + co0;
#pragma unroll
  for (int p = 0; p < 8; ++p) {
    const int ox = tx0 + pcol + p;
    if (ox >= P.ow) break;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = act_apply(P.act, acc[p][j] + bb[j]);
    float* o = orow + (size_t)ox * P.cout;
    if (vec) {
      *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4*>(o + 4) = make_float4(v[4], v[5], v[6], v[7]);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (co0 + j < P.cout) o[j] = v[j];
    }
  }
}

// ------------------------------------------------------------------------------------------ 1^d heads, any width
// prob = sigmoid(f . wp + bp), dist = f . wd + bd.  CTA = 64 pixels x 64 of the R + 1 outputs (output 0 = prob); feature
// chunks of 32 channels and the matching weight tile [32][64] are staged in shared memory, so any cf x (R + 1) fits.
// Per output the sum starts at the bias and adds the features in ascending order with fmaf.
constexpr int kHP = 64, kHO = 64, kHF = 32;

__global__ void __launch_bounds__(256)
k_heads_any(const float* __restrict__ feat, long long npix, int cf, const float* __restrict__ wp, const float* __restrict__ bp,
            const float* __restrict__ wd, const float* __restrict__ bd, int R, float* __restrict__ prob, float* __restrict__ dist) {
  __shared__ float sF[kHP][kHF + 1];
  __shared__ __align__(16) float sW[kHF][kHO];
  const int NO = R + 1;
  const long long p0 = (long long)blockIdx.x * kHP;
  const int o0 = blockIdx.y * kHO;
  const int t = threadIdx.x, og = t % 16, pq = t / 16;
  float acc[4][4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int o = o0 + 4 * og + j;
    const float b = o == 0 ? bp[0] : (o < NO ? bd[o - 1] : 0.f);
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[i][j] = b;
  }
  for (int f0 = 0; f0 < cf; f0 += kHF) {
    for (int e = t; e < kHP * kHF; e += 256) {
      const int f = e % kHF, q = e / kHF;
      sF[q][f] = (p0 + q < npix && f0 + f < cf) ? feat[(p0 + q) * cf + f0 + f] : 0.f;
    }
    for (int e = t; e < kHF * kHO; e += 256) {
      const int o = e % kHO, f = e / kHO, go = o0 + o, gf = f0 + f;
      float v = 0.f;
      if (gf < cf && go < NO) v = go == 0 ? wp[gf] : wd[(size_t)gf * R + go - 1];
      sW[f][o] = v;
    }
    __syncthreads();
    const int fn = min(kHF, cf - f0);
    for (int f = 0; f < fn; ++f) {
      const float4 b = *reinterpret_cast<const float4*>(&sW[f][4 * og]);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float a = sF[4 * pq + i][f];
        acc[i][0] = fmaf(a, b.x, acc[i][0]); acc[i][1] = fmaf(a, b.y, acc[i][1]);
        acc[i][2] = fmaf(a, b.z, acc[i][2]); acc[i][3] = fmaf(a, b.w, acc[i][3]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const long long p = p0 + 4 * pq + i;
    if (p >= npix) break;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int o = o0 + 4 * og + j;
      if (o == 0) prob[p] = 1.f / (1.f + expf(-acc[i][j]));
      else if (o < NO) dist[p * R + o - 1] = acc[i][j];
    }
  }
}

// ------------------------------------------------------------------------------------------ pooling and residual sum
__global__ void k_maxpool_any(const float* __restrict__ in, int N, int D, int H, int W, int C, int pz, int py, int px,
                              float* __restrict__ out) {
  const int Do = D / pz, Ho = H / py, Wo = W / px;
  const long long total = (long long)N * Do * Ho * Wo * C;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(e % C); long long r = e / C;
    const int xo = (int)(r % Wo); r /= Wo;
    const int yo = (int)(r % Ho); r /= Ho;
    const int zo = (int)(r % Do); const long long img = r / Do;
    float m = -INFINITY;
    for (int a = 0; a < pz; ++a) for (int b = 0; b < py; ++b) for (int q = 0; q < px; ++q)
      m = fmaxf(m, in[((((img * D + zo * pz + a) * H + yo * py + b) * W) + xo * px + q) * (size_t)C + c]);
    out[e] = m;
  }
}

__global__ void k_add_act_any(const float* __restrict__ a, const float* __restrict__ b, long long n, int act, float* __restrict__ out) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x)
    out[e] = act_apply(act, a[e] + b[e]);
}

__global__ void k_act_any(const float* __restrict__ z, long long n, int act, float* __restrict__ y) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x)
    y[e] = act_apply(act, z[e]);
}

// g *= act'(z); relu zeroes g where z <= 0 (also an infinite g), like sdb_relu_backward
__global__ void k_act_backward(float* __restrict__ g, const float* __restrict__ z, long long n, int act) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const float v = z[e];
    if (act == 1) { if (!(v > 0.f)) g[e] = 0.f; }
    else g[e] *= act_grad(act, v);
  }
}

template <int COUT_T, int SX>
int launch_conv(dim3 grid, size_t smem, cudaStream_t st, const float* in, const float* lo, const float* w, const float* b,
                const ConvAny& P, float* out) {
  static bool attr = false;
  if (!attr) { SDB_CUDA(cudaFuncSetAttribute(k_conv_any<COUT_T, SX>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); attr = true; }
  SDB_LAUNCH((k_conv_any<COUT_T, SX>), grid, COUT_T * 4, smem, st, in, lo, w, b, P, out);
  return 0;
}

// launches k_conv_any for P with its pads (pz, py, px) already set; the sizes, kernel and channels of P are checked by the caller
int run_conv_any(const char* who, ConvAny& P, int n, const float* d_in, const float* d_in_lo, const float* d_weight, const float* d_bias,
                 float* d_out, cudaStream_t st) {
  P.rows = (kTH - 1) * P.sy + P.ky; P.cols = (kTW - 1) * P.sx + P.kx;
  P.plane = (P.rows * P.cols) | 1;                  // odd: the channel-major halo stores avoid bank conflicts
  P.tiles_x = cdiv(P.ow, kTW);
  const int cout_t = P.cout > 32 ? 64 : 32;
  const long long gx = (long long)P.tiles_x * cdiv(P.oh, kTH), gy = cdiv(P.cout, cout_t), gz = (long long)n * P.od;
  if (gx > 0x7fffffffLL || gy > 65535 || gz > 65535) { sdb::set_error(std::string(who) + ": grid too large"); return 1; }
  const size_t smem = (size_t)(kCK * P.plane + P.ky * P.kx * kCK * cout_t) * sizeof(float);
  dim3 grid((unsigned)gx, (unsigned)gy, (unsigned)gz);
  if (cout_t == 64) {
    if (P.sx == 1) return launch_conv<64, 1>(grid, smem, st, d_in, d_in_lo, d_weight, d_bias, P, d_out);
    return launch_conv<64, 2>(grid, smem, st, d_in, d_in_lo, d_weight, d_bias, P, d_out);
  }
  if (P.sx == 1) return launch_conv<32, 1>(grid, smem, st, d_in, d_in_lo, d_weight, d_bias, P, d_out);
  return launch_conv<32, 2>(grid, smem, st, d_in, d_in_lo, d_weight, d_bias, P, d_out);
}

}  // namespace

extern "C" int sdb_conv_any_nd(const float* d_in, const float* d_in_lo, int n, int d, int h, int w, int cin_skip, int cin_lo,
                               int uz, int uy, int ux, const float* d_weight, const float* d_bias, int cout,
                               int kz, int ky, int kx, int sz, int sy, int sx, int act, float* d_out, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n <= 0 || d <= 0 || h <= 0 || w <= 0 || cin_skip < 0 || cin_lo < 0 || cin_skip + cin_lo < 1 || cout < 1) {
    sdb::set_error("conv_any_nd: bad sizes"); return 1;
  }
  if (kz < 1 || kz > 7 || ky < 1 || ky > 7 || kx < 1 || kx > 7) { sdb::set_error("conv_any_nd: kernel extents must be in 1..7"); return 1; }
  if (sz < 1 || sz > 2 || sy < 1 || sy > 2 || sx < 1 || sx > 2) { sdb::set_error("conv_any_nd: strides must be 1 or 2"); return 1; }
  if (act < 0 || act >= kNumActs) { sdb::set_error("conv_any_nd: unknown activation id"); return 1; }
  if (cin_lo) {
    if (d_in_lo == nullptr) { sdb::set_error("conv_any_nd: cin_lo without in_lo"); return 1; }
    if (sz != 1 || sy != 1 || sx != 1) { sdb::set_error("conv_any_nd: an up-sampled source needs stride 1"); return 1; }
    if (uz < 1 || uy < 1 || ux < 1 || d % uz || h % uy || w % ux) { sdb::set_error("conv_any_nd: size not divisible by the up-sampling factors"); return 1; }
  } else {
    uz = uy = ux = 1;
  }
  ConvAny P;
  P.d = d; P.h = h; P.w = w; P.c_skip = cin_skip; P.c_lo = cin_lo; P.uz = uz; P.uy = uy; P.ux = ux;
  P.cout = cout; P.kz = kz; P.ky = ky; P.kx = kx; P.sz = sz; P.sy = sy; P.sx = sx; P.act = act;
  P.od = (d + sz - 1) / sz; P.oh = (h + sy - 1) / sy; P.ow = (w + sx - 1) / sx;
  // TensorFlow 'same': pad_total = max((out - 1) * s + k - in, 0), pad_before = pad_total / 2
  P.pz = std::max((P.od - 1) * sz + kz - d, 0) / 2;
  P.py = std::max((P.oh - 1) * sy + ky - h, 0) / 2;
  P.px = std::max((P.ow - 1) * sx + kx - w, 0) / 2;
  return run_conv_any("conv_any_nd", P, n, d_in, d_in_lo, d_weight, d_bias, d_out, st);
}

extern "C" int sdb_heads_any(const float* d_feat, long long npix, int cfeat, const float* d_wp, const float* d_bp,
                             const float* d_wd, const float* d_bd, int n_rays, float* d_prob, float* d_dist, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (cfeat < 1 || n_rays < 1 || n_rays > 256) { sdb::set_error("heads_any: need cfeat >= 1 and 1 <= n_rays <= 256"); return 1; }
  if (npix <= 0) return 0;
  const long long gx = (npix + kHP - 1) / kHP;
  if (gx > 0x7fffffffLL) { sdb::set_error("heads_any: too many pixels"); return 1; }
  dim3 grid((unsigned)gx, (unsigned)cdiv(n_rays + 1, kHO), 1);
  SDB_LAUNCH(k_heads_any, grid, 256, 0, st, d_feat, npix, cfeat, d_wp, d_bp, d_wd, d_bd, n_rays, d_prob, d_dist);
  return 0;
}

extern "C" int sdb_maxpool_any_nd(const float* d_in, int n, int d, int h, int w, int c, int pz, int py, int px, float* d_out,
                                  sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n <= 0 || c <= 0 || pz < 1 || py < 1 || px < 1 || d % pz || h % py || w % px) {
    sdb::set_error("maxpool_any_nd: sizes must be divisible by the pool"); return 1;
  }
  const long long total = (long long)n * (d / pz) * (h / py) * (w / px) * c;
  if (total == 0) return 0;
  SDB_LAUNCH(k_maxpool_any, (int)std::min<long long>(cdiv(total, 256LL), 132 * 16), 256, 0, st, d_in, n, d, h, w, c, pz, py, px, d_out);
  return 0;
}

extern "C" int sdb_add_act_any(const float* d_a, const float* d_b, long long n, int act, float* d_out, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (act < 0 || act >= kNumActs) { sdb::set_error("add_act_any: unknown activation id"); return 1; }
  if (n <= 0) return 0;
  SDB_LAUNCH(k_add_act_any, (int)std::min<long long>(cdiv(n, 256LL), 132 * 32), 256, 0, st, d_a, d_b, n, act, d_out);
  return 0;
}

// dX of a stride-1 'same' convolution with kernel (kz, ky, kx, cin, cout): the correlation of dY with the flipped kernel
// wf (kz, ky, kx, cout, cin) of sdb_conv_flip_weights, front offset k - 1 - (k - 1) / 2 per axis (the forward's back
// padding, which differs from its front padding for even k), zero bias, linear output, on the tiled kernel above
extern "C" int sdb_conv_dgrad_any_nd(const float* d_dy, int n, int d, int h, int w, int cout, const float* d_wf, int cin,
                                     int kz, int ky, int kx, float* d_dx, sdb_stream_t stream) {
  if (n <= 0 || d <= 0 || h <= 0 || w <= 0 || cin < 1 || cout < 1) { sdb::set_error("conv_dgrad_any_nd: bad sizes"); return 1; }
  if (kz < 1 || kz > 7 || ky < 1 || ky > 7 || kx < 1 || kx > 7) { sdb::set_error("conv_dgrad_any_nd: kernel extents must be in 1..7"); return 1; }
  ConvAny P;
  P.d = d; P.h = h; P.w = w; P.c_skip = cout; P.c_lo = 0; P.uz = P.uy = P.ux = 1;
  P.cout = cin; P.kz = kz; P.ky = ky; P.kx = kx; P.sz = P.sy = P.sx = 1; P.act = 0;
  P.od = d; P.oh = h; P.ow = w;
  P.pz = kz - 1 - (kz - 1) / 2; P.py = ky - 1 - (ky - 1) / 2; P.px = kx - 1 - (kx - 1) / 2;
  return run_conv_any("conv_dgrad_any_nd", P, n, d_dy, nullptr, d_wf, nullptr, d_dx, (cudaStream_t)stream);
}

extern "C" int sdb_act_any(const float* d_z, long long n, int act, float* d_y, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (act < 0 || act >= kNumActs) { sdb::set_error("act_any: unknown activation id"); return 1; }
  if (n <= 0) return 0;
  SDB_LAUNCH(k_act_any, (int)std::min<long long>(cdiv(n, 256LL), 132 * 32), 256, 0, st, d_z, n, act, d_y);
  return 0;
}

extern "C" int sdb_act_backward(float* d_g, const float* d_z, long long n, int act, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (act < 0 || act >= kNumActs) { sdb::set_error("act_backward: unknown activation id"); return 1; }
  if (n <= 0 || act == 0) return 0;
  SDB_LAUNCH(k_act_backward, (int)std::min<long long>(cdiv(n, 256LL), 132 * 32), 256, 0, st, d_g, d_z, n, act);
  return 0;
}
