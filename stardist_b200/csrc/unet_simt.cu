// unet_simt.cu -- fp32 CUDA-core building blocks of the U-Net forward pass (NHWC / NDHWC).
//
// Reference graph: stardist/models/model2d.py:310-349 (+ csbdeep unet_block, SURVEY A.1):
//   conv3x3('same', bias, ReLU) x2 per level, 2x2 max-pool, nearest 2x up-sampling,
//   Concatenate([UpSampling(x), skip]) (up-sampled tensor FIRST on the channel axis),
//   features = conv3x3(->128, ReLU), prob = sigmoid(1x1), dist = 1x1 (linear).
// Keras kernels are (kh, kw, Cin, Cout) and the op is a cross-correlation with zero padding.
//
// These kernels are the exact-fp32 baseline path (used for the Cin=1 stem, small layers and as
// the in-repo cross-check of the tensor-core path in unet_tc.cu).  The decoder's upsample+concat is
// folded into the loader's address math: no up-sampled or concatenated tensor is materialised.
#include <cuda_fp16.h>
#include <vector>
#include <algorithm>
#include "common.cuh"
#include "../../include/stardist_b200.h"

namespace {

using sdb::cdiv;

// ------------------------------------------------------------------------------------------
// generic 3x3 conv: CTA tile 16x16 output pixels x COUT_T output channels, K chunk of 8 channels
// KZ = 1: 2-D 3x3 convolution (D must be 1); KZ = 3: 3-D 3x3x3 convolution over (D,H,W), weights
// (kz,3,3,Cin,Cout).  The optional low-resolution source is read through nearest up-sampling by
// (uz,uy,ux) (csbdeep UpSampling(pool)).
template <int COUT_T, int KZ>
__global__ void __launch_bounds__(COUT_T * 4)
k_conv3x3(const float* __restrict__ in_skip, const float* __restrict__ in_lo, int D, int H, int W,
          int c_skip, int c_lo, int uz, int uy, int ux, const float* __restrict__ wgt, const float* __restrict__ bias,
          int Cout, int relu, float* __restrict__ out) {
  constexpr int CK = 8, TH = 16, TW = 16, CG = COUT_T / 4, NT = 16 * CG;
  __shared__ __align__(16) float sA[CK][TH + 2][20];
  __shared__ __align__(16) float sB[9][CK][COUT_T];
  const int Cin = c_skip + c_lo;
  const int n_ct = Cout / COUT_T;
  const int zi = (blockIdx.z / n_ct) % D, img = (blockIdx.z / n_ct) / D, n0 = (blockIdx.z % n_ct) * COUT_T;
  const int ty0 = blockIdx.y * TH, tx0 = blockIdx.x * TW;
  const int t = threadIdx.x, cg = t % CG, pg = t / CG;
  const int Dlo = D / uz, Hlo = H / uy, Wlo = W / ux;

  float acc[16][4];
#pragma unroll
  for (int p = 0; p < 16; ++p) { acc[p][0] = acc[p][1] = acc[p][2] = acc[p][3] = 0.f; }

  for (int c0 = 0; c0 < Cin; c0 += CK)
  for (int dz = 0; dz < KZ; ++dz) {
    const int zz = zi + dz - KZ / 2;
    if (zz < 0 || zz >= D) continue;                 // zero padding along z (block-uniform)
    const float* skip_img = in_skip + ((size_t)img * D + zz) * H * W * c_skip;
    const float* lo_img = in_lo ? in_lo + ((size_t)img * Dlo + zz / uz) * Hlo * Wlo * c_lo : nullptr;
    // ---- stage the (TH+2)x(TW+2) halo tile of CK channels, transposed to channel-major
    for (int e = t; e < (TH + 2) * (TW + 2) * (CK / 4); e += NT) {
      const int q = e % (CK / 4), p = e / (CK / 4);
      const int ry = p / (TW + 2), rx = p % (TW + 2);
      const int gy = ty0 + ry - 1, gx = tx0 + rx - 1;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
        const int c = c0 + 4 * q;
        if (c < c_lo) v = *reinterpret_cast<const float4*>(lo_img + ((size_t)(gy / uy) * Wlo + (gx / ux)) * c_lo + c);
        else v = *reinterpret_cast<const float4*>(skip_img + ((size_t)gy * W + gx) * c_skip + (c - c_lo));
      }
      sA[4 * q + 0][ry][rx] = v.x; sA[4 * q + 1][ry][rx] = v.y;
      sA[4 * q + 2][ry][rx] = v.z; sA[4 * q + 3][ry][rx] = v.w;
    }
    // ---- stage weights [9][CK][COUT_T]
    for (int e = t; e < 9 * CK * (COUT_T / 4); e += NT) {
      const int co4 = e % (COUT_T / 4), r = e / (COUT_T / 4);
      const int ci = r % CK, tap = r / CK;
      const float4 v = *reinterpret_cast<const float4*>(wgt + ((size_t)(dz * 9 + tap) * Cin + c0 + ci) * Cout + n0 + 4 * co4);
      *reinterpret_cast<float4*>(&sB[tap][ci][4 * co4]) = v;
    }
    __syncthreads();
#pragma unroll 1
    for (int ci = 0; ci < CK; ++ci) {
#pragma unroll
      for (int dy = 0; dy < 3; ++dy) {
        float a[20];
        const float4* row = reinterpret_cast<const float4*>(&sA[ci][pg + dy][0]);
#pragma unroll
        for (int v4 = 0; v4 < 5; ++v4) {
          const float4 v = row[v4];
          a[4 * v4] = v.x; a[4 * v4 + 1] = v.y; a[4 * v4 + 2] = v.z; a[4 * v4 + 3] = v.w;
        }
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
          const float4 b = *reinterpret_cast<const float4*>(&sB[dy * 3 + dx][ci][4 * cg]);
#pragma unroll
          for (int p = 0; p < 16; ++p) {
            const float av = a[p + dx];
            acc[p][0] = fmaf(av, b.x, acc[p][0]); acc[p][1] = fmaf(av, b.y, acc[p][1]);
            acc[p][2] = fmaf(av, b.z, acc[p][2]); acc[p][3] = fmaf(av, b.w, acc[p][3]);
          }
        }
      }
    }
    __syncthreads();
  }
  const int gy = ty0 + pg;
  if (gy >= H) return;
  const float4 bb = *reinterpret_cast<const float4*>(bias + n0 + 4 * cg);
  float* orow = out + ((((size_t)img * D + zi) * H + gy) * (size_t)W) * Cout + n0 + 4 * cg;
#pragma unroll
  for (int p = 0; p < 16; ++p) {
    const int gx = tx0 + p;
    if (gx >= W) break;
    float4 v = make_float4(acc[p][0] + bb.x, acc[p][1] + bb.y, acc[p][2] + bb.z, acc[p][3] + bb.w);
    if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    *reinterpret_cast<float4*>(orow + (size_t)gx * Cout) = v;
  }
}

// ------------------------------------------------------------------------------------------
// stem: Cin small (1..4), not a multiple of 8: one thread per output voxel, all Cout (<=64) in registers
template <int COUT, int KZ>
__global__ void __launch_bounds__(128)
k_conv3x3_stem(const float* __restrict__ in, int N, int D, int H, int W, int Cin, const float* __restrict__ wgt,
               const float* __restrict__ bias, int relu, float* __restrict__ out) {
  extern __shared__ float sw[];     // [KZ*9*Cin][COUT] + bias[COUT]
  for (int e = threadIdx.x; e < KZ * 9 * Cin * COUT; e += blockDim.x) sw[e] = wgt[e];
  for (int e = threadIdx.x; e < COUT; e += blockDim.x) sw[KZ * 9 * Cin * COUT + e] = bias[e];
  __syncthreads();
  const long long npix = (long long)N * D * H * W;
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npix) return;
  const int x = (int)(p % W), y = (int)((p / W) % H), z = (int)((p / ((long long)W * H)) % D);
  const long long img = p / ((long long)W * H * D);
  float acc[COUT];
#pragma unroll
  for (int o = 0; o < COUT; ++o) acc[o] = sw[KZ * 9 * Cin * COUT + o];
  for (int dz = 0; dz < KZ; ++dz) {
    const int zz = z + dz - KZ / 2;
    if (zz < 0 || zz >= D) continue;
    for (int dy = 0; dy < 3; ++dy) {
      const int yy = y + dy - 1;
      if (yy < 0 || yy >= H) continue;
      for (int dx = 0; dx < 3; ++dx) {
        const int xx = x + dx - 1;
        if (xx < 0 || xx >= W) continue;
        const float* ip = in + (((img * D + zz) * H + yy) * W + xx) * Cin;
        for (int c = 0; c < Cin; ++c) {
          const float v = ip[c];
          const float* wr = sw + (((dz * 3 + dy) * 3 + dx) * Cin + c) * COUT;
#pragma unroll
          for (int o = 0; o < COUT; ++o) acc[o] = fmaf(v, wr[o], acc[o]);
        }
      }
    }
  }
  float4* op = reinterpret_cast<float4*>(out + p * COUT);
#pragma unroll
  for (int o = 0; o < COUT; o += 4) {
    float4 v = make_float4(acc[o], acc[o + 1], acc[o + 2], acc[o + 3]);
    if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    op[o / 4] = v;
  }
}

// ------------------------------------------------------------------------------------------
__global__ void k_maxpool_nd(const float* __restrict__ in, int N, int D, int H, int W, int C, int pz, int py, int px,
                             float* __restrict__ out) {
  const int Do = D / pz, Ho = H / py, Wo = W / px, C4 = C / 4;
  const long long total = (long long)N * Do * Ho * Wo * C4;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(e % C4); long long r = e / C4;
    const int xo = (int)(r % Wo); r /= Wo;
    const int yo = (int)(r % Ho); r /= Ho;
    const int zo = (int)(r % Do); const long long img = r / Do;
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int a = 0; a < pz; ++a) for (int b = 0; b < py; ++b) for (int c = 0; c < px; ++c) {
      const float4 v = reinterpret_cast<const float4*>(in + ((((img * D + zo * pz + a) * H + yo * py + b) * W) + xo * px + c) * (size_t)C)[c4];
      m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
    }
    reinterpret_cast<float4*>(out)[e] = m;
  }
}

// ------------------------------------------------------------------------------------------
// heads: per pixel NO = 1 + n_rays outputs from CF features; block = 32 pixels x 4 warps
template <int CF>
__global__ void __launch_bounds__(128)
k_heads(const float* __restrict__ feat, long long npix, const float* __restrict__ wp, const float* __restrict__ bp,
        const float* __restrict__ wd, const float* __restrict__ bd, int R, float* __restrict__ prob,
        float* __restrict__ dist) {
  extern __shared__ float sm[];
  const int NO = R + 1;
  float* sW = sm;                       // [CF][NO]  (o = 0 prob, 1.. dist)
  float* sF = sW + CF * NO;             // [32][CF+1]
  float* sO = sF + 32 * (CF + 1);       // [32][NO]
  for (int e = threadIdx.x; e < CF * NO; e += blockDim.x) {
    const int f = e / NO, o = e % NO;
    sW[e] = (o == 0) ? wp[f] : wd[(size_t)f * R + (o - 1)];
  }
  const long long p0 = (long long)blockIdx.x * 32;
  for (int e = threadIdx.x; e < 32 * (CF / 4); e += blockDim.x) {
    const int px = e / (CF / 4), f4 = e % (CF / 4);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p0 + px < npix) v = reinterpret_cast<const float4*>(feat + (p0 + px) * CF)[f4];
    float* d = sF + px * (CF + 1) + 4 * f4;
    d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
  }
  __syncthreads();
  const int px = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int o = w; o < NO; o += 4) {
    float acc = (o == 0) ? bp[0] : bd[o - 1];
    const float* fr = sF + px * (CF + 1);
#pragma unroll 8
    for (int f = 0; f < CF; ++f) acc = fmaf(fr[f], sW[f * NO + o], acc);
    if (o == 0) acc = 1.f / (1.f + expf(-acc));
    sO[px * NO + o] = acc;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < 32 * R; e += blockDim.x) {
    const int q = e / R, k = e % R;
    if (p0 + q < npix) dist[(p0 + q) * R + k] = sO[q * NO + 1 + k];
  }
  if (threadIdx.x < 32 && p0 + threadIdx.x < npix) prob[p0 + threadIdx.x] = sO[threadIdx.x * NO];
}


// ---------------------------------------------------------------------------------- generic convolution (ResNet backbone)
// Arbitrary odd/even kernel extent and stride with TensorFlow's padding='same' rule (stardist/models/model3d.py:402-447
// builds the ResNet from Conv3D(7^3), Conv3D(3^3, strides=pool) and Conv3D(1^3, strides=pool) layers):
//   out = ceil(in / stride),  pad_total = max((out - 1) * stride + k - in, 0),  pad_before = pad_total / 2  (rest behind).
// One thread per (output voxel, output channel); consecutive threads = consecutive channels (coalesced weights, broadcast
// activations).  Functional path for the few layers the 3x3x3 stride-1 kernel does not cover; not tuned.
struct GenericConv {
  int n, d, h, w, cin, cout;
  int kz, ky, kx, sz, sy, sx;
  int od, oh, ow, pz, py, px;
  int relu;
};
__global__ void __launch_bounds__(256) k_conv_generic(const float* __restrict__ in, const float* __restrict__ wgt, const float* __restrict__ bias,
                                                      GenericConv P, float* __restrict__ out) {
  const long long total = (long long)P.n * P.od * P.oh * P.ow * P.cout;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(e % P.cout);
    long long v = e / P.cout;
    const int ox = (int)(v % P.ow); v /= P.ow;
    const int oy = (int)(v % P.oh); v /= P.oh;
    const int oz = (int)(v % P.od); const int img = (int)(v / P.od);
    float acc = bias[co];
    for (int a = 0; a < P.kz; ++a) {
      const int iz = oz * P.sz - P.pz + a;
      if (iz < 0 || iz >= P.d) continue;
      for (int b = 0; b < P.ky; ++b) {
        const int iy = oy * P.sy - P.py + b;
        if (iy < 0 || iy >= P.h) continue;
        for (int c = 0; c < P.kx; ++c) {
          const int ix = ox * P.sx - P.px + c;
          if (ix < 0 || ix >= P.w) continue;
          const float* ip = in + ((((size_t)img * P.d + iz) * P.h + iy) * P.w + ix) * P.cin;
          const float* wp = wgt + ((size_t)((a * P.ky + b) * P.kx + c) * P.cin) * P.cout + co;
          for (int ci = 0; ci < P.cin; ++ci) acc = fmaf(ip[ci], wp[(size_t)ci * P.cout], acc);
        }
      }
    }
    if (P.relu) acc = fmaxf(acc, 0.f);
    out[e] = acc;
  }
}
__global__ void k_add_act(const float* __restrict__ a, const float* __restrict__ b, long long n, int relu, float* __restrict__ out) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    float v = a[e] + b[e];
    out[e] = relu ? fmaxf(v, 0.f) : v;
  }
}


// ---------------------------------------------------------------------------------- multi-class head
// prob_class = softmax(features_class . W + b) over n_classes + 1 outputs per pixel (model2d.py:339-347,
// model3d.py:436-444); one thread per pixel, C <= 32.
__global__ void k_class_head(const float* __restrict__ feat, long long npix, int cf, const float* __restrict__ w /*[cf][C]*/,
                             const float* __restrict__ b, int C, float* __restrict__ out /*[npix][C]*/) {
  extern __shared__ float sw[];          // [cf][C] + [C]
  for (int e = threadIdx.x; e < cf * C; e += blockDim.x) sw[e] = w[e];
  for (int e = threadIdx.x; e < C; e += blockDim.x) sw[cf * C + e] = b[e];
  __syncthreads();
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npix) return;
  float acc[32];
  for (int o = 0; o < C; ++o) acc[o] = sw[cf * C + o];
  const float* f = feat + p * cf;
  for (int k = 0; k < cf; ++k) {
    const float v = f[k];
    for (int o = 0; o < C; ++o) acc[o] = fmaf(v, sw[k * C + o], acc[o]);
  }
  float m = acc[0];
  for (int o = 1; o < C; ++o) m = fmaxf(m, acc[o]);
  float sum = 0.f;
  for (int o = 0; o < C; ++o) { acc[o] = expf(acc[o] - m); sum += acc[o]; }
  for (int o = 0; o < C; ++o) out[p * C + o] = acc[o] / sum;
}
// split fp16 activation planes (hi, lo) -> fp32
__global__ void k_merge_split(const __half* __restrict__ hi, const __half* __restrict__ lo, long long n, float* __restrict__ out) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x)
    out[e] = __half2float(hi[e]) + __half2float(lo[e]);
}

}  // namespace

// N-d convolution entry point: kz = 1 (2-D, d must be 1) or 3 (3-D).  (uz,uy,ux): up-sampling factors of
// the optional low-resolution source.
extern "C" int sdb_conv3_nd(const float* d_in, const float* d_in_lo, int n, int d, int h, int w, int cin_skip,
                            int cin_lo, int uz, int uy, int ux, const float* d_weight, const float* d_bias, int cout,
                            int kz, int relu, float* d_out, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int cin = cin_skip + cin_lo;
  if (kz != 1 && kz != 3) { sdb::set_error("conv3_nd: kz must be 1 or 3"); return 1; }
  if (kz == 1 && d != 1) { sdb::set_error("conv3_nd: 2-D convolution needs d == 1"); return 1; }
  if (d_in_lo == nullptr && cin_lo != 0) { sdb::set_error("conv3_nd: cin_lo without in_lo"); return 1; }
  if (cin_lo == 0 && cin <= 4) {
    const size_t smem = (size_t)(kz * 9 * cin * cout + cout) * sizeof(float);
    const long long npix = (long long)n * d * h * w;
    if (cout != 32 && cout != 64) { sdb::set_error("conv3_nd: stem supports cout 32 or 64"); return 1; }
    if (smem > 48 * 1024) { sdb::set_error("conv3_nd: stem weights exceed shared memory"); return 1; }
    if (kz == 1) {
      if (cout == 32) SDB_LAUNCH((k_conv3x3_stem<32, 1>), cdiv(npix, 128), 128, smem, st, d_in, n, d, h, w, cin, d_weight, d_bias, relu, d_out);
      else SDB_LAUNCH((k_conv3x3_stem<64, 1>), cdiv(npix, 128), 128, smem, st, d_in, n, d, h, w, cin, d_weight, d_bias, relu, d_out);
    } else {
      if (cout == 32) SDB_LAUNCH((k_conv3x3_stem<32, 3>), cdiv(npix, 128), 128, smem, st, d_in, n, d, h, w, cin, d_weight, d_bias, relu, d_out);
      else SDB_LAUNCH((k_conv3x3_stem<64, 3>), cdiv(npix, 128), 128, smem, st, d_in, n, d, h, w, cin, d_weight, d_bias, relu, d_out);
    }
    return 0;
  }
  if (cin_skip % 8 || cin_lo % 8 || cout % 32) { sdb::set_error("conv3_nd: channels must be multiples of 8 (in) / 32 (out)"); return 1; }
  if (cin_lo && (uz < 1 || uy < 1 || ux < 1 || d % uz || h % uy || w % ux)) { sdb::set_error("conv3_nd: size not divisible by the up-sampling factors"); return 1; }
  if (!cin_lo) { uz = uy = ux = 1; }
  dim3 grid(cdiv(w, 16), cdiv(h, 16), 1);
  const long long gz = (long long)n * d * (cout % 64 == 0 ? cout / 64 : cout / 32);
  if (gz > 65535) { sdb::set_error("conv3_nd: grid.z too large (n*d*cout tiles > 65535)"); return 1; }
  grid.z = (unsigned)gz;
  if (cout % 64 == 0) {
    if (kz == 1) SDB_LAUNCH((k_conv3x3<64, 1>), grid, 256, 0, st, d_in, d_in_lo, d, h, w, cin_skip, cin_lo, uz, uy, ux, d_weight, d_bias, cout, relu, d_out);
    else SDB_LAUNCH((k_conv3x3<64, 3>), grid, 256, 0, st, d_in, d_in_lo, d, h, w, cin_skip, cin_lo, uz, uy, ux, d_weight, d_bias, cout, relu, d_out);
  } else {
    if (kz == 1) SDB_LAUNCH((k_conv3x3<32, 1>), grid, 128, 0, st, d_in, d_in_lo, d, h, w, cin_skip, cin_lo, uz, uy, ux, d_weight, d_bias, cout, relu, d_out);
    else SDB_LAUNCH((k_conv3x3<32, 3>), grid, 128, 0, st, d_in, d_in_lo, d, h, w, cin_skip, cin_lo, uz, uy, ux, d_weight, d_bias, cout, relu, d_out);
  }
  return 0;
}

extern "C" int sdb_conv3x3_2d(const float* d_in, const float* d_in_lo, int n, int h, int w, int cin_skip,
                              int cin_lo, const float* d_weight, const float* d_bias, int cout, int relu,
                              float* d_out, sdb_stream_t stream) {
  if (cin_lo && ((h & 1) || (w & 1))) { sdb::set_error("conv3x3_2d: upsampled input needs even h, w"); return 1; }
  return sdb_conv3_nd(d_in, d_in_lo, n, 1, h, w, cin_skip, cin_lo, 1, 2, 2, d_weight, d_bias, cout, 1, relu, d_out, stream);
}

extern "C" int sdb_maxpool_nd(const float* d_in, int n, int d, int h, int w, int c, int pz, int py, int px, float* d_out, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (pz < 1 || py < 1 || px < 1 || d % pz || h % py || w % px || (c & 3)) { sdb::set_error("maxpool_nd: sizes must be divisible by the pool and c % 4 == 0"); return 1; }
  const long long total = (long long)n * (d / pz) * (h / py) * (w / px) * (c / 4);
  SDB_LAUNCH(k_maxpool_nd, (int)std::min<long long>(cdiv(total, 256), 132 * 16), 256, 0, st, d_in, n, d, h, w, c, pz, py, px, d_out);
  return 0;
}

extern "C" int sdb_maxpool2x2_2d(const float* d_in, int n, int h, int w, int c, float* d_out, sdb_stream_t stream) {
  return sdb_maxpool_nd(d_in, n, 1, h, w, c, 1, 2, 2, d_out, stream);
}

extern "C" int sdb_heads_2d(const float* d_feat, long long npix, int cfeat, const float* d_wp, const float* d_bp,
                            const float* d_wd, const float* d_bd, int n_rays, float* d_prob, float* d_dist,
                            sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (cfeat != 128) { sdb::set_error("heads_2d: only 128 feature channels (net_conv_after_unet) supported"); return 1; }
  const int NO = n_rays + 1;
  const size_t smem = (size_t)(128 * NO + 32 * 129 + 32 * NO) * sizeof(float);
  static bool attr_set = false;
  if (!attr_set) { SDB_CUDA(cudaFuncSetAttribute(k_heads<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); attr_set = true; }
  if (smem > 200 * 1024) { sdb::set_error("heads_2d: n_rays too large"); return 1; }
  SDB_LAUNCH((k_heads<128>), cdiv(npix, 32), 128, smem, st, d_feat, npix, d_wp, d_bp, d_wd, d_bd, n_rays, d_prob, d_dist);
  return 0;
}

// generic N-d convolution with TF 'same' padding and strides; in [n,d,h,w,cin] fp32, weights (kz,ky,kx,cin,cout), out
// [n,ceil(d/sz),ceil(h/sy),ceil(w/sx),cout].  2-D: d = kz = sz = 1.
extern "C" int sdb_conv_generic_nd(const float* d_in, int n, int d, int h, int w, int cin, const float* d_w, const float* d_b, int cout,
                                   int kz, int ky, int kx, int sz, int sy, int sx, int relu, float* d_out, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n <= 0 || d <= 0 || h <= 0 || w <= 0 || cin <= 0 || cout <= 0 || kz <= 0 || ky <= 0 || kx <= 0 || sz <= 0 || sy <= 0 || sx <= 0) {
    sdb::set_error("conv_generic_nd: bad arguments"); return 1;
  }
  GenericConv P;
  P.n = n; P.d = d; P.h = h; P.w = w; P.cin = cin; P.cout = cout; P.kz = kz; P.ky = ky; P.kx = kx; P.sz = sz; P.sy = sy; P.sx = sx; P.relu = relu;
  P.od = (d + sz - 1) / sz; P.oh = (h + sy - 1) / sy; P.ow = (w + sx - 1) / sx;
  P.pz = std::max((P.od - 1) * sz + kz - d, 0) / 2; P.py = std::max((P.oh - 1) * sy + ky - h, 0) / 2; P.px = std::max((P.ow - 1) * sx + kx - w, 0) / 2;
  const long long total = (long long)n * P.od * P.oh * P.ow * cout;
  SDB_LAUNCH(k_conv_generic, (int)std::min<long long>(sdb::cdiv(total, 256), 132 * 64), 256, 0, st, d_in, d_w, d_b, P, d_out);
  return 0;
}
extern "C" int sdb_add_act(const float* d_a, const float* d_b, long long n, int relu, float* d_out, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n <= 0) return 0;
  SDB_LAUNCH(k_add_act, (int)std::min<long long>(sdb::cdiv(n, 256), 132 * 32), 256, 0, st, d_a, d_b, n, relu, d_out);
  return 0;
}

extern "C" int sdb_class_head(const float* d_feat, long long npix, int cfeat, const float* d_w, const float* d_b, int n_out, float* d_out,
                              sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (npix <= 0) return 0;
  if (n_out < 1 || n_out > 32) { sdb::set_error("class_head: n_classes + 1 must be in [1,32]"); return 1; }
  const size_t smem = (size_t)(cfeat * n_out + n_out) * sizeof(float);
  if (smem > 48 * 1024) { sdb::set_error("class_head: weight table too large"); return 1; }
  SDB_LAUNCH(k_class_head, sdb::cdiv(npix, 128), 128, smem, st, d_feat, npix, cfeat, d_w, d_b, n_out, d_out);
  return 0;
}
extern "C" int sdb_merge_split(const void* d_hi, const void* d_lo, long long n, float* d_out, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n <= 0) return 0;
  SDB_LAUNCH(k_merge_split, (int)std::min<long long>(sdb::cdiv(n, 256), 132 * 32), 256, 0, st, (const __half*)d_hi, (const __half*)d_lo, n, d_out);
  return 0;
}
