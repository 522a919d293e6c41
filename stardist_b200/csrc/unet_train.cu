// unet_train.cu -- fp32 CUDA-core kernels of the U-Net training step (NHWC / NDHWC): weight gradients of the
// 3^d / 1^d convolutions, the decoder split, ReLU and max-pool backward (the float instances of train_elem.cuh), the StarDist loss with its head gradient,
// the multi-class cross-entropy with its softmax-logit gradient, the 1x1 head input gradients, the data-parallel reduction of the
// replicas' gradients and Adam.  The input gradient of the
// convolutions is not here: it is a forward kernel run on dY with the spatially flipped, Cin/Cout-transposed kernel written by
// sdb_conv_flip_weights -- sdb_conv3_nd of unet_simt.cu for the 3^d layers it takes, sdb_conv_dgrad_any_nd of unet_any.cu
// for every other kernel extent and channel count.
//
// Determinism: no float atomics anywhere.  Every reduction splits its work into a count of pieces taken from the shape
// alone, each piece accumulates in a fixed order into its own slot of a workspace, and a second kernel sums the slots
// in index order.  Gradients, loss values and weights are therefore bit-identical from run to run on the same device.
#include <math.h>
#include <string>
#include <algorithm>
#include <cstdint>
#include "common.cuh"
#include "wgrad.cuh"
#include "train_elem.cuh"
#include "../../include/stardist_b200.h"

namespace {

using sdb::cdiv;

__device__ __forceinline__ long long llmin(long long a, long long b) { return a < b ? a : b; }

// ------------------------------------------------------------------------------------------ weight gradient
// dW[tap, ci, co] = sum_p x[p + tap - pad, ci] * dy[p, co] and db[co] = sum_p dy[p, co], as one GEMM over the pixels p of the
// whole batch: row r < taps*Cin is (tap, ci) = (r / Cin, r % Cin), tap = (dz, dy, dx) row-major over the (kz, ky, kx) box,
// row taps*Cin is a constant 1 (the bias).  pad is TensorFlow's 'same' front offset at stride 1, (k - 1) / 2 per axis
// (k / 2 for odd k, so the 3^d / 1^d path of sdb_conv_wgrad_nd reads what it always read).  The decoder
// input [upsample(x_lo), skip] is read through the forward loader's address math (channel c < c_lo from x_lo at the
// up-sampled position).  CTA tile 64 rows x 64 output channels, 16 pixels per K step, 4x4 outputs per thread; split s of
// the pixel range writes work[s][row][co].
constexpr int WG_R = 64, WG_C = 64, WG_K = 16;

using sdb::WgradArgs;

__global__ void __launch_bounds__(256) k_conv_wgrad(WgradArgs A) {
  __shared__ __align__(16) float sX[WG_K][WG_R];
  __shared__ __align__(16) float sD[WG_K][WG_C];
  __shared__ int sRow[WG_R][5];          // dz, dy, dx, channel, kind (0 skip, 1 lo, 2 bias, 3 none)
  __shared__ int sPix[WG_K][4];          // img, z, y, x (img < 0: past the end)
  const int Cin = A.c_skip + A.c_lo, taps = A.kz * A.ky * A.kx;
  const int n_ct = (A.cout + WG_C - 1) / WG_C;
  const int r0 = (blockIdx.x / n_ct) * WG_R, c0 = (blockIdx.x % n_ct) * WG_C;
  const int t = threadIdx.x, tr = t / 16, tc = t % 16;
  if (t < WG_R) {
    const int r = r0 + t;
    int* q = sRow[t];
    if (r < taps * Cin) {
      const int tap = r / Cin, c = r % Cin;
      q[0] = tap / (A.ky * A.kx) - A.pz; q[1] = (tap / A.kx) % A.ky - A.py; q[2] = tap % A.kx - A.px;
      q[3] = c < A.c_lo ? c : c - A.c_lo; q[4] = c < A.c_lo ? 1 : 0;
    } else {
      q[0] = q[1] = q[2] = q[3] = 0; q[4] = (r == taps * Cin) ? 2 : 3;
    }
  }
  const long long p_begin = (long long)blockIdx.y * A.per_split;
  const long long p_end = llmin(A.npix, p_begin + A.per_split);
  const int Dl = A.d / A.uz, Hl = A.h / A.uy, Wl = A.w / A.ux;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
  for (long long p0 = p_begin; p0 < p_end; p0 += WG_K) {
    __syncthreads();
    if (t < WG_K) {
      const long long p = p0 + t;
      int* q = sPix[t];
      if (p < p_end) {
        q[3] = (int)(p % A.w); q[2] = (int)((p / A.w) % A.h); q[1] = (int)((p / ((long long)A.w * A.h)) % A.d);
        q[0] = (int)(p / ((long long)A.w * A.h * A.d));
      } else {
        q[0] = -1; q[1] = q[2] = q[3] = 0;
      }
    }
    __syncthreads();
    for (int e = t; e < WG_K * WG_R; e += 256) {
      const int k = e / WG_R, r = e % WG_R;
      const int* pp = sPix[k]; const int* q = sRow[r];
      float v = 0.f;
      if (pp[0] >= 0) {
        if (q[4] == 2) v = 1.f;
        else if (q[4] < 2) {
          const int zz = pp[1] + q[0], yy = pp[2] + q[1], xx = pp[3] + q[2];
          if (zz >= 0 && zz < A.d && yy >= 0 && yy < A.h && xx >= 0 && xx < A.w) {
            if (q[4] == 1) v = A.x_lo[((((size_t)pp[0] * Dl + zz / A.uz) * Hl + yy / A.uy) * Wl + xx / A.ux) * A.c_lo + q[3]];
            else v = A.x[((((size_t)pp[0] * A.d + zz) * A.h + yy) * A.w + xx) * A.c_skip + q[3]];
          }
        }
      }
      sX[k][r] = v;
    }
    for (int e = t; e < WG_K * WG_C; e += 256) {
      const int k = e / WG_C, c = e % WG_C;
      const long long p = p0 + k;
      sD[k][c] = (p < p_end && c0 + c < A.cout) ? A.dy[p * A.ldy + c0 + c] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < WG_K; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&sX[k][4 * tr]);
      const float4 b = *reinterpret_cast<const float4*>(&sD[k][4 * tc]);
      const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
  }
  float* out = A.work + (size_t)blockIdx.y * A.rows * A.cout;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = r0 + 4 * tr + i;
    if (r >= A.rows) break;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c0 + 4 * tc + j;
      if (c < A.cout) out[(size_t)r * A.cout + c] = acc[i][j];
    }
  }
}

// sum of the per-split partials in split order; row taps*Cin goes to db
__global__ void k_wgrad_reduce(const float* __restrict__ work, int nsplit, int rows, int cout, float* __restrict__ dw,
                               float* __restrict__ db) {
  const long long total = (long long)rows * cout;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < nsplit; ++k) s += work[(size_t)k * total + e];
    if (e < total - cout) dw[e] = s;
    else db[e - (total - cout)] = s;
  }
}

int wgrad_split(long long npix, int rows, int cout, long long* per_split) {
  const int tiles = cdiv(rows, WG_R) * cdiv(cout, WG_C);
  long long ns = std::max(1, cdiv(2048, tiles));
  ns = std::min<long long>(ns, std::max<long long>(1, npix / 256));
  long long ps = (npix + ns - 1) / ns;
  ps = (ps + WG_K - 1) / WG_K * WG_K;
  *per_split = ps;
  return (int)((npix + ps - 1) / ps);
}

// ------------------------------------------------------------------------------------------ small elementwise kernels
// Wf[taps-1-tap][co][ci] = W[tap][ci][co]: flipping every spatial axis of a (kz, ky, kx) box reverses the linear tap index
__global__ void k_flip_weights(const float* __restrict__ w, int taps, int cin, int cout, float* __restrict__ wf) {
  const long long total = (long long)taps * cin * cout;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(e % cout); const long long r = e / cout;
    const int ci = (int)(r % cin), tap = (int)(r / cin);
    wf[((size_t)(taps - 1 - tap) * cout + co) * cin + ci] = w[e];
  }
}

// ------------------------------------------------------------------------------------------ StarDist loss
// Fixed-order block reduction of NV doubles per thread into partial[blockIdx.x][NV] (blockDim 256).
template <int NV>
__device__ void block_reduce_store(double (&v)[NV], double* partial) {
  __shared__ double s[NV][256];
#pragma unroll
  for (int i = 0; i < NV; ++i) s[i][threadIdx.x] = v[i];
  __syncthreads();
  for (int st = 128; st > 0; st >>= 1) {
    if (threadIdx.x < st)
#pragma unroll
      for (int i = 0; i < NV; ++i) s[i][threadIdx.x] += s[i][threadIdx.x + st];
    __syncthreads();
  }
  if (threadIdx.x == 0)
#pragma unroll
    for (int i = 0; i < NV; ++i) partial[(size_t)blockIdx.x * NV + i] = s[i][0];
}

constexpr int LOSS_BLOCKS_MAX = 1024;
constexpr float KEPS = 1e-7f;            // Keras' backend epsilon (float32)

int loss_blocks(long long npix) { return std::max(1, std::min(LOSS_BLOCKS_MAX, cdiv(npix, 2048))); }

// pass 1: n_p = #{prob targets >= 0} and sum of the dist mask (last channel of dist_and_mask)
__global__ void __launch_bounds__(256) k_loss_stats(const float* __restrict__ prob_t, const float* __restrict__ dam, long long npix,
                                                    int R, long long per_block, double* __restrict__ partial) {
  double v[2] = {0.0, 0.0};
  const long long b0 = (long long)blockIdx.x * per_block, b1 = llmin(npix, b0 + per_block);
  for (long long p = b0 + threadIdx.x; p < b1; p += 256) {
    v[0] += prob_t[p] >= 0.f ? 1.0 : 0.0;
    v[1] += (double)dam[p * (R + 1) + R];
  }
  block_reduce_store<2>(v, partial);
}

// stats[0] = n_p, stats[1] = M = mean(mask) in float32 (as K.mean(mask))
__global__ void k_loss_stats_final(const double* __restrict__ partial, int nb, long long npix, float* __restrict__ stats) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double a = 0.0, b = 0.0;
  for (int i = 0; i < nb; ++i) { a += partial[2 * i]; b += partial[2 * i + 1]; }
  stats[0] = (float)a;
  stats[1] = (float)(b / (double)npix);
}

// pass 2: the per-pixel loss terms and, when dhead != nullptr, dL/d(prob logit) in dhead[p][0] and dL/d dist in dhead[p][1..R]
__global__ void __launch_bounds__(256) k_loss(const float* __restrict__ prob, const float* __restrict__ dist, const float* __restrict__ prob_t,
                                              const float* __restrict__ dam, long long npix, int R, int mae, float lam, float w0, float w1,
                                              const float* __restrict__ stats, long long per_block, float* __restrict__ dhead,
                                              double* __restrict__ partial) {
  const float n_p = stats[0], M = stats[1];
  const float gp = w0 / n_p;
  const float gd = w1 / ((float)npix * (float)R * (M + KEPS));
  const float gr = w1 * lam / ((float)npix * (float)R);
  double v[3] = {0.0, 0.0, 0.0};          // sum of prob bce, sum m*pen(dt - d), sum (1-m)*pen(d)
  const long long b0 = (long long)blockIdx.x * per_block, b1 = llmin(npix, b0 + per_block);
  for (long long p = b0 + threadIdx.x; p < b1; p += 256) {
    const float t = prob_t[p], y = prob[p];
    float dz = 0.f;
    if (t >= 0.f) {
      const float c = fminf(fmaxf(y, KEPS), 1.f - KEPS);
      v[0] += (double)(-(t * logf(c + KEPS) + (1.f - t) * logf(1.f - c + KEPS)));
      if (y >= KEPS && y <= 1.f - KEPS) {
        const float dc = -(t / (c + KEPS) - (1.f - t) / (1.f - c + KEPS));
        dz = gp * dc * (y * (1.f - y));
      }
    }
    const float* dt = dam + p * (R + 1);
    const float m = dt[R];
    float s1 = 0.f, s2 = 0.f;
    for (int r = 0; r < R; ++r) {
      const float d = dist[p * R + r], e = dt[r] - d;
      float g;
      if (mae) {
        s1 += m * fabsf(e);
        g = -m * (float)((e > 0.f) - (e < 0.f)) * gd;
        if (lam > 0.f) { s2 += (1.f - m) * fabsf(d); g += (1.f - m) * (float)((d > 0.f) - (d < 0.f)) * gr; }
      } else {
        s1 += m * e * e;
        g = -2.f * m * e * gd;
        if (lam > 0.f) { s2 += (1.f - m) * d * d; g += 2.f * (1.f - m) * d * gr; }
      }
      if (dhead) dhead[p * (R + 1) + 1 + r] = g;
    }
    v[1] += (double)s1; v[2] += (double)s2;
    if (dhead) dhead[p * (R + 1)] = dz;
  }
  block_reduce_store<3>(v, partial);
}

// out = (loss, prob_loss, dist_loss, skipped); state (optional) = (t, n_skipped, skip): a batch without any prob target (n_p = 0)
// is skipped -- Adam leaves the weights and t alone
__global__ void k_loss_final(const double* __restrict__ partial, int nb, long long npix, int R, float lam, float w0, float w1,
                             const float* __restrict__ stats, float* __restrict__ out, int* __restrict__ state) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double a = 0.0, b = 0.0, c = 0.0;
  for (int i = 0; i < nb; ++i) { a += partial[3 * i]; b += partial[3 * i + 1]; c += partial[3 * i + 2]; }
  const double n_p = stats[0], M = stats[1];
  const double NR = (double)npix * R;
  const float lp = (float)(a / n_p);
  const float ld = (float)(b / (NR * ((double)M + (double)KEPS)) + (lam > 0.f ? (double)lam * c / NR : 0.0));
  const int skip = stats[0] == 0.f;
  out[0] = w0 * lp + w1 * ld; out[1] = lp; out[2] = ld; out[3] = (float)skip;
  if (state) {
    state[2] = skip;
    if (skip) state[1] += 1; else state[0] += 1;
  }
}

// ------------------------------------------------------------------------------------------ class loss
// Weighted categorical cross-entropy of the softmax output s [npix][C] against prob_class t [npix][C] (base.py:108-126):
// S = sum_k (s_k + eps), q_k = s_k / S, c_k = clip(q_k, eps, 1 - eps), l = -sum_k w_k [t_k >= 0] t_k log c_k.  When dz !=
// nullptr it receives dL/dz_j = (w2 / npix) s_j (b_j - sum_i s_i b_i), the softmax backward of b_j = a_j / S - (sum_k a_k s_k) / S^2,
// a_k = -w_k [t_k >= 0] t_k / q_k where eps <= q_k <= 1 - eps (the clip passes no gradient outside).  One thread per pixel.
constexpr int CLS_MAX = 32;              // n_classes + 1, as in sdb_class_head

__global__ void __launch_bounds__(256) k_class_loss(const float* __restrict__ s, const float* __restrict__ t, long long npix, int C,
                                                    const float* __restrict__ cw, float w2, long long per_block, float* __restrict__ dz,
                                                    double* __restrict__ partial) {
  __shared__ float sw[CLS_MAX];
  if (threadIdx.x < C) sw[threadIdx.x] = cw[threadIdx.x];
  __syncthreads();
  const float gs = w2 / (float)npix;
  double v[1] = {0.0};
  const long long b0 = (long long)blockIdx.x * per_block, b1 = llmin(npix, b0 + per_block);
  for (long long p = b0 + threadIdx.x; p < b1; p += 256) {
    const float* sp = s + p * C;
    const float* tp = t + p * C;
    float S = 0.f;
    for (int k = 0; k < C; ++k) S += sp[k] + KEPS;
    float l = 0.f, A = 0.f, a[CLS_MAX];
    for (int k = 0; k < C; ++k) {
      const float q = sp[k] / S, tk = tp[k];
      const float c = fminf(fmaxf(q, KEPS), 1.f - KEPS);
      const float wt = tk >= 0.f ? sw[k] * tk : 0.f;
      l += wt * logf(c);
      a[k] = (q >= KEPS && q <= 1.f - KEPS) ? -wt / q : 0.f;
      A += a[k] * sp[k];
    }
    v[0] -= (double)l;
    if (dz) {
      const float AS2 = A / (S * S);
      float sb = 0.f;
      for (int k = 0; k < C; ++k) { a[k] = a[k] / S - AS2; sb += sp[k] * a[k]; }
      for (int k = 0; k < C; ++k) dz[p * C + k] = gs * (sp[k] * (a[k] - sb));
    }
  }
  block_reduce_store<1>(v, partial);
}

// out_class = L_class = sum / npix; total += w2 * L_class (total: the loss sdb_stardist_loss wrote)
__global__ void k_class_loss_final(const double* __restrict__ partial, int nb, long long npix, float w2, float* __restrict__ total,
                                   float* __restrict__ out_class) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double a = 0.0;
  for (int i = 0; i < nb; ++i) a += partial[i];
  const float lc = (float)(a / (double)npix);
  *out_class = lc;
  *total = __fadd_rn(*total, __fmul_rn(w2, lc));
}

// ------------------------------------------------------------------------------------------ heads backward
// dfeat[p][f] = sum_o dhead[p][o] * W[f][o] (W[f][0] = w_prob[f], W[f][1 + r] = w_dist[f][r]), o in order, then the ReLU
// mask of the features layer's output.  32 pixels per CTA.
__global__ void __launch_bounds__(128) k_heads_backward(const float* __restrict__ feat, const float* __restrict__ dhead, long long npix,
                                                        int cf, const float* __restrict__ wp, const float* __restrict__ wd, int R, int relu,
                                                        float* __restrict__ dfeat) {
  extern __shared__ float sm[];
  const int NO = R + 1;
  float* sW = sm;                 // [NO][cf]
  float* sG = sW + NO * cf;       // [32][NO]
  for (int e = threadIdx.x; e < NO * cf; e += blockDim.x) {
    const int o = e / cf, f = e % cf;
    sW[e] = o == 0 ? wp[f] : wd[(size_t)f * R + o - 1];
  }
  const long long p0 = (long long)blockIdx.x * 32;
  for (int e = threadIdx.x; e < 32 * NO; e += blockDim.x) {
    const long long p = p0 + e / NO;
    sG[e] = p < npix ? dhead[p0 * NO + e] : 0.f;
  }
  __syncthreads();
  for (int px = 0; px < 32; ++px) {
    const long long p = p0 + px;
    if (p >= npix) break;
    for (int f = threadIdx.x; f < cf; f += blockDim.x) {
      float acc = 0.f;
      for (int o = 0; o < NO; ++o) acc = fmaf(sG[px * NO + o], sW[o * cf + f], acc);
      if (relu && !(feat[p * cf + f] > 0.f)) acc = 0.f;
      dfeat[p * cf + f] = acc;
    }
  }
}

// dfeat[p][f] (+)= sum_o dz[p][o] * W[f][o] (W [cf][C], the prob_class kernel), o in order, times the ReLU mask of feat when
// relu = 1.  accumulate = 1 adds the class branch's share to a tensor the heads' backward has written (both read one input).
// 32 pixels per CTA.
__global__ void __launch_bounds__(128) k_class_head_backward(const float* __restrict__ feat, const float* __restrict__ dz, long long npix,
                                                             int cf, const float* __restrict__ w, int C, int relu, int accumulate,
                                                             float* __restrict__ dfeat) {
  extern __shared__ float sm[];
  float* sW = sm;                 // [C][cf]
  float* sG = sW + C * cf;        // [32][C]
  for (int e = threadIdx.x; e < C * cf; e += blockDim.x) {
    const int o = e / cf, f = e % cf;
    sW[e] = w[(size_t)f * C + o];
  }
  const long long p0 = (long long)blockIdx.x * 32;
  for (int e = threadIdx.x; e < 32 * C; e += blockDim.x) {
    const long long p = p0 + e / C;
    sG[e] = p < npix ? dz[p0 * C + e] : 0.f;
  }
  __syncthreads();
  for (int px = 0; px < 32; ++px) {
    const long long p = p0 + px;
    if (p >= npix) break;
    for (int f = threadIdx.x; f < cf; f += blockDim.x) {
      float acc = 0.f;
      for (int o = 0; o < C; ++o) acc = fmaf(sG[px * C + o], sW[o * cf + f], acc);
      if (relu && !(feat[p * cf + f] > 0.f)) acc = 0.f;
      dfeat[p * cf + f] = accumulate ? __fadd_rn(dfeat[p * cf + f], acc) : acc;
    }
  }
}

// ------------------------------------------------------------------------------------------ Adam (TF2 Keras)
// m += (g - m)(1 - b1); v += (g^2 - v)(1 - b2); w -= m*alpha / (sqrt(v) + eps), alpha = lr * coef[t - 1] with coef(t) =
// sqrt(1 - b2^t) / (1 - b1^t) tabulated on the host in float32.  Every operation is an explicitly rounded intrinsic, so the
// result does not depend on the TU's contraction flags and equals a float32 numpy restatement with the same order.
__global__ void k_adam(float* __restrict__ w, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, long long n,
                       float lr, float omb1, float omb2, float eps, const float* __restrict__ coef, const int* __restrict__ state) {
  if (state[2]) return;
  const float alpha = __fmul_rn(lr, coef[state[0] - 1]);
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const float gg = g[e];
    const float mm = __fadd_rn(m[e], __fmul_rn(__fsub_rn(gg, m[e]), omb1));
    const float vv = __fadd_rn(v[e], __fmul_rn(__fsub_rn(__fmul_rn(gg, gg), v[e]), omb2));
    m[e] = mm; v[e] = vv;
    w[e] = __fsub_rn(w[e], __fdiv_rn(__fmul_rn(mm, alpha), __fadd_rn(__fsqrt_rn(vv), eps)));
  }
}

int grid_1d(long long n, int per) { return (int)std::max<long long>(1, std::min<long long>(cdiv(n, 256), 132LL * per)); }

// ------------------------------------------------------------------------------------------ data-parallel reduction
constexpr int REDUCE_WORLD_MAX = 4096;   // the member list lives in shared memory
// rows [W][ld]: replica r's flat gradient in rows[r * ld, + P) and its loss row (loss, prob_loss, dist_loss, skipped[, ...]) in
// rows[r * ld + P, + n_out).  S = the replicas with skipped == 0 in ascending rank order, or all W replicas when none is: g[i] =
// (S_0[i] + S_1[i] + ...) / |S| and out[k] likewise, fp32 additions from the first member, then one fp32 division.  Block 0 also
// advances the shared step state as k_loss_final does for one batch, with skip = (no replica ok).  rows and g may alias (W = 1:
// every element is read by the thread that writes it), so neither is __restrict__.  vec = 1: ld % 4 == 0 and 16-byte aligned
// rows and g, read and written as float4 up to P rounded down to 4.
__global__ void __launch_bounds__(256) k_replica_reduce(const float* rows, int W, long long P, int n_out, long long ld, int vec, float* g,
                                                        float* __restrict__ out, int* __restrict__ state) {
  extern __shared__ int sel[];             // [W]: the members of S, then their count in sel[W]
  if (threadIdx.x == 0) {
    int n = 0;
    for (int r = 0; r < W; ++r)
      if (rows[(size_t)r * ld + P + 3] == 0.f) sel[n++] = r;
    const int skip = n == 0;
    if (skip)
      for (int r = 0; r < W; ++r) sel[n++] = r;
    sel[W] = n;
    if (blockIdx.x == 0) {
      for (int k = 0; k < n_out; ++k) {
        float a = rows[(size_t)sel[0] * ld + P + k];
        for (int j = 1; j < n; ++j) a = __fadd_rn(a, rows[(size_t)sel[j] * ld + P + k]);
        out[k] = __fdiv_rn(a, (float)n);
      }
      state[2] = skip;
      if (skip) state[1] += 1; else state[0] += 1;
    }
  }
  __syncthreads();
  const int n = sel[W];
  const float fn = (float)n;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
  long long done = 0;
  if (vec) {
    const long long P4 = P / 4;
    for (long long e = tid; e < P4; e += stride) {
      float4 a = reinterpret_cast<const float4*>(rows + (size_t)sel[0] * ld)[e];
      for (int j = 1; j < n; ++j) {
        const float4 b = reinterpret_cast<const float4*>(rows + (size_t)sel[j] * ld)[e];
        a.x = __fadd_rn(a.x, b.x); a.y = __fadd_rn(a.y, b.y); a.z = __fadd_rn(a.z, b.z); a.w = __fadd_rn(a.w, b.w);
      }
      a.x = __fdiv_rn(a.x, fn); a.y = __fdiv_rn(a.y, fn); a.z = __fdiv_rn(a.z, fn); a.w = __fdiv_rn(a.w, fn);
      reinterpret_cast<float4*>(g)[e] = a;
    }
    done = P4 * 4;
  }
  for (long long e = done + tid; e < P; e += stride) {
    float a = rows[(size_t)sel[0] * ld + e];
    for (int j = 1; j < n; ++j) a = __fadd_rn(a, rows[(size_t)sel[j] * ld + e]);
    g[e] = __fdiv_rn(a, fn);
  }
}

}  // namespace

extern "C" long long sdb_conv_wgrad_workspace(long long npix, int taps, int cin, int cout) {
  long long ps;
  const int rows = taps * cin + 1;
  const int ns = wgrad_split(npix, rows, cout, &ps);
  return (long long)ns * rows * cout;
}

namespace {

// prec selects the partial-sum kernel over the same splits and workspace: WGRAD_FP32 (here), WGRAD_TF32 (the TF32 tensor
// cores, unet_train_tf32.cu) or WGRAD_BF16_* (bf16 tensor cores on bf16 activations, unet_train_bf16.cu)
int conv_wgrad(const char* who, const void* d_x, const void* d_x_lo, int n, int d, int h, int w, int cin_skip, int cin_lo,
               int uz, int uy, int ux, int kz, int ky, int kx, const void* d_dy, int ldy, int cout, float* d_work,
               long long work_floats, float* d_dw, float* d_db, cudaStream_t st, int prec = sdb::WGRAD_FP32) {
  if (n < 1 || d < 1 || h < 1 || w < 1 || cout < 1 || ldy < cout || cin_skip < 0 || cin_lo < 0 || cin_skip + cin_lo < 1) {
    sdb::set_error(std::string(who) + ": bad arguments"); return 1;
  }
  if (cin_lo && (d_x_lo == nullptr || uz < 1 || uy < 1 || ux < 1 || d % uz || h % uy || w % ux)) {
    sdb::set_error(std::string(who) + ": low-resolution source needs a pointer and divisible up-sampling factors"); return 1;
  }
  WgradArgs A;
  A.x = (const float*)d_x; A.x_lo = (const float*)d_x_lo; A.dy = (const float*)d_dy; A.prec = prec;
  A.n = n; A.d = d; A.h = h; A.w = w; A.c_skip = cin_skip; A.c_lo = cin_lo;
  A.uz = cin_lo ? uz : 1; A.uy = cin_lo ? uy : 1; A.ux = cin_lo ? ux : 1;
  A.kz = kz; A.ky = ky; A.kx = kx; A.pz = (kz - 1) / 2; A.py = (ky - 1) / 2; A.px = (kx - 1) / 2;
  A.ldy = ldy; A.cout = cout;
  const int taps = kz * ky * kx;
  A.rows = taps * (cin_skip + cin_lo) + 1;
  A.npix = (long long)n * d * h * w;
  const int ns = wgrad_split(A.npix, A.rows, cout, &A.per_split);
  if ((long long)ns * A.rows * cout > work_floats) { sdb::set_error(std::string(who) + ": workspace too small"); return 1; }
  A.work = d_work;
  if (prec == sdb::WGRAD_TF32) {
    if (sdb::conv_wgrad_tf32_launch(A, ns, st)) return 1;
  } else if (prec != sdb::WGRAD_FP32) {
    if (sdb::conv_wgrad_bf16_launch(A, ns, st)) return 1;
  } else {
    dim3 grid(cdiv(A.rows, WG_R) * cdiv(cout, WG_C), ns);
    SDB_LAUNCH(k_conv_wgrad, grid, 256, 0, st, A);
  }
  SDB_LAUNCH(k_wgrad_reduce, grid_1d((long long)A.rows * cout, 16), 256, 0, st, d_work, ns, A.rows, cout, d_dw, d_db);
  return 0;
}

}  // namespace

extern "C" int sdb_conv_wgrad_nd(const float* d_x, const float* d_x_lo, int n, int d, int h, int w, int cin_skip, int cin_lo,
                                 int uz, int uy, int ux, int kz, int kyx, const float* d_dy, int ldy, int cout, float* d_work,
                                 long long work_floats, float* d_dw, float* d_db, sdb_stream_t stream) {
  if ((kz != 1 && kz != 3) || (kyx != 1 && kyx != 3) || (kz == 3 && kyx != 3)) { sdb::set_error("conv_wgrad_nd: kernel must be 1^d or 3^d"); return 1; }
  return conv_wgrad("conv_wgrad_nd", d_x, d_x_lo, n, d, h, w, cin_skip, cin_lo, uz, uy, ux, kz, kyx, kyx, d_dy, ldy, cout, d_work,
                    work_floats, d_dw, d_db, (cudaStream_t)stream);
}

extern "C" int sdb_conv_wgrad_tf32_nd(const float* d_x, const float* d_x_lo, int n, int d, int h, int w, int cin_skip, int cin_lo,
                                      int uz, int uy, int ux, int kz, int kyx, const float* d_dy, int ldy, int cout, float* d_work,
                                      long long work_floats, float* d_dw, float* d_db, sdb_stream_t stream) {
  if ((kz != 1 && kz != 3) || (kyx != 1 && kyx != 3) || (kz == 3 && kyx != 3)) { sdb::set_error("conv_wgrad_tf32_nd: kernel must be 1^d or 3^d"); return 1; }
  return conv_wgrad("conv_wgrad_tf32_nd", d_x, d_x_lo, n, d, h, w, cin_skip, cin_lo, uz, uy, ux, kz, kyx, kyx, d_dy, ldy, cout, d_work,
                    work_floats, d_dw, d_db, (cudaStream_t)stream, sdb::WGRAD_TF32);
}

extern "C" int sdb_conv_wgrad_bf16_nd(const void* d_x, const void* d_x_lo, int n, int d, int h, int w, int cin_skip, int cin_lo,
                                      int uz, int uy, int ux, int kz, int kyx, const void* d_dy, int dy_bf16, int ldy, int cout,
                                      float* d_work, long long work_floats, float* d_dw, float* d_db, sdb_stream_t stream) {
  if ((kz != 1 && kz != 3) || (kyx != 1 && kyx != 3) || (kz == 3 && kyx != 3)) { sdb::set_error("conv_wgrad_bf16_nd: kernel must be 1^d, 3^d or (1, 3, 3)"); return 1; }
  return conv_wgrad("conv_wgrad_bf16_nd", d_x, d_x_lo, n, d, h, w, cin_skip, cin_lo, uz, uy, ux, kz, kyx, kyx, d_dy, ldy, cout, d_work,
                    work_floats, d_dw, d_db, (cudaStream_t)stream, dy_bf16 ? sdb::WGRAD_BF16_DY_BF16 : sdb::WGRAD_BF16_DY_F32);
}

extern "C" int sdb_conv_wgrad_any_nd(const float* d_x, const float* d_x_lo, int n, int d, int h, int w, int cin_skip, int cin_lo,
                                     int uz, int uy, int ux, int kz, int ky, int kx, const float* d_dy, int ldy, int cout, float* d_work,
                                     long long work_floats, float* d_dw, float* d_db, sdb_stream_t stream) {
  if (kz < 1 || kz > 7 || ky < 1 || ky > 7 || kx < 1 || kx > 7) { sdb::set_error("conv_wgrad_any_nd: kernel extents must be in 1..7"); return 1; }
  return conv_wgrad("conv_wgrad_any_nd", d_x, d_x_lo, n, d, h, w, cin_skip, cin_lo, uz, uy, ux, kz, ky, kx, d_dy, ldy, cout, d_work,
                    work_floats, d_dw, d_db, (cudaStream_t)stream);
}

extern "C" int sdb_conv_flip_weights(const float* d_w, int taps, int cin, int cout, float* d_wf, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (taps < 1 || cin < 1 || cout < 1) { sdb::set_error("conv_flip_weights: bad arguments"); return 1; }
  SDB_LAUNCH(k_flip_weights, grid_1d((long long)taps * cin * cout, 16), 256, 0, st, d_w, taps, cin, cout, d_wf);
  return 0;
}

extern "C" int sdb_decoder_split(const float* d_dcat, int n, int d, int h, int w, int c_lo, int c_skip, int uz, int uy, int ux,
                                 float* d_dlo, float* d_dskip, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (c_lo < 1 || c_skip < 1 || uz < 1 || uy < 1 || ux < 1 || d % uz || h % uy || w % ux) { sdb::set_error("decoder_split: bad arguments"); return 1; }
  const long long total = (long long)n * d * h * w / ((long long)uz * uy * ux) * c_lo + (long long)n * d * h * w * c_skip;
  SDB_LAUNCH(sdb::k_decoder_split<float>, grid_1d(total, 32), 256, 0, st, d_dcat, n, d, h, w, c_lo, c_skip, uz, uy, ux, d_dlo, d_dskip);
  return 0;
}

extern "C" int sdb_relu_backward(float* d_g, const float* d_y, long long n, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n <= 0) return 0;
  SDB_LAUNCH(sdb::k_relu_backward<float>, grid_1d(n, 32), 256, 0, st, d_g, d_y, n);
  return 0;
}

extern "C" int sdb_maxpool_backward_nd(const float* d_x, const float* d_gy, int n, int d, int h, int w, int c, int pz, int py, int px,
                                       int accumulate, float* d_gx, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (pz < 1 || py < 1 || px < 1 || d % pz || h % py || w % px || c < 1) { sdb::set_error("maxpool_backward_nd: sizes must be divisible by the pool"); return 1; }
  const long long total = (long long)n * (d / pz) * (h / py) * (w / px) * c;
  SDB_LAUNCH(sdb::k_maxpool_backward<float>, grid_1d(total, 32), 256, 0, st, d_x, d_gy, n, d, h, w, c, pz, py, px, accumulate, d_gx);
  return 0;
}

extern "C" long long sdb_stardist_loss_workspace(long long npix) {
  return (long long)loss_blocks(npix) * 3 * (long long)sizeof(double);
}

extern "C" int sdb_stardist_loss(const float* d_prob, const float* d_dist, const float* d_prob_t, const float* d_dam, long long npix,
                                 int n_rays, int mae, float lam, float w0, float w1, void* d_work, float* d_stats, float* d_dhead,
                                 float* d_out, int* d_state, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (npix < 1 || n_rays < 1) { sdb::set_error("stardist_loss: bad arguments"); return 1; }
  const int nb = loss_blocks(npix);
  const long long per = (npix + nb - 1) / nb;
  double* part = (double*)d_work;
  SDB_LAUNCH(k_loss_stats, nb, 256, 0, st, d_prob_t, d_dam, npix, n_rays, per, part);
  SDB_LAUNCH(k_loss_stats_final, 1, 32, 0, st, part, nb, npix, d_stats);
  SDB_LAUNCH(k_loss, nb, 256, 0, st, d_prob, d_dist, d_prob_t, d_dam, npix, n_rays, mae, lam, w0, w1, d_stats, per, d_dhead, part);
  SDB_LAUNCH(k_loss_final, 1, 32, 0, st, part, nb, npix, n_rays, lam, w0, w1, d_stats, d_out, d_state);
  return 0;
}

extern "C" int sdb_heads_backward(const float* d_feat, const float* d_dhead, long long npix, int cfeat, const float* d_wp,
                                  const float* d_wd, int n_rays, int relu, float* d_dfeat, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (npix <= 0) return 0;
  const size_t smem = (size_t)((n_rays + 1) * cfeat + 32 * (n_rays + 1)) * sizeof(float);
  if (smem > 200 * 1024) { sdb::set_error("heads_backward: n_rays * features too large"); return 1; }
  static bool attr_set = false;
  if (!attr_set) { SDB_CUDA(cudaFuncSetAttribute(k_heads_backward, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); attr_set = true; }
  SDB_LAUNCH(k_heads_backward, cdiv(npix, 32), 128, smem, st, d_feat, d_dhead, npix, cfeat, d_wp, d_wd, n_rays, relu, d_dfeat);
  return 0;
}

extern "C" long long sdb_stardist_class_loss_workspace(long long npix) {
  return (long long)loss_blocks(npix) * (long long)sizeof(double);
}

extern "C" int sdb_stardist_class_loss(const float* d_s, const float* d_t, long long npix, int n_out, const float* d_class_w, float w2,
                                       void* d_work, float* d_dz, float* d_total, float* d_out_class, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (npix < 1 || n_out < 1 || n_out > CLS_MAX) { sdb::set_error("stardist_class_loss: npix >= 1 and n_classes + 1 in [1,32] required"); return 1; }
  const int nb = loss_blocks(npix);
  const long long per = (npix + nb - 1) / nb;
  double* part = (double*)d_work;
  SDB_LAUNCH(k_class_loss, nb, 256, 0, st, d_s, d_t, npix, n_out, d_class_w, w2, per, d_dz, part);
  SDB_LAUNCH(k_class_loss_final, 1, 32, 0, st, part, nb, npix, w2, d_total, d_out_class);
  return 0;
}

extern "C" int sdb_class_head_backward(const float* d_feat, const float* d_dz, long long npix, int cfeat, const float* d_w, int n_out,
                                       int relu, int accumulate, float* d_dfeat, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (npix <= 0) return 0;
  if (n_out < 1 || n_out > CLS_MAX || cfeat < 1) { sdb::set_error("class_head_backward: n_classes + 1 must be in [1,32]"); return 1; }
  const size_t smem = (size_t)(n_out * cfeat + 32 * n_out) * sizeof(float);
  if (smem > 200 * 1024) { sdb::set_error("class_head_backward: n_classes * features too large"); return 1; }
  static bool attr_set = false;
  if (!attr_set) { SDB_CUDA(cudaFuncSetAttribute(k_class_head_backward, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024)); attr_set = true; }
  SDB_LAUNCH(k_class_head_backward, cdiv(npix, 32), 128, smem, st, d_feat, d_dz, npix, cfeat, d_w, n_out, relu, accumulate, d_dfeat);
  return 0;
}

extern "C" int sdb_adam_step(float* d_w, const float* d_g, float* d_m, float* d_v, long long n, float lr, float one_minus_b1,
                             float one_minus_b2, float eps, const float* d_coef, const int* d_state, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n <= 0) return 0;
  SDB_LAUNCH(k_adam, grid_1d(n, 8), 256, 0, st, d_w, d_g, d_m, d_v, n, lr, one_minus_b1, one_minus_b2, eps, d_coef, d_state);
  return 0;
}

extern "C" int sdb_replica_reduce(const float* d_rows, int world, long long n_params, int n_out, long long ld, float* d_g, float* d_out,
                                  int* d_state, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (world < 1 || world > REDUCE_WORLD_MAX || n_params < 0 || n_out < 4 || ld < n_params + n_out) {
    sdb::set_error("replica_reduce: 1 <= world <= 4096, n_out >= 4 and ld >= n_params + n_out required");
    return 1;
  }
  const int vec = ld % 4 == 0 && (uintptr_t)d_rows % 16 == 0 && (uintptr_t)d_g % 16 == 0;
  const long long work = vec ? std::max(n_params / 4, n_params % 4) : n_params;
  SDB_LAUNCH(k_replica_reduce, grid_1d(work, 8), 256, (size_t)(world + 1) * sizeof(int), st, d_rows, world, n_params, n_out, ld, vec,
             d_g, d_out, d_state);
  return 0;
}
