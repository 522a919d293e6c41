// unet_train_bf16.cu -- the bf16 tensor-core kernels of the U-Net training step under the mixed_bfloat16 policy
// (stardist_b200.mixed_precision, DESIGN.md 4.2).  Activations and the gradients between layers are stored as bf16 NHWC /
// NDHWC; parameters, their gradients, biases, the heads' outputs and the loss stay fp32.  Every GEMM multiplies bf16 values
// on mma.sync.m16n8k16 and accumulates in fp32; an fp32 operand is rounded on load with round-to-nearest-even
// (__float2bfloat16_rn, cvt.rn.bf16.f32).
//   convolution      y[p, co] = act(sum_(tap, ci) x[p + tap - pad, ci] * wb[tap, co, ci] + b[co]) stored as one bf16 rounding;
//                    the decoder input [upsample(x_lo), skip] is read through the forward loader's up-sampling address
//                    math.  The same kernel gives the input gradient (dY with the flipped kernel), the heads (fp32
//                    prob / dist), the heads' and class head's input gradients (an fp32 dY rounded on load) and the class
//                    logits (fp32).
//   weight gradient  dW[tap, ci, co] = sum_p x[p + tap - pad, ci] * dy[p, co] over sdb_conv_wgrad_nd's pixel splits,
//                    workspace and in-order reduction (unet_train.cu); db = sum_p dy[p, co] in fp32 of dy as stored.
// No float atomics: each output element is accumulated by one thread in a fixed order, so results are bit-identical run to run.
#include <stdint.h>
#include <algorithm>
#include <cuda_bf16.h>
#include "common.cuh"
#include "wgrad.cuh"
#include "train_elem.cuh"
#include "../../include/stardist_b200.h"

namespace {

using sdb::cdiv;
using bf16 = __nv_bfloat16;

int grid_1d(long long n, int per) { return (int)std::max<long long>(1, std::min<long long>(cdiv(n, 256), 132LL * per)); }

// c += a * b: a 16x16 (row-major), b 16x8 (column-major), bf16 operands, c 16x8 fp32
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

__device__ __forceinline__ void ldsm_x4_trans(uint32_t (&r)[4], const void* p) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(s));
}

// 16 bytes global -> shared; pred = false fills zeros and reads nothing
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool pred) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" :: "r"(s), "l"(gmem), "r"(pred ? 16 : 0));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N)); }

__device__ __forceinline__ uint32_t ld32(const bf16* p) { return *reinterpret_cast<const uint32_t*>(p); }

// ------------------------------------------------------------------------------------------ convolution
enum { EPI_BF16 = 0, EPI_HEADS = 1, EPI_F32 = 2 };

struct ConvArgs {
  const void* x; const void* x_lo;  // bf16 [n, d, h, w, c_skip] and [n, d/uz, h/uy, w/ux, c_lo]; a_f32: x is fp32, rounded on load
  int a_f32;
  int n, d, h, w, c_skip, c_lo, uz, uy, ux, kz, ky, kx;
  const bf16* wb;                   // [tap][cout][cin]
  const float* bias;                // [cout] or nullptr; EPI_HEADS: the prob bias, bias2 the dist bias
  const float* bias2;
  int cout, relu, mode, accumulate, R;
  void* out;                        // EPI_BF16: bf16 [npix][cout]; EPI_F32: fp32 [npix][cout]; EPI_HEADS: fp32 dist [npix][R]
  float* prob;                      // EPI_HEADS: fp32 [npix]
};

// CTA tile 128 consecutive output pixels x NT output channels (NT = 32 when cout <= 32, else 64); K steps of 32 input channels
// of one tap, double-buffered; 8 warps of 32 columns x (128 / warps along M) rows.  VEC: c_skip, c_lo and cin multiples of
// 8 and bf16 input, so every 8-channel group is one 16-byte cp.async from one source; otherwise element loads.
constexpr int CM = 128, CK = 32, CLD = CK + 8;       // row pitch 80 bytes: the 32-bit fragment loads hit 32 distinct banks

template <int NT, bool VEC>
__global__ void __launch_bounds__(256) k_conv_bf16(ConvArgs A) {
  constexpr int WN = NT / 32, WM = 8 / WN, MT = CM / WM / 16;
  __shared__ __align__(16) bf16 sA[2][CM][CLD];      // input [pixel][channel]
  __shared__ __align__(16) bf16 sB[2][NT][CLD];      // weights [cout][channel]
  __shared__ int sPix[CM][4];                        // img, z, y, x (img < 0: past the end)
  const int cin = A.c_skip + A.c_lo;
  const long long npix = (long long)A.n * A.d * A.h * A.w;
  const long long p0 = (long long)blockIdx.x * CM;
  const int n0 = blockIdx.y * NT;
  const int t = threadIdx.x, warp = t / 32, lane = t % 32, g = lane / 4, t4 = lane % 4;
  const int wm = (warp / WN) * (CM / WM), wn = (warp % WN) * 32;
  if (t < CM) {
    const long long p = p0 + t;
    int* q = sPix[t];
    if (p < npix) {
      q[3] = (int)(p % A.w); q[2] = (int)((p / A.w) % A.h); q[1] = (int)((p / ((long long)A.w * A.h)) % A.d);
      q[0] = (int)(p / ((long long)A.w * A.h * A.d));
    } else {
      q[0] = -1; q[1] = q[2] = q[3] = 0;
    }
  }
  __syncthreads();
  const int n_cc = (cin + CK - 1) / CK, steps = A.kz * A.ky * A.kx * n_cc;
  const int pz = (A.kz - 1) / 2, py = (A.ky - 1) / 2, px = (A.kx - 1) / 2;
  const int Dl = A.d / A.uz, Hl = A.h / A.uy, Wl = A.w / A.ux;
  const bf16* xb = (const bf16*)A.x; const bf16* lb = (const bf16*)A.x_lo;
  auto load = [&](int s, int buf) {
    const int tap = s / n_cc, c0 = (s % n_cc) * CK;
    const int oz = tap / (A.ky * A.kx) - pz, oy = (tap / A.kx) % A.ky - py, ox = tap % A.kx - px;
    if (VEC) {
      for (int e = t; e < CM * (CK / 8); e += 256) {
        const int m = e / (CK / 8), k = 8 * (e % (CK / 8)), c = c0 + k;
        const int* pp = sPix[m];
        const int zz = pp[1] + oz, yy = pp[2] + oy, xx = pp[3] + ox;
        const bool ok = pp[0] >= 0 && c < cin && zz >= 0 && zz < A.d && yy >= 0 && yy < A.h && xx >= 0 && xx < A.w;
        const bf16* src = xb;
        if (ok) src = c < A.c_lo ? lb + ((((size_t)pp[0] * Dl + zz / A.uz) * Hl + yy / A.uy) * Wl + xx / A.ux) * A.c_lo + c
                                 : xb + ((((size_t)pp[0] * A.d + zz) * A.h + yy) * A.w + xx) * A.c_skip + (c - A.c_lo);
        cp_async16(&sA[buf][m][k], src, ok);
      }
      for (int e = t; e < NT * (CK / 8); e += 256) {
        const int nn = e / (CK / 8), k = 8 * (e % (CK / 8)), co = n0 + nn, c = c0 + k;
        const bool ok = co < A.cout && c < cin;
        cp_async16(&sB[buf][nn][k], ok ? A.wb + ((size_t)tap * A.cout + co) * cin + c : A.wb, ok);
      }
      cp_async_commit();
    } else {
      for (int e = t; e < CM * CK; e += 256) {
        const int m = e / CK, k = e % CK, c = c0 + k;
        const int* pp = sPix[m];
        const int zz = pp[1] + oz, yy = pp[2] + oy, xx = pp[3] + ox;
        bf16 v = __float2bfloat16_rn(0.f);
        if (pp[0] >= 0 && c < cin && zz >= 0 && zz < A.d && yy >= 0 && yy < A.h && xx >= 0 && xx < A.w) {
          if (c < A.c_lo) v = lb[((((size_t)pp[0] * Dl + zz / A.uz) * Hl + yy / A.uy) * Wl + xx / A.ux) * A.c_lo + c];
          else {
            const size_t i = ((((size_t)pp[0] * A.d + zz) * A.h + yy) * A.w + xx) * A.c_skip + (c - A.c_lo);
            v = A.a_f32 ? __float2bfloat16_rn(((const float*)A.x)[i]) : xb[i];
          }
        }
        sA[buf][m][k] = v;
      }
      for (int e = t; e < NT * CK; e += 256) {
        const int nn = e / CK, k = e % CK, co = n0 + nn, c = c0 + k;
        sB[buf][nn][k] = (co < A.cout && c < cin) ? A.wb[((size_t)tap * A.cout + co) * cin + c] : __float2bfloat16_rn(0.f);
      }
    }
  };
  float acc[MT][4][4];
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.f;
  load(0, 0);
  for (int s = 0; s < steps; ++s) {
    if (s + 1 < steps) {
      load(s + 1, (s + 1) & 1);
      if (VEC) cp_async_wait<1>();
    } else if (VEC) {
      cp_async_wait<0>();
    }
    __syncthreads();
    const int buf = s & 1, kmax = cin - (s % n_cc) * CK;
#pragma unroll
    for (int kk = 0; kk < CK; kk += 16) {
      if (kk >= kmax) break;                         // the rest of the step is zero padding
      uint32_t a[MT][4], b[4][2];
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        const int m = wm + mt * 16 + g;
        a[mt][0] = ld32(&sA[buf][m][kk + 2 * t4]); a[mt][1] = ld32(&sA[buf][m + 8][kk + 2 * t4]);
        a[mt][2] = ld32(&sA[buf][m][kk + 2 * t4 + 8]); a[mt][3] = ld32(&sA[buf][m + 8][kk + 2 * t4 + 8]);
      }
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const int nn = wn + nt * 8 + g;
        b[nt][0] = ld32(&sB[buf][nn][kk + 2 * t4]); b[nt][1] = ld32(&sB[buf][nn][kk + 2 * t4 + 8]);
      }
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) mma_bf16(acc[mt][nt], a[mt], b[nt]);
    }
    __syncthreads();
  }
  // epilogue: fp32 accumulator + fp32 bias, activation in fp32, one rounding per stored bf16
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const long long p = p0 + wm + mt * 16 + g + (i >= 2 ? 8 : 0);
        const int c = n0 + wn + nt * 8 + 2 * t4 + (i & 1);
        if (p >= npix || c >= A.cout) continue;
        float v = acc[mt][nt][i];
        if (A.mode == EPI_HEADS) {
          v += c == 0 ? A.bias[0] : A.bias2[c - 1];
          if (c == 0) A.prob[p] = 1.f / (1.f + expf(-v));
          else ((float*)A.out)[p * A.R + c - 1] = v;
        } else if (A.mode == EPI_F32) {
          ((float*)A.out)[p * A.cout + c] = A.bias ? v + A.bias[c] : v;
        } else {
          bf16* o = (bf16*)A.out + p * A.cout + c;
          if (A.bias) v += A.bias[c];
          if (A.relu) v = fmaxf(v, 0.f);
          if (A.accumulate) v = __bfloat162float(*o) + v;
          *o = __float2bfloat16_rn(v);
        }
      }
}

int conv_bf16_launch(const ConvArgs& A, cudaStream_t st) {
  const long long npix = (long long)A.n * A.d * A.h * A.w;
  const int cin = A.c_skip + A.c_lo;
  const bool vec = !A.a_f32 && A.c_skip % 8 == 0 && A.c_lo % 8 == 0 && ((uintptr_t)A.x & 15) == 0 &&
                   ((uintptr_t)A.x_lo & 15) == 0 && ((uintptr_t)A.wb & 15) == 0 && cin % 8 == 0;
  void (*kern)(ConvArgs) = A.cout <= 32 ? (vec ? k_conv_bf16<32, true> : k_conv_bf16<32, false>)
                                       : (vec ? k_conv_bf16<64, true> : k_conv_bf16<64, false>);
  const dim3 grid(cdiv(npix, CM), A.cout <= 32 ? 1 : cdiv(A.cout, 64));
  SDB_LAUNCH(kern, grid, 256, 0, st, A);
  return 0;
}

// ------------------------------------------------------------------------------------------ weight gradient
// CTA tile 64 rows (tap, ci) x NT output channels (NT = 32 when cout <= 32, else 64), K steps of 32 pixels, double-buffered;
// 8 warps of 16 columns x (64 / warps along M) rows.  Both operands are staged as they lie in memory, pixel-major (sX[pixel]
// [row], sD[pixel][column]), and ldmatrix.trans turns them into the K-major fragments of mma.sync.  VEC (Cin and c_lo
// multiples of 8): each 8-row group is one 16-byte cp.async of 8 channels of one tap; DY_BF16 (a bf16 dy with ldy % 8 == 0):
// dy rows are 16-byte cp.asyncs too.  Otherwise element loads, an fp32 dy rounded on load.  Row taps*Cin (the bias) is left
// out of the GEMM and written from the fp32 sum of dy, read from global memory as stored.
constexpr int WB_M = 64, WB_K = 32, WB_LX = WB_M + 8;  // row pitch 144 bytes: the 8 rows of an ldmatrix hit distinct banks

template <int NT, bool VEC, bool DY_BF16>
__global__ void __launch_bounds__(256) k_conv_wgrad_bf16(sdb::WgradArgs A) {
  constexpr int WN = NT / 16, WM = 8 / WN, MT = WB_M / WM / 16;
  constexpr int LD = NT + 8;                         // 80 or 144 bytes: distinct banks for ldmatrix
  __shared__ __align__(16) bf16 sX[2][WB_K][WB_LX];
  __shared__ __align__(16) bf16 sD[2][WB_K][LD];
  __shared__ int sRow[WB_M][5];                      // dz, dy, dx, channel, kind (0 skip, 1 lo, 2 bias or none)
  const int Cin = A.c_skip + A.c_lo, brow = A.kz * A.ky * A.kx * Cin;
  const int n_ct = (A.cout + NT - 1) / NT;
  const int r0 = (blockIdx.x / n_ct) * WB_M, c0 = (blockIdx.x % n_ct) * NT;
  const int t = threadIdx.x, warp = t / 32, lane = t % 32;
  const int wm = (warp / WN) * (WB_M / WM), wn = (warp % WN) * 16;
  const bool has_bias = r0 <= brow && brow < r0 + WB_M;
  const bf16* xb = (const bf16*)A.x; const bf16* lb = (const bf16*)A.x_lo;
  if (t < WB_M) {
    const int r = r0 + t;
    int* q = sRow[t];
    if (r < brow) {
      const int tap = r / Cin, c = r % Cin;
      q[0] = tap / (A.ky * A.kx) - A.pz; q[1] = (tap / A.kx) % A.ky - A.py; q[2] = tap % A.kx - A.px;
      q[3] = c < A.c_lo ? c : c - A.c_lo; q[4] = c < A.c_lo ? 1 : 0;
    } else {
      q[0] = q[1] = q[2] = q[3] = 0; q[4] = 2;
    }
  }
  __syncthreads();
  const long long p_begin = (long long)blockIdx.y * A.per_split;
  const long long p_end = p_begin + A.per_split < A.npix ? p_begin + A.per_split : A.npix;
  const int Dl = A.d / A.uz, Hl = A.h / A.uy, Wl = A.w / A.ux;
  // each thread stages one pixel of every K step: VEC 8-row group t % 8 of pixel t / 8, else rows t / 32 + 8j of pixel t % 32
  const int kx_ = VEC ? t / 8 : t % 32;
  auto load = [&](long long p0, int buf) {
    const long long p = p0 + kx_;
    int img = -1, z = 0, y = 0, x = 0;
    if (p < p_end) {
      x = (int)(p % A.w); y = (int)((p / A.w) % A.h); z = (int)((p / ((long long)A.w * A.h)) % A.d);
      img = (int)(p / ((long long)A.w * A.h * A.d));
    }
    if (VEC) {
      const int* q = sRow[8 * (t % 8)];
      const int zz = z + q[0], yy = y + q[1], xx = x + q[2];
      const bool ok = img >= 0 && q[4] < 2 && zz >= 0 && zz < A.d && yy >= 0 && yy < A.h && xx >= 0 && xx < A.w;
      const bf16* src = xb;
      if (ok) src = q[4] == 1 ? lb + ((((size_t)img * Dl + zz / A.uz) * Hl + yy / A.uy) * Wl + xx / A.ux) * A.c_lo + q[3]
                              : xb + ((((size_t)img * A.d + zz) * A.h + yy) * A.w + xx) * A.c_skip + q[3];
      cp_async16(&sX[buf][kx_][8 * (t % 8)], src, ok);
    } else {
#pragma unroll
      for (int j = 0; j < WB_M / 8; ++j) {
        const int r = t / 32 + 8 * j;
        const int* q = sRow[r];
        const int zz = z + q[0], yy = y + q[1], xx = x + q[2];
        bf16 v = __float2bfloat16_rn(0.f);
        if (img >= 0 && q[4] < 2 && zz >= 0 && zz < A.d && yy >= 0 && yy < A.h && xx >= 0 && xx < A.w)
          v = q[4] == 1 ? lb[((((size_t)img * Dl + zz / A.uz) * Hl + yy / A.uy) * Wl + xx / A.ux) * A.c_lo + q[3]]
                        : xb[((((size_t)img * A.d + zz) * A.h + yy) * A.w + xx) * A.c_skip + q[3]];
        sX[buf][kx_][r] = v;
      }
    }
    if (DY_BF16) {
      const bf16* db = (const bf16*)A.dy;
      for (int e = t; e < WB_K * (NT / 8); e += 256) {
        const int k = e / (NT / 8), c = 8 * (e % (NT / 8));
        const long long pp = p0 + k;
        const bool ok = pp < p_end && c0 + c < A.cout;
        cp_async16(&sD[buf][k][c], ok ? db + pp * A.ldy + c0 + c : db, ok);
      }
    } else {
      for (int e = t; e < WB_K * NT; e += 256) {
        const int k = e / NT, c = e % NT;
        const long long pp = p0 + k;
        sD[buf][k][c] = __float2bfloat16_rn((pp < p_end && c0 + c < A.cout) ? A.dy[pp * A.ldy + c0 + c] : 0.f);
      }
    }
    cp_async_commit();
  };
  float acc[MT][2][4];
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.f;
  float bsum = 0.f;                                  // thread t < NT of the bias CTA: db partial of column c0 + t
  if (p_begin < p_end) load(p_begin, 0);
  for (long long p0 = p_begin, s = 0; p0 < p_end; p0 += WB_K, ++s) {
    const int buf = (int)(s & 1);
    if (p0 + WB_K < p_end) {
      load(p0 + WB_K, buf ^ 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (has_bias && t < NT && c0 + t < A.cout) {
      const long long pe = p0 + WB_K < p_end ? p0 + WB_K : p_end;
      for (long long pp = p0; pp < pe; ++pp)
        bsum += DY_BF16 ? __bfloat162float(((const bf16*)A.dy)[pp * A.ldy + c0 + t]) : A.dy[pp * A.ldy + c0 + t];
    }
#pragma unroll
    for (int kk = 0; kk < WB_K; kk += 16) {
      uint32_t a[MT][4], b[4];
      const int mi = lane / 8, lr = lane % 8;
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
        ldsm_x4_trans(a[mt], &sX[buf][kk + (mi >> 1) * 8 + lr][wm + mt * 16 + (mi & 1) * 8]);
      ldsm_x4_trans(b, &sD[buf][kk + (mi & 1) * 8 + lr][wn + (mi >> 1) * 8]);
      const uint32_t b0[2] = {b[0], b[1]}, b1[2] = {b[2], b[3]};
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        mma_bf16(acc[mt][0], a[mt], b0);
        mma_bf16(acc[mt][1], a[mt], b1);
      }
    }
    __syncthreads();
  }
  const int g = lane / 4, t4 = lane % 4;
  float* out = A.work + (size_t)blockIdx.y * A.rows * A.cout;
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = r0 + wm + mt * 16 + g + (i >= 2 ? 8 : 0), c = c0 + wn + nt * 8 + 2 * t4 + (i & 1);
        if (r < brow && c < A.cout) out[(size_t)r * A.cout + c] = acc[mt][nt][i];
      }
  if (has_bias && t < NT && c0 + t < A.cout) out[(size_t)brow * A.cout + c0 + t] = bsum;
}

template <int NT>
int wgrad_bf16_launch_nt(const sdb::WgradArgs& A, dim3 grid, bool vec, bool dyb, cudaStream_t st) {
  void (*kern)(sdb::WgradArgs) = vec ? (dyb ? k_conv_wgrad_bf16<NT, true, true> : k_conv_wgrad_bf16<NT, true, false>)
                                     : (dyb ? k_conv_wgrad_bf16<NT, false, true> : k_conv_wgrad_bf16<NT, false, false>);
  SDB_LAUNCH(kern, grid, 256, 0, st, A);
  return 0;
}

// ------------------------------------------------------------------------------------------ small kernels
__global__ void k_cast_bf16(const float* __restrict__ in, long long n, bf16* __restrict__ out) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x)
    out[e] = __float2bfloat16_rn(in[e]);
}

// w [tap][ci][co] fp32 -> bf16: flip = 0 out[(tap * cout + co) * ld + ci] (the forward kernel's [tap][cout][cin]); flip = 1
// out[((taps-1-tap) * cin + ci) * ld + co] (the input-gradient kernel of sdb_conv_flip_weights, in the same layout)
__global__ void k_weights_bf16(const float* __restrict__ w, int taps, int cin, int cout, int flip, int ld, bf16* __restrict__ out) {
  const long long total = (long long)taps * cin * cout;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(e % cout); const long long r = e / cout;
    const int ci = (int)(r % cin), tap = (int)(r / cin);
    const size_t o = flip ? ((size_t)(taps - 1 - tap) * cin + ci) * ld + co : ((size_t)tap * cout + co) * ld + ci;
    out[o] = __float2bfloat16_rn(w[e]);
  }
}

__global__ void k_maxpool_bf16(const bf16* __restrict__ in, int N, int D, int H, int W, int C, int pz, int py, int px,
                               bf16* __restrict__ out) {
  const int Do = D / pz, Ho = H / py, Wo = W / px;
  const long long total = (long long)N * Do * Ho * Wo * C;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(e % C); long long r = e / C;
    const int xo = (int)(r % Wo); r /= Wo;
    const int yo = (int)(r % Ho); r /= Ho;
    const int zo = (int)(r % Do); const long long img = r / Do;
    bf16 m = in[((((img * D + zo * pz) * H + yo * py) * W) + xo * px) * (size_t)C + c];
    for (int a = 0; a < pz; ++a) for (int b = 0; b < py; ++b) for (int q = 0; q < px; ++q) {
      const bf16 v = in[((((img * D + zo * pz + a) * H + yo * py + b) * W) + xo * px + q) * (size_t)C + c];
      if (__bfloat162float(v) > __bfloat162float(m)) m = v;
    }
    out[e] = m;
  }
}

// softmax over the C <= 32 logits of each pixel, in sdb_class_head's order of operations
__global__ void k_softmax_rows(const float* __restrict__ z, long long npix, int C, float* __restrict__ out) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npix) return;
  float acc[32];
  for (int o = 0; o < C; ++o) acc[o] = z[p * C + o];
  float m = acc[0];
  for (int o = 1; o < C; ++o) m = fmaxf(m, acc[o]);
  float sum = 0.f;
  for (int o = 0; o < C; ++o) { acc[o] = expf(acc[o] - m); sum += acc[o]; }
  for (int o = 0; o < C; ++o) out[p * C + o] = acc[o] / sum;
}

__global__ void k_add_bf16(const bf16* __restrict__ a, const bf16* __restrict__ b, long long n, bf16* __restrict__ out) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x)
    out[e] = __float2bfloat16_rn(__bfloat162float(a[e]) + __bfloat162float(b[e]));
}

}  // namespace

namespace sdb {

int conv_wgrad_bf16_launch(const WgradArgs& A, int nsplit, cudaStream_t st) {
  const int Cin = A.c_skip + A.c_lo;
  const bool vec = A.c_skip % 8 == 0 && A.c_lo % 8 == 0 && Cin % 8 == 0 && ((uintptr_t)A.x & 15) == 0 && ((uintptr_t)A.x_lo & 15) == 0;
  const bool dyb = A.prec == WGRAD_BF16_DY_BF16 && A.ldy % 8 == 0 && A.cout % 8 == 0 && ((uintptr_t)A.dy & 15) == 0;
  if (A.prec == WGRAD_BF16_DY_BF16 && !dyb) { set_error("conv_wgrad_bf16_nd: a bf16 dy needs ldy and cout multiples of 8, 16-byte aligned"); return 1; }
  if (A.cout <= 32) return wgrad_bf16_launch_nt<32>(A, dim3(cdiv(A.rows, WB_M) * cdiv(A.cout, 32), nsplit), vec, dyb, st);
  return wgrad_bf16_launch_nt<64>(A, dim3(cdiv(A.rows, WB_M) * cdiv(A.cout, 64), nsplit), vec, dyb, st);
}

}  // namespace sdb

// ------------------------------------------------------------------------------------------ entry points
static bool bad_kernel(int kz, int ky, int kx) {
  return !((kz == 1 || kz == 3) && (ky == 1 || ky == 3) && (kx == 1 || kx == 3));
}

extern "C" int sdb_conv_bf16_nd(const void* d_x, const void* d_x_lo, int n, int d, int h, int w, int cin_skip, int cin_lo, int uz, int uy,
                                int ux, int kz, int ky, int kx, const void* d_wb, const float* d_b, int cout, int relu, int accumulate,
                                void* d_out, sdb_stream_t stream) {
  if (n < 1 || d < 1 || h < 1 || w < 1 || cout < 1 || cin_skip < 1 || cin_lo < 0 || bad_kernel(kz, ky, kx)) {
    sdb::set_error("conv_bf16_nd: bad arguments (kernel extents 1 or 3 per axis)"); return 1;
  }
  if (cin_lo && (d_x_lo == nullptr || uz < 1 || uy < 1 || ux < 1 || d % uz || h % uy || w % ux)) {
    sdb::set_error("conv_bf16_nd: low-resolution source needs a pointer and divisible up-sampling factors"); return 1;
  }
  ConvArgs A{};
  A.x = d_x; A.x_lo = cin_lo ? d_x_lo : nullptr; A.a_f32 = 0;
  A.n = n; A.d = d; A.h = h; A.w = w; A.c_skip = cin_skip; A.c_lo = cin_lo;
  A.uz = cin_lo ? uz : 1; A.uy = cin_lo ? uy : 1; A.ux = cin_lo ? ux : 1; A.kz = kz; A.ky = ky; A.kx = kx;
  A.wb = (const bf16*)d_wb; A.bias = d_b; A.cout = cout; A.relu = relu; A.mode = EPI_BF16; A.accumulate = accumulate; A.out = d_out;
  return conv_bf16_launch(A, (cudaStream_t)stream);
}

extern "C" int sdb_gemm_bf16_f32in(const float* d_a, long long npix, int k, const void* d_wb, int nout, int accumulate, void* d_out,
                                   sdb_stream_t stream) {
  if (npix < 1 || k < 1 || nout < 1 || npix > 0x7fffffffLL) { sdb::set_error("gemm_bf16_f32in: bad arguments"); return 1; }
  ConvArgs A{};
  A.x = d_a; A.a_f32 = 1;
  A.n = 1; A.d = 1; A.h = 1; A.w = (int)npix; A.c_skip = k; A.c_lo = 0; A.uz = A.uy = A.ux = 1; A.kz = A.ky = A.kx = 1;
  A.wb = (const bf16*)d_wb; A.cout = nout; A.mode = EPI_BF16; A.accumulate = accumulate; A.out = d_out;
  return conv_bf16_launch(A, (cudaStream_t)stream);
}

extern "C" int sdb_heads_bf16(const void* d_feat, long long npix, int cfeat, const void* d_wb, const float* d_bp, const float* d_bd,
                              int n_rays, float* d_prob, float* d_dist, sdb_stream_t stream) {
  if (npix < 1 || cfeat < 1 || n_rays < 1 || npix > 0x7fffffffLL) { sdb::set_error("heads_bf16: bad arguments"); return 1; }
  ConvArgs A{};
  A.x = d_feat; A.n = 1; A.d = 1; A.h = 1; A.w = (int)npix; A.c_skip = cfeat; A.uz = A.uy = A.ux = 1; A.kz = A.ky = A.kx = 1;
  A.wb = (const bf16*)d_wb; A.bias = d_bp; A.bias2 = d_bd; A.cout = n_rays + 1; A.mode = EPI_HEADS; A.R = n_rays;
  A.out = d_dist; A.prob = d_prob;
  return conv_bf16_launch(A, (cudaStream_t)stream);
}

extern "C" int sdb_class_head_bf16(const void* d_feat, long long npix, int cfeat, const void* d_wb, const float* d_b, int n_out,
                                   float* d_logits, float* d_out, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (npix < 1 || cfeat < 1 || n_out < 1 || n_out > 32 || npix > 0x7fffffffLL) { sdb::set_error("class_head_bf16: n_classes + 1 must be in [1,32]"); return 1; }
  ConvArgs A{};
  A.x = d_feat; A.n = 1; A.d = 1; A.h = 1; A.w = (int)npix; A.c_skip = cfeat; A.uz = A.uy = A.ux = 1; A.kz = A.ky = A.kx = 1;
  A.wb = (const bf16*)d_wb; A.bias = d_b; A.cout = n_out; A.mode = EPI_F32; A.out = d_logits;
  if (conv_bf16_launch(A, st)) return 1;
  SDB_LAUNCH(k_softmax_rows, cdiv(npix, 128), 128, 0, st, d_logits, npix, n_out, d_out);
  return 0;
}

extern "C" int sdb_cast_bf16(const float* d_in, long long n, void* d_out, sdb_stream_t stream) {
  if (n <= 0) return 0;
  SDB_LAUNCH(k_cast_bf16, grid_1d(n, 16), 256, 0, (cudaStream_t)stream, d_in, n, (bf16*)d_out);
  return 0;
}

extern "C" int sdb_weights_bf16(const float* d_w, int taps, int cin, int cout, int flip, int ld, void* d_out, sdb_stream_t stream) {
  if (taps < 1 || cin < 1 || cout < 1 || ld < (flip ? cout : cin)) { sdb::set_error("weights_bf16: bad arguments"); return 1; }
  SDB_LAUNCH(k_weights_bf16, grid_1d((long long)taps * cin * cout, 16), 256, 0, (cudaStream_t)stream, d_w, taps, cin, cout, flip, ld,
             (bf16*)d_out);
  return 0;
}

extern "C" int sdb_maxpool_bf16_nd(const void* d_in, int n, int d, int h, int w, int c, int pz, int py, int px, void* d_out,
                                   sdb_stream_t stream) {
  if (pz < 1 || py < 1 || px < 1 || c < 1) { sdb::set_error("maxpool_bf16_nd: bad arguments"); return 1; }
  const long long total = (long long)n * (d / pz) * (h / py) * (w / px) * c;
  if (total <= 0) return 0;
  SDB_LAUNCH(k_maxpool_bf16, grid_1d(total, 32), 256, 0, (cudaStream_t)stream, (const bf16*)d_in, n, d, h, w, c, pz, py, px, (bf16*)d_out);
  return 0;
}

extern "C" int sdb_maxpool_backward_bf16_nd(const void* d_x, const void* d_gy, int n, int d, int h, int w, int c, int pz, int py, int px,
                                            int accumulate, void* d_gx, sdb_stream_t stream) {
  if (pz < 1 || py < 1 || px < 1 || d % pz || h % py || w % px || c < 1) { sdb::set_error("maxpool_backward_bf16_nd: sizes must be divisible by the pool"); return 1; }
  const long long total = (long long)n * (d / pz) * (h / py) * (w / px) * c;
  SDB_LAUNCH(sdb::k_maxpool_backward<bf16>, grid_1d(total, 32), 256, 0, (cudaStream_t)stream, (const bf16*)d_x, (const bf16*)d_gy,
             n, d, h, w, c, pz, py, px, accumulate, (bf16*)d_gx);
  return 0;
}

extern "C" int sdb_relu_backward_bf16(void* d_g, const void* d_y, long long n, sdb_stream_t stream) {
  if (n <= 0) return 0;
  SDB_LAUNCH(sdb::k_relu_backward<bf16>, grid_1d(n, 32), 256, 0, (cudaStream_t)stream, (bf16*)d_g, (const bf16*)d_y, n);
  return 0;
}

extern "C" int sdb_decoder_split_bf16(const void* d_dcat, int n, int d, int h, int w, int c_lo, int c_skip, int uz, int uy, int ux,
                                      void* d_dlo, void* d_dskip, sdb_stream_t stream) {
  if (c_lo < 1 || c_skip < 1 || uz < 1 || uy < 1 || ux < 1 || d % uz || h % uy || w % ux) { sdb::set_error("decoder_split_bf16: bad arguments"); return 1; }
  const long long total = (long long)n * d * h * w / ((long long)uz * uy * ux) * c_lo + (long long)n * d * h * w * c_skip;
  SDB_LAUNCH(sdb::k_decoder_split<bf16>, grid_1d(total, 32), 256, 0, (cudaStream_t)stream, (const bf16*)d_dcat, n, d, h, w, c_lo, c_skip,
             uz, uy, ux, (bf16*)d_dlo, (bf16*)d_dskip);
  return 0;
}

extern "C" int sdb_add_bf16(const void* d_a, const void* d_b, long long n, void* d_out, sdb_stream_t stream) {
  if (n <= 0) return 0;
  SDB_LAUNCH(k_add_bf16, grid_1d(n, 32), 256, 0, (cudaStream_t)stream, (const bf16*)d_a, (const bf16*)d_b, n, (bf16*)d_out);
  return 0;
}
