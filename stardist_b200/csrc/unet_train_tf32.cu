// unet_train_tf32.cu -- the TF32 tensor-core weight and input gradients of the U-Net training step, the precision mode
// behind stardist_b200.enable_tensor_float_32_execution (DESIGN.md 4.2).  Both are GEMMs on mma.sync.m16n8k8 with TF32
// operands and fp32 accumulators; every operand is rounded with cvt.rna.tf32.f32 (10 explicit mantissa bits, nearest, ties
// away from zero) before it enters a fragment:
//   weight gradient  dW[tap, ci, co] = sum_p rna(x[p + tap - pad, ci]) * rna(dy[p, co]), rows (tap, ci), columns co, K = the
//                    batch's pixels; db = sum_p dy[p, co] is summed unrounded in fp32, in pixel order, beside the GEMM.  The
//                    pixel splits, the workspace and the reduction are those of sdb_conv_wgrad_nd (unet_train.cu).
//   input gradient   gin[p, ci] = sum_(tap, co) rna(dy[p + tap - 1, co]) * rna(wf[tap, co, ci]), the stride-1 'same'
//                    correlation of dy with the flipped kernel of sdb_conv_flip_weights: rows p, columns ci, K = (tap, co).
// No float atomics: each output element is accumulated by one thread in a fixed order, so results are bit-identical run to run.
#include <stdint.h>
#include "common.cuh"
#include "wgrad.cuh"
#include "../../include/stardist_b200.h"

namespace {

using sdb::cdiv;

__device__ __forceinline__ uint32_t rna_tf32(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return r;
}

// c += a * b: a 16x8 (row-major), b 8x8 (column-major), c 16x8 fp32
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// ------------------------------------------------------------------------------------------ weight gradient
// CTA tile 64 rows x NT output channels (NT = 32 when cout <= 32, else 64), 32 pixels per K step, 8 warps of 16 columns x
// (64 / warps along M) rows.  Rows as in the fp32 kernel: (tap, ci) = (r / Cin, r % Cin), the decoder input read through the
// up-sampling address math; row taps*Cin (the bias) is left out of the GEMM and written from the fp32 sum of dy instead.
constexpr int TW_M = 64, TW_K = 32;

template <int NT>
__global__ void __launch_bounds__(256) k_conv_wgrad_tf32(sdb::WgradArgs A) {
  constexpr int WN = NT / 16, WM = 8 / WN, MT = TW_M / WM / 16;
  constexpr int LX = TW_M + 8, LD = NT + 8;          // row pitches: the fragment loads hit 32 distinct banks
  __shared__ __align__(16) uint32_t sX[TW_K][LX];    // rna(x) [pixel][row]
  __shared__ __align__(16) float sD[TW_K][LD];       // dy [pixel][column], unrounded (the bias sums it)
  __shared__ int sRow[TW_M][5];                      // dz, dy, dx, channel, kind (0 skip, 1 lo, 2 bias or none)
  __shared__ int sPix[TW_K][4];                      // img, z, y, x (img < 0: past the end)
  const int Cin = A.c_skip + A.c_lo, brow = A.kz * A.ky * A.kx * Cin;
  const int n_ct = (A.cout + NT - 1) / NT;
  const int r0 = (blockIdx.x / n_ct) * TW_M, c0 = (blockIdx.x % n_ct) * NT;
  const int t = threadIdx.x, warp = t / 32, lane = t % 32, g = lane / 4, t4 = lane % 4;
  const int wm = (warp / WN) * (TW_M / WM), wn = (warp % WN) * 16;
  const bool has_bias = r0 <= brow && brow < r0 + TW_M;
  if (t < TW_M) {
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
  const long long p_begin = (long long)blockIdx.y * A.per_split;
  const long long p_end = p_begin + A.per_split < A.npix ? p_begin + A.per_split : A.npix;
  const int Dl = A.d / A.uz, Hl = A.h / A.uy, Wl = A.w / A.ux;
  float acc[MT][2][4];
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.f;
  float bsum = 0.f;                                  // thread t < NT of the bias CTA: db partial of column c0 + t
  for (long long p0 = p_begin; p0 < p_end; p0 += TW_K) {
    __syncthreads();
    if (t < TW_K) {
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
    for (int e = t; e < TW_K * TW_M; e += 256) {
      const int k = e / TW_M, r = e % TW_M;
      const int* pp = sPix[k]; const int* q = sRow[r];
      float v = 0.f;
      if (pp[0] >= 0 && q[4] < 2) {
        const int zz = pp[1] + q[0], yy = pp[2] + q[1], xx = pp[3] + q[2];
        if (zz >= 0 && zz < A.d && yy >= 0 && yy < A.h && xx >= 0 && xx < A.w) {
          if (q[4] == 1) v = A.x_lo[((((size_t)pp[0] * Dl + zz / A.uz) * Hl + yy / A.uy) * Wl + xx / A.ux) * A.c_lo + q[3]];
          else v = A.x[((((size_t)pp[0] * A.d + zz) * A.h + yy) * A.w + xx) * A.c_skip + q[3]];
        }
      }
      sX[k][r] = rna_tf32(v);
    }
    for (int e = t; e < TW_K * NT; e += 256) {
      const int k = e / NT, c = e % NT;
      const long long p = p0 + k;
      sD[k][c] = (p < p_end && c0 + c < A.cout) ? A.dy[p * A.ldy + c0 + c] : 0.f;
    }
    __syncthreads();
    if (has_bias && t < NT) {
#pragma unroll 8
      for (int k = 0; k < TW_K; ++k) bsum += sD[k][t];
    }
#pragma unroll
    for (int kk = 0; kk < TW_K; kk += 8) {
      uint32_t a[MT][4], b[2][2];
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        const int m = wm + mt * 16 + g;
        a[mt][0] = sX[kk + t4][m]; a[mt][1] = sX[kk + t4][m + 8];
        a[mt][2] = sX[kk + t4 + 4][m]; a[mt][3] = sX[kk + t4 + 4][m + 8];
      }
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        const int c = wn + nt * 8 + g;
        b[nt][0] = rna_tf32(sD[kk + t4][c]); b[nt][1] = rna_tf32(sD[kk + t4 + 4][c]);
      }
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) mma_tf32(acc[mt][nt], a[mt], b[nt]);
    }
  }
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

// ------------------------------------------------------------------------------------------ input gradient
// CTA tile 128 consecutive output pixels x NT input channels (NT = 64 when cin % 64 == 0, else 32), K steps of 32 output
// channels of one tap; 8 warps of 32 columns x (128 / warps along M) rows.  vec = 1: dy rows are read as float4 (cout % 4 == 0
// and a 16-byte aligned dy).
constexpr int TD_M = 128, TD_K = 32;

template <int NT>
__global__ void __launch_bounds__(256) k_conv_dgrad_tf32(const float* __restrict__ dy, int n, int d, int h, int w, int cout,
                                                         const float* __restrict__ wf, int cin, int kz, int vec,
                                                         float* __restrict__ gin) {
  constexpr int WN = NT / 32, WM = 8 / WN, MT = TD_M / WM / 16;
  constexpr int LA = TD_K + 4, LB = NT + 8;          // row pitches: the fragment loads hit 32 distinct banks
  __shared__ __align__(16) uint32_t sA[TD_M][LA];    // rna(dy) [pixel][co]
  __shared__ __align__(16) uint32_t sB[TD_K][LB];    // rna(wf) [co][ci]
  __shared__ int sPix[TD_M][4];                      // img, z, y, x (img < 0: past the end)
  const long long npix = (long long)n * d * h * w;
  const long long p0 = (long long)blockIdx.x * TD_M;
  const int ci0 = blockIdx.y * NT;
  const int t = threadIdx.x, warp = t / 32, lane = t % 32, g = lane / 4, t4 = lane % 4;
  const int wm = (warp / WN) * (TD_M / WM), wn = (warp % WN) * 32;
  if (t < TD_M) {
    const long long p = p0 + t;
    int* q = sPix[t];
    if (p < npix) {
      q[3] = (int)(p % w); q[2] = (int)((p / w) % h); q[1] = (int)((p / ((long long)w * h)) % d); q[0] = (int)(p / ((long long)w * h * d));
    } else {
      q[0] = -1; q[1] = q[2] = q[3] = 0;
    }
  }
  float acc[MT][4][4];
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.f;
  const int taps = kz * 9, pz = (kz - 1) / 2;
  for (int tap = 0; tap < taps; ++tap) {
    const int oz = tap / 9 - pz, oy = (tap / 3) % 3 - 1, ox = tap % 3 - 1;
    for (int co0 = 0; co0 < cout; co0 += TD_K) {
      __syncthreads();
      if (vec) {
        for (int e = t; e < TD_M * (TD_K / 4); e += 256) {
          const int m = e / (TD_K / 4), k = 4 * (e % (TD_K / 4));
          const int* pp = sPix[m];
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          const int zz = pp[1] + oz, yy = pp[2] + oy, xx = pp[3] + ox;
          if (pp[0] >= 0 && co0 + k < cout && zz >= 0 && zz < d && yy >= 0 && yy < h && xx >= 0 && xx < w)
            v = *reinterpret_cast<const float4*>(dy + ((((size_t)pp[0] * d + zz) * h + yy) * w + xx) * cout + co0 + k);
          *reinterpret_cast<uint4*>(&sA[m][k]) = make_uint4(rna_tf32(v.x), rna_tf32(v.y), rna_tf32(v.z), rna_tf32(v.w));
        }
      } else {
        for (int e = t; e < TD_M * TD_K; e += 256) {
          const int m = e / TD_K, k = e % TD_K;
          const int* pp = sPix[m];
          float v = 0.f;
          const int zz = pp[1] + oz, yy = pp[2] + oy, xx = pp[3] + ox;
          if (pp[0] >= 0 && co0 + k < cout && zz >= 0 && zz < d && yy >= 0 && yy < h && xx >= 0 && xx < w)
            v = dy[((((size_t)pp[0] * d + zz) * h + yy) * w + xx) * cout + co0 + k];
          sA[m][k] = rna_tf32(v);
        }
      }
      for (int e = t; e < TD_K * NT; e += 256) {
        const int k = e / NT, c = e % NT;
        const int co = co0 + k, ci = ci0 + c;
        sB[k][c] = (co < cout && ci < cin) ? rna_tf32(wf[((size_t)tap * cout + co) * cin + ci]) : 0u;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < TD_K; kk += 8) {
        if (co0 + kk >= cout) break;                 // the rest of the step is zero padding
        uint32_t a[MT][4], b[4][2];
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          const int m = wm + mt * 16 + g;
          a[mt][0] = sA[m][kk + t4]; a[mt][1] = sA[m + 8][kk + t4];
          a[mt][2] = sA[m][kk + t4 + 4]; a[mt][3] = sA[m + 8][kk + t4 + 4];
        }
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
          const int c = wn + nt * 8 + g;
          b[nt][0] = sB[kk + t4][c]; b[nt][1] = sB[kk + t4 + 4][c];
        }
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
          for (int nt = 0; nt < 4; ++nt) mma_tf32(acc[mt][nt], a[mt], b[nt]);
      }
    }
  }
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const long long p = p0 + wm + mt * 16 + g + (i >= 2 ? 8 : 0);
        const int c = ci0 + wn + nt * 8 + 2 * t4 + (i & 1);
        if (p < npix && c < cin) gin[p * cin + c] = acc[mt][nt][i];
      }
}

}  // namespace

namespace sdb {

int conv_wgrad_tf32_launch(const WgradArgs& A, int nsplit, cudaStream_t st) {
  if (A.cout <= 32) {
    dim3 grid(cdiv(A.rows, TW_M) * cdiv(A.cout, 32), nsplit);
    SDB_LAUNCH(k_conv_wgrad_tf32<32>, grid, 256, 0, st, A);
  } else {
    dim3 grid(cdiv(A.rows, TW_M) * cdiv(A.cout, 64), nsplit);
    SDB_LAUNCH(k_conv_wgrad_tf32<64>, grid, 256, 0, st, A);
  }
  return 0;
}

}  // namespace sdb

extern "C" int sdb_conv_dgrad_tf32_nd(const float* d_dy, int n, int d, int h, int w, int cout, const float* d_wf, int cin, int kz,
                                      int kyx, float* d_gin, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n < 1 || d < 1 || h < 1 || w < 1 || kyx != 3 || (kz != 1 && kz != 3) || (kz == 1 && d != 1)) {
    sdb::set_error("conv_dgrad_tf32_nd: a 3^d kernel (kz = 1 with d = 1 in 2-D, kz = 3 in 3-D) is required"); return 1;
  }
  // the layers whose input gradient sdb_conv3_nd takes (conv_dgrad3_accepts): its stem variant and its tiled variant
  if (!((cout >= 1 && cout <= 4 && (cin == 32 || cin == 64)) || (cout >= 8 && cout % 8 == 0 && cin >= 32 && cin % 32 == 0))) {
    sdb::set_error("conv_dgrad_tf32_nd: cout <= 4 with cin 32 or 64, or cout % 8 == 0 with cin % 32 == 0, is required"); return 1;
  }
  const long long npix = (long long)n * d * h * w;
  const int vec = (cout % 4 == 0 && ((uintptr_t)d_dy & 15) == 0) ? 1 : 0;
  if (cin % 64 == 0) {
    SDB_LAUNCH(k_conv_dgrad_tf32<64>, dim3(cdiv(npix, TD_M), cin / 64), 256, 0, st, d_dy, n, d, h, w, cout, d_wf, cin, kz, vec, d_gin);
  } else {
    SDB_LAUNCH(k_conv_dgrad_tf32<32>, dim3(cdiv(npix, TD_M), cin / 32), 256, 0, st, d_dy, n, d, h, w, cout, d_wf, cin, kz, vec, d_gin);
  }
  return 0;
}
