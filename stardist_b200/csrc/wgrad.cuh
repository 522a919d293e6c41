// wgrad.cuh -- the weight-gradient GEMM's arguments, shared by the fp32 kernel (unet_train.cu), the TF32 tensor-core kernel
// (unet_train_tf32.cu) and the bf16 tensor-core kernel (unet_train_bf16.cu).  Both write per-split partials work[split][row][co] with the split count and workspace layout of
// sdb_conv_wgrad_workspace; unet_train.cu sums the slots in index order with one reduction kernel for both.
#pragma once
#include <cuda_runtime.h>

namespace sdb {

enum { WGRAD_FP32 = 0, WGRAD_TF32 = 1, WGRAD_BF16_DY_F32 = 2, WGRAD_BF16_DY_BF16 = 3 };

struct WgradArgs {
  // float data, except under WGRAD_BF16_*: x and x_lo then hold __nv_bfloat16, and dy too under WGRAD_BF16_DY_BF16
  const float* x; const float* x_lo; const float* dy;
  int prec;
  int n, d, h, w, c_skip, c_lo, uz, uy, ux, kz, ky, kx, pz, py, px, ldy, cout;
  int rows;                 // taps * Cin + 1
  long long npix, per_split;
  float* work;
};

// launches the TF32 partial-sum kernel over nsplit pixel ranges of A.per_split pixels (unet_train_tf32.cu)
int conv_wgrad_tf32_launch(const WgradArgs& A, int nsplit, cudaStream_t st);
// the same for the bf16 partial-sum kernel (unet_train_bf16.cu)
int conv_wgrad_bf16_launch(const WgradArgs& A, int nsplit, cudaStream_t st);

}  // namespace sdb
