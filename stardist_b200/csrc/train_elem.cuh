// train_elem.cuh -- elementwise kernels of the U-Net backward pass, templated on the storage type T of activations and
// gradients: float for the fp32 trainer (unet_train.cu), __nv_bfloat16 for the mixed_bfloat16 policy (unet_train_bf16.cu).
// Values are loaded to fp32, combined in fp32 and rounded to T once per stored element (round to nearest even for bf16);
// the float instantiations are the fp32 trainer's kernels.
#pragma once
#include <math.h>
#include <cuda_bf16.h>

namespace sdb {

__device__ __forceinline__ float ldf(float v) { return v; }
__device__ __forceinline__ float ldf(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T stf(float v);
template <> __device__ __forceinline__ float stf<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 stf<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// d[up(x_lo), skip] -> d x_lo (sum over each uz*uy*ux block, row-major) and d skip (the remaining channels)
template <typename T>
__global__ void k_decoder_split(const T* __restrict__ dcat, int n, int d, int h, int w, int c_lo, int c_skip, int uz, int uy,
                                int ux, T* __restrict__ dlo, T* __restrict__ dskip) {
  const int Dl = d / uz, Hl = h / uy, Wl = w / ux, C = c_lo + c_skip;
  const long long n_lo = (long long)n * Dl * Hl * Wl * c_lo, n_sk = (long long)n * d * h * w * c_skip;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n_lo + n_sk; e += (long long)gridDim.x * blockDim.x) {
    if (e < n_lo) {
      const int c = (int)(e % c_lo); long long r = e / c_lo;
      const int xl = (int)(r % Wl); r /= Wl;
      const int yl = (int)(r % Hl); r /= Hl;
      const int zl = (int)(r % Dl); const long long img = r / Dl;
      float s = 0.f;
      for (int a = 0; a < uz; ++a) for (int b = 0; b < uy; ++b) for (int q = 0; q < ux; ++q)
        s += ldf(dcat[((((size_t)img * d + zl * uz + a) * h + yl * uy + b) * w + xl * ux + q) * C + c]);
      dlo[e] = stf<T>(s);
    } else {
      const long long f = e - n_lo;
      const int c = (int)(f % c_skip); const long long p = f / c_skip;
      dskip[f] = dcat[(size_t)p * C + c_lo + c];
    }
  }
}

template <typename T>
__global__ void k_relu_backward(T* __restrict__ g, const T* __restrict__ y, long long n) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x)
    if (!(ldf(y[e]) > 0.f)) g[e] = stf<T>(0.f);
}

// Max-pool backward: the window's gradient goes to its FIRST maximum in row-major order (TF's and torch's tie rule); the
// other window positions receive 0.  Ties are common at 0 after a ReLU; they are harmless, because the ReLU backward of
// the pooled tensor's producer zeroes the gradient at every position whose value is 0, whichever one got it.
// accumulate = 1 adds to dx (a skip tensor whose decoder gradient is already there); windows do not overlap.
template <typename T>
__global__ void k_maxpool_backward(const T* __restrict__ x, const T* __restrict__ gy, int N, int D, int H, int W, int C,
                                   int pz, int py, int px, int accumulate, T* __restrict__ gx) {
  const int Do = D / pz, Ho = H / py, Wo = W / px;
  const long long total = (long long)N * Do * Ho * Wo * C;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(e % C); long long r = e / C;
    const int xo = (int)(r % Wo); r /= Wo;
    const int yo = (int)(r % Ho); r /= Ho;
    const int zo = (int)(r % Do); const long long img = r / Do;
    float m = -INFINITY; int best = 0, k = 0;
    for (int a = 0; a < pz; ++a) for (int b = 0; b < py; ++b) for (int q = 0; q < px; ++q, ++k) {
      const float v = ldf(x[((((size_t)img * D + zo * pz + a) * H + yo * py + b) * W + xo * px + q) * C + c]);
      if (v > m) { m = v; best = k; }
    }
    const float g = ldf(gy[e]);
    k = 0;
    for (int a = 0; a < pz; ++a) for (int b = 0; b < py; ++b) for (int q = 0; q < px; ++q, ++k) {
      const size_t i = ((((size_t)img * D + zo * pz + a) * H + yo * py + b) * W + xo * px + q) * C + c;
      const float v = (k == best) ? g : 0.f;
      gx[i] = accumulate ? stf<T>(ldf(gx[i]) + v) : stf<T>(v);
    }
  }
}

}  // namespace sdb
