// bitonic.cuh -- ascending bitonic sort of unique 64-bit keys in device memory (candidates.cu, overlap.cu).
//
// The keys buffer holds n_pad = a power of two >= BTILE entries; entries n..n_pad-1 are padded with ~0 so they
// sort to the end.  Keys are unique in both users, so the result is fully deterministic.
#pragma once
#include "common.cuh"

namespace sdb {
namespace bitonic {
namespace {            // internal linkage: every translation unit that sorts gets its own kernels

typedef unsigned long long u64;

constexpr int BT = 1024;            // threads per block
constexpr int BTILE = 4 * BT;       // elements per block-local tile (32 KB of smem): 4096 -> 21 global steps for 2^18 keys
constexpr int BPAIRS = BTILE / (2 * BT);   // compare-exchange pairs per thread and step

__global__ void k_pad_keys(u64* keys, unsigned int n, unsigned int n_pad) {
  unsigned int i = blockIdx.x * blockDim.x + threadIdx.x + n;
  if (i < n_pad) keys[i] = ~0ull;
}

__device__ __forceinline__ void cmpx(u64& a, u64& b, bool up) {
  if ((a > b) == up) { u64 t = a; a = b; b = t; }
}

// sort each BTILE tile completely (all stages k <= BTILE)
__global__ void __launch_bounds__(BT) k_bitonic_local_sort(u64* __restrict__ keys) {
  __shared__ u64 sh[BTILE];
  const unsigned int base = blockIdx.x * BTILE;
  for (int e = threadIdx.x; e < BTILE; e += BT) sh[e] = keys[base + e];
  __syncthreads();
  for (unsigned int k = 2; k <= BTILE; k <<= 1) {
    for (unsigned int j = k >> 1; j > 0; j >>= 1) {
#pragma unroll
      for (int q = 0; q < BPAIRS; ++q) {
        const unsigned int t = threadIdx.x + q * BT;
        const unsigned int i = 2 * t - (t & (j - 1));       // lower index of the pair
        const bool up = (((base + i) & k) == 0);
        cmpx(sh[i], sh[i + j], up);
      }
      __syncthreads();
    }
  }
  for (int e = threadIdx.x; e < BTILE; e += BT) keys[base + e] = sh[e];
}
// one global compare-exchange step (j >= BTILE)
__global__ void k_bitonic_global_step(u64* __restrict__ keys, unsigned int k, unsigned int j, unsigned int n_half) {
  const unsigned int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_half) return;
  const unsigned int i = 2 * t - (t & (j - 1));
  const bool up = ((i & k) == 0);
  u64 a = keys[i], b = keys[i + j];
  if ((a > b) == up) { keys[i] = b; keys[i + j] = a; }
}
// finish stage k inside tiles: steps j = BTILE/2 .. 1
__global__ void __launch_bounds__(BT) k_bitonic_local_merge(u64* __restrict__ keys, unsigned int k) {
  __shared__ u64 sh[BTILE];
  const unsigned int base = blockIdx.x * BTILE;
  for (int e = threadIdx.x; e < BTILE; e += BT) sh[e] = keys[base + e];
  __syncthreads();
  for (unsigned int j = BTILE >> 1; j > 0; j >>= 1) {
#pragma unroll
    for (int q = 0; q < BPAIRS; ++q) {
      const unsigned int t = threadIdx.x + q * BT;
      const unsigned int i = 2 * t - (t & (j - 1));
      const bool up = (((base + i) & k) == 0);
      cmpx(sh[i], sh[i + j], up);
    }
    __syncthreads();
  }
  for (int e = threadIdx.x; e < BTILE; e += BT) keys[base + e] = sh[e];
}

// smallest admissible buffer length for n keys
inline unsigned int padded_length(unsigned int n) {
  unsigned int n_pad = BTILE; while (n_pad < n) n_pad <<= 1;
  return n_pad;
}

// pad keys[n..n_pad) and sort keys[0..n_pad) ascending; n_pad = padded_length(n)
inline int sort(u64* keys, unsigned int n, unsigned int n_pad, cudaStream_t st) {
  if (n_pad > n) SDB_LAUNCH(k_pad_keys, cdiv(n_pad - n, 256), 256, 0, st, keys, n, n_pad);
  SDB_LAUNCH(k_bitonic_local_sort, n_pad / BTILE, BT, 0, st, keys);
  for (unsigned int k = 2 * BTILE; k <= n_pad; k <<= 1) {
    for (unsigned int j = k >> 1; j >= (unsigned int)BTILE; j >>= 1)
      SDB_LAUNCH(k_bitonic_global_step, cdiv(n_pad / 2, 256), 256, 0, st, keys, k, j, n_pad / 2);
    SDB_LAUNCH(k_bitonic_local_merge, n_pad / BTILE, BT, 0, st, keys, k);
  }
  return 0;
}

}  // namespace
}  // namespace bitonic
}  // namespace sdb
