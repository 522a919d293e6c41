// scan.cuh -- the one-block row-prefix scan shared by the training-batch sampler (traindata.cu) and the mask compaction of
// sample_points / get_valid_inds (helpers.cu).
#pragma once
#include <cuda_runtime.h>

namespace {

// in-place inclusive scan of pre[1 .. rows] by one block; pre[0] = 0
constexpr int SCAN_THREADS = 1024;
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_rows(long long* __restrict__ pre, long long rows) {
  __shared__ long long part[SCAN_THREADS];
  const long long chunk = (rows + SCAN_THREADS - 1) / SCAN_THREADS;
  const long long a = 1 + threadIdx.x * chunk, e = min(a + chunk, rows + 1);
  long long s = 0;
  for (long long i = a; i < e; ++i) s += pre[i];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int off = 1; off < SCAN_THREADS; off <<= 1) {
    const long long v = threadIdx.x >= off ? part[threadIdx.x - off] : 0;
    __syncthreads();
    part[threadIdx.x] += v;
    __syncthreads();
  }
  long long run = threadIdx.x ? part[threadIdx.x - 1] : 0;
  for (long long i = a; i < e; ++i) { run += pre[i]; pre[i] = run; }
  if (threadIdx.x == 0) pre[0] = 0;
}

}  // namespace
