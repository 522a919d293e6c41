// augment.cu -- the training notebooks' augmenter on the device (stardist_b200.models.Augmenter): numpy's legacy Gaussian
// stream (np.random.normal on the global RandomState) and the per-item transpose / flips / intensity change / noise add on the
// gathered patches.  Compiled with -fmad=false: every rounding below is numpy's.
//
// The Gaussian stream.  MT19937 words w, tempered; two words make one double u = ((w0 >> 5) * 2^26 + (w1 >> 6)) / 2^53; the
// polar method draws x1 = 2u - 1, x2 = 2u - 1 (four words per attempt), rejects r2 = x1^2 + x2^2 >= 1 or == 0, and for
// f = sqrt(-2 log(r2) / r2) returns f*x2 and caches f*x1 as the next value (has_gauss / gauss of get_state()).  Only the word
// recurrence is sequential: k_mt_twist runs it in one block, three dependency levels of <= 227 words per twist of 624, and
// writes every key it passes through ([key_0 | key_1 | ...]), so word j of the stream (from the state's pos) is entry
// pos + j of that buffer and the key numpy holds afterwards is one of its blocks.  Tempering, the acceptance test, a prefix
// count over accepted attempts, f and the output are parallel over attempts.  CUDA's double log is within 1 ulp (glibc's is
// not correctly rounded either), so values may differ from numpy's by a few ulp; the state never does.
#include <algorithm>
#include <climits>
#include <cmath>
#include "common.cuh"
#include "../../include/stardist_b200.h"

namespace {

using sdb::cdiv;

constexpr int MT_N = 624, MT_M = 397;
constexpr unsigned MT_UPPER = 0x80000000u, MT_LOWER = 0x7fffffffu, MT_A = 0x9908b0dfu;
constexpr int ATT_THREADS = 256;       // attempts per block of the counting / emitting kernels

struct MtState {                       // what the host reads back: numpy's (key, pos, has_gauss, gauss) + accepted pairs
  unsigned key[MT_N];
  int pos, has_gauss;
  double gauss;
  long long accepted;
  int last_block, pad;
};

__device__ __forceinline__ unsigned mt_mix(unsigned a, unsigned b, unsigned c) {
  const unsigned y = (a & MT_UPPER) | (b & MT_LOWER);
  return c ^ (y >> 1) ^ ((y & 1u) ? MT_A : 0u);
}

// T twists of keys[0 .. 623] -> keys[t * 624 ...] for t = 1..T; one thread per key word
__global__ void __launch_bounds__(MT_N) k_mt_twist(unsigned* __restrict__ keys, int T) {
  __shared__ unsigned s[2][MT_N];
  const int i = threadIdx.x;
  s[0][i] = keys[i];
  __syncthreads();
  int cur = 0;
  for (int t = 1; t <= T; ++t) {
    const unsigned* P = s[cur];
    unsigned* Q = s[cur ^ 1];
    const unsigned a = P[i], b = i + 1 < MT_N ? P[i + 1] : 0u;
    if (i < MT_N - MT_M) Q[i] = mt_mix(a, b, P[i + MT_M]);                                  // old words only
    __syncthreads();
    if (i >= MT_N - MT_M && i < 2 * (MT_N - MT_M)) Q[i] = mt_mix(a, b, Q[i - (MT_N - MT_M)]);
    __syncthreads();
    if (i >= 2 * (MT_N - MT_M) && i < MT_N - 1) Q[i] = mt_mix(a, b, Q[i - (MT_N - MT_M)]);
    else if (i == MT_N - 1) Q[i] = mt_mix(a, Q[0], Q[MT_M - 1]);
    __syncthreads();
    keys[(long long)t * MT_N + i] = Q[i];
    cur ^= 1;
  }
}

__device__ __forceinline__ unsigned mt_temper(unsigned y) {
  y ^= y >> 11;
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= y >> 18;
  return y;
}

// attempt a: words pos + 4a .. pos + 4a + 3 -> (x1, x2, r2), accepted or not
__device__ __forceinline__ bool polar_attempt(const unsigned* __restrict__ keys, int pos, long long a, double& x1, double& x2,
                                              double& r2) {
  const unsigned* w = keys + pos + 4 * a;
  const unsigned w0 = mt_temper(__ldg(w)), w1 = mt_temper(__ldg(w + 1)), w2 = mt_temper(__ldg(w + 2)), w3 = mt_temper(__ldg(w + 3));
  const double u1 = __ddiv_rn(__dadd_rn(__dmul_rn((double)(w0 >> 5), 67108864.0), (double)(w1 >> 6)), 9007199254740992.0);
  const double u2 = __ddiv_rn(__dadd_rn(__dmul_rn((double)(w2 >> 5), 67108864.0), (double)(w3 >> 6)), 9007199254740992.0);
  x1 = __dsub_rn(__dmul_rn(2.0, u1), 1.0);
  x2 = __dsub_rn(__dmul_rn(2.0, u2), 1.0);
  r2 = __dadd_rn(__dmul_rn(x1, x1), __dmul_rn(x2, x2));
  return !(r2 >= 1.0 || r2 == 0.0);
}

// accepted attempts per block of ATT_THREADS
__global__ void __launch_bounds__(ATT_THREADS) k_polar_count(const unsigned* __restrict__ keys, int pos, long long A,
                                                             long long* __restrict__ counts) {
  const long long a = (long long)blockIdx.x * ATT_THREADS + threadIdx.x;
  double x1, x2, r2;
  const int acc = a < A && polar_attempt(keys, pos, a, x1, x2, r2);
  const int n = __syncthreads_count(acc);
  if (threadIdx.x == 0) counts[blockIdx.x] = n;
}

// exclusive scan of the block counts in place (one block), the total into st->accepted
__global__ void __launch_bounds__(1024) k_polar_scan(long long* __restrict__ counts, int nblk, MtState* __restrict__ st) {
  __shared__ long long part[1024];
  const int chunk = (nblk + 1023) / 1024, a = threadIdx.x * chunk, e = min(a + chunk, nblk);
  long long s = 0;
  for (int i = a; i < e; ++i) s += counts[i];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {
    const long long v = threadIdx.x >= off ? part[threadIdx.x - off] : 0;
    __syncthreads();
    part[threadIdx.x] += v;
    __syncthreads();
  }
  long long run = threadIdx.x ? part[threadIdx.x - 1] : 0;
  for (int i = a; i < e; ++i) { const long long c = counts[i]; counts[i] = run; run += c; }
  if (threadIdx.x == 1023) { st->accepted = part[1023]; st->last_block = 0; }    // k_polar_emit sets the block when M pairs exist
}

// accepted attempt of rank k < M: out[hg + 2k] = f*x2, out[hg + 2k + 1] = f*x1 (or the cache when that is past n); the
// attempt of rank M - 1 writes the state numpy holds afterwards (except the key, which k_mt_state_key copies)
__global__ void __launch_bounds__(ATT_THREADS) k_polar_emit(const unsigned* __restrict__ keys, int pos, long long A,
                                                            const long long* __restrict__ offsets, long long M, int hg,
                                                            double gauss_in, long long n, double* __restrict__ out,
                                                            MtState* __restrict__ st) {
  __shared__ int warp_cnt[ATT_THREADS / 32];
  const long long a = (long long)blockIdx.x * ATT_THREADS + threadIdx.x;
  double x1 = 0, x2 = 0, r2 = 0;
  const bool acc = a < A && polar_attempt(keys, pos, a, x1, x2, r2);
  const unsigned bal = __ballot_sync(0xffffffffu, acc);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) warp_cnt[wid] = __popc(bal);
  __syncthreads();
  long long k = offsets[blockIdx.x] + __popc(bal & ((1u << lane) - 1u));
  for (int w = 0; w < wid; ++w) k += warp_cnt[w];
  if (a == 0 && hg) out[0] = gauss_in;
  if (!acc || k >= M) return;
  const double f = sqrt(__ddiv_rn(__dmul_rn(-2.0, log(r2)), r2));
  const long long v = hg + 2 * k;
  out[v] = __dmul_rn(f, x2);
  const bool cached = v + 1 >= n;
  if (!cached) out[v + 1] = __dmul_rn(f, x1);
  if (k == M - 1) {
    const long long c = pos + 4 * (a + 1);                    // flat index of the next word
    const long long t = (c - 1) / MT_N;
    st->last_block = (int)t;
    st->pos = (int)(c - t * MT_N);
    st->has_gauss = cached;
    st->gauss = cached ? __dmul_rn(f, x1) : 0.0;
  }
}

__global__ void __launch_bounds__(MT_N) k_mt_state_key(const unsigned* __restrict__ keys, MtState* __restrict__ st) {
  st->key[threadIdx.x] = keys[(long long)st->last_block * MT_N + threadIdx.x];
}

// ------------------------------------------------------------------------------------------------------------ augment
// one thread per output pixel of the batch: the item's transpose + flips as source index arithmetic, then x * s + t in float32
// and, with noise, float32(double(x) + sig * n)
constexpr int AUG_PARAM_WORDS = 12;   // per item (int64): src axis per output axis [3], flip [3], bits of s, t (float32), sig (float64), noise on

__global__ void k_augment(const long long* __restrict__ prm, long long n, int pz, int py, int px, int C, int gz, int gy, int gx, int Goy,
                          int Gox, const float* __restrict__ X, const int* __restrict__ Yraw, const int* __restrict__ Ys,
                          const double* __restrict__ noise, float* __restrict__ Xo, int* __restrict__ Yc, int* __restrict__ Yso,
                          int* __restrict__ Ye, unsigned char* __restrict__ neg) {
  const long long P = (long long)pz * py * px;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(e % px);
    long long t = e / px;
    const int y = (int)(t % py);
    t /= py;
    const int z = (int)(t % pz);
    const long long b = t / pz;
    const long long* q = prm + b * AUG_PARAM_WORDS;
    const int o[3] = {z, y, x}, ext[3] = {pz, py, px};
    int j[3];
    for (int a = 0; a < 3; ++a) j[q[a]] = q[3 + a] ? ext[a] - 1 - o[a] : o[a];
    const long long e_in = b * P + ((long long)j[0] * py + j[1]) * px + j[2];
    const float s = __int_as_float((int)q[6]), sh = __int_as_float((int)q[7]);
    const double sig = __longlong_as_double(q[8]);
    const double* nz = q[9] ? noise + b * P * C : nullptr;
    const long long loc = e - b * P;
    for (int c = 0; c < C; ++c) {
      float r = __fadd_rn(__fmul_rn(__ldg(X + e_in * C + c), s), sh);
      if (nz) r = __double2float_rn(__dadd_rn((double)r, __dmul_rn(sig, __ldg(nz + loc * C + c))));
      Xo[e * C + c] = r;
    }
    const int v = __ldg(Yraw + e_in), slot = __ldg(Ys + e_in);
    Yc[e] = max(v, 0);
    Yso[e] = slot;
    if (z % gz == 0 && y % gy == 0 && x % gx == 0) {
      const long long og = ((b * ((pz - 1) / gz + 1) + z / gz) * Goy + y / gy) * Gox + x / gx;
      neg[og] = v < 0;
      if (Ye) Ye[og] = slot;
    }
  }
}

int grid_for(long long work, int threads) { return (int)std::max<long long>(1, std::min<long long>(cdiv(work, threads), 132 * 32)); }

}  // namespace

extern "C" int sdb_mt_normal(const unsigned* h_key, int pos, int has_gauss, double gauss, long long n, double* d_out,
                             unsigned* h_key_out, int* h_pos_out, int* h_has_gauss_out, double* h_gauss_out, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (pos < 0 || pos > MT_N || n < 0) { sdb::set_error("mt_normal: pos must lie in [0, 624] and n >= 0"); return 1; }
  has_gauss = has_gauss ? 1 : 0;
  std::copy(h_key, h_key + MT_N, h_key_out);
  *h_pos_out = pos; *h_has_gauss_out = has_gauss; *h_gauss_out = gauss;
  if (n == 0) return 0;
  const long long M = (n - has_gauss + 1) / 2;              // pairs to draw
  if (M == 0) {                                             // the cached value alone
    SDB_CUDA(cudaMemcpyAsync(d_out, &gauss, sizeof(double), cudaMemcpyHostToDevice, st));
    SDB_CUDA(cudaStreamSynchronize(st));
    *h_has_gauss_out = 0; *h_gauss_out = 0.0;
    return 0;
  }
  // attempts: the expected M / (pi / 4) with a margin of ~13 standard deviations; doubled in the (never seen) case it falls short
  long long A = (long long)std::ceil((M + 6.0 * std::sqrt((double)M) + 32.0) / 0.7853981633974483);
  sdb::DevBuf keys, counts, state;
  MtState h;
  SDB_CUDA(state.alloc(sizeof(MtState), st));
  for (;;) {
    const long long words = pos + 4 * A;
    const long long T = (words + MT_N - 1) / MT_N - 1;        // twists past the current key
    const long long nblk = (A + ATT_THREADS - 1) / ATT_THREADS;
    if (T > INT_MAX || nblk > INT_MAX) { sdb::set_error("mt_normal: n too large"); return 1; }
    SDB_CUDA(keys.alloc((size_t)(T + 1) * MT_N * sizeof(unsigned), st));
    SDB_CUDA(counts.alloc((size_t)nblk * sizeof(long long), st));
    SDB_CUDA(cudaMemcpyAsync(keys.p, h_key, MT_N * sizeof(unsigned), cudaMemcpyHostToDevice, st));
    if (T > 0) SDB_LAUNCH(k_mt_twist, 1, MT_N, 0, st, keys.as<unsigned>(), (int)T);
    SDB_LAUNCH(k_polar_count, (int)nblk, ATT_THREADS, 0, st, keys.as<const unsigned>(), pos, A, counts.as<long long>());
    SDB_LAUNCH(k_polar_scan, 1, 1024, 0, st, counts.as<long long>(), (int)nblk, state.as<MtState>());
    SDB_LAUNCH(k_polar_emit, (int)nblk, ATT_THREADS, 0, st, keys.as<const unsigned>(), pos, A, counts.as<const long long>(), M, has_gauss,
               gauss, n, d_out, state.as<MtState>());
    SDB_LAUNCH(k_mt_state_key, 1, MT_N, 0, st, keys.as<const unsigned>(), state.as<MtState>());
    SDB_CUDA(cudaMemcpyAsync(&h, state.p, sizeof(MtState), cudaMemcpyDeviceToHost, st));
    SDB_CUDA(cudaStreamSynchronize(st));
    if (h.accepted >= M) break;
    A *= 2;
  }
  std::copy(h.key, h.key + MT_N, h_key_out);
  *h_pos_out = h.pos; *h_has_gauss_out = h.has_gauss; *h_gauss_out = h.gauss;
  return 0;
}

extern "C" int sdb_augment_batch(const long long* d_params, int ndim, int batch, const int* patch_size, int n_channels, const int* grid,
                                 const float* d_x, const int* d_y_raw, const int* d_y_slots, const double* d_noise, float* d_x_out,
                                 int* d_y_clamped, int* d_y_slots_out, int* d_y_slots_grid, unsigned char* d_neg, sdb_stream_t stream) {
  if ((ndim != 2 && ndim != 3) || batch < 1 || n_channels < 1) {
    sdb::set_error("augment_batch: ndim must be 2 or 3, batch >= 1 and n_channels >= 1"); return 1;
  }
  int p[3] = {1, 1, 1}, g[3] = {1, 1, 1};
  long long n = batch;
  for (int a = 0; a < ndim; ++a) {
    if (grid[a] < 1 || patch_size[a] < 1) { sdb::set_error("augment_batch: grid and patch sizes must be >= 1"); return 1; }
    p[3 - ndim + a] = patch_size[a]; g[3 - ndim + a] = grid[a];
    n *= patch_size[a];
  }
  SDB_LAUNCH(k_augment, grid_for(n, 256), 256, 0, (cudaStream_t)stream, d_params, n, p[0], p[1], p[2], n_channels, g[0], g[1], g[2],
             (p[1] - 1) / g[1] + 1, (p[2] - 1) / g[2] + 1, d_x, d_y_raw, d_y_slots, d_noise, d_x_out, d_y_clamped, d_y_slots_out,
             d_y_slots_grid, d_neg);
  return 0;
}
