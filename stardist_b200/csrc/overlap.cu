// overlap.cu -- sparse label-overlap table of two label maps (matching.py label_overlap, the optimize_thresholds engine).
//
// Reference: stardist/matching.py:38-52 (_label_overlap: overlap[x[i], y[i]] += 1 over a dense (1+max x, 1+max y) matrix).
// Here only the pairs that occur are kept: every distinct (a, b), background 0 included, with its pixel count, sorted by
// (a, b).  Label maps are spatially coherent, so
//   * each warp merges equal keys with __match_any_sync (one update per run of equal pairs),
//   * each CTA accumulates into a shared-memory open-addressing table (bounded probing),
//   * what does not fit there goes to a global open-addressing table (u64 key CAS, u64 count add),
// and the CTA tables are flushed into the global one at the end.  The keys are then compacted, sorted with the bitonic
// network of bitonic.cuh and emitted with their counts.  The floor is the 8 B per pixel read of the two maps.
#include <algorithm>
#include "common.cuh"
#include "bitonic.cuh"
#include "../../include/stardist_b200.h"

namespace {

using sdb::cdiv;
typedef unsigned long long u64;

constexpr u64 EMPTY = ~0ull;            // never a valid key: both labels are non-negative int32, so bit 63 is clear
constexpr int OT = 256;                 // threads per CTA
constexpr int SH_SLOTS = 2048;          // shared table: 2048 x (8 B key + 8 B count) = 32 KB
constexpr int SH_PROBES = 16;

__device__ __forceinline__ u64 mix(u64 k) {             // splitmix64 finaliser
  k ^= k >> 30; k *= 0xbf58476d1ce4e5b9ull;
  k ^= k >> 27; k *= 0x94d049bb133111ebull;
  return k ^ (k >> 31);
}

// global table of `mask + 1` slots (power of two), linear probing over the whole table; false when it is full
__device__ bool global_add(u64* keys, u64* counts, u64 mask, u64 key, u64 c) {
  u64 s = mix(key) & mask;
  for (u64 probe = 0; probe <= mask; ++probe, s = (s + 1) & mask) {
    u64 k = keys[s];
    if (k == EMPTY) {
      k = atomicCAS(keys + s, EMPTY, key);
      if (k == EMPTY) k = key;
    }
    if (k == key) { atomicAdd(counts + s, c); return true; }
  }
  return false;
}

__global__ void __launch_bounds__(OT) k_overlap_count(const int* __restrict__ a, const int* __restrict__ b, long long n,
                                                      u64* __restrict__ keys, u64* __restrict__ counts, u64 mask,
                                                      unsigned int* __restrict__ flags /* [0] negative label, [1] table full */,
                                                      unsigned long long* __restrict__ dropped) {
  __shared__ u64 sk[SH_SLOTS];
  __shared__ u64 sc[SH_SLOTS];
  for (int i = threadIdx.x; i < SH_SLOTS; i += OT) { sk[i] = EMPTY; sc[i] = 0; }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * OT;
  const long long n_iter = (n + stride - 1) / stride;              // uniform trip count: every lane reaches the warp votes
  const long long base = (long long)blockIdx.x * OT + threadIdx.x;
  for (long long it = 0; it < n_iter; ++it) {
    const long long i = base + it * stride;
    const bool valid = i < n;
    int va = 0, vb = 0;
    if (valid) { va = __ldg(a + i); vb = __ldg(b + i); }
    const bool neg = valid && (va < 0 || vb < 0);
    if (neg) flags[0] = 1u;
    const bool use = valid && !neg;
    const unsigned int active = __ballot_sync(0xffffffffu, use);
    if (!use) continue;
    const u64 key = ((u64)(unsigned int)va << 32) | (u64)(unsigned int)vb;
    const unsigned int peers = __match_any_sync(active, key);
    if (lane != __ffs(peers) - 1) continue;                          // the lowest lane of each run of equal keys adds
    const u64 c = (u64)__popc(peers);
    bool done = false;
    unsigned int s = (unsigned int)(mix(key) & (SH_SLOTS - 1));
    for (int p = 0; p < SH_PROBES && !done; ++p, s = (s + 1) & (SH_SLOTS - 1)) {
      u64 k = sk[s];
      if (k == EMPTY) {
        k = atomicCAS(sk + s, EMPTY, key);
        if (k == EMPTY) k = key;
      }
      if (k == key) { atomicAdd(sc + s, c); done = true; }
    }
    if (!done && !global_add(keys, counts, mask, key, c)) { flags[1] = 1u; atomicAdd(dropped, 1ull); }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < SH_SLOTS; i += OT) {
    const u64 k = sk[i];
    if (k != EMPTY && !global_add(keys, counts, mask, k, sc[i])) { flags[1] = 1u; atomicAdd(dropped, 1ull); }
  }
}

__global__ void k_overlap_compact(const u64* __restrict__ keys, u64 slots, u64* __restrict__ out, unsigned long long* __restrict__ n_out,
                                  u64 capacity) {
  for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < slots; s += (u64)gridDim.x * blockDim.x) {
    const u64 k = keys[s];
    if (k == EMPTY) continue;
    const u64 pos = atomicAdd(n_out, 1ull);
    if (pos < capacity) out[pos] = k;
  }
}

__global__ void k_overlap_emit(const u64* __restrict__ sorted, long long n, const u64* __restrict__ keys,
                               const u64* __restrict__ counts, u64 mask, int* __restrict__ pairs, long long* __restrict__ out_counts) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const u64 key = sorted[r];
  u64 s = mix(key) & mask;
  while (keys[s] != key) s = (s + 1) & mask;                         // present: it was compacted from this table
  pairs[2 * r] = (int)(key >> 32);
  pairs[2 * r + 1] = (int)(key & 0xffffffffull);
  out_counts[r] = (long long)counts[s];
}

}  // namespace

extern "C" int sdb_label_overlap(const int* d_a, const int* d_b, long long n, int* d_pairs, long long* d_counts,
                                 long long capacity, long long* h_n_pairs, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n < 0 || capacity < 1) { sdb::set_error("label_overlap: n must be >= 0 and capacity >= 1"); return 1; }
  if (capacity > (1ll << 28)) { sdb::set_error("label_overlap: capacity above 2^28 pairs"); return 1; }
  *h_n_pairs = 0;
  if (n == 0) return 0;
  // the global table has at least twice the capacity: at most half full whenever the result fits
  u64 slots = 1ull << 12;
  while (slots < 2ull * (u64)capacity) slots <<= 1;
  sdb::DevBuf b_keys, b_counts, b_flags;
  SDB_CUDA(b_keys.alloc(slots * sizeof(u64), st));
  SDB_CUDA(b_counts.alloc(slots * sizeof(u64), st));
  SDB_CUDA(b_flags.alloc(4 * sizeof(u64), st));    // [0] u32 x2 flags, [1] dropped, [2] compacted count
  SDB_CUDA(cudaMemsetAsync(b_keys.p, 0xff, slots * sizeof(u64), st));
  SDB_CUDA(cudaMemsetAsync(b_counts.p, 0, slots * sizeof(u64), st));
  SDB_CUDA(cudaMemsetAsync(b_flags.p, 0, 4 * sizeof(u64), st));
  u64* flags64 = b_flags.as<u64>();
  const int grid = (int)std::min<long long>(std::max<long long>(cdiv(n, OT * 8), 1), 132 * 4);
  SDB_LAUNCH(k_overlap_count, grid, OT, 0, st, d_a, d_b, n, b_keys.as<u64>(), b_counts.as<u64>(), slots - 1,
             reinterpret_cast<unsigned int*>(flags64), flags64 + 1);
  sdb::DevBuf b_sorted;
  const unsigned int cap_pad = sdb::bitonic::padded_length((unsigned int)capacity);
  SDB_CUDA(b_sorted.alloc((size_t)cap_pad * sizeof(u64), st));
  SDB_LAUNCH(k_overlap_compact, (int)std::min<u64>(cdiv((long long)slots, 256), 132 * 8), 256, 0, st, b_keys.as<u64>(), slots,
             b_sorted.as<u64>(), flags64 + 2, (u64)capacity);
  u64 h[3] = {0, 0, 0};
  SDB_CUDA(cudaMemcpyAsync(h, flags64, sizeof(h), cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  const unsigned int* hf = reinterpret_cast<const unsigned int*>(h);
  if (hf[0]) { sdb::set_error("label_overlap: negative label (label maps must be non-negative, matching.py:27-35)"); return 1; }
  const long long n_pairs = (long long)h[2];
  if (hf[1] || n_pairs > capacity) {
    // too small: report an upper bound of the number of distinct pairs, write nothing.  `dropped` counts failed insertions,
    // not distinct keys, so the bound is also clamped to n (there are at most n distinct pairs)
    *h_n_pairs = std::max<long long>(std::min<long long>(n_pairs + (long long)h[1], n), capacity + 1);
    return 0;
  }
  *h_n_pairs = n_pairs;
  if (sdb::bitonic::sort(b_sorted.as<u64>(), (unsigned int)n_pairs, sdb::bitonic::padded_length((unsigned int)n_pairs), st)) return 1;
  SDB_LAUNCH(k_overlap_emit, cdiv(n_pairs, 256), 256, 0, st, b_sorted.as<u64>(), n_pairs, b_keys.as<u64>(), b_counts.as<u64>(),
             slots - 1, d_pairs, d_counts);
  return 0;
}
