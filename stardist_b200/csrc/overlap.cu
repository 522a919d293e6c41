// overlap.cu -- sparse label-overlap tables of label maps (matching.py label_overlap, the optimize_thresholds engine,
// group_matching_labels).
//
// Reference: stardist/matching.py:38-52 (_label_overlap: overlap[x[i], y[i]] += 1 over a dense (1+max x, 1+max y) matrix).
// Here only the pairs that occur are kept: every distinct (a, b), background 0 included, with its pixel count, sorted by
// (a, b).  Label maps are spatially coherent, so
//   * each warp merges equal keys with __match_any_sync (one update per run of equal pairs),
//   * each CTA accumulates into a shared-memory open-addressing table (bounded probing),
//   * what does not fit there goes to a global open-addressing table (u64 key CAS, u64 count add),
// and the CTA tables are flushed into the global one at the end.  The keys are then compacted, sorted with the bitonic
// network of bitonic.cuh and emitted with their counts.  The floor is the 8 B per pixel read of the two maps.
//
// The same machinery runs over a stack of T frames [T, S] (group_matching_labels, matching.py:409-472), one grid row
// (blockIdx.y) per frame or frame pair, with the group index folded into the key:
//   * sdb_stack_labels: the distinct (frame, label) of every frame, key (frame << 32) | label;
//   * sdb_stack_overlap: the overlap of the consecutive pairs (p, p + 1), on ids compacted per frame to 0..n_f as
//     relabel_sequential would (0 = background, the others in ascending order, looked up in the sorted ids of the frame
//     that sdb_stack_labels gave), key ((p - p0) << 2w) | (a' << w) | b' with w = key_bits;
//   * sdb_stack_group_remap writes the grouped stack: frame 0 copied, frame f > 0 through a lookup table indexed by the
//     compacted ids.
#include <algorithm>
#include "common.cuh"
#include "bitonic.cuh"
#include "../../include/stardist_b200.h"

namespace {

using sdb::cdiv;
typedef unsigned long long u64;

constexpr u64 EMPTY = ~0ull;            // never a valid key: every key layout below keeps bit 63 clear
constexpr int OT = 256;                 // threads per CTA
constexpr int SH_SLOTS = 2048;          // shared table: 2048 x (8 B key + 8 B count) = 32 KB
constexpr int SH_PROBES = 16;
constexpr long long MAX_CAPACITY = 1ll << 28;

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

// 1 + rank of label v among the sorted non-zero ids[lo, hi) of its frame (where it occurs), 0 for the background
__device__ __forceinline__ u64 compact_id(const int* __restrict__ ids, long long lo, long long hi, int v) {
  if (v == 0) return 0;
  const long long first = lo;
  while (lo < hi) {
    const long long mid = lo + ((hi - lo) >> 1);
    if (__ldg(ids + mid) < v) lo = mid + 1; else hi = mid;
  }
  return (u64)(lo - first + 1);
}

// pixel sources of k_overlap_count: load(g, i, va, vb) reads pixel i of group g (= blockIdx.y); the warp merges equal
// (va, vb), and the lowest lane of each run turns them into the table key with key(g, va, vb)
struct PairSrc {                        // sdb_label_overlap: two maps, one group
  const int* a; const int* b;
  __device__ void load(long long, long long i, int& va, int& vb) const { va = __ldg(a + i); vb = __ldg(b + i); }
  __device__ u64 key(long long, int va, int vb) const { return ((u64)(unsigned int)va << 32) | (u64)(unsigned int)vb; }
};

struct FrameSrc {                       // sdb_stack_labels: group = frame, key (frame << 32) | label
  const int* y; long long S;
  __device__ void load(long long g, long long i, int& va, int& vb) const { va = (int)g; vb = __ldg(y + g * S + i); }
  __device__ u64 key(long long, int va, int vb) const { return ((u64)(unsigned int)va << 32) | (u64)(unsigned int)vb; }
};

struct StackPairSrc {                   // sdb_stack_overlap: group g = pair p0 + g of frames (p, p + 1), compacted ids
  const int* y; long long S; long long p0; const int* ids; const long long* off; int w;
  __device__ void load(long long g, long long i, int& va, int& vb) const {
    const int* f = y + (p0 + g) * S;
    va = __ldg(f + i); vb = __ldg(f + S + i);
  }
  __device__ u64 key(long long g, int va, int vb) const {
    const long long p = p0 + g;
    const u64 ca = compact_id(ids, __ldg(off + p), __ldg(off + p + 1), va);
    const u64 cb = compact_id(ids, __ldg(off + p + 1), __ldg(off + p + 2), vb);
    return ((u64)g << (2 * w)) | (ca << w) | cb;
  }
};

template <class Src>
__global__ void __launch_bounds__(OT) k_overlap_count(Src src, long long n, long long n_groups,
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
  for (long long g = blockIdx.y; g < n_groups; g += gridDim.y) {
    for (long long it = 0; it < n_iter; ++it) {
      const long long i = base + it * stride;
      const bool valid = i < n;
      int va = 0, vb = 0;
      if (valid) src.load(g, i, va, vb);
      const bool neg = valid && (va < 0 || vb < 0);
      if (neg) flags[0] = 1u;
      const bool use = valid && !neg;
      const unsigned int active = __ballot_sync(0xffffffffu, use);
      if (!use) continue;
      const unsigned int peers = __match_any_sync(active, ((u64)(unsigned int)va << 32) | (u64)(unsigned int)vb);
      if (lane != __ffs(peers) - 1) continue;                        // the lowest lane of each run of equal pairs adds
      const u64 key = src.key(g, va, vb);
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

// row r of the sorted table: either split into int32 (a, b) pairs (sdb_label_overlap) or kept as the 64-bit key
__global__ void k_overlap_emit(const u64* __restrict__ sorted, long long n, const u64* __restrict__ keys,
                               const u64* __restrict__ counts, u64 mask, int* __restrict__ pairs, long long* __restrict__ out_keys,
                               long long* __restrict__ out_counts) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const u64 key = sorted[r];
  u64 s = mix(key) & mask;
  while (keys[s] != key) s = (s + 1) & mask;                         // present: it was compacted from this table
  if (pairs) {
    pairs[2 * r] = (int)(key >> 32);
    pairs[2 * r + 1] = (int)(key & 0xffffffffull);
  } else {
    out_keys[r] = (long long)key;
  }
  out_counts[r] = (long long)counts[s];
}

// count the distinct keys of `src` over n pixels x n_groups groups and emit them sorted, with the capacity protocol of
// sdb_label_overlap (*h_n > capacity: nothing written, an upper bound of the number of keys reported)
template <class Src>
int overlap_table(const Src& src, long long n, long long n_groups, int* d_pairs, long long* d_keys, long long* d_counts,
                  long long capacity, long long* h_n, const char* what, cudaStream_t st) {
  if (n < 0 || capacity < 1) { sdb::set_error(std::string(what) + ": n must be >= 0 and capacity >= 1"); return 1; }
  if (capacity > MAX_CAPACITY) { sdb::set_error(std::string(what) + ": capacity above 2^28 pairs"); return 1; }
  *h_n = 0;
  if (n == 0 || n_groups == 0) return 0;
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
  const dim3 grid((unsigned int)std::min<long long>(std::max<long long>(cdiv(n, OT * 8), 1), 132 * 4),
                  (unsigned int)std::min<long long>(n_groups, 65535));
  SDB_LAUNCH(k_overlap_count<Src>, grid, OT, 0, st, src, n, n_groups, b_keys.as<u64>(), b_counts.as<u64>(), slots - 1,
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
  if (hf[0]) { sdb::set_error(std::string(what) + ": negative label (label maps must be non-negative, matching.py:27-35)"); return 1; }
  const long long n_keys = (long long)h[2];
  if (hf[1] || n_keys > capacity) {
    // too small: report an upper bound of the number of distinct keys, write nothing.  `dropped` counts failed insertions,
    // not distinct keys, so the bound is also clamped to the pixel count (there are at most that many distinct keys)
    *h_n = std::max<long long>(std::min<long long>(n_keys + (long long)h[1], n * n_groups), capacity + 1);
    return 0;
  }
  *h_n = n_keys;
  if (sdb::bitonic::sort(b_sorted.as<u64>(), (unsigned int)n_keys, sdb::bitonic::padded_length((unsigned int)n_keys), st)) return 1;
  SDB_LAUNCH(k_overlap_emit, cdiv(n_keys, 256), 256, 0, st, b_sorted.as<u64>(), n_keys, b_keys.as<u64>(), b_counts.as<u64>(),
             slots - 1, d_pairs, d_keys, d_counts);
  return 0;
}

// grouped stack: frame 0 copied, frame f > 0 -> lut[off[f] + compact_id - 1] (0 stays 0); the lowest lane of each run of
// equal labels in a warp does the lookup
__global__ void __launch_bounds__(OT) k_group_remap(const int* __restrict__ y, long long S, long long T, const int* __restrict__ ids,
                                                    const long long* __restrict__ off, const int* __restrict__ lut,
                                                    int* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * OT;
  const long long n_iter = (S + stride - 1) / stride;
  const long long base = (long long)blockIdx.x * OT + threadIdx.x;
  for (long long f = blockIdx.y; f < T; f += gridDim.y) {
    const int* src = y + f * S;
    int* dst = out + f * S;
    for (long long it = 0; it < n_iter; ++it) {
      const long long i = base + it * stride;
      const bool valid = i < S;
      const int v = valid ? __ldg(src + i) : 0;
      if (f == 0) { if (valid) dst[i] = v; continue; }
      const unsigned int active = __ballot_sync(0xffffffffu, valid);
      if (!valid) continue;
      const unsigned int peers = __match_any_sync(active, v);
      const int leader = __ffs(peers) - 1;
      int r = 0;
      if (lane == leader && v != 0) {
        const long long lo = __ldg(off + f);
        r = __ldg(lut + lo + (long long)compact_id(ids, lo, __ldg(off + f + 1), v) - 1);
      }
      r = __shfl_sync(active, r, leader);
      dst[i] = r;
    }
  }
}

}  // namespace

extern "C" int sdb_label_overlap(const int* d_a, const int* d_b, long long n, int* d_pairs, long long* d_counts,
                                 long long capacity, long long* h_n_pairs, sdb_stream_t stream) {
  return overlap_table(PairSrc{d_a, d_b}, n, 1, d_pairs, nullptr, d_counts, capacity, h_n_pairs, "label_overlap",
                       (cudaStream_t)stream);
}

extern "C" int sdb_stack_labels(const int* d_stack, long long n_frames, long long frame_size, long long* d_keys,
                                long long* d_counts, long long capacity, long long* h_n_keys, sdb_stream_t stream) {
  if (n_frames < 0 || n_frames > 0x7fffffffll || frame_size < 0) { sdb::set_error("stack_labels: bad stack shape"); return 1; }
  return overlap_table(FrameSrc{d_stack, frame_size}, frame_size, n_frames, nullptr, d_keys, d_counts, capacity, h_n_keys,
                       "stack_labels", (cudaStream_t)stream);
}

extern "C" int sdb_stack_overlap(const int* d_stack, long long frame_size, long long first_pair, long long n_pairs,
                                 const int* d_ids, const long long* d_offsets, int key_bits, long long* d_keys, long long* d_counts,
                                 long long capacity, long long* h_n_keys, sdb_stream_t stream) {
  if (frame_size < 0 || first_pair < 0 || n_pairs < 0) { sdb::set_error("stack_overlap: bad stack shape"); return 1; }
  if (key_bits < 1 || key_bits > 31) { sdb::set_error("stack_overlap: key_bits must be in [1, 31]"); return 1; }
  if (n_pairs > 1 && (u64)(n_pairs - 1) >> (63 - 2 * key_bits)) {
    sdb::set_error("stack_overlap: the pair index does not fit the 63 - 2 * key_bits bits left in the key"); return 1;
  }
  return overlap_table(StackPairSrc{d_stack, frame_size, first_pair, d_ids, d_offsets, key_bits}, frame_size, n_pairs, nullptr,
                       d_keys, d_counts, capacity, h_n_keys, "stack_overlap", (cudaStream_t)stream);
}

extern "C" int sdb_stack_group_remap(const int* d_stack, long long n_frames, long long frame_size, const int* d_ids,
                                     const long long* d_offsets, const int* d_lut, int* d_out, sdb_stream_t stream) {
  if (n_frames < 0 || frame_size < 0) { sdb::set_error("stack_group_remap: bad stack shape"); return 1; }
  if (n_frames == 0 || frame_size == 0) return 0;
  const dim3 grid((unsigned int)std::min<long long>(std::max<long long>(cdiv(frame_size, OT * 8), 1), 132 * 4),
                  (unsigned int)std::min<long long>(n_frames, 65535));
  SDB_LAUNCH(k_group_remap, grid, OT, 0, (cudaStream_t)stream, d_stack, frame_size, n_frames, d_ids, d_offsets, d_lut, d_out);
  return 0;
}
