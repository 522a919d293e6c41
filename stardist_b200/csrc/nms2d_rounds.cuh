// nms2d_rounds.cuh -- frontier / suppress kernels of the 2D NMS, templated on the polygon
// capacity NV.  Included by exactly one TU per NV (the clipping sweep is large; separate TUs
// compile in parallel).  Must be compiled with -fmad=false.
#pragma once
#include "nms2d_common.cuh"
#include "clip2d.cuh"
#include "polyfast.cuh"
#include <algorithm>
#include <vector>

namespace sdnms {
namespace {

struct DevVerts {
  const int2* v;
  __device__ int32_t x(int i) const { return v[i].x; }
  __device__ int32_t y(int i) const { return v[i].y; }
};

// overlap test of kept h against candidate c; returns 1 suppressed, 0 not, -1 pool overflow
template <int NV, int SC>
__device__ int pair_suppresses(const NmsArrays& A, int h, int c, sdclip::ClipSweep<NV, SC>& S) {
  DevVerts va{A.verts + (size_t)h * A.R}, vb{A.verts + (size_t)c * A.R};
  int status;
  const float inter = sdclip::clip_intersection_area(va, vb, A.R, S, &status);
  if (status == sdclip::CLIP_OVERFLOW) return -1;
  // overlap = area_inter / fmin(areas[i]+1e-10, areas[j]+1e-10)  (double), stored to float (:580)
  const double den = fmin((double)A.area[h] + 1.e-10, (double)A.area[c] + 1.e-10);
  const float overlap = (float)((double)inter / den);
  return overlap > A.threshold ? 1 : 0;
}

// counters: [0] undecided at round start, [1] pairs emitted this round, [2] pair tests (total),
//           [3] slow-path pool overflows (fatal), [4] slow pairs this round, [5] sticky "pair list
//           overflowed" flag: every later kernel of the batch becomes a no-op until the host recovers,
//           [6] candidates kept in this round (length of the kept list)
//
// K_frontier is PULL based with a per-candidate cursor: the 3x3 cell neighbourhood is scanned in a
// fixed order and the scan resumes where it stopped in the previous round -- an item that did not
// block once (h >= c, h decided, or h cannot reach c) never blocks later, so the total scan work over
// all rounds is one pass over the neighbourhood.  K_pairs is PUSH based: one warp per candidate kept
// in this round enumerates the undecided candidates it reaches (only ~n_kept * degree work in total).
// The undecided candidates are kept in a compacted list (double buffered: blocked candidates are
// appended to list_out, counters[7] = its length; round 0 reads the identity list).
// (device function shared by the stand-alone kernel and the tail kernel k_tail; the arrays written during the rounds carry
// no __restrict__ / const-cache qualifiers: inside k_tail they are re-read after grid-wide barriers)
__device__ __forceinline__ void d_frontier2(const NmsArrays& A, int round, int2* cursor, int* kept_list,
                            const int* list_in, unsigned int n_in_or_all, const unsigned int* n_in_dev,
                            int* list_out, unsigned int* counters, const int* pend = nullptr) {
  // one WARP per undecided candidate: the neighbourhood scan is a chain of dependent loads, so the lanes
  // test 32 list items per step (a kept candidate scans its whole 3x3 neighbourhood: ~2000 items)
  if (counters[5]) return;
  const unsigned int n_in = n_in_dev ? *n_in_dev : n_in_or_all;
  const unsigned int warps = (gridDim.x * blockDim.x) >> 5, lane = threadIdx.x & 31;
  const int kept_now = ST_KEPT_BASE + round;
  unsigned int n_undecided = 0;
  for (unsigned int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n_in; i += warps) {
    const int c = list_in ? list_in[i] : (int)i;
    if (A.state[c] != ST_UNDECIDED) continue;
    ++n_undecided;
    const float cy = A.points[2 * c], cx = A.points[2 * c + 1];
    const int4 bc = A.bbox[c];
    int ccx = 0, ccy = 0;
    if (!A.G.all_pairs) { ccx = cell_of(cx, A.G.minx, A.G.cell, A.G.gx); ccy = cell_of(cy, A.G.miny, A.G.cell, A.G.gy); }
    int2 cur = cursor[c];          // (neighbour cell 0..8, offset inside that cell)
    bool blocked = false, first_step = true;
    for (int k = cur.x; k < 9 && !blocked; ++k) {
      // own cell first, then the edge neighbours, then the corners: a blocker is nearly always found among the
      // first (= highest scored) items of the candidate's own cell
      const int kk = (0x862075314 >> (4 * k)) & 15;       // k -> 4,1,3,5,7,0,2,6,8
      const int yy = ccy + kk / 3 - 1, xx = ccx + kk % 3 - 1;
      if (yy < 0 || yy >= A.G.gy || xx < 0 || xx >= A.G.gx) { cur.x = k + 1; cur.y = 0; continue; }
      const int cell = yy * A.G.gx + xx;
      const unsigned int b = A.cell_start[cell], e = A.cell_start[cell + 1];
      // The scan is a chain of dependent L2 round trips (items -> state / centre / radius / bbox), ~1 us per step
      // whatever its width: the first step of a candidate looks at 32 items (in round 0 that nearly always finds
      // the blocker), later steps at 128 (4 per lane, loads in flight together).
      unsigned int t0 = b + (unsigned int)cur.y;
      if (first_step && t0 < e) {
        first_step = false;
        const unsigned int t = t0 + lane;
        bool hit = false, past = false;
        if (t < e) {
          const int h = A.items[t];
          if (h < c) {
            const int sh = A.state[h];
            if (sh == ST_UNDECIDED || sh == kept_now) hit = reaches(A, h, c, cy, cx, bc);
          } else past = true;
        }
        const unsigned int m = __ballot_sync(0xffffffffu, hit);
        if (m) { blocked = true; cur.x = k; cur.y = (int)(t0 + (unsigned int)(__ffs(m) - 1) - b); }
        else if (__any_sync(0xffffffffu, past)) t0 = e;
        else t0 += 32;
      }
      for (; t0 < e && !blocked; t0 += 128) {
        int hs[4];
        bool hit[4], past = false;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const unsigned int t = t0 + 32u * u + lane;
          hs[u] = (t < e) ? A.items[t] : 0x7fffffff;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          hit[u] = false;
          const int h = hs[u];
          if (h < c) {
            const int sh = A.state[h];
            if (sh == ST_UNDECIDED || sh == kept_now) hit[u] = reaches(A, h, c, cy, cx, bc);
          } else if (h != 0x7fffffff) past = true;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const unsigned int m = __ballot_sync(0xffffffffu, hit[u]);
          if (m && !blocked) { blocked = true; cur.x = k; cur.y = (int)(t0 + 32u * u + (unsigned int)(__ffs(m) - 1) - b); }
        }
        if (__any_sync(0xffffffffu, past)) break;     // cell lists are sorted by index: nothing below c is left
      }
      if (!blocked) { cur.x = k + 1; cur.y = 0; }
    }
    if (lane == 0) {
      cursor[c] = cur;
      // (k_tail only) a candidate with open pairs -- tests against kept polygons the pre-filter left to the exact sweep,
      // not yet run -- stays undecided: it keeps blocking what it reaches and is looked at again after the next flush
      if (!blocked && pend && pend[c] > 0) blocked = true;
      if (!blocked) {
        A.state[c] = kept_now;
        kept_list[atomicAdd(&counters[6], 1u)] = c;
      } else {
        list_out[atomicAdd(&counters[7], 1u)] = c;
      }
    }
  }
  if (lane == 0 && n_undecided) atomicAdd(&counters[0], n_undecided);
}
__global__ void __launch_bounds__(256) k_frontier2(NmsArrays A, int round, int2* cursor, int* kept_list, const int* list_in, unsigned int n_in_or_all,
                                                   const unsigned int* n_in_dev, int* list_out, unsigned int* counters) {
  d_frontier2(A, round, cursor, kept_list, list_in, n_in_or_all, n_in_dev, list_out, counters);
}

// one BLOCK per candidate kept in this round: emit the (h, c) pairs the reference would test (:548-576).
// (A warp per h walked ~2000 neighbour items in 60 dependent steps: ~100 us per round regardless of the count.)
__device__ __forceinline__ void d_pairs(const NmsArrays& A, int round, const int* kept_list, int2* pairs, unsigned int cap, unsigned int* counters) {
  if (counters[5]) return;
  const unsigned int n_kept = counters[6];
  for (unsigned int w = blockIdx.x; w < n_kept; w += gridDim.x) {
    const int h = kept_list[w];
    const float hy = A.points[2 * h], hx = A.points[2 * h + 1];
    const int4 bh = A.bbox[h];
    const float rr = A.max_dist + A.radius[h];
    int hcx = 0, hcy = 0;
    if (!A.G.all_pairs) { hcx = cell_of(hx, A.G.minx, A.G.cell, A.G.gx); hcy = cell_of(hy, A.G.miny, A.G.cell, A.G.gy); }
    // the (up to) nine neighbour cells as one flat index range: their item loads are independent, so all threads of
    // the block walk the concatenation instead of nine short dependent passes
    unsigned int beg[9], pre[10];
    pre[0] = 0;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const int yy = hcy + k / 3 - 1, xx = hcx + k % 3 - 1;
      unsigned int b = 0, e = 0;
      if (yy >= 0 && yy < A.G.gy && xx >= 0 && xx < A.G.gx) { const int cell = yy * A.G.gx + xx; b = A.cell_start[cell]; e = A.cell_start[cell + 1]; }
      beg[k] = b; pre[k + 1] = pre[k] + (e - b);
    }
    for (unsigned int u = threadIdx.x; u < pre[9]; u += blockDim.x) {
      unsigned int t = 0;
#pragma unroll
      for (int q = 0; q < 9; ++q) if (u >= pre[q] && u < pre[q + 1]) t = beg[q] + (u - pre[q]);     // static indices: registers
      {
        {
          const int c = A.items[t];
          if (c <= h) continue;
          if (A.state[c] != ST_UNDECIDED) continue;
          if (!A.G.all_pairs) {
            const float d0 = hy - A.points[2 * c], d1 = hx - A.points[2 * c + 1];
            const float dd = d0 * d0 + d1 * d1;
            if (!(dd < rr * rr)) continue;
          }
          if (A.use_bbox) {
            const int4 bc = A.bbox[c];
            if (!(bc.x <= bh.y && bh.x <= bc.y && bc.z <= bh.w && bh.z <= bc.w)) continue;
          }
          const unsigned int k2 = atomicAdd(&counters[1], 1u);
          if (k2 < cap) { int2 pr; pr.x = h; pr.y = c; pairs[k2] = pr; }
        }
      }
    }
  }
}
__global__ void __launch_bounds__(256) k_pairs(NmsArrays A, int round, const int* kept_list, int2* pairs, unsigned int cap, unsigned int* counters) {
  d_pairs(A, round, kept_list, pairs, cap, counters);
}
__global__ void k_check_overflow(unsigned int cap, unsigned int* __restrict__ counters) {
  if (counters[1] > cap) counters[5] = 1;
}

// Pre-filter (polyfast.cuh): one WARP per pair.  Lane j owns edge j of the candidate's polygon (and j+32, ...
// for n_rays > 32) and walks the suppressor's edges, which are warp-uniform loads; the closed-form overlap
// integral and its bound decide most pairs, the rest is appended to the exact list (counters[9]).
// verify != 0: nothing is decided here, the verdict is stored per pair for k_clip to compare.
template <typename T>
__device__ __forceinline__ void d_fast(const NmsArrays& A, const int2* pairs, int2* xpairs, signed char* verdict, int verify, unsigned int* counters,
                                       int* pend = nullptr) {
  if (counters[5]) return;
  const unsigned int n_pairs = counters[1];
  const unsigned int warps = (gridDim.x * blockDim.x) >> 5, lane = threadIdx.x & 31;
  const int R = A.R;
  for (unsigned int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n_pairs; w += warps) {
    const int2 pr = pairs[w];
    const int h = pr.x, c = pr.y;
    if (!verify && A.state[c] == ST_SUPPRESSED) continue;
    const int2* __restrict__ va = A.verts + (size_t)h * R;
    const int2* __restrict__ vb = A.verts + (size_t)c * R;
    const double* __restrict__ sa = A.suf + (size_t)h * R;
    const double* __restrict__ sb = A.suf + (size_t)c * R;
    const int2 p0 = va[0], q0 = vb[0];
    sdfast::Accum acc; acc.clear();
    int wq = 0, wp = 0;
    bool overflow = false;
    for (int j = lane; j < R; j += 32) {
      const int j1 = (j + 1 == R) ? 0 : j + 1;
      const int2 b0 = vb[j], b1 = vb[j1], a0 = va[j], a1 = va[j1];
      sdfast::Edge f; f.x0 = b0.x; f.y0 = b0.y; f.x1 = b1.x; f.y1 = b1.y;
      sdfast::Edge e2; e2.x0 = a0.x; e2.y0 = a0.y; e2.x1 = a1.x; e2.y1 = a1.y;
      wq += sdfast::wind_Q_edge(f, p0.x, p0.y);
      wp += sdfast::wind_P_edge(e2, q0.x, q0.y);
      // pass 1, branch free: which edges of P does f properly cross?  (at most two are remembered; a third sends
      // the pair to the exact sweep.)  A crossing costs ~150 instructions; taken inside this loop it ran ~14 times
      // per pair with one or two active lanes.
      const T fx = (T)f.x1 - (T)f.x0, fy = (T)f.y1 - (T)f.y0;
      const int tieQ = sdfast::tie_edge(fx, fy);
      int cnt = 0, ci0 = -1, ci1 = -1;
      int2 prev = p0;
      T o3 = fx * ((T)prev.y - (T)f.y0) - fy * ((T)prev.x - (T)f.x0);
      for (int i = 0; i < R; ++i) {
        const int2 cur = va[(i + 1 == R) ? 0 : i + 1];      // warp-uniform
        const T ex = (T)cur.x - (T)prev.x, ey = (T)cur.y - (T)prev.y;
        const T o1 = ex * ((T)f.y0 - (T)prev.y) - ey * ((T)f.x0 - (T)prev.x);
        const T o2 = ex * ((T)f.y1 - (T)prev.y) - ey * ((T)f.x1 - (T)prev.x);
        const T o4 = fx * ((T)cur.y - (T)f.y0) - fy * ((T)cur.x - (T)f.x0);
        const bool cross = sdfast::crossing_test(ex, ey, fx, fy, o1, o2, o3, o4, sdfast::tie_point(ex, ey), tieQ);
        ci1 = (cross && cnt == 1) ? i : ci1;
        ci0 = (cross && cnt == 0) ? i : ci0;
        cnt += cross ? 1 : 0;
        o3 = o4;                                            // orient(q0,q1,p1) of this edge = orient(q0,q1,p0) of the next
        prev = cur;
      }
      overflow |= (cnt > 2);
      // pass 2, lock step: every lane handles its first recorded crossing, then its second
#pragma unroll 1
      for (int c = 0; c < 2; ++c) {
        const int i = c ? ci1 : ci0;
        if (i >= 0) {
          const int2 e0 = va[i], e1 = va[(i + 1 == R) ? 0 : i + 1];
          sdfast::Edge e; e.x0 = e0.x; e.y0 = e0.y; e.x1 = e1.x; e.y1 = e1.y;
          const T ex = (T)e.x1 - (T)e.x0, ey = (T)e.y1 - (T)e.y0;
          const T o1 = ex * ((T)f.y0 - (T)e.y0) - ey * ((T)f.x0 - (T)e.x0);
          const T o2 = ex * ((T)f.y1 - (T)e.y0) - ey * ((T)f.x1 - (T)e.x0);
          const T q3 = fx * ((T)e.y0 - (T)f.y0) - fy * ((T)e.x0 - (T)f.x0);
          const T q4 = fx * ((T)e.y1 - (T)f.y0) - fy * ((T)e.x1 - (T)f.x0);
          sdfast::crossing_contrib(e, f, ex, ey, fx, fy, o1, o2, q3, q4, tieQ, sa[i], sb[j], acc);
        }
      }
    }
    overflow = __any_sync(0xffffffffu, overflow);
    for (int o = 16; o > 0; o >>= 1) {
      acc.I += __shfl_xor_sync(0xffffffffu, acc.I, o);
      acc.len += __shfl_xor_sync(0xffffffffu, acc.len, o);
      acc.K += __shfl_xor_sync(0xffffffffu, acc.K, o);
      wq += __shfl_xor_sync(0xffffffffu, wq, o);
      wp += __shfl_xor_sync(0xffffffffu, wp, o);
    }
    if (lane == 0) {
      const double I = acc.I + (double)wq * A.sarea[h] + (double)wp * A.sarea[c];
      const double bound = sdfast::clipper_bound(acc, (double)A.maxlen[h] + (double)A.maxlen[c], A.max_abs_coord, R);
      const double den = fmin((double)A.area[h] + 1.e-10, (double)A.area[c] + 1.e-10);
      const int d = overflow ? -1 : sdfast::decide(I, bound, den, A.threshold);
      if (verify) verdict[w] = (signed char)d;
      else if (d == 1) A.state[c] = ST_SUPPRESSED;
      else if (d < 0) { xpairs[atomicAdd(&counters[9], 1u)] = pr; if (pend) atomicAdd(&pend[c], 1); }
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256) k_fast(NmsArrays A, const int2* pairs, int2* xpairs, signed char* verdict, int verify, unsigned int* counters,
                                              int* pend) {
  d_fast<T>(A, pairs, xpairs, verdict, verify, counters, pend);
}

// Exact sweep: ONE PAIR PER WARP, executed by lane 0 with the sweep state (~8 KB of pools for 32-gons) in
// SHARED memory.  The sweep is ~3e4 dependent, branchy instructions per pair: lanes running different pairs
// serialise anyway (a 32-pairs-per-warp version was no faster in aggregate), and a single active lane in local
// memory touches 4 bytes of every 128-byte line -- its 8 KB of state occupied ~70 KB of L1 and ran out of L2.
// n_list: &counters[1] (all pairs) or &counters[9] (pairs the pre-filter left open).
template <int NV> struct ClipCfg { static constexpr int WARPS = (NV <= 32) ? 4 : 1; };

template <int NV>
__device__ __forceinline__ void d_clip(const NmsArrays& A, const int2* pairs, const unsigned int* n_list, const signed char* verdict,
                                       int2* slow_pairs, unsigned int* counters, unsigned char* clip_smem, int* pend = nullptr, int wpb = 0) {
  if (counters[5]) return;
  const unsigned int n_pairs = *n_list;
  // wpb: warps of a block that sweep (0 = all); their sweep states occupy the first wpb slots of clip_smem
  const unsigned int W = wpb ? (unsigned int)wpb : (blockDim.x >> 5);
  const unsigned int G = gridDim.x * W;                                       // sweeping warps in the grid
  const unsigned int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned int warp_g = blockIdx.x * W + wib;
  if (wib >= W || warp_g >= n_pairs || lane != 0) return;
  sdclip::ClipSweep<NV, 1>& S = *reinterpret_cast<sdclip::ClipSweep<NV, 1>*>(clip_smem + (size_t)(threadIdx.x >> 5) * sizeof(sdclip::ClipSweep<NV, 1>));
  for (unsigned int t = warp_g; t < n_pairs; t += G) {
    const int2 pr = pairs[t];
    if (pend) atomicSub(&pend[pr.y], 1);                             // this open pair is resolved by the end of the phase
    if (!verdict && A.state[pr.y] == ST_SUPPRESSED) continue;        // already suppressed by another pair (benign race)
    const int r = pair_suppresses<NV, 1>(A, pr.x, pr.y, S);
    if (r == 1) A.state[pr.y] = ST_SUPPRESSED;
    else if (r < 0) { const unsigned int k = atomicAdd(&counters[4], 1u); slow_pairs[k] = pr; }
    if (verdict && r >= 0) {
      const int d = verdict[t];
      if (d < 0) atomicAdd(&counters[9], 1u);            // would have gone to the exact sweep
      else if (d != r) atomicAdd(&counters[10], 1u);     // the pre-filter would have decided wrongly
    }
  }
}

template <int NV>
__global__ void __launch_bounds__(32 * ClipCfg<NV>::WARPS) k_clip(NmsArrays A, const int2* pairs, const unsigned int* n_list, const signed char* verdict,
                                                                  int2* slow_pairs, unsigned int* counters) {
  extern __shared__ __align__(16) unsigned char clip_smem_k[];
  d_clip<NV>(A, pairs, n_list, verdict, slow_pairs, counters, clip_smem_k);
}

template <int NV>
__global__ void __launch_bounds__(64) k_clip_slow(NmsArrays A, const int2* __restrict__ slow_pairs, unsigned int* __restrict__ counters) {
  if (counters[5]) return;
  const unsigned int n_slow = counters[4];
  if (blockIdx.x * blockDim.x >= n_slow) return;
  sdclip::ClipSweep<NV, 4> S;
  for (unsigned int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_slow; t += gridDim.x * blockDim.x) {
    const int2 pr = slow_pairs[t];
    const int r = pair_suppresses<NV, 4>(A, pr.x, pr.y, S);
    if (r == 1) A.state[pr.y] = ST_SUPPRESSED;
    else if (r < 0) atomicAdd(&counters[3], 1u);
  }
}

__device__ __forceinline__ void d_reset_counters(unsigned int* counters) {
  counters[2] += counters[1]; counters[0] = 0; counters[1] = 0; counters[4] = 0; counters[6] = 0; counters[8] = counters[7]; counters[7] = 0;
  counters[12] += counters[9]; counters[9] = 0;
}
__global__ void k_reset_counters(unsigned int* counters) {
  if (counters[5]) return;
  if (threadIdx.x == 0) d_reset_counters(counters);
}

// ---------------------------------------------------------------------------------------------------------
// Tail of the frontier peeling in ONE cooperative launch.  Round 0 carries the bulk of the work (all candidates scanned,
// ~70 % of the pair tests) and runs as full-occupancy kernels; the rounds after it touch a few thousand candidates each
// and were dominated by launch gaps and host round trips (7 launches per round, a synchronisation every 4 rounds).
// Here the phases of a round are separated by grid-wide barriers, the termination test (no undecided candidate left)
// is evaluated on the device, and the host reads the counters once at the end.  The kernel hands back to the host loop
// (which knows how to grow the pair list / run the slow exact path) by leaving: counters[5] set (pair list overflow),
// counters[4] != 0 (pairs for the slow path) or simply counters[0] != 0 after max_rounds; counters[13] = round in progress.
struct TailCtx {
  int2* cursor; int* kept; int* list0; int* list1; int2* pairs; int2* xpairs; int2* slow; int* pend;
  unsigned int* counters; unsigned int* bar; unsigned int cap; int round0, max_rounds, filter;
  unsigned long long* dbg;      // optional phase time stamps (verbose >= 2): [round][8] globaltimer ns, written by the lead thread
};
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
#define TAIL_STAMP(slot) do { if (C.dbg && lead && round - C.round0 < 64) C.dbg[(round - C.round0) * 8 + (slot)] = gtime(); } while (0)

// Grid-wide barrier of the cooperative launch (all blocks are resident): arrival counter + generation word, with a bounded
// wait -- if the blocks ever disagree on the control flow, the kernel gives up (bar[2] = 1, every block returns) instead of
// hanging the device; the host then reports an error.  bar = {count, generation, abort}, zeroed by the host.
struct GridBarrier {
  unsigned int* bar; bool dead;
  __device__ GridBarrier(unsigned int* b) : bar(b), dead(false) {}
  __device__ void sync() {
    __shared__ int s_dead;
    __syncthreads();
    if (threadIdx.x == 0) {
      volatile unsigned int* vb = bar;
      int d = dead || vb[2] != 0;
      if (!d) {
        __threadfence();
        const unsigned int gen = vb[1];
        if (atomicAdd(&bar[0], 1u) == gridDim.x - 1) { bar[0] = 0; __threadfence(); atomicAdd(&bar[1], 1u); }
        else {
          const long long t0 = clock64();
          while (vb[1] == gen) {
            if (vb[2] != 0) { d = 1; break; }
            if (clock64() - t0 > 3000000000LL) { atomicExch(&bar[2], 1u); d = 1; break; }      // ~1.5 s at 1.9 GHz
          }
        }
        __threadfence();
      }
      s_dead = d;
    }
    __syncthreads();
    dead = dead || s_dead != 0;
  }
};
constexpr int TAIL_CLIP_WARPS = 8;                // sweeping warps per block (8 KB of shared sweep state each for 32-gons): all of them --
                                                  // a flush of <= 3.5 k pairs is then one sweep latency (~0.2 ms) long (r02h: 4 warps -> 0.4 ms)
constexpr unsigned int TAIL_FLUSH_MIN = 1024;     // open pairs that make an exact-sweep phase worth its ~0.2 ms latency

template <int NV, int MINB>
__global__ void __launch_bounds__(256, MINB) k_tail(NmsArrays A, TailCtx C) {
  GridBarrier grid(C.bar);
  extern __shared__ __align__(16) unsigned char tail_smem[];
  unsigned int* cnt = C.counters;
  volatile unsigned int* vc = cnt;
  if (vc[5] || vc[3] || vc[4]) return;                  // round 0 left work for the host (uniform: nothing writes before the first barrier)
  const bool lead = blockIdx.x == 0 && threadIdx.x == 0;
  // The exact sweep costs ~0.2 ms of pure latency per phase whatever the number of pairs (one 3e4-instruction dependent
  // chain per pair).  With the pre-filter on, pairs it leaves open are therefore DEFERRED: the candidate is marked pending
  // (d_frontier2 will not keep it, it goes on blocking what it reaches) and the open pairs of several rounds are swept
  // together -- when enough have accumulated, when the frontier cannot advance without them, or before leaving.
  int* pend = C.filter == 1 ? C.pend : nullptr;
  for (int round = C.round0; round < C.round0 + C.max_rounds; ++round) {
    // barrier BEFORE the counters are reset: the decisions at the end of the previous round (flush / leave) read
    // counters[4], [6], [9] after that round's last barrier -- every block must have taken them before they change
    grid.sync(); if (grid.dead) return;
    if (lead) {
      cnt[2] += cnt[1]; cnt[0] = 0; cnt[1] = 0; cnt[4] = 0; cnt[6] = 0; cnt[8] = cnt[7]; cnt[7] = 0;      // d_reset_counters without the open list
      if (!pend) { cnt[12] += cnt[9]; cnt[9] = 0; }
      cnt[13] = (unsigned int)round;
    }
    grid.sync(); if (grid.dead) return;
    TAIL_STAMP(0);
    const unsigned int n_open_start = vc[9];              // open pairs carried over; nothing changes it before this round's d_fast
    int* lin = (round & 1) ? C.list1 : C.list0;
    int* lout = (round & 1) ? C.list0 : C.list1;
    d_frontier2(A, round, C.cursor, C.kept, lin, 0u, cnt + 8, lout, cnt, pend);
    grid.sync(); if (grid.dead) return;
    TAIL_STAMP(1);
    if (vc[0] == 0) break;                                // no undecided candidate was left: done (nothing can be pending)
    bool leave = false;
    d_pairs(A, round, C.kept, C.pairs, C.cap, cnt);
    grid.sync(); if (grid.dead) return;
    TAIL_STAMP(2);
    // pair list overflow: the host grows it and redoes this round's pair stage (the flag is raised on the way out, after
    // the open pairs have been swept: every phase is a no-op once counters[5] is set)
    const bool overflow = vc[1] > C.cap;
    if (C.filter == 1) {
      if (!overflow && n_open_start + vc[1] > C.cap) {    // the open list could overflow: sweep what is there first (both values are stable here)
        d_clip<NV>(A, C.xpairs, cnt + 9, nullptr, C.slow, cnt, tail_smem, pend, TAIL_CLIP_WARPS);
        grid.sync(); if (grid.dead) return;
        if (lead) { cnt[12] += cnt[9]; cnt[9] = 0; }
        grid.sync(); if (grid.dead) return;
      }
      if (!overflow) {
        d_fast<int32_t>(A, C.pairs, C.xpairs, nullptr, 0, cnt, pend);
        grid.sync(); if (grid.dead) return;
      }
      TAIL_STAMP(3);
      // flush: enough open pairs, or no candidate was kept in this round (the frontier is waiting for them), or leaving
      const bool must_leave = overflow || vc[4] != 0;
      const unsigned int n_open = vc[9];
      if (n_open > 0 && (must_leave || n_open >= TAIL_FLUSH_MIN || vc[6] == 0)) {
        d_clip<NV>(A, C.xpairs, cnt + 9, nullptr, C.slow, cnt, tail_smem, pend, TAIL_CLIP_WARPS);
        grid.sync(); if (grid.dead) return;
        if (lead) { cnt[12] += cnt[9]; cnt[9] = 0; }
        grid.sync(); if (grid.dead) return;
      }
      TAIL_STAMP(4);
      if (C.dbg && lead && round - C.round0 < 64) { C.dbg[(round - C.round0) * 8 + 5] = n_open; C.dbg[(round - C.round0) * 8 + 6] = vc[6]; C.dbg[(round - C.round0) * 8 + 7] = vc[0]; }
      leave = must_leave || vc[4] != 0;                   // (a flush that produced slow pairs has swept everything: nothing is pending)
    } else {
      if (!overflow) {
        d_clip<NV>(A, C.pairs, cnt + 1, nullptr, C.slow, cnt, tail_smem, nullptr, TAIL_CLIP_WARPS);
        grid.sync(); if (grid.dead) return;
      }
      leave = overflow || vc[4] != 0;                     // pool overflow in the fast sweep: slow exact path on the host loop
    }
    if (overflow && lead) cnt[5] = 1;
    if (leave) break;
  }
}

template <int NV>
int run_rounds(NmsArrays A, int* d_slow_unused, unsigned int* d_counters, cudaStream_t st, int verbose,
               unsigned int* h_pin /* pinned [8*BATCH] */) {
  (void)d_slow_unused;
  const int n = A.n;
  constexpr int BATCH = 4;     // rounds launched per host synchronisation (host loop)
  size_t cap = std::max<size_t>((size_t)n * 2, 1 << 15);
  sdb::DevBuf b_pairs, b_slow, b_cursor, b_kept, b_list0, b_list1, b_xpairs, b_verdict;
  const int filter = A.filter;
  auto alloc_filter_lists = [&]() -> int {
    if (filter == 1) SDB_CUDA(b_xpairs.alloc(cap * sizeof(int2), st));
    if (filter == 2) SDB_CUDA(b_verdict.alloc(cap, st));
    return 0;
  };
  if (alloc_filter_lists()) return 1;
  SDB_CUDA(b_list0.alloc((size_t)n * sizeof(int), st));
  SDB_CUDA(b_list1.alloc((size_t)n * sizeof(int), st));
  SDB_CUDA(b_cursor.alloc((size_t)n * sizeof(int2), st));
  SDB_CUDA(b_kept.alloc((size_t)n * sizeof(int), st));
  SDB_CUDA(cudaMemsetAsync(b_cursor.p, 0, (size_t)n * sizeof(int2), st));
  SDB_CUDA(b_pairs.alloc(cap * sizeof(int2), st));
  SDB_CUDA(b_slow.alloc(cap * sizeof(int2), st));
  SDB_CUDA(cudaMemsetAsync(d_counters, 0, 16 * sizeof(unsigned int), st));
  int round = 0;
  auto launch_frontier = [&](int r) -> int {
    SDB_LAUNCH(k_reset_counters, 1, 32, 0, st, d_counters);
    // round r reads the list written by round r-1 (length saved in counters[8] by k_reset_counters)
    int* lin = (r & 1) ? b_list1.as<int>() : b_list0.as<int>();
    int* lout = (r & 1) ? b_list0.as<int>() : b_list1.as<int>();
    sdb::ProfSpan spf;
    sdb::profile_begin("nms2d_frontier", st, &spf);
    if (r == 0) SDB_LAUNCH(k_frontier2, 132 * 8, 256, 0, st, A, r, b_cursor.as<int2>(), b_kept.as<int>(), (const int*)nullptr, (unsigned int)n, (const unsigned int*)nullptr, lout, d_counters);
    else SDB_LAUNCH(k_frontier2, 132 * 8, 256, 0, st, A, r, b_cursor.as<int2>(), b_kept.as<int>(), (const int*)lin, 0u, (const unsigned int*)(d_counters + 8), lout, d_counters);
    sdb::profile_end("nms2d_frontier", st, &spf);
    return 0;
  };
  auto launch_clip_slow = [&]() -> int {
    SDB_LAUNCH((k_clip_slow<NV>), 8, 64, 0, st, A, b_slow.as<int2>(), d_counters);
    return 0;
  };
  int* d_pend = nullptr;          // set on the k_tail path: round 0 leaves its open pairs to the tail kernel's first flush
  auto launch_pair_stage = [&](int r, bool defer_exact = false) -> int {
    sdb::ProfSpan sp;
    sdb::profile_begin("nms2d_pairs", st, &sp);
    SDB_LAUNCH(k_pairs, 132 * 8, 256, 0, st, A, r, b_kept.as<int>(), b_pairs.as<int2>(), (unsigned int)cap, d_counters);
    sdb::profile_end("nms2d_pairs", st, &sp);
    SDB_LAUNCH(k_check_overflow, 1, 1, 0, st, (unsigned int)cap, d_counters);
    if (filter) {
      sdb::profile_begin("nms2d_fast", st, &sp);
      int* pend = defer_exact ? d_pend : nullptr;
      if (A.max_abs_coord <= 8191.0) SDB_LAUNCH(k_fast<int32_t>, 132 * 8, 256, 0, st, A, b_pairs.as<int2>(), b_xpairs.as<int2>(), b_verdict.as<signed char>(), filter == 2 ? 1 : 0, d_counters, pend);
      else SDB_LAUNCH(k_fast<long long>, 132 * 8, 256, 0, st, A, b_pairs.as<int2>(), b_xpairs.as<int2>(), b_verdict.as<signed char>(), filter == 2 ? 1 : 0, d_counters, pend);
      sdb::profile_end("nms2d_fast", st, &sp);
      if (defer_exact && filter == 1) return 0;       // the open pairs (counters[9], pend[]) are swept by k_tail
    }
    sdb::profile_begin("nms2d_clip", st, &sp);
    {
      constexpr int CW = ClipCfg<NV>::WARPS;
      const size_t csm = (size_t)CW * sizeof(sdclip::ClipSweep<NV, 1>);
      static bool attr = false;
      if (!attr) { SDB_CUDA(cudaFuncSetAttribute(k_clip<NV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)csm)); attr = true; }
      const int cblocks = 132 * (NV <= 32 ? 6 : 4);
      if (filter == 1) SDB_LAUNCH((k_clip<NV>), cblocks, 32 * CW, csm, st, A, b_xpairs.as<int2>(), d_counters + 9, (const signed char*)nullptr, b_slow.as<int2>(), d_counters);
      else SDB_LAUNCH((k_clip<NV>), cblocks, 32 * CW, csm, st, A, b_pairs.as<int2>(), d_counters + 1, filter == 2 ? b_verdict.as<signed char>() : (const signed char*)nullptr, b_slow.as<int2>(), d_counters);
    }
    sdb::profile_end("nms2d_clip", st, &sp);
    return launch_clip_slow();
  };
  // pair list overflowed in round r: its frontier marks are in place, the later kernels of the round were no-ops.
  // Grow the lists, clear the flag, redo the pair stage of that round (c = the counters read back).
  auto recover_overflow = [&](const unsigned int* c, int r) -> int {
    cap = (size_t)c[1] + (size_t)c[1] / 2 + 1024;
    SDB_CUDA(b_pairs.alloc(cap * sizeof(int2), st));
    SDB_CUDA(b_slow.alloc(cap * sizeof(int2), st));
    if (alloc_filter_lists()) return 1;
    const unsigned int zeros[10] = {c[0], 0, c[2], 0, 0, 0, c[6], c[7], c[8], 0};
    SDB_CUDA(cudaMemcpyAsync(d_counters, zeros, sizeof(zeros), cudaMemcpyHostToDevice, st));
    if (launch_pair_stage(r)) return 1;
    SDB_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  auto finish_stats = [&](const unsigned int* c) {
    // pairs tested = counters[2] (accumulated by the counter reset) + the pairs of the last counted round
    unsigned int tot = c[2] + c[1], exact = c[12] + c[9], bad = c[10];
    if (!filter) exact = tot;
    sdb::profile_add_units("nms2d_clip", (double)exact);
    sdb::profile_add_units("nms2d_fast", (double)tot);
    g_filter_stats[0] += tot; g_filter_stats[1] += exact; g_filter_stats[2] += bad; g_filter_stats[3] += 1;
    if (verbose) printf("NMS2D(b200): pair tests=%u, exact sweeps=%u (filter mode %d), verify mismatches=%u\n", tot, exact, filter, bad);
  };

  // ---- round 0 as full-occupancy kernels, the remaining rounds in one cooperative launch (k_tail)
  if (g_tail_mode && NV <= 32 && filter != 2 && A.max_abs_coord <= 8191.0) {
    // g_tail_mode 1: 3 blocks per SM (no register spills), 2: 4 blocks per SM (64 registers; more warps for the latency-bound
    // frontier phase, some spills in the sweep)
    const bool four = g_tail_mode == 2;
    const void* tail_fn = four ? (const void*)k_tail<NV, 4> : (const void*)k_tail<NV, 3>;
    static int tail_blocks_v[2] = {-1, -1};
    int& tail_blocks = tail_blocks_v[four ? 1 : 0];
    const size_t tsm = (size_t)TAIL_CLIP_WARPS * sizeof(sdclip::ClipSweep<NV, 1>);
    if (tail_blocks < 0) {
      int dev = 0, coop = 0, sms = 0, per_sm = 0;
      cudaGetDevice(&dev);
      cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
      cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
      cudaError_t e1 = four ? cudaFuncSetAttribute(k_tail<NV, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tsm)
                            : cudaFuncSetAttribute(k_tail<NV, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tsm);
      cudaError_t e2 = four ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_tail<NV, 4>, 256, tsm)
                            : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_tail<NV, 3>, 256, tsm);
      if (coop && e1 == cudaSuccess && e2 == cudaSuccess && per_sm > 0) tail_blocks = sms * std::min(per_sm, four ? 4 : 3);
      else { tail_blocks = 0; cudaGetLastError(); }
    }
    if (tail_blocks > 0) {
      sdb::DevBuf b_pend;
      SDB_CUDA(b_pend.alloc((size_t)n * sizeof(int), st));
      SDB_CUDA(cudaMemsetAsync(b_pend.p, 0, (size_t)n * sizeof(int), st));
      d_pend = b_pend.as<int>();
      if (launch_frontier(0) || launch_pair_stage(0, filter == 1)) return 1;
      d_pend = nullptr;
      sdb::DevBuf b_bar;
      SDB_CUDA(b_bar.alloc(4 * sizeof(unsigned int), st));
      SDB_CUDA(cudaMemsetAsync(b_bar.p, 0, 4 * sizeof(unsigned int), st));
      sdb::DevBuf b_dbg;
      if (verbose > 1) { SDB_CUDA(b_dbg.alloc(64 * 8 * sizeof(unsigned long long), st)); SDB_CUDA(cudaMemsetAsync(b_dbg.p, 0, 64 * 8 * sizeof(unsigned long long), st)); }
      TailCtx C{b_cursor.as<int2>(), b_kept.as<int>(), b_list0.as<int>(), b_list1.as<int>(), b_pairs.as<int2>(), b_xpairs.as<int2>(), b_slow.as<int2>(),
                b_pend.as<int>(), d_counters, b_bar.as<unsigned int>(), (unsigned int)cap, 1, 4 * n + 8, filter,
                verbose > 1 ? b_dbg.as<unsigned long long>() : nullptr};
      void* args[] = {(void*)&A, (void*)&C};
      sdb::ProfSpan spt;
      sdb::profile_begin("nms2d_tail", st, &spt);
      SDB_CUDA(cudaLaunchCooperativeKernel(tail_fn, dim3(tail_blocks), dim3(256), args, tsm, st));
      sdb::g_launch_count++;
      sdb::profile_end("nms2d_tail", st, &spt);
      SDB_CUDA(cudaMemcpyAsync(h_pin, d_counters, 16 * sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
      SDB_CUDA(cudaMemcpyAsync(h_pin + 16, b_bar.p, 4 * sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
      SDB_CUDA(cudaStreamSynchronize(st));
      if (h_pin[16 + 2] != 0) { sdb::set_error("nms2d: grid barrier of the tail kernel timed out (inconsistent control flow)"); return 1; }
      if (verbose > 1) {
        std::vector<unsigned long long> dbg(64 * 8);
        SDB_CUDA(cudaMemcpy(dbg.data(), b_dbg.p, dbg.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        printf("NMS2D(b200) tail phases per round (us): frontier | pairs | fast | flush   [open pairs, kept, undecided]\n");
        for (int r = 0; r < 64 && dbg[r * 8]; ++r) {
          const unsigned long long* d = &dbg[r * 8];
          if (!d[1]) break;
          printf("  round %2d: %7.1f | %6.1f | %6.1f | %6.1f   [%llu, %llu, %llu]\n", r + 1, (d[1] - d[0]) / 1e3, d[2] ? (d[2] - d[1]) / 1e3 : 0.0,
                 d[3] ? (d[3] - d[2]) / 1e3 : 0.0, d[4] ? (d[4] - d[3]) / 1e3 : 0.0, d[5], d[6], d[7]);
        }
      }
      const unsigned int* c = h_pin;
      const int r = (int)c[13];                      // round in progress when the tail kernel left (0: it never started)
      if (verbose) printf("NMS2D(b200): tail kernel left in round %d: undecided=%u overflow=%u slow=%u\n", r, c[0], c[5], c[4]);
      if (c[3] != 0) { sdb::set_error("nms2d: polygon clipping pools overflowed in the slow path"); return 1; }
      if (c[5] != 0) { if (recover_overflow(c, r)) return 1; round = r + 1; }
      else if (c[4] != 0 && r > 0) { if (launch_clip_slow()) return 1; round = r + 1; }     // (round 0 ran its slow path already)
      else if (r > 0 && c[0] == 0) { finish_stats(c); return 0; }
      else round = r + 1;
      // anything else continues in the host loop below from `round`
    }
  }

  for (;;) {
    const int round0 = round;
    for (int b = 0; b < BATCH; ++b, ++round) {
      if (launch_frontier(round)) return 1;
      if (launch_pair_stage(round)) return 1;
      SDB_CUDA(cudaMemcpyAsync(h_pin + 16 * b, d_counters, 16 * sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
    }
    SDB_CUDA(cudaStreamSynchronize(st));
    bool done = false;
    const unsigned int* c_done = nullptr;
    for (int b = 0; b < BATCH; ++b) {
      const unsigned int* c = h_pin + 16 * b;
      if (c[3] != 0) { sdb::set_error("nms2d: polygon clipping pools overflowed in the slow path"); return 1; }
      if (c[5] != 0) {
        round = round0 + b;
        if (recover_overflow(c, round)) return 1;
        round += 1;
        break;
      }
      if (c[0] == 0) { done = true; c_done = c; break; }
    }
    if (verbose > 1)
      for (int b = 0; b < BATCH; ++b) { const unsigned int* c = h_pin + 16 * b; printf("  round %d: undecided=%u kept=%u pairs=%u exact=%u slow=%u\n", round0 + b, c[0], c[6], c[1], c[9], c[4]); }
    if (verbose) printf("NMS2D(b200): rounds=%d undecided(last)=%u pair tests so far=%u\n", round, h_pin[16 * (BATCH - 1)], h_pin[16 * (BATCH - 1) + 2] + h_pin[16 * (BATCH - 1) + 1]);
    if (done) { finish_stats(c_done); break; }
    if (round > 4 * n + 8) { sdb::set_error("nms2d: no progress"); return 1; }
  }
  return 0;
}

}  // namespace
}  // namespace sdnms
