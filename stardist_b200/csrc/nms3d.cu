// nms3d.cu -- star-convex polyhedron non-maximum suppression on the GPU.
//
// Reference: stardist/lib/stardist3d_impl.cpp:956-1385 (_COMMON_non_maximum_suppression_sparse):
//   precompute per candidate: volume (:257), integer bbox (:536), anisotropy = running float sum of
//   bbox extents / n (:1007-1010, summed here in index order == the OMP_NUM_THREADS=1 result),
//   outer / inner (isotropic) bounding radii (:1032-1052); kd-tree radius (max_dist + r_outer_i)^2;
//   greedy loop in score order; for every candidate pair the cascade (:1192-1334)
//     S1 upper bound  min(sphere_outer ∩, bbox ∩)        -> keep   if iou <= thr (use_bbox)
//     S2 lower bound  sphere_inner ∩                      -> suppress if iou > thr
//     S3 kernel ∩ kernel (Qhull halfspace intersection)   -> suppress if iou > thr
//     S4 hull ∩ hull                                      -> keep   if iou <= thr
//     S5 voxel render of i, count voxels also inside j    -> suppress if iou > thr   (early exit)
// Every stage is a pure function of the pair, so the greedy loop is resolved by the same
// frontier peeling as the 2D NMS (nms2d.cu): per round K_frontier, K_pretest (S1,S2 per candidate,
// emits the surviving pairs), K_heavy (one CTA per emitted pair: S3, S4, S5).
// S3/S4: geom3d.cuh (Q) -- Qhull-free, float-bit-equal on all fuzzed pairs (tests/tools/qhull_fuzz.py).
// S5 early exit is emulated on the full count: res = min(full, floor(overlap_maximal)+1) (SURVEY H4).
// Compile with -fmad=false.
#include <math.h>
#include <string.h>
#include <vector>
#include <algorithm>
#include "common.cuh"
#include "geom3d.cuh"
#include "bins3d.cuh"
#include "nms3d_pair.cuh"
#include "../../include/stardist_b200.h"

namespace {

using sdb::cdiv;
using sd3::Plane;

enum { ST_UNDECIDED = 0, ST_SUPPRESSED = 1, ST_KEPT_BASE = 2 };
constexpr int MAXR = sd3::SD3_MAX_RAYS, MAXF = sd3::SD3_MAX_FACES;

struct Grid3 { float mn[3]; float cell; int g[3]; int all_pairs; };

struct Arr {
  const float* dist; const float* points; const float* verts; const int* faces;
  int n, R, F;
  float* volume; int* bbox; float* r_outer; float* r_outer_iso; float* r_inner_iso;
  float* aniso_terms;    // [3][n]
  float* aniso;          // [3]
  const unsigned int* cell_start; const int* items; int* state;
  float max_dist, threshold; int use_bbox;
  int fan_subdiv;        // fan bounds on the refined fan (one extra ray per face)
  int s3_bound;          // k_heavy: lower-bound short cut in front of the S3 volume (decisions identical)
  int norm_planes;       // k_heavy: S3/S4 volumes on pre-normalised planes (face_cone_volume_n; bit-identical, see geom3d.cuh)
  int dup_dirs;          // the ray set has coincident directions (Rays_Cartesian poles): polyhedra can have duplicate vertices
  Grid3 G;
};

// ------------------------------------------------------------------------------------------
__global__ void k_pre1(Arr A, unsigned int* __restrict__ stats) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  const float* d = A.dist + (size_t)i * A.R;
  const float* c = A.points + 3 * i;
  A.volume[i] = sd3::polyhedron_volume(d, A.verts, A.faces, A.F);
  int bb[6];
  sd3::polyhedron_bbox(d, c, A.verts, A.R, bb);
  for (int k = 0; k < 6; ++k) A.bbox[6 * i + k] = bb[k];
  // anisotropy[k] += (float)(bbox extent) / n_polys   -- the terms; summed serially by k_aniso
  A.aniso_terms[i] = (float)(bb[1] - bb[0]) / A.n;
  A.aniso_terms[A.n + i] = (float)(bb[3] - bb[2]) / A.n;
  A.aniso_terms[2 * A.n + i] = (float)(bb[5] - bb[4]) / A.n;
  const float ro = sd3::bounding_radius_outer(d, A.R);
  A.r_outer[i] = ro;
  atomicMax(&stats[0], __float_as_uint(ro));
  for (int k = 0; k < 3; ++k) {
    const float v = fminf(fmaxf(c[k], -1.0e9f), 1.0e9f);
    atomicMin((int*)&stats[1 + 2 * k], (int)floorf(v)); atomicMax((int*)&stats[2 + 2 * k], (int)floorf(v));
  }
}

// serial float accumulation in index order (one warp per axis stages 32 terms at a time)
__global__ void k_aniso(Arr A) {
  const int axis = blockIdx.x;
  const float* t = A.aniso_terms + (size_t)axis * A.n;
  __shared__ float buf[1024];
  float acc = 0.f;
  for (int base = 0; base < A.n; base += 1024) {
    const int m = min(1024, A.n - base);
    for (int k = threadIdx.x; k < m; k += blockDim.x) buf[k] = t[base + k];
    __syncthreads();
    if (threadIdx.x == 0) for (int k = 0; k < m; ++k) acc = acc + buf[k];
    __syncthreads();
  }
  if (threadIdx.x == 0) A.aniso[axis] = acc;
}
__global__ void k_aniso_norm(Arr A) {
  // _tmp = fmax(fmax(a0,a1),a2); a_k = _tmp / a_k     (:1020-1023)
  const float a0 = A.aniso[0], a1 = A.aniso[1], a2 = A.aniso[2];
  const float tmp = fmaxf(fmaxf(a0, a1), a2);
  A.aniso[0] = tmp / a0; A.aniso[1] = tmp / a1; A.aniso[2] = tmp / a2;
}
__global__ void k_pre2(Arr A) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  const float* d = A.dist + (size_t)i * A.R;
  const float an[3] = {A.aniso[0], A.aniso[1], A.aniso[2]};
  A.r_outer_iso[i] = sd3::bounding_radius_outer_isotropic(d, A.verts, A.R, an);
  A.r_inner_iso[i] = sd3::bounding_radius_inner_isotropic(d, A.verts, A.faces, A.F, an);
}

// ---- uniform grid (same scheme as nms2d.cu) ------------------------------------------------
__device__ __forceinline__ int cell_of(float v, float mn, float cell, int g) {
  int c = (int)((v - mn) / cell);
  return c < 0 ? 0 : (c >= g ? g - 1 : c);
}
__device__ __forceinline__ int cell_index(const Grid3& G, const float* p) {
  if (G.all_pairs) return 0;
  return (cell_of(p[0], G.mn[0], G.cell, G.g[0]) * G.g[1] + cell_of(p[1], G.mn[1], G.cell, G.g[1])) * G.g[2] +
         cell_of(p[2], G.mn[2], G.cell, G.g[2]);
}
__global__ void k_cell_count(const float* __restrict__ points, int n, Grid3 G, int* __restrict__ cell_of_pt, unsigned int* __restrict__ counts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = cell_index(G, points + 3 * i);
  cell_of_pt[i] = c;
  atomicAdd(&counts[c], 1u);
}
__global__ void k_scan_serial(const unsigned int* __restrict__ counts, unsigned int* __restrict__ start, int n_cells) {
  // single block: chunked Hillis-Steele scan with carry
  __shared__ unsigned int sh[1024];
  __shared__ unsigned int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base <= n_cells; base += 1024) {
    const int i = base + threadIdx.x;
    const unsigned int v = (i < n_cells) ? counts[i] : 0u;
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int off = 1; off < 1024; off <<= 1) {
      const unsigned int t = (threadIdx.x >= off) ? sh[threadIdx.x - off] : 0u;
      __syncthreads();
      sh[threadIdx.x] += t;
      __syncthreads();
    }
    if (i <= n_cells) start[i] = carry + sh[threadIdx.x] - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry += sh[1023];
    __syncthreads();
  }
}
__global__ void k_cell_fill(const int* __restrict__ cell_of_pt, int n, unsigned int* __restrict__ cursor, int* __restrict__ items) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  items[atomicAdd(&cursor[cell_of_pt[i]], 1u)] = i;
}

// would h (higher score) test c ?  kd-tree radius query (:1169-1171), strict <
__device__ __forceinline__ bool reaches(const Arr& A, int h, const float* pc) {
  if (A.G.all_pairs) return true;
  const float* ph = A.points + 3 * h;
  const float d0 = ph[0] - pc[0], d1 = ph[1] - pc[1], d2 = ph[2] - pc[2];
  const float dd = d0 * d0 + d1 * d1 + d2 * d2;
  const float rr = A.max_dist + A.r_outer[h];
  return dd < rr * rr;
}

template <typename F>
__device__ __forceinline__ void for_neighbors(const Arr& A, int c, F&& f) {
  const float* pc = A.points + 3 * c;
  int cz = 0, cy = 0, cx = 0;
  if (!A.G.all_pairs) {
    cz = cell_of(pc[0], A.G.mn[0], A.G.cell, A.G.g[0]); cy = cell_of(pc[1], A.G.mn[1], A.G.cell, A.G.g[1]);
    cx = cell_of(pc[2], A.G.mn[2], A.G.cell, A.G.g[2]);
  }
  for (int zz = max(cz - 1, 0); zz <= min(cz + 1, A.G.g[0] - 1); ++zz)
    for (int yy = max(cy - 1, 0); yy <= min(cy + 1, A.G.g[1] - 1); ++yy)
      for (int xx = max(cx - 1, 0); xx <= min(cx + 1, A.G.g[2] - 1); ++xx) {
        const int cell = (zz * A.G.g[1] + yy) * A.G.g[2] + xx;
        const unsigned int e = A.cell_start[cell + 1];
        for (unsigned int t = A.cell_start[cell]; t < e; ++t) {
          const int h = A.items[t];
          if (h >= c) continue;
          if (!f(h, pc)) return;
        }
      }
}

// counters: [0] undecided at round start, [1] heavy pairs emitted, [3] S3 pairs decided by the lower bound, [4] pair tests,
//           [5] S3, [6] S4, [7] S5 evaluations, [8] candidates kept in this round, [9] length of the undecided list written by
//           this round, [10] length of the list this round reads
// k_frontier is pull based over the COMPACTED list of undecided candidates (double buffered; round 0 reads the identity):
// a candidate without an undecided / just-kept neighbour of higher score that reaches it is kept and appended to kept_list.
__global__ void __launch_bounds__(256) k_frontier(Arr A, int round, const int* __restrict__ list_in, int n_all, int* __restrict__ list_out,
                                                  int* __restrict__ kept_list, int2* __restrict__ cursor, unsigned int* __restrict__ counters) {
  // one WARP per undecided candidate: the lanes test 32 items of a cell per step (a chain of dependent loads otherwise), and
  // the scan of the 27 cells RESUMES where it stopped in the previous round (cursor = cell 0..26, offset): an item that did
  // not block once -- index above c, decided, or out of reach -- never blocks later, so every neighbourhood is walked once
  // over all rounds.
  const unsigned int n_in = list_in ? counters[10] : (unsigned int)n_all;
  const unsigned int warps = (gridDim.x * blockDim.x) >> 5, lane = threadIdx.x & 31;
  const int kept_now = ST_KEPT_BASE + round;
  unsigned int n_und = 0;
  for (unsigned int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n_in; i += warps) {
    const int c = list_in ? list_in[i] : (int)i;
    if (A.state[c] != ST_UNDECIDED) continue;
    ++n_und;
    const float* pc = A.points + 3 * c;
    int cz = 0, cy = 0, cx = 0;
    if (!A.G.all_pairs) {
      cz = cell_of(pc[0], A.G.mn[0], A.G.cell, A.G.g[0]); cy = cell_of(pc[1], A.G.mn[1], A.G.cell, A.G.g[1]);
      cx = cell_of(pc[2], A.G.mn[2], A.G.cell, A.G.g[2]);
    }
    int2 cur = cursor[c];
    bool blocked = false;
    for (int k = cur.x; k < 27 && !blocked; ++k) {
      const int zz = cz + k / 9 - 1, yy = cy + (k / 3) % 3 - 1, xx = cx + k % 3 - 1;
      if (zz < 0 || zz >= A.G.g[0] || yy < 0 || yy >= A.G.g[1] || xx < 0 || xx >= A.G.g[2]) { cur.x = k + 1; cur.y = 0; continue; }
      const int cell = (zz * A.G.g[1] + yy) * A.G.g[2] + xx;
      const unsigned int b = A.cell_start[cell], e = A.cell_start[cell + 1];
      for (unsigned int t0 = b + (unsigned int)cur.y; t0 < e && !blocked; t0 += 32) {
        const unsigned int t = t0 + lane;
        bool hit = false;
        if (t < e) {
          const int h = A.items[t];
          if (h < c) {
            const int sh = A.state[h];
            if (sh == ST_UNDECIDED || sh == kept_now) hit = reaches(A, h, pc);
          }
        }
        const unsigned int m = __ballot_sync(0xffffffffu, hit);
        if (m) { blocked = true; cur.x = k; cur.y = (int)(t0 + (unsigned int)(__ffs(m) - 1) - b); }
      }
      if (!blocked) { cur.x = k + 1; cur.y = 0; }
    }
    if (lane == 0) {
      cursor[c] = cur;
      if (!blocked) { A.state[c] = kept_now; kept_list[atomicAdd(&counters[8], 1u)] = c; }
      else list_out[atomicAdd(&counters[9], 1u)] = c;
    }
  }
  if (lane == 0 && n_und) atomicAdd(&counters[0], n_und);
}

// S1 + S2 for every (h kept in this round, undecided c > h that h reaches); emits the pairs that need the heavy stages.
// Push based: one block per kept polyhedron walks its 27 cells once -- the work is (kept polyhedra) x (neighbourhood) over
// the whole run instead of (undecided candidates) x (neighbourhood) per round.
__global__ void __launch_bounds__(128) k_pretest(Arr A, int round, const int* __restrict__ kept_list, int2* __restrict__ pairs, unsigned int pair_cap,
                                                 unsigned int* __restrict__ counters) {
  const unsigned int n_kept = counters[8];
  const float an[3] = {A.aniso[0], A.aniso[1], A.aniso[2]};
  for (unsigned int w = blockIdx.x; w < n_kept; w += gridDim.x) {
    const int h = kept_list[w];
    const float* ph = A.points + 3 * h;
    const float rr = A.max_dist + A.r_outer[h];
    int cz = 0, cy = 0, cx = 0;
    if (!A.G.all_pairs) {
      cz = cell_of(ph[0], A.G.mn[0], A.G.cell, A.G.g[0]); cy = cell_of(ph[1], A.G.mn[1], A.G.cell, A.G.g[1]);
      cx = cell_of(ph[2], A.G.mn[2], A.G.cell, A.G.g[2]);
    }
    for (int zz = max(cz - 1, 0); zz <= min(cz + 1, A.G.g[0] - 1); ++zz)
      for (int yy = max(cy - 1, 0); yy <= min(cy + 1, A.G.g[1] - 1); ++yy)
        for (int xx = max(cx - 1, 0); xx <= min(cx + 1, A.G.g[2] - 1); ++xx) {
          const int cell = (zz * A.G.g[1] + yy) * A.G.g[2] + xx;
          const unsigned int e = A.cell_start[cell + 1];
          for (unsigned int t = A.cell_start[cell] + threadIdx.x; t < e; t += blockDim.x) {
            const int c = A.items[t];
            if (c <= h) continue;
            if (A.state[c] != ST_UNDECIDED) continue;
            const float* pc = A.points + 3 * c;
            if (!A.G.all_pairs) {
              const float d0 = ph[0] - pc[0], d1 = ph[1] - pc[1], d2 = ph[2] - pc[2];
              const float dd = d0 * d0 + d1 * d1 + d2 * d2;
              if (!(dd < rr * rr)) continue;                       // reaches(A, h, pc)
            }
            atomicAdd(&counters[4], 1u);
            const float A_min = fminf(A.volume[h], A.volume[c]);
            // S1 (:1213-1228)
            float A_inter = fminf(sd3::intersect_sphere_isotropic(A.r_outer_iso[h], ph, A.r_outer_iso[c], pc, an),
                                  sd3::intersect_bbox(A.bbox + 6 * h, A.bbox + 6 * c));
            float iou = (float)fmin(1.0, (double)A_inter / ((double)A_min + 1e-10));
            if (A.use_bbox && (((double)A_inter < 1.e-10) || (iou <= A.threshold))) continue;
            // S2 (:1232-1248)
            A_inter = sd3::intersect_sphere_isotropic(A.r_inner_iso[h], ph, A.r_inner_iso[c], pc, an);
            iou = (float)fmax(0.0, (double)A_inter / ((double)A_min + 1e-10));
            if (iou > A.threshold) { A.state[c] = ST_SUPPRESSED; continue; }
            const unsigned int k = atomicAdd(&counters[1], 1u);
            if (k < pair_cap) { int2 pr; pr.x = h; pr.y = c; pairs[k] = pr; }
          }
        }
  }
}

// ---- heavy stages: one CTA (128 threads) per pair ------------------------------------------
struct PlaneAt { const Plane* p; __device__ Plane operator()(int i) const { return p[i]; } };

__device__ __forceinline__ double block_sum(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  double s = 0;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += red[i];
  return s;
}

// warp-cooperative gift wrapping pivot: lanes scan the points, then a shuffle tournament
__device__ int warp_pivot(const double* pts, int n, int a, int b, int skip) {
  const int lane = threadIdx.x & 31;
  auto orient = [&](int p, int q, int r, int s) -> double {
    const double b0 = pts[3 * q] - pts[3 * p], b1 = pts[3 * q + 1] - pts[3 * p + 1], b2 = pts[3 * q + 2] - pts[3 * p + 2];
    const double c0 = pts[3 * r] - pts[3 * p], c1 = pts[3 * r + 1] - pts[3 * p + 1], c2 = pts[3 * r + 2] - pts[3 * p + 2];
    const double d0 = pts[3 * s] - pts[3 * p], d1 = pts[3 * s + 1] - pts[3 * p + 1], d2 = pts[3 * s + 2] - pts[3 * p + 2];
    return d0 * (b1 * c2 - b2 * c1) + d1 * (b2 * c0 - b0 * c2) + d2 * (b0 * c1 - b1 * c0);
  };
  int q = -1;
  for (int r = lane; r < n; r += 32) {
    if (r == a || r == b || r == skip) continue;
    if (q < 0) { q = r; continue; }
    if (orient(a, b, q, r) > 0) q = r;
  }
  for (int o = 16; o > 0; o >>= 1) {
    const int other = __shfl_xor_sync(0xffffffffu, q, o);
    int best = q;
    if (q < 0) best = other;
    else if (other >= 0 && other != q) {
      // deterministic tournament: both lanes evaluate the same comparison
      const int lo = min(q, other), hi = max(q, other);
      best = (orient(a, b, lo, hi) > 0) ? hi : lo;
    }
    q = best;
  }
  return q;
}

// hull facet planes by warp 0 (other warps idle); identical facet set to sd3::convex_hull_planes up to order
__device__ int hull_planes_warp(double* pts, int n, Plane* out, int max_planes, uint32_t* edge_done, int16_t* stack, int max_stack, int dedup) {
  const int lane = threadIdx.x & 31;
  if (dedup) {      // warp-uniform; only for ray sets with coincident directions: repeated points go to the centroid (geom3d.cuh)
    if (lane == 0) sd3::demote_duplicate_points(pts, n);
    __syncwarp();
  }
  for (int i = lane; i < (n * n + 31) / 32; i += 32) edge_done[i] = 0;
  __syncwarp();
  // start edge (serial scan by every lane redundantly: cheap, n <= 256)
  int p0 = 0;
  for (int i = 1; i < n; ++i)
    if (pts[3 * i] < pts[3 * p0] || (pts[3 * i] == pts[3 * p0] && (pts[3 * i + 1] < pts[3 * p0 + 1] ||
        (pts[3 * i + 1] == pts[3 * p0 + 1] && pts[3 * i + 2] < pts[3 * p0 + 2])))) p0 = i;
  int p1 = -1;
  for (int i = 0; i < n; ++i) {
    if (i == p0) continue;
    if (p1 < 0) { p1 = i; continue; }
    const double ax = pts[3 * p1] - pts[3 * p0], ay = pts[3 * p1 + 1] - pts[3 * p0 + 1];
    const double bx = pts[3 * i] - pts[3 * p0], by = pts[3 * i + 1] - pts[3 * p0 + 1];
    const double cr = ax * by - ay * bx;
    if (cr < 0 || (cr == 0 && (bx * bx + by * by) > (ax * ax + ay * ay))) p1 = i;
  }
  if (p1 < 0) return -1;
  int p2 = warp_pivot(pts, n, p0, p1, -1);
  if (p2 < 0) return -1;
  int nf = 0, sp = 0;
  auto done = [&](int a, int b) -> bool { const int e = a * n + b; return (edge_done[e >> 5] >> (e & 31)) & 1u; };
  auto emit = [&](int a, int b, int c) -> bool {
    if (nf >= max_planes) return false;
    if (lane == 0) {
      const double b0 = pts[3 * b] - pts[3 * a], b1 = pts[3 * b + 1] - pts[3 * a + 1], b2 = pts[3 * b + 2] - pts[3 * a + 2];
      const double c0 = pts[3 * c] - pts[3 * a], c1 = pts[3 * c + 1] - pts[3 * a + 1], c2 = pts[3 * c + 2] - pts[3 * a + 2];
      double n0 = b1 * c2 - b2 * c1, n1 = b2 * c0 - b0 * c2, n2 = b0 * c1 - b1 * c0;
      const double l = sqrt(n0 * n0 + n1 * n1 + n2 * n2);
      if (l > 0) { n0 /= l; n1 /= l; n2 /= l; }
      Plane P; P.n0 = n0; P.n1 = n1; P.n2 = n2; P.d = -(n0 * pts[3 * a] + n1 * pts[3 * a + 1] + n2 * pts[3 * a + 2]);
      out[nf] = P;
      int e;
      e = a * n + b; edge_done[e >> 5] |= (1u << (e & 31));
      e = b * n + c; edge_done[e >> 5] |= (1u << (e & 31));
      e = c * n + a; edge_done[e >> 5] |= (1u << (e & 31));
    }
    nf++;
    __syncwarp();
    return true;
  };
  auto push = [&](int a, int b, int c) {
    if (sp < max_stack) { if (lane == 0) { stack[3 * sp] = (int16_t)a; stack[3 * sp + 1] = (int16_t)b; stack[3 * sp + 2] = (int16_t)c; } sp++; }
  };
  if (!emit(p0, p1, p2)) return -1;
  push(p1, p0, p2); push(p2, p1, p0); push(p0, p2, p1);
  __syncwarp();
  int guard = 0;
  while (sp > 0) {
    if (++guard > 16 * n + 64) return -1;
    --sp;
    const int a = stack[3 * sp], b = stack[3 * sp + 1], opp = stack[3 * sp + 2];
    __syncwarp();
    if (done(a, b)) continue;
    const int q = warp_pivot(pts, n, a, b, opp);
    if (q < 0) return -1;
    if (!emit(a, b, q)) return -1;
    if (!done(q, b)) push(q, b, a);
    if (!done(a, q)) push(a, q, b);
    __syncwarp();
  }
  return nf;
}

// Rigorous two-sided bounds of the volume of the convex polytope {x : planes[j](x) <= 0, j < np} around an interior point p,
// from the ray triangulation of the model (directions v_k = A.verts[k], faces A.faces):
//   lower: the tetrahedra (p, p + t_a v_a, p + t_b v_b, p + t_c v_c), t_k = distance to the first plane along v_k, lie inside;
//   upper: the polytope's part inside the cone over a face lies below EVERY plane of the polytope, in particular below each
//          of the (up to three) planes that stop the face's rays; below plane j the cone is the tetrahedron with the
//          ray-plane distances t^j_a, t^j_b, t^j_c -- the smallest of the three bounds that part.
// The cones tile space when every face determinant det(v_a, v_b, v_c) is positive (checked; otherwise upper = +inf).
// ~2F*R plane-ray products instead of ~(2F)^2 polygon clips.  scratch: 3R doubles (tmin) + R ints (first plane) in shared memory.
__device__ void fan_bounds(const Arr& A, const Plane* planes, int np, const double* p, double Lext, const int* sfaces,
                           double* tmin, int* jhit, double* red, double* lower, double* upper, double* tm = nullptr, int* jm = nullptr) {
  // tm / jm (F entries each, optional): one extra ray per face along v_a + v_b + v_c; every face cone is then split into the
  // three sub-cones (a,b,m), (b,c,m), (c,a,m) -- same construction, finer fan, bounds a few times tighter
  const int G = 3;
  __syncthreads();
  const int n_ray_jobs = G * A.R, n_jobs = n_ray_jobs + (tm ? A.F : 0);
  for (int idx = threadIdx.x; idx < n_jobs; idx += blockDim.x) {       // (the job count exceeds the block for large R / F)
    double v0, v1, v2; int j0, jstep;
    if (idx < n_ray_jobs) {
      const int k = idx % A.R;
      v0 = (double)A.verts[3 * k]; v1 = (double)A.verts[3 * k + 1]; v2 = (double)A.verts[3 * k + 2];
      j0 = idx / A.R; jstep = G;
    } else {
      const int f = idx - n_ray_jobs, ia = sfaces[3 * f], ib = sfaces[3 * f + 1], ic = sfaces[3 * f + 2];
      v0 = (double)A.verts[3 * ia] + (double)A.verts[3 * ib] + (double)A.verts[3 * ic];
      v1 = (double)A.verts[3 * ia + 1] + (double)A.verts[3 * ib + 1] + (double)A.verts[3 * ic + 1];
      v2 = (double)A.verts[3 * ia + 2] + (double)A.verts[3 * ib + 2] + (double)A.verts[3 * ic + 2];
      j0 = 0; jstep = 1;
    }
    double tn = Lext, td = 1.0; int jb = -1;        // running minimum of sd / a as a fraction (no division per plane)
    for (int j = j0; j < np; j += jstep) {
      const Plane P = planes[j];
      const double a = P.n0 * v0 + P.n1 * v1 + P.n2 * v2;
      if (a > 0) {
        const double sd = -(P.d + P.n0 * p[0] + P.n1 * p[1] + P.n2 * p[2]);
        if (sd * td < tn * a) { tn = sd; td = a; jb = j; }
      }
    }
    if (idx < n_ray_jobs) { tmin[idx] = tn / td; jhit[idx] = jb; }
    else { tm[idx - n_ray_jobs] = tn / td; jm[idx - n_ray_jobs] = jb; }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < A.R; k += blockDim.x) {
    double t = tmin[k]; int jb = jhit[k];
    for (int g = 1; g < G; ++g) if (tmin[g * A.R + k] < t) { t = tmin[g * A.R + k]; jb = jhit[g * A.R + k]; }
    tmin[k] = t; jhit[k] = jb;
  }
  __syncthreads();
  double pl = 0, pu = 0; int bad = 0;
  // det of the tetrahedron_volume0 orientation: M = (B - A, C - A, -A)
  auto det3v = [](const double* Av, double ta, const double* Bv, double tb, const double* Cv, double tc) {
    const double Az = ta * Av[0], Ay = ta * Av[1], Ax = ta * Av[2], Bz = tb * Bv[0], By = tb * Bv[1], Bx = tb * Bv[2], Cz = tc * Cv[0], Cy = tc * Cv[1], Cx = tc * Cv[2];
    const double M00 = Bz - Az, M01 = By - Ay, M02 = Bx - Ax, M10 = Cz - Az, M11 = Cy - Ay, M12 = Cx - Ax, M20 = -Az, M21 = -Ay, M22 = -Ax;
    return M00 * (M11 * M22 - M21 * M12) - M01 * (M10 * M22 - M12 * M20) + M02 * (M10 * M21 - M11 * M20);
  };
  // lower / upper contribution of the cone over (A, B, C) with first-plane distances tA.. and stopping planes jA..
  auto cone = [&](const double* Av, double tA, int jA, const double* Bv, double tB, int jB, const double* Cv, double tC, int jC, double* lo, double* up) -> bool {
    if (!(det3v(Av, 1.0, Bv, 1.0, Cv, 1.0) > 0)) return false;
    const double l = det3v(Av, tA, Bv, tB, Cv, tC);
    *lo += l > 0 ? l : 0.0;
    double u = 1e300;
    const int js[3] = {jA, jB, jC};
#pragma unroll
    for (int e = 0; e < 3; ++e) {
      const int j = js[e];
      if (j < 0) continue;
      const Plane P = planes[j];
      const double sd = -(P.d + P.n0 * p[0] + P.n1 * p[1] + P.n2 * p[2]);
      const double qa = P.n0 * Av[0] + P.n1 * Av[1] + P.n2 * Av[2], qb = P.n0 * Bv[0] + P.n1 * Bv[1] + P.n2 * Bv[2], qc = P.n0 * Cv[0] + P.n1 * Cv[1] + P.n2 * Cv[2];
      if (qa > 0 && qb > 0 && qc > 0) u = fmin(u, det3v(Av, sd / qa, Bv, sd / qb, Cv, sd / qc));
    }
    if (u >= 1e299) return false;
    *up += u;
    return true;
  };
  for (int f = threadIdx.x; f < A.F; f += blockDim.x) {
    const int ia = sfaces[3 * f], ib = sfaces[3 * f + 1], ic = sfaces[3 * f + 2];
    const double va[3] = {A.verts[3 * ia], A.verts[3 * ia + 1], A.verts[3 * ia + 2]};
    const double vb[3] = {A.verts[3 * ib], A.verts[3 * ib + 1], A.verts[3 * ib + 2]};
    const double vc[3] = {A.verts[3 * ic], A.verts[3 * ic + 1], A.verts[3 * ic + 2]};
    if (!(det3v(va, 1.0, vb, 1.0, vc, 1.0) > 0)) { bad = 1; continue; }
    bool ok;
    if (tm) {
      const double vm[3] = {va[0] + vb[0] + vc[0], va[1] + vb[1] + vc[1], va[2] + vb[2] + vc[2]};
      const double t_m = tm[f]; const int j_m = jm[f];
      ok = cone(va, tmin[ia], jhit[ia], vb, tmin[ib], jhit[ib], vm, t_m, j_m, &pl, &pu);
      ok = cone(vb, tmin[ib], jhit[ib], vc, tmin[ic], jhit[ic], vm, t_m, j_m, &pl, &pu) && ok;
      ok = cone(vc, tmin[ic], jhit[ic], va, tmin[ia], jhit[ia], vm, t_m, j_m, &pl, &pu) && ok;
    } else {
      ok = cone(va, tmin[ia], jhit[ia], vb, tmin[ib], jhit[ib], vc, tmin[ic], jhit[ic], &pl, &pu);
    }
    if (!ok) bad = 1;
  }
  bad = __syncthreads_or(bad);
  const double sl = block_sum(pl, red);
  const double su = block_sum(pu, red);
  *lower = sl / 6.0;
  *upper = bad ? 1e300 : su / 6.0;
}

struct HeavyCtx {
  int stage; int2* list4; int* slot; int* uniq; Plane* hull_planes; int* hull_n; int hull_cap;
  sdbins::FaceBins bins;      // direction bins of the ray triangulation for the S5 rendering (count == nullptr: all faces)
};

// hull facet planes of the polyhedra registered by the S3 launch: ONE WARP per polyhedron (gift wrapping is a serial chain of
// pivots; 4 warps per block, each with its own points / edge bit map / stack in shared memory)
__global__ void __launch_bounds__(128) k_hulls(Arr A, HeavyCtx X, const unsigned int* __restrict__ counters) {
  extern __shared__ __align__(16) unsigned char hsm[];
  const int wpb = blockDim.x >> 5, wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t per_warp = (size_t)3 * A.R * sizeof(double) + (size_t)((A.R * A.R + 31) / 32) * 4 + (size_t)3 * 4 * A.R * 2 + 16;
  unsigned char* base = hsm + (size_t)wid * ((per_warp + 15) / 16 * 16);
  double* pts = reinterpret_cast<double*>(base);
  uint32_t* edge_done = reinterpret_cast<uint32_t*>(base + (size_t)3 * A.R * sizeof(double));
  int16_t* stack = reinterpret_cast<int16_t*>(base + (size_t)3 * A.R * sizeof(double) + (size_t)((A.R * A.R + 31) / 32) * 4);
  const unsigned int n_uniq = min(counters[12], (unsigned int)X.hull_cap);
  for (unsigned int u = blockIdx.x * wpb + wid; u < n_uniq; u += gridDim.x * wpb) {
    const int i = X.uniq[u];
    const float* d = A.dist + (size_t)i * A.R;
    const float c0 = A.points[3 * i], c1 = A.points[3 * i + 1], c2 = A.points[3 * i + 2];
    __syncwarp();
    for (int j = lane; j < A.R; j += 32) {
      pts[3 * j] = (double)(c0 + d[j] * A.verts[3 * j]);
      pts[3 * j + 1] = (double)(c1 + d[j] * A.verts[3 * j + 1]);
      pts[3 * j + 2] = (double)(c2 + d[j] * A.verts[3 * j + 2]);
    }
    __syncwarp();
    const int nf = hull_planes_warp(pts, A.R, X.hull_planes + (size_t)u * A.F, A.F, edge_done, stack, 4 * A.R, A.dup_dirs);
    if (lane == 0) X.hull_n[u] = nf;
    __syncwarp();
  }
}

// Stage S3 lower bound, ONE WARP per pair (the first of the three launches of a round).  The work of a pair is small (2F
// planes, R rays x 2F plane-ray products, F tetrahedra) and a CTA per pair spent it mostly in block-wide barriers: 46 us per
// pair, 41 ms per bench volume; a warp needs no barrier.  Any valid lower bound decides correctly (the summation order of the
// fan volume differs from the block-wide version by ulps; the 1e-5 margin covers it): decided pairs are suppressed, the rest
// go to X.list4 and their polyhedra are registered for k_hulls -- exactly what k_heavy's stage 1 does.
__global__ void __launch_bounds__(256) k_s3_bound_warp(Arr A, const int2* __restrict__ pairs, unsigned int* __restrict__ counters, unsigned int pair_cap,
                                                       HeavyCtx X, int warps_per_block) {
  extern __shared__ __align__(16) unsigned char wsm[];
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (wid >= warps_per_block) return;
  const size_t per_warp = (((size_t)2 * A.F * sizeof(Plane) + (size_t)A.R * sizeof(double) + (size_t)6 * A.R * sizeof(float)) + 15) / 16 * 16;
  unsigned char* base = wsm + (size_t)wid * per_warp;
  Plane* planes = reinterpret_cast<Plane*>(base);                               // [2F]
  double* tmin = reinterpret_cast<double*>(base + (size_t)2 * A.F * sizeof(Plane));      // [R]
  float* pv1 = reinterpret_cast<float*>(base + (size_t)2 * A.F * sizeof(Plane) + (size_t)A.R * sizeof(double));   // [R][3]
  float* pv2 = pv1 + 3 * A.R;
  const unsigned int n_pairs = min(counters[1], pair_cap);
  const int np = 2 * A.F;
  for (;;) {
    unsigned int pi = 0;
    if (lane == 0) pi = atomicAdd(&counters[14], 1u);
    pi = __shfl_sync(0xffffffffu, pi, 0);
    if (pi >= n_pairs) break;
    const int h = pairs[pi].x, c = pairs[pi].y;
    if (A.state[c] == ST_SUPPRESSED) continue;                        // (warp-uniform)
    const float c1[3] = {A.points[3 * h], A.points[3 * h + 1], A.points[3 * h + 2]};
    const float c2[3] = {A.points[3 * c], A.points[3 * c + 1], A.points[3 * c + 2]};
    const float* d1 = A.dist + (size_t)h * A.R; const float* d2 = A.dist + (size_t)c * A.R;
    __syncwarp();
    for (int j = lane; j < A.R; j += 32)
      for (int k = 0; k < 3; ++k) {
        pv1[3 * j + k] = c1[k] + d1[j] * A.verts[3 * j + k];
        pv2[3 * j + k] = c2[k] + d2[j] * A.verts[3 * j + k];
      }
    __syncwarp();
    if (lane == 0) atomicAdd(&counters[5], 1u);
    for (int f = lane; f < A.F; f += 32) {
      const int ia = A.faces[3 * f], ib = A.faces[3 * f + 1], ic = A.faces[3 * f + 2];
      double hs[4];
      sd3::build_halfspace(&pv1[3 * ia], &pv1[3 * ib], &pv1[3 * ic], hs);
      Plane P; P.n0 = hs[0]; P.n1 = hs[1]; P.n2 = hs[2]; P.d = hs[3]; planes[2 * f] = P;
      sd3::build_halfspace(&pv2[3 * ia], &pv2[3 * ib], &pv2[3 * ic], hs);
      P.n0 = hs[0]; P.n1 = hs[1]; P.n2 = hs[2]; P.d = hs[3]; planes[2 * f + 1] = P;
    }
    __syncwarp();
    double p[3];
    for (int k = 0; k < 3; ++k) p[k] = .5 * (double)(c1[k] + c2[k]);
    bool decided = false;
    if (A.s3_bound) {
      int infeasible = 0;
      for (int k = lane; k < np; k += 32) if (!sd3::plane_feasible(planes[k], p)) infeasible = 1;
      infeasible = __any_sync(0xffffffffu, infeasible);
      if (!infeasible) {
        double m = 0;
        for (int k = lane; k < 3 * A.R; k += 32) { m = fmax(m, fabs((double)pv1[k] - p[k % 3])); m = fmax(m, fabs((double)pv2[k] - p[k % 3])); }
        for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
        const double L = 4.0 * m + 1.0;
        for (int k = lane; k < A.R; k += 32) {
          const double v0 = (double)A.verts[3 * k], v1 = (double)A.verts[3 * k + 1], v2 = (double)A.verts[3 * k + 2];
          // min over the planes of sd / a (both positive) kept as a fraction: one fp64 division per ray instead of one per
          // plane (the divisions were ~80 % of this kernel)
          double tn = L, td = 1.0;
          for (int j = 0; j < np; ++j) {
            const Plane P = planes[j];
            const double a = P.n0 * v0 + P.n1 * v1 + P.n2 * v2;
            if (a > 0) {
              const double sd = -(P.d + P.n0 * p[0] + P.n1 * p[1] + P.n2 * p[2]);
              if (sd * td < tn * a) { tn = sd; td = a; }
            }
          }
          tmin[k] = tn / td;
        }
        __syncwarp();
        double part = 0;
        for (int f = lane; f < A.F; f += 32) {
          const int ia = A.faces[3 * f], ib = A.faces[3 * f + 1], ic = A.faces[3 * f + 2];
          const double ta = tmin[ia], tb = tmin[ib], tc = tmin[ic];
          const double Az = ta * A.verts[3 * ia], Ay = ta * A.verts[3 * ia + 1], Ax = ta * A.verts[3 * ia + 2];
          const double Bz = tb * A.verts[3 * ib], By = tb * A.verts[3 * ib + 1], Bx = tb * A.verts[3 * ib + 2];
          const double Cz = tc * A.verts[3 * ic], Cy = tc * A.verts[3 * ic + 1], Cx = tc * A.verts[3 * ic + 2];
          const double M00 = Bz - Az, M01 = By - Ay, M02 = Bx - Ax, M10 = Cz - Az, M11 = Cy - Ay, M12 = Cx - Ax, M20 = -Az, M21 = -Ay, M22 = -Ax;
          const double det = M00 * (M11 * M22 - M21 * M12) - M01 * (M10 * M22 - M12 * M20) + M02 * (M10 * M21 - M11 * M20);
          if (det > 0) part += det;
        }
        for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
        const double den = (double)fminf(A.volume[h], A.volume[c]) + 1e-10;
        if (part / 6.0 > (double)A.threshold * den * (1.0 + 1e-5)) {
          decided = true;
          if (lane == 0) { A.state[c] = ST_SUPPRESSED; atomicAdd(&counters[3], 1u); }
        }
      }
    }
    if (!decided && lane == 0) {
      const unsigned int q = atomicAdd(&counters[11], 1u);
      if (q < pair_cap) X.list4[q] = pairs[pi];
      const int two[2] = {h, c};
      for (int e = 0; e < 2; ++e) {
        const int i = two[e];
        if (atomicCAS(&X.slot[i], -1, -2) == -1) {
          const unsigned int u = atomicAdd(&counters[12], 1u);
          if (u < (unsigned int)X.hull_cap) { X.uniq[u] = i; X.slot[i] = (int)u; } else X.slot[i] = -3;
        }
      }
    }
  }
}

__global__ void __launch_bounds__(512)
k_heavy(Arr A, const int2* __restrict__ pairs, unsigned int* __restrict__ counters, unsigned int pair_cap, HeavyCtx X) {
  // X.stage 0: all stages for the pairs of k_pretest (single launch);  1: S3 only, the pairs it leaves open go to X.list4 and
  // their polyhedra are registered for k_hulls;  2: S4 + S5 for X.list4 with the hull facets k_hulls computed (one warp per
  // polyhedron, all warps of the device busy -- inside this kernel the gift wrapping occupies 1 warp of 16)
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int stage = X.stage;
  if (stage == 2) pairs = X.list4;
  const unsigned int n_pairs = stage == 2 ? min(counters[11], pair_cap) : min(counters[1], pair_cap);
  float* pv1 = reinterpret_cast<float*>(smem_raw);                 // [R][3]
  float* pv2 = pv1 + 3 * A.R;
  int* sfaces = reinterpret_cast<int*>(pv2 + 3 * A.R);             // [F][3]
  size_t off = ((size_t)(6 * A.R + 3 * A.F) * 4 + 15) / 16 * 16;
  Plane* planes = reinterpret_cast<Plane*>(smem_raw + off);        // [2F]
  off += (size_t)2 * A.F * sizeof(Plane);
  double* pts = reinterpret_cast<double*>(smem_raw + off);         // [R][3] (hull stage)
  off += (size_t)3 * A.R * sizeof(double);
  uint32_t* edge_done = reinterpret_cast<uint32_t*>(smem_raw + off);
  off += (size_t)((A.R * A.R + 31) / 32) * 4;
  int16_t* stack = reinterpret_cast<int16_t*>(smem_raw + off);     // [3*4R]
  off = (off + (size_t)3 * 4 * A.R * 2 + 15) / 16 * 16;
  double* fan_tm = reinterpret_cast<double*>(smem_raw + off);      // [F] face-centroid rays of the refined fan bounds
  int* fan_jm = reinterpret_cast<int*>(smem_raw + off + (size_t)A.F * sizeof(double));   // [F]
  __shared__ double red[16];          // one slot per warp (up to 512 threads)
  __shared__ int sh_i[4];
  __shared__ int sh_cnt;              // S5: running count of voxels inside both polyhedra
  __shared__ float c1[3], c2[3];
  for (int j = threadIdx.x; j < 3 * A.F; j += blockDim.x) sfaces[j] = A.faces[j];

  // pairs are handed out one at a time (atomic ticket): the expensive ones -- a few per cent -- would otherwise pile up in
  // whichever CTAs a static stride gives them to, and the slowest CTA sets the length of the round
  __shared__ unsigned int sh_pi;
  for (;;) {
    __syncthreads();
    if (threadIdx.x == 0) sh_pi = atomicAdd(&counters[stage == 2 ? 15 : 14], 1u);
    __syncthreads();
    const unsigned int pi = sh_pi;
    if (pi >= n_pairs) break;
    const int h = pairs[pi].x, c = pairs[pi].y;
    __syncthreads();
    if (threadIdx.x == 0) sh_i[2] = A.state[c];
    __syncthreads();
    if (sh_i[2] == ST_SUPPRESSED) continue;             // another pair already suppressed c (uniform per block)
    if (threadIdx.x < 3) { c1[threadIdx.x] = A.points[3 * h + threadIdx.x]; c2[threadIdx.x] = A.points[3 * c + threadIdx.x]; }
    __syncthreads();
    const float* d1 = A.dist + (size_t)h * A.R; const float* d2 = A.dist + (size_t)c * A.R;
    for (int j = threadIdx.x; j < A.R; j += blockDim.x)
      for (int k = 0; k < 3; ++k) {
        pv1[3 * j + k] = c1[k] + d1[j] * A.verts[3 * j + k];
        pv2[3 * j + k] = c2[k] + d2[j] * A.verts[3 * j + k];
      }
    __syncthreads();
    const float A_min = fminf(A.volume[h], A.volume[c]);
    const double den = (double)A_min + 1e-10;
    double p[3];
    for (int k = 0; k < 3; ++k) p[k] = .5 * (double)(c1[k] + c2[k]);
    int np = 2 * A.F;
    double L = 0;
    {
      double m = 0;
      for (int k = threadIdx.x; k < 3 * A.R; k += blockDim.x) {
        m = fmax(m, fabs((double)pv1[k] - p[k % 3])); m = fmax(m, fabs((double)pv2[k] - p[k % 3]));
      }
      for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
      __syncthreads();
      if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
      __syncthreads();
      m = 0;
      for (int i = 0; i < (int)(blockDim.x >> 5); ++i) m = fmax(m, red[i]);
      L = 4.0 * m + 1.0;
    }
    float iou = 0.f;
    if (stage != 2) {
    atomicAdd(&counters[5], threadIdx.x == 0 ? 1u : 0u);

    // ---- S3: kernel ∩ kernel (:1261-1277) ------------------------------------------------
    for (int f = threadIdx.x; f < A.F; f += blockDim.x) {
      double hs[4];
      sd3::build_halfspace(&pv1[3 * sfaces[3 * f]], &pv1[3 * sfaces[3 * f + 1]], &pv1[3 * sfaces[3 * f + 2]], hs);
      Plane P; P.n0 = hs[0]; P.n1 = hs[1]; P.n2 = hs[2]; P.d = hs[3]; planes[2 * f] = P;
      sd3::build_halfspace(&pv2[3 * sfaces[3 * f]], &pv2[3 * sfaces[3 * f + 1]], &pv2[3 * sfaces[3 * f + 2]], hs);
      P.n0 = hs[0]; P.n1 = hs[1]; P.n2 = hs[2]; P.d = hs[3]; planes[2 * f + 1] = P;
    }
    __syncthreads();
    int infeasible = 0;
    for (int k = threadIdx.x; k < np; k += blockDim.x) if (!sd3::plane_feasible(planes[k], p)) infeasible = 1;
    infeasible = __syncthreads_or(infeasible);
    float vol_kernel = 0.f;
    // ---- S3 short cut: a rigorous LOWER bound of vol(kernel_h ∩ kernel_c) that is ~80x cheaper than the volume itself.
    // Both kernels are convex and contain the midpoint p (feasibility above), so for every ray direction v_k the point
    // p + t_k v_k, t_k = distance from p to the nearest of the 2F planes along v_k, lies in the intersection, and so does
    // every tetrahedron (p, p+t_a v_a, p+t_b v_b, p+t_c v_c) of the ray triangulation; the cones over the faces tile space,
    // so the tetrahedra do not overlap and  L_low = sum_f det(t_a v_a, t_b v_b, t_c v_c)/6  <=  vol(intersection).
    // If L_low already exceeds threshold * (A_min + 1e-10) by a 1e-5 relative margin (the volume stage is accurate to
    // ~1e-12, its float rounding to 6e-8), the reference's test `iou > threshold` (:1270-1277) is decided: suppress.
    // Near-duplicate candidates of one object -- the bulk of the pairs that reach this stage -- end here.
    if (!infeasible && A.s3_bound) {
      const int G = 3;                                   // pts holds 3R doubles: G partial minima per ray
      double* tmin = pts;
      __syncthreads();
      for (int idx = threadIdx.x; idx < G * A.R; idx += blockDim.x) {     // (G*R exceeds the block for R > 170)
        const int g = idx / A.R, k = idx % A.R;
        const double v0 = (double)A.verts[3 * k], v1 = (double)A.verts[3 * k + 1], v2 = (double)A.verts[3 * k + 2];
        double t = L;                                    // extent bound of the polytope around p (never binding for closed kernels)
        for (int j = g; j < np; j += G) {
          const Plane P = planes[j];
          const double a = P.n0 * v0 + P.n1 * v1 + P.n2 * v2;
          if (a > 0) {
            const double sd = -(P.d + P.n0 * p[0] + P.n1 * p[1] + P.n2 * p[2]);     // > 0 (feasible)
            t = fmin(t, sd / a);
          }
        }
        tmin[g * A.R + k] = t;
      }
      __syncthreads();
      for (int k = threadIdx.x; k < A.R; k += blockDim.x) tmin[k] = fmin(tmin[k], fmin(tmin[A.R + k], tmin[2 * A.R + k]));
      __syncthreads();
      double partl = 0;
      for (int f = threadIdx.x; f < A.F; f += blockDim.x) {
        const int ia = sfaces[3 * f], ib = sfaces[3 * f + 1], ic = sfaces[3 * f + 2];
        const double ta = tmin[ia], tb = tmin[ib], tc = tmin[ic];
        const double Az = ta * A.verts[3 * ia], Ay = ta * A.verts[3 * ia + 1], Ax = ta * A.verts[3 * ia + 2];
        const double Bz = tb * A.verts[3 * ib], By = tb * A.verts[3 * ib + 1], Bx = tb * A.verts[3 * ib + 2];
        const double Cz = tc * A.verts[3 * ic], Cy = tc * A.verts[3 * ic + 1], Cx = tc * A.verts[3 * ic + 2];
        // orientation of tetrahedron_volume0 (positive for the ray faces, as in polyhedron_volume)
        const double M00 = Bz - Az, M01 = By - Ay, M02 = Bx - Ax, M10 = Cz - Az, M11 = Cy - Ay, M12 = Cx - Ax, M20 = -Az, M21 = -Ay, M22 = -Ax;
        const double det = M00 * (M11 * M22 - M21 * M12) - M01 * (M10 * M22 - M12 * M20) + M02 * (M10 * M21 - M11 * M20);
        if (det > 0) partl += det;
      }
      const double L_low = block_sum(partl, red) / 6.0;
      if (L_low > (double)A.threshold * den * (1.0 + 1e-5)) {
        if (threadIdx.x == 0) { A.state[c] = ST_SUPPRESSED; atomicAdd(&counters[3], 1u); }
        continue;
      }
    }
    if (!infeasible && stage == 0) {
      PlaneAt PA{planes};
      double part = 0; int ovf = 0;
      if (A.norm_planes) {
        // (block-uniform branch) scale every plane once instead of once per (k, j) pair
        for (int k = threadIdx.x; k < np; k += blockDim.x) planes[k] = sd3::normalized_plane(planes[k]);
        __syncthreads();
        for (int k = threadIdx.x; k < np; k += blockDim.x) part += sd3::face_cone_volume_n(PA, np, k, p, L, &ovf);
      } else {
        for (int k = threadIdx.x; k < np; k += blockDim.x) part += sd3::face_cone_volume(PA, np, k, p, L, &ovf);
      }
      vol_kernel = (float)block_sum(part, red);     // NOTE: summation order differs from the serial host version (ulp-level in double)
    }
    iou = (float)((double)vol_kernel / den);
    if (iou > A.threshold) { if (threadIdx.x == 0) A.state[c] = ST_SUPPRESSED; continue; }
    if (stage == 1) {
      // not decided by the lower bound: hand the pair to the second launch (S4, then the S3 volume only if S4 leaves the pair
      // open) and register both polyhedra for the hull kernel (once per round)
      if (threadIdx.x == 0) {
        const unsigned int q = atomicAdd(&counters[11], 1u);
        if (q < pair_cap) X.list4[q] = pairs[pi];
        const int two[2] = {h, c};
        for (int e = 0; e < 2; ++e) {
          const int i = two[e];
          if (atomicCAS(&X.slot[i], -1, -2) == -1) {
            const unsigned int u = atomicAdd(&counters[12], 1u);
            if (u < (unsigned int)X.hull_cap) { X.uniq[u] = i; X.slot[i] = (int)u; } else X.slot[i] = -3;      // -3: no room, hull inside the CTA
          }
        }
      }
      continue;
    }
    }   // stage != 2

    // ---- S4: hull ∩ hull (:1282-1295) -----------------------------------------------------
    atomicAdd(&counters[6], threadIdx.x == 0 ? 1u : 0u);
    float vol_convex = 1.e10f;
    {
      int n1 = -1, n2 = -1;
      __syncthreads();
      const int s1 = stage == 2 ? X.slot[h] : -1, s2 = stage == 2 ? X.slot[c] : -1;
      if (s1 >= 0 && s2 >= 0) {
        // facets from k_hulls (same routine, same numbers as the in-CTA gift wrapping below)
        n1 = X.hull_n[s1]; n2 = X.hull_n[s2];
        if (n1 >= 4 && n2 >= 4) {
          for (int k = threadIdx.x; k < n1; k += blockDim.x) planes[k] = X.hull_planes[(size_t)s1 * A.F + k];
          for (int k = threadIdx.x; k < n2; k += blockDim.x) planes[n1 + k] = X.hull_planes[(size_t)s2 * A.F + k];
        }
        __syncthreads();
      } else {
      for (int k = threadIdx.x; k < 3 * A.R; k += blockDim.x) pts[k] = (double)pv1[k];
      __syncthreads();
      if (threadIdx.x < 32) { n1 = hull_planes_warp(pts, A.R, planes, A.F, edge_done, stack, 4 * A.R, A.dup_dirs); if (threadIdx.x == 0) sh_i[0] = n1; }
      __syncthreads();
      n1 = sh_i[0];
      if (n1 >= 4) {
        for (int k = threadIdx.x; k < 3 * A.R; k += blockDim.x) pts[k] = (double)pv2[k];
        __syncthreads();
        if (threadIdx.x < 32) { n2 = hull_planes_warp(pts, A.R, planes + n1, A.F, edge_done, stack, 4 * A.R, A.dup_dirs); if (threadIdx.x == 0) sh_i[1] = n2; }
        __syncthreads();
        n2 = sh_i[1];
      }
      }
      if (n1 >= 4 && n2 >= 4) {
        np = n1 + n2;
        for (int k = 0; k < 3; ++k) p[k] = .5 * ((double)c1[k] + (double)c2[k]);
        int inf2 = 0;
        for (int k = threadIdx.x; k < np; k += blockDim.x) if (!sd3::plane_feasible(planes[k], p)) inf2 = 1;
        inf2 = __syncthreads_or(inf2);
        int decided4 = 0;
        if (!inf2 && stage == 2 && A.s3_bound) {
          // two-sided fan bounds decide `iou_hull <= t` / `> t` for all but the pairs within a few per cent of the threshold
          double lo4, up4;
          fan_bounds(A, planes, np, p, L, sfaces, pts, reinterpret_cast<int*>(edge_done), red, &lo4, &up4, A.fan_subdiv ? fan_tm : nullptr, fan_jm);
          const double tden = (double)A.threshold * den;
          if (up4 * (1.0 + 1e-5) <= tden) { vol_convex = 0.f; decided4 = 1; }             // certainly <= t: the pair is kept (S4 exit)
          else if (lo4 > tden * (1.0 + 1e-5)) { vol_convex = 1.e10f; decided4 = 1; }      // certainly > t (value itself is not used)
          if (decided4) atomicAdd(&counters[2], threadIdx.x == 0 ? 1u : 0u);
        }
        if (!inf2 && !decided4) {
          PlaneAt PA{planes};
          double part = 0; int ovf = 0;
          if (A.norm_planes) {
            for (int k = threadIdx.x; k < np; k += blockDim.x) planes[k] = sd3::normalized_plane(planes[k]);
            __syncthreads();
            for (int k = threadIdx.x; k < np; k += blockDim.x) part += sd3::face_cone_volume_n(PA, np, k, p, L, &ovf);
          } else {
            for (int k = threadIdx.x; k < np; k += blockDim.x) part += sd3::face_cone_volume(PA, np, k, p, L, &ovf);
          }
          vol_convex = (float)block_sum(part, red);
        }
      }
    }
    if (stage == 2) {
      // The reference evaluates S3 (suppress if iou_kernel > t) before S4 (keep if iou_hull <= t).  kernel_h ∩ kernel_c is a
      // subset of hull_h ∩ hull_c, so iou_hull <= t implies iou_kernel <= t: neither stage suppresses and the S3 volume --
      // as expensive as S4 -- is not needed.  (1e-4 relative margin against the independent roundings of the two stages;
      // the sentinel 1e10 of an infeasible hull midpoint never takes this exit.)  ~3/4 of the open pairs end here.
      if ((double)vol_convex * (1.0 + 1e-4) <= (double)A.threshold * den) continue;
      atomicAdd(&counters[13], threadIdx.x == 0 ? 1u : 0u);
      __syncthreads();
      for (int f = threadIdx.x; f < A.F; f += blockDim.x) {
        double hs[4];
        sd3::build_halfspace(&pv1[3 * sfaces[3 * f]], &pv1[3 * sfaces[3 * f + 1]], &pv1[3 * sfaces[3 * f + 2]], hs);
        Plane P; P.n0 = hs[0]; P.n1 = hs[1]; P.n2 = hs[2]; P.d = hs[3]; planes[2 * f] = P;
        sd3::build_halfspace(&pv2[3 * sfaces[3 * f]], &pv2[3 * sfaces[3 * f + 1]], &pv2[3 * sfaces[3 * f + 2]], hs);
        P.n0 = hs[0]; P.n1 = hs[1]; P.n2 = hs[2]; P.d = hs[3]; planes[2 * f + 1] = P;
      }
      __syncthreads();
      for (int k = 0; k < 3; ++k) p[k] = .5 * (double)(c1[k] + c2[k]);
      np = 2 * A.F;
      int infeasible = 0;
      for (int k = threadIdx.x; k < np; k += blockDim.x) if (!sd3::plane_feasible(planes[k], p)) infeasible = 1;
      infeasible = __syncthreads_or(infeasible);
      float vol_kernel = 0.f;
      int decided3 = 0;
      if (!infeasible && A.s3_bound) {
        double lo3, up3;
        fan_bounds(A, planes, np, p, L, sfaces, pts, reinterpret_cast<int*>(edge_done), red, &lo3, &up3, A.fan_subdiv ? fan_tm : nullptr, fan_jm);
        const double tden = (double)A.threshold * den;
        if (lo3 > tden * (1.0 + 1e-5)) { vol_kernel = 1.e30f; decided3 = 1; }             // certainly > t: suppressed at S3
        else if (up3 * (1.0 + 1e-5) <= tden) { vol_kernel = 0.f; decided3 = 1; }          // certainly <= t: S3 does not suppress
      }
      if (!infeasible && !decided3) {
        PlaneAt PA{planes};
        double part = 0; int ovf = 0;
        if (A.norm_planes) {
          for (int k = threadIdx.x; k < np; k += blockDim.x) planes[k] = sd3::normalized_plane(planes[k]);
          __syncthreads();
          for (int k = threadIdx.x; k < np; k += blockDim.x) part += sd3::face_cone_volume_n(PA, np, k, p, L, &ovf);
        } else {
          for (int k = threadIdx.x; k < np; k += blockDim.x) part += sd3::face_cone_volume(PA, np, k, p, L, &ovf);
        }
        vol_kernel = (float)block_sum(part, red);
      }
      const float iou3 = (float)((double)vol_kernel / den);
      if (iou3 > A.threshold) { if (threadIdx.x == 0) A.state[c] = ST_SUPPRESSED; continue; }
    }
    iou = (float)((double)vol_convex / den);
    if (iou <= A.threshold) continue;

    // ---- S5: rendered overlap inside bbox(h) (:1305-1330) ------------------------------------
    atomicAdd(&counters[7], threadIdx.x == 0 ? 1u : 0u);
    const int* bb = A.bbox + 6 * h;
    const int Nz = bb[1] - bb[0] + 1, Ny = bb[3] - bb[2] + 1, Nx = bb[5] - bb[4] + 1;
    const long long nv = (long long)Nz * Ny * Nx;
    const float overlap_maximal = (float)(den * (double)A.threshold);      // (A_min+1e-10)*threshold passed as float
    // The reference loop returns as soon as the running count exceeds overlap_maximal (:1305-1330); the outcome only
    // depends on min(full count, stop), so the block stops once its shared count reaches `stop`.
    const long long stop_ll = (overlap_maximal < 0.f) ? 1 : (long long)floorf(overlap_maximal) + 1;
    __syncthreads();
    if (threadIdx.x == 0) { sh_cnt = 0; sh_i[3] = 0; }
    __syncthreads();
    int cnt = 0;
    for (long long q0 = 0; q0 < nv; q0 += (long long)blockDim.x * 8) {
      if ((long long)(*(volatile int*)&sh_cnt) >= stop_ll) break;
      int local = 0;
#pragma unroll 1
      for (int u = 0; u < 8; ++u) {
        const long long q = q0 + (long long)u * blockDim.x + threadIdx.x;
        if (q >= nv) break;
        const int x = (int)(q % Nx), y = (int)((q / Nx) % Ny), z = (int)(q / ((long long)Nx * Ny));
        const float fz = (float)(z + bb[0]), fy = (float)(y + bb[2]), fx = (float)(x + bb[4]);
        if (sdbins::inside_polyhedron_binned(fz, fy, fx, c1, pv1, sfaces, A.F, X.bins) && sdbins::inside_polyhedron_binned(fz, fy, fx, c2, pv2, sfaces, A.F, X.bins)) {
          local++; if (q == 0) sh_i[3] = 1;
        }
      }
      for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
      if ((threadIdx.x & 31) == 0 && local) atomicAdd(&sh_cnt, local);
      cnt += local;
    }
    (void)cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
      const int full = sh_cnt;
      const int first_hit = sh_i[3];
      // early exit emulation: the serial loop returns the first running count with (float)res > overlap_maximal
      int res;
      if (overlap_maximal < 0.f) res = (nv > 0) ? first_hit : 0;
      else {
        const long long stop = (long long)floorf(overlap_maximal) + 1;      // smallest integer > overlap_maximal
        res = (full >= stop) ? (int)stop : full;
      }
      const float A_inter_render = (float)res;
      const float iou5 = (float)((double)A_inter_render / den);
      if (iou5 > A.threshold) A.state[c] = ST_SUPPRESSED;
    }
  }
}

// full: start of a round; !full: retry of the pair stages after the pair list was enlarged
__global__ void k_reset(unsigned int* counters, int* slot, const int* uniq, int hull_cap, int full) {
  const unsigned int nu = min(counters[12], (unsigned int)hull_cap);
  for (unsigned int u = threadIdx.x; u < nu; u += blockDim.x) slot[uniq[u]] = -1;
  __syncthreads();
  if (threadIdx.x == 0) {
    counters[1] = 0; counters[11] = 0; counters[12] = 0; counters[14] = 0; counters[15] = 0;
    if (full) { counters[0] = 0; counters[10] = counters[9]; counters[9] = 0; counters[8] = 0; }
  }
}
__global__ void k_finish(const int* __restrict__ state, int n, unsigned char* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) keep[i] = (state[i] != ST_SUPPRESSED) ? 1 : 0;
}

}  // namespace

// 0 (default): face_cone_volume as validated on the GPU in round 1; 1: face_cone_volume_n on pre-normalised planes.
// The two are bit-identical functions (host build, 7 500 fuzzed pairs: tests/test_cpu_oracle.py); the switch exists because
// variant 1 has not been run on a GPU yet (tests/test_gpu_3d.py runs it under STARDIST_B200_EXPERIMENTAL=1).
static int g_nms3d_norm_planes = 1;      // face_cone_volume_n (bit-identical on the host build; goldens green on the GPU)
static int g_nms3d_fan_subdiv = 1;    // refined fan (sdb_nms3d_set_s3_bound(2) = bounds on the coarse fan only)
static int g_nms3d_s5_bins = 1;       // direction-binned tetrahedra in the S5 rendering (off together with the S3 bound switch)
static int g_nms3d_warp_bound = 1;    // S3 lower bound by one warp per pair (0: k_heavy stage 1, a CTA per pair)
static int g_nms3d_split = 1;         // S3 | hull kernel | S4+S5 as separate launches (sdb_nms3d_set_split; decisions identical)
extern "C" int sdb_nms3d_set_split(int on) { g_nms3d_split = on ? 1 : 0; g_nms3d_warp_bound = (on & 2) ? 0 : 1; return 0; }   // on = 3: split with the CTA-per-pair bound
static int g_nms3d_s3_bound = 1;      // S3 lower-bound short cut (sdb_nms3d_set_s3_bound; decisions identical)
extern "C" int sdb_nms3d_set_s3_bound(int on) { g_nms3d_s3_bound = on ? 1 : 0; g_nms3d_s5_bins = on ? 1 : 0; g_nms3d_fan_subdiv = on == 2 ? 0 : 1; return 0; }
extern "C" int sdb_nms3d_set_variant(int norm_planes) { g_nms3d_norm_planes = norm_planes ? 1 : 0; return 0; }

extern "C" int sdb_nms3d(const float* d_dist, const float* d_points, const float* d_verts, const int* d_faces,
                         int n_polys, int n_rays, int n_faces, float threshold, int use_bbox, int use_kdtree,
                         int verbose, unsigned char* d_keep, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int n = n_polys;
  if (n <= 0) return 0;
  if (n_rays < 4 || n_rays > MAXR || n_faces > MAXF || n_faces < 1) { sdb::set_error("nms3d: unsupported n_rays / n_faces"); return 1; }
  sdb::DevBuf b_vol, b_bbox, b_ro, b_roi, b_rii, b_terms, b_aniso, b_stats, b_cellpt, b_counts, b_start, b_items, b_state, b_pairs, b_counters, b_list0, b_list1, b_kept;
  SDB_CUDA(b_list0.alloc((size_t)n * 4, st)); SDB_CUDA(b_list1.alloc((size_t)n * 4, st)); SDB_CUDA(b_kept.alloc((size_t)n * 4, st));
  sdb::DevBuf b_cursor; SDB_CUDA(b_cursor.alloc((size_t)n * 8, st)); SDB_CUDA(cudaMemsetAsync(b_cursor.p, 0, (size_t)n * 8, st));
  SDB_CUDA(b_vol.alloc((size_t)n * 4, st)); SDB_CUDA(b_bbox.alloc((size_t)n * 24, st)); SDB_CUDA(b_ro.alloc((size_t)n * 4, st));
  SDB_CUDA(b_roi.alloc((size_t)n * 4, st)); SDB_CUDA(b_rii.alloc((size_t)n * 4, st)); SDB_CUDA(b_terms.alloc((size_t)n * 12, st));
  SDB_CUDA(b_aniso.alloc(16, st)); SDB_CUDA(b_stats.alloc(32, st)); SDB_CUDA(b_state.alloc((size_t)n * 4, st));
  SDB_CUDA(b_counters.alloc(64, st));
  const int init_stats[8] = {0, INT32_MAX, INT32_MIN, INT32_MAX, INT32_MIN, INT32_MAX, INT32_MIN, 0};
  SDB_CUDA(cudaMemcpyAsync(b_stats.p, init_stats, sizeof(init_stats), cudaMemcpyHostToDevice, st));
  SDB_CUDA(cudaMemsetAsync(b_state.p, 0, (size_t)n * 4, st));
  SDB_CUDA(cudaMemsetAsync(b_counters.p, 0, 64, st));
  Arr A;
  A.dist = d_dist; A.points = d_points; A.verts = d_verts; A.faces = d_faces; A.n = n; A.R = n_rays; A.F = n_faces;
  A.volume = b_vol.as<float>(); A.bbox = b_bbox.as<int>(); A.r_outer = b_ro.as<float>(); A.r_outer_iso = b_roi.as<float>();
  A.r_inner_iso = b_rii.as<float>(); A.aniso_terms = b_terms.as<float>(); A.aniso = b_aniso.as<float>();
  A.state = b_state.as<int>(); A.threshold = threshold; A.use_bbox = use_bbox; A.norm_planes = g_nms3d_norm_planes; A.s3_bound = g_nms3d_s3_bound; A.fan_subdiv = g_nms3d_fan_subdiv; A.dup_dirs = 0;
  A.cell_start = nullptr; A.items = nullptr; A.max_dist = 0; memset(&A.G, 0, sizeof(A.G));
  SDB_LAUNCH(k_pre1, cdiv(n, 128), 128, 0, st, A, b_stats.as<unsigned int>());
  SDB_LAUNCH(k_aniso, 3, 256, 0, st, A);
  SDB_LAUNCH(k_aniso_norm, 1, 1, 0, st, A);
  SDB_LAUNCH(k_pre2, cdiv(n, 128), 128, 0, st, A);
  int h_stats[8]; float h_aniso[3];
  std::vector<float> h_verts((size_t)3 * n_rays);
  SDB_CUDA(cudaMemcpyAsync(h_verts.data(), d_verts, h_verts.size() * 4, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaMemcpyAsync(h_stats, b_stats.p, sizeof(h_stats), cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaMemcpyAsync(h_aniso, b_aniso.p, 12, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  float max_dist; { unsigned int u = (unsigned int)h_stats[0]; memcpy(&max_dist, &u, 4); }
  A.max_dist = max_dist;
  A.dup_dirs = sd3::rays_have_coincident_directions(h_verts.data(), n_rays) ? 1 : 0;
  Grid3 G; G.all_pairs = use_kdtree ? 0 : 1;
  {
    double cell = 2.0 * (double)max_dist * (1.0 + 1e-5) + 1e-3;
    if (cell < 1.0) cell = 1.0;
    double ext[3];
    for (int k = 0; k < 3; ++k) { G.mn[k] = (float)h_stats[1 + 2 * k]; ext[k] = (double)h_stats[2 + 2 * k] - h_stats[1 + 2 * k] + 1.0; }
    while ((floor(ext[0] / cell) + 1) * (floor(ext[1] / cell) + 1) * (floor(ext[2] / cell) + 1) > 4.0e6) cell *= 2;
    G.cell = (float)cell;
    for (int k = 0; k < 3; ++k) G.g[k] = G.all_pairs ? 1 : (int)floor(ext[k] / cell) + 1;
  }
  A.G = G;
  const int n_cells = G.g[0] * G.g[1] * G.g[2];
  SDB_CUDA(b_cellpt.alloc((size_t)n * 4, st)); SDB_CUDA(b_counts.alloc((size_t)(n_cells + 1) * 4, st));
  SDB_CUDA(b_start.alloc((size_t)(n_cells + 1) * 4, st)); SDB_CUDA(b_items.alloc((size_t)n * 4, st));
  SDB_CUDA(cudaMemsetAsync(b_counts.p, 0, (size_t)(n_cells + 1) * 4, st));
  SDB_LAUNCH(k_cell_count, cdiv(n, 256), 256, 0, st, d_points, n, G, b_cellpt.as<int>(), b_counts.as<unsigned int>());
  SDB_LAUNCH(k_scan_serial, 1, 1024, 0, st, b_counts.as<unsigned int>(), b_start.as<unsigned int>(), n_cells);
  SDB_CUDA(cudaMemcpyAsync(b_counts.p, b_start.p, (size_t)(n_cells + 1) * 4, cudaMemcpyDeviceToDevice, st));
  SDB_LAUNCH(k_cell_fill, cdiv(n, 256), 256, 0, st, b_cellpt.as<int>(), n, b_counts.as<unsigned int>(), b_items.as<int>());
  A.cell_start = b_start.as<unsigned int>(); A.items = b_items.as<int>();

  // pair list: grown on overflow (the round is re-run, decisions are idempotent)
  size_t pair_cap = std::max<size_t>(1 << 16, (size_t)n * 4);
  SDB_CUDA(b_pairs.alloc(pair_cap * sizeof(int2), st));
  // S3 | hulls | S4+S5 split: open pairs of S3, per-round hull cache (slot: polyhedron -> cache row, -1 unregistered)
  sdb::DevBuf b_list4, b_slot, b_uniq, b_hull, b_hulln;
  const int hull_cap = 16384;
  SDB_CUDA(b_list4.alloc(pair_cap * sizeof(int2), st));
  SDB_CUDA(b_slot.alloc((size_t)n * 4, st)); SDB_CUDA(cudaMemsetAsync(b_slot.p, 0xff, (size_t)n * 4, st));
  SDB_CUDA(b_uniq.alloc((size_t)hull_cap * 4, st));
  SDB_CUDA(b_hull.alloc((size_t)hull_cap * n_faces * sizeof(Plane), st));
  SDB_CUDA(b_hulln.alloc((size_t)hull_cap * 4, st));
  // direction bins for the S5 rendering (same lists as k_paint3d; off with the rendering's switch sdb_label3d_set_cull(0/1))
  sdb::DevBuf b_bcnt, b_bfaces;
  sdbins::FaceBins FB{nullptr, nullptr};
  if (g_nms3d_s5_bins) {
    SDB_CUDA(b_bcnt.alloc(sdbins::BIN_N * sizeof(int), st)); SDB_CUDA(b_bfaces.alloc((size_t)sdbins::BIN_N * sdbins::BIN_CAP * sizeof(int), st));
    FB.count = b_bcnt.as<int>(); FB.faces = b_bfaces.as<int>();
    SDB_LAUNCH(sdbins::k_build_bins, sdbins::BIN_N, 128, 0, st, d_verts, d_faces, n_faces, FB);
  }
  const size_t hull_per_warp = (((size_t)3 * n_rays * sizeof(double) + (size_t)((n_rays * n_rays + 31) / 32) * 4 + (size_t)3 * 4 * n_rays * 2 + 16) + 15) / 16 * 16;
  const size_t hull_smem = 4 * hull_per_warp;
  // warp-per-pair S3 bound: per-warp scratch (2F planes, R distances, two vertex sets); as many warps per block as fit
  const size_t bound_per_warp = (((size_t)2 * n_faces * sizeof(Plane) + (size_t)n_rays * sizeof(double) + (size_t)6 * n_rays * sizeof(float)) + 15) / 16 * 16;
  const int bound_wpb = g_nms3d_warp_bound ? (int)std::min<size_t>(8, (size_t)(200 * 1024) / bound_per_warp) : 0;
  const int bound_bps = bound_wpb > 0 ? std::max(1, std::min(4, (int)((size_t)(200 * 1024) / (bound_per_warp * bound_wpb)))) : 0;
  const size_t bound_smem = bound_per_warp * (size_t)std::max(bound_wpb, 0);
  if (bound_wpb > 0) SDB_CUDA(cudaFuncSetAttribute(k_s3_bound_warp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(bound_smem, 48 * 1024)));
  SDB_CUDA(cudaFuncSetAttribute(k_hulls, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(hull_smem, 48 * 1024)));
  const size_t smem = ((size_t)(6 * n_rays + 3 * n_faces) * 4 + 15) / 16 * 16 + (size_t)2 * n_faces * sizeof(Plane) +
                      (size_t)3 * n_rays * 8 + (size_t)((n_rays * n_rays + 31) / 32) * 4 + (size_t)3 * 4 * n_rays * 2 + 64 +
                      (size_t)n_faces * 12 + 32;      // + face-centroid rays of the refined fan bounds
  SDB_CUDA(cudaFuncSetAttribute(k_heavy, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem, 48 * 1024)));
  if (verbose) {
    printf("Non Maximum Suppression (3D, GPU) ++++ \nNMS: n_polys  = %d \nNMS: n_rays   = %d  \nNMS: n_faces  = %d \nNMS: thresh   = %.3f \nNMS: use_bbox = %d \nNMS: use_kdtree = %d \n",
           n, n_rays, n_faces, threshold, use_bbox, use_kdtree);
    printf("NMS: calculated anisotropy: %.2f \t %.2f \t %.2f \n", h_aniso[0], h_aniso[1], h_aniso[2]);
  }
  unsigned int* h_pin = sdb::pinned_scratch();
  if (!h_pin) { sdb::set_error("nms3d: pinned host allocation failed"); return 1; }
  int rc = 0;
  for (int round = 0;; ++round) {
    SDB_LAUNCH(k_reset, 1, 256, 0, st, b_counters.as<unsigned int>(), b_slot.as<int>(), b_uniq.as<int>(), hull_cap, 1);
    sdb::ProfSpan sp;
    sdb::profile_begin("nms3d_frontier", st, &sp);
    {
      const int* lin = round == 0 ? (const int*)nullptr : ((round & 1) ? b_list1.as<int>() : b_list0.as<int>());
      int* lout = (round & 1) ? b_list0.as<int>() : b_list1.as<int>();
      SDB_LAUNCH(k_frontier, std::min(cdiv((long long)n * 32, 256), 132 * 8), 256, 0, st, A, round, lin, n, lout, b_kept.as<int>(), b_cursor.as<int2>(), b_counters.as<unsigned int>());
    }
    sdb::profile_end("nms3d_frontier", st, &sp);
    for (;;) {
      sdb::profile_begin("nms3d_pretest", st, &sp);
      SDB_LAUNCH(k_pretest, 132 * 8, 128, 0, st, A, round, b_kept.as<int>(), b_pairs.as<int2>(), (unsigned int)pair_cap, b_counters.as<unsigned int>());
      sdb::profile_end("nms3d_pretest", st, &sp);
      sdb::profile_begin("nms3d_heavy", st, &sp);
      if (g_nms3d_split) {
        HeavyCtx X{1, b_list4.as<int2>(), b_slot.as<int>(), b_uniq.as<int>(), b_hull.as<Plane>(), b_hulln.as<int>(), hull_cap, FB};
        sdb::ProfSpan s2;
        sdb::profile_begin("nms3d_heavy_bound", st, &s2);
        if (bound_wpb > 0) SDB_LAUNCH(k_s3_bound_warp, 132 * bound_bps, 256, bound_smem, st, A, b_pairs.as<int2>(), b_counters.as<unsigned int>(), (unsigned int)pair_cap, X, bound_wpb);
        else SDB_LAUNCH(k_heavy, 132 * 2, 512, smem, st, A, b_pairs.as<int2>(), b_counters.as<unsigned int>(), (unsigned int)pair_cap, X);
        sdb::profile_end("nms3d_heavy_bound", st, &s2);
        sdb::profile_begin("nms3d_hulls", st, &s2);
        SDB_LAUNCH(k_hulls, 132 * 4, 128, hull_smem, st, A, X, b_counters.as<unsigned int>());
        sdb::profile_end("nms3d_hulls", st, &s2);
        X.stage = 2;
        sdb::profile_begin("nms3d_heavy_s4s3s5", st, &s2);
        SDB_LAUNCH(k_heavy, 132 * 2, 512, smem, st, A, b_pairs.as<int2>(), b_counters.as<unsigned int>(), (unsigned int)pair_cap, X);
        sdb::profile_end("nms3d_heavy_s4s3s5", st, &s2);
      } else {
        HeavyCtx X{0, nullptr, nullptr, nullptr, nullptr, nullptr, 0, FB};
        SDB_LAUNCH(k_heavy, 132 * 2, 512, smem, st, A, b_pairs.as<int2>(), b_counters.as<unsigned int>(), (unsigned int)pair_cap, X);
      }
      sdb::profile_end("nms3d_heavy", st, &sp);
      if (cudaMemcpyAsync(h_pin, b_counters.p, 64, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) {
        sdb::set_error(std::string("nms3d: round failed: ") + cudaGetErrorString(cudaGetLastError())); rc = 1; break;
      }
      if (h_pin[1] <= pair_cap) break;
      // overflow: enlarge the list and redo the pretest/heavy stages of this round (already suppressed
      // candidates are skipped, nothing is lost)
      pair_cap = (size_t)h_pin[1] + (size_t)h_pin[1] / 2;
      SDB_CUDA(b_pairs.alloc(pair_cap * sizeof(int2), st));
      SDB_CUDA(b_list4.alloc(pair_cap * sizeof(int2), st));
      SDB_LAUNCH(k_reset, 1, 256, 0, st, b_counters.as<unsigned int>(), b_slot.as<int>(), b_uniq.as<int>(), hull_cap, 0);
    }
    if (rc) break;
    if (verbose) printf("NMS3D(b200): round %d undecided=%u heavy pairs=%u (pretests %u, kernel %u [decided by the lower bound: %u, S3 after S4: %u], convex %u [decided by the fan bounds: %u], render %u so far)\n",
                        round, h_pin[0], h_pin[1], h_pin[4], h_pin[5], h_pin[3], h_pin[13], h_pin[6], h_pin[2], h_pin[7]);
    if (h_pin[0] == 0) break;
    if (round > 4 * n + 8) { sdb::set_error("nms3d: no progress"); rc = 1; break; }
  }
  if (rc) return rc;
  SDB_LAUNCH(k_finish, cdiv(n, 256), 256, 0, st, b_state.as<int>(), n, d_keep);
  return 0;
}

// reference C ABI (stardist3d_lib.h:55-65): host pointers
extern "C" void _LIB_non_maximum_suppression_sparse(const float* scores, const float* dist, const float* points,
                                                    const int n_polys, const int n_rays, const int n_faces,
                                                    const float* verts, const int* faces, const float threshold,
                                                    const int use_bbox, const int use_kdtree, const int verbose,
                                                    bool* result) {
  (void)scores;     // not used by the reference either (the arrays arrive sorted)
  if (n_polys <= 0) return;
  // The reference signature returns void (stardist3d_lib.h:55-65).  A failure must not take the host process down (the
  // consumer may be a JVM): the result is zeroed (nothing kept), the message is left in sdb_last_error() and one line goes
  // to stderr; callers that can should use the int-returning sdb_nms3d / check sdb_last_error().
  auto fail = [&](const char* what) {
    fprintf(stderr, "stardist_b200: _LIB_non_maximum_suppression_sparse failed: %s: %s\n", what, sdb_last_error());
    for (int i = 0; i < n_polys; ++i) result[i] = false;
    cudaGetLastError();
  };
  cudaStream_t st = 0;
  sdb::DevBuf d_dist, d_points, d_verts, d_faces, d_keep;
  if (d_dist.alloc((size_t)n_polys * n_rays * 4, st) || d_points.alloc((size_t)n_polys * 12, st) || d_verts.alloc((size_t)n_rays * 12, st) ||
      d_faces.alloc((size_t)n_faces * 12, st) || d_keep.alloc((size_t)n_polys, st)) { sdb::set_error("device allocation failed"); return fail("alloc"); }
  cudaMemcpyAsync(d_dist.p, dist, (size_t)n_polys * n_rays * 4, cudaMemcpyHostToDevice, st);
  cudaMemcpyAsync(d_points.p, points, (size_t)n_polys * 12, cudaMemcpyHostToDevice, st);
  cudaMemcpyAsync(d_verts.p, verts, (size_t)n_rays * 12, cudaMemcpyHostToDevice, st);
  cudaMemcpyAsync(d_faces.p, faces, (size_t)n_faces * 12, cudaMemcpyHostToDevice, st);
  if (sdb_nms3d(d_dist.as<float>(), d_points.as<float>(), d_verts.as<float>(), d_faces.as<int>(), n_polys, n_rays, n_faces,
                threshold, use_bbox, use_kdtree, verbose, d_keep.as<unsigned char>(), (sdb_stream_t)st)) return fail("kernel");
  if (cudaMemcpyAsync(result, d_keep.p, (size_t)n_polys, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) {
    sdb::set_error("copy back failed"); return fail("copy back");
  }
  sdb::set_error("");
}
