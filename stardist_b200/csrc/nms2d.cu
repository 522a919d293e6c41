// nms2d.cu -- star-convex polygon non-maximum suppression on the GPU.
//
// Reference semantics: stardist/lib/stardist2d.cpp:390-615 (c_non_max_suppression_inds).
//   * vertices x = px + d*cosf(k*2pi/R), y = py + d*sinf(..) in float32 (no FMA), truncated to
//     integers (:453-471); float bbox, radius_outer = max d, float shoelace area (:128-138)
//   * greedy loop in score order (:525-587): a kept polygon i suppresses every later, not yet
//     suppressed j inside the kd-tree radius (max_dist + r_i)^2 (:548-549, strict <) whose
//     integer bbox intersects (:575) and whose Clipper overlap / min(area) > thresh (:579-581)
//
// GPU formulation (SURVEY A.5): every pair decision is a pure function of (i,j); the greedy
// loop is the resolution of a DAG in score order.  We peel it by frontiers:
//   round r:  K_frontier  -- an undecided candidate with no undecided higher-scored candidate
//                            that *could* test it (same radius/bbox predicate) is kept;
//             K_suppress  -- every undecided candidate is tested against the candidates kept in
//                            this round that can reach it; first overlap > thresh suppresses it.
// The set of evaluated pairs is a superset of the CPU's, the decisions are identical.
// The pair test itself is clip2d.cuh (bit-exact restatement of the Clipper result).
//
// Must be compiled with -fmad=false (the reference's float/double expressions are not fused).
#include <math.h>
#include <string.h>
#include <vector>
#include "nms2d_common.cuh"
#include "../../include/stardist_b200.h"

namespace sdnms {
int g_filter_mode = 1;
unsigned long long g_filter_stats[4] = {0, 0, 0, 0};
int g_tail_mode = 1;
namespace {

// ------------------------------------------------------------------------------------------
__global__ void k_precompute(const float* __restrict__ dist, const float* __restrict__ points,
                             const float* __restrict__ sn, const float* __restrict__ cs,
                             int n, int R, int2* __restrict__ verts, int4* __restrict__ bbox,
                             float* __restrict__ radius, float* __restrict__ area,
                             double* __restrict__ suf, double* __restrict__ sarea, float* __restrict__ maxlen,
                             unsigned int* __restrict__ stats /* [0]=max radius bits,[1..4]= minx,maxx,miny,maxy (int) */) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float py = points[2 * i], px = points[2 * i + 1];
  float bx1 = 0, bx2 = 0, by1 = 0, by2 = 0, rmax = 0;
  int2* v = verts + (size_t)i * R;
  for (int k = 0; k < R; ++k) {
    const float d = dist[(size_t)i * R + k];
    const float y = py + d * sn[k];
    const float x = px + d * cs[k];
    if (k == 0) { bx1 = x; bx2 = x; by1 = y; by2 = y; }
    else {
      bx1 = (x < bx1) ? x : bx1; bx2 = (x > bx2) ? x : bx2;
      by1 = (y < by1) ? y : by1; by2 = (y > by2) ? y : by2;
    }
    int2 q; q.x = (int)(long long)x; q.y = (int)(long long)y;   // IntPoint(x,y): trunc toward zero
    v[k] = q;
    rmax = fmaxf(d, rmax);
  }
  // area_from_path (stardist2d.cpp:128-138): float accumulator over int64 cross products
  float a = 0;
  for (int k = 0; k < R; ++k) {
    int2 p = v[k], q = v[(k + 1) % R];
    long long cr = (long long)p.x * (long long)q.y - (long long)p.y * (long long)q.x;
    a = a + (float)cr;
  }
  a = (float)(0.5 * (double)fabsf(a));
  area[i] = a;
  radius[i] = rmax;
  if (suf) {
    // pre-filter data (polyfast.cuh): suffix sums of F_k = ∫ x dy over edge k, ∮ x dy, longest edge
    double s = 0; float ml = 0;
    for (int k = R - 1; k >= 0; --k) {
      const int2 p = v[k], q = v[(k + 1) % R];
      suf[(size_t)i * R + k] = s;
      s += 0.5 * (double)((long long)q.y - p.y) * (double)((long long)p.x + q.x);
      const float ex = (float)(q.x - p.x), ey = (float)(q.y - p.y);
      ml = fmaxf(ml, sqrtf(ex * ex + ey * ey));
    }
    sarea[i] = s;
    maxlen[i] = ml * 1.000001f;
  }
  // bbox_intersect() takes int parameters: the float bbox is truncated at the call (:114-120,575)
  int4 b; b.x = (int)bx1; b.y = (int)bx2; b.z = (int)by1; b.w = (int)by2;
  bbox[i] = b;
  atomicMax(&stats[0], __float_as_uint(rmax));
  float cx = fminf(fmaxf(px, -1.0e9f), 1.0e9f), cy = fminf(fmaxf(py, -1.0e9f), 1.0e9f);
  atomicMin((int*)&stats[1], (int)floorf(cx)); atomicMax((int*)&stats[2], (int)floorf(cx));
  atomicMin((int*)&stats[3], (int)floorf(cy)); atomicMax((int*)&stats[4], (int)floorf(cy));
}

// Same results as k_precompute, one WARP per polygon (lane = ray; coalesced vertex / suffix rows).  The float
// shoelace sum keeps the reference's left-to-right order: the 32 cross products of a chunk are broadcast in turn.
__global__ void __launch_bounds__(256) k_precompute_w(const float* __restrict__ dist, const float* __restrict__ points,
                             const float* __restrict__ sn, const float* __restrict__ cs,
                             int n, int R, int2* __restrict__ verts, int4* __restrict__ bbox,
                             float* __restrict__ radius, float* __restrict__ area,
                             double* __restrict__ suf, double* __restrict__ sarea, float* __restrict__ maxlen,
                             unsigned int* __restrict__ stats) {
  const int lane = threadIdx.x & 31;
  // running statistics of this warp (one set of atomics per block at the end: one per polygon serialised on 5 words)
  float st_r = 0.f; int st_x0 = INT32_MAX, st_x1 = INT32_MIN, st_y0 = INT32_MAX, st_y1 = INT32_MIN;
  const int warps = (gridDim.x * blockDim.x) >> 5;
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
  const float py = points[2 * i], px = points[2 * i + 1];
  int2* v = verts + (size_t)i * R;
  const int2 v0 = [&]() { const float d = dist[(size_t)i * R]; int2 q; q.x = (int)(long long)(px + d * cs[0]); q.y = (int)(long long)(py + d * sn[0]); return q; }();
  float bx1 = 0, bx2 = 0, by1 = 0, by2 = 0, rmax = 0, a = 0, ml = 0;
  bool first = true;
  double s_total = 0;          // filled below (second sweep, right to left)
  const int n_chunks = (R + 31) / 32;
  for (int c = 0; c < n_chunks; ++c) {
    const int k = c * 32 + lane;
    const bool act = k < R;
    float x = 0, y = 0, d = 0;
    int2 q = make_int2(0, 0);
    if (act) {
      d = dist[(size_t)i * R + k];
      y = py + d * sn[k];
      x = px + d * cs[k];
      q.x = (int)(long long)x; q.y = (int)(long long)y;   // IntPoint(x,y): trunc toward zero
      v[k] = q;
    }
    // float bbox / max radius: min and max are exact, any order
    float lx1 = act ? x : INFINITY, lx2 = act ? x : -INFINITY, ly1 = act ? y : INFINITY, ly2 = act ? y : -INFINITY, lr = act ? d : 0.f;
    for (int o = 16; o > 0; o >>= 1) {
      lx1 = fminf(lx1, __shfl_xor_sync(0xffffffffu, lx1, o)); lx2 = fmaxf(lx2, __shfl_xor_sync(0xffffffffu, lx2, o));
      ly1 = fminf(ly1, __shfl_xor_sync(0xffffffffu, ly1, o)); ly2 = fmaxf(ly2, __shfl_xor_sync(0xffffffffu, ly2, o));
      lr = fmaxf(lr, __shfl_xor_sync(0xffffffffu, lr, o));
    }
    if (first) { bx1 = lx1; bx2 = lx2; by1 = ly1; by2 = ly2; first = false; }
    else { bx1 = fminf(bx1, lx1); bx2 = fmaxf(bx2, lx2); by1 = fminf(by1, ly1); by2 = fmaxf(by2, ly2); }
    rmax = fmaxf(rmax, lr);
    // next vertex (wraps to vertex 0 at the end)
    int2 qn;
    qn.x = __shfl_down_sync(0xffffffffu, q.x, 1); qn.y = __shfl_down_sync(0xffffffffu, q.y, 1);
    if (lane == 31 || k + 1 >= R) {
      if (k + 1 >= R) qn = v0;
      else {   // first vertex of the next chunk
        const float dn = dist[(size_t)i * R + k + 1];
        qn.x = (int)(long long)(px + dn * cs[k + 1]); qn.y = (int)(long long)(py + dn * sn[k + 1]);
      }
    }
    const long long cr = act ? ((long long)q.x * (long long)qn.y - (long long)q.y * (long long)qn.x) : 0;
    const float crf = (float)cr;
    const int lim = min(32, R - c * 32);
    for (int kk = 0; kk < lim; ++kk) a = a + __shfl_sync(0xffffffffu, crf, kk);      // area_from_path order (:128-138)
    if (suf) {
      const float ex = (float)(qn.x - q.x), ey = (float)(qn.y - q.y);
      float l = act ? sqrtf(ex * ex + ey * ey) : 0.f;
      for (int o = 16; o > 0; o >>= 1) l = fmaxf(l, __shfl_xor_sync(0xffffffffu, l, o));
      ml = fmaxf(ml, l);
    }
  }
  if (suf) {
    // suffix sums of F_k = 0.5 (y_{k+1} - y_k)(x_k + x_{k+1}), right to left over the chunks
    __syncwarp();              // the vertex row written above is read across lanes
    double carry = 0;
    for (int c = n_chunks - 1; c >= 0; --c) {
      const int k = c * 32 + lane;
      const bool act = k < R;
      double F = 0;
      if (act) {
        const int2 p = v[k], q = (k + 1 == R) ? v0 : v[k + 1];      // own row, just written by this warp
        F = 0.5 * (double)((long long)q.y - p.y) * (double)((long long)p.x + q.x);
      }
      // inclusive suffix scan inside the chunk
      double inc = F;
      for (int o = 1; o < 32; o <<= 1) {
        const double t = __shfl_down_sync(0xffffffffu, inc, o);
        if (lane + o < 32) inc += t;
      }
      if (act) suf[(size_t)i * R + k] = carry + (inc - F);           // Σ over edges after k
      carry += __shfl_sync(0xffffffffu, inc, 0);
    }
    s_total = carry;
  }
  if (lane == 0) {
    a = (float)(0.5 * (double)fabsf(a));
    area[i] = a;
    radius[i] = rmax;
    if (suf) { sarea[i] = s_total; maxlen[i] = ml * 1.000001f; }
    int4 b; b.x = (int)bx1; b.y = (int)bx2; b.z = (int)by1; b.w = (int)by2;
    bbox[i] = b;
    st_r = fmaxf(st_r, rmax);
    float cx = fminf(fmaxf(px, -1.0e9f), 1.0e9f), cy = fminf(fmaxf(py, -1.0e9f), 1.0e9f);
    st_x0 = min(st_x0, (int)floorf(cx)); st_x1 = max(st_x1, (int)floorf(cx));
    st_y0 = min(st_y0, (int)floorf(cy)); st_y1 = max(st_y1, (int)floorf(cy));
  }
  }
  __shared__ unsigned int sh_r; __shared__ int sh_b[4];
  if (threadIdx.x == 0) { sh_r = 0u; sh_b[0] = INT32_MAX; sh_b[1] = INT32_MIN; sh_b[2] = INT32_MAX; sh_b[3] = INT32_MIN; }
  __syncthreads();
  if (lane == 0) {
    atomicMax(&sh_r, __float_as_uint(st_r));
    atomicMin(&sh_b[0], st_x0); atomicMax(&sh_b[1], st_x1); atomicMin(&sh_b[2], st_y0); atomicMax(&sh_b[3], st_y1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    atomicMax(&stats[0], sh_r);
    atomicMin((int*)&stats[1], sh_b[0]); atomicMax((int*)&stats[2], sh_b[1]);
    atomicMin((int*)&stats[3], sh_b[2]); atomicMax((int*)&stats[4], sh_b[3]);
  }
}

__global__ void k_cell_count(const float* __restrict__ points, int n, GridDesc G, int* __restrict__ cell_of_pt,
                             unsigned int* __restrict__ counts) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int c = 0;
  if (!G.all_pairs) {
    int cx = cell_of(points[2 * i + 1], G.minx, G.cell, G.gx);
    int cy = cell_of(points[2 * i], G.miny, G.cell, G.gy);
    c = cy * G.gx + cx;
  }
  cell_of_pt[i] = c;
  atomicAdd(&counts[c], 1u);
}

// exclusive scan, three small kernels (n_cells is at most a few million)
constexpr int SCAN_T = 256, SCAN_ITEMS = 8, SCAN_TILE = SCAN_T * SCAN_ITEMS;
__global__ void k_scan_tiles(const unsigned int* __restrict__ in, unsigned int* __restrict__ out, int n,
                             unsigned int* __restrict__ tile_sums) {
  __shared__ unsigned int sh[SCAN_T];
  int base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
  unsigned int v[SCAN_ITEMS], s = 0;
  for (int k = 0; k < SCAN_ITEMS; ++k) { v[k] = (base + k < n) ? in[base + k] : 0u; s += v[k]; }
  sh[threadIdx.x] = s;
  __syncthreads();
  for (int off = 1; off < SCAN_T; off <<= 1) {
    unsigned int t = (threadIdx.x >= off) ? sh[threadIdx.x - off] : 0u;
    __syncthreads();
    sh[threadIdx.x] += t;
    __syncthreads();
  }
  unsigned int excl = sh[threadIdx.x] - s;
  for (int k = 0; k < SCAN_ITEMS; ++k) { if (base + k < n) out[base + k] = excl; excl += v[k]; }
  if (threadIdx.x == SCAN_T - 1) tile_sums[blockIdx.x] = sh[threadIdx.x];
}
__global__ void k_scan_sums(unsigned int* tile_sums, int n_tiles) {   // single block, serial over chunks
  __shared__ unsigned int sh[1024];
  __shared__ unsigned int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n_tiles; base += 1024) {
    int i = base + threadIdx.x;
    unsigned int v = (i < n_tiles) ? tile_sums[i] : 0u;
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int off = 1; off < 1024; off <<= 1) {
      unsigned int t = (threadIdx.x >= off) ? sh[threadIdx.x - off] : 0u;
      __syncthreads();
      sh[threadIdx.x] += t;
      __syncthreads();
    }
    if (i < n_tiles) tile_sums[i] = carry + sh[threadIdx.x] - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry += sh[1023];
    __syncthreads();
  }
}
__global__ void k_scan_add(unsigned int* __restrict__ out, int n, const unsigned int* __restrict__ tile_sums) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] += tile_sums[i / SCAN_TILE];
}

__global__ void k_cell_fill(const int* __restrict__ cell_of_pt, int n, unsigned int* __restrict__ cursor,
                            int* __restrict__ items) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned int pos = atomicAdd(&cursor[cell_of_pt[i]], 1u);
  items[pos] = i;
}

// sort every cell's item list by candidate index (= score order): the frontier scan of candidate c then only
// walks the prefix h < c, which is EMPTY for the local maxima that used to scan their whole neighbourhood.
// Rank by counting; a cell holds a few hundred items (cell edge = 2 max_dist).
__global__ void __launch_bounds__(256) k_cell_sort(const unsigned int* __restrict__ cell_start, const int* __restrict__ items_in,
                                                   int* __restrict__ items_out) {
  const unsigned int b = cell_start[blockIdx.x], e = cell_start[blockIdx.x + 1];
  __shared__ int sh[2048];
  const unsigned int m = e - b;
  if (m <= 2048) {
    for (unsigned int i = threadIdx.x; i < m; i += blockDim.x) sh[i] = items_in[b + i];
    __syncthreads();
    for (unsigned int i = threadIdx.x; i < m; i += blockDim.x) {
      const int v = sh[i];
      unsigned int r = 0;
      for (unsigned int j = 0; j < m; ++j) r += (sh[j] < v) ? 1u : 0u;
      items_out[b + r] = v;
    }
  } else {
    for (unsigned int i = threadIdx.x; i < m; i += blockDim.x) {
      const int v = items_in[b + i];
      unsigned int r = 0;
      for (unsigned int j = 0; j < m; ++j) r += (items_in[b + j] < v) ? 1u : 0u;
      items_out[b + r] = v;
    }
  }
}
__global__ void k_iota(int* __restrict__ out, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = i;
}

__global__ void k_finish(const int* __restrict__ state, int n, unsigned char* __restrict__ keep, unsigned int* __restrict__ flag /*[n+1] or null*/) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  const unsigned int k = (i < n && state[i] != ST_SUPPRESSED) ? 1u : 0u;
  if (i < n && keep) keep[i] = (unsigned char)k;
  if (flag) flag[i] = k;
}
__global__ void k_scatter_kept(const unsigned int* __restrict__ flag, const unsigned int* __restrict__ pos, int n, int* __restrict__ kept_index) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && flag[i]) kept_index[pos[i]] = i;
}
// paint order of survivors listed by descending score with ties in list order reversed (= np.argsort(prob,
// kind='stable')[::-1]): rank under np.argsort(prob_k, kind='stable') (geom2d.py:191), ids[rank] = index + 1
__global__ void k_paint_order(const float* __restrict__ prob, int nk, int* __restrict__ rank, int* __restrict__ id_by_rank) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nk) return;
  const float p = prob[i];
  int s = i, e = i + 1;
  while (s > 0 && prob[s - 1] == p) --s;
  while (e < nk && prob[e] == p) ++e;
  const int r = (nk - e) + (i - s);
  rank[i] = r;
  id_by_rank[r] = i + 1;
}


}  // namespace
}  // namespace sdnms

using namespace sdnms;

// ------------------------------------------------------------------------------------------
extern "C" int sdb_nms2d(const float* d_dist, const float* d_points, int n_polys, int n_rays,
                         float threshold, int use_bbox, int use_kdtree, int verbose,
                         unsigned char* d_keep, sdb_stream_t stream) {
  return sdb_nms2d_survivors(d_dist, d_points, n_polys, n_rays, threshold, use_bbox, use_kdtree, verbose, d_keep, nullptr, nullptr, stream);
}

extern "C" int sdb_paint_order_2d(const float* d_prob_desc, int n, int* d_rank, int* d_id_by_rank, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n <= 0) return 0;
  SDB_LAUNCH(k_paint_order, cdiv(n, 256), 256, 0, st, d_prob_desc, n, d_rank, d_id_by_rank);
  return 0;
}

extern "C" int sdb_nms2d_survivors(const float* d_dist, const float* d_points, int n_polys, int n_rays,
                                   float threshold, int use_bbox, int use_kdtree, int verbose,
                                   unsigned char* d_keep, int* d_kept_index, int* h_n_kept, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int n = n_polys, R = n_rays;
  if (h_n_kept) *h_n_kept = 0;
  if (n <= 0) return 0;
  if (R < 1 || R > 128) { sdb::set_error("nms2d: n_rays must be in [1,128]"); return 1; }

  // ray tables with the host libm, exactly like stardist2d.cpp:423,454-455:
  //   const float ANGLE_PI = 2*M_PI/n_rays;  sin(ANGLE_PI*k) / cos(ANGLE_PI*k) on float -> sinf/cosf
  std::vector<float> tab(2 * R);
  const float ANGLE_PI = (float)(2 * M_PI / R);
  for (int k = 0; k < R; ++k) { float a = ANGLE_PI * k; tab[k] = sinf(a); tab[R + k] = cosf(a); }

  const int filter = g_filter_mode;
  sdb::DevBuf b_suf, b_sarea, b_maxlen;
  if (filter) {
    SDB_CUDA(b_suf.alloc((size_t)n * R * sizeof(double), st));
    SDB_CUDA(b_sarea.alloc((size_t)n * sizeof(double), st));
    SDB_CUDA(b_maxlen.alloc((size_t)n * sizeof(float), st));
  }
  sdb::DevBuf b_tab, b_verts, b_bbox, b_radius, b_area, b_stats, b_cellpt, b_counts, b_start, b_tiles, b_items, b_state, b_slow, b_counters;
  SDB_CUDA(b_tab.alloc(2 * R * sizeof(float), st));
  SDB_CUDA(b_verts.alloc((size_t)n * R * sizeof(int2), st));
  SDB_CUDA(b_bbox.alloc((size_t)n * sizeof(int4), st));
  SDB_CUDA(b_radius.alloc((size_t)n * sizeof(float), st));
  SDB_CUDA(b_area.alloc((size_t)n * sizeof(float), st));
  SDB_CUDA(b_stats.alloc(8 * sizeof(unsigned int), st));
  SDB_CUDA(cudaMemcpyAsync(b_tab.p, tab.data(), 2 * R * sizeof(float), cudaMemcpyHostToDevice, st));
  const int init_stats[8] = {0, INT32_MAX, INT32_MIN, INT32_MAX, INT32_MIN, 0, 0, 0};
  SDB_CUDA(cudaMemcpyAsync(b_stats.p, init_stats, sizeof(init_stats), cudaMemcpyHostToDevice, st));
  SDB_LAUNCH(k_precompute_w, std::min(cdiv((long long)n * 32, 256), 132 * 16), 256, 0, st, d_dist, d_points, b_tab.as<float>(), b_tab.as<float>() + R, n, R,
             b_verts.as<int2>(), b_bbox.as<int4>(), b_radius.as<float>(), b_area.as<float>(),
             filter ? b_suf.as<double>() : (double*)nullptr, b_sarea.as<double>(), b_maxlen.as<float>(), b_stats.as<unsigned int>());
  int h_stats[8];
  SDB_CUDA(cudaMemcpyAsync(h_stats, b_stats.p, sizeof(h_stats), cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  float max_dist; { unsigned int u = (unsigned int)h_stats[0]; memcpy(&max_dist, &u, 4); }

  GridDesc G;
  G.all_pairs = use_kdtree ? 0 : 1;
  G.minx = (float)h_stats[1]; G.miny = (float)h_stats[3];
  {
    // cell edge >= largest search radius (max_dist + r_i <= 2*max_dist), with slack for rounding
    double cell = 2.0 * (double)max_dist * (1.0 + 1e-5) + 1e-3;
    if (cell < 1.0) cell = 1.0;
    double ex = (double)h_stats[2] - h_stats[1] + 1.0, ey = (double)h_stats[4] - h_stats[3] + 1.0;
    while ((floor(ex / cell) + 1) * (floor(ey / cell) + 1) > 4.0e6) cell *= 2;
    G.cell = (float)cell;
    G.gx = (int)floor(ex / cell) + 1; G.gy = (int)floor(ey / cell) + 1;
    if (G.all_pairs) { G.gx = G.gy = 1; }
  }
  const int n_cells = G.gx * G.gy;
  const int n_tiles = cdiv(n_cells + 1, SCAN_TILE);
  SDB_CUDA(b_cellpt.alloc((size_t)n * sizeof(int), st));
  SDB_CUDA(b_counts.alloc((size_t)(n_cells + 1) * sizeof(unsigned int), st));
  SDB_CUDA(b_start.alloc((size_t)(n_cells + 1) * sizeof(unsigned int), st));
  SDB_CUDA(b_tiles.alloc((size_t)n_tiles * sizeof(unsigned int), st));
  SDB_CUDA(b_items.alloc((size_t)n * sizeof(int), st));
  SDB_CUDA(b_state.alloc((size_t)n * sizeof(int), st));
  SDB_CUDA(b_slow.alloc((size_t)n * sizeof(int), st));
  SDB_CUDA(b_counters.alloc(16 * sizeof(unsigned int), st));
  SDB_CUDA(cudaMemsetAsync(b_counts.p, 0, (size_t)(n_cells + 1) * sizeof(unsigned int), st));
  SDB_CUDA(cudaMemsetAsync(b_state.p, 0, (size_t)n * sizeof(int), st));
  SDB_CUDA(cudaMemsetAsync(b_counters.p, 0, 16 * sizeof(unsigned int), st));
  SDB_LAUNCH(k_cell_count, cdiv(n, 256), 256, 0, st, d_points, n, G, b_cellpt.as<int>(), b_counts.as<unsigned int>());
  SDB_LAUNCH(k_scan_tiles, n_tiles, SCAN_T, 0, st, b_counts.as<unsigned int>(), b_start.as<unsigned int>(), n_cells + 1, b_tiles.as<unsigned int>());
  SDB_LAUNCH(k_scan_sums, 1, 1024, 0, st, b_tiles.as<unsigned int>(), n_tiles);
  SDB_LAUNCH(k_scan_add, cdiv(n_cells + 1, 256), 256, 0, st, b_start.as<unsigned int>(), n_cells + 1, b_tiles.as<unsigned int>());
  // cursor = copy of starts (counts buffer reused)
  SDB_CUDA(cudaMemcpyAsync(b_counts.p, b_start.p, (size_t)(n_cells + 1) * sizeof(unsigned int), cudaMemcpyDeviceToDevice, st));
  sdb::DevBuf b_items_raw;
  if (G.all_pairs) {
    SDB_LAUNCH(k_iota, cdiv(n, 256), 256, 0, st, b_items.as<int>(), n);        // single cell: already sorted
  } else {
    SDB_CUDA(b_items_raw.alloc((size_t)n * sizeof(int), st));
    SDB_LAUNCH(k_cell_fill, cdiv(n, 256), 256, 0, st, b_cellpt.as<int>(), n, b_counts.as<unsigned int>(), b_items_raw.as<int>());
    SDB_LAUNCH(k_cell_sort, n_cells, 256, 0, st, b_start.as<unsigned int>(), b_items_raw.as<int>(), b_items.as<int>());
  }

  NmsArrays A;
  A.points = d_points; A.radius = b_radius.as<float>(); A.area = b_area.as<float>();
  A.bbox = b_bbox.as<int4>(); A.verts = b_verts.as<int2>();
  A.cell_start = b_start.as<unsigned int>(); A.items = b_items.as<int>();
  A.state = b_state.as<int>(); A.n = n; A.R = R;
  A.max_dist = max_dist; A.threshold = threshold; A.use_bbox = use_bbox; A.G = G;
  A.suf = b_suf.as<double>(); A.sarea = b_sarea.as<double>(); A.maxlen = b_maxlen.as<float>(); A.filter = filter;
  {
    double m = 0;
    for (int k = 1; k <= 4; ++k) m = fmax(m, fabs((double)h_stats[k]));
    A.max_abs_coord = m + (double)max_dist + 2.0;
  }

  if (verbose) {
    printf("Non Maximum Suppression (2D, GPU) ++++ \n");
    printf("NMS: n_polys    = %d \nNMS: n_rays     = %d  \nNMS: thresh     = %.3f \nNMS: use_bbox   = %d\nNMS: use_kdtree = %d\n", n, R, threshold, use_bbox, use_kdtree);
    printf("NMS: max_dist = %g grid = %d x %d cell = %g\n", max_dist, G.gx, G.gy, G.cell);
  }
  unsigned int* h_pin = sdb::pinned_scratch();
  if (!h_pin) { sdb::set_error("nms2d: pinned host allocation failed"); return 1; }
  int rc;
  if (R <= 32) rc = run_rounds_nv32(A, b_slow.as<int>(), b_counters.as<unsigned int>(), st, verbose, h_pin);
  else rc = run_rounds_nv128(A, b_slow.as<int>(), b_counters.as<unsigned int>(), st, verbose, h_pin);
  if (rc) return rc;
  if (!d_kept_index) {
    SDB_LAUNCH(k_finish, cdiv(n + 1, 256), 256, 0, st, b_state.as<int>(), n, d_keep, (unsigned int*)nullptr);
    return 0;
  }
  // ordered list of survivors + their number on the host (one 4-byte read-back)
  sdb::DevBuf b_flag, b_pos, b_ft;
  const int nt = cdiv(n + 1, SCAN_TILE);
  SDB_CUDA(b_flag.alloc((size_t)(n + 1) * sizeof(unsigned int), st));
  SDB_CUDA(b_pos.alloc((size_t)(n + 1) * sizeof(unsigned int), st));
  SDB_CUDA(b_ft.alloc((size_t)nt * sizeof(unsigned int), st));
  SDB_LAUNCH(k_finish, cdiv(n + 1, 256), 256, 0, st, b_state.as<int>(), n, d_keep, b_flag.as<unsigned int>());
  SDB_LAUNCH(k_scan_tiles, nt, SCAN_T, 0, st, b_flag.as<unsigned int>(), b_pos.as<unsigned int>(), n + 1, b_ft.as<unsigned int>());
  SDB_LAUNCH(k_scan_sums, 1, 1024, 0, st, b_ft.as<unsigned int>(), nt);
  SDB_LAUNCH(k_scan_add, cdiv(n + 1, 256), 256, 0, st, b_pos.as<unsigned int>(), n + 1, b_ft.as<unsigned int>());
  SDB_LAUNCH(k_scatter_kept, cdiv(n, 256), 256, 0, st, b_flag.as<unsigned int>(), b_pos.as<unsigned int>(), n, d_kept_index);
  SDB_CUDA(cudaMemcpyAsync(h_pin, b_pos.as<unsigned int>() + n, sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  if (h_n_kept) *h_n_kept = (int)h_pin[0];
  return 0;
}

extern "C" int sdb_nms2d_set_filter(int mode) {
  if (mode < 0 || mode > 2) { sdb::set_error("nms2d: filter mode must be 0, 1 or 2"); return 1; }
  g_filter_mode = mode;
  return 0;
}
extern "C" int sdb_nms2d_set_tail(int on) { g_tail_mode = on < 0 ? 0 : (on > 2 ? 2 : on); return 0; }
extern "C" void sdb_nms2d_filter_stats(unsigned long long* out4, int reset) {
  for (int k = 0; k < 4; ++k) { out4[k] = g_filter_stats[k]; if (reset) g_filter_stats[k] = 0; }
}

extern "C" int _LIB_non_maximum_suppression_2d(const float* dist, const float* points, const int n_polys,
                                               const int n_rays, const float threshold, const int use_bbox,
                                               const int use_kdtree, const int verbose, bool* result) {
  if (n_polys <= 0) return 0;
  cudaStream_t st = 0;
  sdb::DevBuf d_dist, d_points, d_keep;
  SDB_CUDA(d_dist.alloc((size_t)n_polys * n_rays * sizeof(float), st));
  SDB_CUDA(d_points.alloc((size_t)n_polys * 2 * sizeof(float), st));
  SDB_CUDA(d_keep.alloc((size_t)n_polys, st));
  SDB_CUDA(cudaMemcpyAsync(d_dist.p, dist, (size_t)n_polys * n_rays * sizeof(float), cudaMemcpyHostToDevice, st));
  SDB_CUDA(cudaMemcpyAsync(d_points.p, points, (size_t)n_polys * 2 * sizeof(float), cudaMemcpyHostToDevice, st));
  int rc = sdb_nms2d(d_dist.as<float>(), d_points.as<float>(), n_polys, n_rays, threshold, use_bbox, use_kdtree, verbose,
                     d_keep.as<unsigned char>(), (sdb_stream_t)st);
  if (rc) return rc;
  static_assert(sizeof(bool) == 1, "bool must be one byte");
  SDB_CUDA(cudaMemcpyAsync(result, d_keep.p, (size_t)n_polys, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  return 0;
}
