// labelprep.cu -- the training targets of a label map: edt_prob (normalised exact Euclidean distance transform of every
// object) and fill_label_holes.  Both take a sequential int32 label map (values 0..n_labels, negative labels already
// mapped to 0: they are never an object and count as "another label", exactly like background).
//
// edt_prob (reference: stardist/utils.py:98-125, _edt_prob_scipy).  For a pixel p of label l > 0, d2(p) = the smallest
// sum_a ((q_a - p_a) * s_a)^2 over pixels q of the image with a label != l, evaluated in float64 in axis order 0, 1, ...
// (scipy's distance_transform_edt on the grown object box gives exactly this; positions outside the image do not count,
// except for a constant image, where the reference pads with background: black_border).  prob(p) =
// float(sqrt(d2) / (sqrt(max over the label of d2) + 1e-10)).
//
// The transform is separable over runs of equal labels: one pass per axis, last axis first.  Along a line, a run of
// label l only sees candidates of the same run (their earlier-pass value is the distance to another label inside their
// own sub-space) and the two positions just outside the run, which have another label and enter with cost 0: any
// candidate beyond such a position is farther along this axis and no closer.  Each run is a lower envelope of parabolas
// (Felzenszwalb & Huttenlocher), built with an exact cross-multiplied test.  Every pass carries the arg-min offset
// vector instead of a distance, and the last pass recomputes d2 from it in scipy's order and rounding, so integer and
// dyadic sampling are exact (all products and sums stay below 2^53 for extents <= 65535).  This unit is built with
// -fmad=false so no product is contracted into an FMA.  sdb_edt_prob_batch runs the same passes over training patches laid
// end to end: no pass runs along the batch (an object at a patch edge sees only its own patch, as the reference's per-patch
// call does), labels are distinct across items, and the constant-image rule is decided per item.
//
// fill_label_holes (reference: stardist/utils.py:137-153).  For label i, holes are the pixels with a label != i inside
// i's bounding box grown by one pixel on the sides that do not touch the image border, which cannot reach the boundary
// of that box through label-!=-i pixels under the connectivity generate_binary_structure(ndim, c).  out(p) = the largest
// i whose label or holes contain p (the reference writes labels in ascending order).  All boxes are laid end to end in
// one work array and labelled by one union-find (Playne & Hawick): a union pass over the backward half of the
// neighbourhood, a pass that compresses every path and flags roots seen on a box boundary, and a write pass.
#include <algorithm>
#include <climits>
#include <cmath>
#include <vector>
#include "common.cuh"
#include "../../include/stardist_b200.h"

namespace {

using sdb::cdiv;

constexpr int OFF_INF = INT_MIN;      // no candidate with another label in the sub-space resolved so far
constexpr int EDT_THREADS = 128;
constexpr int MAX_EXTENT = 65535;

struct Samp { double s[3]; };         // sampling of the pass axis and of the axes after it

// one thread per line along the pass axis; lines are numbered with the inner (faster) axes fastest, so the threads of
// a warp read neighbouring addresses in the column passes.  in: NB offset components (axes a+1 .. a+NB), planes of N;
// out: NB + 1 components (axes a .. a+NB), or, in the last pass (FINAL), d2 and the per-label maximum of d2.
// Envelope scratch: sv / sf [len + 2][n_lines] (position and cost of each parabola).
template <int NB, bool FINAL>
__global__ void __launch_bounds__(EDT_THREADS) k_edt_pass(const int* __restrict__ lbl, int len, long long inner, long long n_lines,
                                                          long long N, const int* __restrict__ in, int* __restrict__ out,
                                                          double* __restrict__ d2, unsigned long long* __restrict__ lmax, Samp sp,
                                                          int black, const int* __restrict__ item_minmax, long long item_lines,
                                                          int* __restrict__ sv, double* __restrict__ sf) {
  const long long l = (long long)blockIdx.x * EDT_THREADS + threadIdx.x;
  if (l >= n_lines) return;
  const long long o = l / inner, base = o * len * inner + (l - o * inner);
  if (item_minmax) {                        // batch: the constant-image rule per item (its label minimum equals its maximum > 0)
    const long long it = l / item_lines;
    black = item_minmax[2 * it] == item_minmax[2 * it + 1] && item_minmax[2 * it + 1] > 0;
  }
  const double s = sp.s[0], w = s * s;
  int* v = sv + l;
  double* f = sf + l;
  auto at = [&](int k) { return (long long)k * n_lines; };
  auto cost_of = [&](long long idx) {       // cost of an interior candidate: its offsets in the resolved sub-space
    double c = 0.0;
    if (NB > 0) {
      const int c0 = __ldg(in + idx);
      if (c0 == OFF_INF) return (double)INFINITY;
      const double t = (double)c0 * sp.s[1];
      c = t * t;
      if (NB > 1) {
        const double u = (double)__ldg(in + N + idx) * sp.s[2];
        c = c + u * u;
      }
    }
    return c;
  };
  int y = 0;
  while (y < len) {
    const int L = __ldg(lbl + base + (long long)y * inner);
    int k = 0;
    auto push = [&](int q, double fq) {
      while (k >= 2) {
        const int top = v[at(k - 1)], prev = v[at(k - 2)];
        const double ftop = f[at(k - 1)], fprev = f[at(k - 2)];
        const double A = (double)(q - top), B = (double)(top - prev);
        // intersection(top, q) <= intersection(prev, top), multiplied by 2 w A B > 0
        if (w * A * B * (A + B) + (fq - ftop) * B - (ftop - fprev) * A <= 0.0) --k;
        else break;
      }
      v[at(k)] = q; f[at(k)] = fq; ++k;
    };
    if (L > 0 && (y > 0 || black)) push(y - 1, 0.0);
    int b = y;
    for (; b < len; ++b) {
      const long long idx = base + (long long)b * inner;
      if (__ldg(lbl + idx) != L) break;
      if (L > 0 && NB > 0) {
        const double c = cost_of(idx);
        if (c != (double)INFINITY) push(b, c);
      }
    }
    if (L > 0) {                           // the run is [y, b)
      if (b < len || black) push(b, 0.0);
      int kp = 0;
      for (int p = y; p < b; ++p) {
        const long long idx = base + (long long)p * inner;
        while (kp + 1 < k) {
          const double t1 = (double)(v[at(kp + 1)] - p) * s, t0 = (double)(v[at(kp)] - p) * s;
          if (t1 * t1 + f[at(kp + 1)] <= t0 * t0 + f[at(kp)]) ++kp;
          else break;
        }
        int off[3] = {OFF_INF, 0, 0};
        if (k > 0) {
          const int q = v[at(kp)];
          off[0] = q - p;
          if (q >= y && q < b) {                          // interior candidate: its resolved offsets
            const long long qi = base + (long long)q * inner;
            for (int c = 0; c < NB; ++c) off[1 + c] = __ldg(in + c * N + qi);
          }
        }
        if (FINAL) {
          double dd = (double)INFINITY;
          if (off[0] != OFF_INF) {
            const double t0 = (double)off[0] * s;
            dd = t0 * t0;                                   // scipy: dt[0]^2 + dt[1]^2 (+ dt[2]^2)
            for (int c = 0; c < NB; ++c) {
              const double t = (double)off[1 + c] * sp.s[1 + c];
              dd = dd + t * t;
            }
          }
          d2[idx] = dd;
          atomicMax(lmax + (L - 1), (unsigned long long)__double_as_longlong(dd));   // non-negative: bit order = value order
        } else {
          for (int c = 0; c <= NB; ++c) out[c * N + idx] = off[c];
        }
      }
    }
    y = b;
  }
}

__global__ void k_edt_norm(const int* __restrict__ lbl, const double* __restrict__ d2, const unsigned long long* __restrict__ lmax,
                           long long N, float* __restrict__ prob) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (long long)gridDim.x * blockDim.x) {
    const int L = __ldg(lbl + i);
    float r = 0.f;
    if (L > 0) {
      const double m = __longlong_as_double((long long)__ldg(lmax + (L - 1)));
      r = __double2float_rn(__ddiv_rn(__dsqrt_rn(d2[i]), __dadd_rn(__dsqrt_rn(m), 1e-10)));
    }
    prob[i] = r;
  }
}

// ---------------------------------------------------------------------------------------------------- hole filling

struct Box { int lo[3], ext[3]; };                 // grown box of a label, 2-D maps as [1, H, W]
struct Nbrs { int n; int d[13][3]; };              // backward half of the neighbourhood (first non-zero component < 0)

__device__ __forceinline__ int box_of(const long long* __restrict__ off, int n, long long e) {
  int lo = 0, hi = n - 1;                          // largest i with off[i] <= e
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(off + mid) <= e) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ void local_coords(const Box& b, long long r, int& z, int& y, int& x) {
  x = (int)(r % b.ext[2]);
  const long long t = r / b.ext[2];
  y = (int)(t % b.ext[1]);
  z = (int)(t / b.ext[1]);
}

__device__ __forceinline__ int uf_find(const int* P, int x) {
  int p = __ldcg(P + x);
  while (p != x) { x = p; p = __ldcg(P + x); }
  return x;
}

__device__ __forceinline__ void uf_unite(int* P, int a, int b) {
  for (;;) {
    a = uf_find(P, a); b = uf_find(P, b);
    if (a == b) return;
    if (a < b) { const int old = atomicMin(P + b, a); if (old == b) return; b = old; }
    else { const int old = atomicMin(P + a, b); if (old == a) return; a = old; }
  }
}

// parent[e] = -1 for pixels of the box's own label, e otherwise
__global__ void k_fill_init(const int* __restrict__ lbl, int H, int W, const Box* __restrict__ boxes, const long long* __restrict__ off,
                            int n, long long total, int* __restrict__ parent) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int i = box_of(off, n, e);
    const Box b = boxes[i];
    int z, y, x;
    local_coords(b, e - off[i], z, y, x);
    const long long p = ((long long)(b.lo[0] + z) * H + b.lo[1] + y) * W + b.lo[2] + x;
    parent[e] = __ldg(lbl + p) == i + 1 ? -1 : (int)e;
  }
}

__global__ void k_fill_union(const Box* __restrict__ boxes, const long long* __restrict__ off, int n, long long total, Nbrs nb,
                             int* __restrict__ parent) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    if (__ldcg(parent + e) == -1) continue;      // -1 never changes
    const int i = box_of(off, n, e);
    const Box b = boxes[i];
    int z, y, x;
    local_coords(b, e - off[i], z, y, x);
    for (int k = 0; k < nb.n; ++k) {
      const int zz = z + nb.d[k][0], yy = y + nb.d[k][1], xx = x + nb.d[k][2];
      if (zz < 0 || zz >= b.ext[0] || yy < 0 || yy >= b.ext[1] || xx < 0 || xx >= b.ext[2]) continue;
      const long long ne = e + ((long long)nb.d[k][0] * b.ext[1] + nb.d[k][1]) * b.ext[2] + nb.d[k][2];
      if (__ldcg(parent + ne) != -1) uf_unite(parent, (int)e, (int)ne);
    }
  }
}

// every path compressed to its root; roots of components with a pixel on the box boundary are flagged as outside
__global__ void k_fill_roots(const Box* __restrict__ boxes, const long long* __restrict__ off, int n, long long total, int ndim,
                             int* __restrict__ parent, unsigned char* __restrict__ outside) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    if (__ldcg(parent + e) == -1) continue;
    const int r = uf_find(parent, (int)e);
    parent[e] = r;
    const int i = box_of(off, n, e);
    const Box b = boxes[i];
    int c[3];
    local_coords(b, e - off[i], c[0], c[1], c[2]);
    bool edge = false;
    for (int a = 3 - ndim; a < 3; ++a) edge |= c[a] == 0 || c[a] == b.ext[a] - 1;
    if (edge) outside[r] = 1;
  }
}

__global__ void k_fill_write(int H, int W, const Box* __restrict__ boxes, const long long* __restrict__ off, int n, long long total,
                             const int* __restrict__ parent, const unsigned char* __restrict__ outside, int* __restrict__ out) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int r = parent[e];
    if (r != -1 && outside[r]) continue;
    const int i = box_of(off, n, e);
    const Box b = boxes[i];
    int z, y, x;
    local_coords(b, e - off[i], z, y, x);
    atomicMax(out + ((long long)(b.lo[0] + z) * H + b.lo[1] + y) * W + b.lo[2] + x, i + 1);
  }
}

// ---------------------------------------------------------------------------------------------------- host side

int check_shape(const char* what, int ndim, const int* shape, int dims[3], long long* N) {
  char m[256];
  if (ndim != 2 && ndim != 3) { snprintf(m, sizeof(m), "%s: ndim must be 2 or 3", what); sdb::set_error(m); return 1; }
  dims[0] = 1;
  *N = 1;
  for (int a = 0; a < ndim; ++a) {
    if (shape[a] < 0 || shape[a] > MAX_EXTENT) {
      snprintf(m, sizeof(m), "%s: every extent must lie in [0, %d]", what, MAX_EXTENT); sdb::set_error(m); return 1;
    }
    dims[3 - ndim + a] = shape[a];
    *N *= shape[a];
  }
  if (*N > INT_MAX) { snprintf(m, sizeof(m), "%s: more than 2^31 - 1 pixels are not supported", what); sdb::set_error(m); return 1; }
  return 0;
}

int grid_for(long long work, int threads) { return (int)std::max<long long>(1, std::min<long long>(cdiv(work, threads), 132 * 32)); }

// the passes of the transform over `batch` maps of `shape` laid end to end (no pass runs along the batch): d2 of every pixel
// and the per-label maximum lmax[n_labels] (labels distinct across items).  item_minmax (device [batch][2], or NULL for the
// scalar black_border) gives each item's constant-image rule.
int edt_passes(const int* d_labels, int ndim, const int* shape, int batch, long long N, const double* s, int black_border,
               const int* item_minmax, int n_labels, double* D2, unsigned long long* M, cudaStream_t st) {
  long long stack = 0;                               // envelope entries of the largest pass: (len + 2) per line
  for (int a = 0; a < ndim; ++a) stack = std::max(stack, (shape[a] + 2LL) * (N / shape[a]));
  sdb::DevBuf offs_a, offs_b, sv, sf;
  SDB_CUDA(offs_a.alloc((size_t)N * 4, st));
  if (ndim == 3) SDB_CUDA(offs_b.alloc((size_t)N * 4 * 2, st));
  SDB_CUDA(sv.alloc((size_t)stack * 4, st));
  SDB_CUDA(sf.alloc((size_t)stack * 8, st));
  SDB_CUDA(cudaMemsetAsync(M, 0, (size_t)n_labels * 8, st));
  auto geom = [&](int a, int& len, long long& inner, long long& lines) {
    len = shape[a];
    inner = 1;
    for (int b = a + 1; b < ndim; ++b) inner *= shape[b];
    lines = N / len;
  };
  auto samp = [&](int a) { Samp p{{1.0, 1.0, 1.0}}; for (int b = a; b < ndim; ++b) p.s[b - a] = s[b]; return p; };
  int len;
  long long inner, lines;
  int* A = offs_a.as<int>();
  int* B = offs_b.as<int>();
  int* SV = sv.as<int>();
  double* SF = sf.as<double>();
  const int* MM = item_minmax;
  geom(ndim - 1, len, inner, lines);
  SDB_LAUNCH((k_edt_pass<0, false>), cdiv(lines, EDT_THREADS), EDT_THREADS, 0, st, d_labels, len, inner, lines, N, nullptr, A, nullptr,
             nullptr, samp(ndim - 1), black_border, MM, lines / batch, SV, SF);
  if (ndim == 2) {
    geom(0, len, inner, lines);
    SDB_LAUNCH((k_edt_pass<1, true>), cdiv(lines, EDT_THREADS), EDT_THREADS, 0, st, d_labels, len, inner, lines, N, A, nullptr, D2, M,
               samp(0), black_border, MM, lines / batch, SV, SF);
  } else {
    geom(1, len, inner, lines);
    SDB_LAUNCH((k_edt_pass<1, false>), cdiv(lines, EDT_THREADS), EDT_THREADS, 0, st, d_labels, len, inner, lines, N, A, B, nullptr,
               nullptr, samp(1), black_border, MM, lines / batch, SV, SF);
    geom(0, len, inner, lines);
    SDB_LAUNCH((k_edt_pass<2, true>), cdiv(lines, EDT_THREADS), EDT_THREADS, 0, st, d_labels, len, inner, lines, N, B, nullptr, D2, M,
               samp(0), black_border, MM, lines / batch, SV, SF);
  }
  return 0;
}

}  // namespace

extern "C" int sdb_edt_prob(const int* d_labels, int ndim, const int* shape, int n_labels, const double* h_sampling, int black_border,
                            float* d_prob, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  int dims[3];
  long long N;
  if (check_shape("edt_prob", ndim, shape, dims, &N)) return 1;
  if (n_labels < 0) { sdb::set_error("edt_prob: n_labels must be >= 0"); return 1; }
  double s[3] = {1.0, 1.0, 1.0};
  for (int a = 0; a < ndim; ++a) {
    if (h_sampling) s[a] = h_sampling[a];
    if (!(s[a] > 0.0) || !std::isfinite(s[a])) { sdb::set_error("edt_prob: sampling must be positive and finite"); return 1; }
  }
  if (N == 0) return 0;
  if (n_labels == 0) { SDB_CUDA(cudaMemsetAsync(d_prob, 0, (size_t)N * 4, st)); return 0; }
  sdb::DevBuf d2, lmax;
  SDB_CUDA(d2.alloc((size_t)N * 8, st));
  SDB_CUDA(lmax.alloc((size_t)n_labels * 8, st));
  double* D2 = d2.as<double>();
  unsigned long long* M = lmax.as<unsigned long long>();
  if (edt_passes(d_labels, ndim, shape, 1, N, s, black_border, nullptr, n_labels, D2, M, st)) return 1;
  SDB_LAUNCH(k_edt_norm, grid_for(N, 256), 256, 0, st, d_labels, D2, M, N, d_prob);
  return 0;
}

namespace {

__global__ void k_minmax_init(int* __restrict__ mm, int batch) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < batch) { mm[2 * b] = INT_MAX; mm[2 * b + 1] = INT_MIN; }
}

// per-item label minimum and maximum; grid (blocks per item, batch)
__global__ void k_item_minmax(const int* __restrict__ lbl, long long n_item, int* __restrict__ mm) {
  const int b = blockIdx.y;
  const int* l = lbl + (long long)b * n_item;
  int lo = INT_MAX, hi = INT_MIN;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_item; i += (long long)gridDim.x * blockDim.x) {
    const int v = __ldg(l + i);
    lo = min(lo, v); hi = max(hi, v);
  }
  for (int o = 16; o > 0; o >>= 1) {
    lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if ((threadIdx.x & 31) == 0) { atomicMin(mm + 2 * b, lo); atomicMax(mm + 2 * b + 1, hi); }
}

// normalisation at the grid positions of every item: prob[b, o] (-1 where neg[b, o]) and dam[(b, o) * dm_stride], the
// unmasked value
__global__ void k_edt_norm_grid(const int* __restrict__ lbl, const double* __restrict__ d2, const unsigned long long* __restrict__ lmax,
                                int D, int H, int W, int gz, int gy, int gx, int Do, int Ho, int Wo, long long n_out,
                                const unsigned char* __restrict__ neg, float* __restrict__ prob, float* __restrict__ dam, int dm_stride) {
  for (long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x; o < n_out; o += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(o % Wo);
    const long long t = o / Wo;
    const int j = (int)(t % Ho);
    const long long u = t / Ho;
    const int i = (int)(u % Do);
    const long long b = u / Do;
    const long long src = ((b * D + (long long)i * gz) * H + (long long)j * gy) * W + (long long)k * gx;
    const int L = __ldg(lbl + src);
    float r = 0.f;
    if (L > 0) {
      const double m = __longlong_as_double((long long)__ldg(lmax + (L - 1)));
      r = __double2float_rn(__ddiv_rn(__dsqrt_rn(d2[src]), __dadd_rn(__dsqrt_rn(m), 1e-10)));
    }
    prob[o] = (neg && neg[o]) ? -1.f : r;
    if (dam) dam[o * dm_stride] = r;
  }
}

}  // namespace

extern "C" int sdb_edt_prob_batch(const int* d_labels, int ndim, int batch, const int* shape, int n_labels, const double* h_sampling,
                                  const int* grid, const unsigned char* d_neg, int* d_item_minmax, float* d_prob, float* d_dist_and_mask,
                                  int dm_stride, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  int dims[3];
  long long n_item;
  if (check_shape("edt_prob", ndim, shape, dims, &n_item)) return 1;
  if (batch < 1 || n_labels < 0) { sdb::set_error("edt_prob: batch must be >= 1 and n_labels >= 0"); return 1; }
  double s[3] = {1.0, 1.0, 1.0};
  int g[3] = {1, 1, 1}, od[3] = {1, 1, 1};
  for (int a = 0; a < ndim; ++a) {
    if (h_sampling) s[a] = h_sampling[a];
    if (!(s[a] > 0.0) || !std::isfinite(s[a])) { sdb::set_error("edt_prob: sampling must be positive and finite"); return 1; }
    if (grid[a] < 1) { sdb::set_error("edt_prob: grid values must be >= 1"); return 1; }
    g[3 - ndim + a] = grid[a];
    od[3 - ndim + a] = (shape[a] - 1) / grid[a] + 1;
  }
  if (n_item == 0) return 0;
  const long long N = n_item * batch;
  SDB_LAUNCH(k_minmax_init, cdiv(batch, 128), 128, 0, st, d_item_minmax, batch);
  SDB_LAUNCH(k_item_minmax, dim3((unsigned)std::min<long long>(cdiv(n_item, 256), 64), (unsigned)batch), 256, 0, st, d_labels, n_item,
             d_item_minmax);
  sdb::DevBuf d2, lmax;
  SDB_CUDA(d2.alloc((size_t)N * 8, st));
  SDB_CUDA(lmax.alloc((size_t)n_labels * 8, st));
  if (edt_passes(d_labels, ndim, shape, batch, N, s, 0, d_item_minmax, n_labels, d2.as<double>(), lmax.as<unsigned long long>(), st))
    return 1;
  const long long n_out = (long long)batch * od[0] * od[1] * od[2];
  SDB_LAUNCH(k_edt_norm_grid, grid_for(n_out, 256), 256, 0, st, d_labels, d2.as<double>(), lmax.as<unsigned long long>(), dims[0], dims[1],
             dims[2], g[0], g[1], g[2], od[0], od[1], od[2], n_out, d_neg, d_prob, d_dist_and_mask, dm_stride);
  return 0;
}

extern "C" int sdb_fill_label_holes(const int* d_labels, int ndim, const int* shape, int n_labels, int connectivity, int* d_out,
                                    sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  int dims[3];
  long long N;
  if (check_shape("fill_label_holes", ndim, shape, dims, &N)) return 1;
  if (n_labels < 0) { sdb::set_error("fill_label_holes: n_labels must be >= 0"); return 1; }
  if (connectivity < 1 || connectivity > ndim) { sdb::set_error("fill_label_holes: connectivity must lie in [1, ndim]"); return 1; }
  if (N == 0) return 0;
  SDB_CUDA(cudaMemsetAsync(d_out, 0, (size_t)N * 4, st));
  if (n_labels == 0) return 0;
  sdb::DevBuf cnt, sum, bmin, bmax;
  SDB_CUDA(cnt.alloc((size_t)n_labels * 8, st));
  SDB_CUDA(sum.alloc((size_t)n_labels * ndim * 8, st));
  SDB_CUDA(bmin.alloc((size_t)n_labels * ndim * 4, st));
  SDB_CUDA(bmax.alloc((size_t)n_labels * ndim * 4, st));
  if (sdb_region_stats(d_labels, ndim, shape, n_labels, cnt.as<long long>(), sum.as<long long>(), bmin.as<int>(), bmax.as<int>(), stream))
    return 1;
  std::vector<int> hmin((size_t)n_labels * ndim), hmax((size_t)n_labels * ndim);
  SDB_CUDA(cudaMemcpyAsync(hmin.data(), bmin.p, hmin.size() * 4, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaMemcpyAsync(hmax.data(), bmax.p, hmax.size() * 4, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  std::vector<Box> boxes(n_labels);
  std::vector<long long> off(n_labels + 1, 0);
  for (int i = 0; i < n_labels; ++i) {
    Box b{{0, 0, 0}, {1, 1, 1}};
    long long vol = 1;
    if (hmax[(size_t)i * ndim] >= 0) {                 // absent labels (none after a sequential relabelling) get an empty box
      for (int a = 0; a < ndim; ++a) {
        const int lo = std::max(hmin[(size_t)i * ndim + a] - 1, 0), hi = std::min(hmax[(size_t)i * ndim + a] + 1, shape[a] - 1);
        b.lo[3 - ndim + a] = lo;
        b.ext[3 - ndim + a] = hi - lo + 1;
        vol *= hi - lo + 1;
      }
    } else {
      vol = 0;
    }
    boxes[i] = b;
    off[i + 1] = off[i] + vol;
  }
  const long long total = off[n_labels];
  if (total > INT_MAX) {
    sdb::set_error("fill_label_holes: the grown bounding boxes hold more than 2^31 - 1 pixels in all; not supported");
    return 1;
  }
  Nbrs nb{};
  for (int dz = -1; dz <= 1; ++dz)
    for (int dy = -1; dy <= 1; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        const int d[3] = {dz, dy, dx};
        if (ndim == 2 && dz != 0) continue;
        int nz = 0, first = 0;
        for (int a = 0; a < 3; ++a) if (d[a]) { ++nz; if (!first) first = d[a]; }
        if (nz == 0 || nz > connectivity || first > 0) continue;
        nb.d[nb.n][0] = dz; nb.d[nb.n][1] = dy; nb.d[nb.n][2] = dx; ++nb.n;
      }
  sdb::DevBuf d_boxes, d_off, parent, outside;
  SDB_CUDA(d_boxes.alloc(sizeof(Box) * n_labels, st));
  SDB_CUDA(d_off.alloc(sizeof(long long) * (n_labels + 1), st));
  SDB_CUDA(parent.alloc((size_t)total * 4, st));
  SDB_CUDA(outside.alloc((size_t)total, st));
  SDB_CUDA(cudaMemcpyAsync(d_boxes.p, boxes.data(), sizeof(Box) * n_labels, cudaMemcpyHostToDevice, st));
  SDB_CUDA(cudaMemcpyAsync(d_off.p, off.data(), sizeof(long long) * (n_labels + 1), cudaMemcpyHostToDevice, st));
  SDB_CUDA(cudaMemsetAsync(outside.p, 0, (size_t)total, st));
  SDB_CUDA(cudaStreamSynchronize(st));               // the host vectors go out of scope on return
  if (total == 0) return 0;
  const Box* BX = d_boxes.as<Box>();
  const long long* OF = d_off.as<long long>();
  int* P = parent.as<int>();
  const int g = grid_for(total, 256);
  SDB_LAUNCH(k_fill_init, g, 256, 0, st, d_labels, dims[1], dims[2], BX, OF, n_labels, total, P);
  SDB_LAUNCH(k_fill_union, g, 256, 0, st, BX, OF, n_labels, total, nb, P);
  SDB_LAUNCH(k_fill_roots, g, 256, 0, st, BX, OF, n_labels, total, ndim, P, outside.as<unsigned char>());
  SDB_LAUNCH(k_fill_write, g, 256, 0, st, dims[1], dims[2], BX, OF, n_labels, total, P, outside.as<unsigned char>(), d_out);
  return 0;
}

namespace {

__global__ void k_clamp_minmax(int* __restrict__ lbl, long long n, int* __restrict__ mm) {
  int lo = INT_MAX, hi = INT_MIN;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int v = lbl[i];
    lo = min(lo, v); hi = max(hi, v);
    if (v < 0) lbl[i] = 0;
  }
  atomicMin(mm, lo);
  atomicMax(mm + 1, hi);
}

__global__ void k_inverse_map(const int* __restrict__ fwd, int max_label, int* __restrict__ inv) {
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v <= max_label; v += (long long)gridDim.x * blockDim.x) {
    const int t = fwd[v];
    if (v == 0) inv[0] = 0;
    else if (t > 0) inv[t] = (int)v;
  }
}

__global__ void k_apply_map(int* __restrict__ x, long long n, const int* __restrict__ map) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) x[i] = map[x[i]];
}

// host labels -> device map relabelled sequentially in ascending order (negative labels -> 0); the raw minimum and maximum
// (for the constant-image rule) and, when inv is given, the inverse map new id -> original label
int prepare_host_labels(const int* h_lbl, long long N, sdb::DevBuf& d, int* n_labels, int* raw_min, int* raw_max, sdb::DevBuf* inv,
                        cudaStream_t st) {
  SDB_CUDA(d.alloc((size_t)N * 4, st));
  SDB_CUDA(cudaMemcpyAsync(d.p, h_lbl, (size_t)N * 4, cudaMemcpyHostToDevice, st));
  sdb::DevBuf mm;
  SDB_CUDA(mm.alloc(8, st));
  const int init[2] = {INT_MAX, INT_MIN};
  SDB_CUDA(cudaMemcpyAsync(mm.p, init, 8, cudaMemcpyHostToDevice, st));
  SDB_LAUNCH(k_clamp_minmax, grid_for(N, 256), 256, 0, st, d.as<int>(), N, mm.as<int>());
  int h_mm[2];
  SDB_CUDA(cudaMemcpyAsync(h_mm, mm.p, 8, cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  *raw_min = h_mm[0]; *raw_max = h_mm[1];
  if (h_mm[1] > (1 << 30) - 1) { sdb::set_error("labels above 2^30 - 1 are not supported"); return 1; }
  const int max_label = std::max(h_mm[1], 0);
  sdb::DevBuf fwd;
  SDB_CUDA(fwd.alloc(((size_t)max_label + 3) * 4, st));
  if (sdb_relabel_sequential(d.as<int>(), N, max_label, 1, fwd.as<int>(), n_labels, st)) return 1;
  if (inv) {
    SDB_CUDA(inv->alloc(((size_t)*n_labels + 1) * 4, st));
    SDB_LAUNCH(k_inverse_map, grid_for((long long)max_label + 1, 256), 256, 0, st, fwd.as<int>(), max_label, inv->as<int>());
  }
  return 0;
}

}  // namespace

extern "C" void _LIB_edt_prob(const int* lbl, int ndim, const int* shape, const double* sampling, float* prob) {
  cudaStream_t st = 0;
  int dims[3];
  long long N = 0;
  auto run = [&]() -> int {
    if (check_shape("edt_prob", ndim, shape, dims, &N)) return 1;
    if (N == 0) return 0;
    sdb::DevBuf d, d_prob;
    int n_labels = 0, mn = 0, mx = 0;
    if (prepare_host_labels(lbl, N, d, &n_labels, &mn, &mx, nullptr, st)) return 1;
    SDB_CUDA(d_prob.alloc((size_t)N * 4, st));
    if (sdb_edt_prob(d.as<int>(), ndim, shape, n_labels, sampling, mn == mx && mx > 0, d_prob.as<float>(), st)) return 1;
    SDB_CUDA(cudaMemcpyAsync(prob, d_prob.p, (size_t)N * 4, cudaMemcpyDeviceToHost, st));
    SDB_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  if (run()) {
    for (long long i = 0; i < N; ++i) prob[i] = 0.f;
    cudaGetLastError();
    return;
  }
  sdb::set_error("");
}

extern "C" void _LIB_fill_label_holes(const int* lbl, int ndim, const int* shape, int connectivity, int* out) {
  cudaStream_t st = 0;
  int dims[3];
  long long N = 0;
  auto run = [&]() -> int {
    if (check_shape("fill_label_holes", ndim, shape, dims, &N)) return 1;
    if (N == 0) return 0;
    sdb::DevBuf d, d_out, inv;
    int n_labels = 0, mn = 0, mx = 0;
    if (prepare_host_labels(lbl, N, d, &n_labels, &mn, &mx, &inv, st)) return 1;
    SDB_CUDA(d_out.alloc((size_t)N * 4, st));
    if (sdb_fill_label_holes(d.as<int>(), ndim, shape, n_labels, connectivity, d_out.as<int>(), st)) return 1;
    SDB_LAUNCH(k_apply_map, grid_for(N, 256), 256, 0, st, d_out.as<int>(), N, inv.as<int>());
    SDB_CUDA(cudaMemcpyAsync(out, d_out.p, (size_t)N * 4, cudaMemcpyDeviceToHost, st));
    SDB_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  if (run()) {
    for (long long i = 0; i < N; ++i) out[i] = 0;
    cudaGetLastError();
    return;
  }
  sdb::set_error("");
}
