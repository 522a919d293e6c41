// polyfast.cuh -- closed-form overlap integral of two integer polygons, used as a conservative
// PRE-FILTER in front of the exact Clipper-equivalent sweep (clip2d.cuh).
//
// The reference decides   area(Clipper(P ∩ Q)) / min(area P, area Q) > threshold   (stardist2d.cpp:579-581)
// where Clipper works on integer coordinates and rounds every intersection vertex to the integer
// grid.  Its result therefore differs from the exact area of the intersection of the two integer
// polygons only by the area swept by those roundings.  This header computes
//
//     I = ∬ w_P · w_Q dA        (w = winding number; = area(P ∩ Q) for simple, equally oriented P, Q)
//
// exactly (integer predicates, fp64 accumulation) with one pass over the n×n edge pairs and no
// sorting, plus the data of a bound E on |area_Clipper − I|.  A pair whose ratio is farther than the
// bound from the threshold is decided here; everything else goes through the exact sweep, so the
// kept/suppressed result stays bit-identical to the reference (DESIGN.md §3.4 states the bound and
// how it is validated against the reference Clipper).
//
// Formula (Green / integration by parts for piecewise-constant integer fields):
//     I = ∮_∂P w_Q x dy + ∮_∂Q w_P x dy
// and along an edge the other polygon's winding number only changes at proper crossings, so with
// F_e(t,1) = ∫_t^1 x dy along e and Suf(i) = Σ_{k>=i} F_k(0,1):
//     I = w_Q(p_0)·A_P + w_P(q_0)·A_Q + Σ_crossings s·[F_e(t,1)+SufP(i+1)] − s·[F_f(u,1)+SufQ(j+1)]
// Degenerate contacts (shared vertices, collinear overlapping edges -- the rule, not the exception, on
// an integer grid) are resolved by a symbolic shift of Q by (ε, ε²): every predicate below is the sign
// of the ε-polynomial, so the computed I is that of a configuration in general position arbitrarily
// close to the input, and I is continuous in the vertices.
#pragma once
#include <stdint.h>
#include <math.h>
#ifndef SD_HD
#ifdef __CUDACC__
#define SD_HD __host__ __device__
#else
#define SD_HD
#endif
#endif

namespace sdfast {

typedef long long i64;

struct Edge {           // directed edge v0 -> v1
  int32_t x0, y0, x1, y1;
};
struct Box { int32_t xl, xh, yl, yh; };
SD_HD inline Box edge_box(const Edge& e) {
  Box b;
  b.xl = e.x0 < e.x1 ? e.x0 : e.x1; b.xh = e.x0 < e.x1 ? e.x1 : e.x0;
  b.yl = e.y0 < e.y1 ? e.y0 : e.y1; b.yh = e.y0 < e.y1 ? e.y1 : e.y0;
  return b;
}

SD_HD inline double edge_F(int32_t x0, int32_t y0, int32_t x1, int32_t y1) {   // ∫ x dy over the edge
  return 0.5 * (double)((i64)y1 - y0) * (double)((i64)x0 + x1);
}

// Symbolic perturbation: Q is shifted by δ = (ε, ε²).
//   orient(q0+δ, q1+δ, p) = base + fy·ε − fx·ε²   (f = q1 − q0)   -> sign at base == 0: tie_edge(fx, fy)
//   orient(p0, p1, q+δ)   = base − ey·ε + ex·ε²   (e = p1 − p0)   -> sign at base == 0: tie_point(ex, ey)
template <typename T> SD_HD inline int tie_edge(T fx, T fy) { return (fy > 0 || (fy == 0 && fx < 0)) ? 1 : -1; }
template <typename T> SD_HD inline int tie_point(T ex, T ey) { return (ey < 0 || (ey == 0 && ex > 0)) ? 1 : -1; }
template <typename T> SD_HD inline int sgn_tie(T o, int tie) { return o > 0 ? 1 : (o < 0 ? -1 : tie); }
SD_HD inline int sgn_shifted_edge(i64 base, i64 fx, i64 fy) { return sgn_tie(base, tie_edge(fx, fy)); }
SD_HD inline int sgn_shifted_point(i64 base, i64 ex, i64 ey) { return sgn_tie(base, tie_point(ex, ey)); }

struct Accum {
  double I;        // crossing terms of the overlap integral
  double len;      // Σ over crossings of (|e| + |f|)
  int K;           // number of proper crossings
  SD_HD void clear() { I = 0; len = 0; K = 0; }
};

// Proper-crossing predicate of the edge pair (e of P, f of Q) under the perturbation, branch free.
// T = int32_t is exact while every coordinate difference is below 2^14 (|coordinates| <= 8191: products < 2^28,
// orientations < 2^29), T = int64 otherwise.   o1 = orient(p0,p1,q0), o2 = orient(p0,p1,q1),
// o3 = orient(q0,q1,p0), o4 = orient(q0,q1,p1).
template <typename T>
SD_HD inline bool crossing_test(T ex, T ey, T fx, T fy, T o1, T o2, T o3, T o4, int tieP, int tieQ) {
  const int s1 = sgn_tie(o1, tieP), s2 = sgn_tie(o2, tieP), s3 = sgn_tie(o3, tieQ), s4 = sgn_tie(o4, tieQ);
  return (s1 != s2) & (s3 != s4) & ((ex | ey) != 0) & ((fx | fy) != 0);
}
// Contribution of an established proper crossing.  e_suf / f_suf = Σ_{k > edge} F_k(0,1) of the two polygons.
// Moving along e we end on the left of f (w_Q += 1) iff o4 (perturbed) > 0.
// t, u only need ~1e-7: an error dt moves F by |ey * x| dt, far below the bound (which is >= 2).
template <typename T>
SD_HD inline void crossing_contrib(const Edge& e, const Edge& f, T ex, T ey, T fx, T fy, T o1, T o2, T o3, T o4, int tieQ,
                                   double e_suf, double f_suf, Accum& acc) {
  const double s = (double)sgn_tie(o4, tieQ);
  const double t = (double)((float)o3 / ((float)o3 - (float)o4));      // on e   (o3 != o4: signs differ, not both 0)
  const double u = (double)((float)o1 / ((float)o1 - (float)o2));      // on f
  const double Fe = (double)ey * ((double)e.x0 * (1.0 - t) + 0.5 * (double)ex * (1.0 - t * t));
  const double Ff = (double)fy * ((double)f.x0 * (1.0 - u) + 0.5 * (double)fx * (1.0 - u * u));
  acc.I += s * ((Fe + e_suf) - (Ff + f_suf));
  acc.len += (double)(sqrtf((float)(ex * ex + ey * ey)) + sqrtf((float)(fx * fx + fy * fy))) * 1.000001;
  acc.K += 1;
}
template <typename T>
SD_HD inline void edge_pair(const Edge& e, const double* e_suf, const Edge& f, const double* f_suf, Accum& acc) {
  const T ex = (T)e.x1 - (T)e.x0, ey = (T)e.y1 - (T)e.y0;
  const T fx = (T)f.x1 - (T)f.x0, fy = (T)f.y1 - (T)f.y0;
  const T o1 = ex * ((T)f.y0 - (T)e.y0) - ey * ((T)f.x0 - (T)e.x0);
  const T o2 = ex * ((T)f.y1 - (T)e.y0) - ey * ((T)f.x1 - (T)e.x0);
  const T o3 = fx * ((T)e.y0 - (T)f.y0) - fy * ((T)e.x0 - (T)f.x0);
  const T o4 = fx * ((T)e.y1 - (T)f.y0) - fy * ((T)e.x1 - (T)f.x0);
  const int tieP = tie_point(ex, ey), tieQ = tie_edge(fx, fy);
  if (!crossing_test(ex, ey, fx, fy, o1, o2, o3, o4, tieP, tieQ)) return;
  crossing_contrib(e, f, ex, ey, fx, fy, o1, o2, o3, o4, tieQ, *e_suf, *f_suf, acc);
}

// winding-number contribution of edge f of Q around p0 − δ (ray towards +x)
SD_HD inline int wind_Q_edge(const Edge& f, int32_t px, int32_t py) {
  const bool a0 = f.y0 >= py, a1 = f.y1 >= py;
  if (a0 == a1) return 0;
  const i64 fx = (i64)f.x1 - f.x0, fy = (i64)f.y1 - f.y0;
  const i64 base = fx * ((i64)py - f.y0) - fy * ((i64)px - f.x0);
  const int sg = sgn_shifted_edge(base, fx, fy);
  if (a1) return sg > 0 ? 1 : 0;     // upward edge, point on its left
  return sg < 0 ? -1 : 0;            // downward edge, point on its right
}
// winding-number contribution of edge e of P around q0 + δ
SD_HD inline int wind_P_edge(const Edge& e, int32_t qx, int32_t qy) {
  const bool a0 = e.y0 > qy, a1 = e.y1 > qy;
  if (a0 == a1) return 0;
  const i64 ex = (i64)e.x1 - e.x0, ey = (i64)e.y1 - e.y0;
  const i64 base = ex * ((i64)qy - e.y0) - ey * ((i64)qx - e.x0);
  const int sg = sgn_shifted_point(base, ex, ey);
  if (a1) return sg > 0 ? 1 : 0;
  return sg < 0 ? -1 : 0;
}

// Bound on |area_Clipper − I|.
//  * every true intersection vertex of the result is moved by at most (1/2, 1/2) by Clipper's rounding;
//    moving one vertex of a polygon by d changes its area by |d × (next − prev)|/2, and next/prev lie on
//    the two crossing edges (possibly moved themselves): <= 0.354·(|e|+|f|) + 1/2 per crossing;
//  * edges whose rounded scanline positions swap without a true crossing, and contacts along shared
//    edges, add or drop slivers at most one pixel wide along one edge: covered by 2 (maxlen_P + maxlen_Q) + 4
//    (near-tangent, almost congruent polygons are the worst observed case: |area_Clipper - I| = 6.0 at K = 2);
//  * the float32 accumulation of the shoelace sum (area_from_path, stardist2d.cpp:128-138): partial sums
//    are below n_out·max|coord|·maxlen, n_out additions of relative error 2^-24 each.
// The geometric part carries a factor 1.25.  tests/tools/polyfast_fuzz.py measures the observed maximum of
// |area_Clipper − I| / bound over tens of millions of pairs (tests/tools/polyfast_fuzz.py, DESIGN.md §5).
SD_HD inline double clipper_bound(const Accum& acc, double maxlen_sum, double max_abs_coord, int n) {
  const double geom = 1.25 * (0.354 * acc.len + 0.5 * acc.K) + 2.0 * maxlen_sum + 4.0
                      + 4.0e-7 * acc.K * max_abs_coord * maxlen_sum;        // float t, u at the crossings
  const double n_out = (double)(2 * n + 8);
  const double f32 = n_out * n_out * max_abs_coord * maxlen_sum * 6.0e-8;
  return geom + f32;
}

// Decision against the reference's test  (float)(area / den) > threshold  (stardist2d.cpp:580-581), with
// area_Clipper in [I - bound, I + bound] and the float conversion monotone:
//   1 = suppressed for sure, 0 = not suppressed for sure, -1 = needs the exact sweep.
SD_HD inline int decide(double I, double bound, double den, float threshold) {
  const float lo = (float)((I - bound) / den), hi = (float)((I + bound) / den);
  if (lo > threshold) return 1;
  if (!(hi > threshold)) return 0;
  return -1;
}

}  // namespace sdfast
