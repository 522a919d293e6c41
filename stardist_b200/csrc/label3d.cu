// label3d.cu -- polyhedron_to_label on the GPU.
//
// Reference: stardist/lib/stardist3d_impl.cpp:1404-1525 (_COMMON_polyhedron_to_label), called from
// stardist/geometry/geom3d.py:100-198 with polyhedra sorted by descending probability.  Per
// polyhedron: integer bbox via lrint (:536-567), then every voxel of the (clipped) bbox is tested;
// the first polyhedron that covers a voxel wins (`result==0 ? labels[i] : result`), or, with
// use_overlap_label, every further cover writes overlap_label (:1508-1517).
//
// render_mode 0 "full":  inside = kernel(p) || (hull(p) && polyhedron(p))            (:1469-1476)
//   kernel(p)     -- float-built face planes evaluated in double (build_halfspace / point_in_halfspaces)
//   polyhedron(p) -- union of the (centre,A,B,C) tetrahedra, float determinants `det >= 0`
//   hull(p)       -- Qhull facet planes of the vertices.  polyhedron(p) implies hull(p) geometrically
//                    (every tetrahedron lies in the hull), so the hull test is only an accelerator in
//                    the reference; it is dropped here.  A voxel can differ only if it lies on a hull
//                    facet to within Qhull's last-bit rounding (lattice-aligned inputs), DESIGN.md.
// render_mode 1 "kernel", 3 "bbox", 4 "debug" as in the reference; 2 "hull" uses gift-wrapped facets.
//
// "First cover wins" == per-voxel minimum over the polyhedron index -> atomicMin on a rank image,
// then one pass maps ranks to labels (and overlaps to overlap_label).  Compile with -fmad=false.
#include <vector>
#include <algorithm>
#include "common.cuh"
#include "geom3d.cuh"
#include "bins3d.cuh"
#include "nms3d_pair.cuh"
#include "../../include/stardist_b200.h"

namespace {

using sdb::cdiv;
constexpr int MAXR = sd3::SD3_MAX_RAYS, MAXF = sd3::SD3_MAX_FACES;
constexpr int RANK_NONE = 0x7fffffff;
__device__ int g_cull3d = 3;      // bit 0: sphere culling, bit 1: direction bins in k_paint3d (sdb_label3d_set_cull; results identical)

struct PaintArgs {
  const float* dist; const float* points; const float* verts; const int* faces;
  int n_polys, n_rays, n_faces, nz, ny, nx, mode;
  // sequential variant (labels == 0 among the inputs, or overlap_label == 0): one launch per polyhedron, the reference's
  // update rule applied in place (stardist3d_impl.cpp:1508-1517)
  int poly0; int* direct; const int* labels; int use_overlap, overlap_label;
  int hull_conj;      // mode 0 only: apply the reference's hull conjunct (ray sets with degenerate faces, see sdb_polyhedron_to_label)
};

// render_mode 2 only: hull facet planes per polyhedron (one thread each; gift wrapping is serial)
__global__ void k_hull3d(PaintArgs A, double* __restrict__ hull_planes, int* __restrict__ hull_count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n_polys) return;
  double pts[3 * MAXR]; uint32_t ed[(MAXR * MAXR + 31) / 32]; int16_t st[3 * 4 * MAXR];
  const float* d = A.dist + (size_t)i * A.n_rays;
  for (int j = 0; j < A.n_rays; ++j)
    for (int c = 0; c < 3; ++c) pts[3 * j + c] = (double)(A.points[3 * i + c] + d[j] * A.verts[3 * j + c]);
  sd3::demote_duplicate_points(pts, A.n_rays);      // coincident ray directions with equal distances (Rays_Cartesian poles)
  hull_count[i] = sd3::convex_hull_planes(pts, A.n_rays, reinterpret_cast<sd3::Plane*>(hull_planes + (size_t)i * 4 * A.n_faces),
                                          A.n_faces, ed, st, 4 * MAXR);
}

using sdbins::FaceBins; using sdbins::bin_of; using sdbins::k_build_bins; using sdbins::BIN_N; using sdbins::BIN_CAP;

// one block per polyhedron
__global__ void __launch_bounds__(256)
k_paint3d(PaintArgs A, int* __restrict__ rank_img, int* __restrict__ second_img, int* __restrict__ debug_img,
          const double* __restrict__ hull_planes, const int* __restrict__ hull_count, FaceBins B) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* pv = reinterpret_cast<float*>(smem_raw);                         // [R][3]
  int* sfaces = reinterpret_cast<int*>(pv + 3 * A.n_rays);                // [F][3]
  double* hs = reinterpret_cast<double*>(smem_raw + ((3 * A.n_rays * 4 + 3 * A.n_faces * 4 + 15) / 16) * 16);   // [F][4] kernel planes / hull planes
  __shared__ int bbox[6];
  __shared__ float center[3];
  __shared__ int n_hull;
  const int i = blockIdx.x + A.poly0;
  const float* d = A.dist + (size_t)i * A.n_rays;
  if (threadIdx.x < 3) center[threadIdx.x] = A.points[3 * i + threadIdx.x];
  __syncthreads();
  for (int j = threadIdx.x; j < A.n_rays; j += blockDim.x) {
    pv[3 * j] = center[0] + d[j] * A.verts[3 * j];
    pv[3 * j + 1] = center[1] + d[j] * A.verts[3 * j + 1];
    pv[3 * j + 2] = center[2] + d[j] * A.verts[3 * j + 2];
  }
  for (int j = threadIdx.x; j < 3 * A.n_faces; j += blockDim.x) sfaces[j] = A.faces[j];
  if (threadIdx.x == 0) {
    int z1 = INT32_MAX, z2 = -1, y1 = INT32_MAX, y2 = -1, x1 = INT32_MAX, x2 = -1;
    for (int j = 0; j < A.n_rays; ++j) {
      const int iz = sd3::round_to_int(center[0] + d[j] * A.verts[3 * j]);
      const int iy = sd3::round_to_int(center[1] + d[j] * A.verts[3 * j + 1]);
      const int ix = sd3::round_to_int(center[2] + d[j] * A.verts[3 * j + 2]);
      z1 = min(z1, iz); z2 = max(z2, iz); y1 = min(y1, iy); y2 = max(y2, iy); x1 = min(x1, ix); x2 = max(x2, ix);
    }
    bbox[0] = max(0, z1); bbox[1] = min(A.nz - 1, z2); bbox[2] = max(0, y1); bbox[3] = min(A.ny - 1, y2);
    bbox[4] = max(0, x1); bbox[5] = min(A.nx - 1, x2);
    n_hull = 0;
  }
  __syncthreads();
  if (A.mode == 2) {
    // hull facets were computed by k_hull3d (rarely used render mode)
    if (threadIdx.x == 0) n_hull = hull_count[i];
    for (int f = threadIdx.x; f < 4 * A.n_faces; f += blockDim.x) hs[f] = hull_planes[(size_t)i * 4 * A.n_faces + f];
  } else {
    for (int f = threadIdx.x; f < A.n_faces; f += blockDim.x)
      sd3::build_halfspace(&pv[3 * sfaces[3 * f]], &pv[3 * sfaces[3 * f + 1]], &pv[3 * sfaces[3 * f + 2]], &hs[4 * f]);
    if (A.mode == 0 && A.hull_conj) {      // hull facets behind the kernel planes (the launch reserved the room)
      if (threadIdx.x == 0) n_hull = hull_count[i];
      for (int f = threadIdx.x; f < 4 * A.n_faces; f += blockDim.x) hs[4 * A.n_faces + f] = hull_planes[(size_t)i * 4 * A.n_faces + f];
    }
  }
  __syncthreads();
  // Sphere culling of the bounding box (render modes "full" / "kernel"), exactness preserving by margin:
  //  * a voxel farther from the centre than every vertex (+ margin) lies outside the polyhedron -- every tetrahedron
  //    (centre, A, B, C) is inside that ball -- so the kernel planes and the float determinants reject it anyway;
  //  * a voxel inside the ball inscribed in the kernel planes (the planes as built above, in double; - margin) satisfies
  //    every plane inequality, i.e. point_in_halfspaces(kernel) is true and the voxel is labelled in both modes.
  // The margins (1e-3 relative + 0.05 voxel) are ~1e4 x the rounding of the tests they short-cut.  Switched off for
  // polyhedra with a near-degenerate face (|normal| < 1e-6 r^2), where the determinant signs are noise-dominated.
  __shared__ double cull_out2, cull_in2;
  if (threadIdx.x == 0) {
    double r2 = 0, rho = 1e300, nmin = 1e300;
    for (int j = 0; j < A.n_rays; ++j) {
      const double a = (double)pv[3 * j] - center[0], b = (double)pv[3 * j + 1] - center[1], c = (double)pv[3 * j + 2] - center[2];
      r2 = fmax(r2, a * a + b * b + c * c);
    }
    if (A.mode <= 1) {
      for (int f = 0; f < A.n_faces; ++f) {
        const double nn = sqrt(hs[4 * f] * hs[4 * f] + hs[4 * f + 1] * hs[4 * f + 1] + hs[4 * f + 2] * hs[4 * f + 2]);
        const double v = hs[4 * f] * center[0] + hs[4 * f + 1] * center[1] + hs[4 * f + 2] * center[2] + hs[4 * f + 3];
        nmin = fmin(nmin, nn);
        rho = fmin(rho, nn > 0 ? -v / nn : -1.0);
      }
    }
    const double r = sqrt(r2);
    const bool ok = (g_cull3d & 1) && A.mode <= 1 && nmin >= 1e-6 * r2 && r2 > 0;
    const double ro = r * 1.001 + 0.05, ri = rho * 0.999 - 0.05;
    cull_out2 = ok ? ro * ro : 1e300;
    cull_in2 = (ok && ri > 0) ? ri * ri : -1.0;
  }
  __syncthreads();
  const int bz = bbox[1] - bbox[0] + 1, by = bbox[3] - bbox[2] + 1, bx = bbox[5] - bbox[4] + 1;
  if (bz <= 0 || by <= 0 || bx <= 0) return;
  const long long nvox = (long long)bz * by * bx;
  for (long long q = threadIdx.x; q < nvox; q += blockDim.x) {
    const int x = bbox[4] + (int)(q % bx), y = bbox[2] + (int)((q / bx) % by), z = bbox[0] + (int)(q / ((long long)bx * by));
    const float fz = (float)z, fy = (float)y, fx = (float)x;
    bool inside = false;
    {
      const double a = (double)z - center[0], b = (double)y - center[1], c = (double)x - center[2];
      const double d2 = a * a + b * b + c * c;
      if (d2 > cull_out2) continue;
      if (d2 < cull_in2) inside = true;
    }
    auto in_planes = [&](int cnt) {
      for (int f = 0; f < cnt; ++f)
        if (hs[4 * f] * fz + hs[4 * f + 1] * fy + hs[4 * f + 2] * fx + hs[4 * f + 3] > 0) return false;
      return true;
    };
    if (inside) { /* inside the kernel's inscribed ball: labelled in modes "full" and "kernel" */ }
    else if (A.mode == 0 && B.count && (g_cull3d & 2)) {
      // kernel || polyhedron with the direction bins: the tetrahedra whose cone can contain this voxel first (the OR over
      // all F reduces to them); if none contains it, the kernel planes -- the binned faces' planes first, they are the
      // ones an outside voxel violates -- decide
      const int b = bin_of(fz - center[0], fy - center[1], fx - center[2]);
      const int cnt = b >= 0 ? __ldg(B.count + b) : -1;
      if (cnt < 0) inside = in_planes(A.n_faces) || sd3::inside_polyhedron(fz, fy, fx, center, pv, sfaces, A.n_faces);
      else {
        const int* lst = B.faces + b * BIN_CAP;
        bool poly = false;
        for (int i = 0; i < cnt && !poly; ++i) {
          const int f = __ldg(lst + i);
          const int iA = sfaces[3 * f], iB = sfaces[3 * f + 1], iC = sfaces[3 * f + 2];
          poly = sd3::inside_tetrahedron(fz, fy, fx, center[0], center[1], center[2], pv[3 * iA], pv[3 * iA + 1], pv[3 * iA + 2],
                                         pv[3 * iB], pv[3 * iB + 1], pv[3 * iB + 2], pv[3 * iC], pv[3 * iC + 1], pv[3 * iC + 2]);
        }
        if (poly) inside = true;
        else {
          bool ker = true;
          for (int i = 0; i < cnt && ker; ++i) {
            const int f = __ldg(lst + i);
            ker = !(hs[4 * f] * fz + hs[4 * f + 1] * fy + hs[4 * f + 2] * fx + hs[4 * f + 3] > 0);
          }
          inside = ker && in_planes(A.n_faces);
        }
      }
    }
    else if (A.mode == 0 && A.hull_conj) {
      // kernel || (hull && polyhedron), the reference's rule in full (stardist3d_impl.cpp:1475-1477)
      inside = in_planes(A.n_faces);
      if (!inside && n_hull >= 4 && sd3::inside_polyhedron(fz, fy, fx, center, pv, sfaces, A.n_faces)) {
        const double* hh = hs + 4 * A.n_faces;
        bool in_hull = true;
        for (int f = 0; f < n_hull && in_hull; ++f) in_hull = !(hh[4 * f] * fz + hh[4 * f + 1] * fy + hh[4 * f + 2] * fx + hh[4 * f + 3] > 0);
        inside = in_hull;
      }
    }
    else if (A.mode == 0) inside = in_planes(A.n_faces) || sd3::inside_polyhedron(fz, fy, fx, center, pv, sfaces, A.n_faces);
    else if (A.mode == 1) inside = in_planes(A.n_faces);
    else if (A.mode == 2) inside = (n_hull >= 4) && in_planes(n_hull);
    else if (A.mode == 3) inside = true;
    else {
      // "debug": flag kernel && !polyhedron with -1, label nothing
      bool ker = true;
      for (int f = 0; f < A.n_faces && ker; ++f)
        ker = sd3::inside_halfspace(fz, fy, fx, pv[3 * sfaces[3 * f]], pv[3 * sfaces[3 * f] + 1], pv[3 * sfaces[3 * f] + 2],
                                    pv[3 * sfaces[3 * f + 1]], pv[3 * sfaces[3 * f + 1] + 1], pv[3 * sfaces[3 * f + 1] + 2],
                                    pv[3 * sfaces[3 * f + 2]], pv[3 * sfaces[3 * f + 2] + 1], pv[3 * sfaces[3 * f + 2] + 2]);
      if (ker && !sd3::inside_polyhedron(fz, fy, fx, center, pv, sfaces, A.n_faces))
        debug_img[((size_t)z * A.ny + y) * A.nx + x] = 1;
      continue;
    }
    if (inside && A.direct) {
      const size_t off = ((size_t)z * A.ny + y) * A.nx + x;
      const int cur = A.direct[off];
      A.direct[off] = cur == 0 ? A.labels[i] : (A.use_overlap ? A.overlap_label : cur);
    } else if (inside) {
      const size_t off = ((size_t)z * A.ny + y) * A.nx + x;
      const int old = atomicMin(&rank_img[off], i);
      if (second_img) {
        // track the second smallest covering index as well (needed for labels==0 corner cases and
        // overlap_label): second = min over covers excluding the minimum
        const int loser = max(old, i);
        if (old != i && loser != RANK_NONE) atomicMin(&second_img[off], loser);
      }
    }
  }
}

__global__ void k_finalize3d(int* __restrict__ out, const int* __restrict__ rank_img, const int* __restrict__ second_img,
                             const int* __restrict__ debug_img, long long nvox, const int* __restrict__ labels,
                             int use_overlap, int overlap_label, int mode) {
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < nvox; v += (long long)gridDim.x * blockDim.x) {
    if (mode == 4) { out[v] = debug_img[v] ? -1 : 0; continue; }
    const int r = rank_img[v];
    int val = 0;
    if (r != RANK_NONE) {
      val = labels[r];
      if (use_overlap && second_img[v] != RANK_NONE) val = overlap_label;
    }
    out[v] = val;
  }
}

__global__ void k_count_zero(const int* __restrict__ labels, int n, int* __restrict__ flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && labels[i] == 0) *flag = 1;
}

__global__ void k_fill(int* p, long long n, int v) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = v;
}

}  // namespace

extern "C" int sdb_polyhedron_to_label(const float* d_dist, const float* d_points, const float* d_verts,
                                       const int* d_faces, int n_polys, int n_rays, int n_faces,
                                       const int* d_labels, int nz, int ny, int nx, int render_mode,
                                       int use_overlap_label, int overlap_label, int* d_result,
                                       sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (n_rays > MAXR || n_faces > MAXF) { sdb::set_error("polyhedron_to_label: too many rays/faces"); return 1; }
  if (render_mode < 0 || render_mode > 4) { sdb::set_error("polyhedron_to_label: unknown render mode"); return 1; }
  const long long nvox = (long long)nz * ny * nx;
  const int fb = (int)std::min<long long>(cdiv(nvox, 256), 132 * 16);
  if (nvox == 0) return 0;
  // Render mode "full" here is kernel || inside_polyhedron, the reference's is kernel || (hull && inside_polyhedron)
  // (stardist3d_impl.cpp:1475-1477).  inside_polyhedron lies inside the hull -- except for DEGENERATE faces of the ray
  // triangulation (Rays_Cartesian's zero-area pole faces): their tetrahedra "contain" whole planes through the centre, which
  // the reference's hull test cuts back to the hull and which would otherwise be painted across the bounding box.  For a ray
  // set with such faces the hull conjunct is applied with the gift-wrapping facets (k_hull3d); the direction bins are not
  // used.  Ray sets without degenerate faces (every golden-spiral / subdivision set) are rendered as before.
  bool hull_conj = false;
  if (render_mode == 0 && n_polys > 0 && n_faces > 0) {
    std::vector<float> hv((size_t)3 * n_rays); std::vector<int> hf((size_t)3 * n_faces);
    SDB_CUDA(cudaMemcpyAsync(hv.data(), d_verts, hv.size() * 4, cudaMemcpyDeviceToHost, st));
    SDB_CUDA(cudaMemcpyAsync(hf.data(), d_faces, hf.size() * 4, cudaMemcpyDeviceToHost, st));
    SDB_CUDA(cudaStreamSynchronize(st));
    bool valid = true;
    for (size_t k = 0; k < hf.size() && valid; ++k) valid = hf[k] >= 0 && hf[k] < n_rays;
    for (int f = 0; f < n_faces && valid && !hull_conj; ++f) hull_conj = sd3::ray_face_is_degenerate(hv.data(), hf.data(), f);
  }
  // labels == 0 ("paints nothing, and is painted over") and overlap_label == 0 make the reference's in-place rule order
  // dependent beyond "first cover wins": detect them (one 4-byte read-back) and run the polyhedra one launch at a time
  bool sequential = use_overlap_label && overlap_label == 0;
  if (!sequential && n_polys > 0 && render_mode != 4) {
    sdb::DevBuf b_z;
    SDB_CUDA(b_z.alloc(4, st));
    SDB_CUDA(cudaMemsetAsync(b_z.p, 0, 4, st));
    SDB_LAUNCH(k_count_zero, cdiv(n_polys, 256), 256, 0, st, d_labels, n_polys, b_z.as<int>());
    int hz = 0;
    SDB_CUDA(cudaMemcpyAsync(&hz, b_z.p, 4, cudaMemcpyDeviceToHost, st));
    SDB_CUDA(cudaStreamSynchronize(st));
    sequential = hz != 0;
  }
  if (sequential && render_mode != 4) {
    SDB_CUDA(cudaMemsetAsync(d_result, 0, (size_t)nvox * sizeof(int), st));
    PaintArgs A{d_dist, d_points, d_verts, d_faces, n_polys, n_rays, n_faces, nz, ny, nx, render_mode, 0, d_result, d_labels, use_overlap_label, overlap_label, hull_conj ? 1 : 0};
    const size_t smem = ((3 * n_rays * 4 + 3 * n_faces * 4 + 15) / 16) * 16 + (size_t)n_faces * 4 * sizeof(double) * (hull_conj ? 2 : 1);
    sdb::DevBuf b_hull, b_hcnt;
    if (render_mode == 2 || hull_conj) {
      SDB_CUDA(b_hull.alloc((size_t)n_polys * n_faces * 4 * sizeof(double), st));
      SDB_CUDA(b_hcnt.alloc((size_t)n_polys * sizeof(int), st));
      SDB_LAUNCH(k_hull3d, cdiv(n_polys, 32), 32, 0, st, A, b_hull.as<double>(), b_hcnt.as<int>());
    }
    for (int i = 0; i < n_polys; ++i) {
      A.poly0 = i;
      SDB_LAUNCH(k_paint3d, 1, 256, smem, st, A, nullptr, nullptr, nullptr, b_hull.as<double>(), b_hcnt.as<int>(), FaceBins{nullptr, nullptr});
    }
    return 0;
  }
  sdb::DevBuf b_rank, b_second, b_debug;
  SDB_CUDA(b_rank.alloc((size_t)nvox * sizeof(int), st));
  SDB_LAUNCH(k_fill, fb, 256, 0, st, b_rank.as<int>(), nvox, RANK_NONE);
  if (use_overlap_label) {
    SDB_CUDA(b_second.alloc((size_t)nvox * sizeof(int), st));
    SDB_LAUNCH(k_fill, fb, 256, 0, st, b_second.as<int>(), nvox, RANK_NONE);
  }
  if (render_mode == 4) {
    SDB_CUDA(b_debug.alloc((size_t)nvox * sizeof(int), st));
    SDB_CUDA(cudaMemsetAsync(b_debug.p, 0, (size_t)nvox * sizeof(int), st));
  }
  if (n_polys > 0) {
    PaintArgs A{d_dist, d_points, d_verts, d_faces, n_polys, n_rays, n_faces, nz, ny, nx, render_mode, 0, nullptr, d_labels, use_overlap_label, overlap_label, hull_conj ? 1 : 0};
    const size_t smem = ((3 * n_rays * 4 + 3 * n_faces * 4 + 15) / 16) * 16 + (size_t)n_faces * 4 * sizeof(double) * (hull_conj ? 2 : 1);
    sdb::DevBuf b_hull, b_hcnt;
    if (render_mode == 2 || hull_conj) {
      SDB_CUDA(b_hull.alloc((size_t)n_polys * n_faces * 4 * sizeof(double), st));
      SDB_CUDA(b_hcnt.alloc((size_t)n_polys * sizeof(int), st));
      SDB_LAUNCH(k_hull3d, cdiv(n_polys, 32), 32, 0, st, A, b_hull.as<double>(), b_hcnt.as<int>());
    }
    sdb::ProfSpan sp;
    sdb::profile_begin("nms3d_paint", st, &sp);
    sdb::DevBuf b_bcnt, b_bfaces;
    FaceBins FB{nullptr, nullptr};
    if (render_mode == 0 && !hull_conj) {
      SDB_CUDA(b_bcnt.alloc(BIN_N * sizeof(int), st)); SDB_CUDA(b_bfaces.alloc((size_t)BIN_N * BIN_CAP * sizeof(int), st));
      FB.count = b_bcnt.as<int>(); FB.faces = b_bfaces.as<int>();
      SDB_LAUNCH(k_build_bins, BIN_N, 128, 0, st, d_verts, d_faces, n_faces, FB);
    }
    SDB_LAUNCH(k_paint3d, n_polys, 256, smem, st, A, b_rank.as<int>(), use_overlap_label ? b_second.as<int>() : nullptr,
               render_mode == 4 ? b_debug.as<int>() : nullptr, b_hull.as<double>(), b_hcnt.as<int>(), FB);
    sdb::profile_end("nms3d_paint", st, &sp);
  }
  SDB_LAUNCH(k_finalize3d, fb, 256, 0, st, d_result, b_rank.as<int>(), use_overlap_label ? b_second.as<int>() : nullptr,
             render_mode == 4 ? b_debug.as<int>() : nullptr, nvox, d_labels, use_overlap_label, overlap_label, render_mode);
  return 0;
}

// sphere culling of the bounding-box voxels in k_paint3d: 1 (default) on, 0 off -- identical label maps (tests)
extern "C" int sdb_label3d_set_cull(int on) {
  const int v = on & 3;          // 0: off, 1: sphere culling, 2: direction bins, 3: both (default)
  SDB_CUDA(cudaMemcpyToSymbol(g_cull3d, &v, sizeof(int)));
  return 0;
}

// ---------------------------------------------------------------------------------------------------------
// relabel_sequential (stardist/matching.py:319-406; caller model3d.py:645): the labels that occur in the map
// are renumbered offset, offset+1, ... in ascending order, 0 stays 0.  Three passes: presence flags (one int per
// label, benign store race), a single-CTA scan of the flags into the forward map, and -- only if some label is
// missing or offset != 1 -- the rewrite of the map.  Integer work, bit-exact.
namespace {
__global__ void __launch_bounds__(256) k_mark_labels(const int* __restrict__ lab, long long n, int max_label,
                                                     int* __restrict__ present, int* __restrict__ bad) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long n4 = n >> 2;
  const int4* lab4 = reinterpret_cast<const int4*>(lab);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const int4 v = lab4[i];
    const int a[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (a[k] < 0 || a[k] > max_label) *bad = 1;
      else if (a[k] > 0) present[a[k]] = 1;
    }
  }
  for (long long i = (n4 << 2) + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int v = lab[i];
    if (v < 0 || v > max_label) *bad = 1;
    else if (v > 0) present[v] = 1;
  }
}

// present[1..max_label] (0/1) -> forward map in place; count[0] = number of labels present
__global__ void __launch_bounds__(1024) k_scan_labels(int* __restrict__ present, int max_label, int offset, int* __restrict__ count) {
  __shared__ int s_warp[32];
  __shared__ int s_carry;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) s_carry = 0;
  __syncthreads();
  for (int base = 1; base <= max_label; base += 1024) {
    const int idx = base + tid;
    const int f = (idx <= max_label) ? (present[idx] != 0) : 0;
    int incl = f;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
    if (lane == 31) s_warp[wid] = incl;
    __syncthreads();
    if (wid == 0) {
      int w = s_warp[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const int t = __shfl_up_sync(0xffffffffu, w, d); if (lane >= d) w += t; }
      s_warp[lane] = w;
    }
    __syncthreads();
    const int carry = s_carry;
    const int before = carry + (wid ? s_warp[wid - 1] : 0) + incl - f;      // labels present below idx
    if (idx <= max_label) present[idx] = f ? offset + before : 0;
    __syncthreads();
    if (tid == 0) s_carry = carry + s_warp[31];
    __syncthreads();
  }
  if (tid == 0) { present[0] = 0; count[0] = s_carry; }
}

__global__ void __launch_bounds__(256) k_apply_labels(int* __restrict__ lab, long long n, const int* __restrict__ fwd) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long n4 = n >> 2;
  int4* lab4 = reinterpret_cast<int4*>(lab);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    int4 v = lab4[i];
    if ((v.x | v.y | v.z | v.w) == 0) continue;
    v.x = __ldg(fwd + v.x); v.y = __ldg(fwd + v.y); v.z = __ldg(fwd + v.z); v.w = __ldg(fwd + v.w);
    lab4[i] = v;
  }
  for (long long i = (n4 << 2) + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int v = lab[i];
    if (v) lab[i] = __ldg(fwd + v);
  }
}
}  // namespace

extern "C" int sdb_relabel_sequential(int* d_labels, long long n, int max_label, int offset, int* d_forward_map,
                                      int* h_count, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (offset <= 0) { sdb::set_error("relabel_sequential: offset must be strictly positive"); return 1; }   // matching.py:372
  if (max_label < 0 || n < 0) { sdb::set_error("relabel_sequential: negative size"); return 1; }
  if ((reinterpret_cast<uintptr_t>(d_labels) & 15) != 0) { sdb::set_error("relabel_sequential: label map must be 16-byte aligned"); return 1; }
  // d_forward_map: max_label + 3 ints; [max_label+1] = count, [max_label+2] = out-of-range flag
  SDB_CUDA(cudaMemsetAsync(d_forward_map, 0, (size_t)(max_label + 3) * sizeof(int), st));
  int* d_count = d_forward_map + max_label + 1;
  int* d_bad = d_forward_map + max_label + 2;
  const int grid = (int)std::min<long long>(std::max<long long>(cdiv(n >> 2, 256), 1), 132 * 8);
  if (n > 0) SDB_LAUNCH(k_mark_labels, grid, 256, 0, st, d_labels, n, max_label, d_forward_map, d_bad);
  SDB_LAUNCH(k_scan_labels, 1, 1024, 0, st, d_forward_map, max_label, offset, d_count);
  int h[2] = {0, 0};
  SDB_CUDA(cudaMemcpyAsync(h, d_count, 2 * sizeof(int), cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  if (h[1]) { sdb::set_error("relabel_sequential: label outside [0, max_label] (negative values cannot be relabelled, matching.py:374)"); return 1; }
  if (h_count) *h_count = h[0];
  if (n > 0 && !(h[0] == max_label && offset == 1))                       // otherwise the map is already sequential
    SDB_LAUNCH(k_apply_labels, grid, 256, 0, st, d_labels, n, d_forward_map);
  return 0;
}

// reference C ABI (stardist3d_lib.h:67-82): host pointers, result int32[nz*ny*nx] zero-initialised by the caller
extern "C" void _LIB_polyhedron_to_label(const float* dist, const float* points, const float* verts, const int* faces,
                                         const int n_polys, const int n_rays, const int n_faces, const int* labels,
                                         const int nz, const int ny, const int nx, const int render_mode,
                                         const int verbose, const int use_overlap_label, const int overlap_label,
                                         int* result) {
  // void signature (stardist3d_lib.h:67-82): on failure the result is zeroed and the message stays in sdb_last_error();
  // the host process is never aborted
  const long long nvox = (long long)nz * ny * nx;
  auto fail = [&](const char* what) {
    fprintf(stderr, "stardist_b200: _LIB_polyhedron_to_label failed: %s: %s\n", what, sdb_last_error());
    for (long long i = 0; i < nvox; ++i) result[i] = 0;
    cudaGetLastError();
  };
  cudaStream_t st = 0;
  sdb::DevBuf d_dist, d_points, d_verts, d_faces, d_labels, d_out;
  if (d_dist.alloc((size_t)n_polys * n_rays * 4, st) || d_points.alloc((size_t)n_polys * 12, st) || d_verts.alloc((size_t)n_rays * 12, st) ||
      d_faces.alloc((size_t)n_faces * 12, st) || d_labels.alloc((size_t)n_polys * 4, st) || d_out.alloc((size_t)nvox * 4, st)) { sdb::set_error("device allocation failed"); return fail("alloc"); }
  if (n_polys > 0) {
    cudaMemcpyAsync(d_dist.p, dist, (size_t)n_polys * n_rays * 4, cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(d_points.p, points, (size_t)n_polys * 12, cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(d_labels.p, labels, (size_t)n_polys * 4, cudaMemcpyHostToDevice, st);
  }
  cudaMemcpyAsync(d_verts.p, verts, (size_t)n_rays * 12, cudaMemcpyHostToDevice, st);
  cudaMemcpyAsync(d_faces.p, faces, (size_t)n_faces * 12, cudaMemcpyHostToDevice, st);
  if (verbose >= 1) printf("+++++++++++++++ polyhedra to label (GPU) +++++++++++++++ \nn_polys = %d n_rays = %d n_faces = %d nz,ny,nx = %d %d %d\n", n_polys, n_rays, n_faces, nz, ny, nx);
  if (sdb_polyhedron_to_label(d_dist.as<float>(), d_points.as<float>(), d_verts.as<float>(), d_faces.as<int>(), n_polys, n_rays, n_faces,
                              d_labels.as<int>(), nz, ny, nx, render_mode, use_overlap_label, overlap_label, d_out.as<int>(), (sdb_stream_t)st)) return fail("kernel");
  if (cudaMemcpyAsync(result, d_out.p, (size_t)nvox * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) {
    sdb::set_error("copy back failed"); return fail("copy back");
  }
  sdb::set_error("");
}
