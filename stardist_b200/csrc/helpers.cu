// helpers.cu -- the public helpers around the prediction and training paths that read a whole label, mask or distance map:
//   * mask_to_categorical (stardist/utils.py:318-380): sdb_label_class_map writes the (n_classes + 1)-channel class map of a
//     label map, one thread per output value; the label's class comes from a sorted (label, code) table by binary search;
//   * sample_points (utils.py:156-177) and get_valid_inds (sample_patches.py:38-66): sdb_mask_compact_count /
//     sdb_mask_compact_write are one order-preserving compaction of a box of a mask (flag, per-row count, the row scan of
//     scan.cuh, scatter), with a gather of a float32 weight map at the survivors;
//   * sample_patches (sample_patches.py:7-35): sdb_gather_patches copies equally shaped crops of an array, its elements as
//     1, 2, 4, 8 or 16-byte words (other element types are viewed as bytes by the caller), so values cannot change;
//   * dist_to_volume / dist_to_centroid (geometry/geom3d.py:220-258 over stardist3d_impl.cpp:1529-1585): the volume and
//     centroid of the star-convex polyhedron of every voxel of a 3-D distance map.  Exact unit (-fmad=false): the float and
//     double operations are the reference's, in its order.
#include <algorithm>
#include "common.cuh"
#include "scan.cuh"
#include "geom3d.cuh"
#include "nms3d_pair.cuh"
#include "../../include/stardist_b200.h"

namespace {

using sdb::cdiv;

int grid_for(long long work, int threads) { return (int)std::max<long long>(1, std::min<long long>(cdiv(work, threads), 132 * 32)); }

// ----------------------------------------------------------------------------------------------- mask_to_categorical
// codes: 1..n_classes = one-hot class, 0 = background class (all channels 0 once channel 0 is set to y == 0), -1 = None
// (channel 0 is 0, the others -1).  Every non-zero label of the map is in keys (checked on the host).
__global__ void k_label_class_map(const int* __restrict__ y, long long n_out, const int* __restrict__ keys,
                                  const int* __restrict__ codes, int n_keys, int n_classes, float* __restrict__ out) {
  const int C = n_classes + 1;
  for (long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x; o < n_out; o += (long long)gridDim.x * blockDim.x) {
    const long long p = o / C;
    const int c = (int)(o - p * C);
    const int v = __ldg(y + p);
    float r;
    if (v == 0) {
      r = c == 0 ? 1.f : 0.f;
    } else {
      int lo = 0, hi = n_keys - 1;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(keys + mid) < v) lo = mid + 1; else hi = mid;
      }
      const int code = __ldg(codes + lo);
      if (c == 0) r = 0.f;                                               // y_mask[..., 0] = (y == 0), written last
      else if (code < 0) r = -1.f;
      else r = code == c ? 1.f : 0.f;
    }
    out[o] = r;
  }
}

// ----------------------------------------------------------------------------------------------- mask compaction
// The mask is contiguous with shape S[4] (leading axes padded with 1), the box [lo, lo + e) per axis; rows are the box's
// lines along the last axis, in C order.  An element is set when the low bit of its first byte is (NONZERO false: numpy's
// `mask & 1` on a little-endian bool or integer) or when any of its elem_size bytes is non-zero (NONZERO true: np.where).
struct Box {
  long long S[4], lo[4], e[4];
  __device__ long long line_offset(long long r) const {            // flat element offset of the first element of row r
    const long long a2 = r % e[2], t = r / e[2];
    const long long a1 = t % e[1], a0 = t / e[1];
    return (((lo[0] + a0) * S[1] + lo[1] + a1) * S[2] + lo[2] + a2) * S[3] + lo[3];
  }
};

template <bool NONZERO>
__device__ __forceinline__ bool is_set(const unsigned char* __restrict__ m, long long off, int elem) {
  const unsigned char* p = m + off * elem;
  if (!NONZERO) return __ldg(p) & 1;
  unsigned char any = 0;
  for (int b = 0; b < elem; ++b) any |= __ldg(p + b);
  return any != 0;
}

constexpr int CW = 8;                  // warps (rows in flight) per CTA

template <bool NONZERO>
__global__ void __launch_bounds__(CW * 32) k_mask_row_counts(const unsigned char* __restrict__ m, int elem, Box box, long long rows,
                                                             long long* __restrict__ pre) {
  const int lane = threadIdx.x & 31;
  for (long long r = (long long)blockIdx.x * CW + (threadIdx.x >> 5); r < rows; r += (long long)gridDim.x * CW) {
    const long long base = box.line_offset(r);
    long long c = 0;
    for (long long x = 0; x < box.e[3]; x += 32) {
      const bool set = x + lane < box.e[3] && is_set<NONZERO>(m, base + x + lane, elem);
      c += __popc(__ballot_sync(0xffffffffu, set));
    }
    if (lane == 0) pre[r + 1] = c;
  }
}

// survivors of row r go to [pre[r], pre[r + 1]) in order: coordinates (absolute, int32) axis after axis into
// coords[axis][n], and w[k] = prob[flat offset] when prob is given
template <bool NONZERO>
__global__ void __launch_bounds__(CW * 32) k_mask_row_write(const unsigned char* __restrict__ m, int elem, Box box, long long rows,
                                                            int ndim, const long long* __restrict__ pre, long long n,
                                                            int* __restrict__ coords, const float* __restrict__ prob,
                                                            float* __restrict__ w) {
  const int lane = threadIdx.x & 31;
  const unsigned int below = (1u << lane) - 1u;
  for (long long r = (long long)blockIdx.x * CW + (threadIdx.x >> 5); r < rows; r += (long long)gridDim.x * CW) {
    const long long base = box.line_offset(r);
    const long long a2 = r % box.e[2], t = r / box.e[2];
    const int c[3] = {(int)(box.lo[0] + t / box.e[1]), (int)(box.lo[1] + t % box.e[1]), (int)(box.lo[2] + a2)};
    long long k = pre[r];
    for (long long x = 0; x < box.e[3]; x += 32) {
      const bool set = x + lane < box.e[3] && is_set<NONZERO>(m, base + x + lane, elem);
      const unsigned int vote = __ballot_sync(0xffffffffu, set);
      if (set) {
        const long long pos = k + __popc(vote & below);
        for (int a = 0; a < ndim - 1; ++a) coords[(long long)a * n + pos] = c[3 - ndim + 1 + a];
        coords[(long long)(ndim - 1) * n + pos] = (int)(box.lo[3] + x + lane);
        if (prob) w[pos] = __ldg(prob + base + x + lane);
      }
      k += __popc(vote);
    }
  }
}

int make_box(int ndim, const long long* shape, const long long* lo, const long long* hi, Box& box, long long& rows, const char* what) {
  if (ndim < 1 || ndim > 4) { sdb::set_error(std::string(what) + ": ndim must be in [1, 4]"); return 1; }
  for (int a = 0; a < 4; ++a) { box.S[a] = 1; box.lo[a] = 0; box.e[a] = 1; }
  for (int a = 0; a < ndim; ++a) {
    const int b = 4 - ndim + a;
    if (shape[a] < 0 || lo[a] < 0 || hi[a] > shape[a]) { sdb::set_error(std::string(what) + ": box outside the mask"); return 1; }
    box.S[b] = shape[a]; box.lo[b] = lo[a]; box.e[b] = std::max<long long>(0, hi[a] - lo[a]);
  }
  rows = box.e[0] * box.e[1] * box.e[2];
  return 0;
}

// ----------------------------------------------------------------------------------------------- patch gather
template <typename T>
__global__ void k_gather_patches(const T* __restrict__ src, Box box, long long n_out, long long per,
                                 const long long* __restrict__ starts, int ndim, T* __restrict__ out) {
  // box.S: the array's shape, box.e: the crop's shape (both padded to 4 axes); starts [n_samples][ndim]
  for (long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x; o < n_out; o += (long long)gridDim.x * blockDim.x) {
    const long long s = o / per;
    long long q = o - s * per, off = 0, stride = 1;
    for (int a = 3; a >= 0; --a) {
      const long long qa = q % box.e[a];
      q /= box.e[a];
      const long long st = a >= 4 - ndim ? __ldg(starts + s * ndim + (a - (4 - ndim))) : 0;
      off += (st + qa) * stride;
      stride *= box.S[a];
    }
    out[o] = src[off];
  }
}

struct alignas(16) Bytes16 { unsigned long long a, b; };

template <typename T>
int gather_as(const void* src, const Box& box, long long n_out, long long per, const long long* starts, int ndim, void* out,
              cudaStream_t st) {
  SDB_LAUNCH(k_gather_patches<T>, grid_for(n_out, 256), 256, 0, st, (const T*)src, box, n_out, per, starts, ndim, (T*)out);
  return 0;
}

// ----------------------------------------------------------------------------------------------- polyhedra of a dist map
constexpr int VPB = 64;                // voxels (threads) per CTA; their ray rows are staged in shared memory

__host__ __device__ inline int row_pitch(int n_rays) { return n_rays | 1; }     // odd pitch: one voxel per bank
size_t poly_smem(int n_rays, int n_faces) {
  return sizeof(float) * (3 * (size_t)n_rays + (size_t)VPB * row_pitch(n_rays)) + sizeof(int) * 3 * (size_t)n_faces;
}

// stardist3d_impl.cpp:1529-1585: one voxel per thread; dist [n_vox][n_rays] read into shared memory with coalesced loads
template <bool CENTROID>
__global__ void __launch_bounds__(VPB) k_dist_to_poly(const float* __restrict__ dist, long long n_vox, int n_rays,
                                                      const float* __restrict__ verts, const int* __restrict__ faces, int n_faces,
                                                      int ny, int nx, int absolute, float* __restrict__ out) {
  extern __shared__ float smem[];
  const int pitch = row_pitch(n_rays);
  float* sv = smem;                                   // [3 n_rays]
  float* sd = sv + 3 * n_rays;                        // [VPB][pitch]
  int* sf = reinterpret_cast<int*>(sd + VPB * pitch); // [3 n_faces]
  for (int i = threadIdx.x; i < 3 * n_rays; i += VPB) sv[i] = __ldg(verts + i);
  for (int i = threadIdx.x; i < 3 * n_faces; i += VPB) sf[i] = __ldg(faces + i);
  const long long v0 = (long long)blockIdx.x * VPB;
  const int nv = (int)min((long long)VPB, n_vox - v0);
  const float* src = dist + v0 * n_rays;
  for (int i = threadIdx.x; i < nv * n_rays; i += VPB) {
    const int v = i / n_rays;
    sd[v * pitch + (i - v * n_rays)] = __ldg(src + i);
  }
  __syncthreads();
  if ((int)threadIdx.x >= nv) return;
  const float* d = sd + threadIdx.x * pitch;
  const long long v = v0 + threadIdx.x;
  if (!CENTROID) {
    out[v] = sd3::polyhedron_volume(d, sv, sf, n_faces);              // :257-291
    return;
  }
  // polyhedron_centroid :293-340.  R += .25 * (A + B + C) * vol: a float sum, a double literal, so a double product (the
  // .25 is exact) and a double add, rounded to float on assignment
  float vol = 0.f, Rz = 0.f, Ry = 0.f, Rx = 0.f;
  for (int f = 0; f < n_faces; ++f) {
    const int iA = sf[3 * f], iB = sf[3 * f + 1], iC = sf[3 * f + 2];
    const float Az = __fmul_rn(d[iA], sv[3 * iA]), Ay = __fmul_rn(d[iA], sv[3 * iA + 1]), Ax = __fmul_rn(d[iA], sv[3 * iA + 2]);
    const float Bz = __fmul_rn(d[iB], sv[3 * iB]), By = __fmul_rn(d[iB], sv[3 * iB + 1]), Bx = __fmul_rn(d[iB], sv[3 * iB + 2]);
    const float Cz = __fmul_rn(d[iC], sv[3 * iC]), Cy = __fmul_rn(d[iC], sv[3 * iC + 1]), Cx = __fmul_rn(d[iC], sv[3 * iC + 2]);
    const float cv = sd3::tetrahedron_volume0(Az, Ay, Ax, Bz, By, Bx, Cz, Cy, Cx);
    const double dv = (double)cv;
    Rz = __double2float_rn(__dadd_rn((double)Rz, __dmul_rn(__dmul_rn(0.25, (double)__fadd_rn(__fadd_rn(Az, Bz), Cz)), dv)));
    Ry = __double2float_rn(__dadd_rn((double)Ry, __dmul_rn(__dmul_rn(0.25, (double)__fadd_rn(__fadd_rn(Ay, By), Cy)), dv)));
    Rx = __double2float_rn(__dadd_rn((double)Rx, __dmul_rn(__dmul_rn(0.25, (double)__fadd_rn(__fadd_rn(Ax, Bx), Cx)), dv)));
    vol = __fadd_rn(vol, cv);
  }
  const bool ok = (double)vol > 1.e-10;
  const long long i = v % nx, t = v / nx;
  const long long j = t % ny, k = t / ny;
  // _COMMON_dist_to_centroid :1580-1582: centroid + absolute * index, an int converted to float
  out[3 * v] = __fadd_rn(ok ? __fdiv_rn(Rz, vol) : 0.f, (float)(absolute * (int)k));
  out[3 * v + 1] = __fadd_rn(ok ? __fdiv_rn(Ry, vol) : 0.f, (float)(absolute * (int)j));
  out[3 * v + 2] = __fadd_rn(ok ? __fdiv_rn(Rx, vol) : 0.f, (float)(absolute * (int)i));
}

template <bool CENTROID>
int dist_to_poly(const float* d_dist, int nz, int ny, int nx, int n_rays, const float* d_verts, const int* d_faces, int n_faces,
                 int absolute, float* d_out, cudaStream_t st, const char* what) {
  if (nz < 0 || ny < 0 || nx < 0) { sdb::set_error(std::string(what) + ": bad map shape"); return 1; }
  if (n_rays < 1 || n_rays > sd3::SD3_MAX_RAYS || n_faces < 0 || n_faces > sd3::SD3_MAX_FACES) {
    sdb::set_error(std::string(what) + ": n_rays must be in [1, 256] and n_faces in [0, 512]"); return 1;
  }
  const long long n_vox = (long long)nz * ny * nx;
  if (n_vox == 0) return 0;
  const size_t smem = poly_smem(n_rays, n_faces);
  SDB_CUDA(cudaFuncSetAttribute(k_dist_to_poly<CENTROID>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  SDB_LAUNCH(k_dist_to_poly<CENTROID>, cdiv(n_vox, VPB), VPB, smem, st, d_dist, n_vox, n_rays, d_verts, d_faces, n_faces, ny, nx,
             absolute, d_out);
  return 0;
}

}  // namespace

extern "C" int sdb_label_class_map(const int* d_labels, long long n, const int* d_keys, const int* d_codes, int n_keys,
                                   int n_classes, float* d_out, sdb_stream_t stream) {
  if (n < 0 || n_keys < 0 || n_classes < 1) { sdb::set_error("label_class_map: n, n_keys must be >= 0 and n_classes >= 1"); return 1; }
  const long long n_out = n * (n_classes + 1);
  if (n_out == 0) return 0;
  SDB_LAUNCH(k_label_class_map, grid_for(n_out, 256), 256, 0, (cudaStream_t)stream, d_labels, n_out, d_keys, d_codes, n_keys,
             n_classes, d_out);
  return 0;
}

extern "C" int sdb_mask_compact_count(const void* d_mask, int elem_size, int nonzero, int ndim, const long long* shape,
                                      const long long* lo, const long long* hi, long long* d_prefix, long long* h_n,
                                      sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  Box box; long long rows;
  if (elem_size < 1) { sdb::set_error("mask_compact: elem_size must be >= 1"); return 1; }
  if (make_box(ndim, shape, lo, hi, box, rows, "mask_compact")) return 1;
  *h_n = 0;
  if (rows == 0 || box.e[3] == 0) return 0;
  const int grid = (int)std::min<long long>(cdiv(rows, CW), 132 * 64);
  if (nonzero) SDB_LAUNCH(k_mask_row_counts<true>, grid, CW * 32, 0, st, (const unsigned char*)d_mask, elem_size, box, rows, d_prefix);
  else SDB_LAUNCH(k_mask_row_counts<false>, grid, CW * 32, 0, st, (const unsigned char*)d_mask, elem_size, box, rows, d_prefix);
  SDB_LAUNCH(k_scan_rows, 1, SCAN_THREADS, 0, st, d_prefix, rows);
  SDB_CUDA(cudaMemcpyAsync(h_n, d_prefix + rows, sizeof(long long), cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int sdb_mask_compact_write(const void* d_mask, int elem_size, int nonzero, int ndim, const long long* shape,
                                      const long long* lo, const long long* hi, const long long* d_prefix, long long n,
                                      int* d_coords, const float* d_prob, float* d_w, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  Box box; long long rows;
  if (elem_size < 1) { sdb::set_error("mask_compact: elem_size must be >= 1"); return 1; }
  if (make_box(ndim, shape, lo, hi, box, rows, "mask_compact")) return 1;
  if (rows == 0 || box.e[3] == 0 || n == 0) return 0;
  const int grid = (int)std::min<long long>(cdiv(rows, CW), 132 * 64);
  if (nonzero)
    SDB_LAUNCH(k_mask_row_write<true>, grid, CW * 32, 0, st, (const unsigned char*)d_mask, elem_size, box, rows, ndim, d_prefix, n,
               d_coords, d_prob, d_w);
  else
    SDB_LAUNCH(k_mask_row_write<false>, grid, CW * 32, 0, st, (const unsigned char*)d_mask, elem_size, box, rows, ndim, d_prefix, n,
               d_coords, d_prob, d_w);
  return 0;
}

extern "C" int sdb_gather_patches(const void* d_src, int elem_size, int ndim, const long long* shape, const long long* patch,
                                  const long long* d_starts, long long n_samples, void* d_out, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (ndim < 1 || ndim > 4 || elem_size < 1 || n_samples < 0) {
    sdb::set_error("gather_patches: ndim must be in [1, 4], elem_size >= 1 and n_samples >= 0"); return 1;
  }
  Box box;
  long long per = 1;
  for (int a = 0; a < 4; ++a) { box.S[a] = 1; box.lo[a] = 0; box.e[a] = 1; }
  for (int a = 0; a < ndim; ++a) {
    if (shape[a] < 0 || patch[a] < 0 || patch[a] > shape[a]) { sdb::set_error("gather_patches: crop larger than the array"); return 1; }
    box.S[4 - ndim + a] = shape[a]; box.e[4 - ndim + a] = patch[a]; per *= patch[a];
  }
  const long long n_out = per * n_samples;
  if (n_out == 0) return 0;
  switch (elem_size) {
    case 1: return gather_as<unsigned char>(d_src, box, n_out, per, d_starts, ndim, d_out, st);
    case 2: return gather_as<unsigned short>(d_src, box, n_out, per, d_starts, ndim, d_out, st);
    case 4: return gather_as<unsigned int>(d_src, box, n_out, per, d_starts, ndim, d_out, st);
    case 8: return gather_as<unsigned long long>(d_src, box, n_out, per, d_starts, ndim, d_out, st);
    case 16: return gather_as<Bytes16>(d_src, box, n_out, per, d_starts, ndim, d_out, st);
    default: sdb::set_error("gather_patches: elem_size must be 1, 2, 4, 8 or 16"); return 1;
  }
}

extern "C" int sdb_dist_to_volume(const float* d_dist, int nz, int ny, int nx, int n_rays, const float* d_verts, const int* d_faces,
                                  int n_faces, float* d_out, sdb_stream_t stream) {
  return dist_to_poly<false>(d_dist, nz, ny, nx, n_rays, d_verts, d_faces, n_faces, 0, d_out, (cudaStream_t)stream, "dist_to_volume");
}

extern "C" int sdb_dist_to_centroid(const float* d_dist, int nz, int ny, int nx, int n_rays, const float* d_verts, const int* d_faces,
                                    int n_faces, int absolute, float* d_out, sdb_stream_t stream) {
  return dist_to_poly<true>(d_dist, nz, ny, nx, n_rays, d_verts, d_faces, n_faces, absolute ? 1 : 0, d_out, (cudaStream_t)stream,
                            "dist_to_centroid");
}
