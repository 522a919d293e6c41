// traindata.cu -- the batch side of StarDistData2D / StarDistData3D (stardist/models/model2d.py:29-120, model3d.py:30-127,
// base.py:129-225, sample_patches.py): foreground-restricted sampling positions, the patch gather and the class maps.  The
// targets themselves are the batched star distances (stardist.cu) and edt_prob (labelprep.cu).
//
// Sampling.  Without a filter every position of the box [p//2, s-p+p//2] (inclusive, per axis) is valid, in C order.  With
// the foreground filter the box is restricted to maximum_filter(Y, f, mode='constant') > 0, i.e. to the dilation of Y > 0 by
// a box of offsets -(f//2) .. f-1-f//2 along each axis (scipy's origin; outside the image counts as 0), in np.where (C)
// order.  sdb_fg_valid_index builds that mask with one sliding-window pass per axis and a prefix count over the box rows;
// sdb_sample_select maps a batch of drawn ranks to positions on the device (binary search over the rows, then a scan of the
// row), so the index list never exists.
//
// Items are described by a host-built int64 table [batch][TD_ITEM_WORDS] (pointers into the resident images):
//   0 x (float32 [..., C])   1 y (int32 labels)   2 seq (int32, the image's labels relabelled 1..n in ascending order, 0 for
//   background and negative labels)   3 foreground mask (uint8, 0 = no filter)   4 row prefix (int64 [rows + 1])
//   5 drawn rank   6 slot offset (added to seq: labels of different items never coincide)   7..9 image shape (D, H, W; D = 1
//   for 2-D).
#include <algorithm>
#include <climits>
#include "common.cuh"
#include "scan.cuh"
#include "../../include/stardist_b200.h"

namespace {

using sdb::cdiv;

constexpr int TD_ITEM_WORDS = 10;
constexpr int CLASS_NONE = -1;        // the object is ignored: -1 in every class channel
constexpr int CLASS_MISSING = -2;     // the label has no entry in the class dict (an error when it occurs in a patch)

int grid_for(long long work, int threads) { return (int)std::max<long long>(1, std::min<long long>(cdiv(work, threads), 132 * 32)); }

// one thread per line along the pass axis: out = 1 where some input of the window [i - f//2, i + f-1-f//2] is set
template <bool FROM_LABELS>
__global__ void k_fg_dilate(const void* __restrict__ in, unsigned char* __restrict__ out, int len, long long inner, long long n_lines, int f) {
  const long long l = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= n_lines) return;
  const long long o = l / inner, base = o * len * inner + (l - o * inner);
  auto val = [&](int k) -> int {
    const long long idx = base + (long long)k * inner;
    return FROM_LABELS ? (__ldg((const int*)in + idx) > 0) : (int)__ldg((const unsigned char*)in + idx);
  };
  const int lo = f / 2, hi = f - 1 - f / 2;
  int cnt = 0;
  for (int k = 0; k <= min(hi, len - 1); ++k) cnt += val(k);
  for (int i = 0; i < len; ++i) {
    out[base + (long long)i * inner] = cnt > 0;
    if (i + 1 + hi < len) cnt += val(i + 1 + hi);
    if (i - lo >= 0) cnt -= val(i - lo);
  }
}

// set positions per box row (rows in C order over the box's leading axes) -> pre[row + 1]
__global__ void k_box_row_counts(const unsigned char* __restrict__ m, int H, int W, int pz, int py, int px, int ey, int ex, long long rows,
                                 long long* __restrict__ pre) {
  for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(r % ey), z = (int)(r / ey);
    const unsigned char* line = m + ((long long)(z + pz / 2) * H + (y + py / 2)) * W + px / 2;
    long long c = 0;
    for (int x = 0; x < ex; ++x) c += line[x];
    pre[r + 1] = c;
  }
}

__global__ void k_sample_select(const long long* __restrict__ items, int batch, int pz, int py, int px, int* __restrict__ pos) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  const long long* it = items + (long long)b * TD_ITEM_WORDS;
  const int H = (int)it[8], W = (int)it[9];
  const int ey = H - py + 1, ex = W - px + 1;
  const long long rank = it[5];
  int z, y, x;
  if (!it[3]) {
    x = (int)(rank % ex);
    const long long t = rank / ex;
    y = (int)(t % ey); z = (int)(t / ey);
  } else {
    const unsigned char* m = (const unsigned char*)it[3];
    const long long* pre = (const long long*)it[4];
    const long long rows = (long long)((int)it[7] - pz + 1) * ey;
    long long lo = 0, hi = rows - 1;                 // the row r with pre[r] <= rank < pre[r + 1]
    while (lo < hi) {
      const long long mid = (lo + hi + 1) >> 1;
      if (pre[mid] <= rank) lo = mid; else hi = mid - 1;
    }
    y = (int)(lo % ey); z = (int)(lo / ey);
    long long rem = rank - pre[lo];
    const unsigned char* line = m + ((long long)(z + pz / 2) * H + (y + py / 2)) * W + px / 2;
    for (x = 0; x < ex - 1; ++x)
      if (line[x] && rem-- == 0) break;
  }
  pos[3 * b] = z + pz / 2; pos[3 * b + 1] = y + py / 2; pos[3 * b + 2] = x + px / 2;
}

// one thread per patch pixel: X channels, clamped labels, slot labels, and at the grid positions the negative-label mask
// (and, for 2-D, the subsampled slot labels edt_prob runs on); flags[0] |= 1 where a label without a class occurs
__global__ void k_train_gather(const long long* __restrict__ items, const int* __restrict__ pos, long long n, int pz, int py, int px, int C,
                               int gz, int gy, int gx, int Goy, int Gox, const int* __restrict__ table, float* __restrict__ X,
                               int* __restrict__ Yc, int* __restrict__ Ys, int* __restrict__ Ye, unsigned char* __restrict__ neg,
                               int* __restrict__ flags, int clamp) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(e % px);
    long long t = e / px;
    const int y = (int)(t % py);
    t /= py;
    const int z = (int)(t % pz);
    const long long b = t / pz;
    const long long* it = items + b * TD_ITEM_WORDS;
    const long long H = it[8], W = it[9];
    const long long src = ((long long)(pos[3 * b] - pz / 2 + z) * H + (pos[3 * b + 1] - py / 2 + y)) * W + (pos[3 * b + 2] - px / 2 + x);
    const int v = __ldg((const int*)it[1] + src);
    const int s = __ldg((const int*)it[2] + src);
    const int slot = s > 0 ? s + (int)it[6] : 0;
    Yc[e] = clamp ? max(v, 0) : v;
    Ys[e] = slot;
    if (table && slot > 0 && __ldg(table + slot) == CLASS_MISSING) atomicOr(flags, 1);
    const float* xs = (const float*)it[0] + src * C;
    for (int c = 0; c < C; ++c) X[e * C + c] = __ldg(xs + c);
    if (z % gz == 0 && y % gy == 0 && x % gx == 0) {
      const long long o = ((b * ((pz - 1) / gz + 1) + z / gz) * Goy + y / gy) * Gox + x / gx;
      neg[o] = v < 0;
      if (Ye) Ye[o] = slot;
    }
  }
}

// prob_class: mask_to_categorical of the slot labels at the order-0 zoom positions (index -1: zoom's constant 0), -1
// where neg
__global__ void k_class_map(const int* __restrict__ Ys, int pz, int py, int px, const int* __restrict__ zi, const int* __restrict__ yi,
                            const int* __restrict__ xi, int oz, int oy, int ox, long long n_out, const int* __restrict__ table, int n_classes,
                            const unsigned char* __restrict__ neg, float* __restrict__ out) {
  for (long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x; o < n_out; o += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(o % ox);
    long long t = o / ox;
    const int j = (int)(t % oy);
    t /= oy;
    const int i = (int)(t % oz);
    const long long b = t / oz;
    float* r = out + o * (n_classes + 1);
    const bool masked = neg[o];
    if (zi[i] < 0 || yi[j] < 0 || xi[k] < 0) {                       // zoom's constant 0 (see zoom_order0_index)
      for (int c = 0; c <= n_classes; ++c) r[c] = masked ? -1.f : 0.f;
      continue;
    }
    const int slot = __ldg(Ys + ((b * pz + zi[i]) * py + yi[j]) * px + xi[k]);
    const int cls = slot > 0 ? __ldg(table + slot) : 0;
    for (int c = 0; c <= n_classes; ++c) {
      float v;
      if (masked) v = -1.f;
      else if (slot == 0) v = c == 0 ? 1.f : 0.f;
      else if (c == 0) v = 0.f;                                      // y_mask[..., 0] = (y == 0), written last
      else if (cls == CLASS_NONE) v = -1.f;
      else v = cls == c ? 1.f : 0.f;
      r[c] = v;
    }
  }
}

}  // namespace

extern "C" int sdb_fg_valid_index(const int* d_labels, int ndim, const int* shape, const int* filter_size, const int* patch_size,
                                  unsigned char* d_mask, long long* d_prefix, long long* h_n_valid, sdb_stream_t stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (ndim != 2 && ndim != 3) { sdb::set_error("fg_valid_index: ndim must be 2 or 3"); return 1; }
  int d[3] = {1, 1, 1}, p[3] = {1, 1, 1};
  long long N = 1;
  for (int a = 0; a < ndim; ++a) {
    if (filter_size[a] < 1) { sdb::set_error("fg_valid_index: filter sizes must be >= 1"); return 1; }
    if (patch_size[a] < 1 || patch_size[a] > shape[a]) { sdb::set_error("fg_valid_index: patch size must lie in [1, image extent]"); return 1; }
    d[3 - ndim + a] = shape[a]; p[3 - ndim + a] = patch_size[a];
    N *= shape[a];
  }
  sdb::DevBuf tmp;
  SDB_CUDA(tmp.alloc((size_t)N, st));
  unsigned char* T = tmp.as<unsigned char>();
  for (int a = ndim - 1; a >= 0; --a) {
    const int len = shape[a];
    long long inner = 1;
    for (int b = a + 1; b < ndim; ++b) inner *= shape[b];
    const long long lines = N / len;
    // 2-D: labels -> tmp -> mask; 3-D: labels -> mask -> tmp -> mask
    unsigned char* out = ((ndim - 1 - a) % 2 == (ndim == 2 ? 0 : 1)) ? T : d_mask;
    if (a == ndim - 1)
      SDB_LAUNCH(k_fg_dilate<true>, cdiv(lines, 128), 128, 0, st, (const void*)d_labels, out, len, inner, lines, filter_size[a]);
    else
      SDB_LAUNCH(k_fg_dilate<false>, cdiv(lines, 128), 128, 0, st, (const void*)(out == T ? d_mask : T), out, len, inner, lines,
                 filter_size[a]);
  }
  const int ey = d[1] - p[1] + 1, ex = d[2] - p[2] + 1;
  const long long rows = (long long)(d[0] - p[0] + 1) * ey;
  SDB_LAUNCH(k_box_row_counts, grid_for(rows, 256), 256, 0, st, d_mask, d[1], d[2], p[0], p[1], p[2], ey, ex, rows, d_prefix);
  SDB_LAUNCH(k_scan_rows, 1, SCAN_THREADS, 0, st, d_prefix, rows);
  SDB_CUDA(cudaMemcpyAsync(h_n_valid, d_prefix + rows, sizeof(long long), cudaMemcpyDeviceToHost, st));
  SDB_CUDA(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int sdb_sample_select(const long long* d_items, int ndim, int batch, const int* patch_size, int* d_pos, sdb_stream_t stream) {
  if ((ndim != 2 && ndim != 3) || batch < 1) { sdb::set_error("sample_select: ndim must be 2 or 3 and batch >= 1"); return 1; }
  const int pz = ndim == 3 ? patch_size[0] : 1, py = patch_size[ndim - 2], px = patch_size[ndim - 1];
  SDB_LAUNCH(k_sample_select, cdiv(batch, 128), 128, 0, (cudaStream_t)stream, d_items, batch, pz, py, px, d_pos);
  return 0;
}

extern "C" int sdb_train_gather(const long long* d_items, const int* d_pos, int ndim, int batch, const int* patch_size, int n_channels,
                                const int* grid, const int* d_class_table, float* d_x, int* d_y_clamped, int* d_y_slots,
                                int* d_y_slots_grid, unsigned char* d_neg, int* d_flags, int clamp, sdb_stream_t stream) {
  if ((ndim != 2 && ndim != 3) || batch < 1 || n_channels < 1) {
    sdb::set_error("train_gather: ndim must be 2 or 3, batch >= 1 and n_channels >= 1"); return 1;
  }
  int p[3] = {1, 1, 1}, g[3] = {1, 1, 1};
  long long n = batch;
  for (int a = 0; a < ndim; ++a) {
    if (grid[a] < 1 || patch_size[a] < 1) { sdb::set_error("train_gather: grid and patch sizes must be >= 1"); return 1; }
    p[3 - ndim + a] = patch_size[a]; g[3 - ndim + a] = grid[a];
    n *= patch_size[a];
  }
  SDB_LAUNCH(k_train_gather, grid_for(n, 256), 256, 0, (cudaStream_t)stream, d_items, d_pos, n, p[0], p[1], p[2], n_channels, g[0], g[1],
             g[2], (p[1] - 1) / g[1] + 1, (p[2] - 1) / g[2] + 1, d_class_table, d_x, d_y_clamped, d_y_slots, d_y_slots_grid, d_neg, d_flags, clamp);
  return 0;
}

extern "C" int sdb_class_map(const int* d_y_slots, int ndim, int batch, const int* patch_size, const int* d_zoom_index,
                             const int* out_shape, const int* d_class_table, int n_classes, const unsigned char* d_neg, float* d_out,
                             sdb_stream_t stream) {
  if ((ndim != 2 && ndim != 3) || batch < 1 || n_classes < 1) {
    sdb::set_error("class_map: ndim must be 2 or 3, batch >= 1 and n_classes >= 1"); return 1;
  }
  int p[3] = {1, 1, 1}, o[3] = {1, 1, 1};
  for (int a = 0; a < ndim; ++a) { p[3 - ndim + a] = patch_size[a]; o[3 - ndim + a] = out_shape[a]; }
  // d_zoom_index: the source index of every output index, axis after axis ([o_0] [o_1] (...)); a 2-D map gets a 0 in front
  sdb::DevBuf zero;
  const int* zi = d_zoom_index;
  if (ndim == 2) {
    SDB_CUDA(zero.alloc(sizeof(int), (cudaStream_t)stream));
    SDB_CUDA(cudaMemsetAsync(zero.p, 0, sizeof(int), (cudaStream_t)stream));
    zi = zero.as<int>();
  }
  const int* yi = ndim == 3 ? d_zoom_index + o[0] : d_zoom_index;
  const int* xi = yi + o[1];
  const long long n_out = (long long)batch * o[0] * o[1] * o[2];
  SDB_LAUNCH(k_class_map, grid_for(n_out, 256), 256, 0, (cudaStream_t)stream, d_y_slots, p[0], p[1], p[2], zi, yi, xi, o[0], o[1], o[2],
             n_out, d_class_table, n_classes, d_neg, d_out);
  return 0;
}
