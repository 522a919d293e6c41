/* stardist_b200.h -- C ABI of libstardist_b200.so (H100 / sm_90a prediction hot path).
 *
 * Two families of entry points:
 *
 *  (1) _LIB_*  : HOST pointers, blocking.  These are the drop-in boundary: the first two have
 *      exactly the signatures of the reference's own C ABI
 *      (stardist/lib/stardist3d_lib.h:55-82, implemented by stardist3d_lib.c:5-41 on top of
 *      _COMMON_* in stardist3d_impl.cpp:956,1404); the 2D ones are the analogues of the CPython
 *      entry point c_non_max_suppression_inds (stardist/lib/stardist2d.cpp:390-615, called from
 *      stardist/nms.py:220-225) and of polygons_to_label (stardist/geometry/geom2d.py:149-197).
 *      Inputs are copied to the device, the CUDA kernels run, the result is copied back.
 *
 *  (2) sdb_*   : DEVICE pointers + cudaStream_t, stream ordered.  Used by the Python host layer
 *      (stardist_b200/) to keep the whole predict_instances pipeline resident in HBM.
 *
 * All functions returning int return 0 on success, non-zero on error; sdb_last_error() gives the
 * message.  There is no CPU fallback: without a usable CUDA device every call fails.
 */
#ifndef STARDIST_B200_H
#define STARDIST_B200_H

#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
#include <cstdbool>
extern "C" {
#else
#include <stdbool.h>
#endif

typedef void* sdb_stream_t; /* a cudaStream_t (0 = default stream) */

/* ----------------------------------------------------------------------------- misc */
const char* sdb_last_error(void);
int sdb_device_info(int* n_devices, int* sm_count, int* cc_major, int* cc_minor);
/* number of kernel launches issued by this library since the last reset (bench "gpu_launches") */
long long sdb_launch_count(int reset);

/* optional live profiling with CUDA events on the launching stream (bench.py's roofline): names are
 * "nms2d_clip" (units = polygon pairs tested) and "conv_tc" (units = algorithmic FLOPs) */
int sdb_profile_enable(int on);
int sdb_profile_get(const char* name, double* ms, long long* launches, double* units);

/* ----------------------------------------------------------------------------- (1) host ABI */

/* reference: stardist3d_lib.h:55-65 (identical signature) */
void _LIB_non_maximum_suppression_sparse(
    const float* scores, const float* dist, const float* points,
    const int n_polys, const int n_rays, const int n_faces,
    const float* verts, const int* faces,
    const float threshold, const int use_bbox, const int use_kdtree,
    const int verbose, bool* result);

/* reference: stardist3d_lib.h:67-82 (identical signature) */
void _LIB_polyhedron_to_label(
    const float* dist, const float* points, const float* verts, const int* faces,
    const int n_polys, const int n_rays, const int n_faces, const int* labels,
    const int nz, const int ny, const int nx,
    const int render_mode, const int verbose,
    const int use_overlap_label, const int overlap_label,
    int* result);

/* 2D analogue of c_non_max_suppression_inds (stardist2d.cpp:390): dist[n_polys*n_rays],
 * points[n_polys*2] (y,x), sorted by descending score; result[n_polys] = kept. Returns status. */
int _LIB_non_maximum_suppression_2d(
    const float* dist, const float* points, const int n_polys, const int n_rays,
    const float threshold, const int use_bbox, const int use_kdtree, const int verbose,
    bool* result);

/* 2D analogue of polygons_to_label_coord (geom2d.py:149-166): coord[n_polys*2*n_rays] as
 * (n_polys, 2, n_rays) float32 with row 0 = y(r), row 1 = x(c); polygons are painted in the
 * given order (later overwrite earlier) with value labels[i]+1. result is int32[ny*nx]. */
int _LIB_polygons_to_label_2d(
    const float* coord, const int* labels, const int n_polys, const int n_rays,
    const int ny, const int nx, int* result);

/* ----------------------------------------------------------------------------- (2) device ABI */

/* 2D NMS, all pointers are device pointers; d_keep is uint8[n_polys]. */
int sdb_nms2d(const float* d_dist, const float* d_points, int n_polys, int n_rays,
              float threshold, int use_bbox, int use_kdtree, int verbose,
              unsigned char* d_keep, sdb_stream_t stream);
/* sdb_nms2d + the ordered list of survivors: d_kept_index[0..*h_n_kept) = indices with keep == 1, ascending
 * (= descending score); d_keep may be NULL.  One 4-byte device->host read-back, stream synchronised on return. */
int sdb_nms2d_survivors(const float* d_dist, const float* d_points, int n_polys, int n_rays,
                        float threshold, int use_bbox, int use_kdtree, int verbose,
                        unsigned char* d_keep, int* d_kept_index, int* h_n_kept, sdb_stream_t stream);
/* Paint order of polygons_to_label (geom2d.py:191-197) for survivors listed by descending score (ties in the
 * order np.argsort(prob, kind='stable')[::-1] leaves them): rank[i] = position of i in
 * np.argsort(prob, kind='stable'), id_by_rank[rank[i]] = i + 1. */
int sdb_paint_order_2d(const float* d_prob_desc, int n, int* d_rank, int* d_id_by_rank, sdb_stream_t stream);
/* Pre-filter of the 2D pair test (csrc/polyfast.cuh): 0 = exact Clipper-equivalent sweep on every pair,
 * 1 (default) = closed-form overlap integral with a conservative bound first, exact sweep for the rest,
 * 2 = verify: both on every pair, disagreements are counted.  Results are identical in all modes.
 * stats: out4 = {pairs tested, pairs that needed the exact sweep, verify mismatches, nms calls}. */
int sdb_nms2d_set_filter(int mode);
/* 1 (default): frontier rounds >= 1 run inside one cooperative kernel with on-device termination; 0: host-driven rounds.
 * Results are identical. */
int sdb_nms2d_set_tail(int on);
void sdb_nms2d_filter_stats(unsigned long long* out4, int reset);

/* paint polygons (geom2d.py:149-197): d_rank[i] = paint rank of polygon i (0 = painted first;
 * a pixel takes the covering polygon of highest rank), d_id_by_rank[r] = value written for
 * rank r (reference: original index + 1); d_out int32[ny*nx] is zeroed first. */
int sdb_polygons_to_label_2d(const float* d_coord, const int* d_rank, const int* d_id_by_rank,
                             int n_polys, int n_rays, int ny, int nx, int* d_out,
                             sdb_stream_t stream);

/* dist_to_coord (geom2d.py:130-146): coord[n,2,R] = f32(dist * sincos(phi_k) in f64) * scale + points.
 * d_sincos = float64[2*R] = [sin(phi_k) | cos(phi_k)] evaluated by the caller with numpy (same
 * libm/SIMD routine as the reference); d_points float64[n,2] (y,x) (integer pixel centres, or
 * already multiplied by the predict_instances(scale=...) rescale, model2d.py:539-546). */
int sdb_dist_to_coord_2d(const float* d_dist, const double* d_points, int n_polys, int n_rays,
                         const double* d_sincos, double scale_y, double scale_x,
                         float* d_coord, sdb_stream_t stream);

/* 3D label painting on device arrays (see _LIB_polyhedron_to_label): polyhedra in painting order
 * (descending probability, geom3d.py:176-180), first cover wins; d_labels[n_polys] must be non-zero. */
int sdb_polyhedron_to_label(const float* d_dist, const float* d_points, const float* d_verts,
                            const int* d_faces, int n_polys, int n_rays, int n_faces,
                            const int* d_labels, int nz, int ny, int nx, int render_mode,
                            int use_overlap_label, int overlap_label, int* d_result,
                            sdb_stream_t stream);

/* sphere culling of bounding-box voxels in the 3-D label rendering (1 = default); label maps are identical either way */
int sdb_label3d_set_cull(int on);

/* k_heavy volume stages (S3 kernel / S4 hull intersection): 0 (default) = per-(k, j) plane scaling as validated by the GPU goldens,
 * 1 = planes scaled once per pair + early-out for non-cutting planes (sd3::face_cone_volume_n; bit-identical results on the
 * host build, not yet run on a GPU -- experimental until then). */
int sdb_nms3d_set_variant(int norm_planes);
/* 1 (default): a rigorous lower bound of the kernel-intersection volume (ray-wise distances to the 2F planes from the centre
 * midpoint, fan of tetrahedra) decides `iou > threshold` of stage S3 before the volume itself is computed; 0: always the
 * volume.  Decisions are identical (margin 1e-5 relative).  The same switch governs the two-sided fan bounds of S4 / S3 in the
 * second launch and the direction bins of S5 (2: bounds on the coarse ray fan, without the extra ray per face). */
int sdb_nms3d_set_s3_bound(int on);
/* 1 (default): the heavy stages run as three launches per round -- S3 for all pairs, hull facets of the polyhedra that stay open
 * (one warp each), S4 + S5 with those facets; 0: one launch doing everything per pair.  Decisions identical. */
int sdb_nms3d_set_split(int on);

/* relabel_sequential on a device label map (stardist/matching.py:319-406; callers model3d.py:645, base.py:959):
 * labels occurring in d_labels[n] (values in [0, max_label], 16-byte aligned) are renumbered offset, offset+1, ...
 * in ascending order, 0 stays 0, in place.  d_forward_map: scratch of max_label + 3 ints; on return [0..max_label]
 * holds the forward map (matching.py:399-401).  *h_count = number of distinct non-zero labels.  Negative labels
 * are an error like in the reference (matching.py:374).  Synchronises the stream once (count read-back). */
int sdb_relabel_sequential(int* d_labels, long long n, int max_label, int offset, int* d_forward_map,
                           int* h_count, sdb_stream_t stream);

/* sparse label-overlap table (stardist/matching.py:38-52, _label_overlap): every distinct pair (a, b) = (d_a[i], d_b[i]) of
 * two int32 label maps of n pixels / voxels, background 0 included, with its pixel count, sorted by (a, b).  Results go to
 * d_pairs[capacity][2] (int32 a, b) and d_counts[capacity] (int64); *h_n_pairs = number of pairs, after one stream
 * synchronisation.  When the pairs do not fit in `capacity`, nothing is written and *h_n_pairs > capacity is returned: an
 * upper bound of the number of distinct pairs, so the caller can retry once with that capacity.  Negative labels are an
 * error (matching.py:27-35).  capacity in [1, 2^28]: maps with more than 2^28 distinct pairs are not supported. */
int sdb_label_overlap(const int* d_a, const int* d_b, long long n, int* d_pairs, long long* d_counts,
                      long long capacity, long long* h_n_pairs, sdb_stream_t stream);

/* group_matching_labels (stardist/matching.py:409-472) on an int32 stack d_stack[n_frames][frame_size]; the three calls
 * share the table machinery and capacity protocol of sdb_label_overlap (d_keys / d_counts [capacity], *h_n_keys after one
 * stream synchronisation, > capacity = nothing written and an upper bound returned; negative labels are an error).
 * sdb_stack_labels: every distinct (frame, label) of the stack, background 0 included, as the sorted keys
 *   (frame << 32) | label with their pixel counts.
 * sdb_stack_overlap: the overlap tables of the frame pairs (p, p + 1), p in [first_pair, first_pair + n_pairs), on ids
 *   compacted per frame as relabel_sequential numbers them (0 stays 0, the non-zero labels of frame f become 1..n_f in
 *   ascending order): d_ids holds the sorted non-zero labels of every frame, those of frame f at
 *   [d_offsets[f], d_offsets[f + 1]).  Sorted keys ((p - first_pair) << 2 key_bits) | (a' << key_bits) | b' with their
 *   pixel counts; key_bits in [1, 31] must hold every compacted id, and n_pairs - 1 must fit in 63 - 2 key_bits bits.
 * sdb_stack_group_remap: d_out[0] = d_stack[0]; d_out[f] = d_lut[d_offsets[f] + a' - 1] where d_stack[f] has a
 *   compacted id a' > 0, else 0 (d_lut is laid out like d_ids).  Asynchronous. */
int sdb_stack_labels(const int* d_stack, long long n_frames, long long frame_size, long long* d_keys, long long* d_counts,
                     long long capacity, long long* h_n_keys, sdb_stream_t stream);
int sdb_stack_overlap(const int* d_stack, long long frame_size, long long first_pair, long long n_pairs, const int* d_ids,
                      const long long* d_offsets, int key_bits, long long* d_keys, long long* d_counts, long long capacity,
                      long long* h_n_keys, sdb_stream_t stream);
int sdb_stack_group_remap(const int* d_stack, long long n_frames, long long frame_size, const int* d_ids,
                          const long long* d_offsets, const int* d_lut, int* d_out, sdb_stream_t stream);

/* star distances (stardist2d.cpp:55-125 c_star_dist, stardist3d.cpp:245-345 c_star_dist3d), bit-identical to the reference.
 * d_labels: label map [H, W] / [D, H, W], uint16 (label_bytes 2) or int32 (label_bytes 4); labels are compared by their low
 * 16 bits (the reference's astype(np.uint16)).  h_dirs: HOST float32 table [2][n_rays] = [dy | dx] (dy = cosf(phi_k),
 * dx = sinf(phi_k), phi_k = float(k) * float(2 pi / n_rays), libm's single-precision functions) or h_rays [3][n_rays] =
 * [dz | dy | dx] (Rays.vertices as float32).  Dense mode (d_points NULL): d_out float32 [Ho, Wo(, ...), n_rays] with
 * Ho = (H - 1) / grid_y + 1 etc.  Point mode: d_points int32 [n_points][2 or 3] indices into that subsampled grid, d_out
 * float32 [n_points][n_rays].  A ray set whose walk cannot be bounded for the shape is an error (sdb_star_dist_walk_bound). */
int sdb_star_dist_2d(const void* d_labels, int label_bytes, int H, int W, int grid_y, int grid_x, int n_rays,
                     const float* h_dirs, const int* d_points, long long n_points, float* d_out, sdb_stream_t stream);
int sdb_star_dist_3d(const void* d_labels, int label_bytes, int D, int H, int W, int grid_z, int grid_y, int grid_x,
                     int n_rays, const float* h_rays, const int* d_points, long long n_points, float* d_out,
                     sdb_stream_t stream);
/* host-only check of a direction table ([ndim][n_rays], as above) for an image of the given shape: every ray needs a
 * component of magnitude >= max(2^-8, 2 ulp(max extent + 1 + max component)).  On success *h_cap = a step count after
 * which every walk has left the image (the kernels' loop cap); otherwise an error and a message. */
int sdb_star_dist_walk_bound(const float* h_dirs, int ndim, int n_rays, const int* shape, long long* h_cap);
/* host-pointer versions with the reference's semantics: src uint16, dst float32 dense; void, on failure dst is zeroed and
 * sdb_last_error() holds the message (cleared on success) */
void _LIB_star_dist_2d(const unsigned short* src, int H, int W, int n_rays, int grid_y, int grid_x, const float* dirs,
                       float* dst);
void _LIB_star_dist_3d(const unsigned short* src, int D, int H, int W, int n_rays, int grid_z, int grid_y, int grid_x,
                       const float* rays, float* dst);

/* batched dense star distances for training batches: d_labels int32 [batch][shape...] (maps laid end to end, each walked on
 * its own), d_out float32 [batch][Ho][Wo](...) with n_rays values at the start of every out_stride floats (out_stride
 * n_rays + 1 leaves a channel free: the dist_and_mask layout).  Same walk and table as sdb_star_dist_2d / _3d. */
int sdb_star_dist_batch(const int* d_labels, int ndim, int batch, const int* shape, const int* grid, int n_rays,
                        const float* h_dirs, int out_stride, float* d_out, sdb_stream_t stream);

/* per-label statistics of a sequential int32 label map (values in [0, n_labels], e.g. after sdb_relabel_sequential):
 * for label l >= 1, index l - 1: d_count[n_labels] pixel count, d_sum[n_labels][ndim] coordinate sums, d_bbox_min /
 * d_bbox_max [n_labels][ndim] smallest / largest coordinate (inclusive), axes in array order.  What regionprops gives
 * relabel_image_stardist (centroid = sum / count) and calculate_extents (bbox).  shape is a host int[ndim].  Negative
 * labels or labels above n_labels are an error.  Synchronises the stream once. */
int sdb_region_stats(const int* d_labels, int ndim, const int* shape, int n_labels, long long* d_count, long long* d_sum,
                     int* d_bbox_min, int* d_bbox_max, sdb_stream_t stream);

/* training targets (stardist/utils.py:98-153, _edt_prob_scipy and fill_label_holes), bit-identical to the reference.
 * d_labels: sequential int32 label map (values 0..n_labels, e.g. after sdb_relabel_sequential; negative labels mapped to 0
 * first), shape a host int[ndim], ndim 2 or 3, every extent <= 65535, at most 2^31 - 1 pixels.
 * sdb_edt_prob: d_prob float32 = float(sqrt(d2) / (sqrt(max of d2 over the label) + 1e-10)), d2 = squared distance to the
 * nearest pixel of another label, sum_a ((q_a - p_a) * s_a)^2 in float64 in axis order; h_sampling: HOST double[ndim]
 * (NULL = 1); black_border: positions just outside the image count as another label (the reference's constant-image rule).
 * sdb_fill_label_holes: d_out int32 = the largest label whose pixels or holes contain the pixel, 0 elsewhere; holes are
 * connected under generate_binary_structure(ndim, connectivity), connectivity in [1, ndim].  Uses sdb_region_stats and
 * synchronises the stream once (box sizes). */
int sdb_edt_prob(const int* d_labels, int ndim, const int* shape, int n_labels, const double* h_sampling, int black_border,
                 float* d_prob, sdb_stream_t stream);
int sdb_fill_label_holes(const int* d_labels, int ndim, const int* shape, int n_labels, int connectivity, int* d_out,
                         sdb_stream_t stream);
/* edt_prob of `batch` maps of `shape` laid end to end (no pass crosses an item; the constant-image rule is decided per item
 * from its label minimum and maximum, written to d_item_minmax int32 [batch][2]).  Labels are distinct across items, values
 * 0..n_labels.  Output at the grid positions (Do = (D - 1) / grid + 1 ...): d_prob float32 [batch][Do..] (-1 where d_neg,
 * uint8 [batch][Do..] or NULL, is set) and, when d_dist_and_mask is not NULL, the unmasked value at d_dist_and_mask[o *
 * dm_stride].  Does not synchronise. */
int sdb_edt_prob_batch(const int* d_labels, int ndim, int batch, const int* shape, int n_labels, const double* h_sampling,
                       const int* grid, const unsigned char* d_neg, int* d_item_minmax, float* d_prob, float* d_dist_and_mask,
                       int dm_stride, sdb_stream_t stream);

/* training batches (stardist/models/base.py:129-225, model2d.py:29-120, model3d.py:30-127, sample_patches.py).
 * sdb_fg_valid_index: d_mask uint8 [shape] = maximum_filter(labels, filter_size, mode='constant') > 0 and d_prefix int64
 * [rows + 1] = the prefix count of set positions over the rows of the box [p//2, s-p+p//2] (rows: every axis but the last,
 * C order); *h_n_valid (host) = d_prefix[rows].  Synchronises the stream once.
 * sdb_sample_select: positions (int32 [batch][3], 2-D: 0 first) of the drawn ranks of the items d_items (int64
 * [batch][10], see traindata.cu).  sdb_train_gather: patches at those positions -> d_x float32 [batch][patch][n_channels],
 * d_y_clamped int32 max(label, 0) (the label itself when clamp is 0), d_y_slots int32 (per-item sequential labels + the item's slot offset), and at the grid
 * positions d_neg uint8 (label < 0) and, if not NULL, d_y_slots_grid; d_flags[0] |= 1 where a slot with class -2 (no class
 * given) occurs.  sdb_class_map: prob_class float32 [batch][out_shape][n_classes + 1] (mask_to_categorical of the slots'
 * classes d_class_table, -1 = None, then scipy's order-0 zoom with the source indices d_zoom_index int32 [sum out_shape],
 * then -1 where d_neg). */
int sdb_fg_valid_index(const int* d_labels, int ndim, const int* shape, const int* filter_size, const int* patch_size,
                       unsigned char* d_mask, long long* d_prefix, long long* h_n_valid, sdb_stream_t stream);
int sdb_sample_select(const long long* d_items, int ndim, int batch, const int* patch_size, int* d_pos, sdb_stream_t stream);
int sdb_train_gather(const long long* d_items, const int* d_pos, int ndim, int batch, const int* patch_size, int n_channels,
                     const int* grid, const int* d_class_table, float* d_x, int* d_y_clamped, int* d_y_slots,
                     int* d_y_slots_grid, unsigned char* d_neg, int* d_flags, int clamp, sdb_stream_t stream);
int sdb_class_map(const int* d_y_slots, int ndim, int batch, const int* patch_size, const int* d_zoom_index,
                  const int* out_shape, const int* d_class_table, int n_classes, const unsigned char* d_neg, float* d_out,
                  sdb_stream_t stream);
/* The training notebooks' augmenter (augment.cu, DESIGN.md 4.2).  sdb_mt_normal: np.random.normal(0, 1, n) of numpy's legacy
 * RandomState from its state (h_key [624], pos, has_gauss, gauss as get_state() gives them) -> d_out float64 [n] and the state
 * numpy holds afterwards (h_key_out may be h_key); synchronises the stream.  Values may differ from numpy's by the ulps of
 * the device's double log; the state is numpy's.  sdb_augment_batch: per item b the output patch of d_params int64 [batch][12]
 * = (source axis of output axis 0..2, flip of output axis 0..2, float32 bits of scale and shift, float64 bits of sigma, noise
 * on, 0, 0), axes counted with a leading unit axis in 2-D; from the gathered d_x [batch][patch][n_channels], raw labels d_y_raw
 * and slots d_y_slots (sdb_train_gather with clamp 0) it writes d_x_out = x * s + t (float32), plus float32(double(.) +
 * sigma * d_noise[b][patch][n_channels]) with noise on, d_y_clamped = max(label, 0), d_y_slots_out, and at the grid positions
 * d_neg (label < 0) and, if not NULL, d_y_slots_grid -- what sdb_train_gather writes for the augmented patch. */
int sdb_mt_normal(const unsigned* h_key, int pos, int has_gauss, double gauss, long long n, double* d_out, unsigned* h_key_out,
                  int* h_pos_out, int* h_has_gauss_out, double* h_gauss_out, sdb_stream_t stream);
int sdb_augment_batch(const long long* d_params, int ndim, int batch, const int* patch_size, int n_channels, const int* grid,
                      const float* d_x, const int* d_y_raw, const int* d_y_slots, const double* d_noise, float* d_x_out,
                      int* d_y_clamped, int* d_y_slots_out, int* d_y_slots_grid, unsigned char* d_neg, sdb_stream_t stream);
/* helpers.cu: the public helpers that read a whole label, mask or distance map (DESIGN.md §4).
 * sdb_label_class_map: mask_to_categorical (stardist/utils.py:318-380) of an int32 label map of n pixels -> d_out float32
 *   [n][n_classes + 1]: 0 -> channel 0 is 1; a label -> its code in d_codes at its position in the ascending d_keys [n_keys]
 *   (every non-zero label of the map must be there): 1..n_classes one-hot, 0 all zeros, -1 (None) channel 0 is 0 and the
 *   others -1.  Asynchronous.
 * sdb_mask_compact_count / _write: the set elements of the box [lo, hi) of a contiguous mask d_mask [shape] (ndim in [1, 4],
 *   elements of elem_size bytes), in C order.  An element is set when the low bit of its first byte is (nonzero 0: numpy's
 *   mask & 1 on a bool or integer mask) or when any of its bytes is non-zero (nonzero 1: np.where).  _count writes the row
 *   prefix d_prefix int64 [rows + 1] (rows: the box's extents over every axis but the last, multiplied) and *h_n, after one
 *   stream synchronisation; _write then writes the n absolute coordinates axis after axis, d_coords int32 [ndim][n], and, when
 *   d_prob (float32, the mask's shape) is not NULL, d_w [n] = d_prob at them.  Asynchronous.
 * sdb_gather_patches: n_samples crops of shape patch [ndim] (ndim in [1, 4]) of the contiguous array d_src [shape] with
 *   elements of elem_size in {1, 2, 4, 8, 16} bytes, starting at d_starts int64 [n_samples][ndim] -> d_out [n_samples][patch],
 *   copied as words.  Asynchronous.
 * sdb_dist_to_volume / sdb_dist_to_centroid: c_dist_to_volume / c_dist_to_centroid (stardist3d.cpp:146-234) on a float32 map
 *   d_dist [nz][ny][nx][n_rays] with the rays' d_verts float32 [n_rays][3] and d_faces int32 [n_faces][3] (indices below
 *   n_rays), n_rays <= 256, n_faces <= 512: d_out float32 [nz][ny][nx] (volume) or [nz][ny][nx][3] (centroid, plus the
 *   voxel's (k, j, i) when absolute), bit-identical to the reference.  Asynchronous. */
int sdb_label_class_map(const int* d_labels, long long n, const int* d_keys, const int* d_codes, int n_keys, int n_classes,
                        float* d_out, sdb_stream_t stream);
int sdb_mask_compact_count(const void* d_mask, int elem_size, int nonzero, int ndim, const long long* shape, const long long* lo,
                           const long long* hi, long long* d_prefix, long long* h_n, sdb_stream_t stream);
int sdb_mask_compact_write(const void* d_mask, int elem_size, int nonzero, int ndim, const long long* shape, const long long* lo,
                           const long long* hi, const long long* d_prefix, long long n, int* d_coords, const float* d_prob,
                           float* d_w, sdb_stream_t stream);
int sdb_gather_patches(const void* d_src, int elem_size, int ndim, const long long* shape, const long long* patch,
                       const long long* d_starts, long long n_samples, void* d_out, sdb_stream_t stream);
int sdb_dist_to_volume(const float* d_dist, int nz, int ny, int nx, int n_rays, const float* d_verts, const int* d_faces,
                       int n_faces, float* d_out, sdb_stream_t stream);
int sdb_dist_to_centroid(const float* d_dist, int nz, int ny, int nx, int n_rays, const float* d_verts, const int* d_faces,
                         int n_faces, int absolute, float* d_out, sdb_stream_t stream);
/* host-pointer versions on any int32 label map (negative labels are never an object; relabelling, the constant-image rule and
 * the mapping back to the original labels happen inside): void, on failure the result is zeroed and sdb_last_error() holds
 * the message (cleared on success) */
void _LIB_edt_prob(const int* lbl, int ndim, const int* shape, const double* sampling, float* prob);
void _LIB_fill_label_holes(const int* lbl, int ndim, const int* shape, int connectivity, int* out);

/* 3D NMS on device arrays (see _LIB_non_maximum_suppression_sparse); d_keep is uint8[n_polys]. */
int sdb_nms3d(const float* d_dist, const float* d_points, const float* d_verts, const int* d_faces,
              int n_polys, int n_rays, int n_faces, float threshold, int use_bbox, int use_kdtree,
              int verbose, unsigned char* d_keep, sdb_stream_t stream);

/* threshold + border mask + compaction + sort (nms.py:6-17, base.py:606-610, nms.py:167):
 * prob is [H*W] (2D) / [D*H*W] (3D) float32; candidates are pixels with prob > thresh that lie at
 * least b_lo/b_hi pixels inside along each axis and inside valid_* (un-padded) extents.
 * Output sorted by (prob desc, flat index desc) == np.argsort(prob, kind='stable')[::-1].
 * d_count receives the number of candidates (also returned through *h_count after a sync). */
int sdb_threshold_sort(const float* d_prob, int ndim, const int* shape, const int* valid_shape,
                       const int* b_lo, const int* b_hi, float prob_thresh,
                       int* d_sorted_index, float* d_sorted_prob, int capacity, int* h_count,
                       sdb_stream_t stream);

/* gather: out_dist[r,:] = max(1e-3, dist[idx[r],:]), out_points[r,:] = unravel(idx[r]) * grid */
int sdb_gather_candidates(const float* d_dist, const int* d_index, int n, int n_rays, int ndim,
                          const int* shape, const int* grid, float* d_out_dist,
                          float* d_out_points, sdb_stream_t stream);

/* sparse candidate store (large volumes: the dense dist map is never written, SURVEY H7 / base.py:580-593) */
int sdb_count_above(const float* d_prob, long long n, float thresh, int* h_count, sdb_stream_t stream);
int sdb_store_rows_above(const float* d_prob, const float* d_dist, long long n, int n_rays, float thresh, long long flat0,
                         int row0, int capacity, float* d_store, int* d_slot, sdb_stream_t stream);
int sdb_gather_candidates_slots(const float* d_store, const int* d_slot, const int* d_index, int n, int n_rays, int ndim,
                                const int* shape, const int* grid, float* d_out_dist, float* d_out_points, sdb_stream_t stream);

/* ---- U-Net forward building blocks (NHWC float32; see stardist_b200/csrc/unet*.cu) ---- */

/* 3x3 'same' convolution + bias + optional ReLU.  The input may be the channel concatenation
 * [nearest-upsample2x(in_lo), in_skip] (csbdeep unet_block decoder, SURVEY A.1): pass in_lo=NULL,
 * cin_lo=0 for a plain convolution.  weights are Keras layout (3,3,Cin,Cout), Cin = cin_lo+cin_skip. */
int sdb_conv3x3_2d(const float* d_in, const float* d_in_lo, int n, int h, int w, int cin_skip,
                   int cin_lo, const float* d_weight, const float* d_bias, int cout, int relu,
                   float* d_out, sdb_stream_t stream);

int sdb_maxpool2x2_2d(const float* d_in, int n, int h, int w, int c, float* d_out, sdb_stream_t stream);

/* N-d variants (NDHWC): kz = 1 -> 2-D (d == 1), kz = 3 -> 3x3x3 with Keras kernels (3,3,3,Cin,Cout);
 * (uz,uy,ux) = nearest up-sampling factors of the optional low-resolution source; pooling (pz,py,px). */
int sdb_conv3_nd(const float* d_in, const float* d_in_lo, int n, int d, int h, int w, int cin_skip,
                 int cin_lo, int uz, int uy, int ux, const float* d_weight, const float* d_bias, int cout,
                 int kz, int relu, float* d_out, sdb_stream_t stream);
int sdb_maxpool_nd(const float* d_in, int n, int d, int h, int w, int c, int pz, int py, int px, float* d_out, sdb_stream_t stream);
/* ResNet backbone (model3d.py:402-447): convolution with arbitrary kernel extent and strides under TensorFlow's
 * padding='same' rule (asymmetric: pad_before = pad_total / 2), fp32 CUDA cores; residual add (+ ReLU). */
int sdb_conv_generic_nd(const float* d_in, int n, int d, int h, int w, int cin, const float* d_w, const float* d_b, int cout,
                        int kz, int ky, int kx, int sz, int sy, int sx, int relu, float* d_out, sdb_stream_t stream);
int sdb_add_act(const float* d_a, const float* d_b, long long n, int relu, float* d_out, sdb_stream_t stream);
/* multi-class head (model2d.py:339-347): prob_class = softmax over n_out = n_classes + 1 outputs of a 1x1 convolution of
 * fp32 features [npix, cfeat] with weights [cfeat][n_out]; sdb_merge_split: split fp16 planes (hi, lo) -> fp32. */
int sdb_class_head(const float* d_feat, long long npix, int cfeat, const float* d_w, const float* d_b, int n_out, float* d_out,
                   sdb_stream_t stream);
int sdb_merge_split(const void* d_hi, const void* d_lo, long long n, float* d_out, sdb_stream_t stream);

/* Any layer shape (csrc/unet_any.cu), for the models outside the default architecture family.  `act` is an activation
 * id: 0 linear, 1 relu, 2 elu, 3 selu, 4 tanh, 5 sigmoid, 6 softplus, 7 softsign, 8 exponential, 9 swish, 10 gelu.
 * sdb_conv_any_nd: tiled convolution, NDHWC fp32 (2-D: d = kz = sz = 1), Keras kernels (kz,ky,kx,Cin,Cout) with extents
 * 1..7, strides 1 or 2 under TensorFlow's padding='same' (out = ceil(in / s), pad_before = pad_total / 2), output
 * [n, ceil(d/sz), ceil(h/sy), ceil(w/sx), cout] = act(conv + bias).  Input channels are [upsample(in_lo), in] when
 * cin_lo > 0 (stride 1 only; (uz,uy,ux) nearest up-sampling factors, (d,h,w) the skip's size).
 * sdb_heads_any: the 1^d heads of sdb_heads_2d for any cfeat >= 1 and 1 <= n_rays <= 256.
 * sdb_maxpool_any_nd: sdb_maxpool_nd for any c.  sdb_add_act_any: out = act(a + b). */
int sdb_conv_any_nd(const float* d_in, const float* d_in_lo, int n, int d, int h, int w, int cin_skip, int cin_lo,
                    int uz, int uy, int ux, const float* d_weight, const float* d_bias, int cout,
                    int kz, int ky, int kx, int sz, int sy, int sx, int act, float* d_out, sdb_stream_t stream);
int sdb_heads_any(const float* d_feat, long long npix, int cfeat, const float* d_wp, const float* d_bp,
                  const float* d_wd, const float* d_bd, int n_rays, float* d_prob, float* d_dist, sdb_stream_t stream);
int sdb_maxpool_any_nd(const float* d_in, int n, int d, int h, int w, int c, int pz, int py, int px, float* d_out,
                       sdb_stream_t stream);
int sdb_add_act_any(const float* d_a, const float* d_b, long long n, int act, float* d_out, sdb_stream_t stream);
/* sdb_act_any: y = act(z) elementwise (y may be z), the epilogue of sdb_conv_any_nd as a separate pass: a convolution run
 * linear and then this gives the fused result bit for bit.  sdb_act_backward: g *= act'(z) in place, z the pre-activation;
 * relu zeroes g where z <= 0.  sdb_conv_dgrad_any_nd: input gradient of a stride-1 'same' convolution with kernel extents
 * (kz,ky,kx) in 1..7, any cin and cout: dx [n,d,h,w,cin] from dy [n,d,h,w,cout] and wf (kz,ky,kx,cout,cin), the kernel
 * flipped by sdb_conv_flip_weights; a decoder layer's dx is d[upsample(x_lo), skip], split by sdb_decoder_split. */
int sdb_act_any(const float* d_z, long long n, int act, float* d_y, sdb_stream_t stream);
int sdb_act_backward(float* d_g, const float* d_z, long long n, int act, sdb_stream_t stream);
int sdb_conv_dgrad_any_nd(const float* d_dy, int n, int d, int h, int w, int cout, const float* d_wf, int cin,
                          int kz, int ky, int kx, float* d_dx, sdb_stream_t stream);

/* 1x1 heads: prob = sigmoid(x.Wp+bp) [npix], dist = x.Wd+bd [npix*n_rays] */
int sdb_heads_2d(const float* d_feat, long long npix, int cfeat, const float* d_wp, const float* d_bp,
                 const float* d_wd, const float* d_bd, int n_rays, float* d_prob, float* d_dist,
                 sdb_stream_t stream);

/* ---- wgmma / TMA U-Net path (stardist_b200/csrc/unet_tc.cu) -------------------------------------
 * Activations are two fp16 planes (hi, lo) per tensor, hi = fp16(v), lo = fp16(v - hi); weights are
 * split the same way into [9][cout][cin] planes by sdb_split_weights.  fp32 accumulation in registers. */
int sdb_conv3x3_tc(const void* src0_hi, const void* src0_lo, int c_src0, const void* src1_hi, const void* src1_lo,
                   int c_src1, int n, int h, int w, const void* w_hi, const void* w_lo, float w_scale, const float* d_bias, int cout,
                   int relu, int up2x, void* out_hi, void* out_lo, sdb_stream_t stream);
/* 1x1 heads on the tensor cores (one tap, K = cfeat): head weights [1][np][cfeat] split fp16, row 0 = prob,
 * rows 1..n_rays = dist, zero padded to np in {48, 80, 112, 144}; outputs fp32 */
int sdb_heads_tc(const void* f_hi, const void* f_lo, int cfeat, int n, int h, int w, const void* w_hi, const void* w_lo,
                 float w_scale, const float* d_bias, int np, int n_rays, float* d_prob, float* d_dist, sdb_stream_t stream);
/* Last convolution of the backbone fused with the 1x1 heads (model2d.py:329-337: features conv3x3 + ReLU, then
 * Conv2D(1,1,sigmoid) -> prob and Conv2D(n_rays,1,linear) -> dist): src as in sdb_conv3x3_tc, cout = 128,
 * heads_w fp32 [128][36] (columns 0..n_rays-1 = dist kernels, column 32 = prob kernel, rest 0), heads_b fp32 [36];
 * n_rays <= 32.  Outputs prob [n,h,w] and dist [n,h,w,n_rays] fp32; the feature map is not materialised. */
int sdb_conv3x3_heads_tc(const void* src0_hi, const void* src0_lo, int c_src0, const void* src1_hi, const void* src1_lo,
                         int c_src1, int n, int h, int w, const void* w_hi, const void* w_lo, float w_scale, const float* d_bias,
                         int relu, const float* d_heads_w, const float* d_heads_b, int n_rays, float* d_prob, float* d_dist,
                         sdb_stream_t stream);
/* 3-D U-Net on the tensor cores (model3d.py:360-399): 3x3x3 convolution of ONE volume [d,h,w,c] in split fp16 planes
 * (the z planes as the tensor map's image axis; weights [27][cout][cin] from sdb_split_weights_3d,
 * tap = dz*9 + dy*3 + dx; up2x: 0 none, 2 = nearest 2x2x2 up-sampling written by the epilogue), max-pooling on split
 * planes, and the fp32 -> split conversion behind the CUDA-core stem. */
int sdb_conv3x3x3_tc(const void* src0_hi, const void* src0_lo, int c_src0, const void* src1_hi, const void* src1_lo,
                     int c_src1, int d, int h, int w, const void* w_hi, const void* w_lo, float w_scale, const float* d_bias, int cout,
                     int relu, int up2x, void* out_hi, void* out_lo, sdb_stream_t stream);
int sdb_split_weights_3d(const float* d_w, int cin, int cout, float w_scale, void* w_hi, void* w_lo, sdb_stream_t stream);
int sdb_maxpool3d_split(const void* in_hi, const void* in_lo, int d, int h, int w, int c, int pz, int py, int px,
                        void* out_hi, void* out_lo, sdb_stream_t stream);
int sdb_split_f32(const float* d_in, long long n, void* out_hi, void* out_lo, sdb_stream_t stream);
/* kernel variant of sdb_conv3x3_tc: 0 (default) = the measured best, currently the same kernel as 3; 1 = one 8x16 tile per
 * CTA, 3 = persistent CTAs with 64-channel K blocks where the channel counts allow, 4 = persistent CTAs with 32-channel K blocks
 * (per-layer timings: tests/tools/conv_layers.py, DESIGN.md 4.1).  Results are identical up to fp32 summation order. */
int sdb_tc_set_variant(int variant);
/* 1 (default): the small split-fp16 products (lo*Whi, hi*Wlo) accumulate in their own registers, the main accumulator
 * takes one truncating tensor-core add per k-step; 0: all products into one accumulator (kept for A/B error
 * measurements: tests/tools/tc_split_error.py).  Applies to every tensor-core convolution. */
int sdb_tc_set_split_acc(int on);
int sdb_tc_error_check(sdb_stream_t stream);
/* w_scale: power of two the weights are multiplied by before the split (undone on the accumulator) */
int sdb_split_weights(const float* d_w, int cin, int cout, float w_scale, void* w_hi, void* w_lo, sdb_stream_t stream);
int sdb_stem_split(const float* d_in, int n, int h, int w, int cin, const float* d_w, const float* d_b, int cout, int relu,
                   void* out_hi, void* out_lo, sdb_stream_t stream);
int sdb_maxpool_split(const void* in_hi, const void* in_lo, int n, int h, int w, int c, void* out_hi, void* out_lo, sdb_stream_t stream);
int sdb_heads_split(const void* f_hi, const void* f_lo, long long npix, int cfeat, const float* d_wp, const float* d_bp,
                    const float* d_wd, const float* d_bd, int n_rays, float* d_prob, float* d_dist, sdb_stream_t stream);

/* ---- predict_instances_big on the device (stardist/big.py:340-413 filter_objects, :319-326 write; base.py:959) ---- */
/* per-label bounding boxes of a C-contiguous int32 label tile (ndim 2 or 3): d_bbox int32[(max_label+1)*6] =
 * {min0,min1,min2,max0,max1,max2} (inclusive; 2-D tiles use columns 1,2,4,5), absent labels keep {INT_MAX.., -1..};
 * d_bad[0] != 0 when a value lies outside [0, max_label].  Replaces skimage.measure.regionprops (big.py:373). */
int sdb_label_bbox(const int* d_labels, int ndim, const int* shape, int max_label, int* d_bbox, int* d_bad, sdb_stream_t stream);
/* in place labels[i] = lut[labels[i]] for non-zero entries (foreign objects -> 0, kept objects -> 1..n_kept) */
int sdb_label_remap(int* d_labels, long long n, const int* d_lut, sdb_stream_t stream);
/* BlockND.write with the running label offset folded in: dst[origin+idx] = tile[idx] + add where tile[idx] > 0 */
int sdb_label_write(const int* d_tile, int ndim, const int* tile_shape, int add, int* d_dst, const int* dst_shape,
                    const int* origin, sdb_stream_t stream);

/* ---- the steps in front of the network (SURVEY 8 f3): csbdeep.utils.normalize / PercentileNormalizer and the `scale=` zoom ---- */
/* exact order statistics of the region [0,valid) of a C-contiguous float32 array: h_out[q] = sorted(region)[ranks[q]], <= 8 ranks */
int sdb_select_ranks(const float* d_x, int ndim, const int* shape, const int* valid, const long long* ranks, int n_ranks,
                     float* h_out, sdb_stream_t stream);
/* in place x = (x - mi) / den in float32 (den = ma - mi + eps computed by the caller in float32), optional clip to [0,1] */
int sdb_normalize_mi_ma(float* d_x, long long n, float mi, float den, int clip, sdb_stream_t stream);
/* scipy.ndimage.zoom(x, zoom, order=1) (stardist/models/base.py:735) for ndim 2 / 3; out_shape = round(in_shape * zoom) */
int sdb_zoom_linear(const float* d_in, int ndim, const int* in_shape, const int* out_shape, float* d_out, int round_int,
                    double int_lo, double int_hi, sdb_stream_t stream);   /* round_int: integer source image -> scipy's rounding */
/* numpy.pad(mode='reflect') at the end of each spatial axis of a channels-last array (StarDistPadAndCropResizer.before) */
int sdb_pad_reflect_end(const float* d_in, int ndim, const int* in_shape, const int* out_shape, int channels, float* d_out,
                        sdb_stream_t stream);

/* ---- the network boundary as C entry points (SURVEY 8b: keras_model.predict, stardist/models/base.py:408-410) ----
 * A network object is built from the configuration fields that define the graph (model2d.py:310-349 / model3d.py:360-399) and
 * the Keras kernels / biases (HOST pointers, layout (k..., Cin, Cout) / (Cout,)) in the order sdb_unet_layer_name(cfg, i)
 * reports for i in [0, sdb_unet_layer_count(cfg)): the convolution layers in topology order, then "prob", "dist".
 * _LIB_unet_forward_2d/3d take a DEVICE input [h, w, Cin] / [d, h, w, Cin] float32 (normalised, padded to multiples of
 * 2^depth) and write prob [h, w] / [d, h, w] and dist [..., n_rays] (raw head outputs: sigmoid applied to prob, dist
 * not yet clamped to 1e-3).  Default architecture family only (U-Net, 3^d kernels, pool 2, ReLU, no batch norm, grid 1);
 * sdb_unet_create returns NULL (see sdb_last_error) for anything else. */
typedef struct sdb_unet sdb_unet;
typedef struct {
  int ndim, n_channel_in, n_rays, unet_n_depth, unet_n_filter_base, unet_n_conv_per_depth, net_conv_after_unet;
  int grid[3];
} sdb_unet_config;
int sdb_unet_layer_count(const sdb_unet_config* cfg);
const char* sdb_unet_layer_name(const sdb_unet_config* cfg, int i);
sdb_unet* sdb_unet_create(const sdb_unet_config* cfg, const float* const* kernels, const float* const* biases);
void sdb_unet_destroy(sdb_unet* net);
int _LIB_unet_forward_2d(sdb_unet* net, const float* d_x, int h, int w, float* d_prob, float* d_dist, sdb_stream_t stream);
int _LIB_unet_forward_3d(sdb_unet* net, const float* d_x, int d, int h, int w, float* d_prob, float* d_dist, sdb_stream_t stream);

/* ---- training step of the U-Net (csrc/unet_train.cu): fp32 CUDA cores, fixed-order reductions, no float atomics ----
 * Weight gradient of a 3^d (kz = 3 in 3-D, 1 in 2-D; kyx = 3) or 1^d (kz = kyx = 1) 'same' convolution over the whole batch:
 * dw (k..., cin, cout) = sum_p x[p + tap] * dy[p], db = sum_p dy[p]; the input is [upsample(x_lo), skip] as in sdb_conv3_nd,
 * dy has row stride ldy >= cout.  d_work holds sdb_conv_wgrad_workspace(n*d*h*w, taps, cin_skip + cin_lo, cout) floats. */
long long sdb_conv_wgrad_workspace(long long npix, int taps, int cin, int cout);
int sdb_conv_wgrad_nd(const float* d_x, const float* d_x_lo, int n, int d, int h, int w, int cin_skip, int cin_lo,
                      int uz, int uy, int ux, int kz, int kyx, const float* d_dy, int ldy, int cout, float* d_work,
                      long long work_floats, float* d_dw, float* d_db, sdb_stream_t stream);
/* the same for any kernel extents (kz,ky,kx) in 1..7 at stride 1, TensorFlow 'same' front offsets (k - 1) / 2; the
 * workspace is sdb_conv_wgrad_workspace(n*d*h*w, kz*ky*kx, cin_skip + cin_lo, cout) floats */
int sdb_conv_wgrad_any_nd(const float* d_x, const float* d_x_lo, int n, int d, int h, int w, int cin_skip, int cin_lo,
                          int uz, int uy, int ux, int kz, int ky, int kx, const float* d_dy, int ldy, int cout, float* d_work,
                          long long work_floats, float* d_dw, float* d_db, sdb_stream_t stream);
/* wf (k..., cout, cin) = w (k..., cin, cout) flipped along every spatial axis (taps = the kernel's box volume): the input
 * gradient of a stride-1 3^d 'same' convolution is sdb_conv3_nd of dy with wf, zero bias, no ReLU (sdb_conv_dgrad_any_nd
 * for other extents) */
int sdb_conv_flip_weights(const float* d_w, int taps, int cin, int cout, float* d_wf, sdb_stream_t stream);
/* TF32 tensor-core variants of the two gradients above (csrc/unet_train_tf32.cu), the precision mode of
 * stardist_b200.enable_tensor_float_32_execution (DESIGN.md 4.2).  rna(v) is cvt.rna.tf32.f32: v rounded to 10 explicit
 * mantissa bits, nearest, ties away from zero; products accumulate in fp32, with no float atomics (bit-identical run to run).
 * sdb_conv_wgrad_tf32_nd: sdb_conv_wgrad_nd's arguments, shapes and workspace; dw = sum_p rna(x[p + tap]) * rna(dy[p]) and
 * db = sum_p dy[p] unrounded, in fp32.  sdb_conv_dgrad_tf32_nd: the input gradient of a stride-1 3^d 'same' convolution,
 * gin [n,d,h,w,cin] = sum over (tap, co) of rna(dy[p + tap - 1, co]) * rna(wf[tap, co, ci]) with wf (k..., cout, cin) from
 * sdb_conv_flip_weights (kz = 1 with d = 1 in 2-D, kz = 3 in 3-D; kyx = 3); the shapes sdb_conv3_nd takes for it: cout <= 4
 * with cin 32 or 64, or cout % 8 == 0 with cin % 32 == 0. */
int sdb_conv_wgrad_tf32_nd(const float* d_x, const float* d_x_lo, int n, int d, int h, int w, int cin_skip, int cin_lo,
                           int uz, int uy, int ux, int kz, int kyx, const float* d_dy, int ldy, int cout, float* d_work,
                           long long work_floats, float* d_dw, float* d_db, sdb_stream_t stream);
int sdb_conv_dgrad_tf32_nd(const float* d_dy, int n, int d, int h, int w, int cout, const float* d_wf, int cin, int kz, int kyx,
                           float* d_gin, sdb_stream_t stream);
/* bf16 tensor-core training kernels (csrc/unet_train_bf16.cu), the mixed_bfloat16 policy of stardist_b200.mixed_precision
 * (DESIGN.md 4.2).  Activations and gradients between layers are bf16 (void* below: __nv_bfloat16); parameters, biases and
 * gradients of parameters are fp32.  Every GEMM multiplies bf16 values and accumulates in fp32; an fp32 operand is rounded
 * to bf16 on load (round to nearest even); every bf16 store is one such rounding of an fp32 value.  No float atomics.
 * sdb_cast_bf16: out = bf16(in).  sdb_weights_bf16: w (taps, cin, cout) fp32 -> bf16, flip = 0 to out[(tap*cout + co)*ld +
 * ci] (the layout sdb_conv_bf16_nd reads, ld = cin), flip = 1 to out[((taps-1-tap)*cin + ci)*ld + co] (the flipped kernel
 * of sdb_conv_flip_weights in that layout, ld = cout: the input gradient's weights).
 * sdb_conv_bf16_nd: y = act(conv(x) + b) with 'same' padding, stride 1, extents kz, ky, kx in {1, 3}, over the input
 * [upsample(x_lo), skip] (x = skip, cin_lo = 0 for none); wb [taps][cout][cin_skip + cin_lo] bf16, b fp32 [cout] or NULL;
 * relu = 1 applies ReLU; accumulate = 1 adds the result to the bf16 already in d_out (one rounding of the sum).  The input
 * gradient is this kernel on dy with the flip = 1 weights, no bias.
 * sdb_gemm_bf16_f32in: out [npix][nout] bf16 (+)= a [npix][k] (fp32, rounded on load) . wb [nout][k] -- the heads' and class
 * head's input gradients.  sdb_heads_bf16: prob = sigmoid(f . wp + bp), dist = f . wd + bd in fp32 from bf16 features, wb
 * [n_rays + 1][cfeat] (row 0 the prob kernel).  sdb_class_head_bf16: softmax(f . w + b) in fp32, wb [n_out][cfeat], logits
 * fp32 [npix][n_out] scratch.
 * sdb_conv_wgrad_bf16_nd: sdb_conv_wgrad_nd on bf16 x, x_lo and a dy that is bf16 (dy_bf16 = 1: ldy and cout multiples of 8)
 * or fp32 (rounded on load); kernels 1^d, 3^d and (1, 3, 3) (kz = 1, kyx = 3); same workspace and split reduction; db = sum_p
 * dy[p] in fp32 of dy as stored.
 * The rest are the bf16 versions of sdb_maxpool_any_nd, sdb_maxpool_backward_nd, sdb_relu_backward, sdb_decoder_split and
 * out = bf16(a + b). */
int sdb_cast_bf16(const float* d_in, long long n, void* d_out, sdb_stream_t stream);
int sdb_weights_bf16(const float* d_w, int taps, int cin, int cout, int flip, int ld, void* d_out, sdb_stream_t stream);
int sdb_conv_bf16_nd(const void* d_x, const void* d_x_lo, int n, int d, int h, int w, int cin_skip, int cin_lo, int uz, int uy,
                     int ux, int kz, int ky, int kx, const void* d_wb, const float* d_b, int cout, int relu, int accumulate,
                     void* d_out, sdb_stream_t stream);
int sdb_gemm_bf16_f32in(const float* d_a, long long npix, int k, const void* d_wb, int nout, int accumulate, void* d_out,
                        sdb_stream_t stream);
int sdb_heads_bf16(const void* d_feat, long long npix, int cfeat, const void* d_wb, const float* d_bp, const float* d_bd,
                   int n_rays, float* d_prob, float* d_dist, sdb_stream_t stream);
int sdb_class_head_bf16(const void* d_feat, long long npix, int cfeat, const void* d_wb, const float* d_b, int n_out,
                        float* d_logits, float* d_out, sdb_stream_t stream);
int sdb_conv_wgrad_bf16_nd(const void* d_x, const void* d_x_lo, int n, int d, int h, int w, int cin_skip, int cin_lo,
                           int uz, int uy, int ux, int kz, int kyx, const void* d_dy, int dy_bf16, int ldy, int cout,
                           float* d_work, long long work_floats, float* d_dw, float* d_db, sdb_stream_t stream);
int sdb_maxpool_bf16_nd(const void* d_in, int n, int d, int h, int w, int c, int pz, int py, int px, void* d_out,
                        sdb_stream_t stream);
int sdb_maxpool_backward_bf16_nd(const void* d_x, const void* d_gy, int n, int d, int h, int w, int c, int pz, int py, int px,
                                 int accumulate, void* d_gx, sdb_stream_t stream);
int sdb_relu_backward_bf16(void* d_g, const void* d_y, long long n, sdb_stream_t stream);
int sdb_decoder_split_bf16(const void* d_dcat, int n, int d, int h, int w, int c_lo, int c_skip, int uz, int uy, int ux,
                           void* d_dlo, void* d_dskip, sdb_stream_t stream);
int sdb_add_bf16(const void* d_a, const void* d_b, long long n, void* d_out, sdb_stream_t stream);
/* gradient of [upsample(x_lo), skip] -> d x_lo (block sums, the backward of nearest up-sampling) and d skip (overwritten) */
int sdb_decoder_split(const float* d_dcat, int n, int d, int h, int w, int c_lo, int c_skip, int uz, int uy, int ux,
                      float* d_dlo, float* d_dskip, sdb_stream_t stream);
/* g *= (y > 0) in place, y the saved ReLU output */
int sdb_relu_backward(float* d_g, const float* d_y, long long n, sdb_stream_t stream);
/* gradient of sdb_maxpool_nd to the first maximum of each window (row-major); accumulate = 1 adds to d_gx */
int sdb_maxpool_backward_nd(const float* d_x, const float* d_gy, int n, int d, int h, int w, int c, int pz, int py, int px,
                            int accumulate, float* d_gx, sdb_stream_t stream);
/* StarDist loss (DESIGN.md 4.2): prob = sigmoid output [npix], dist [npix][n_rays], targets prob_t [npix] and dist_and_mask
 * [npix][n_rays + 1].  Writes stats (n_p, mean mask), out = (loss, prob_loss, dist_loss, n_p == 0) and, if d_dhead is not NULL,
 * dhead [npix][n_rays + 1] = (dL/d prob logit, dL/d dist).  d_state (optional) = (t, n_skipped, skip) of the training step.
 * d_work holds sdb_stardist_loss_workspace(npix) bytes. */
long long sdb_stardist_loss_workspace(long long npix);
int sdb_stardist_loss(const float* d_prob, const float* d_dist, const float* d_prob_t, const float* d_dam, long long npix,
                      int n_rays, int mae, float lam, float w0, float w1, void* d_work, float* d_stats, float* d_dhead,
                      float* d_out, int* d_state, sdb_stream_t stream);
/* dfeat = dhead . [w_prob | w_dist]^T, times the features ReLU mask when relu = 1 */
int sdb_heads_backward(const float* d_feat, const float* d_dhead, long long npix, int cfeat, const float* d_wp,
                       const float* d_wd, int n_rays, int relu, float* d_dfeat, sdb_stream_t stream);
/* Weighted categorical cross-entropy of multi-class models (DESIGN.md 4.2): s = softmax output [npix][n_out], targets
 * prob_class t [npix][n_out] (all channels < 0 on ignored pixels), class weights d_class_w [n_out] on the device, n_out =
 * n_classes + 1 <= 32.  Writes *d_out_class = L_class, adds w2 * L_class to *d_total (the loss sdb_stardist_loss wrote) and, if
 * d_dz is not NULL, dz [npix][n_out] = dL/d(softmax logits).  d_work holds sdb_stardist_class_loss_workspace(npix) bytes. */
long long sdb_stardist_class_loss_workspace(long long npix);
int sdb_stardist_class_loss(const float* d_s, const float* d_t, long long npix, int n_out, const float* d_class_w, float w2,
                            void* d_work, float* d_dz, float* d_total, float* d_out_class, sdb_stream_t stream);
/* dfeat (+)= dz . W^T with W [cfeat][n_out] the prob_class kernel, times the ReLU mask of feat when relu = 1; accumulate = 1 adds
 * to d_dfeat instead of overwriting it */
int sdb_class_head_backward(const float* d_feat, const float* d_dz, long long npix, int cfeat, const float* d_w, int n_out,
                            int relu, int accumulate, float* d_dfeat, sdb_stream_t stream);
/* Data-parallel reduction of one training step (DESIGN.md 4.2).  d_rows [world][ld]: replica r's flat gradient in
 * d_rows[r * ld, + n_params) followed by its loss row (loss, prob_loss, dist_loss, skipped[, prob_class_loss]) of n_out >= 4
 * floats.  S = the replicas with skipped == 0 in ascending rank order, all replicas when none is.  Writes d_g = (sum over S) / |S|
 * and d_out [n_out] likewise (fp32 additions from S's first member, then one fp32 division), and advances the step state
 * d_state = (t, n_skipped, skip) once, skipped when no replica is.  d_rows and d_g may alias for world = 1.  No atomics. */
int sdb_replica_reduce(const float* d_rows, int world, long long n_params, int n_out, long long ld, float* d_g, float* d_out,
                       int* d_state, sdb_stream_t stream);
/* TF2 Keras Adam over n parameters; alpha = lr * coef[t - 1] with t = d_state[0]; nothing when d_state[2] (skipped step) */
int sdb_adam_step(float* d_w, const float* d_g, float* d_m, float* d_v, long long n, float lr, float one_minus_b1,
                  float one_minus_b2, float eps, const float* d_coef, const int* d_state, sdb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* STARDIST_B200_H */
