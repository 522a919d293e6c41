"""ctypes binding of libstardist_b200.so (the C ABI declared in include/stardist_b200.h).

The library is the product's only compute path: if it is missing, or no CUDA device is
usable, importing the ops fails loudly -- there is no CPU fallback.
"""
import ctypes, os
from ctypes import c_int, c_float, c_double, c_void_p, c_char_p, c_longlong, c_bool, POINTER

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libstardist_b200.so")

class StarDistB200Error(RuntimeError):
    pass

_lib = None

def _declare(lib):
    P = c_void_p
    lib.sdb_last_error.restype = c_char_p
    lib.sdb_last_error.argtypes = []
    lib.sdb_launch_count.restype = c_longlong
    lib.sdb_launch_count.argtypes = [c_int]
    lib.sdb_device_info.argtypes = [POINTER(c_int)] * 4
    lib.sdb_profile_enable.argtypes = [c_int]
    lib.sdb_profile_get.argtypes = [c_char_p, POINTER(c_double), POINTER(c_longlong), POINTER(c_double)]
    lib._LIB_non_maximum_suppression_2d.argtypes = [P, P, c_int, c_int, c_float, c_int, c_int, c_int, P]
    lib._LIB_polygons_to_label_2d.argtypes = [P, P, c_int, c_int, c_int, c_int, P]
    lib.sdb_nms2d.argtypes = [P, P, c_int, c_int, c_float, c_int, c_int, c_int, P, P]
    lib.sdb_nms2d_survivors.argtypes = [P, P, c_int, c_int, c_float, c_int, c_int, c_int, P, P, POINTER(c_int), P]
    lib.sdb_nms2d_survivors.restype = c_int
    lib.sdb_paint_order_2d.argtypes = [P, c_int, P, P, P]
    lib.sdb_paint_order_2d.restype = c_int
    lib.sdb_nms2d_set_filter.argtypes = [c_int]
    lib.sdb_nms2d_set_filter.restype = c_int
    lib.sdb_nms3d_set_split.argtypes = [c_int]
    lib.sdb_nms3d_set_split.restype = c_int
    lib.sdb_nms3d_set_s3_bound.argtypes = [c_int]
    lib.sdb_nms3d_set_s3_bound.restype = c_int
    lib.sdb_label3d_set_cull.argtypes = [c_int]
    lib.sdb_label3d_set_cull.restype = c_int
    lib.sdb_nms2d_set_tail.argtypes = [c_int]
    lib.sdb_nms2d_set_tail.restype = c_int
    lib.sdb_nms2d_filter_stats.argtypes = [POINTER(ctypes.c_ulonglong), c_int]
    lib.sdb_nms2d_filter_stats.restype = None
    lib.sdb_polygons_to_label_2d.argtypes = [P, P, P, c_int, c_int, c_int, c_int, P, P]
    lib.sdb_dist_to_coord_2d.argtypes = [P, P, c_int, c_int, P, c_double, c_double, P, P]
    lib.sdb_threshold_sort.argtypes = [P, c_int, POINTER(c_int), POINTER(c_int), POINTER(c_int), POINTER(c_int),
                                       c_float, P, P, c_int, POINTER(c_int), P]
    lib.sdb_gather_candidates.argtypes = [P, P, c_int, c_int, c_int, POINTER(c_int), POINTER(c_int), P, P, P]
    lib.sdb_conv3x3_2d.argtypes = [P, P, c_int, c_int, c_int, c_int, c_int, P, P, c_int, c_int, P, P]
    lib.sdb_maxpool2x2_2d.argtypes = [P, c_int, c_int, c_int, c_int, P, P]
    lib.sdb_conv3_nd.argtypes = [P, P] + [c_int] * 9 + [P, P, c_int, c_int, c_int, P, P]
    lib.sdb_maxpool_nd.argtypes = [P] + [c_int] * 8 + [P, P]
    lib.sdb_conv_generic_nd.argtypes = [P] + [c_int] * 5 + [P, P] + [c_int] * 8 + [P, P]
    lib.sdb_conv_generic_nd.restype = c_int
    lib.sdb_add_act.argtypes = [P, P, c_longlong, c_int, P, P]
    lib.sdb_add_act.restype = c_int
    lib.sdb_class_head.argtypes = [P, c_longlong, c_int, P, P, c_int, P, P]
    lib.sdb_class_head.restype = c_int
    lib.sdb_merge_split.argtypes = [P, P, c_longlong, P, P]
    lib.sdb_merge_split.restype = c_int
    lib.sdb_conv_any_nd.argtypes = [P, P] + [c_int] * 9 + [P, P] + [c_int] * 8 + [P, P]
    lib.sdb_conv_any_nd.restype = c_int
    lib.sdb_heads_any.argtypes = [P, c_longlong, c_int, P, P, P, P, c_int, P, P, P]
    lib.sdb_heads_any.restype = c_int
    lib.sdb_maxpool_any_nd.argtypes = [P] + [c_int] * 8 + [P, P]
    lib.sdb_maxpool_any_nd.restype = c_int
    lib.sdb_add_act_any.argtypes = [P, P, c_longlong, c_int, P, P]
    lib.sdb_add_act_any.restype = c_int
    lib.sdb_conv_wgrad_workspace.argtypes = [c_longlong, c_int, c_int, c_int]
    lib.sdb_conv_wgrad_workspace.restype = c_longlong
    lib.sdb_conv_wgrad_nd.argtypes = [P, P] + [c_int] * 11 + [P, c_int, c_int, P, c_longlong, P, P, P]
    lib.sdb_conv_wgrad_nd.restype = c_int
    lib.sdb_conv_wgrad_tf32_nd.argtypes = [P, P] + [c_int] * 11 + [P, c_int, c_int, P, c_longlong, P, P, P]
    lib.sdb_conv_wgrad_tf32_nd.restype = c_int
    lib.sdb_conv_dgrad_tf32_nd.argtypes = [P] + [c_int] * 5 + [P] + [c_int] * 3 + [P, P]
    lib.sdb_conv_dgrad_tf32_nd.restype = c_int
    lib.sdb_cast_bf16.argtypes = [P, c_longlong, P, P]
    lib.sdb_cast_bf16.restype = c_int
    lib.sdb_weights_bf16.argtypes = [P] + [c_int] * 5 + [P, P]
    lib.sdb_weights_bf16.restype = c_int
    lib.sdb_conv_bf16_nd.argtypes = [P, P] + [c_int] * 12 + [P, P, c_int, c_int, c_int, P, P]
    lib.sdb_conv_bf16_nd.restype = c_int
    lib.sdb_gemm_bf16_f32in.argtypes = [P, c_longlong, c_int, P, c_int, c_int, P, P]
    lib.sdb_gemm_bf16_f32in.restype = c_int
    lib.sdb_heads_bf16.argtypes = [P, c_longlong, c_int, P, P, P, c_int, P, P, P]
    lib.sdb_heads_bf16.restype = c_int
    lib.sdb_class_head_bf16.argtypes = [P, c_longlong, c_int, P, P, c_int, P, P, P]
    lib.sdb_class_head_bf16.restype = c_int
    lib.sdb_conv_wgrad_bf16_nd.argtypes = [P, P] + [c_int] * 11 + [P, c_int, c_int, c_int, P, c_longlong, P, P, P]
    lib.sdb_conv_wgrad_bf16_nd.restype = c_int
    lib.sdb_maxpool_bf16_nd.argtypes = [P] + [c_int] * 8 + [P, P]
    lib.sdb_maxpool_bf16_nd.restype = c_int
    lib.sdb_maxpool_backward_bf16_nd.argtypes = [P, P] + [c_int] * 9 + [P, P]
    lib.sdb_maxpool_backward_bf16_nd.restype = c_int
    lib.sdb_relu_backward_bf16.argtypes = [P, P, c_longlong, P]
    lib.sdb_relu_backward_bf16.restype = c_int
    lib.sdb_decoder_split_bf16.argtypes = [P] + [c_int] * 9 + [P, P, P]
    lib.sdb_decoder_split_bf16.restype = c_int
    lib.sdb_add_bf16.argtypes = [P, P, c_longlong, P, P]
    lib.sdb_add_bf16.restype = c_int
    lib.sdb_conv_wgrad_any_nd.argtypes = [P, P] + [c_int] * 12 + [P, c_int, c_int, P, c_longlong, P, P, P]
    lib.sdb_conv_wgrad_any_nd.restype = c_int
    lib.sdb_conv_dgrad_any_nd.argtypes = [P] + [c_int] * 5 + [P] + [c_int] * 4 + [P, P]
    lib.sdb_conv_dgrad_any_nd.restype = c_int
    lib.sdb_act_any.argtypes = [P, c_longlong, c_int, P, P]
    lib.sdb_act_any.restype = c_int
    lib.sdb_act_backward.argtypes = [P, P, c_longlong, c_int, P]
    lib.sdb_act_backward.restype = c_int
    lib.sdb_conv_flip_weights.argtypes = [P, c_int, c_int, c_int, P, P]
    lib.sdb_conv_flip_weights.restype = c_int
    lib.sdb_decoder_split.argtypes = [P] + [c_int] * 9 + [P, P, P]
    lib.sdb_decoder_split.restype = c_int
    lib.sdb_relu_backward.argtypes = [P, P, c_longlong, P]
    lib.sdb_relu_backward.restype = c_int
    lib.sdb_maxpool_backward_nd.argtypes = [P, P] + [c_int] * 9 + [P, P]
    lib.sdb_maxpool_backward_nd.restype = c_int
    lib.sdb_stardist_loss_workspace.argtypes = [c_longlong]
    lib.sdb_stardist_loss_workspace.restype = c_longlong
    lib.sdb_stardist_loss.argtypes = [P, P, P, P, c_longlong, c_int, c_int, c_float, c_float, c_float, P, P, P, P, P, P]
    lib.sdb_stardist_loss.restype = c_int
    lib.sdb_heads_backward.argtypes = [P, P, c_longlong, c_int, P, P, c_int, c_int, P, P]
    lib.sdb_heads_backward.restype = c_int
    lib.sdb_stardist_class_loss_workspace.argtypes = [c_longlong]
    lib.sdb_stardist_class_loss_workspace.restype = c_longlong
    lib.sdb_stardist_class_loss.argtypes = [P, P, c_longlong, c_int, P, c_float, P, P, P, P, P]
    lib.sdb_stardist_class_loss.restype = c_int
    lib.sdb_class_head_backward.argtypes = [P, P, c_longlong, c_int, P, c_int, c_int, c_int, P, P]
    lib.sdb_class_head_backward.restype = c_int
    lib.sdb_adam_step.argtypes = [P, P, P, P, c_longlong, c_float, c_float, c_float, c_float, P, P, P]
    lib.sdb_adam_step.restype = c_int
    lib.sdb_heads_2d.argtypes = [P, c_longlong, c_int, P, P, P, P, c_int, P, P, P]
    lib.sdb_conv3x3_tc.argtypes = [P, P, c_int, P, P, c_int, c_int, c_int, c_int, P, P, c_float, P, c_int, c_int, c_int, P, P, P]
    lib.sdb_heads_tc.argtypes = [P, P, c_int, c_int, c_int, c_int, P, P, c_float, P, c_int, c_int, P, P, P]
    lib.sdb_conv3x3_heads_tc.argtypes = [P, P, c_int, P, P, c_int, c_int, c_int, c_int, P, P, c_float, P, c_int, P, P, c_int, P, P, P]
    lib.sdb_conv3x3_heads_tc.restype = c_int
    lib.sdb_conv3x3x3_tc.argtypes = [P, P, c_int, P, P, c_int, c_int, c_int, c_int, P, P, c_float, P, c_int, c_int, c_int, P, P, P]
    lib.sdb_conv3x3x3_tc.restype = c_int
    lib.sdb_split_weights_3d.argtypes = [P, c_int, c_int, c_float, P, P, P]
    lib.sdb_split_weights_3d.restype = c_int
    lib.sdb_maxpool3d_split.argtypes = [P, P] + [c_int] * 7 + [P, P, P]
    lib.sdb_maxpool3d_split.restype = c_int
    lib.sdb_split_f32.argtypes = [P, c_longlong, P, P, P]
    lib.sdb_split_f32.restype = c_int
    lib.sdb_tc_error_check.argtypes = [P]
    lib.sdb_tc_set_variant.argtypes = [c_int]
    lib.sdb_tc_set_variant.restype = c_int
    lib.sdb_tc_set_split_acc.argtypes = [c_int]
    lib.sdb_tc_set_split_acc.restype = c_int
    lib.sdb_split_weights.argtypes = [P, c_int, c_int, c_float, P, P, P]
    lib.sdb_stem_split.argtypes = [P, c_int, c_int, c_int, c_int, P, P, c_int, c_int, P, P, P]
    lib.sdb_maxpool_split.argtypes = [P, P, c_int, c_int, c_int, c_int, P, P, P]
    lib.sdb_heads_split.argtypes = [P, P, c_longlong, c_int, P, P, P, P, c_int, P, P, P]
    lib.sdb_polyhedron_to_label.argtypes = [P, P, P, P, c_int, c_int, c_int, P, c_int, c_int, c_int, c_int, c_int, c_int, P, P]
    lib.sdb_nms3d_set_variant.argtypes = [c_int]
    lib.sdb_nms3d_set_variant.restype = c_int
    lib.sdb_relabel_sequential.argtypes = [P, c_longlong, c_int, c_int, P, POINTER(c_int), P]
    lib.sdb_relabel_sequential.restype = c_int
    lib.sdb_label_overlap.argtypes = [P, P, c_longlong, P, P, c_longlong, POINTER(c_longlong), P]
    lib.sdb_label_overlap.restype = c_int
    lib.sdb_stack_labels.argtypes = [P, c_longlong, c_longlong, P, P, c_longlong, POINTER(c_longlong), P]
    lib.sdb_stack_labels.restype = c_int
    lib.sdb_stack_overlap.argtypes = [P, c_longlong, c_longlong, c_longlong, P, P, c_int, P, P, c_longlong, POINTER(c_longlong), P]
    lib.sdb_stack_overlap.restype = c_int
    lib.sdb_stack_group_remap.argtypes = [P, c_longlong, c_longlong, P, P, P, P, P]
    lib.sdb_stack_group_remap.restype = c_int
    lib.sdb_star_dist_2d.argtypes = [P, c_int, c_int, c_int, c_int, c_int, c_int, P, P, c_longlong, P, P]
    lib.sdb_star_dist_2d.restype = c_int
    lib.sdb_star_dist_3d.argtypes = [P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P, P, c_longlong, P, P]
    lib.sdb_star_dist_3d.restype = c_int
    lib.sdb_star_dist_walk_bound.argtypes = [P, c_int, c_int, P, POINTER(c_longlong)]
    lib.sdb_star_dist_walk_bound.restype = c_int
    lib._LIB_star_dist_2d.argtypes = [P, c_int, c_int, c_int, c_int, c_int, P, P]
    lib._LIB_star_dist_2d.restype = None
    lib._LIB_star_dist_3d.argtypes = [P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P, P]
    lib._LIB_star_dist_3d.restype = None
    lib.sdb_region_stats.argtypes = [P, c_int, P, c_int, P, P, P, P, P]
    lib.sdb_region_stats.restype = c_int
    lib.sdb_edt_prob.argtypes = [P, c_int, P, c_int, P, c_int, P, P]
    lib.sdb_edt_prob.restype = c_int
    lib.sdb_star_dist_batch.argtypes = [P, c_int, c_int, P, P, c_int, P, c_int, P, P]
    lib.sdb_star_dist_batch.restype = c_int
    lib.sdb_edt_prob_batch.argtypes = [P, c_int, c_int, P, c_int, P, P, P, P, P, P, c_int, P]
    lib.sdb_edt_prob_batch.restype = c_int
    lib.sdb_fg_valid_index.argtypes = [P, c_int, P, P, P, P, P, POINTER(c_longlong), P]
    lib.sdb_fg_valid_index.restype = c_int
    lib.sdb_sample_select.argtypes = [P, c_int, c_int, P, P, P]
    lib.sdb_sample_select.restype = c_int
    lib.sdb_train_gather.argtypes = [P, P, c_int, c_int, P, c_int, P, P, P, P, P, P, P, P, c_int, P]
    lib.sdb_train_gather.restype = c_int
    lib.sdb_class_map.argtypes = [P, c_int, c_int, P, P, P, P, c_int, P, P, P]
    lib.sdb_class_map.restype = c_int
    lib.sdb_mt_normal.argtypes = [P, c_int, c_int, c_double, c_longlong, P, P, POINTER(c_int), POINTER(c_int), POINTER(c_double), P]
    lib.sdb_mt_normal.restype = c_int
    lib.sdb_augment_batch.argtypes = [P, c_int, c_int, P, c_int, P, P, P, P, P, P, P, P, P, P, P]
    lib.sdb_augment_batch.restype = c_int
    lib.sdb_label_class_map.argtypes = [P, c_longlong, P, P, c_int, c_int, P, P]
    lib.sdb_label_class_map.restype = c_int
    lib.sdb_mask_compact_count.argtypes = [P, c_int, c_int, c_int, POINTER(c_longlong), POINTER(c_longlong), POINTER(c_longlong), P,
                                           POINTER(c_longlong), P]
    lib.sdb_mask_compact_count.restype = c_int
    lib.sdb_mask_compact_write.argtypes = [P, c_int, c_int, c_int, POINTER(c_longlong), POINTER(c_longlong), POINTER(c_longlong), P,
                                           c_longlong, P, P, P, P]
    lib.sdb_mask_compact_write.restype = c_int
    lib.sdb_gather_patches.argtypes = [P, c_int, c_int, POINTER(c_longlong), POINTER(c_longlong), P, c_longlong, P, P]
    lib.sdb_gather_patches.restype = c_int
    lib.sdb_dist_to_volume.argtypes = [P, c_int, c_int, c_int, c_int, P, P, c_int, P, P]
    lib.sdb_dist_to_volume.restype = c_int
    lib.sdb_dist_to_centroid.argtypes = [P, c_int, c_int, c_int, c_int, P, P, c_int, c_int, P, P]
    lib.sdb_dist_to_centroid.restype = c_int
    lib.sdb_fill_label_holes.argtypes = [P, c_int, P, c_int, c_int, P, P]
    lib.sdb_fill_label_holes.restype = c_int
    lib._LIB_edt_prob.argtypes = [P, c_int, P, P, P]
    lib._LIB_edt_prob.restype = None
    lib._LIB_fill_label_holes.argtypes = [P, c_int, P, c_int, P]
    lib._LIB_fill_label_holes.restype = None
    lib.sdb_nms3d.argtypes = [P, P, P, P, c_int, c_int, c_int, c_float, c_int, c_int, c_int, P, P]
    lib.sdb_unet_layer_count.argtypes = [P]
    lib.sdb_unet_layer_count.restype = c_int
    lib.sdb_unet_layer_name.argtypes = [P, c_int]
    lib.sdb_unet_layer_name.restype = c_char_p
    lib.sdb_unet_create.argtypes = [P, P, P]
    lib.sdb_unet_create.restype = c_void_p
    lib.sdb_unet_destroy.argtypes = [P]
    lib.sdb_unet_destroy.restype = None
    lib._LIB_unet_forward_2d.argtypes = [P, P, c_int, c_int, P, P, P]
    lib._LIB_unet_forward_2d.restype = c_int
    lib._LIB_unet_forward_3d.argtypes = [P, P, c_int, c_int, c_int, P, P, P]
    lib._LIB_unet_forward_3d.restype = c_int
    lib.sdb_count_above.argtypes = [P, c_longlong, c_float, POINTER(c_int), P]
    lib.sdb_count_above.restype = c_int
    lib.sdb_store_rows_above.argtypes = [P, P, c_longlong, c_int, c_float, c_longlong, c_int, c_int, P, P, P]
    lib.sdb_store_rows_above.restype = c_int
    lib.sdb_gather_candidates_slots.argtypes = [P, P, P, c_int, c_int, c_int, POINTER(c_int), POINTER(c_int), P, P, P]
    lib.sdb_gather_candidates_slots.restype = c_int
    lib.sdb_select_ranks.argtypes = [P, c_int, POINTER(c_int), POINTER(c_int), POINTER(c_longlong), c_int, POINTER(c_float), P]
    lib.sdb_select_ranks.restype = c_int
    lib.sdb_normalize_mi_ma.argtypes = [P, c_longlong, c_float, c_float, c_int, P]
    lib.sdb_normalize_mi_ma.restype = c_int
    lib.sdb_zoom_linear.argtypes = [P, c_int, POINTER(c_int), POINTER(c_int), P, c_int, c_double, c_double, P]
    lib.sdb_zoom_linear.restype = c_int
    lib.sdb_pad_reflect_end.argtypes = [P, c_int, POINTER(c_int), POINTER(c_int), c_int, P, P]
    lib.sdb_pad_reflect_end.restype = c_int
    lib.sdb_label_bbox.argtypes = [P, c_int, POINTER(c_int), c_int, P, P, P]
    lib.sdb_label_bbox.restype = c_int
    lib.sdb_label_remap.argtypes = [P, c_longlong, P, P]
    lib.sdb_label_remap.restype = c_int
    lib.sdb_label_write.argtypes = [P, c_int, POINTER(c_int), c_int, P, POINTER(c_int), POINTER(c_int), P]
    lib.sdb_label_write.restype = c_int
    for name in ("_LIB_non_maximum_suppression_2d", "_LIB_polygons_to_label_2d", "sdb_nms2d",
                 "sdb_polygons_to_label_2d", "sdb_dist_to_coord_2d", "sdb_threshold_sort",
                 "sdb_gather_candidates", "sdb_conv3x3_2d", "sdb_maxpool2x2_2d", "sdb_heads_2d",
                 "sdb_device_info", "sdb_conv3x3_tc", "sdb_heads_tc", "sdb_tc_error_check", "sdb_split_weights", "sdb_stem_split",
                 "sdb_maxpool_split", "sdb_heads_split", "sdb_polyhedron_to_label", "sdb_nms3d", "sdb_conv3_nd", "sdb_maxpool_nd"):
        getattr(lib, name).restype = c_int
    # optional (added as the build widens)
    for name, argtypes in _OPTIONAL.items():
        if hasattr(lib, name):
            f = getattr(lib, name); f.argtypes = argtypes[0]; f.restype = argtypes[1]

_OPTIONAL = {}

def register_optional(name, argtypes, restype=c_int):
    _OPTIONAL[name] = (argtypes, restype)
    if _lib is not None and hasattr(_lib, name):
        f = getattr(_lib, name); f.argtypes = argtypes; f.restype = restype

def load():
    """Load the shared library (once). Raises StarDistB200Error when it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise StarDistB200Error(
                "libstardist_b200.so not found at %s -- build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback)" % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        _declare(lib)
        _lib = lib
    return _lib

def check(rc):
    if rc != 0:
        raise StarDistB200Error(load().sdb_last_error().decode("utf-8", "replace"))

def profile_enable(on=True):
    load().sdb_profile_enable(1 if on else 0)


def profile_get(name):
    ms, n, u = c_double(0), c_longlong(0), c_double(0)
    load().sdb_profile_get(name.encode(), ctypes.byref(ms), ctypes.byref(n), ctypes.byref(u))
    return dict(ms=ms.value, launches=n.value, units=u.value)


def launch_count(reset=False):
    return int(load().sdb_launch_count(1 if reset else 0))

def require_cuda():
    import torch
    if not torch.cuda.is_available():
        raise StarDistB200Error("stardist_b200 needs a CUDA device (sm_90a); none is visible and there is no CPU fallback")
    return load()

def ptr(t):
    """device/host pointer of a torch tensor or numpy array as c_void_p (None -> NULL)"""
    if t is None:
        return c_void_p(0)
    if hasattr(t, "data_ptr"):
        return c_void_p(t.data_ptr())
    return c_void_p(t.ctypes.data)

def stream_ptr(stream=None):
    import torch
    s = torch.cuda.current_stream() if stream is None else stream
    return c_void_p(s.cuda_stream)

def iarr(vals):
    return (c_int * len(vals))(*[int(v) for v in vals])


def larr(vals):
    return (c_longlong * len(vals))(*[int(v) for v in vals])


def nms2d_set_filter(mode):
    """0 = exact sweep on every pair, 1 = pre-filter + exact sweep (default), 2 = verify (both, count mismatches)."""
    check(load().sdb_nms2d_set_filter(int(mode)))


def nms2d_filter_stats(reset=False):
    out = (ctypes.c_ulonglong * 4)()
    load().sdb_nms2d_filter_stats(out, 1 if reset else 0)
    return dict(pairs=int(out[0]), exact=int(out[1]), mismatches=int(out[2]), calls=int(out[3]))


class UNetConfigC(ctypes.Structure):
    """sdb_unet_config of include/stardist_b200.h"""
    _fields_ = [(n, c_int) for n in ("ndim", "n_channel_in", "n_rays", "unet_n_depth", "unet_n_filter_base", "unet_n_conv_per_depth",
                                     "net_conv_after_unet")] + [("grid", c_int * 3)]


def c_unet_create(config, weights):
    """network object of the C boundary (_LIB_unet_forward_2d/3d) from a Config2D/3D and a weights dict; returns
    (handle, config struct).  The kernels are handed over in the order the library names the layers.
    sdb_unet_config has no fields for activations, batch norm, kernel size or pooling: the C executor always runs ReLU,
    3^d kernels and 2^d pooling without batch norm, so any other config is refused here rather than run as a different net."""
    import numpy as np
    unsupported = [(k, getattr(config, k)) for k in ("unet_activation", "unet_last_activation") if getattr(config, k) != 'relu']
    if config.unet_batch_norm:
        unsupported.append(("unet_batch_norm", config.unet_batch_norm))
    if any(int(k) != 3 for k in config.unet_kernel_size):
        unsupported.append(("unet_kernel_size", tuple(config.unet_kernel_size)))
    if any(int(p) != 2 for p in config.unet_pool):
        unsupported.append(("unet_pool", tuple(config.unet_pool)))
    if unsupported:
        raise StarDistB200Error("the C executor runs ReLU, 3^d kernels, pool 2 and no batch norm only; unsupported: %s"
                                % ", ".join("%s=%r" % kv for kv in unsupported))
    lib = require_cuda()
    g = tuple(config.grid) + (1,) * (3 - len(config.grid))
    cfg = UNetConfigC(config.n_dim, config.n_channel_in, config.n_rays, config.unet_n_depth, config.unet_n_filter_base,
                      config.unet_n_conv_per_depth, config.net_conv_after_unet, (c_int * 3)(*g))
    n = lib.sdb_unet_layer_count(ctypes.byref(cfg))
    names = [lib.sdb_unet_layer_name(ctypes.byref(cfg), i).decode() for i in range(n)]
    ks = [np.ascontiguousarray(weights[nm][0], np.float32) for nm in names]
    bs = [np.ascontiguousarray(weights[nm][1], np.float32) for nm in names]
    kp = (c_void_p * n)(*[k.ctypes.data for k in ks]); bp = (c_void_p * n)(*[b.ctypes.data for b in bs])
    h = lib.sdb_unet_create(ctypes.byref(cfg), kp, bp)
    if not h:
        raise StarDistB200Error(lib.sdb_last_error().decode("utf-8", "replace"))
    return c_void_p(h), cfg
