"""ctypes binding of libvirconv_sm90.so (include/virconv_b200.h).

The library is the product: there is no CPU / PyTorch fallback.  If the shared object is missing the
first op that needs it raises — loudly — instead of computing anything elsewhere.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_int32, c_size_t, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('VIRCONV_LIB') or os.path.join(_HERE, 'lib', 'libvirconv_sm90.so')

_P = c_void_p
_I = c_int
_F = c_float
_Z = c_size_t
_HOST = ctypes.POINTER(c_int32)
_HOSTF = ctypes.POINTER(c_float)
_HOSTD = ctypes.POINTER(c_double)
_HOSTP = ctypes.POINTER(c_void_p)        # host array of device pointers
_D = c_double
# vc_bn_exchange_fn: (user, layer, direction, slot, n doubles) -> 0 on success
EXCHANGE_FN = ctypes.CFUNCTYPE(c_int, c_void_p, c_int, c_int, c_void_p, c_int)

# name -> (restype, argtypes).  Every symbol include/virconv_b200.h declares.
SIGNATURES = {
    'vc_version': (_I, []),
    'vc_last_error': (c_char_p, []),
    'vc_launch_count': (ctypes.c_longlong, []),
    'vc_set_bn_fused': (_I, [_I]),
    'vc_set_conv_bn_fused': (_I, [_I]),
    'vc_set_tc_variant': (_I, [_I]),
    'vc_conv_tc2_config': (_I, [_I]),
    'vc_conv_tc2_plan': (_I, [_I, _I, _I, _I, _HOST]),
    'vc_conv_wgrad_tc3_config': (_I, [_I, _I]),
    'vc_wgrad_launch_geometry': (_I, [_I, _I, _I, _I, _I, _HOST]),
    'vc_subm_rulebook_ws_bytes': (_Z, [_I]),
    'vc_subm_rulebook': (_I, [_P, _I, _I, _I, _HOST, _HOST, _HOST, _P, _P, _P, _Z, _P]),
    'vc_conv_rulebook_ws_bytes': (_Z, [_I, _I, _HOST]),
    'vc_conv_out_shape': (_I, [_I, _HOST, _HOST, _HOST, _HOST, _HOST, _HOST]),
    'vc_conv_rulebook_count': (_I, [_P, _I, _I, _I, _HOST, _HOST, _HOST, _HOST, _HOST, _P, _P, _Z, _P]),
    'vc_conv_rulebook_fill': (_I, [_P, _I, _I, _I, _HOST, _HOST, _HOST, _HOST, _HOST, _I, _P, _P, _P, _P, _P, _Z, _P]),
    'vc_pairs_from_nbr': (_I, [_P, _I, _I, _P, _P, _P]),
    'vc_conv_ws_bytes': (_Z, [_I, _I, _I]),
    'vc_conv_fwd_f32': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _Z, _P]),
    'vc_conv_dgrad_f32': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _Z, _P]),
    'vc_conv_dgrad_scatter_f32': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _Z, _P]),
    'vc_conv_wgrad_ws_bytes': (_Z, [_I, _I, _I, _I]),
    'vc_conv_wgrad_f32': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _Z, _P]),
    'vc_cast_f32_bf16': (_I, [_P, _P, ctypes.c_longlong, _P]),
    'vc_conv_tc_ws_bytes': (_Z, [_I, _I, _I]),
    'vc_conv_fwd_tc': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _Z, _P, _P]),
    'vc_conv_fwd_tc_ld': (_I, [_P, _I, _P, _P, _P, _I, _I, _I, _I, _P, _P, _Z, _P, _P]),
    'vc_conv_dgrad_tc': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _Z, _P, _P]),
    'vc_conv_dgrad_scatter_tc': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _Z, _P, _P]),
    'vc_conv_wgrad_tc_ws_bytes': (_Z, [_I, _I, _I, _I]),
    'vc_conv_wgrad_tc': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _Z, _P, _P]),
    'vc_conv_fwd_det_ws_bytes': (_Z, [_I, _I, _I, _I]),
    'vc_conv_fwd_det': (_I, [_I, _P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _Z, _P, _P]),
    'vc_conv_bn_relu_tc_ws_bytes': (_Z, [_I, _I, _I, _I]),
    'vc_conv_bn_relu_tc': (_I, [_P, _P, _P, _P, _I, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _F, _F, _I, _P, _I, _P, _I, _P, _P, _Z,
                                _P, _P]),
    'vc_conv_wgrad_tc_det_ws_bytes': (_Z, [_I, _I, _I, _I]),
    'vc_conv_wgrad_tc_det': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _Z, _P, _P]),
    'vc_conv_wgrad_tc_det_ld': (_I, [_P, _I, _P, _P, _P, _I, _I, _I, _I, _P, _Z, _P, _P]),
    'vc_bn_bwd_det_ws_bytes': (_Z, [_I, _I]),
    'vc_bn_relu_bwd_det_f32': (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _Z, _P]),
    'vc_subm_rulebook_rep': (_I, [_P, _I, _I, _I, _HOST, _HOST, _HOST, _P, _P, _P, _P, _Z, _P]),
    'vc_conv_dgrad_gather2d_ws_bytes': (_Z, [_I, _I, _I, _I]),
    'vc_conv_dgrad_gather2d_f32': (_I, [_P, _P, _P, _P, _P, _I, _P, _I, _I, _I, _P, _Z, _P]),
    'vc_conv_dgrad_gather2d_tc': (_I, [_P, _P, _P, _P, _P, _I, _P, _I, _I, _I, _P, _Z, _P, _P]),
    'vc_bn_apply_relu_f32': (_I, [_P, _P, _I, _I, _P, _P, _P, _P, _P, _F, _F, _I, _P, _P, _P, _I, _P]),
    'vc_bn_relu_bwd_f32': (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _P]),
    'vc_index2uv': (_I, [_P, _I, _I, _P, _HOSTF, _I, _I, _I, _P, _P]),
    'vc_dense_f32': (_I, [_P, _P, _I, _I, _I, _I, _HOST, _P, _P]),
    'vc_dense_bwd_f32': (_I, [_P, _P, _I, _I, _I, _I, _HOST, _P, _P]),
    'vc_voxelize_ws_bytes': (_Z, [_I, _I, _I]),
    'vc_voxelize_mean': (_I, [_P, _I, _I, _I, _HOSTF, _HOSTF, _I, _I, _I, _P, _P, _P, _P, _P, _P, _Z, _P]),
    'vc_voxel2pinds': (_I, [_P, _I, _I, _I, _HOST, _P, _P]),
    'vc_voxel2pinds_rows': (_I, [_P, _I, _P, _I, _I, _HOST, _P, _P]),
    'vc_dense_rows_f32': (_I, [_P, _P, _I, _P, _I, _I, _I, _HOST, _P, _P]),
    'vc_dense_rows_bwd_f32': (_I, [_P, _P, _I, _P, _I, _I, _I, _HOST, _P, _P]),
    'vc_xbatch_pack': (_I, [_HOSTP, _HOSTP, _HOSTP, _HOST, _I, _I, _I, _I, _P, _P, _P, _P]),
    'vc_xbatch_split_ws_bytes': (_Z, [_I, _I]),
    'vc_xbatch_split': (_I, [_P, _P, _I, _P, _I, _I, _I, _HOSTP, _HOSTP, _HOSTP, _P, _Z, _P]),
    'vc_cat2_f32': (_I, [_P, _P, _P, _P, _I, _I, _I, _P]),
    'vc_masked_mean_ws_bytes': (_Z, []),
    'vc_masked_mean_f32': (_I, [_P, ctypes.c_longlong, _I, _P, _P, _P, _Z, _P]),
    'vc_masked_mean_bwd_f32': (_I, [_P, ctypes.c_longlong, _I, _P, _P, _P]),
    'vc_gather_rows': (_I, [_P, _P, _P, _I, _I, _P]),
    'vc_stvd_ws_bytes': (_Z, [_I]),
    'vc_stvd_partition': (_I, [_P, _I, _I, _I, ctypes.c_double, _P, _P, _Z, _P]),
    'vc_stvd_gather': (_I, [_P, _I, _I, _HOST, _I, _P, _P, _I, _P, _Z, _P]),
    'vc_stvd_input_ws_bytes': (_Z, [_I, _I]),
    'vc_stvd_input_front_end': (_I, [_P, _I, _P, _I, _I, _I, _D, _D, _HOSTF, _I, _I, _P, _I, _P, _P, _I, _P, _P, _I, _P, _P, _P,
                                     _P, _Z, _P]),
    'vc_stvd_layer_keep_ws_bytes': (_Z, [_I]),
    'vc_stvd_layer_keep': (_I, [_P, _P, _I, _I, _P, _D, _P, _P, _P, _P, _Z, _P]),
    'vc_voxel_query': (_I, [_I, _I, _I, _I, _I, _F, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P]),
    'vc_group_points': (_I, [_I, _I, _I, _I, _P, _P, _P, _P, _P, _P]),
    'vc_group_points_grad': (_I, [_I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P]),
    'vc_group_points_grad_det_ws_bytes': (_Z, [_I, _I, _I]),
    'vc_group_points_grad_det': (_I, [_I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _Z, _P]),
    'vc_voxel_pool_query': (_I, [_I, _I, _I, _I, _I, _F, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P]),
    'vc_voxel_pool_bn_fold': (_I, [_I, ctypes.c_longlong, _I, _P, _P, _P, _P, _P, _P, _P, ctypes.c_double, ctypes.c_double,
                                   _P, _P, _P, _P]),
    'vc_voxel_pool_bn_grad': (_I, [_I, ctypes.c_longlong, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    'vc_voxel_pool_bn_fold_sync': (_I, [_I, _I, _P, _P, _P, _P, _P, _P, _P, ctypes.c_double, ctypes.c_double, _P, _P, _P, _P]),
    'vc_voxel_pool_bn_grad_sync': (_I, [_I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    'vc_voxel_pool_fwd': (_I, [_I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    'vc_voxel_pool_bwd': (_I, [_I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    'vc_voxel_pool_det_config': (_I, [_I]),
    'vc_voxel_pool_query_det_ws_bytes': (_Z, [_I]),
    'vc_voxel_pool_query_det': (_I, [_I, _I, _I, _I, _I, _F, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _Z, _P]),
    'vc_voxel_pool_bwd_det_ws_bytes': (_Z, [_I, _I, _I, _I]),
    'vc_voxel_pool_bwd_det': (_I, [_I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _Z, _P]),
    'vc_boxes_overlap_bev': (_I, [_P, _I, _P, _I, _P, _P]),
    'vc_boxes_iou_bev': (_I, [_P, _I, _P, _I, _P, _P]),
    'vc_boxes_iou3d': (_I, [_P, _I, _P, _I, _P, _P]),
    'vc_boxes_iou_bev_host': (_I, [_P, _I, _P, _I, _P]),
    'vc_nms_ws_bytes': (_Z, [_I, _I]),
    'vc_nms_boxes': (_I, [_P, _I, _I, _I, _P, _F, _I, _I, _P, _P, _P, _Z, _P]),
    'vc_anchor_mask': (_I, [_P, _I, _I, _F, _F, _F, _I, _I, _P, _P, _P]),
    'vc_anchor_targets_ws_bytes': (_Z, [_I, _I, _I]),
    'vc_anchor_targets': (_I, [_P, _P, _I, _I, _HOSTF, _HOSTF, _P, _I, _I, _I, _HOST, _I, _P, _P, _P, _P, _P, _Z, _P]),
    'vc_roi_targets_ws_bytes': (_Z, [_I, _I, _I]),
    'vc_roi_targets': (_I, [_P, _P, _P, _I, _I, _I, _P, _I, _I, _I, _HOSTD, _HOSTD, _HOSTD, _D, _HOSTD, _HOSTD, _I, _I, _I,
                            _D, _P, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _Z, _P]),
    'vc_rpn_loss_ws_bytes': (_Z, [_I, _I]),
    'vc_rpn_loss': (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _D, _D, _D, _HOSTD, _D, _D, _D, _D, _P, _P, _P, _P, _P, _Z,
                         _P]),
    'vc_rcnn_loss_ws_bytes': (_Z, [_I]),
    'vc_rcnn_loss': (_I, [_P, _I, _D, _HOSTD, _D, _D, _D, _I, _P, _P, _Z, _P]),
    'vc_part_pool_fwd': (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _F, _F, _F, _P, _P]),
    'vc_part_pool_bwd_ws_bytes': (_Z, [_I, _I, _I]),
    'vc_part_pool_bwd': (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _F, _F, _F, _P, _P, _Z, _P]),
    'vc_roi_grid_points': (_I, [_P, _I, _I, _I, _I, _HOSTF, _HOSTF, _HOST, _I, _P, _P, _P]),
    'vc_anchor_decode': (_I, [_P, _P, _P, _I, _I, _I, _F, _F, _F, _P, _P]),
    'vc_anchor_decode_bwd': (_I, [_P, _P, _P, _I, _I, _I, _P, _P]),
    'vc_roi_decode': (_I, [_P, _P, _I, _I, _I, _P, _P]),
    'vc_roi_decode_bwd': (_I, [_P, _P, _P, _I, _I, _I, _P, _P]),
    'vc_box_xtrans': (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _P, _P]),
    'vc_optim_ws_bytes': (_Z, [_I]),
    'vc_optim_step': (_I, [_P, _I, _P, _I, _D, _HOSTP, _I, _P, _P, _P, _I, _P, _Z, _P]),
    'vc_exec_state_bytes': (_Z, []),
    'vc_exec_forward': (_I, [_P, _P, _I, _P, _P, _I, _P, _I, _P, _I, _HOST, _I, _P, _I, _I, _I, _P, _Z, _P, _P, _P, _Z, _P, _P, _I,
                             _P, _P, _P, _P]),
    'vc_exec_forward_seeded': (_I, [_P, _P, _I, _P, _P, _I, _P, _I, _P, _I, _HOST, _I, _P, _I, _I, _I, _P, _Z, _P, _P, _P, _Z, _P, _P,
                                    _I, _P, _P, _P, _P, _P]),
    'vc_exec_forward_sync': (_I, [_P, _P, _I, _P, _P, _I, _P, _I, _P, _I, _HOST, _I, _P, _I, _I, _I, _P, _Z, _P, _P, _P, _Z, _P, _P,
                                  _I, _P, _P, _P, _P, _P, _P, _P, EXCHANGE_FN, _P]),
    'vc_exec_backward': (_I, [_P, _P, _I, _P, _P, _I, _P, _P, _I, _P, _Z, _P, _P, _P, _P]),
    'vc_exec_backward_sync': (_I, [_P, _P, _I, _P, _P, _I, _P, _P, _I, _P, _Z, _P, _P, _P, _P, _P, _P, EXCHANGE_FN, _P]),
    'vc_exec_query': (_I, [_P, _I, _I, _P]),
    'vc_exec_timing': (_I, [_I]),
    'vc_exec_timing_read': (_I, [_P, _P, _I]),
    'vc_kitti_overlaps': (_I, [_P, _P, _P, _I, ctypes.c_longlong, _I, _P, _P]),
    'vc_kitti_rotate_iou': (_I, [_P, _P, _I, _I, _I, _P, _P]),
    'vc_kitti_eval_ws_bytes': (_Z, [_I, _I, _I, _I, _I]),
    'vc_kitti_eval': (_I, [_P, _P, _P, _P, _I, _I, _I, ctypes.c_longlong, _I, _HOST, _I, _I, _P, _P, _P, _Z, _P]),
    'vc_allreduce_peer_flag_words': (_I, [_I]),
    'vc_allreduce_peer_f32': (_I, [_P, _P, _I, _I, _P, ctypes.c_longlong, ctypes.c_longlong, ctypes.c_uint, _F, _P, _P]),
}

_lib = None


class VirConvLibraryError(RuntimeError):
    pass


def load():
    """Load the shared library (once).  Raises if it has not been built: no fallback exists."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise VirConvLibraryError(
            f'{LIB_PATH} is missing: build it with `python -m virconv_b200.build` '
            f'(or __graft_entry__.build()).  virconv_b200 has no CPU or PyTorch fallback.')
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    # BatchNorm + ReLU inside the tensor-core conv forward (one cooperative launch per layer); 0 for A/B runs
    lib.vc_set_conv_bn_fused(0 if os.environ.get('VIRCONV_CONV_BN_FUSED', '1') == '0' else 1)
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc != 0:
        msg = load().vc_last_error()
        raise VirConvLibraryError(f'{what} failed (rc={rc}): {msg.decode() if msg else ""}')


def host_i32(vals):
    return (c_int32 * len(vals))(*[int(v) for v in vals])


def host_f32(vals):
    return (c_float * len(vals))(*[float(v) for v in vals])


def host_ptrs(vals):
    return (c_void_p * len(vals))(*[int(v) for v in vals])


def host_f64(vals):
    return (c_double * len(vals))(*[float(v) for v in vals])
