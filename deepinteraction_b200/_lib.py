"""ctypes binding of libdi_b200.so (the C-ABI declared in include/di_b200.h).

There is no fallback: if the library is missing or a call fails, a RuntimeError is raised.
"""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, 'libdi_b200.so')

_p = ctypes.c_void_p
_i = ctypes.c_int
_ll = ctypes.c_longlong
_f = ctypes.c_float
_fp = ctypes.POINTER(ctypes.c_float)

# name -> argument ctypes (all functions return int; see include/di_b200.h)
SIGNATURES = {
    'di_version': [],
    'di_built_arch': [],
    # gemm.cu
    'di_linear_f32': [_p, _i, _i, _p, _i, _i, _p, _i, _i, _p, _p, _p, _i, _i, _p, _i, _i, _i, _i, _i, _ll, _p],
    'di_conv3x3_f32': [_p, _i, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _p],
    'di_linear_tc_f32': [_p, _i, _i, _p, _i, _i, _p, _i, _i, _p, _p, _p, _p, _i, _i, _p, _i, _i, _i, _i, _p],
    'di_linear_tcb_f32': [_p, _i, _i, _p, _i, _i, _p, _i, _i, _p, _p, _p, _p, _i, _i, _p, _i, _i, _i, _i, _p],
    'di_linear_tcb_split_f32': [_p, _i, _i, _p, _i, _i, _p, _i, _i, _p, _p, _p, _p, _i, _i, _p, _i, _i, _i, _i, _i, _i, _p],
    'di_attn_planes_f32': [_p, _i, _p, _i, _p, _i, _p, _p, _ll, _p],
    'di_xattn_tc_splits': [_i, _i],
    'di_xattn_tc_f32': [_p, _p, _p, _p, _p, _i, _i, _i, _i, _p],
    'di_xattn_tc_lse_f32': [_p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _p],
    'di_xattn_bwd_workspace': [_i, _i, _i],
    'di_xattn_bwd_f32': [_p, _p, _p, _p, _p, _i, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _p],
    'di_conv3x3_tc_f32': [_p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    'di_conv3x3_tcb_f32': [_p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    'di_conv3x3_tc_nchw_f32': [_p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    'di_conv3x3_tcb_nchw_f32': [_p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    'di_tc_set_debug': [_i],
    'di_tc_set_mode': [_i],
    'di_tc_set_sm_limit': [_i],
    'di_tc_debug_read': [ctypes.POINTER(ctypes.c_longlong)],
    # lcab.cu
    'di_lcab_window_f32': [_p, _i, _p, _i, _p, _i, _p, _i, _i, _i, _i, _i, _i, _p],
    'di_lcab_window_pre_f32': [_p, _i, _p, _i, _p, _i, _p, _i, _i, _i, _i, _i, _p],
    'di_lcab_window_tc_f32': [_p, _i, _p, _i, _p, _i, _p, _i, _i, _i, _i, _i, _p],
    'di_lcab_proj_f32': [_p, _i, _p, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i, _p],
    'di_lcab_proj_grid': [_i, ctypes.POINTER(_i), ctypes.POINTER(_i), ctypes.POINTER(_i)],
    'di_lcab_forward_f32': [_p, _i, _p, _i, _p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _p],
    'di_set_window_ffma': [_i],
    'di_locatt_cc2k_f32': [_p, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    'di_locatt_ck2c_ori_f32': [_p, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    'di_locatt_ck2c_loc_f32': [_p, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    # geometry.cu
    'di_gather_rows_f32': [_p, _p, _p, _i, _i, _i, _i, _p, _p],
    'di_scatter_rows_f32': [_p, _p, _p, _p, _i, _i, _i, _i, _p, _p],
    'di_i2p_attend_f32': [_p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p, _p],
    'di_depth_scatter': [_p, _i, _i, _p, _p, _i, _i, _i, _i, _i, _p, _p],
    'di_depth_complete': [_p, _p, _p, _p, _i, _i, _i, _p],
    'di_lift_grid': [_p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _fp, _p],
    'di_bev_sample_f32': [_p, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    # pillar.cu
    'di_pillarize_f32': [ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_int), _p, _i, _i, _i, _i, _i, _i, _fp, _p, _p, _p, _p, _p, _i, _p],
    # deform.cu
    'di_msdeform_f32': [_p, _p, _p, _i, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, ctypes.POINTER(ctypes.c_int), _p],
    'di_axpy_f32': [_p, _p, _p, _p, _ll, _p],
    'di_polar_grid_f32': [_p, _p, _i, _i, _i, _i, _f, _f, _f, _fp, _i, _i, _p],
    'di_add_rows_mod_f32': [_p, _p, _p, _ll, _i, _ll, _p],
    'di_seq_attn_f32': [_p, _i, _p, _i, _p, _i, _p, _i, _i, _i, _i, _i, _i, _i, _p],
    'di_polar_gather_f32': [_p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _fp, _f, _f, _p],
    'di_scatter_rows_add_f32': [_p, _p, _p, _p, _i, _i, _i, _i, _p, _p],
    'di_msdeform_bwd_f32': [_p, _p, _p, _i, _p, _i, _p, _i, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i,
                            ctypes.POINTER(ctypes.c_int), _p],
    'di_seq_attn_bwd_f32': [_p, _i, _p, _i, _p, _i, _p, _i, _p, _i, _p, _i, _p, _i, _p, _i, _i, _i, _i, _i, _i, _i, _p],
    'di_polar_gather_bwd_f32': [_p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _fp, _f, _f, _p],
    'di_axpy_bwd_workspace': [],
    'di_axpy_bwd_f32': [_p, _p, _p, _p, _p, _p, _ll, _p],
    # decoder.cu
    'di_heatmap_nms_f32': [_p, _p, _i, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    'di_topk_f32': [_p, _p, _i, _i, _i, _p, _i, _p],
    'di_query_init_f32': [_p, _p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    'di_query_init_bwd_f32': [_p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _p],
    'di_mha_small_f32': [_p, _i, _p, _i, _p, _i, _p, _i, _p, _p, _i, _i, _i, _i, _p],
    'di_mha_small_bwd_f32': [_p, _i, _p, _i, _p, _i, _p, _i, _p, _p, _p, _i, _p, _p, _p, _i, _i, _i, _i, _p],
    'di_cross_attn_f32': [_p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    'di_rows_finish_f32': [_p, _i, _ll, _i, _p, _p, _i, _p, _p, _p, _i, _p, _i, _i, _i, _f, _p],
    'di_rows_mlp_f32': [_p, _i, _i, _p, _i, _i, _p, _p, _i, _i, _p, _p, _i, _p, _i, _p, _p, _f, _i, _p, _p, _i, _i, _p],
    'di_pred_finish_f32': [_p, _p, _p, _p, _i, _i, _p],
    'di_i2p_attend_bwd_f32': [_p, _p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p, _p],
    'di_i2p_attend_dropout_f32': [_p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p, _f, ctypes.c_uint, _p],
    'di_i2p_attend_bwd_dropout_f32': [_p, _p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p, _f, ctypes.c_uint, _p],
    'di_i2p_dropout_mask_f32': [_p, _i, _i, _f, ctypes.c_uint, _p],
    'di_bev_sample_bwd_f32': [_p, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    'di_gather_rows_masked_f32': [_p, _p, _p, _p, _i, _i, _i, _i, _p],
    'di_win_dot_f32': [_p, _i, _p, _i, _p, _i, _i, _i, _i, _i, _p],
    'di_win_gather_f32': [_p, _p, _i, _p, _i, _i, _i, _i, _i, _i, _p],
    'di_win_scatter_f32': [_p, _p, _i, _p, _i, _i, _i, _i, _i, _i, _p],
    'di_win_softmax_f32': [_p, _p, _ll, _i, _f, _p],
    'di_win_softmax_bwd_f32': [_p, _p, _p, _ll, _i, _f, _p],
    'di_relu_bwd_f32': [_p, _p, _p, _ll, _p],
    'di_col_sum_f32': [_p, _i, _ll, _i, _p, _p, _p],
    'di_ln_bwd_f32': [_p, _i, _p, _i, _p, _p, _i, _p, _p, _p, _i, _i, _f, _p],
    'di_shift_map_f32': [_p, _p, _i, _i, _i, _i, _i, _i, _p],
    # bn_train.cu
    'di_bn_stats_f32': [_p, _ll, _i, _p, _p, _p, _p, _p, _f, _p],
    'di_bn_apply_f32': [_p, _ll, _i, _p, _p, _p, _p, _f, _i, _p, _p],
    'di_bn_bwd_f32': [_p, _p, _p, _ll, _i, _p, _p, _p, _f, _p, _p, _p, _p, _p],
    'di_match_cost_f32': [_p, _i, _p, _i, _p, _p, _p, _i, _i, _i, _p, _p, _p, _p],
    'di_heuristic_assign_f32': [_p, _i, _i, _p, _p, _i, _p, _f, _p, _p, _p, _p, _p],
    'di_hungarian_f32': [_p, _p, _p, _i, _i, _i, _i, _p, _p, _p],
    'di_loss_targets_f32': [_p, _p, _p, _p, _i, _p, _i, _i, _i, _i, _i, _i, _i, _f, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p],
    'di_gaussian_heatmap_f32': [_p, _i, _p, _p, _i, _i, _i, _i, _i, _p, _p, _p],
    'di_mmpi_losses_f32': [_p, _p, _ll, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _p, _p, _p,
                           _p, _p, _p, _p],
    'di_mmpi_losses_bwd_f32': [_p, _p, _ll, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _p, _p, _p, _p,
                               _p, _p, _p, _p, _p],
    'di_pred_finish_pp_f32': [_p, _p, _p, _p, _p, _p, _i, _i, _i, _p],
    'di_rcnn_leaders': [_p, _p, _p, _i, _i, _i, _p],
    'di_mha_small_rows_f32': [_p, _i, _p, _i, _p, _i, _p, _i, _p, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    'di_take_rows_f32': [_p, _i, _p, _p, _i, _i, _p],
    'di_branch_mix_f32': [_p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _p],
    'di_mha_small_rows_bwd_f32': [_p, _i, _p, _i, _p, _i, _p, _i, _p, _i, _p, _p, _i, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i,
                                  _p],
    'di_rows_scatter_add_f32': [_p, _i, _p, _p, _i, _i, _i, _p],
    'di_branch_mix_bwd_f32': [_p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _p],
    'di_pred_finish_pp_bwd_f32': [_p, _p, _p, _p, _i, _i, _i, _p],
    'di_rcnn_rois_f32': [_p, _i, _p, _p, _p, _p, _p, _i, _i, _i, _i, _fp, _p],
    'di_roi_align_f32': [_p, _p, _p, _i, _i, _i, _i, _f, _p],
    'di_dynconv_f32': [_p, _p, _p, _p, _p, _p, _p, _i, _f, _p],
    'di_roi_align_bwd_f32': [_p, _p, _p, _i, _i, _i, _i, _i, _f, _p],
    'di_dynconv_bwd_f32': [_p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i, _f, _p],
    'di_gelu_bwd_f32': [_p, _p, _p, _ll, _p],
    'di_nchw_to_nhwc_f32': [_p, _p, _i, _i, _i, _p],
    'di_nhwc_to_nchw_f32': [_p, _p, _i, _i, _i, _p],
    'di_bbox_decode_f32': [_p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _f, _f, _f, _f, _fp, _f, _i, _p, _p, _p, _p, _p],
    'di_bbox_encode_f32': [_p, _i, _p, _i, _i, _f, _f, _f, _f, _p],
    'di_circle_nms_f32': [_p, _i, _p, _p, _p, _i, _i, ctypes.c_uint, _f, _i, _p],
}

_lib = None


def lib():
    """Load the library once; raise loudly when it is absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f'{LIB_PATH} not found: build it with `python -m deepinteraction_b200.build` '
                '(nvcc, sm_90a).  There is no CPU/PyTorch fallback for the MMRI/MMPI kernels.')
        L = ctypes.CDLL(LIB_PATH)
        L.di_last_error.restype = ctypes.c_char_p
        L.di_last_error.argtypes = []
        for name, args in SIGNATURES.items():
            fn = getattr(L, name)          # AttributeError if a declared symbol is missing
            fn.restype = ctypes.c_int
            fn.argtypes = args
        _lib = L
    return _lib


def last_error():
    return lib().di_last_error().decode()


def check(rc, what=''):
    if rc < 0:
        raise RuntimeError(f'libdi_b200 {what}: {last_error()} (status {rc})')
    return rc
