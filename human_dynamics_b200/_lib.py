"""ctypes binding of libhd_b200.so (the C-ABI declared in include/hd_b200.h).

There is NO CPU fallback: if the shared library is missing this module raises at import,
and every op raises if it is handed a non-CUDA tensor.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libhd_b200.so')

HD_IMPL_SIMT, HD_IMPL_TC_3XTF32, HD_IMPL_TC_1XTF32, HD_IMPL_TC_3XF16 = 0, 1, 2, 3
HD_CONV_NO_TMA_EPILOGUE = 1
HD_CONV_INPUT_PLANES = 2
HD_PACK_FORWARD, HD_PACK_BACKWARD_DATA = 0, 1
IMPL_BY_NAME = {'simt': HD_IMPL_SIMT, 'tc3': HD_IMPL_TC_3XTF32, 'tc1': HD_IMPL_TC_1XTF32, 'tc3h': HD_IMPL_TC_3XF16}


class ConvDesc(C.Structure):
    """Mirror of hd_conv_desc (include/hd_b200.h)."""
    _fields_ = [
        ('in_', C.c_void_p), ('in_ld', C.c_longlong),
        ('n_img', C.c_int), ('H', C.c_int), ('W', C.c_int), ('Cin', C.c_int),
        ('Ho', C.c_int), ('Wo', C.c_int), ('KH', C.c_int), ('KW', C.c_int),
        ('stride', C.c_int), ('pad_t', C.c_int), ('pad_l', C.c_int),
        ('w_kn', C.c_void_p), ('w_nk_hi', C.c_void_p), ('w_nk_lo', C.c_void_p),
        ('Cout', C.c_int), ('K_pad', C.c_int),
        ('pre_scale', C.c_void_p), ('pre_shift', C.c_void_p), ('pre_img_stride', C.c_int), ('pre_relu', C.c_int),
        ('post_scale', C.c_void_p), ('post_shift', C.c_void_p), ('post_relu', C.c_int),
        ('res', C.c_void_p), ('res_ld', C.c_longlong), ('res_H', C.c_int), ('res_W', C.c_int), ('res_stride', C.c_int),
        ('out', C.c_void_p), ('out_ld', C.c_longlong),
        ('impl', C.c_int),
        ('tmap_hi', C.c_void_p), ('tmap_lo', C.c_void_p),
        ('in_hi', C.c_void_p), ('in_lo', C.c_void_p),
        ('out_hi', C.c_void_p), ('out_lo', C.c_void_p), ('out2_ld', C.c_longlong),
        ('post2_scale', C.c_void_p), ('post2_shift', C.c_void_p), ('post2_relu', C.c_int),
        ('tmap_res', C.c_void_p), ('tmap_out', C.c_void_p), ('tmap_out_hi', C.c_void_p), ('tmap_out_lo', C.c_void_p),
        ('flags', C.c_int),
        ('tmap_hi_n64', C.c_void_p), ('tmap_lo_n64', C.c_void_p),
        ('out_subsample', C.c_int),
    ]


WEIGHT_FN = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_char_p, C.POINTER(C.c_longlong))      # hd_weight_fn


class SmplConsts(C.Structure):
    """Mirror of hd_smpl_consts."""
    _fields_ = [
        ('num_verts', C.c_int), ('num_kps', C.c_int), ('lbs_nnz', C.c_int), ('kp_nnz_total', C.c_int),
        ('v_template', C.c_void_p), ('dirs', C.c_void_p), ('J_template', C.c_void_p), ('J_shapedirs', C.c_void_p),
        ('lbs_idx', C.c_void_p), ('lbs_w', C.c_void_p),
        ('kp_ptr', C.c_void_p), ('kp_vidx', C.c_void_p), ('kp_w', C.c_void_p),
        ('parents', C.c_int * 24),
    ]


class SmplGradConsts(C.Structure):
    """Mirror of hd_smpl_grad_consts."""
    _fields_ = [
        ('num_verts', C.c_int), ('num_kps', C.c_int), ('num_tiles', C.c_int), ('tile_verts', C.c_int),
        ('kpv_ptr', C.c_void_p), ('kpv_kidx', C.c_void_p), ('kpv_w', C.c_void_p),
        ('lbt_ptr', C.c_void_p), ('lbt_v', C.c_void_p), ('lbt_w', C.c_void_p),
    ]


SMPL_GRAD_TILE, SMPL_GRAD_CLD = 256, 224       # HD_SMPL_GRAD_TILE, HD_SMPL_GRAD_CLD


class RenderParams(C.Structure):
    """Mirror of hd_render_params."""
    _fields_ = [
        ('color', C.c_float * 3), ('light_dir', C.c_float * 3), ('ambient', C.c_float), ('directional', C.c_float),
        ('bg', C.c_float * 3), ('near_z', C.c_float), ('far_z', C.c_float), ('eye_z', C.c_float),
        ('rot', C.c_float * 9), ('use_rot', C.c_int),
    ]


HD_LOSS_KP_L1, HD_LOSS_MSE_ROWS = 0, 1
HD_LOSS_KP_CAMERA, HD_LOSS_KP_OPTCAM, HD_LOSS_KP_RAW = 0, 1, 2
HD_LOSS_MAX_TERMS, HD_LOSS_MAX_GRADS = 64, 16


class LossTerm(C.Structure):
    """Mirror of hd_loss_term."""
    _fields_ = [
        ('kind', C.c_int), ('proj', C.c_int), ('B', C.c_int), ('Tw', C.c_int), ('p_t0', C.c_int), ('q_t0', C.c_int),
        ('p_T', C.c_int), ('q_T', C.c_int), ('K', C.c_int), ('D', C.c_int),
        ('p', C.c_void_p), ('p_clip', C.c_longlong), ('p_frame', C.c_longlong),
        ('q', C.c_void_p), ('q_clip', C.c_longlong), ('q_frame', C.c_longlong),
        ('cam', C.c_void_p), ('cam_clip', C.c_longlong), ('cam_frame', C.c_longlong),
        ('w', C.c_void_p), ('cam_out', C.c_void_p), ('scale', C.c_float),
    ]


class LossGrad(C.Structure):
    """Mirror of hd_loss_grad."""
    _fields_ = [('src', C.c_void_p), ('grad', C.c_void_p), ('numel', C.c_longlong)]


HD_AUG_SRC_U8, HD_AUG_ROTATE, HD_AUG_FLIP = 1, 2, 4


class TubeAugArgs(C.Structure):
    """Mirror of hd_tube_aug_args."""
    _fields_ = [
        ('frames', C.c_void_p), ('F', C.c_int), ('H', C.c_int), ('W', C.c_int), ('flags', C.c_int),
        ('trans', C.c_void_p), ('scale', C.c_void_p), ('rot', C.c_void_p), ('flip', C.c_void_p),
        ('labels', C.c_void_p), ('K', C.c_int), ('centers', C.c_void_p), ('poses', C.c_void_p), ('gt3ds', C.c_void_p),
        ('S', C.c_int), ('trans_max', C.c_int), ('geom', C.c_void_p),
        ('labels_out', C.c_void_p), ('centers_out', C.c_void_p), ('poses_out', C.c_void_p), ('gt3ds_out', C.c_void_p),
        ('crops', C.c_void_p), ('plane_hi', C.c_void_p), ('plane_lo', C.c_void_p), ('WP', C.c_int),
    ]


HD_EVAL_KP, HD_EVAL_KP_PA, HD_EVAL_KP_PCK, HD_EVAL_JOINTS, HD_EVAL_JOINTS_PA, HD_EVAL_ACCEL, HD_EVAL_ACCEL_ERROR, HD_EVAL_VIS3D = range(8)
HD_EVAL_COLS = 8


class EvalFramesArgs(C.Structure):
    """Mirror of hd_eval_frames_args."""
    _fields_ = [
        ('N', C.c_int), ('n_seq', C.c_int), ('seq_start', C.c_void_p), ('K', C.c_int), ('J', C.c_int),
        ('kps_gt', C.c_void_p), ('kps_gt_ld', C.c_longlong), ('kps_pred', C.c_void_p), ('kps_pred_ld', C.c_longlong),
        ('joints_gt', C.c_void_p), ('joints_gt_ld', C.c_longlong), ('joints_pred', C.c_void_p), ('joints_pred_ld', C.c_longlong),
        ('img_size', C.c_float), ('min_visible', C.c_int), ('out', C.c_void_p),
    ]


# name -> (restype, argtypes); must list every symbol include/hd_b200.h declares.
_vp, _i, _ll, _f, _sz = C.c_void_p, C.c_int, C.c_longlong, C.c_float, C.c_size_t
SIGNATURES = {
    'hd_version': (_i, []),
    'hd_status_string': (C.c_char_p, [_i]),
    'hd_last_error': (C.c_char_p, []),
    'hd_launch_count': (_ll, []),
    'hd_launch_count_reset': (None, []),
    'hd_conv_gemm': (_i, [C.POINTER(ConvDesc), _vp]),
    'hd_conv_gemm_profile': (_i, [C.POINTER(ConvDesc), _vp, _vp]),
    'hd_make_weight_tmap': (_i, [_vp, _i, _i, _i, _i, _vp]),
    'hd_make_act_tmap': (_i, [_vp, _ll, _i, _ll, _i, _vp]),
    'hd_pack_conv1_planes': (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    'hd_conv1_7x7s2': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    'hd_maxpool3x3s2_same': (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    'hd_subsample': (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp]),
    'hd_bnrelu_avgpool': (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    'hd_bn_stats_workspace_bytes': (_sz, [_ll, _i]),
    'hd_bn_batch_stats': (_i, [_vp, _ll, _i, _ll, _vp, _vp, _f] + [_vp] * 6 + [C.c_double, _vp, _sz, _vp]),
    'hd_bn_moving_update': (_i, [_vp, _vp, _ll, _i, C.c_double, _vp, _vp, _vp]),
    'hd_conv_wgrad_workspace_bytes': (_sz, [_ll, _i, _i, _i]),
    'hd_conv_wgrad': (_i, [_vp, _ll] + [_i] * 11 + [_vp, _vp, _vp, _ll, _i, _vp, _vp, _vp, _sz, _vp]),
    'hd_bn_relu_backward_workspace_bytes': (_sz, [_ll, _i]),
    'hd_bn_relu_backward': (_i, [_vp, _vp, _i, _ll, _i, _vp, _vp, _vp, _vp, _f, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    'hd_maxpool3x3s2_same_backward': (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    'hd_zero_insert': (_i, [_vp, _vp] + [_i] * 7 + [_vp]),
    'hd_process_image': (_i, [_vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _i, _vp]),
    'hd_crop_geometry': (_i, [_i, _i, _vp, _i, _vp, _vp, _vp]),
    'hd_groupnorm_stats': (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _vp]),
    'hd_groupnorm_relu_split': (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _vp]),
    'hd_split_f16': (_i, [_vp, _vp, _vp, _ll, _vp]),
    'hd_ief_fc1_theta': (_i, [_vp, _vp, _i, _vp, _i, _i, _vp, _vp, _vp, _i, _vp]),
    'hd_ief_fc3': (_i, [_vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _vp]),
    'hd_ief_delta_init': (_i, [_vp, _vp, _i, _i, _vp]),
    'hd_net_destroy': (None, [_vp]),
    'hd_net_error': (C.c_char_p, [_vp]),
    'hd_net_num_launches': (_ll, [_vp]),
    'hd_resnet50_create': (_i, [_vp, _vp, _i, _i, C.POINTER(_vp)]),
    'hd_resnet50_forward': (_i, [_vp, _vp, _vp, _vp]),
    'hd_fmovie_create': (_i, [_vp, _vp, _i, _i, _i, C.POINTER(_vp)]),
    'hd_fmovie_forward': (_i, [_vp, _vp, _vp, _vp]),
    'hd_ief_create': (_i, [_vp, _vp, _i, C.POINTER(_i), _i, C.POINTER(_vp)]),
    'hd_ief_forward': (_i, [_vp, _vp, _vp, _vp, _vp]),
    'hd_smpl_pack_sizes': (_i, [_i, _i, _vp, _vp, C.POINTER(_i), C.POINTER(_i)]),
    'hd_smpl_pack': (_i, [_i, _i] + [_vp] * 13 + [_i] + [_vp] * 4),
    'hd_smpl_workspace_bytes': (_sz, [_i]),
    'hd_smpl_forward': (_i, [C.POINTER(SmplConsts), _vp, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _vp, _sz, _vp]),
    'hd_smpl_pose': (_i, [C.POINTER(SmplConsts), _vp, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _i, _vp, _sz, _vp]),
    'hd_smpl_lbs_tc': (_i, [_vp, _vp, _vp, _vp, _vp, _ll, _vp, _i, _i, _i, _i, _vp]),
    'hd_smpl_lbs': (_i, [C.POINTER(SmplConsts), _vp, _ll, _vp, _vp, _i, _i, _i, _vp]),
    'hd_smpl_joints': (_i, [C.POINTER(SmplConsts), _vp, _vp, _i, _vp, _vp, _i, _i, _i, _vp]),
    'hd_rodrigues': (_i, [_vp, _vp, _i, _vp]),
    'hd_rot2aa': (_i, [_vp, _vp, _i, _vp]),
    'hd_global_rigid': (_i, [_vp, _vp, C.POINTER(C.c_int), _vp, _vp, _i, _i, _vp]),
    'hd_orth_proj': (_i, [_vp, _vp, _vp, _i, _i, _vp]),
    'hd_smpl_backward_workspace_bytes': (_sz, [_i, _i]),
    'hd_smpl_lbs_backward': (_i, [C.POINTER(SmplConsts), C.POINTER(SmplGradConsts), _vp, _ll, _vp, _vp, _vp, _vp, _vp, _i, _vp]),
    'hd_smpl_pose_backward': (_i, [C.POINTER(SmplConsts), _vp, _i, _vp, _i, _i, _vp, _vp, _i, _vp, _vp, _vp, _i, _vp, _i, _vp]),
    'hd_rodrigues_backward': (_i, [_vp, _vp, _vp, _i, _vp]),
    'hd_global_rigid_backward': (_i, [_vp, _vp, C.POINTER(C.c_int), _vp, _vp, _vp, _vp, _i, _i, _vp]),
    'hd_orth_proj_backward': (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _vp]),
    'hd_pack_weight': (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _i, _i, _vp]),
    'hd_transpose_split': (_i, [_vp, _ll, _i, _ll, _i, _vp, _vp, _ll, _i, _ll, _vp]),
    'hd_im2col_t': (_i, [_vp, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp, _ll, _ll, _vp]),
    'hd_groupnorm_relu_backward': (_i, [_vp] * 8 + [_i, _i, _i, _i, _f, _i, _vp]),
    'hd_col_sum': (_i, [_vp, _ll, _i, _ll, _vp, _vp]),
    'hd_relu_backward': (_i, [_vp, _vp, _vp, _ll, _vp]),
    'hd_fc_small_dgrad': (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _i, _vp]),
    'hd_add_strided': (_i, [_vp, _ll, _vp, _ll, _vp, _ll, _i, _i, _vp]),
    'hd_dpose_workspace_bytes': (_sz, [_i]),
    'hd_dpose_trunk_forward': (_i, [_vp] * 10 + [_i, _vp]),
    'hd_dpose_out_forward': (_i, [_vp] * 4 + [_i, _vp]),
    'hd_dpose_trunk_backward': (_i, [_vp] * 11 + [_sz, _i, _vp]),
    'hd_dpose_grad_reduce': (_i, [_vp, _sz, _i, _vp, _vp]),
    'hd_loss_workspace_bytes': (_sz, [_vp, _i]),
    'hd_loss_forward': (_i, [_vp, _i, _vp, _vp, _sz, _vp]),
    'hd_loss_backward': (_i, [_vp, _i, _vp, _i, _vp, _vp, _sz, _vp]),
    'hd_render_workspace_bytes': (_sz, [_i, _i, _i]),
    'hd_tube_augment': (_i, [C.POINTER(TubeAugArgs), _vp]),
    'hd_render_mesh': (_i, [_vp, _ll, _i, _i, _vp, _i, _vp, _i, C.POINTER(RenderParams), _vp, _i, _vp, _vp, _vp, _sz, _vp]),
    'hd_eval_frames': (_i, [C.POINTER(EvalFramesArgs), _vp]),
    'hd_eval_mesh_tpose': (_i, [C.POINTER(SmplConsts), _vp, _i, _vp, _i, _i, _vp, _vp]),
    'hd_eval_verts_error': (_i, [_vp, _ll, _vp, _ll, _i, _i, _vp, _vp]),
}


def _load():
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            'human_dynamics_b200: %s is missing -- build it with `make -C human_dynamics_b200/csrc` '
            '(or `python -c "import __graft_entry__ as g; g.build()"`). There is no CPU fallback.' % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError here = header/library mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


class HDError(RuntimeError):
    pass


def check(rc: int, what: str = ''):
    if rc != 0:
        raise HDError('%s failed: %s [%s]' % (what or 'libhd_b200 call', lib.hd_status_string(rc).decode(),
                                              lib.hd_last_error().decode()))


def dptr(t, dtype=None):
    """Device pointer of a CUDA tensor (contiguity is the caller's business: strided views are allowed)."""
    import torch
    if t is None:
        return None
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise HDError('expected a CUDA torch.Tensor (no CPU fallback exists), got %r' % (type(t),))
    if dtype is not None and t.dtype != dtype:
        raise HDError('expected dtype %s, got %s' % (dtype, t.dtype))
    return C.c_void_p(t.data_ptr())


def fptr(t):
    import torch
    return dptr(t, torch.float32)


def current_stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
