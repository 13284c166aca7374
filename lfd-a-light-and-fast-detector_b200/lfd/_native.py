# -*- coding: utf-8 -*-
"""ctypes binding of liblfd_b200.so (C-ABI declared in include/lfd_b200.h).

The library is built in-tree by ../build.py (nvcc, sm_90a).  Loading never falls back to anything else:
if the shared object is missing and cannot be built, importing a native entry point raises.
"""
import ctypes as C
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
_PKG = os.path.dirname(_HERE)
LIB_PATH = os.environ.get('LFD_B200_LIB') or os.path.join(_PKG, 'liblfd_b200.so')   # LFD_B200_LIB: an alternative build of the SAME library (tuning experiments)
MAX_LEVELS = 8

OP_STEM0, OP_CONV, OP_GN_APPLY, OP_HEAD_FINAL, OP_STEM4 = 0, 1, 2, 3, 4
INPUT_F32_NCHW, INPUT_U8_NHWC = 0, 1
CONV_UMMA, CONV_SIMT = 0, 1
DTYPE_BF16, DTYPE_FP16 = 0, 1
CLS_SIGMOID, CLS_SOFTMAX, CLS_BCE, CLS_QFL = 0, 1, 2, 3
REG_IOU, REG_GIOU, REG_DIOU, REG_CIOU, REG_SMOOTH_L1, REG_MSE = range(6)
BBOX_SIGMOID, BBOX_EXP, BBOX_INDEPENDENT = 0, 1, 2
ASSIGN_DIST, ASSIGN_LONGER, ASSIGN_SHORTER = 0, 1, 2


class LfdError(RuntimeError):
    pass


class Op(C.Structure):
    _fields_ = [('kind', C.c_int32),
                ('N', C.c_int32), ('H', C.c_int32), ('W', C.c_int32), ('Cin', C.c_int32),
                ('Ho', C.c_int32), ('Wo', C.c_int32), ('Cout', C.c_int32),
                ('ksize', C.c_int32), ('stride', C.c_int32), ('relu', C.c_int32), ('gn_groups', C.c_int32),
                ('n_cls', C.c_int32), ('n_reg', C.c_int32), ('point_off', C.c_int32), ('cc', C.c_int32),
                ('branch', C.c_int32), ('wait_mask', C.c_int32),
                ('in_off', C.c_int64), ('out_off', C.c_int64), ('res_off', C.c_int64), ('stats_off', C.c_int64),
                ('weight', C.c_void_p), ('scale', C.c_void_p), ('shift', C.c_void_p),
                ('gamma', C.c_void_p), ('beta', C.c_void_p),
                ('tail_cout', C.c_int32), ('tail_relu', C.c_int32),
                ('tail_weight', C.c_void_p), ('tail_scale', C.c_void_p), ('tail_shift', C.c_void_p),
                ('ds_cout', C.c_int32), ('dtype', C.c_int32), ('max_ctas', C.c_int32), ('pad_', C.c_int32), ('ds_out_off', C.c_int64),
                ('ds_weight', C.c_void_p), ('ds_shift', C.c_void_p),
                ('s2_relu', C.c_int32), ('s3_relu', C.c_int32),
                ('s2_weight', C.c_void_p), ('s2_shift', C.c_void_p), ('s3_weight', C.c_void_p), ('s3_shift', C.c_void_p)]


class PostCfg(C.Structure):
    _fields_ = [('N', C.c_int32), ('P', C.c_int32), ('C', C.c_int32), ('cls_channels', C.c_int32),
                ('cls_mode', C.c_int32), ('bbox_mode', C.c_int32), ('class_agnostic', C.c_int32),
                ('num_levels', C.c_int32),
                ('level_off', C.c_int32 * MAX_LEVELS), ('level_w', C.c_int32 * MAX_LEVELS),
                ('level_stride', C.c_int32 * MAX_LEVELS), ('level_hi', C.c_float * MAX_LEVELS),
                ('score_thr', C.c_float), ('iou_thr', C.c_float), ('cap', C.c_int32), ('max_ctas', C.c_int32)]


class Levels(C.Structure):
    _fields_ = [('num_levels', C.c_int32),
                ('off', C.c_int32 * MAX_LEVELS), ('w', C.c_int32 * MAX_LEVELS), ('stride', C.c_int32 * MAX_LEVELS),
                ('lo', C.c_float * MAX_LEVELS), ('hi', C.c_float * MAX_LEVELS),
                ('glo', C.c_float * MAX_LEVELS), ('ghi', C.c_float * MAX_LEVELS)]


class LossCfg(C.Structure):
    _fields_ = [('N', C.c_int32), ('P', C.c_int32), ('C', C.c_int32), ('cls_mode', C.c_int32), ('bbox_mode', C.c_int32), ('reg_loss', C.c_int32),
                ('gamma', C.c_float), ('alpha', C.c_float), ('reg_eps', C.c_float), ('smooth_l1_beta', C.c_float),
                ('cls_weight', C.c_float), ('reg_weight', C.c_float), ('max_ctas', C.c_int32)]


# training plan ops (include/lfd_b200.h, lfd_top).  TOP_INFER runs one inference op (an Op: STEM0 / CONV with tail and shortcut /
# STEM4, bf16) inside a training plan: ptr[0] = the host address of the Op, off[0..3] = its input / output / residual / shortcut
# output, which replace the Op's own offsets (the frozen backbone prefix of a fine-tuning step, lfd/_train.py)
(TOP_PACK, TOP_STEM0, TOP_CONV, TOP_BN_STATS, TOP_BN_APPLY, TOP_GN_APPLY, TOP_HEAD_FINAL, TOP_HEAD_FINAL_BWD, TOP_NORM_BWD_REDUCE,
 TOP_NORM_BWD_APPLY, TOP_WGRAD, TOP_WGRAD_STEM, TOP_UNPACK, TOP_ZERO, TOP_INFER) = range(15)
WGRAD_UMMA, WGRAD_SIMT = 0, 1
PACK_CONV_FWD, PACK_CONV_DGRAD, PACK_STEM, PACK_ROUND_F32, PACK_SCALE_SHIFT = range(5)
UNPACK_CONV, UNPACK_ADD = 0, 1


MAX_BRANCHES = 8          # LFD_MAX_BRANCHES

RESIZE_COPY, RESIZE_LINEAR, RESIZE_AREA2 = 0, 1, 2
INPUT_OUT_U8_NHWC, INPUT_OUT_F32_NCHW = 0, 1


class InputDesc(C.Structure):
    _fields_ = [('src_off', C.c_int64), ('inv_scale', C.c_double), ('pitch', C.c_int32), ('channels', C.c_int32),
                ('win_x', C.c_int32), ('win_y', C.c_int32), ('win_w', C.c_int32), ('win_h', C.c_int32),
                ('src_w', C.c_int32), ('src_h', C.c_int32), ('dw', C.c_int32), ('dh', C.c_int32), ('mode', C.c_int32),
                ('crop_x', C.c_int32), ('crop_y', C.c_int32), ('out_w', C.c_int32), ('out_h', C.c_int32), ('flip', C.c_int32)]


class Top(C.Structure):
    _fields_ = [('kind', C.c_int32),
                ('N', C.c_int32), ('H', C.c_int32), ('W', C.c_int32), ('Cin', C.c_int32), ('Ho', C.c_int32), ('Wo', C.c_int32),
                ('Cout', C.c_int32), ('ksize', C.c_int32), ('stride', C.c_int32),
                ('relu', C.c_int32), ('groups', C.c_int32), ('cc', C.c_int32), ('n_cls', C.c_int32), ('n_reg', C.c_int32),
                ('point_off', C.c_int32), ('P', C.c_int32), ('cls_stride', C.c_int32),
                ('accumulate', C.c_int32), ('upH', C.c_int32), ('upW', C.c_int32), ('n_desc', C.c_int32), ('max_n', C.c_int32),
                ('impl', C.c_int32), ('frozen', C.c_int32), ('branch', C.c_int32), ('wait_mask', C.c_int32), ('max_ctas', C.c_int32), ('eps', C.c_float), ('momentum', C.c_float),
                ('off', C.c_int64 * 8), ('ptr', C.c_void_p * 6)]


class PackDesc(C.Structure):
    _fields_ = [('kind', C.c_int32), ('Cout', C.c_int32), ('Cin', C.c_int32), ('k', C.c_int32), ('cc', C.c_int32), ('n', C.c_int32),
                ('src', C.c_void_p), ('src2', C.c_void_p), ('dst', C.c_void_p), ('dst2', C.c_void_p), ('dst3', C.c_void_p)]


class UnpackDesc(C.Structure):
    _fields_ = [('kind', C.c_int32), ('Cout', C.c_int32), ('Cin', C.c_int32), ('kk', C.c_int32), ('n', C.c_int32), ('pad_', C.c_int32),
                ('src', C.c_void_p), ('dst', C.c_void_p)]


# every symbol include/lfd_b200.h declares: name -> (restype, argtypes)
_vp, _i, _f, _i64 = C.c_void_p, C.c_int, C.c_float, C.c_int64
SYMBOLS = {
    'lfd_abi_version': (_i, []),
    'lfd_struct_bytes': (_i, [_i]),
    'lfd_last_error': (C.c_char_p, []),
    'lfd_device_sm_count': (_i, []),
    'lfd_conv_query': (_i, [_i] * 11 + [C.POINTER(_i)] * 4 + [C.POINTER(_i64)]),
    'lfd_stem4_query': (_i, [_i] * 3 + [C.POINTER(_i), C.POINTER(_i64), C.POINTER(_i), C.POINTER(_i)]),
    'lfd_plan_create': (_i, [C.POINTER(Op), _i, _i, _i, _i, _i64, _i64, _i64, _i, C.POINTER(_vp)]),
    'lfd_plan_destroy': (_i, [_vp]),
    'lfd_plan_num_launches': (_i, [_vp]),
    'lfd_plan_forward': (_i, [_vp, _vp, _i, _vp, _vp, _vp, _i, _vp]),
    'lfd_plan_profile': (_i, [_vp, _vp, _i, _vp, _vp, _vp, C.POINTER(C.c_float), _vp]),
    'lfd_debug_set_trace': (_i, [_vp]),
    'lfd_debug_set_timeline': (_i, [_vp]),
    'lfd_run_op': (_i, [C.POINTER(Op), _vp, _i, _vp, _vp, _vp, _i, _i, _i, _vp]),
    'lfd_postprocess_workspace_bytes': (C.c_size_t, [C.POINTER(PostCfg)]),
    'lfd_postprocess': (_i, [C.POINTER(PostCfg)] + [_vp] * 11),
    'lfd_multiclass_nms_workspace_bytes': (C.c_size_t, [_i]),
    'lfd_multiclass_nms': (_i, [_vp, _i, _vp, _i, _vp, _i, _i, _f, _f, _i, _i] + [_vp] * 7),
    'lfd_nms_workspace_bytes': (C.c_size_t, [_i]),
    'lfd_nms': (_i, [_vp, _i, _f, _vp, _vp, _vp, _vp]),
    'lfd_assign_targets': (_i, [C.POINTER(Levels), _i, _i, _i, _i, _i, _i] + [_vp] * 8),
    'lfd_detection_loss': (_i, [C.POINTER(Levels), C.POINTER(LossCfg)] + [_vp] * 10),
    'lfd_box_loss': (_i, [_i, _vp, _vp, _i, _f, _vp, _vp, _vp]),
    'lfd_sigmoid_focal_loss_forward': (_i, [_vp, _vp, _i, _i, _f, _f, _vp, _vp]),
    'lfd_sigmoid_focal_loss_backward': (_i, [_vp, _vp, _vp, _i, _i, _f, _f, _vp, _vp]),
    'lfd_train_plan_create': (_i, [C.POINTER(Top), _i, _i64, C.POINTER(_vp)]),
    'lfd_train_plan_destroy': (_i, [_vp]),
    'lfd_train_plan_num_ops': (_i, [_vp]),
    'lfd_train_plan_run': (_i, [_vp, _vp, _i, _vp, _i, _vp]),
    'lfd_train_plan_profile': (_i, [_vp, _vp, _i, _vp, C.POINTER(C.c_float), _vp]),
    'lfd_run_top': (_i, [C.POINTER(Top), _vp, _i, _vp, _vp]),
    'lfd_grad_sqnorm': (_i, [_vp, _i64, _vp, _vp]),
    'lfd_sgd_step': (_i, [_vp, _vp, _vp, _i64, _f, _f, _f, _f, _i, _f, _f, _vp, _vp]),
    'lfd_input_batch': (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _i, C.POINTER(_f), C.POINTER(_f), _vp]),
}

_lib = None


def build(force=False):
    """Compile the shared library in-tree (needs nvcc, not a GPU)."""
    if _PKG not in sys.path:
        sys.path.insert(0, _PKG)
    import importlib
    b = importlib.import_module('build')
    return b.build(force=force)


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        try:
            build()
        except Exception as e:  # no silent fallback: the native library IS the product
            raise LfdError('liblfd_b200.so is missing and could not be built (%s); there is no CPU / PyTorch '
                           'fallback for the LFD hot path' % (e,))
    L = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args
    if L.lfd_abi_version() != 5:
        raise LfdError('liblfd_b200.so ABI version mismatch')
    for which, st in enumerate((Op, Top, PackDesc, UnpackDesc, PostCfg, LossCfg, Levels, InputDesc)):
        if L.lfd_struct_bytes(which) != C.sizeof(st):
            raise LfdError('liblfd_b200.so: %s is %d bytes in the library, %d in lfd/_native.py' % (st.__name__, L.lfd_struct_bytes(which), C.sizeof(st)))
    _lib = L
    return L


def check(rc):
    if rc != 0:
        raise LfdError('liblfd_b200 error %d: %s' % (rc, lib().lfd_last_error().decode()))


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def conv_query(N, H, W, Cin, Ho, Wo, Cout, ksize, stride, tail_cout=0, ds_cout=0):
    cc, st, res, nt = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    smem = C.c_int64()
    check(lib().lfd_conv_query(N, H, W, Cin, Ho, Wo, Cout, ksize, stride, tail_cout, ds_cout, C.byref(cc), C.byref(st), C.byref(res),
                               C.byref(nt), C.byref(smem)))
    return dict(cc=cc.value, stages=st.value, weights_resident=res.value, num_tiles=nt.value, smem_bytes=smem.value)


def stem4_query(N, H, W):
    """Tiles, shared memory and stem3 output size of the fused four-conv stem (LFD_OP_STEM4) on N images of H x W."""
    nt, ho, wo = C.c_int(), C.c_int(), C.c_int()
    smem = C.c_int64()
    check(lib().lfd_stem4_query(N, H, W, C.byref(nt), C.byref(smem), C.byref(ho), C.byref(wo)))
    return dict(num_tiles=nt.value, smem_bytes=smem.value, Ho=ho.value, Wo=wo.value)
