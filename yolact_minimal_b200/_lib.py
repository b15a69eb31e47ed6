"""ctypes binding of libyolact_b200.so (the C ABI in include/yolact_b200.h).

There is no fallback: if the library is missing or a call fails this raises.  Build it with
`python -m yolact_minimal_b200.build` (nvcc, sm_90a).
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libyolact_b200.so')

c_f32p = C.POINTER(C.c_float)
c_i32p = C.POINTER(C.c_int32)
c_u8p = C.POINTER(C.c_uint8)
vp = C.c_void_p


class DetectParams(C.Structure):
    _fields_ = [('score_thr', C.c_float), ('iou_thr', C.c_float), ('top_k', C.c_int), ('max_det', C.c_int),
                ('num_classes', C.c_int), ('coef_dim', C.c_int), ('traditional', C.c_int), ('img_size', C.c_float), ('no_clip', C.c_int)]


class ProfEntry(C.Structure):
    _fields_ = [('name', C.c_char * 32), ('launches', C.c_int), ('forwards', C.c_int), ('ms', C.c_double),
                ('flops', C.c_double), ('bytes', C.c_double)]


class NetConfig(C.Structure):
    _fields_ = [('depth', C.c_int), ('img_size', C.c_int), ('num_classes', C.c_int), ('num_ratios', C.c_int),
                ('coef_dim', C.c_int)]


class LossParams(C.Structure):
    _fields_ = [('batch', C.c_int), ('num_anchors', C.c_int), ('num_classes', C.c_int), ('coef_dim', C.c_int), ('proto_size', C.c_int),
                ('seg_size', C.c_int), ('mask_size', C.c_int), ('pos_iou_thr', C.c_float), ('neg_iou_thr', C.c_float),
                ('neg_pos_ratio', C.c_int), ('masks_to_train', C.c_int), ('conf_alpha', C.c_float), ('bbox_alpha', C.c_float),
                ('mask_alpha', C.c_float), ('semantic_alpha', C.c_float)]


EVAL_MAX_THR = 16


class EvalParams(C.Structure):
    _fields_ = [('num_classes', C.c_int), ('num_thr', C.c_int), ('thr', C.c_double * EVAL_MAX_THR)]


class TrainHparams(C.Structure):
    _fields_ = [('pos_iou_thr', C.c_float), ('neg_iou_thr', C.c_float), ('neg_pos_ratio', C.c_int), ('masks_to_train', C.c_int),
                ('conf_alpha', C.c_float), ('bbox_alpha', C.c_float), ('mask_alpha', C.c_float), ('semantic_alpha', C.c_float),
                ('bn_momentum', C.c_float), ('bn_eps', C.c_float)]


# name -> (restype, argtypes); every symbol declared in include/yolact_b200.h
PROTOTYPES = {
    'yb_version': (C.c_int, []),
    'yb_last_error': (C.c_char_p, []),
    'yb_launch_count': (C.c_uint64, []),
    'yb_device_info': (C.c_int, [C.POINTER(C.c_int)] * 3),
    'yb_detect_workspace_bytes': (C.c_size_t, [C.c_int, C.c_int, C.POINTER(DetectParams)]),
    'yb_detect': (C.c_int, [vp, vp, vp, vp, C.c_int, C.c_int, C.POINTER(DetectParams), vp, C.c_size_t,
                            vp, vp, vp, vp, vp, vp, vp]),
    'yb_detect_host': (C.c_int, [vp, vp, vp, vp, C.c_int, C.c_int, C.POINTER(DetectParams),
                                 vp, vp, vp, vp, vp, vp]),
    'yb_hard_nms': (C.c_int, [vp, C.c_int, C.c_float, vp, vp]),
    'yb_hard_nms_host': (C.c_int, [vp, C.c_int, C.c_float, vp]),
    'yb_mask_workspace_bytes': (C.c_size_t, [C.c_int, C.c_int]),
    'yb_mask_assemble': (C.c_int, [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                   vp, C.c_size_t, vp, vp, vp]),
    'yb_val_aug': (C.c_int, [vp, C.c_int, C.c_int, C.c_int, vp, vp]),
    'yb_pack_mask_bits': (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp]),
    'yb_mask_iou_bits': (C.c_int, [vp, C.c_int, vp, C.c_int, C.c_int64, vp, vp]),
    'yb_box_iou': (C.c_int, [vp, C.c_int, vp, C.c_int, vp, vp]),
    'yb_mask_rle': (C.c_int, [vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, vp, vp]),
    'yb_eval_state_bytes': (C.c_size_t, [C.POINTER(EvalParams)]),
    'yb_eval_match_workspace_bytes': (C.c_size_t, [C.c_int, C.c_int, C.c_int64, C.POINTER(EvalParams)]),
    'yb_eval_ap_workspace_bytes': (C.c_size_t, [C.c_int64, C.POINTER(EvalParams)]),
    'yb_eval_match': (C.c_int, [C.POINTER(EvalParams), C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, C.c_int64, vp, vp, vp, C.c_int64,
                                vp, vp, C.c_int64, vp, vp, vp, C.c_int64, vp, vp, C.c_size_t, vp]),
    'yb_eval_ap': (C.c_int, [C.POINTER(EvalParams), vp, vp, vp, C.c_int64, vp, vp, C.c_size_t, vp, vp, vp]),
    'yb_net_create': (C.c_int, [C.POINTER(NetConfig), C.POINTER(vp)]),
    'yb_net_destroy': (None, [vp]),
    'yb_net_num_params': (C.c_int, [vp]),
    'yb_net_param_info': (C.c_int, [vp, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int64)]),
    'yb_net_set_param': (C.c_int, [vp, C.c_char_p, vp, C.c_int64]),
    'yb_net_finalize': (C.c_int, [vp, C.c_int, C.c_int]),
    'yb_net_num_anchors': (C.c_int, [vp]),
    'yb_net_proto_size': (C.c_int, [vp]),
    'yb_net_anchors_host': (C.c_int, [vp, vp]),
    'yb_net_anchors_device': (vp, [vp]),
    'yb_net_set_anchors': (C.c_int, [vp, vp, C.c_int]),
    'yb_net_forward': (C.c_int, [vp, vp, C.c_int, vp, vp, vp, vp, vp]),
    'yb_net_read_activation': (C.c_int, [vp, C.c_char_p, C.c_int, vp, C.c_int64, C.POINTER(C.c_int),
                                         C.POINTER(C.c_int), C.POINTER(C.c_int), vp]),
    'yb_net_set_profiling': (C.c_int, [vp, C.c_int]),
    'yb_net_profile': (C.c_int, [vp, C.POINTER(ProfEntry), C.c_int, C.POINTER(C.c_int)]),
    'yb_conv2d': (C.c_int, [vp, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int, C.c_int, vp]),
    'yb_net_detect_host': (C.c_int, [vp, vp, C.c_int, C.POINTER(DetectParams), vp, vp, vp, vp, vp, vp]),
    'yb_net_last_proto': (vp, [vp]),
    'yb_net_submit_host': (C.c_int, [vp, vp, C.c_int, C.POINTER(DetectParams), C.POINTER(C.c_int)]),
    'yb_net_collect_host': (C.c_int, [vp, C.c_int, vp, vp, vp, vp, vp, vp]),
    'yb_losses_workspace_bytes': (C.c_size_t, [C.POINTER(LossParams), C.c_int]),
    'yb_losses': (C.c_int, [C.POINTER(LossParams), vp, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp, C.c_int, C.c_int, C.c_uint32, vp, vp,
                            vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_size_t, vp]),
    'yb_train_create': (C.c_int, [C.POINTER(NetConfig), C.c_int, C.c_int, C.POINTER(vp)]),
    'yb_train_destroy': (None, [vp]),
    'yb_train_num_tensors': (C.c_int, [vp]),
    'yb_train_tensor_info': (C.c_int, [vp, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int64), C.POINTER(C.c_int)]),
    'yb_train_bind': (C.c_int, [vp, C.c_char_p, vp, vp]),
    'yb_train_set_anchors': (C.c_int, [vp, vp, C.c_int]),
    'yb_train_forward': (C.c_int, [vp, vp, vp, vp, vp, C.c_int, C.c_int, C.POINTER(TrainHparams), C.c_uint32, vp, vp]),
    'yb_train_backward': (C.c_int, [vp, vp, vp]),
    'yb_train_read': (C.c_int, [vp, C.c_char_p, C.c_int, vp, C.c_int64, C.POINTER(C.c_int), C.POINTER(C.c_int), vp]),
    'yb_train_launches_per_step': (C.c_uint64, [vp]),
}

_lib = None


class YolactB200Error(RuntimeError):
    pass


def lib():
    """Load (once) and return the ctypes library.  Raises if it is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise YolactB200Error(
                f'{LIB_PATH} not found: the CUDA library is not built (run `python -m yolact_minimal_b200.build`). '
                'There is no CPU fallback.')
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in PROTOTYPES.items():
            fn = getattr(l, name)          # AttributeError if the symbol is missing -> loud
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(status, what=''):
    if status != 0:
        msg = lib().yb_last_error()
        raise YolactB200Error(f'{what} failed with status {status}: {msg.decode() if msg else ""}')


def launch_count():
    return int(lib().yb_launch_count())
