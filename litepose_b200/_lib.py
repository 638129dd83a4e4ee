"""ctypes binding of the C-ABI shared library (include/litepose_b200.h, and include/litepose_b200_train.h and
include/litepose_b200_train_bn.h for the training kernels, include/litepose_b200_debug.h for the SM limit).

The CUDA library is the product: there is no Python/PyTorch fallback.  Importing
this module never compiles anything; ``load()`` raises ``LitePoseLibraryError`` if the
in-tree ``litepose_b200/_C/liblitepose_b200.so`` is missing (build it with
``python -m litepose_b200.build``) and ``LitePoseError`` when an entry point fails.
"""
import ctypes
import os
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "_C", "liblitepose_b200.so")

LP_OK = 0
ACT_NONE, ACT_RELU, ACT_RELU6 = 0, 1, 2
LP_DT_F32, LP_DT_F16 = 0, 1


class LitePoseLibraryError(RuntimeError):
    pass


class LitePoseError(RuntimeError):
    pass


_c = ctypes
_vp, _i, _sz, _d, _f = _c.c_void_p, _c.c_int, _c.c_size_t, _c.c_double, _c.c_float

# name -> (restype, argtypes); every symbol declared in include/litepose_b200.h
SIGNATURES = {
    "lp_version": (_i, []),
    "lp_last_error": (_c.c_char_p, []),
    "lp_device_check": (_i, []),
    "lp_launch_count": (_c.c_uint64, []),
    "lp_reset_launch_count": (None, []),
    "lp_stem_conv3x3_s2": (_i, [_vp, _i, _i, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "lp_stem_conv3x3_s2_act": (_i, [_vp, _i, _i, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "lp_stem_fused_supported": (_i, [_i, _i, _i]),
    "lp_stem_fused_f16": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "lp_dwconv_f16": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "lp_set_dw_precision": (None, [_i]),
    "lp_get_dw_precision": (_i, []),
    "lp_pw1x1_packed_elems": (_sz, [_i, _i]),
    "lp_pw1x1_packed_bias_elems": (_sz, [_i]),
    "lp_pw1x1_pack": (_i, [_vp, _vp, _i, _i, _vp, _vp]),
    "lp_pw1x1_f16": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "lp_dw7_project_f16": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "lp_block_s1_supported": (_i, [_i, _i, _i]),
    "lp_block_s1_wexp_elems": (_sz, [_i, _i]),
    "lp_block_s1_pack_wexp": (_i, [_vp, _i, _i, _vp]),
    "lp_block_s1_f16": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "lp_block_s2_supported": (_i, [_i, _i, _i]),
    "lp_block_s2_f16": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "lp_deconv_packed_elems": (_sz, [_i, _i, _i]),
    "lp_deconv_packed_bias_elems": (_sz, [_i]),
    "lp_deconv_pack": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "lp_fusion_deconv_f16": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "lp_fusion_deconv_act_f16": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "lp_bn_stats_workspace_bytes": (_sz, [_i, _i]),
    "lp_bn_stats_f16": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _d, _d, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "lp_bn_apply_f16": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "lp_head_packed_elems": (_sz, [_i, _i, _i]),
    "lp_head_pack": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "lp_head_pw_dual_f16": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "lp_head_fused_dw_elems": (_sz, [_i, _i]),
    "lp_head_fused_pw_elems": (_sz, [_i, _i, _i]),
    "lp_head_fused_pack": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "lp_head_fused_f16": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "lp_nms_topk_workspace_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "lp_nms_topk_f32": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _d, _vp, _vp, _vp, _vp, _sz, _vp]),
    "lp_tag_match_workspace_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "lp_tag_match_f32": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _d, _d, _i, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "lp_adjust_refine_workspace_bytes": (_sz, [_i, _i, _i]),
    "lp_adjust_refine_f32": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i, _i, _vp, _sz, _vp]),
    "lp_glue_f32": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "lp_glue_scale_f32": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _f, _vp, _vp, _vp]),
    "lp_pack_payload_f32": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "lp_plant_crowd_f32": (_i, [_vp, _vp, _vp, _c.c_int64, _vp, _vp, _vp, _c.c_int64, _vp]),
    "lp_warp_affine_normalize_u8": (_i, [_vp, _i, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _i, _vp]),
    "lp_warp_affine_normalize_ragged_u8": (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _vp, _i, _vp]),
    "lp_nms_topk_ragged_workspace_bytes": (_sz, [_i, _vp, _i, _i]),
    "lp_nms_topk_ragged_f32": (_i, [_vp, _vp, _i, _vp, _vp, _i, _i, _i, _i, _d, _vp, _vp, _vp, _vp, _sz, _vp]),
    "lp_tag_match_ragged_f32": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _d, _d, _i, _i, _i, _i, _vp, _vp, _vp, _sz,
                                     _vp]),
    "lp_adjust_refine_ragged_f32": (_i, [_vp, _vp, _i, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _i, _i, _vp, _sz, _vp]),
    "lp_transform_preds_f32": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "lp_find_peaks_f32": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _f, _i, _vp, _vp, _vp, _vp, _vp]),
    "lp_assign_f32": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _f, _vp, _vp, _vp, _vp]),
    "lp_find_peaks_maps_f32": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _i, _i, _i, _i, _f, _i, _vp, _vp, _vp, _vp, _vp]),
    "lp_pack_fast_payload_f32": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp]),
}

# every symbol declared in include/litepose_b200_train.h (the same library)
TRAIN_SIGNATURES = {
    "lp_dw_nchw_fwd": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "lp_dw_nchw_dgrad": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "lp_dw_nchw_wgrad_workspace_bytes": (_sz, [_i, _i, _i, _i, _i, _i]),
    "lp_dw_nchw_wgrad": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _sz, _vp]),
}

# every symbol declared in include/litepose_b200_train_bn.h (the same library)
TRAIN_BN_SIGNATURES = {
    "lp_bn_nchw_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "lp_bn_nchw_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _d, _d, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _sz, _vp]),
    "lp_bn_nchw_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _sz, _vp]),
}

# every symbol declared in include/litepose_b200_debug.h (the same library): library state for tests and debugging,
# launching nothing
DEBUG_SIGNATURES = {
    "lp_set_sm_limit": (None, [_i]),
    "lp_get_sm_limit": (_i, []),
}

_lock = threading.Lock()
_lib = None


def load():
    """Load (once) and return the ctypes library with typed entry points."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.isfile(LIB_PATH):
            raise LitePoseLibraryError(
                "CUDA library %s not found: run `python -m litepose_b200.build` "
                "(there is no CPU/PyTorch fallback for the inference path)" % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in (list(SIGNATURES.items()) + list(TRAIN_SIGNATURES.items()) +
                                  list(TRAIN_BN_SIGNATURES.items()) + list(DEBUG_SIGNATURES.items())):
            fn = getattr(lib, name)   # AttributeError if the .so lacks a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(rc, what=""):
    if rc != LP_OK:
        msg = load().lp_last_error()
        raise LitePoseError("%s failed (code %d): %s" % (what or "litepose_b200 call", rc,
                                                         msg.decode() if msg else "?"))


def ptr(t):
    """Device/host pointer of a torch tensor (or None)."""
    return None if t is None else t.data_ptr()


def current_stream_ptr():
    import torch
    return torch.cuda.current_stream().cuda_stream
