"""ctypes binding of libvd3d_b200.so (C ABI declared in include/vd3d_b200.h).

The product path has NO fallback: if the shared library is missing or a symbol is absent, `load()` raises, and every
op raises `Vd3dError` when a kernel entry returns non-zero.
"""
from __future__ import annotations

import ctypes
import os
import re
from ctypes import c_char_p, c_double, c_float, c_int, c_longlong, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("VD3D_LIB") or os.path.join(_HERE, "libvd3d_b200.so")      # VD3D_LIB: A/B timing against another build of the same ABI
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "vd3d_b200.h")

_lib = None


class Vd3dError(RuntimeError):
    pass


def header_symbols(path: str = HEADER_PATH):
    """Every function name declared in include/vd3d_b200.h."""
    txt = open(path).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(vd3d_[a-z0-9_]+)\s*\(", txt)))


P = c_void_p
I = c_int
F = c_float

_SIGS = {
    "vd3d_last_error": (c_char_p, []),
    "vd3d_version": (I, []),
    "vd3d_launch_count": (c_longlong, []),
    "vd3d_launch_count_reset": (None, []),
    "vd3d_nchw_to_nhwc": (I, [P, P, I, I, I, I, I, I, P]),
    "vd3d_nhwc_to_nchw": (I, [P, P, I, I, I, I, I, I, P]),
    "vd3d_conv2d_nhwc": (I, [P, I, I, I, I, I, I, P, P, I, I, I, I, I, P, I, I, P, I, I, I, I, P]),
    "vd3d_dwconv3x3_nhwc": (I, [P, I, I, I, I, I, I, P, P, P, I, I, I, P]),
    "vd3d_maxpool3x3s2_nhwc": (I, [P, I, I, I, I, I, I, P, I, I, P]),
    "vd3d_maxpool2x2s2_nhwc": (I, [P, I, I, I, I, I, I, P, I, I, P]),
    "vd3d_dw_convtranspose_nhwc": (I, [P, I, I, I, I, I, I, P, I, P, I, I, P, I, I, P]),
    "vd3d_avgpool2_nhwc": (I, [P, I, I, I, I, I, I, P, I, I, P]),
    "vd3d_copy_channels_nhwc": (I, [P, I, I, I, I, P, I, I, P]),
    "vd3d_psm_cosine_nhwc": (I, [P, P, I, I, I, I, I, I, I, P, I, I, P]),
    "vd3d_psm_cosine_nchw": (I, [P, P, I, I, I, I, I, P, P]),
    "vd3d_concat_volume_conv3d": (I, [P, P, I, I, I, I, I, P, P, P, P, P, P, I, I, P]),
    "vd3d_tc_set_trace": (None, [P, I]),
    "vd3d_tc_pick_bn": (I, [I]),
    "vd3d_tc_pick_bn_persistent": (I, [I]),
    "vd3d_conv2d_tc": (I, [P, P, I, I, I, I, I, I, P, P, P, I, I, I, I, P, I, I, P, P, I, I, I, I, I, I, P]),
    "vd3d_conv2d_tc16": (I, [I, P, P, P, P, I, I, I, I, P, P, F, P, I, I, I, I, I, P, P, P, P, P, I, I, P, P, P, I, I, I, I, I, I, P]),
    "vd3d_convtranspose2d_tc16": (I, [P, P, I, I, I, I, I, I, P, P, F, P, P, P, P, I, I, I, I, I, P]),
    "vd3d_conv2d_tc16_gather": (I, [P, P, I, I, I, I, I, I, P, P, F, P, I, I, I, I, P, P, I, P, I, I, I, P]),
    "vd3d_conv2d_tc16_tiles": (I, [P, P, I, I, I, I, I, I, P, P, F, P, I, I, I, I, P, P, P, I, I, P, P, P, I, I, I, I, I, P, P, P, P]),
    "vd3d_stem_row_pitch": (I, [I, I, I, I]),
    "vd3d_image_to_h16_rows": (I, [P, I, I, I, I, P, P, I, I, P]),
    "vd3d_conv2d_tc16_stem": (I, [P, P, I, I, I, I, I, I, I, I, I, P, P, F, P, P, P, P, I, I, I, I, P]),
    "vd3d_conv2d_tc16_stem_pool": (I, [P, P, I, I, I, I, I, I, I, I, I, P, P, F, P, P, I, I, I, P]),
    "vd3d_stem_pool_row_pitch": (I, [I]),
    "vd3d_stem_pool_xoff": (I, []),
    "vd3d_stem_pool_fused": (I, [P, P, I, I, I, I, P, P, F, P, P, P, P, I, I, P]),
    "vd3d_row_conv_pitch": (I, [I, I, I, I, I, I]),
    "vd3d_image_to_h16_rows_c": (I, [P, I, I, I, I, P, P, I, I, I, P]),
    "vd3d_row_conv": (I, [P, P, I, I, I, I, I, I, I, I, I, I, P, P, F, P, I, I, P, P, P, I, I, I, I, P]),
    "vd3d_split_h16_nhwc": (I, [P, P, P, c_longlong, I, I, I, P]),
    "vd3d_psm_cosine_h16": (I, [P, P, P, P, c_longlong, I, I, I, I, I, P, I, I, P]),
    "vd3d_split_lo_nhwc": (I, [P, P, c_longlong, I, I, I, P]),
    "vd3d_deform_im2col_nhwc": (I, [P, I, I, I, I, I, I, P, I, I, P, I, I, I, I, I, I, I, I, I, P, P, I, P]),
    "vd3d_deform_im2col_h16": (I, [P, I, I, I, I, I, I, P, I, I, P, I, I, I, I, I, I, I, I, I, I, P, P, P, I, P]),
    "vd3d_deform_conv_fused": (I, [P, I, I, I, I, I, I, P, I, I, I, I, I, I, I, I, I, I, I, P, P, F, P, P, I, I, P, P, P, I, I, I, I, P]),
    "vd3d_deform_col2im_nhwc": (I, [P, I, I, I, I, I, I, P, I, I, P, I, I, I, I, I, I, I, I, P, I, P, I, I, P, I, I, P, I, I, P]),
    "vd3d_boxes_overlap_bev": (I, [P, I, P, I, P, P]),
    "vd3d_boxes_iou_bev": (I, [P, I, P, I, P, P]),
    "vd3d_nms_bev_workspace": (c_longlong, [I]),
    "vd3d_nms_bev": (I, [P, I, F, I, P, P, P, P]),
    "vd3d_monoflex_decode_workspace": (c_longlong, [I, I]),
    "vd3d_monoflex_decode": (I, [P, I, I, I, I, I, I, I, I, I, I, I, I, I, I, P, F, c_double, I, F, F, F, F, I, P, I, P, P, P, P, P, P, P]),
    "vd3d_km3d_decode_workspace": (c_longlong, [I, I, I]),
    "vd3d_km3d_decode": (I, [P, I, I, I, I, I, I, I, I, I, I, I, I, I, I, P, F, c_double, I, F, F, I, I, P, I, P, P, P, P, P, P, P]),
    "vd3d_train_augment_host": (I, [P, I, I, I, P, P, P]),
    "vd3d_train_augment_desc_bytes": (I, []),
    "vd3d_train_augment_describe": (I, [P, P, I, I, I, I, I, I, I, I, P, I, I, P, P, P]),
    "vd3d_train_augment": (I, [P, I, I, I, I, P, P, P, P]),
    "vd3d_center_targets_record_bytes": (I, []),
    "vd3d_center_targets_splat_bytes": (I, []),
    "vd3d_center_targets_pack": (I, [P, I, I, I, I, P, I, P, P]),
    "vd3d_center_targets_host": (I, [P, I, I, I, I, P]),
    "vd3d_center_targets": (I, [P, I, I, I, I, I, P, P, P]),
    "vd3d_post_opt_host": (I, [P, P, I, P, P, P, P, P, P, P, P, c_double, c_double, c_double, c_double, P, P]),
    "vd3d_post_opt": (I, [P, P, P, P, I, I, F, F, F, F, F, I, P]),
    "vd3d_fp16_range_check": (I, [P, I, P]),
    "vd3d_pack_records": (I, [P, P, P, P, I, I, I, P, P]),
    "vd3d_post_forward": (I, [P, P, P, P, I, I, P, P, P, P, P, P]),
    "vd3d_pack_records_geo": (I, [P, P, P, P, P, P, P, I, I, I, P, P]),
    "vd3d_look_ground_sample": (I, [P, I, I, I, I, I, I, P, I, I, P, F, F, P, P, I, P]),
    "vd3d_anchor_mask": (I, [P, P, P, I, I, I, F, F, F, P, P]),
    "vd3d_reg_candidates": (I, [P, P, I, I, I, I, F, I, P, P, P, P]),
    "vd3d_reg_tower_tile_cap": (I, [I, I, I]),
    "vd3d_reg_tower_tiles": (I, [P, I, I, I, I, P, P, P, P]),
    "vd3d_decode_nms_workspace": (c_longlong, [I, I]),
    "vd3d_decode_nms": (I, [P, P, P, P, P, I, I, I, I, F, c_double, F, F, I, P, P, P, P, P, P, P, P]),
    "vd3d_retina_decode_workspace": (c_longlong, [I, I, I]),
    "vd3d_retina_decode": (I, [I, P, P, P, I, I, P, I, I, I, I, I, P, P, F, c_double, I, P, P, P, P, P, P, P, P]),
    "vd3d_kitti_rotate_iou": (I, [P, I, P, I, I, P, P]),
    "vd3d_kitti_eval_workspace_bytes": (c_longlong, [I, c_longlong, c_longlong, c_longlong, I, I]),
    "vd3d_kitti_eval": (I, [P, P, P, I, c_longlong, c_longlong, c_longlong, c_longlong, P, I, P, I, I, P, P, P, P, P, P, c_longlong, P]),
    "vd3d_anchor_loss_workspace_bytes": (c_longlong, [I, I, I]),
    "vd3d_anchor_loss_forward": (I, [P, P, P, P, P, P, I, I, I, I, P, I, I, P, c_longlong, P, P, P, P, P, P]),
    "vd3d_anchor_loss_backward": (I, [P, P, P, P, P, I, I, I, I, P, P, P, P, P, P, P]),
    "vd3d_retina_loss_workspace_bytes": (c_longlong, [I, I, I]),
    "vd3d_retina_loss_forward": (I, [P, P, P, P, I, I, I, I, I, P, I, I, P, c_longlong, P, P, P, P, P, P]),
    "vd3d_retina_loss_backward": (I, [P, P, P, P, I, I, I, I, I, P, P, P, P, P, P, P]),
    "vd3d_monoflex_loss_workspace_bytes": (c_longlong, [I, I, I, I, I]),
    "vd3d_monoflex_loss_forward": (I, [P, P, I, I, I, I, I, F, F, F, P, c_longlong, P, P, P]),
    "vd3d_monoflex_loss_backward": (I, [P, P, I, I, I, I, I, F, F, F, P, P, P, P, P]),
    "vd3d_km3d_loss_workspace_bytes": (c_longlong, [I, I, I, I, I]),
    "vd3d_km3d_loss_forward": (I, [P, P, I, I, I, I, I, F, F, P, c_longlong, P, P, P]),
    "vd3d_km3d_loss_backward": (I, [P, P, I, I, I, I, I, F, F, P, P, P, P, P]),
    "vd3d_disparity_loss_workspace_bytes": (c_longlong, [I, I, I, I]),
    "vd3d_disparity_loss_forward": (I, [P, P, I, I, I, I, P, c_longlong, P, P, P]),
    "vd3d_disparity_loss_backward": (I, [P, P, P, I, I, I, I, P, P, P]),
    "vd3d_stereo_bm_workspace_bytes": (c_longlong, [I, I, I]),
    "vd3d_stereo_bm": (I, [P, P, I, I, I, P, P, P]),
    "vd3d_stereo_bm_f32": (I, [P, P, I, I, I, P, P, P, P, P, P]),
    "vd3d_disparity_block_max": (I, [P, I, I, I, I, P, P]),
    "vd3d_velo_disparity": (I, [P, I, I, P, P, P, c_double, I, I, P, P, P]),
    "vd3d_disparity_grey_host": (I, [P, I, I, P, P, P]),
    "vd3d_stereo_bm_host": (I, [P, P, I, I, P]),
    "vd3d_disparity_block_max_host": (I, [P, I, I, I, P]),
    "vd3d_velo_disparity_host": (I, [P, I, I, P, P, P, c_double, I, I, P]),
    "vd3d_anchor_prior_workspace_bytes": (c_longlong, [I, I, I, I, I]),
    "vd3d_anchor_prior_accumulate": (I, [P, P, P, I, I, P, I, I, P, I, P, I, c_double, P, P, P, P, P, c_longlong, P]),
    "vd3d_anchor_prior_host": (I, [P, P, P, I, I, P, I, I, P, I, P, I, c_double, P, P, P, P]),
}


def load():
    """dlopen the library and bind every symbol the header declares.  Raises if anything is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise Vd3dError(f"{LIB_PATH} not built: run `python __graft_entry__.py` (there is no CPU / eager fallback)")
    lib = ctypes.CDLL(LIB_PATH)
    for name in header_symbols():
        if not hasattr(lib, name):
            raise Vd3dError(f"symbol {name} declared in include/vd3d_b200.h is not exported by {LIB_PATH}")
        if name not in _SIGS:
            raise Vd3dError(f"no ctypes signature registered for {name}")
    for name, (res, args) in _SIGS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def call(name: str, *args):
    """Call an int-returning entry; raise Vd3dError with the library's message on failure."""
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise Vd3dError(f"{name} failed ({rc}): {lib.vd3d_last_error().decode()}")


def launch_count() -> int:
    return int(load().vd3d_launch_count())


def launch_count_reset() -> None:
    load().vd3d_launch_count_reset()
