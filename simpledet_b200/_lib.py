"""ctypes binding of the C ABI declared in include/simpledet_b200.h.

There is no CPU fallback: if the shared library is missing or a call fails this raises.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_size_t, c_uint64, c_void_p

from .build import LIB_PATH

_lib = None


class SdetError(RuntimeError):
    """A C-ABI entry point returned a non-zero sdet_status."""

    def __init__(self, code: int, msg: str):
        super().__init__(f"simpledet_b200 error {code}: {msg}")
        self.code = code


# name -> (argtypes); every function returns int status unless listed in _RESTYPES.
_P = c_void_p
_SIGNATURES = {
    "sdet_abi_version": [],
    "sdet_last_error": [],
    "sdet_build_digest": [],
    "sdet_launch_count": [],
    "sdet_roi_align_v2_workspace": [c_int, c_int],
    "sdet_roi_align_v2_forward": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int,
                                  c_int, c_float, _P, c_size_t, _P],
    "sdet_roi_align_v2_forward_ex": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int,
                                     c_int, c_float, _P, c_size_t, _P, c_int, POINTER(c_int)],
    "sdet_roi_align_v2_backward": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int,
                                   c_int, c_int, _P],
    "sdet_fpn_roi_align_v2_forward": [POINTER(_P), POINTER(c_int), POINTER(c_int), POINTER(c_int),
                                      c_int, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int,
                                      c_int, c_int, _P, c_size_t, _P],
    "sdet_fpn_roi_align_v2_forward_ex": [POINTER(_P), POINTER(c_int), POINTER(c_int), POINTER(c_int),
                                         c_int, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int,
                                         c_int, c_int, _P, c_size_t, _P, c_int, POINTER(c_int)],
    "sdet_fpn_roi_align_v2_workspace": [c_int, c_int, c_int, POINTER(c_int), POINTER(c_int), c_int],
    "sdet_fpn_roi_align_v2_forward_nhwc": [POINTER(_P), POINTER(c_int), POINTER(c_int), POINTER(c_int), c_int, _P, _P, _P,
                                           c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P, c_size_t, _P],
    "sdet_fpn_assign": [_P, c_int, POINTER(c_int), c_int, c_int, c_int, POINTER(_P), _P, _P],
    "sdet_fpn_roi_align_v2_backward": [_P, _P, _P, _P, POINTER(_P), POINTER(c_int), POINTER(c_int),
                                       c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P],
    "sdet_roi_pooling_v1_forward": [_P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int,
                                    c_int, c_float, _P],
    "sdet_roi_pooling_v1_backward": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int,
                                     c_int, c_float, c_int, _P],
    "sdet_roi_align_v2_backward_ordered": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int,
                                           c_int, c_int, _P],
    "sdet_fpn_roi_align_v2_backward_ordered": [_P, _P, _P, _P, POINTER(_P), POINTER(c_int), POINTER(c_int),
                                               c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P],
    "sdet_roi_pooling_v1_backward_ordered": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int,
                                             c_int, c_float, c_int, _P],
    "sdet_decode_bbox": [_P, _P, _P, _P, c_int, c_int, c_int, POINTER(c_float), POINTER(c_float), c_int,
                         c_int, _P],
    "sdet_proposal_v3_workspace": [c_int, c_int, c_int, c_int, c_int],
    "sdet_proposal_v3": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, POINTER(c_float), c_int,
                         POINTER(c_float), c_int, c_int, c_int, c_float, c_int, c_int, c_int, _P,
                         c_size_t, _P],
    "sdet_proposal_v3_fpn_workspace": [c_int, c_int, POINTER(c_int), POINTER(c_int), c_int, c_int],
    "sdet_proposal_v3_fpn": [POINTER(_P), POINTER(_P), _P, _P, _P, c_int, c_int, POINTER(c_int),
                             POINTER(c_int), POINTER(c_int), c_int, POINTER(c_float), c_int,
                             POINTER(c_float), c_int, c_int, c_int, c_float, c_int, c_int, c_int, _P,
                             c_size_t, _P],
    "sdet_proposal_legacy_workspace": [c_int, c_int, c_int, c_int, c_int],
    "sdet_proposal_legacy": [_P, _P, _P, _P, c_int, _P, _P, c_int, c_int, c_int, c_int, c_int, POINTER(c_float),
                             c_int, POINTER(c_float), c_int, c_int, c_int, c_float, c_int, c_int, c_int, c_int,
                             _P, c_size_t, _P],
    "sdet_gen_proposal_workspace": [c_int, c_int, c_int, c_int, c_int],
    "sdet_gen_proposal": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P, c_size_t, _P],
    "sdet_gen_anchor": [_P, c_int, c_int, c_int, POINTER(c_double), c_int, POINTER(c_double), c_int, _P],
    "sdet_gen_proposal_retina_workspace": [c_int, c_int, c_int, c_int],
    "sdet_gen_proposal_retina": [_P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                 c_float, POINTER(c_float), POINTER(c_float), c_int, c_int, c_int, _P, c_size_t, _P],
    "sdet_modulated_deformable_im2col": [_P, _P, _P, _P] + [c_int] * 13 + [_P],
    "sdet_modulated_deformable_col2im": [_P, _P, _P, _P, _P, _P, _P] + [c_int] * 13 + [_P],
    "sdet_final_detections": [_P, _P, _P, c_int, c_int, c_int, c_int, _P, _P, _P],
    "sdet_final_detections_ex": [_P, _P, _P, c_int, c_int, c_int, c_int, _P, _P, c_int, c_int, _P],
    "sdet_set_nms_sorted": [_P, _P, _P, c_int, c_int, c_float, _P, _P, _P, c_size_t, _P],
    "sdet_weighted_nms_workspace": [c_int, c_int],
    "sdet_weighted_nms_sorted": [_P, _P, c_int, c_int, c_float, c_float, _P, _P, _P, c_size_t, _P],
    "sdet_bbox_flip": [_P, _P, c_size_t, c_double, c_int, _P],
    "sdet_box_voting": [_P, _P, _P, c_int, c_int, c_float, c_int, c_float, _P],
    "sdet_bbox_overlaps": [_P, _P, _P, c_int, c_int, c_int, _P],
    "sdet_bbox_nonlinear_transform": [_P, _P, _P, c_int, _P],
    "sdet_bbox_pred": [_P, _P, _P, c_int, c_int, c_int, c_int, c_double, c_double, _P],
    "sdet_anchor_target_workspace": [c_int, c_int, c_int],
    "sdet_anchor_target": [_P, _P, c_int, _P, _P, _P, c_int, c_int, c_int, POINTER(c_int), POINTER(c_int),
                           POINTER(c_int), POINTER(c_double), c_int, POINTER(c_double), c_int, c_float, c_float,
                           c_float, c_float, c_int, c_int, _P, c_uint64, _P, c_size_t, _P],
    "sdet_contrib_nms_workspace": [c_int, c_int, c_int],
    "sdet_contrib_nms": [_P, _P, _P, c_int, c_int, c_int, c_int, c_float, c_int, _P, c_size_t, _P],
    "sdet_get_top_proposal": [_P, _P, _P, _P, c_int, c_int, c_int, _P],
    "sdet_mask_paste_count": [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P, _P],
    "sdet_mask_paste_write": [_P, _P, _P, c_int, c_int, c_int, c_int, c_int, _P, _P, _P],
    "sdet_multiclass_nms_workspace": [c_int, c_int, c_int, c_int],
    "sdet_multiclass_nms": [_P, _P, c_int, c_int, c_int, c_int, c_int, c_float, c_float, _P, _P, _P, _P,
                            _P, _P, c_size_t, _P],
    "sdet_proposal_target": [_P, _P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_float,
                             c_float, c_float, c_float, c_int, c_int, POINTER(c_float), POINTER(c_float),
                             POINTER(c_float), c_uint64, _P, c_int, _P, _P, _P, _P],
    "sdet_proposal_target_v2": [_P, _P, _P, _P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_float,
                                c_float, c_float, c_float, c_int, c_int, c_int, POINTER(c_float),
                                POINTER(c_float), POINTER(c_float), c_uint64, _P, c_int, _P, _P, _P, _P],
    "sdet_poly_mask_target": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P],
    "sdet_poly_mask_target_ratio": [_P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, _P],
    "sdet_focal_loss_forward": [_P, _P, c_size_t, _P],
    "sdet_focal_loss_backward": [_P, _P, _P, _P, c_int, c_int, c_int, c_float, c_float, c_float, c_int, _P,
                                 c_size_t, _P],
    "sdet_bbox_norm_backward": [_P, _P, _P, c_size_t, c_size_t, _P, c_size_t, _P],
    "sdet_sigmoid_ce_forward": [_P, _P, _P, c_int, c_size_t, _P, c_size_t, _P],
    "sdet_sigmoid_ce_backward": [_P, _P, _P, c_int, c_size_t, c_float, _P, c_size_t, _P],
    "sdet_soft_nms": [_P, _P, c_int, c_int, c_float, c_float, c_float, c_int, _P, _P, _P, _P],
    "sdet_deformable_im2col": [_P, _P, _P] + [c_int] * 13 + [_P],
    "sdet_deformable_im2col_plan": [c_int] * 13 + [POINTER(c_int)] * 3,
    "sdet_deformable_im2col_nhwc": [_P, _P, _P] + [c_int] * 13 + [_P],
    "sdet_deformable_col2im": [_P, _P, _P, _P, _P] + [c_int] * 13 + [_P],
    "sdet_nms_workspace": [c_int, c_int],
    "_nms": [_P, POINTER(c_int), _P, c_int, c_int, c_float, c_int],
    "sdet_nms_sorted": [_P, _P, c_int, c_int, c_float, c_int, _P, _P, _P, c_size_t, _P],
    "sdet_group_norm_workspace": [c_int, c_int, c_int, c_int],
    "sdet_group_norm_forward": [_P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_float, c_int, c_int, _P,
                                c_size_t, _P],
    "sdet_fcos_proposal_workspace": [c_int, c_int, c_int, c_int],
    "sdet_fcos_proposal": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_int, _P,
                           c_size_t, _P],
    "sdet_fcos_batch_proposal": [_P, _P, _P, _P, c_int, c_int, _P],
}
_RESTYPES = {"_nms": None, "sdet_last_error": c_char_p, "sdet_build_digest": c_char_p, "sdet_launch_count": c_uint64,
             "sdet_proposal_v3_workspace": c_size_t, "sdet_proposal_legacy_workspace": c_size_t,
             "sdet_gen_proposal_workspace": c_size_t, "sdet_anchor_target_workspace": c_size_t, "sdet_weighted_nms_workspace": c_size_t, "sdet_gen_proposal_retina_workspace": c_size_t, "sdet_proposal_v3_fpn_workspace": c_size_t, "sdet_contrib_nms_workspace": c_size_t,
             "sdet_nms_workspace": c_size_t, "sdet_roi_align_v2_workspace": c_size_t, "sdet_fpn_roi_align_v2_workspace": c_size_t, "sdet_multiclass_nms_workspace": c_size_t,
             "sdet_group_norm_workspace": c_size_t, "sdet_fcos_proposal_workspace": c_size_t}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def lib() -> ctypes.CDLL:
    """Load libsimpledet_b200.so (built in-tree by simpledet_b200.build / __graft_entry__.build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU fallback)")
        L = ctypes.CDLL(LIB_PATH)
        for name, argtypes in _SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError if the header and the library disagree
            fn.argtypes = argtypes
            fn.restype = _RESTYPES.get(name, c_int)
        _lib = L
    return _lib


def check(status: int) -> None:
    if status != 0:
        raise SdetError(status, lib().sdet_last_error().decode())


def build_digest() -> str:
    return lib().sdet_build_digest().decode()


def launch_count() -> int:
    return int(lib().sdet_launch_count())
