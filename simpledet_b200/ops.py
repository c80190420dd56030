"""Host-side mirror of the reference's operator interface for the detection hot path.

Every public callable keeps the reference operator's name, argument names, defaults, output
arity and shape rules (SURVEY.md §8b) and forwards to the C ABI (include/simpledet_b200.h).
PyTorch is used for device memory, streams and autograd plumbing only — all arithmetic happens in
libsimpledet_b200.so.  There is no CPU path: CPU tensors raise.

`OPS` maps the reference's registry strings (``_contrib_ROIAlign_v2``, ``ROIPooling_v1`` …) to
these callables, which is what a symbol/builder façade binds to.
"""
from __future__ import annotations

import ctypes
from typing import Sequence

import torch

from . import _lib
from ._lib import check

__all__ = ["decode_retina", "fpn_roi_align_nhwc", "gpu_nms", "greedy_nms", "bbox_overlaps_cython", "assign_layer_fpn", "BboxPostProcessing", "ROIAlign_v2", "roi_align_v2_raw", "ROIPooling_v1", "roi_pooling_v1_raw",
           "fpn_roi_align", "fpn_roi_align_raw", "DecodeBBox", "Proposal_v3", "Proposal_v3_fpn", "NMS", "nms_sorted", "get_top_proposal",
           "multiclass_nms", "ProposalTarget", "FocalLoss", "BBoxNorm",
           "SigmoidCrossEntropy", "soft_nms", "soft_nms_batched",
           "cython_soft_nms_wrapper", "DeformableConvolution", "ProposalMaskTarget", "ProposalTarget_v2", "Proposal", "Proposal_v2", "GenAnchor", "GenProposal", "GenProposalRetina", "AnchorTarget2D", "PyramidAnchorTarget2D", "bbox_overlaps",
           "nonlinear_transform", "nonlinear_pred", "iou_pred", "set_nms", "py_weighted_nms", "py_set_nms_wrapper",
           "wnms_wrapper", "flip_boxes", "box_voting", "final_detections", "ModulatedDeformableConvolution",
           "GroupNorm", "group_norm_raw", "get_proposal_single_stage", "get_batch_proposal", "OPS"]


def _dev(t: torch.Tensor | None, name: str, dtype=torch.float32) -> torch.Tensor | None:
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError(f"{name}: simpledet_b200 ops are CUDA-only (no CPU fallback)")
    _same_device(t, name)
    if t.dtype != dtype:
        raise TypeError(f"{name}: expected {dtype}, got {t.dtype} (the reference path is fp32, "
                        "symbol/builder.py:882-894)")
    return t.contiguous()


def _same_device(t: torch.Tensor, name: str) -> None:
    """The C ABI launches on the calling thread's current device and stream: a tensor that lives elsewhere would be
    dereferenced on the wrong GPU.  Fail loudly instead (wrap the call in `with torch.cuda.device(t.device):`)."""
    cur = torch.cuda.current_device()
    if t.device.index != cur:
        raise RuntimeError(f"{name} is on cuda:{t.device.index} but the current device is cuda:{cur}: "
                           "run the operator under `with torch.cuda.device(tensor.device):`")


def _dev_any_layout(t: torch.Tensor, name: str, dtype=torch.float32) -> torch.Tensor:
    """The checks of _dev without forcing NCHW contiguity (for operators that take channels-last tensors as they are)."""
    if not t.is_cuda:
        raise RuntimeError(f"{name}: simpledet_b200 ops are CUDA-only (no CPU fallback)")
    _same_device(t, name)
    if t.dtype != dtype:
        raise TypeError(f"{name}: expected {dtype}, got {t.dtype}")
    return t


def _p(t: torch.Tensor | None):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _pair(v) -> tuple[int, int]:
    if isinstance(v, int):
        return v, v
    v = tuple(int(x) for x in v)
    if len(v) != 2:
        raise ValueError("pooled_size must have 2 dims (set_expect_ndim(2))")
    return v


# --------------------------------------------------------------------------------------------
# _contrib_ROIAlign_v2  (operator_cxx/contrib/roi_align_v2.cc:170-228)
# --------------------------------------------------------------------------------------------
def roi_align_v2_raw(data, rois, pooled_size, spatial_scale, with_argmax=True, use_plan=True, path=0,
                     return_path=False):
    """All three outputs of the reference op: (out, argmax_x, argmax_y), each (B,N,C,PH,PW).

    Shape rules of ROIAlign_v2 FInferShape (roi_align_v2.cc:187-210): data 4-D, rois 3-D
    (B,N,4) with rois.shape[0] == data.shape[0].
    """
    data, rois = _dev(data, "data"), _dev(rois, "rois")
    if data.dim() != 4:
        raise ValueError("data should be a 4D tensor")
    if rois.dim() != 3 or rois.shape[2] != 4:
        raise ValueError("bbox should be a 3D tensor of shape [batch, rois, 4]")
    if rois.shape[0] != data.shape[0]:
        raise ValueError("rois.shape[0] must equal data.shape[0]")
    ph, pw = _pair(pooled_size)
    B, C, H, W = data.shape
    N = rois.shape[1]
    out = torch.empty((B, N, C, ph, pw), device=data.device, dtype=torch.float32)
    ax = torch.empty_like(out) if with_argmax else None
    ay = torch.empty_like(out) if with_argmax else None
    L = _lib.lib()
    nbytes = L.sdet_roi_align_v2_workspace(B, N) if use_plan else 0
    if use_plan and not with_argmax and path == 3:  # room for the NHWC re-layout: channels-last kernel
        nbytes = L.sdet_fpn_roi_align_v2_workspace(B, N, C, (ctypes.c_int * 1)(H), (ctypes.c_int * 1)(W), 1)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=data.device) if nbytes else None
    used = ctypes.c_int(-1)
    check(L.sdet_roi_align_v2_forward_ex(_p(data), _p(rois), _p(out), _p(ax), _p(ay), B, N, C, H, W, ph, pw,
                                         float(spatial_scale), _p(ws), nbytes, _stream(), int(path),
                                         ctypes.byref(used)))
    if return_path:
        return out, ax, ay, used.value
    return out, ax, ay


def _backward_entry(name: str):
    """The RoI pooling backward entry `name`, or its `_ordered` twin under torch.use_deterministic_algorithms(True):
    the default entries scatter with float atomics, the ordered ones return the serial sum in index order, bit for bit
    the same on every run."""
    if torch.are_deterministic_algorithms_enabled():
        name += "_ordered"
    return getattr(_lib.lib(), name)


class _ROIAlignV2Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, data, rois, ph, pw, spatial_scale):
        need = data.requires_grad
        out, ax, ay = roi_align_v2_raw(data, rois, (ph, pw), spatial_scale, with_argmax=need)
        if need:
            ctx.save_for_backward(ax, ay)
            ctx.dshape = tuple(data.shape)
            ctx.rshape = tuple(rois.shape)
        return out

    @staticmethod
    def backward(ctx, ograd):
        if not ctx.saved_tensors:  # data did not require grad (only rois did): their gradient is identically zero
            return None, None, None, None, None
        ax, ay = ctx.saved_tensors
        B, C, H, W = ctx.dshape
        N = ctx.rshape[1]
        ograd = _dev(ograd, "ograd")
        grad = torch.empty(ctx.dshape, device=ograd.device, dtype=torch.float32)
        ph, pw = ograd.shape[3], ograd.shape[4]
        check(_backward_entry("sdet_roi_align_v2_backward")(_p(ograd), _p(ax), _p(ay), _p(grad), None, B, N,
                                                            C, H, W, ph, pw, 0, _stream()))
        # grad_rois is identically zero in the reference (roi_align_v2.cu:139-141)
        return grad, None, None, None, None


def ROIAlign_v2(data, rois, pooled_size, spatial_scale):
    """mx.sym.contrib.ROIAlign_v2(data, rois, pooled_size=(h,w), spatial_scale=s) — one visible
    output (B,N,C,PH,PW); differentiable w.r.t. data."""
    ph, pw = _pair(pooled_size)
    return _ROIAlignV2Fn.apply(data, rois, ph, pw, float(spatial_scale))


# --------------------------------------------------------------------------------------------
# Fused FPN RoIAlign = fpn_roi_assign + 4 x ROIAlign_v2 + add_n (models/FPN/builder.py:573-605)
# --------------------------------------------------------------------------------------------
def _level_arrays(feats: Sequence[torch.Tensor], strides: Sequence[int]):
    L = len(feats)
    if L != len(strides):
        raise ValueError("one stride per feature level")
    feats = [_dev(f, f"feat[{i}]") for i, f in enumerate(feats)]
    B, C = feats[0].shape[:2]
    for f in feats:
        if f.dim() != 4 or f.shape[0] != B or f.shape[1] != C:
            raise ValueError("all levels must be (B,C,H_l,W_l) with the same B and C")
    ptrs = (ctypes.c_void_p * L)(*[f.data_ptr() for f in feats])
    Hs = (ctypes.c_int * L)(*[f.shape[2] for f in feats])
    Ws = (ctypes.c_int * L)(*[f.shape[3] for f in feats])
    Ss = (ctypes.c_int * L)(*[int(s) for s in strides])
    return feats, ptrs, Hs, Ws, Ss, B, C


def fpn_roi_align_raw(feats, rois, strides, out_size, roi_canonical_scale=224,
                      roi_canonical_level=4, with_argmax=True, use_plan=True, path=0, return_path=False):
    """-> (out, argmax_x, argmax_y, levels).  out (B,N,C,PH,PW); levels (B,N) int32 index into
    `strides` (-1: the roi matched no level and pools to zeros)."""
    feats, ptrs, Hs, Ws, Ss, B, C = _level_arrays(feats, strides)
    rois = _dev(rois, "rois")
    if rois.dim() != 3 or rois.shape[2] != 4 or rois.shape[0] != B:
        raise ValueError("rois must be (B,N,4)")
    ph, pw = _pair(out_size)
    N = rois.shape[1]
    out = torch.empty((B, N, C, ph, pw), device=rois.device, dtype=torch.float32)
    ax = torch.empty_like(out) if with_argmax else None
    ay = torch.empty_like(out) if with_argmax else None
    levels = torch.empty((B, N), device=rois.device, dtype=torch.int32)
    L = _lib.lib()
    nbytes = L.sdet_roi_align_v2_workspace(B, N) if use_plan else 0
    if use_plan and not with_argmax and path == 3:  # room for the NHWC re-layout: channels-last kernel
        nbytes = L.sdet_fpn_roi_align_v2_workspace(B, N, C, Hs, Ws, len(feats))
    ws = _ws_cached(nbytes, rois.device) if nbytes else None
    used = ctypes.c_int(-1)
    check(L.sdet_fpn_roi_align_v2_forward_ex(
        ptrs, Hs, Ws, Ss, len(feats), _p(rois), _p(out), _p(ax), _p(ay), _p(levels), B, N, C, ph, pw,
        int(roi_canonical_scale), int(roi_canonical_level), _p(ws), nbytes, _stream(), int(path),
        ctypes.byref(used)))
    if return_path:  # 0 inline per-roi, 1 planned per-roi, 2 band-stationary (+ per-roi leftovers)
        return out, ax, ay, levels, used.value
    return out, ax, ay, levels


_WS_CACHE: dict = {}


def _ws_cached(nbytes: int, device) -> torch.Tensor:
    """One grow-only workspace per device and stream (the RoIAlign workspace holds a re-layout of the feature maps:
    allocating ~100 MB per call would cost more than the kernels)."""
    key = (str(device), torch.cuda.current_stream(device).cuda_stream)
    t = _WS_CACHE.get(key)
    if t is None or t.numel() < nbytes:
        t = torch.empty(nbytes, dtype=torch.uint8, device=device)
        _WS_CACHE[key] = t
    return t


def fpn_roi_align_nhwc(feats_nhwc, rois, strides, out_size, roi_canonical_scale=224, roi_canonical_level=4):
    """Fused FPN RoIAlign over channels-last features: feats_nhwc[l] is (B, H_l, W_l, C) contiguous (what a
    tensor-core convolution in channels_last memory format produces: `y.permute(0, 2, 3, 1)` of it is such a
    view).  Inference (no argmax planes).  -> (out (B,N,C,PH,PW), levels (B,N))."""
    feats = [_dev(f, f"feat[{i}]") for i, f in enumerate(feats_nhwc)]
    rois = _dev(rois, "rois")
    B, C = feats[0].shape[0], feats[0].shape[3]
    ph, pw = _pair(out_size)
    N = rois.shape[1]
    Lv = len(feats)
    out = torch.empty((B, N, C, ph, pw), device=rois.device, dtype=torch.float32)
    levels = torch.empty((B, N), device=rois.device, dtype=torch.int32)
    ptrs = (ctypes.c_void_p * Lv)(*[f.data_ptr() for f in feats])
    Hs = (ctypes.c_int * Lv)(*[f.shape[1] for f in feats])
    Ws = (ctypes.c_int * Lv)(*[f.shape[2] for f in feats])
    Ss = (ctypes.c_int * Lv)(*[int(s) for s in strides])
    L = _lib.lib()
    nbytes = L.sdet_roi_align_v2_workspace(B, N)
    ws = _ws_cached(nbytes, rois.device)
    check(L.sdet_fpn_roi_align_v2_forward_nhwc(ptrs, Hs, Ws, Ss, Lv, _p(rois), _p(out), _p(levels), B, N, C, ph, pw,
                                               int(roi_canonical_scale), int(roi_canonical_level), _p(ws), nbytes,
                                               _stream()))
    return out, levels


class _FpnRoiAlignFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rois, strides, ph, pw, scale0, lvl0, *feats):
        need = any(f.requires_grad for f in feats)
        ctx.num_inputs = 6 + len(feats)
        out, ax, ay, levels = fpn_roi_align_raw(feats, rois, strides, (ph, pw), scale0, lvl0,
                                                with_argmax=need)
        if need:
            ctx.save_for_backward(ax, ay, levels)
            ctx.shapes = [tuple(f.shape) for f in feats]
            ctx.N = rois.shape[1]
        return out

    @staticmethod
    def backward(ctx, ograd):
        if not ctx.saved_tensors:  # no feature map required grad
            return (None,) * ctx.num_inputs
        ax, ay, levels = ctx.saved_tensors
        ograd = _dev(ograd, "ograd")
        grads = [torch.empty(s, device=ograd.device, dtype=torch.float32) for s in ctx.shapes]
        L = len(grads)
        B, C = ctx.shapes[0][:2]
        ptrs = (ctypes.c_void_p * L)(*[g.data_ptr() for g in grads])
        Hs = (ctypes.c_int * L)(*[s[2] for s in ctx.shapes])
        Ws = (ctypes.c_int * L)(*[s[3] for s in ctx.shapes])
        check(_backward_entry("sdet_fpn_roi_align_v2_backward")(
            _p(ograd), _p(ax), _p(ay), _p(levels), ptrs, Hs, Ws, L, B, ctx.N, C, ograd.shape[3],
            ograd.shape[4], 0, _stream()))
        return (None, None, None, None, None, None, *grads)


def fpn_roi_align(feats, rois, strides=(4, 8, 16, 32), out_size=7, roi_canonical_scale=224,
                  roi_canonical_level=4):
    """FPNRoiAlign.get_roi_feature (models/FPN/builder.py:567-610) in one kernel.  Returns the
    5-D (B,N,C,PH,PW) tensor the reference reshapes with (-3,-2)."""
    ph, pw = _pair(out_size)
    return _FpnRoiAlignFn.apply(rois, tuple(int(s) for s in strides), ph, pw,
                                int(roi_canonical_scale), int(roi_canonical_level), *feats)


# --------------------------------------------------------------------------------------------
# operator_py/bbox_transform.py + operator_py/cython/{bbox,bbox_self}.pyx on the device
# --------------------------------------------------------------------------------------------
def bbox_overlaps(boxes, query_boxes, mode="iou"):
    """bbox_overlaps_cython (mode='iou') / bbox_selfoverlaps_cython (mode='ioa'): (N,4),(K,4) -> (N,K)."""
    boxes, query_boxes = _dev(boxes, "boxes"), _dev(query_boxes, "query_boxes")
    N, K = int(boxes.shape[0]), int(query_boxes.shape[0])
    out = torch.empty((N, K), device=boxes.device, dtype=torch.float32)
    check(_lib.lib().sdet_bbox_overlaps(_p(boxes), _p(query_boxes), _p(out), N, K, {"iou": 0, "ioa": 1}[mode],
                                        _stream()))
    return out


def nonlinear_transform(ex_rois, gt_rois):
    """bbox_transform.nonlinear_transform in float64: (N,4),(N,4) -> (N,4)."""
    ex_rois, gt_rois = _dev(ex_rois, "ex_rois", torch.float64), _dev(gt_rois, "gt_rois", torch.float64)
    if ex_rois.shape != gt_rois.shape:
        raise ValueError("inconsistent rois number")
    out = torch.empty_like(ex_rois)
    check(_lib.lib().sdet_bbox_nonlinear_transform(_p(ex_rois), _p(gt_rois), _p(out), int(ex_rois.shape[0]),
                                                   _stream()))
    return out


def _bbox_pred(boxes, box_deltas, iou, im_shape):
    boxes, box_deltas = _dev(boxes, "boxes"), _dev(box_deltas, "box_deltas", torch.float64)
    N, K4 = int(box_deltas.shape[0]), int(box_deltas.shape[1])
    out = torch.empty_like(box_deltas)
    h, w = (float(im_shape[0]), float(im_shape[1])) if im_shape is not None else (0.0, 0.0)
    check(_lib.lib().sdet_bbox_pred(_p(boxes), _p(box_deltas), _p(out), N, K4 // 4, int(iou),
                                    int(im_shape is not None), h, w, _stream()))
    return out


def nonlinear_pred(boxes, box_deltas, im_shape=None):
    """bbox_transform.nonlinear_pred (boxes float32 (N,4), deltas float64 (N,4K)); im_shape=(h,w) fuses
    clip_boxes."""
    return _bbox_pred(boxes, box_deltas, False, im_shape)


def iou_pred(boxes, box_deltas, im_shape=None):
    """bbox_transform.iou_pred, optionally fused with clip_boxes."""
    return _bbox_pred(boxes, box_deltas, True, im_shape)


def flip_boxes(boxes, im_width):
    """bbox_transform.flip_boxes: (N, 4K) float32 or float64."""
    if boxes.dtype not in (torch.float32, torch.float64):
        raise TypeError("boxes must be float32 or float64")
    boxes = _dev(boxes, "boxes", boxes.dtype)
    out = torch.empty_like(boxes)
    check(_lib.lib().sdet_bbox_flip(_p(boxes), _p(out), boxes.numel() // 4, float(im_width),
                                    int(boxes.dtype == torch.float64), _stream()))
    return out


_VOTE_METHODS = {"ID": 0, "TEMP_AVG": 1, "AVG": 2, "IOU_AVG": 3, "GENERALIZED_AVG": 4, "QUASI_SUM": 5}


def box_voting(top_dets, all_dets, thresh=0.5, scoring_method="ID", beta=1.0):
    """bbox_transform.box_voting: top_dets (T,5), all_dets (N,5) float32 on the device -> (T,5)."""
    if scoring_method not in _VOTE_METHODS:
        raise NotImplementedError("Unknown scoring method {}".format(scoring_method))
    top_dets, all_dets = _dev(top_dets, "top_dets"), _dev(all_dets, "all_dets")
    out = torch.empty_like(top_dets)
    check(_lib.lib().sdet_box_voting(_p(top_dets), _p(all_dets), _p(out), int(top_dets.shape[0]),
                                     int(all_dets.shape[0]), float(thresh), _VOTE_METHODS[scoring_method],
                                     float(beta), _stream()))
    return out


# --------------------------------------------------------------------------------------------
# AnchorTarget2D / PyramidAnchorTarget2D  (core/detection_input.py:353-565, models/FPN/input.py:55-148)
# --------------------------------------------------------------------------------------------
def _seq(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v,)


def PyramidAnchorTarget2D(im_info, gt_bbox, stride, short, long, scales, aspects, allowed_border=9999, pos_thr=0.7,
                          neg_thr=0.3, min_pos_thr=0.0, image_anchor=256, pos_fraction=0.5, priorities=None,
                          seed=0):
    """Batched RPN targets.  im_info (B,3), gt_bbox (B,G,4|5) device tensors; stride/short/long per
    pyramid level (scalars = one level).  Returns rpn_cls_label (B, A*S), rpn_reg_target (B,4A,S),
    rpn_reg_weight (B,4A,S), S = sum of level cells — the arrays the reference's loader emits per image."""
    im_info, gt_bbox = _dev(im_info, "im_info"), _dev(gt_bbox, "gt_bbox")
    strides, shorts, longs = _seq(stride), _seq(short), _seq(long)
    if not (len(strides) == len(shorts) == len(longs)):
        raise ValueError("stride / short / long must have one entry per level")
    if gt_bbox.dim() != 3 or gt_bbox.shape[2] not in (4, 5) or gt_bbox.shape[0] != im_info.shape[0]:
        raise ValueError("gt_bbox must be (B,G,4) or (B,G,5)")
    B, G = int(gt_bbox.shape[0]), int(gt_bbox.shape[1])
    A = len(scales) * len(aspects)
    S = sum(int(a) * int(b) for a, b in zip(shorts, longs))
    N = A * S
    dev = im_info.device
    label = torch.empty((B, N), device=dev, dtype=torch.float32)
    target = torch.empty((B, 4 * A, S), device=dev, dtype=torch.float32)
    weight = torch.empty((B, 4 * A, S), device=dev, dtype=torch.float32)
    if priorities is not None:
        if not priorities.is_cuda or priorities.dtype not in (torch.int32, torch.uint32) or priorities.numel() != B * N:
            raise ValueError("priorities must be a CUDA int32/uint32 tensor with B*A*S elements")
        priorities = priorities.contiguous()
    L = _lib.lib()
    nbytes = L.sdet_anchor_target_workspace(B, N, G)
    ws = _ws(nbytes, dev)
    ia = lambda v: (ctypes.c_int * len(v))(*[int(x) for x in v])  # noqa: E731
    da = lambda v: (ctypes.c_double * len(v))(*[float(x) for x in v])  # noqa: E731
    check(L.sdet_anchor_target(_p(im_info), _p(gt_bbox), int(gt_bbox.shape[2]), _p(label), _p(target), _p(weight),
                               B, G, len(strides), ia(strides), ia(shorts), ia(longs), da(scales), len(scales),
                               da(aspects), len(aspects), float(allowed_border), float(neg_thr), float(pos_thr),
                               float(min_pos_thr), int(image_anchor), int(pos_fraction * image_anchor),
                               _p(priorities), int(seed), _p(ws), nbytes, _stream()))
    return label, target, weight


def AnchorTarget2D(im_info, gt_bbox, stride, short, long, scales, aspects, allowed_border=0, **kw):
    """Single-level variant: rpn_reg_target / weight come back as (B, 4A, fh, fw) with (fh, fw) =
    (long, short) when h >= w else (short, long) — fixed per call, so one orientation per batch."""
    label, target, weight = PyramidAnchorTarget2D(im_info, gt_bbox, (stride,), (short,), (long,), scales, aspects,
                                                  allowed_border=allowed_border, **kw)
    return label, target, weight


# --------------------------------------------------------------------------------------------
# ROIPooling_v1  (operator_cxx/roi_pooling_v1.cc:243; shape rules roi_pooling_v1-inl.h:170-195)
# --------------------------------------------------------------------------------------------
def roi_pooling_v1_raw(data, rois, pooled_size, spatial_scale):
    """-> (out, maxidx), each (R,C,PH,PW); rois (R,5) = [batch_index, x1, y1, x2, y2]."""
    data, rois = _dev(data, "data"), _dev(rois, "rois")
    if data.dim() != 4:
        raise ValueError("data should be a 4D tensor")
    if rois.dim() != 2 or rois.shape[1] != 5:
        raise ValueError("bbox should be a 2D tensor of shape [batch, 5]")
    ph, pw = _pair(pooled_size)
    B, C, H, W = data.shape
    R = rois.shape[0]
    out = torch.empty((R, C, ph, pw), device=data.device, dtype=torch.float32)
    idx = torch.empty_like(out)
    check(_lib.lib().sdet_roi_pooling_v1_forward(_p(data), _p(rois), _p(out), _p(idx), B, R, C, H, W,
                                                 ph, pw, float(spatial_scale), _stream()))
    return out, idx


class _ROIPoolingV1Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, data, rois, ph, pw, spatial_scale):
        out, idx = roi_pooling_v1_raw(data, rois, (ph, pw), spatial_scale)
        ctx.save_for_backward(idx, rois)
        ctx.dshape = tuple(data.shape)
        ctx.scale = float(spatial_scale)
        return out

    @staticmethod
    def backward(ctx, ograd):
        idx, rois = ctx.saved_tensors
        B, C, H, W = ctx.dshape
        ograd = _dev(ograd, "ograd")
        R, _, ph, pw = ograd.shape
        grad = torch.empty(ctx.dshape, device=ograd.device, dtype=torch.float32)
        check(_backward_entry("sdet_roi_pooling_v1_backward")(_p(ograd), _p(idx), _p(rois), _p(grad), None, B,
                                                              R, C, H, W, ph, pw, ctx.scale, 0, _stream()))
        return grad, None, None, None, None


def ROIPooling_v1(data, rois, pooled_size, spatial_scale):
    """mx.sym.ROIPooling_v1(data, rois, pooled_size, spatial_scale) — one visible output."""
    ph, pw = _pair(pooled_size)
    return _ROIPoolingV1Fn.apply(data, rois, ph, pw, float(spatial_scale))


# --------------------------------------------------------------------------------------------
# _contrib_DecodeBBox  (operator_cxx/contrib/decodebbox.cc:150-209; params decodebbox-inl.h:50-69)
# --------------------------------------------------------------------------------------------
def _f4(v, name):
    v = tuple(float(x) for x in v)
    if len(v) != 4:
        raise ValueError(f"{name} must have 4 values")
    return (ctypes.c_float * 4)(*v)


def DecodeBBox(rois, bbox_pred, im_info, bbox_mean=(0.0, 0.0, 0.0, 0.0), bbox_std=(0.1, 0.1, 0.2, 0.2),
               class_agnostic=True, bbox_decode_type="xywh"):
    """mx.sym.contrib.DecodeBBox / X.decode_bbox.  rois (B,N,4), bbox_pred (B,N,4K), im_info (B,3)
    -> (B,N,4) if class_agnostic (the op's default!) else (B,N,4K).  No gradient (Backward writes
    zeros, decodebbox.cc:212-229)."""
    rois, bbox_pred, im_info = _dev(rois, "rois"), _dev(bbox_pred, "bbox_pred"), _dev(im_info, "im_info")
    if rois.dim() != 3 or rois.shape[2] != 4:
        raise ValueError("rois must be (B,N,4)")
    if bbox_pred.dim() != 3 or bbox_pred.shape[:2] != rois.shape[:2] or bbox_pred.shape[2] % 4:
        raise ValueError("bbox_pred must be (B,N,4K)")
    if bbox_decode_type not in ("xywh", "xyxy"):
        raise ValueError("bbox_decode_type must be 'xywh' or 'xyxy'")
    B, N, K4 = bbox_pred.shape
    out = torch.empty((B, N, 4 if class_agnostic else K4), device=rois.device, dtype=torch.float32)
    check(_lib.lib().sdet_decode_bbox(_p(rois), _p(bbox_pred), _p(im_info), _p(out), B, N, K4,
                                      _f4(bbox_mean, "bbox_mean"), _f4(bbox_std, "bbox_std"),
                                      int(bool(class_agnostic)), 0 if bbox_decode_type == "xywh" else 1,
                                      _stream()))
    return out


# --------------------------------------------------------------------------------------------
# _contrib_Proposal_v3  (operator_cxx/contrib/proposal_v3.cu:435-638)
# --------------------------------------------------------------------------------------------
def _ws(nbytes: int, device) -> torch.Tensor:
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def Proposal_v3(cls_prob, bbox_pred, im_info, rpn_pre_nms_top_n=6000, rpn_post_nms_top_n=300,
                threshold=0.7, rpn_min_size=16, scales=(4.0, 8.0, 16.0, 32.0), ratios=(0.5, 1.0, 2.0),
                feature_stride=16, output_score=False, iou_loss=False, is_train=False):
    """mx.sym.contrib.Proposal_v3 with the op's own defaults (proposal_v3-inl.h:141-183).
    Returns rois (B,post,4) — and scores (B,post,1) when output_score — exactly the visible
    outputs of the reference op."""
    cls_prob, bbox_pred, im_info = _dev(cls_prob, "cls_prob"), _dev(bbox_pred, "bbox_pred"), _dev(im_info, "im_info")
    if cls_prob.dim() != 4 or cls_prob.shape[1] % 2:
        raise ValueError("cls_prob must be (B,2A,H,W)")
    B, A2, H, W = cls_prob.shape
    A = A2 // 2
    if tuple(bbox_pred.shape) != (B, 4 * A, H, W):
        raise ValueError("bbox_pred must be (B,4A,H,W)")
    if im_info.shape != (B, 3):
        raise ValueError("im_info must be (B,3)")
    count = A * H * W
    pre = min(rpn_pre_nms_top_n if rpn_pre_nms_top_n > 0 else count, count)
    post = rpn_post_nms_top_n if not is_train else min(rpn_post_nms_top_n, pre)
    out = torch.empty((B, post, 4), device=cls_prob.device, dtype=torch.float32)
    score = torch.empty((B, post, 1), device=cls_prob.device, dtype=torch.float32)
    L = _lib.lib()
    nbytes = L.sdet_proposal_v3_workspace(B, A, H, W, int(rpn_pre_nms_top_n))
    ws = _ws(nbytes, cls_prob.device)
    sc = (ctypes.c_float * len(scales))(*[float(x) for x in scales])
    ra = (ctypes.c_float * len(ratios))(*[float(x) for x in ratios])
    check(L.sdet_proposal_v3(_p(cls_prob), _p(bbox_pred), _p(im_info), _p(out), _p(score), B, A, H, W,
                             int(feature_stride), sc, len(scales), ra, len(ratios),
                             int(rpn_pre_nms_top_n), int(rpn_post_nms_top_n), float(threshold),
                             int(rpn_min_size), int(bool(iou_loss)), int(bool(is_train)), _p(ws), nbytes,
                             _stream()))
    return (out, score) if output_score else out


def _proposal_legacy(version, cls_prob, bbox_pred, im_info, valid_ranges, rpn_pre_nms_top_n, rpn_post_nms_top_n,
                     threshold, rpn_min_size, scales, ratios, feature_stride, output_score, iou_loss, is_train,
                     filter_scales):
    cls_prob, bbox_pred, im_info = _dev(cls_prob, "cls_prob"), _dev(bbox_pred, "bbox_pred"), _dev(im_info, "im_info")
    valid_ranges = _dev(valid_ranges, "valid_ranges")
    B, A2, H, W = cls_prob.shape
    A = A2 // 2
    if tuple(bbox_pred.shape) != (B, 4 * A, H, W):
        raise ValueError("bbox_pred must be (B,4A,H,W)")
    count = A * H * W
    pre = min(rpn_pre_nms_top_n if rpn_pre_nms_top_n > 0 else count, count)
    post = min(rpn_post_nms_top_n, pre)
    if version == 1 and not is_train:
        post = rpn_post_nms_top_n
    out = torch.empty((B, post, 4), device=cls_prob.device, dtype=torch.float32)
    score = torch.empty((B, post, 1), device=cls_prob.device, dtype=torch.float32)
    L = _lib.lib()
    nbytes = L.sdet_proposal_legacy_workspace(B, A, H, W, int(rpn_pre_nms_top_n))
    ws = _ws(nbytes, cls_prob.device)
    sc = (ctypes.c_float * len(scales))(*[float(x) for x in scales])
    ra = (ctypes.c_float * len(ratios))(*[float(x) for x in ratios])
    check(L.sdet_proposal_legacy(_p(cls_prob), _p(bbox_pred), _p(im_info), _p(valid_ranges), version, _p(out),
                                 _p(score), B, A, H, W, int(feature_stride), sc, len(scales), ra, len(ratios),
                                 int(rpn_pre_nms_top_n), int(rpn_post_nms_top_n), float(threshold),
                                 int(rpn_min_size), int(bool(iou_loss)), int(bool(is_train)),
                                 int(bool(filter_scales)), _p(ws), nbytes, _stream()))
    return (out, score) if output_score else out


def Proposal(cls_prob, bbox_pred, im_info, rpn_pre_nms_top_n=6000, rpn_post_nms_top_n=300, threshold=0.7,
             rpn_min_size=16, scales=(4.0, 8.0, 16.0, 32.0), ratios=(0.5, 1.0, 2.0), feature_stride=16,
             output_score=False, iou_loss=False, is_train=False):
    """mx.sym.contrib.Proposal / X.proposal (symbol/builder.py:241-255): the legacy RPN proposal op."""
    return _proposal_legacy(1, cls_prob, bbox_pred, im_info, None, rpn_pre_nms_top_n, rpn_post_nms_top_n, threshold,
                            rpn_min_size, scales, ratios, feature_stride, output_score, iou_loss, is_train, False)


def Proposal_v2(cls_prob, bbox_pred, im_info, valid_ranges, rpn_pre_nms_top_n=6000, rpn_post_nms_top_n=300,
                threshold=0.7, rpn_min_size=16, scales=(4.0, 8.0, 16.0, 32.0), ratios=(0.5, 1.0, 2.0),
                feature_stride=16, output_score=False, iou_loss=False, filter_scales=False):
    """mx.sym.contrib.Proposal_v2 (TridentNet, models/tridentnet/builder.py:239): Proposal + valid_ranges."""
    return _proposal_legacy(2, cls_prob, bbox_pred, im_info, valid_ranges, rpn_pre_nms_top_n, rpn_post_nms_top_n,
                            threshold, rpn_min_size, scales, ratios, feature_stride, output_score, iou_loss, False,
                            filter_scales)


def GenAnchor(cls_prob, scales=(4.0, 8.0, 16.0, 32.0), ratios=(0.5, 1.0, 2.0), feature_stride=16):
    """mx.sym.contrib.GenAnchor (models/retinanet/builder.py:365): only cls_prob's (H, W) is used."""
    cls_prob = _dev(cls_prob, "cls_prob")
    H, W = int(cls_prob.shape[2]), int(cls_prob.shape[3])
    A = len(scales) * len(ratios)
    out = torch.empty((H * W * A, 4), device=cls_prob.device, dtype=torch.float32)
    sc = (ctypes.c_double * len(scales))(*[float(x) for x in scales])
    ra = (ctypes.c_double * len(ratios))(*[float(x) for x in ratios])
    check(_lib.lib().sdet_gen_anchor(_p(out), H, W, int(feature_stride), sc, len(scales), ra, len(ratios), _stream()))
    return out


def GenProposal(cls_prob, bbox_pred, im_info, anchors, rpn_pre_nms_top_n=6000, rpn_min_size=16, feature_stride=16,
                iou_loss=False):
    """mx.sym.contrib.GenProposal (generate_proposal.cu): sorted pre-NMS proposals (B, pre, 5), no NMS."""
    cls_prob, bbox_pred, im_info = _dev(cls_prob, "cls_prob"), _dev(bbox_pred, "bbox_pred"), _dev(im_info, "im_info")
    anchors = _dev(anchors, "anchors")
    B, A2, H, W = cls_prob.shape
    A = A2 // 2
    if tuple(bbox_pred.shape) != (B, 4 * A, H, W) or anchors.numel() != H * W * A * 4:
        raise ValueError("bbox_pred must be (B,4A,H,W) and anchors (H*W*A,4)")
    out = torch.empty((B, int(rpn_pre_nms_top_n), 5), device=cls_prob.device, dtype=torch.float32)
    L = _lib.lib()
    nbytes = L.sdet_gen_proposal_workspace(B, A, H, W, int(rpn_pre_nms_top_n))
    ws = _ws(nbytes, cls_prob.device)
    check(L.sdet_gen_proposal(_p(cls_prob), _p(bbox_pred), _p(im_info), _p(anchors), _p(out), B, A, H, W,
                              int(feature_stride), int(rpn_pre_nms_top_n), int(rpn_min_size), int(bool(iou_loss)),
                              _p(ws), nbytes, _stream()))
    return out


def GenProposalRetina(cls_prob, bbox_pred, im_info, anchors, num_anchors, feature_stride=16, rpn_pre_nms_top_n=6000,
                      rpn_min_size=16, thresh=0.0, anchor_mean=(0.0, 0.0, 0.0, 0.0), anchor_std=(1.0, 1.0, 1.0, 1.0),
                      iou_loss=False, output_one_hot=True, batch_wise_anchor=False, workspace=None):
    """mx.sym.contrib.GenProposalRetina (models/retinanet/builder.py:374-387) -> (bbox_xyxy, cls_score)."""
    cls_prob, bbox_pred, im_info = _dev(cls_prob, "cls_prob"), _dev(bbox_pred, "bbox_pred"), _dev(im_info, "im_info")
    anchors = _dev(anchors, "anchors")
    B, AK, H, W = cls_prob.shape
    if AK % num_anchors:
        raise ValueError("cls_prob channels must be a multiple of num_anchors")
    if tuple(bbox_pred.shape) != (B, 4 * num_anchors, H, W):
        raise ValueError("bbox_pred must be (B, 4*num_anchors, H, W)")
    K = AK // num_anchors
    oc = K + 1 if output_one_hot else 1
    pre = int(rpn_pre_nms_top_n)
    out = torch.empty((B, pre, 4), device=cls_prob.device, dtype=torch.float32)
    score = torch.empty((B, pre, oc), device=cls_prob.device, dtype=torch.float32)
    L = _lib.lib()
    nbytes = L.sdet_gen_proposal_retina_workspace(B, AK, H, W)
    ws = _ws(nbytes, cls_prob.device)
    m = (ctypes.c_float * 4)(*[float(x) for x in anchor_mean])
    sd = (ctypes.c_float * 4)(*[float(x) for x in anchor_std])
    check(L.sdet_gen_proposal_retina(_p(cls_prob), _p(bbox_pred), _p(im_info), _p(anchors), _p(out), _p(score), B, AK,
                                     H, W, int(num_anchors), int(feature_stride), pre, int(rpn_min_size),
                                     float(thresh), m, sd, int(bool(iou_loss)), int(bool(output_one_hot)),
                                     int(bool(batch_wise_anchor)), _p(ws), nbytes, _stream()))
    return out, score


def Proposal_v3_fpn(cls_probs, bbox_preds, im_info, feature_strides, rpn_pre_nms_top_n=6000,
                    rpn_post_nms_top_n=300, threshold=0.7, rpn_min_size=16, scales=(4.0, 8.0, 16.0, 32.0),
                    ratios=(0.5, 1.0, 2.0), iou_loss=False, is_train=False):
    """All FPN levels at once: [Proposal_v3(level) for level in strides] + Concat(dim=1), exactly
    FPNRpnHead.get_all_proposal (models/FPN/builder.py:267-317).  -> (rois (B,L*post,4),
    scores (B,L*post,1)), level-major."""
    L_ = len(cls_probs)
    cls_probs = [_dev(c, f"cls_prob[{i}]") for i, c in enumerate(cls_probs)]
    bbox_preds = [_dev(c, f"bbox_pred[{i}]") for i, c in enumerate(bbox_preds)]
    im_info = _dev(im_info, "im_info")
    B, A2 = cls_probs[0].shape[:2]
    A = A2 // 2
    for c, d in zip(cls_probs, bbox_preds):
        if c.dim() != 4 or c.shape[0] != B or c.shape[1] != A2 or tuple(d.shape) != (B, 4 * A, c.shape[2], c.shape[3]):
            raise ValueError("each level needs cls_prob (B,2A,H,W) and bbox_pred (B,4A,H,W)")
    pres = [min(rpn_pre_nms_top_n if rpn_pre_nms_top_n > 0 else A * c.shape[2] * c.shape[3],
                A * c.shape[2] * c.shape[3]) for c in cls_probs]
    # is_train: a level writes min(post, its pre) rows; equal levels shrink the output, unequal ones keep `post` rows
    # per level with zero rows after what a small level (P6) can fill - sdet_proposal_v3_fpn's rule
    post = rpn_post_nms_top_n if (not is_train or min(pres) != max(pres)) else min(rpn_post_nms_top_n, min(pres))
    dev = cls_probs[0].device
    out = torch.empty((B, L_ * post, 4), device=dev, dtype=torch.float32)
    score = torch.empty((B, L_ * post, 1), device=dev, dtype=torch.float32)
    cp = (ctypes.c_void_p * L_)(*[c.data_ptr() for c in cls_probs])
    bp = (ctypes.c_void_p * L_)(*[c.data_ptr() for c in bbox_preds])
    Hs = (ctypes.c_int * L_)(*[c.shape[2] for c in cls_probs])
    Ws = (ctypes.c_int * L_)(*[c.shape[3] for c in cls_probs])
    Ss = (ctypes.c_int * L_)(*[int(s) for s in feature_strides])
    sc = (ctypes.c_float * len(scales))(*[float(x) for x in scales])
    ra = (ctypes.c_float * len(ratios))(*[float(x) for x in ratios])
    Lb = _lib.lib()
    nbytes = Lb.sdet_proposal_v3_fpn_workspace(B, A, Hs, Ws, L_, int(rpn_pre_nms_top_n))
    ws = _ws(nbytes, dev)
    check(Lb.sdet_proposal_v3_fpn(cp, bp, _p(im_info), _p(out), _p(score), B, A, Hs, Ws, Ss, L_, sc, len(scales),
                                  ra, len(ratios), int(rpn_pre_nms_top_n), int(rpn_post_nms_top_n),
                                  float(threshold), int(rpn_min_size), int(bool(iou_loss)), int(bool(is_train)),
                                  _p(ws), nbytes, _stream()))
    return out, score


# --------------------------------------------------------------------------------------------
# _contrib_NMS  (operator_cxx/contrib/nms.cu:274-364)
# --------------------------------------------------------------------------------------------
def NMS(data, rpn_pre_nms_top_n=6000, rpn_post_nms_top_n=300, threshold=0.7, output_score=False,
        already_sorted=False):
    """mx.sym.contrib.NMS: data (B,count,5) -> rois (B,post,4) [, scores (B,post,1)].  Rows past
    min(post, pre) are never written by the reference; they are zero here."""
    data = _dev(data, "data")
    if data.dim() != 3 or data.shape[2] != 5:
        raise ValueError("data must be (B,count,5)")
    B, count, _ = data.shape
    out = torch.zeros((B, rpn_post_nms_top_n, 4), device=data.device, dtype=torch.float32)
    score = torch.zeros((B, rpn_post_nms_top_n, 1), device=data.device, dtype=torch.float32)
    L = _lib.lib()
    nbytes = L.sdet_contrib_nms_workspace(B, count, int(rpn_pre_nms_top_n))
    ws = _ws(nbytes, data.device)
    check(L.sdet_contrib_nms(_p(data), _p(out), _p(score), B, count, int(rpn_pre_nms_top_n),
                             int(rpn_post_nms_top_n), float(threshold), int(bool(already_sorted)), _p(ws),
                             nbytes, _stream()))
    return (out, score) if output_score else out


def nms_sorted(dets, thresh, ge=True, counts=None):
    """Batched greedy NMS over boxes already sorted by descending score.
    dets (P,n,5) -> keep (P,n) int32 (kept positions, zero padded), nkeep (P) int32."""
    dets = _dev(dets, "dets")
    if dets.dim() != 3 or dets.shape[2] != 5:
        raise ValueError("dets must be (P,n,5)")
    P, n, _ = dets.shape
    counts = _dev(counts, "counts", torch.int32)
    keep = torch.empty((P, n), device=dets.device, dtype=torch.int32)
    nkeep = torch.empty((P,), device=dets.device, dtype=torch.int32)
    L = _lib.lib()
    nbytes = L.sdet_nms_workspace(P, n)
    ws = _ws(nbytes, dets.device)
    check(L.sdet_nms_sorted(_p(dets), _p(counts), P, n, float(thresh), int(bool(ge)), _p(keep), _p(nkeep),
                            _p(ws), nbytes, _stream()))
    return keep, nkeep


def set_nms(dets, thresh):
    """operator_py/nms.py set_nms: dets (m,6) rows [x1,y1,x2,y2,score,set] on the device -> kept rows."""
    dets = _dev(dets, "dets")
    if dets.dim() != 2 or dets.shape[1] != 6:
        raise ValueError("dets must be (m,6)")
    if dets.shape[0] == 0:
        return dets
    order = torch.sort(dets[:, 4], descending=True, stable=True).indices
    srt = dets[order].contiguous()
    boxes, sets = srt[:, :5].contiguous()[None], srt[:, 5].contiguous()[None]
    n = int(srt.shape[0])
    keep = torch.empty((1, n), device=dets.device, dtype=torch.int32)
    nkeep = torch.empty((1,), device=dets.device, dtype=torch.int32)
    L = _lib.lib()
    nbytes = L.sdet_nms_workspace(1, n)
    ws = _ws(nbytes, dets.device)
    check(L.sdet_set_nms_sorted(_p(boxes), _p(sets), None, 1, n, float(thresh), _p(keep), _p(nkeep), _p(ws), nbytes,
                                _stream()))
    return srt[keep[0, :int(nkeep.item())].long()]


def py_weighted_nms(dets, thresh_lo, thresh_hi):
    """operator_py/nms.py py_weighted_nms: dets (m,5) -> (m',5) voted boxes with the top boxes' scores."""
    dets = _dev(dets, "dets")
    if dets.dim() != 2 or dets.shape[1] != 5:
        raise ValueError("dets must be (m,5)")
    if dets.shape[0] == 0:
        return dets
    order = torch.sort(dets[:, 4], descending=True, stable=True).indices
    srt = dets[order].contiguous()[None]
    n = int(srt.shape[1])
    out = torch.empty((1, n, 5), device=dets.device, dtype=torch.float32)
    nout = torch.empty((1,), device=dets.device, dtype=torch.int32)
    L = _lib.lib()
    nbytes = L.sdet_weighted_nms_workspace(1, n)
    ws = _ws(nbytes, dets.device)
    check(L.sdet_weighted_nms_sorted(_p(srt), None, 1, n, float(thresh_lo), float(thresh_hi), _p(out), _p(nout),
                                     _p(ws), nbytes, _stream()))
    return out[0, :int(nout.item())]


def py_set_nms_wrapper(thresh):
    return lambda dets: set_nms(dets, thresh)


def wnms_wrapper(thresh_lo, thresh_hi):
    return lambda dets: py_weighted_nms(dets, thresh_lo, thresh_hi)


# --------------------------------------------------------------------------------------------
# ProposalTarget  (operator_cxx/proposal_target-inl.h:81-114 params; X.proposal_target at
# models/FPN/builder.py:347-363)
# --------------------------------------------------------------------------------------------
_PT_CALLS = [0]


def ProposalTarget(rois, gt_boxes, num_classes, batch_images, image_rois, fg_thresh, bg_thresh_hi,
                   bg_thresh_lo, proposal_without_gt, fg_fraction=0.25, class_agnostic=False,
                   output_iou=False, bbox_mean=(0.0, 0.0, 0.0, 0.0), bbox_std=(0.1, 0.1, 0.2, 0.2),
                   bbox_weight=(1.0, 1.0, 1.0, 1.0), seed=None, priorities=None, num_draws=8,
                   return_debug=False, _match_out=None):
    """mx.sym.ProposalTarget.  rois (B,R,4), gt_boxes (B,G,5) -> rois (B,IR,4), label (B,IR),
    bbox_target (B,IR,4*num_classes), bbox_weight (same) [, match_gt_iou (B,IR) if output_iou].
    `seed` (int) keys the on-device Philox sampling (default: a per-process call counter);
    `priorities` (B,D,R+G) uint32-in-int32/int64 tensor injects the shuffles instead.
    return_debug adds (kept (B,IR) int32, priorities_used (B,D,R+G) int32 bit patterns)."""
    rois, gt_boxes = _dev(rois, "rois"), _dev(gt_boxes, "gt_boxes")
    B = int(batch_images)
    R = rois.numel() // (B * 4)       # -inl.h:139-140: shapes are re-derived from batch_images
    G = gt_boxes.numel() // (B * 5)
    IR = int(image_rois)
    if IR <= 0:
        raise ValueError("image_rois must be > 0 (ProposalTarget_v2 handles -1)")
    dev = rois.device
    NC4 = 4 * int(num_classes)
    o_rois = torch.empty((B, IR, 4), device=dev, dtype=torch.float32)
    o_lab = torch.empty((B, IR), device=dev, dtype=torch.float32)
    o_tgt = torch.empty((B, IR, NC4), device=dev, dtype=torch.float32)
    o_wgt = torch.empty((B, IR, NC4), device=dev, dtype=torch.float32)
    o_iou = torch.empty((B, IR), device=dev, dtype=torch.float32)
    kept = torch.empty((B, IR), device=dev, dtype=torch.int32) if return_debug else None
    T = R + G
    if priorities is not None:
        priorities = priorities.to(device=dev, dtype=torch.int64).contiguous()
        if priorities.shape[0] != B or priorities.shape[2] != T:
            raise ValueError("priorities must be (B, D, R+G)")
        num_draws = priorities.shape[1]
        priorities = (priorities & 0xFFFFFFFF).to(torch.int64)
        priorities = torch.where(priorities >= 2 ** 31, priorities - 2 ** 32, priorities).to(torch.int32).contiguous()
    used = torch.zeros((B, num_draws, T), device=dev, dtype=torch.int32) if return_debug else None
    if seed is None:
        _PT_CALLS[0] += 1
        seed = 0x5DE7B200 + _PT_CALLS[0]
    check(_lib.lib().sdet_proposal_target(
        _p(rois), _p(gt_boxes), _p(o_rois), _p(o_lab), _p(o_tgt), _p(o_wgt), _p(o_iou), _p(kept), B, R, G,
        int(num_classes), IR, float(fg_fraction), float(fg_thresh), float(bg_thresh_hi), float(bg_thresh_lo),
        int(bool(proposal_without_gt)), int(bool(class_agnostic)), _f4(bbox_mean, "bbox_mean"),
        _f4(bbox_std, "bbox_std"), _f4(bbox_weight, "bbox_weight"), int(seed) & (2 ** 64 - 1), _p(priorities),
        int(num_draws), _p(used), _p(_match_out[0]) if _match_out else None,
        _p(_match_out[1]) if _match_out else None, _stream()))
    outs = [o_rois, o_lab, o_tgt, o_wgt]
    if output_iou:
        outs.append(o_iou)
    if return_debug:
        outs += [o_iou, kept, used]
    return tuple(outs)


# --------------------------------------------------------------------------------------------
# _contrib_FocalLoss / _contrib_BBoxNorm / _contrib_SigmoidCrossEntropy
# --------------------------------------------------------------------------------------------
_NORM = {"null": 0, "batch": 1, "valid": 2}


class _FocalLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, data, label, alpha, gamma, normalization, grad_scale, out_grad):
        data, label = _dev(data, "data"), _dev(label, "label")
        out = torch.empty_like(data)
        check(_lib.lib().sdet_focal_loss_forward(_p(data), _p(out), data.numel(), _stream()))
        ctx.save_for_backward(out, label)
        ctx.cfg = (alpha, gamma, normalization, grad_scale, out_grad)
        return out

    @staticmethod
    def backward(ctx, ograd):
        out, label = ctx.saved_tensors
        alpha, gamma, normalization, grad_scale, use_og = ctx.cfg
        B, N, K = out.shape
        g = torch.empty_like(out)
        og = _dev(ograd, "ograd") if use_og else None
        ws = _ws(16, out.device)
        check(_lib.lib().sdet_focal_loss_backward(_p(out), _p(label), _p(og), _p(g), B, N, K, float(alpha),
                                                  float(gamma), float(grad_scale), _NORM[normalization], _p(ws),
                                                  16, _stream()))
        return g, None, None, None, None, None, None


def FocalLoss(data, label, alpha=0.25, gamma=2.0, normalization="null", grad_scale=1.0, out_grad=False,
              workspace=256):
    """mx.sym.contrib.FocalLoss / X.focal_loss: data (B,N,K) logits, label (B,N) -> sigmoid(data);
    the loss gradient is produced in backward like the reference (the incoming gradient is
    ignored unless out_grad=True).  `workspace` is accepted and unused (no temporaries)."""
    if data.dim() != 3 or label.shape != data.shape[:2]:
        raise ValueError("data must be (B,N,K) and label (B,N)")
    return _FocalLossFn.apply(data, label, float(alpha), float(gamma), normalization, float(grad_scale),
                              bool(out_grad))


class _BBoxNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, data, label):
        ctx.save_for_backward(label)
        return data.clone()  # Assign(out, identity(data)), bbox_norm-inl.h:96

    @staticmethod
    def backward(ctx, gout):
        (label,) = ctx.saved_tensors
        gout, label = _dev(gout, "gout"), _dev(label, "label")
        g = torch.empty_like(gout)
        ws = _ws(16, gout.device)
        check(_lib.lib().sdet_bbox_norm_backward(_p(gout), _p(label), _p(g), gout.numel(), label.numel(), _p(ws),
                                                 16, _stream()))
        return g, None


def BBoxNorm(data, label, normalization="valid"):
    """mx.sym.contrib.BBoxNorm / X.bbox_norm: identity forward; backward divides the gradient by
    max(sum(label >= 1) + 1, 1) (the reference ignores `normalization` in Backward too)."""
    return _BBoxNormFn.apply(data, label)


class _SigmoidCEFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, data, label, grad_scale):
        data, label = _dev(data, "data"), _dev(label, "label")
        R, D = data.shape
        out = torch.empty((R,), device=data.device, dtype=torch.float32)
        ws = _ws(8 * R, data.device)
        check(_lib.lib().sdet_sigmoid_ce_forward(_p(data), _p(label), _p(out), R, D, _p(ws), 8 * R, _stream()))
        ctx.save_for_backward(data, label)
        ctx.scale = grad_scale
        return out

    @staticmethod
    def backward(ctx, ograd):
        data, label = ctx.saved_tensors
        R, D = data.shape
        g = torch.empty_like(data)
        ws = _ws(8 * R, data.device)
        check(_lib.lib().sdet_sigmoid_ce_backward(_p(data), _p(label), _p(g), R, D, float(ctx.scale), _p(ws), 8 * R,
                                                  _stream()))
        return g, None, None


def SigmoidCrossEntropy(data, label, grad_scale=1.0):
    """mx.sym.contrib.SigmoidCrossEntropy: data, label (R,D), label -1 ignored -> loss (R,)."""
    if data.dim() != 2 or data.shape != label.shape:
        raise ValueError("data and label must both be (R,D)")
    return _SigmoidCEFn.apply(data, label, float(grad_scale))


def ProposalTarget_v2(rois, gt_boxes, valid_ranges, num_classes, batch_images, image_rois, fg_thresh, bg_thresh_hi,
                      bg_thresh_lo, proposal_without_gt, fg_fraction=0.25, class_agnostic=False, output_iou=False,
                      filter_scales=False, bbox_mean=(0.0, 0.0, 0.0, 0.0), bbox_std=(0.1, 0.1, 0.2, 0.2),
                      bbox_weight=(1.0, 1.0, 1.0, 1.0), seed=None, priorities=None, num_draws=8, return_debug=False,
                      _match_out=None):
    """mx.sym.ProposalTarget_v2 (TridentNet): ProposalTarget + valid_ranges (B,2) / filter_scales,
    and image_rois = -1 to keep every foreground roi (R rows per image)."""
    rois, gt_boxes = _dev(rois, "rois"), _dev(gt_boxes, "gt_boxes")
    valid_ranges = _dev(valid_ranges, "valid_ranges")
    B = int(batch_images)
    R = rois.numel() // (B * 4)
    G = gt_boxes.numel() // (B * 5)
    IR = R if int(image_rois) == -1 else int(image_rois)
    dev = rois.device
    NC4 = 4 * int(num_classes)
    o_rois = torch.empty((B, IR, 4), device=dev, dtype=torch.float32)
    o_lab = torch.empty((B, IR), device=dev, dtype=torch.float32)
    o_tgt = torch.empty((B, IR, NC4), device=dev, dtype=torch.float32)
    o_wgt = torch.empty((B, IR, NC4), device=dev, dtype=torch.float32)
    o_iou = torch.empty((B, IR), device=dev, dtype=torch.float32)
    kept = torch.empty((B, IR), device=dev, dtype=torch.int32) if return_debug else None
    T = R + G
    if priorities is not None:
        priorities = priorities.to(device=dev, dtype=torch.int64).contiguous()
        num_draws = priorities.shape[1]
        priorities = (priorities & 0xFFFFFFFF)
        priorities = torch.where(priorities >= 2 ** 31, priorities - 2 ** 32, priorities).to(torch.int32).contiguous()
    if seed is None:
        _PT_CALLS[0] += 1
        seed = 0x5DE7B200 + _PT_CALLS[0]
    check(_lib.lib().sdet_proposal_target_v2(
        _p(rois), _p(gt_boxes), _p(valid_ranges), _p(o_rois), _p(o_lab), _p(o_tgt), _p(o_wgt), _p(o_iou), _p(kept), B,
        R, G, int(num_classes), int(image_rois), float(fg_fraction), float(fg_thresh), float(bg_thresh_hi),
        float(bg_thresh_lo), int(bool(proposal_without_gt)), int(bool(class_agnostic)), int(bool(filter_scales)),
        _f4(bbox_mean, "bbox_mean"), _f4(bbox_std, "bbox_std"), _f4(bbox_weight, "bbox_weight"),
        int(seed) & (2 ** 64 - 1), _p(priorities), int(num_draws), None,
        _p(_match_out[0]) if _match_out else None, _p(_match_out[1]) if _match_out else None, _stream()))
    outs = [o_rois, o_lab, o_tgt, o_wgt]
    if output_iou or return_debug:
        outs.append(o_iou)
    if return_debug:
        outs.append(kept)
    return tuple(outs)


def ProposalMaskTarget(rois, gt_boxes, gt_polys, num_classes, batch_images, image_rois, mask_size, fg_thresh,
                       bg_thresh_hi, bg_thresh_lo, proposal_without_gt, fg_fraction=0.25, class_agnostic=False,
                       output_iou=False, output_ratio=False, filter_scales=False, num_args=3,
                       bbox_mean=(0.0, 0.0, 0.0, 0.0), bbox_std=(0.1, 0.1, 0.2, 0.2),
                       bbox_weight=(1.0, 1.0, 1.0, 1.0), seed=None, priorities=None, valid_ranges=None):
    """mx.sym.ProposalMaskTarget (models/maskrcnn/builder.py:184-203): ProposalTarget's outputs +
    mask_target (B, int(image_rois*fg_fraction), M, M) with -1 = ignore.  filter_scales=True takes the
    4th input valid_ranges (B,2) (models/tridentnet/builder.py:377-398): gt boxes outside the range are
    not appended to the candidates (proposal_mask_target-inl.h:222-229).  output_ratio=True (Mask Scoring R-CNN,
    models/msrcnn/builder.py:219-239) appends mask_ratio (B, int(image_rois*fg_fraction)): the share of the
    instance's polygon area that lies inside the roi (convertPoly2MaskWithRatio, proposal_mask_target.cc:20-152)."""
    if filter_scales and valid_ranges is None:
        raise ValueError("filter_scales=True needs valid_ranges (B,2)")
    del num_args
    gt_polys = _dev(gt_polys, "gt_polys")
    B = int(batch_images)
    IR = int(image_rois)
    G = gt_boxes.numel() // (B * 5)
    PL = gt_polys.numel() // (B * G)
    dev = rois.device
    gt_index = torch.empty((B, IR), device=dev, dtype=torch.int32)
    fg_count = torch.empty((B,), device=dev, dtype=torch.int32)
    common = dict(fg_fraction=fg_fraction, class_agnostic=class_agnostic, output_iou=output_iou, bbox_mean=bbox_mean,
                  bbox_std=bbox_std, bbox_weight=bbox_weight, seed=seed, priorities=priorities,
                  _match_out=(gt_index, fg_count))
    if filter_scales:
        outs = ProposalTarget_v2(rois, gt_boxes, valid_ranges, num_classes, B, IR, fg_thresh, bg_thresh_hi,
                                 bg_thresh_lo, proposal_without_gt, filter_scales=True, **common)
    else:
        outs = ProposalTarget(rois, gt_boxes, num_classes, B, IR, fg_thresh, bg_thresh_hi, bg_thresh_lo,
                              proposal_without_gt, **common)
    NM = int(IR * fg_fraction)
    M = int(mask_size)
    mask = torch.empty((B, NM, M, M), device=dev, dtype=torch.float32)
    if output_ratio:
        ratio = torch.empty((B, NM), device=dev, dtype=torch.float32)
        check(_lib.lib().sdet_poly_mask_target_ratio(_p(outs[0]), _p(gt_polys), _p(gt_index), _p(fg_count), _p(mask),
                                                     _p(ratio), B, IR, G, PL, NM, M, _stream()))
        return tuple(outs) + (mask, ratio)
    check(_lib.lib().sdet_poly_mask_target(_p(outs[0]), _p(gt_polys), _p(gt_index), _p(fg_count), _p(mask), B, IR, G,
                                           PL, NM, M, _stream()))
    return tuple(outs) + (mask,)


# --------------------------------------------------------------------------------------------
# _contrib_DeformableConvolution (DCNv1; models/dcn/builder.py:14-17)
# --------------------------------------------------------------------------------------------
class _DeformConvFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, data, offset, weight, bias, geo):
        kh, kw, ph_, pw_, sh, sw, dh, dw, ng, dg = geo
        data, offset, weight = _dev_any_layout(data, "data"), _dev(offset, "offset"), _dev(weight, "weight")
        B, C, H, W = data.shape
        F = weight.shape[0]
        Ho = (H + 2 * ph_ - (dh * (kh - 1) + 1)) // sh + 1
        Wo = (W + 2 * pw_ - (dw * (kw - 1) + 1)) // sw + 1
        if tuple(offset.shape) != (B, dg * 2 * kh * kw, Ho, Wo):
            raise ValueError(f"offset must be {(B, dg * 2 * kh * kw, Ho, Wo)}, got {tuple(offset.shape)}")
        P, T = Ho * Wo, kh * kw
        if ng == 1 and (C // dg) % 2 == 0:
            # channels-last: sample into col_t (B, P, T*C), contract with W'[(tap, c)][f]; input and output stay NHWC
            # in memory (the tensors handed back are NCHW-shaped views, torch's channels_last format)
            x = data.permute(0, 2, 3, 1)
            if not x.is_contiguous():
                x = x.contiguous()  # NCHW-contiguous input: one re-layout pass
            col_t = torch.empty((B, P, T * C), device=data.device, dtype=torch.float32)
            check(_lib.lib().sdet_deformable_im2col_nhwc(_p(x), _p(offset), _p(col_t), B, C, H, W, kh, kw, ph_, pw_,
                                                         sh, sw, dh, dw, dg, _stream()))
            wp = weight.permute(2, 3, 1, 0).reshape(T * C, F)
            out = torch.matmul(col_t, wp)  # library GEMM (cuBLAS via torch)
            if bias is not None:
                out = out + bias.view(1, 1, F)
            ctx.save_for_backward(data, offset, weight, col_t)
            ctx.geo, ctx.has_bias, ctx.cl = geo, bias is not None, True
            return out.view(B, Ho, Wo, F).permute(0, 3, 1, 2)
        data = data.contiguous()
        col = torch.empty((B, C * kh * kw, Ho * Wo), device=data.device, dtype=torch.float32)
        check(_lib.lib().sdet_deformable_im2col(_p(data), _p(offset), _p(col), B, C, H, W, kh, kw, ph_, pw_, sh,
                                                sw, dh, dw, dg, _stream()))
        # dense contraction: library GEMM (cuBLAS via torch), grouped like the reference's num_group
        wg = weight.reshape(ng, F // ng, (C // ng) * kh * kw)
        cg = col.reshape(B, ng, (C // ng) * kh * kw, Ho * Wo)
        out = torch.einsum("gfk,bgkp->bgfp", wg, cg).reshape(B, F, Ho, Wo)
        if bias is not None:
            out = out + bias.view(1, F, 1, 1)
        ctx.save_for_backward(data, offset, weight, col)
        ctx.geo, ctx.has_bias, ctx.cl = geo, bias is not None, False
        return out

    @staticmethod
    def backward(ctx, gout):
        data, offset, weight, col = ctx.saved_tensors
        kh, kw, ph_, pw_, sh, sw, dh, dw, ng, dg = ctx.geo
        B, C, H, W = data.shape
        F = weight.shape[0]
        gout = gout if gout.is_cuda else _dev(gout, "gout")
        P = gout.shape[2] * gout.shape[3]
        data, offset = data.contiguous(), offset.contiguous()
        if ctx.cl:
            T = kh * kw
            go = gout.permute(0, 2, 3, 1).reshape(B, P, F)
            wp = weight.permute(2, 3, 1, 0).reshape(T * C, F)
            gcol_t = torch.matmul(go, wp.t())                                    # (B, P, T*C)
            gcol = gcol_t.view(B, P, T, C).permute(0, 3, 2, 1).reshape(B, C * T, P).contiguous()
            gweight = torch.einsum("bpk,bpf->kf", col, go).view(kh, kw, C, F).permute(3, 2, 0, 1).contiguous()
        else:
            gout = gout.contiguous()
            go = gout.reshape(B, ng, F // ng, P)
            wg = weight.reshape(ng, F // ng, (C // ng) * kh * kw)
            gcol = torch.einsum("gfk,bgfp->bgkp", wg, go).reshape(B, C * kh * kw, P).contiguous()
            gweight = torch.einsum("bgfp,bgkp->gfk", go, col.reshape(B, ng, (C // ng) * kh * kw, P)).reshape(weight.shape)
        gdata = torch.empty_like(data)
        goff = torch.empty_like(offset)
        check(_lib.lib().sdet_deformable_col2im(_p(gcol), _p(data), _p(offset), _p(gdata), _p(goff), B, C, H, W, kh,
                                                kw, ph_, pw_, sh, sw, dh, dw, dg, _stream()))
        gbias = gout.sum((0, 2, 3)) if ctx.has_bias else None
        return gdata, goff, gweight, gbias, None


def DeformableConvolution(data, offset, weight, bias=None, kernel=(3, 3), stride=(1, 1), dilate=(1, 1),
                          pad=(0, 0), num_filter=None, num_group=1, num_deformable_group=1, no_bias=False):
    """mx.sym.contrib.DeformableConvolution (DCNv1).  data (B,C,H,W), offset
    (B, 2*KH*KW*num_deformable_group, Ho, Wo), weight (num_filter, C/num_group, KH, KW)."""
    kh, kw = _pair(kernel)
    sh, sw = _pair(stride)
    dh, dw = _pair(dilate)
    ph_, pw_ = _pair(pad)
    if num_filter is not None and weight.shape[0] != num_filter:
        raise ValueError("weight.shape[0] != num_filter")
    geo = (kh, kw, ph_, pw_, sh, sw, dh, dw, int(num_group), int(num_deformable_group))
    return _DeformConvFn.apply(data, offset, weight, None if no_bias else bias, geo)


class _ModDeformConvFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, data, offset, mask, weight, bias, geo):
        kh, kw, ph_, pw_, sh, sw, dh, dw, ng, dg = geo
        data, offset, mask, weight = (_dev(data, "data"), _dev(offset, "offset"), _dev(mask, "mask"),
                                      _dev(weight, "weight"))
        B, C, H, W = data.shape
        F = weight.shape[0]
        Ho = (H + 2 * ph_ - (dh * (kh - 1) + 1)) // sh + 1
        Wo = (W + 2 * pw_ - (dw * (kw - 1) + 1)) // sw + 1
        if tuple(offset.shape) != (B, dg * 2 * kh * kw, Ho, Wo) or tuple(mask.shape) != (B, dg * kh * kw, Ho, Wo):
            raise ValueError("offset must be (B, 2*dg*KH*KW, Ho, Wo) and mask (B, dg*KH*KW, Ho, Wo)")
        col = torch.empty((B, C * kh * kw, Ho * Wo), device=data.device, dtype=torch.float32)
        check(_lib.lib().sdet_modulated_deformable_im2col(_p(data), _p(offset), _p(mask), _p(col), B, C, H, W, kh, kw,
                                                          ph_, pw_, sh, sw, dh, dw, dg, _stream()))
        wg = weight.reshape(ng, F // ng, (C // ng) * kh * kw)
        out = torch.einsum("gfk,bgkp->bgfp", wg, col.reshape(B, ng, (C // ng) * kh * kw, Ho * Wo)).reshape(B, F, Ho, Wo)
        if bias is not None:
            out = out + bias.view(1, F, 1, 1)
        ctx.save_for_backward(data, offset, mask, weight, col)
        ctx.geo, ctx.has_bias = geo, bias is not None
        return out

    @staticmethod
    def backward(ctx, gout):
        data, offset, mask, weight, col = ctx.saved_tensors
        kh, kw, ph_, pw_, sh, sw, dh, dw, ng, dg = ctx.geo
        B, C, H, W = data.shape
        F = weight.shape[0]
        gout = _dev(gout, "gout")
        P = gout.shape[2] * gout.shape[3]
        go = gout.reshape(B, ng, F // ng, P)
        wg = weight.reshape(ng, F // ng, (C // ng) * kh * kw)
        gcol = torch.einsum("gfk,bgfp->bgkp", wg, go).reshape(B, C * kh * kw, P).contiguous()
        gweight = torch.einsum("bgfp,bgkp->gfk", go, col.reshape(B, ng, (C // ng) * kh * kw, P)).reshape(weight.shape)
        gdata, goff, gmask = torch.empty_like(data), torch.empty_like(offset), torch.empty_like(mask)
        check(_lib.lib().sdet_modulated_deformable_col2im(_p(gcol), _p(data), _p(offset), _p(mask), _p(gdata), _p(goff),
                                                          _p(gmask), B, C, H, W, kh, kw, ph_, pw_, sh, sw, dh, dw, dg,
                                                          _stream()))
        gbias = gout.sum((0, 2, 3)) if ctx.has_bias else None
        return gdata, goff, gmask, gweight, gbias, None


def ModulatedDeformableConvolution(data, offset, mask, weight, bias=None, kernel=(3, 3), stride=(1, 1),
                                   dilate=(1, 1), pad=(0, 0), num_filter=None, num_group=1, num_deformable_group=1,
                                   no_bias=False):
    """mx.sym.contrib.ModulatedDeformableConvolution (DCNv2): DeformableConvolution with a per-tap mask
    (B, num_deformable_group*KH*KW, Ho, Wo) — the caller applies the sigmoid, as the upstream models do."""
    kh, kw = _pair(kernel)
    sh, sw = _pair(stride)
    dh, dw = _pair(dilate)
    ph_, pw_ = _pair(pad)
    if num_filter is not None and weight.shape[0] != num_filter:
        raise ValueError("weight.shape[0] != num_filter")
    geo = (kh, kw, ph_, pw_, sh, sw, dh, dw, int(num_group), int(num_deformable_group))
    return _ModDeformConvFn.apply(data, offset, mask, weight, None if no_bias else bias, geo)


# --------------------------------------------------------------------------------------------
# get_top_proposal (models/FPN/get_top_proposal.py) and test-time per-class NMS
# (detection_test.py:233-260 + operator_py/nms.py:41-75)
# --------------------------------------------------------------------------------------------
def get_top_proposal(bbox, score, top_n):
    """CustomOp `get_top_proposal` / mxnext.tvm.get_top_proposal: bbox (B,M,4), score (B,M,1)
    -> (bbox (B,top_n,4), score (B,top_n,1)) sorted by descending score."""
    bbox, score = _dev(bbox, "bbox"), _dev(score, "score")
    B, M, _ = bbox.shape
    if score.shape[:2] != (B, M):
        raise ValueError("score must be (B,M,1)")
    ob = torch.empty((B, top_n, 4), device=bbox.device, dtype=torch.float32)
    os_ = torch.empty((B, top_n, 1), device=bbox.device, dtype=torch.float32)
    check(_lib.lib().sdet_get_top_proposal(_p(bbox), _p(score), _p(ob), _p(os_), B, M, int(top_n), _stream()))
    return ob, os_


def multiclass_nms(cls_score, bbox_xyxy, nms_thresh, min_det_score=0.05, first_class=0):
    """All (image, class) problems of detection_test.py's `do_nms` at once.
    cls_score (B,N,K), bbox_xyxy (B,N,4K) or (B,N,4).
    -> dets (P,n_pad,5) candidates in descending score order, counts (P), keep (P,n_pad), nkeep (P),
       src (P,n_pad) roi index per candidate;  P = B*(K-first_class), problem p = b*(K-fc)+(cid-fc).
    The reference's per-class result is dets[p][keep[p,:nkeep[p]]]."""
    cls_score, bbox_xyxy = _dev(cls_score, "cls_score"), _dev(bbox_xyxy, "bbox_xyxy")
    B, N, K = cls_score.shape
    bd = bbox_xyxy.shape[2]
    P = B * (K - first_class)
    n_pad = 1 << (N - 1).bit_length()
    dev = cls_score.device
    dets = torch.empty((P, n_pad, 5), device=dev, dtype=torch.float32)
    counts = torch.empty((P,), device=dev, dtype=torch.int32)
    keep = torch.empty((P, n_pad), device=dev, dtype=torch.int32)
    nkeep = torch.empty((P,), device=dev, dtype=torch.int32)
    src = torch.empty((P, n_pad), device=dev, dtype=torch.int32)
    L = _lib.lib()
    nbytes = L.sdet_multiclass_nms_workspace(B, N, K, int(first_class))
    ws = _ws(nbytes, dev)
    check(L.sdet_multiclass_nms(_p(cls_score), _p(bbox_xyxy), B, N, K, bd, int(first_class),
                                float(min_det_score), float(nms_thresh), _p(dets), _p(counts), _p(keep),
                                _p(nkeep), _p(src), _p(ws), nbytes, _stream()))
    return dets, counts, keep, nkeep, src


def final_detections(cls_score, bbox_xyxy, nms_thresh, min_det_score=0.05, max_det_per_image=100, first_class=0):
    """detection_test.py:233-291 on the device: per-class NMS, then the `max_det_per_image` best detections of
    every image.  -> (out (B, max_det, 6) rows [x, y, w, h, score, class index] ascending by score,
    count (B)); class index counts from `first_class` (map it through coco.getCatIds() on the host)."""
    dets, counts, keep, nkeep, _ = multiclass_nms(cls_score, bbox_xyxy, nms_thresh, min_det_score, first_class)
    B, _, K = cls_score.shape
    ncls = K - first_class
    out = torch.empty((B, int(max_det_per_image), 6), device=dets.device, dtype=torch.float32)
    cnt = torch.empty((B,), device=dets.device, dtype=torch.int32)
    check(_lib.lib().sdet_final_detections(_p(dets), _p(keep), _p(nkeep), B, ncls, int(dets.shape[1]),
                                           int(max_det_per_image), _p(out), _p(cnt), _stream()))
    return out, cnt


# --------------------------------------------------------------------------------------------
# soft_nms  (operator_py/cython/cpu_nms.pyx:98-203, operator_py/nms.py:5-16)
# --------------------------------------------------------------------------------------------
_SOFT_METHODS = {"hard": 0, "linear": 1, "gaussian": 2}


def soft_nms_batched(dets, sigma=0.5, Nt=0.3, threshold=0.001, method=0, counts=None):
    """All problems at once: dets (P,m,5) -> (boxes (P,m,5), inds (P,m) int32, counts (P) int32)."""
    dets = _dev(dets, "dets")
    if dets.dim() != 3 or dets.shape[2] != 5:
        raise ValueError("dets must be (P,m,5)")
    P, m, _ = dets.shape
    counts = _dev(counts, "counts", torch.int32)
    ob = torch.empty_like(dets)
    oi = torch.empty((P, m), device=dets.device, dtype=torch.int32)
    oc = torch.empty((P,), device=dets.device, dtype=torch.int32)
    check(_lib.lib().sdet_soft_nms(_p(dets), _p(counts), P, m, float(sigma), float(Nt), float(threshold),
                                   int(method), _p(ob), _p(oi), _p(oc), _stream()))
    return ob, oi, oc


def soft_nms(boxes_in, sigma=0.5, Nt=0.3, threshold=0.001, method=0):
    """Same signature and result as the Cython `soft_nms`: (boxes[:N], inds[:N])."""
    ob, oi, oc = soft_nms_batched(boxes_in[None], sigma, Nt, threshold, method)
    n = int(oc[0])
    return ob[0, :n], oi[0, :n].to(torch.int64)


def cython_soft_nms_wrapper(thresh, sigma=0.5, score_thresh=0.001, method="linear"):
    """operator_py/nms.py:5-16 — returns fn(dets (m,5)) -> dets, as pTest.nms.type expects
    (detection_test.py:224-231)."""
    assert method in _SOFT_METHODS, "Unknown soft_nms method: {}".format(method)

    def _nms(dets):
        return soft_nms(dets, sigma, thresh, score_thresh, _SOFT_METHODS[method])[0]

    return _nms


# --------------------------------------------------------------------------------------------
# Drop-in callables and CustomOp twins (SURVEY §8b "Secondary API 1/2/3")
# --------------------------------------------------------------------------------------------
def gpu_nms(dets, thresh, device_id=0):
    """operator_py/cython/gpu_nms.pyx:16-31 with the library's `_nms` export behind it: dets (m,5) float32 NUMPY
    array on the host -> list of kept indices into dets (descending score, `IoU > thresh` suppressed)."""
    import numpy as np

    dets = np.ascontiguousarray(dets, dtype=np.float32)
    n, dim = dets.shape
    order = dets[:, 4].argsort()[::-1]
    sorted_dets = np.ascontiguousarray(dets[order, :])
    keep = np.zeros(n, dtype=np.int32)
    num_out = ctypes.c_int(0)
    _lib.lib()._nms(keep.ctypes.data, ctypes.byref(num_out), sorted_dets.ctypes.data, int(n), int(dim), float(thresh),
                    int(device_id))
    return list(order[keep[:num_out.value]])


def greedy_nms(dets, thresh):
    """operator_py/cython/cpu_nms.pyx:37-87 greedy_nms: dets (m,5) CUDA tensor -> kept indices ascending
    (`np.where(suppressed == 0)[0]`), suppression at IoU >= thresh."""
    dets = _dev(dets, "dets")
    if dets.shape[0] == 0:
        return torch.empty((0,), dtype=torch.int64, device=dets.device)
    order = torch.sort(dets[:, 4], descending=True, stable=True).indices
    keep, nkeep = nms_sorted(dets[order].contiguous()[None], thresh, ge=True)
    return torch.sort(order[keep[0, :int(nkeep.item())].long()]).values


def bbox_overlaps_cython(boxes, query_boxes):
    """operator_py/cython/bbox.pyx:32-73 on the device: (N,4), (K,4) -> (N,K) IoU."""
    return bbox_overlaps(boxes, query_boxes, "iou")


def assign_layer_fpn(rois, rcnn_stride=(4, 8, 16, 32), roi_canonical_scale=224, roi_canonical_level=4,
                     return_levels=False):
    """CustomOp 'assign_layer_fpn' (models/FPN/assign_layer_fpn.py:17-40): rois (B,N,4) -> one (B,N,4) tensor per
    stride holding the roi where it is assigned to that level and zeros elsewhere."""
    rois = _dev(rois, "rois")
    if rois.dim() != 3 or rois.shape[2] != 4:
        raise ValueError("rois must be (B,N,4)")
    L = len(rcnn_stride)
    outs = [torch.empty_like(rois) for _ in range(L)]
    levels = torch.empty(rois.shape[:2], device=rois.device, dtype=torch.int32)
    ptrs = (ctypes.c_void_p * L)(*[o.data_ptr() for o in outs])
    Ss = (ctypes.c_int * L)(*[int(s) for s in rcnn_stride])
    check(_lib.lib().sdet_fpn_assign(_p(rois), rois.shape[0] * rois.shape[1], Ss, L, int(roi_canonical_scale),
                                     int(roi_canonical_level), ptrs, _p(levels), _stream()))
    return (tuple(outs), levels) if return_levels else tuple(outs)


def BboxPostProcessing(cls_score, bbox_xyxy, max_det_per_image=100, min_det_score=0.05, nms_type="nms", nms_thr=0.5):
    """CustomOp 'BboxPostProcessing' (models/maskrcnn/bbox_post_processing.py:6-76): background column dropped,
    per-class py_nms, the max_det_per_image highest scores of the image -> post_score (B,M,1), post_bbox_xyxy
    (B,M,4), post_cls (B,M,1) (class index without background, -1 padding), descending score.  Among equal scores
    the reference's `np.argsort(scores)[::-1]` order is numpy's introsort order; here ties go to the later class."""
    if nms_type != "nms":
        raise NotImplementedError
    dets, counts, keep, nkeep, _ = multiclass_nms(cls_score, bbox_xyxy, nms_thr, min_det_score, first_class=1)
    B, _, K = cls_score.shape
    M = int(max_det_per_image)
    out = torch.empty((B, M, 6), device=dets.device, dtype=torch.float32)
    cnt = torch.empty((B,), device=dets.device, dtype=torch.int32)
    check(_lib.lib().sdet_final_detections_ex(_p(dets), _p(keep), _p(nkeep), B, K - 1, int(dets.shape[1]), M, _p(out),
                                              _p(cnt), 1, 1, _stream()))
    # rows beyond the count are [0,0,0,0,0,-1]: exactly the reference's zero / -1 initialised outputs
    post_bbox, post_score, post_cls = out[..., :4].contiguous(), out[..., 4:5].contiguous(), out[..., 5:6].contiguous()
    return post_score, post_bbox, post_cls


# Registry keyed by the reference's operator names (what symbol/builder.py binds by string).

# --------------------------------------------------------------------------------------------
# CustomOp 'decode_retina' (models/retinanet/decode_retina.py:35-146; the test branch of
# models/retinanet/builder.py:395-413 when the config does not ask for GenProposalRetina)
# --------------------------------------------------------------------------------------------
def decode_retina(cls_probs, bbox_preds, im_info, stride, scales, ratios, per_level_top_n, thresh):
    """-> (bbox_xyxy (1, L*per_level_top_n, 4), cls_score (1, L*per_level_top_n, num_class)), float32, zero-padded.

    Per level: pairs with score > thresh (0.0 on the coarsest level), the per_level_top_n best of them, anchors =
    cell * stride + base anchor (AnchorTarget2D.base_anchor, core/detection_input.py:374-400), nonlinear_pred
    decode in float64 with the float32 exp and the BBOX_XFORM_CLIP clamp the numpy code has, clip to the image.
    The reference keeps the selected pairs in np.argpartition's (unspecified) order; here each level's block is
    ordered by descending score, ties by flat index - the same set of rows.  Batch size 1 like the reference.
    A host-composed operator: the selection is torch.topk (library), everything stays on the device and nothing
    synchronises."""
    import math

    import numpy as np

    L_ = len(stride)
    cls_probs = [_dev(c, f"cls_prob[{i}]") for i, c in enumerate(cls_probs)]
    bbox_preds = [_dev(c, f"bbox_pred[{i}]") for i, c in enumerate(bbox_preds)]
    im_info = _dev(im_info, "im_info")
    if cls_probs[0].shape[0] != 1:
        raise ValueError("Multiple images each device is not implemented")  # the reference's message
    A = len(scales) * len(ratios)
    K = cls_probs[0].shape[1] // A
    dev = cls_probs[0].device
    top = int(per_level_top_n)
    boxes_out = torch.zeros((1, top * L_, 4), device=dev, dtype=torch.float32)
    score_out = torch.zeros((1, top * L_, K + 1), device=dev, dtype=torch.float32)
    clip = float(np.float32(math.log(1000.0 / 16.0)))  # np.minimum(float32 array, python float) stays float32
    hmax, wmax = im_info[0, 0].double() - 1.0, im_info[0, 1].double() - 1.0
    blocks, nvalid = [], []
    for s_, cp, bp in zip(stride, cls_probs, bbox_preds):
        H, W = cp.shape[2], cp.shape[3]
        # base anchors: aspect-major, np.round = round-half-even, float64
        side = float(s_)
        ctr = 0.5 * (side - 1)
        asp = np.asarray(ratios, np.float64)
        wr = np.round(np.sqrt(side * side / asp))
        hr = np.round(wr * asp)
        sc = np.asarray(scales, np.float64)
        ws_, hs_ = np.outer(wr, sc).ravel(), np.outer(hr, sc).ravel()
        base = torch.from_numpy(np.stack([ctr - 0.5 * (ws_ - 1), ctr - 0.5 * (hs_ - 1), ctr + 0.5 * (ws_ - 1),
                                          ctr + 0.5 * (hs_ - 1)], 1)).to(dev)                      # (A, 4) float64
        thr = float(thresh) if s_ != max(stride) else 0.0
        flat = cp.reshape(-1)                                                                       # (a, k, y, x) order
        k_ = min(top, flat.numel())
        vals, inds = torch.topk(torch.where(flat > thr, flat, torch.full_like(flat, -1.0)), k_, sorted=True)
        ok = vals > thr
        x = inds % W
        y = (inds // W) % H
        cls = (inds // (H * W)) % K
        a = inds // (H * W * K)
        cell = torch.stack([x, y, x, y], 1).to(torch.float32) * float(s_)
        anchors = (cell.double() + base[a]).to(torch.float32).double()   # float32 `+=` float64 rounds to float32 first
        d = bp.reshape(A, 4, H, W)[a, :, y, x]                                                      # (k, 4) float32
        wdt = anchors[:, 2] - anchors[:, 0] + 1.0
        hgt = anchors[:, 3] - anchors[:, 1] + 1.0
        cx = anchors[:, 0] + 0.5 * (wdt - 1.0)
        cy = anchors[:, 1] + 0.5 * (hgt - 1.0)
        pcx = d[:, 0].double() * wdt + cx
        pcy = d[:, 1].double() * hgt + cy
        pw = torch.exp(torch.clamp(d[:, 2], max=clip)).double() * wdt
        ph = torch.exp(torch.clamp(d[:, 3], max=clip)).double() * hgt
        bx = torch.stack([pcx - 0.5 * (pw - 1.0), pcy - 0.5 * (ph - 1.0), pcx + 0.5 * (pw - 1.0),
                          pcy + 0.5 * (ph - 1.0)], 1)
        lim = torch.stack([wmax, hmax, wmax, hmax])
        bx = torch.clamp(torch.minimum(bx, lim), min=0.0)
        blocks.append((bx.to(torch.float32), vals, cls, ok))
        nvalid.append(ok.sum())
    # the reference concatenates the levels' kept rows: row offsets are running counts of valid rows (on the device);
    # rows that did not pass the threshold are sent to a scratch row past the end
    nrow = top * L_
    bbuf = torch.zeros((nrow + 1, 4), device=dev, dtype=torch.float32)
    sbuf = torch.zeros((nrow + 1, K + 1), device=dev, dtype=torch.float32)
    off = torch.zeros((), device=dev, dtype=torch.long)
    for (bx, vals, cls, ok), n in zip(blocks, nvalid):
        rank = torch.cumsum(ok.long(), 0) - 1 + off          # valid rows are a prefix of the sorted block
        rows = torch.where(ok, rank, torch.full_like(rank, nrow)).clamp(max=nrow)
        bbuf.index_put_((rows,), bx)
        sbuf.index_put_((rows, cls + 1), vals)
        off = off + n
    boxes_out[0] = bbuf[:nrow]
    score_out[0] = sbuf[:nrow]
    return boxes_out, score_out


# --------------------------------------------------------------------------------------------
# test-time mask paste + COCO result records  (models/maskrcnn/utils.py:26-67, mask_test.py:283-313,
# detection_test.py:268-291)
# --------------------------------------------------------------------------------------------
def rle_counts_to_strings(counts, row_ptr):
    """cocoapi maskApi.c rleToString for many masks at once, on the host (numpy): `counts` is the concatenation of
    the masks' run lengths, mask n owning counts[row_ptr[n]:row_ptr[n+1]].  -> list of bytes, what
    pycocotools.mask.encode puts under 'counts'.  Each count (from a mask's 4th on: its difference to the count two
    places back) becomes 5-bit groups, least significant first, 0x20 = continuation, 0x10 of the last group = sign,
    + 48."""
    import numpy as np

    counts = np.asarray(counts, np.int64)
    row_ptr = np.asarray(row_ptr, np.int64)
    n = counts.size
    if n == 0:
        return [b"" for _ in range(len(row_ptr) - 1)]
    idx_in_row = np.arange(n, dtype=np.int64) - np.repeat(row_ptr[:-1], np.diff(row_ptr))
    x = counts.copy()
    d = idx_in_row > 2
    x[d] -= counts[np.nonzero(d)[0] - 2]
    chars = np.zeros((n, 13), np.uint8)           # 64-bit value: at most 13 groups of 5 bits
    length = np.zeros(n, np.int64)
    alive = np.ones(n, bool)
    for k in range(13):
        c = x & 0x1F
        x = x >> 5                                # arithmetic shift on int64, like the C `long`
        more = np.where((c & 0x10) != 0, x != -1, x != 0)
        c = np.where(more, c | 0x20, c) + 48
        chars[alive, k] = c[alive]
        length[alive] = k + 1
        alive = alive & more
        if not alive.any():
            break
    keep = np.arange(13)[None, :] < length[:, None]
    flat = chars[keep]                            # row-major: each count's characters in order
    ends = np.cumsum(length)
    char_ptr = np.concatenate([[0], ends])[row_ptr]
    raw = flat.tobytes()
    return [raw[char_ptr[i]:char_ptr[i + 1]] for i in range(len(row_ptr) - 1)]


def _segm_results_impl(bbox_xyxy, cls, masks, im_h, im_w, count_fn, write_fn):
    """The host side of `segm_results` around the two passes (count_fn / write_fn: the C-ABI calls on CUDA tensors in
    the product, the host emulation of the same kernel source in tests/test_mask_paste_host.py)."""
    import numpy as np

    N = int(bbox_xyxy.shape[0])
    im_h, im_w = int(im_h), int(im_w)
    if N == 0:
        return np.array([], dtype=object)
    dev = bbox_xyxy.device
    col_counts = torch.empty((N, im_w), device=dev, dtype=torch.int32)
    count_fn(bbox_xyxy, cls, masks, col_counts)
    incl = torch.cumsum(col_counts.reshape(-1).to(torch.int64), 0)
    col_offsets = (incl - col_counts.reshape(-1)).contiguous()                 # exclusive scan, (N * im_w) int64
    total = int(incl[-1].item())                                               # the one synchronisation
    positions = torch.empty((max(total, 1),), device=dev, dtype=torch.int32)
    if total:
        write_fn(bbox_xyxy, cls, masks, col_offsets, positions)
    per_det = col_counts.sum(1, dtype=torch.int64).cpu().numpy()               # flips per detection
    pos = positions[:total].cpu().numpy().astype(np.int64)
    # run lengths: differences of consecutive flip positions, bracketed by 0 and im_h * im_w
    det_ptr = np.concatenate([[0], np.cumsum(per_det)])
    row_ptr = det_ptr + np.arange(N + 1)                                        # one more count than flips per mask
    ext = np.empty(total + 2 * N, np.int64)                                     # per mask: 0, its flips, im_h*im_w
    ext_ptr = det_ptr + 2 * np.arange(N + 1)
    is_flip = np.ones(total + 2 * N, bool)
    is_flip[ext_ptr[:-1]] = False
    is_flip[ext_ptr[1:] - 1] = False
    ext[ext_ptr[:-1]] = 0
    ext[ext_ptr[1:] - 1] = im_h * im_w
    ext[is_flip] = pos
    diffs = np.diff(ext)
    keep = np.ones(diffs.size, bool)
    keep[ext_ptr[1:-1] - 1] = False                                             # the differences across two masks
    strings = rle_counts_to_strings(diffs[keep], row_ptr)
    out = np.empty(N, dtype=object)
    for i in range(N):
        out[i] = {"size": [im_h, im_w], "counts": strings[i]}
    return out


def segm_results(bbox_xyxy, cls, masks, im_h, im_w):
    """models/maskrcnn/utils.py:26-67 `segm_results` (the body of mask_test.py's pTest.process_output,
    models/maskrcnn/process_output.py:6-19): bbox_xyxy (N,4) float32, cls (N) int, masks (N,K,M,M) float32 (background
    channel already removed) -> numpy object array of N dicts {'size': [im_h, im_w], 'counts': bytes}, what
    `pycocotools.mask.encode` returns for the pasted binary masks.  Inputs may be numpy arrays (copied to the
    current CUDA device, like the reference's host arrays) or CUDA tensors (CPU tensors raise: no CPU fallback).

    expand_boxes, the int32 truncation, cv2.resize's bilinear interpolation (as the opencv-python wheel's IPP path
    rounds it), `> 0.5` and the paste run in two launches that never materialise the im_h x im_w images: only the
    positions where a pasted mask flips leave the device; the run-length strings are formed on the host.  A box with
    no pixel inside the image gives the empty mask (the reference raises there)."""
    import numpy as np

    def dev_of(a, dtype):   # numpy arrays go to the current device; tensors must already be there (CPU tensors raise)
        if isinstance(a, np.ndarray):
            a = torch.from_numpy(np.ascontiguousarray(a)).to(torch.device("cuda", torch.cuda.current_device()))
        return a.to(dtype).contiguous()

    boxes = _dev(dev_of(bbox_xyxy, torch.float32), "bbox_xyxy")
    masks_t = _dev(dev_of(masks, torch.float32), "masks")
    cls_t = _dev(dev_of(cls, torch.int32), "cls", dtype=torch.int32)
    if boxes.dim() != 2 or boxes.shape[1] != 4 or masks_t.dim() != 4 or masks_t.shape[0] != boxes.shape[0] \
            or masks_t.shape[2] != masks_t.shape[3] or cls_t.shape != (boxes.shape[0],):
        raise ValueError("segm_results: bbox_xyxy (N,4), cls (N), masks (N,K,M,M)")
    N, K, M = int(masks_t.shape[0]), int(masks_t.shape[1]), int(masks_t.shape[2])
    L = _lib.lib()

    def count_fn(b, c, m, col_counts):
        check(L.sdet_mask_paste_count(_p(b), _p(c), _p(m), N, K, M, int(im_h), int(im_w), _p(col_counts), _stream()))

    def write_fn(b, c, m, col_offsets, positions):
        check(L.sdet_mask_paste_write(_p(b), _p(c), _p(m), N, K, M, int(im_h), int(im_w), _p(col_offsets),
                                      _p(positions), _stream()))

    return _segm_results_impl(boxes, cls_t, masks_t, im_h, im_w, count_fn, write_fn)


def coco_bbox_records(image_id, dets_by_category, max_det_per_image):
    """detection_test.py:268-289 for one image: dets_by_category {dataset category id: (n,5) float32 rows
    [x1,y1,x2,y2,score]} (insertion order = the reference's class loop) -> the image's COCO result dicts, the
    `max_det_per_image` best in ascending score order (Python's stable sort, then [-max:])."""
    result = []
    for cid, det in dets_by_category.items():
        if det.shape[0] == 0:
            continue
        xs, ys = det[:, 0], det[:, 1]
        ws, hs = det[:, 2] - xs + 1, det[:, 3] - ys + 1
        scores = det[:, 4]
        result += [{"image_id": int(image_id), "category_id": int(cid),
                    "bbox": [float(xs[k]), float(ys[k]), float(ws[k]), float(hs[k])], "score": float(scores[k])}
                   for k in range(det.shape[0])]
    return sorted(result, key=lambda r: r["score"])[-int(max_det_per_image):]


def coco_records_from_final_detections(image_ids, out, count, category_ids):
    """The same records from `final_detections`' device result: out (B, max_det, 6) rows [x, y, w, h, score, class
    index] ascending by score, count (B); category_ids = coco.getCatIds() (class index -> dataset id).  One
    device-to-host copy; the rows are already the reference's selection and order."""
    out_h, cnt_h = out.cpu().numpy(), count.cpu().numpy()
    recs = []
    for b, iid in enumerate(image_ids):
        n = int(cnt_h[b])
        rows = out_h[b, :n]                                             # the valid rows come first
        recs += [{"image_id": int(iid), "category_id": int(category_ids[int(r[5])]),
                  "bbox": [float(r[0]), float(r[1]), float(r[2]), float(r[3])], "score": float(r[4])} for r in rows]
    return recs


def coco_segm_records(image_id, dets_by_category, segms_by_category, mask_scores_by_category, max_det_per_image):
    """mask_test.py:283-313 for one image: like coco_bbox_records plus 'mask_score' and 'segmentation' (the RLE dict
    with its counts decoded to str)."""
    result = []
    for cid, det in dets_by_category.items():
        if det.shape[0] == 0:
            continue
        seg, ms = segms_by_category[cid], mask_scores_by_category[cid]
        xs, ys = det[:, 0], det[:, 1]
        ws, hs = det[:, 2] - xs + 1, det[:, 3] - ys + 1
        scores = det[:, -1]
        result += [{"image_id": int(image_id), "category_id": int(cid),
                    "bbox": [float(xs[k]), float(ys[k]), float(ws[k]), float(hs[k])], "score": float(scores[k]),
                    "mask_score": float(ms[k]),
                    "segmentation": {"size": seg[k]["size"], "counts": seg[k]["counts"].decode("utf8")}}
                   for k in range(det.shape[0])]
    return sorted(result, key=lambda r: r["score"])[-int(max_det_per_image):]


def write_coco_json(coco_result, path):
    """detection_test.py:286-290 / mask_test.py:317-321: json.dump(coco_result, f, sort_keys=True, indent=2)."""
    import json

    with open(path, "w") as f:
        json.dump(coco_result, f, sort_keys=True, indent=2)



def mask_test_records(im_id, im_info, im_h, im_w, post_cls_score, post_box, post_cls, mask, category_ids,
                      max_det_per_image=100, mask_score=None):
    """One image of mask_test.py's result loop (:159-200 un-padding and rescaling, :207 process_output =
    segm_results, :236-311 per-class grouping and COCO records; the `multi_branch_nms is None` route every shipped
    Mask R-CNN config takes).  Inputs are the squeezed network outputs of one image as numpy arrays or CUDA tensors:
    post_cls_score (D,), post_box (D,4) in network-input pixels, post_cls (D,) with -1 padding, mask (D, 1+K, M, M)
    with the background channel first; im_info = (h, w, scale); im_h, im_w = roidb[rec_id]['h'], ['w'];
    category_ids = coco.getCatIds().  -> the image's COCO result dicts (bbox + score + mask_score + segmentation)."""
    import numpy as np

    def host(a):
        return a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)

    info = host(im_info).reshape(-1)
    scale = info[2]
    cls_all = host(post_cls).reshape(-1).astype(np.int32)
    valid = np.where(cls_all > -1)[0]                                   # remove pad bbox and mask
    bbox_xyxy = (host(post_box).reshape(-1, 4) / scale)[valid]          # scale to the original image
    cls_score = host(post_cls_score).reshape(-1)[valid]
    cls = cls_all[valid]
    ms = np.zeros_like(cls_score) if mask_score is None else host(mask_score).reshape(-1)[valid]
    if isinstance(mask, torch.Tensor):
        vt = torch.from_numpy(valid).to(mask.device)
        m = mask[:, 1:][vt].contiguous()                                # remove bg; stays on the device
    else:
        m = np.ascontiguousarray(np.asarray(mask)[:, 1:][valid])
    segm = segm_results(np.ascontiguousarray(bbox_xyxy, np.float32), cls, m, im_h, im_w) if len(valid) else np.array([], object)
    dets, segs, mscores = {}, {}, {}
    for cid in np.unique(cls):
        ind = np.where(cls == cid)[0]
        det = np.concatenate((bbox_xyxy[ind], cls_score[ind].reshape(-1, 1)), axis=1).astype(np.float32)
        dataset_cid = category_ids[int(cid)]
        dets[dataset_cid], segs[dataset_cid], mscores[dataset_cid] = det, segm[ind], ms[ind]
    return coco_segm_records(im_id, dets, segs, mscores, max_det_per_image)



def maskiou_compute(mask_pred_logits, mask_target, mask_ratio, mask_inds):
    """CustomOp 'maskiou_compute' (models/msrcnn/maskiou_compute.py:10-44; Mask Scoring R-CNN's MaskIoU regression
    target, fed by ProposalMaskTarget(output_ratio=True)): mask_pred_logits, mask_target (R,M,M), mask_ratio (R) or
    (R,1), mask_inds (R) class per slot -> (maskiou_target (R,1), weight_list (R,1)) float32.
    iou = max(sum(target * pred), 0) / max(sum(target) / ratio + sum(pred) - sum(target * pred), 1) with pred =
    `mask_pred_logits` > 0.5 (the operator's own threshold on its first input, which models/msrcnn/builder.py feeds with the
    sigmoid probabilities `mask_pred_prob`); the sums are small integers (exact in float32), the
    division by the ratio and the quotient are float64 like numpy's, rounded to float32 on output.  Host-composed on the
    device (elementwise + row reductions from the library); no gradient (need_top_grad=False, zero in_grad)."""
    logits = _dev(mask_pred_logits, "mask_pred_logits")
    target = _dev(mask_target, "mask_target")
    ratio = _dev(mask_ratio, "mask_ratio").reshape(-1)
    inds = _dev(mask_inds, "mask_inds").reshape(-1)
    with torch.no_grad():
        pred = logits > 0.5
        inter = (target * pred).sum((1, 2))                          # float32, exact
        pred_sum = pred.sum((1, 2)).double()
        tgt_sum = target.sum((1, 2)).double() / ratio.double()
        union = torch.clamp(tgt_sum + pred_sum - inter.double(), min=1.0)
        iou = (torch.clamp(inter, min=0.0).double() / union).to(torch.float32).reshape(-1, 1)
        weight = (inds > 0).to(torch.float32).reshape(-1, 1)
    return iou, weight



def _bbox_target_impl(proposal, gt_bbox, num_class, add_gt_to_proposal, image_rois, fg_fraction, fg_thresh, bg_thresh_hi,
                      bg_thresh_lo, bbox_target_std, rng, overlaps):
    """The body of `bbox_target` over tensors on one device, with the IoU operator passed in (the product passes the
    CUDA `bbox_overlaps`; tests/test_bbox_target_host.py drives the same host logic on CPU tensors)."""
    import numpy as np

    B, R, C = proposal.shape[0], int(image_rois), int(num_class)
    dev = proposal.device
    inv = [1.0 / float(s) for s in bbox_target_std]
    fg_per_image = int(np.round(float(fg_fraction) * R))        # np.round: half to even (bbox_target.py:27)
    rois = torch.zeros((B, R, 4), device=dev, dtype=torch.float32)
    label = torch.zeros((B, R), device=dev, dtype=torch.float32)
    target = torch.zeros((B, R, 4 * C), device=dev, dtype=torch.float32)
    weight = torch.zeros((B, R, 4 * C), device=dev, dtype=torch.float32)
    for b in range(B):
        gt = gt_bbox[b][gt_bbox[b][:, 4] != -1]                 # class == -1 is padding
        prop = proposal[b][proposal[b][:, 3] != 0]              # y2 == 0 is padding
        if add_gt_to_proposal:
            prop = torch.cat([prop, gt[:, :4]], 0)
        if gt.shape[0] == 0:
            raise ValueError("bbox_target: an image without ground-truth boxes (the reference's argmax over an empty "
                             "axis raises too)")
        ov = overlaps(prop.contiguous(), gt[:, :4].contiguous())
        mx, arg = ov.max(dim=1)                                  # first maximum, like numpy's argmax
        mx_h = mx.cpu().numpy()
        fg = np.where(mx_h >= fg_thresh)[0]
        nfg = int(np.minimum(fg_per_image, fg.size))
        if fg.size > 0:
            fg = rng.choice(fg, size=nfg, replace=False)
        bg = np.where((mx_h < bg_thresh_hi) & (mx_h >= bg_thresh_lo))[0]
        nbg = int(np.minimum(R - nfg, bg.size))
        if bg.size > 0:
            bg = rng.choice(bg, size=nbg, replace=False)
        keep = np.append(fg, bg).astype(np.int64)
        if keep.size != R:
            raise ValueError(f"bbox_target: image {b} has {keep.size} candidates for image_rois={R}; the reference "
                             "returns ragged lists here, which it cannot stack either")
        keep = torch.from_numpy(keep).to(dev)
        agt = gt[arg[keep]]
        lab = agt[:, 4].clone()
        lab[nfg:] = 0
        ex = prop[keep]
        # detectron_bbox_utils.bbox_transform_inv:205-219, float32 throughout (python scalars are weak)
        ew = ex[:, 2] - ex[:, 0] + 1.0
        eh = ex[:, 3] - ex[:, 1] + 1.0
        ecx = ex[:, 0] + 0.5 * ew
        ecy = ex[:, 1] + 0.5 * eh
        gw = agt[:, 2] - agt[:, 0] + 1.0
        gh = agt[:, 3] - agt[:, 1] + 1.0
        gcx = agt[:, 0] + 0.5 * gw
        gcy = agt[:, 1] + 0.5 * gh
        t = torch.stack([inv[0] * (gcx - ecx) / ew, inv[1] * (gcy - ecy) / eh, inv[2] * torch.log(gw / ew),
                         inv[3] * torch.log(gh / eh)], 1)
        cls = (lab > 0).to(torch.long) if C == 2 else lab.to(torch.long)
        pos = torch.nonzero(cls > 0)[:, 0]
        col = 4 * cls[pos][:, None] + torch.arange(4, device=dev)[None, :]
        target[b][pos[:, None], col] = t[pos]
        weight[b][pos[:, None], col] = 1.0
        rois[b], label[b] = ex, lab
    return rois, label, target, weight


def bbox_target(proposal, gt_bbox, num_class, add_gt_to_proposal, image_rois, fg_fraction, fg_thresh, bg_thresh_hi,
                bg_thresh_lo, bbox_target_std, rng=None):
    """CustomOp 'bbox_target' (operator_py/bbox_target.py:12-170; the Detectron-style roi sampler of
    models/crowdhuman/builder.py:380-396).  proposal (B,K,4), gt_bbox (B,M,5) float32 on the device ->
    (sampled_proposal (B,R,4), bbox_cls (B,R), bbox_target (B,R,4C), bbox_target_weight (B,R,4C)), R = image_rois.

    A host-composed operator: IoU (the `bbox_overlaps_cython` kernel), the arg-max match, the gather and the float32
    target arithmetic run on the device; the sampling is the reference's own two `numpy.random.choice(..., replace=
    False)` draws per image on the host, in the reference's order (foreground, then background), so under
    `numpy.random.seed(s)` the sampled rows are the reference's rows.  `rng` defaults to the global `numpy.random`
    module like the reference; a `numpy.random.RandomState` may be passed instead.  Where the reference cannot work
    either (an image with fewer candidates than image_rois: ragged lists; an image without gt: argmax of an empty
    axis) a ValueError says so.  No gradient flows (need_top_grad=False, zero in_grad)."""
    import numpy as np

    proposal = _dev(proposal, "proposal")
    gt_bbox = _dev(gt_bbox, "gt_bbox")
    if proposal.dim() != 3 or proposal.shape[2] != 4 or gt_bbox.dim() != 3 or gt_bbox.shape[2] != 5 \
            or gt_bbox.shape[0] != proposal.shape[0]:
        raise ValueError("bbox_target: proposal (B,K,4), gt_bbox (B,M,5)")
    if isinstance(add_gt_to_proposal, str):
        add_gt_to_proposal = add_gt_to_proposal == "True"     # CustomOp kwargs arrive as strings
    if isinstance(bbox_target_std, str):
        from ast import literal_eval
        bbox_target_std = literal_eval(bbox_target_std)
    with torch.no_grad():
        return _bbox_target_impl(proposal.detach(), gt_bbox.detach(), int(num_class), bool(add_gt_to_proposal),
                                 int(image_rois), float(fg_fraction), float(fg_thresh), float(bg_thresh_hi),
                                 float(bg_thresh_lo), bbox_target_std, rng if rng is not None else np.random,
                                 bbox_overlaps)


# --------------------------------------------------------------------------------------------
# _contrib_GroupNorm forward (operator_cxx/contrib/group_norm.cu) and the FCOS test-time CustomOps
# (models/FCOS/utils.py)
# --------------------------------------------------------------------------------------------
def _channels_last_4d(t: torch.Tensor) -> bool:
    """(N, H, W, C) memory that is not also plain NCHW memory (C == 1 or H*W == 1 are both at once: NCHW then)."""
    return t.dim() == 4 and not t.is_contiguous() and t.is_contiguous(memory_format=torch.channels_last)


def group_norm_raw(data, gamma, beta, num_group=32, eps=1e-5, relu=False):
    """-> (y, mean (N, G), rsig (N, G)).  data (N, C, ...) fp32; a 4-D channels_last tensor is normalised in place
    of its (N, H, W, C) memory and y keeps that layout.  relu=True applies ReLU to y in the same pass."""
    data = _dev_any_layout(data, "data")
    gamma, beta = _dev(gamma, "gamma"), _dev(beta, "beta")
    if data.dim() < 2:
        raise ValueError("GroupNorm: data must be (N, C, ...)")
    N, C = int(data.shape[0]), int(data.shape[1])
    HxW = data.numel() // max(N * C, 1)
    G = int(num_group)
    if gamma.numel() != C or beta.numel() != C:
        raise ValueError(f"GroupNorm: gamma and beta must have C = {C} elements")
    cl = _channels_last_4d(data)
    if not cl:
        data = data.contiguous()
    y = torch.empty_like(data)
    mean = torch.empty((N, G), device=data.device, dtype=torch.float32)
    rsig = torch.empty((N, G), device=data.device, dtype=torch.float32)
    L = _lib.lib()
    nbytes = L.sdet_group_norm_workspace(N, C, HxW, G)
    ws = _ws(nbytes, data.device)
    check(L.sdet_group_norm_forward(_p(data), _p(gamma), _p(beta), _p(y), _p(mean), _p(rsig), N, C, HxW, G,
                                    float(eps), int(cl), int(bool(relu)), _p(ws), nbytes, _stream()))
    return y, mean, rsig


def GroupNorm(data, gamma, beta, num_group=32, eps=1e-5, relu=False):
    """mx.sym.contrib.GroupNorm / X.gn forward: the one visible output.  Inference only: there is no backward yet
    (GroupNorm training comes with FCOS training), so a tensor that requires grad raises NotImplementedError."""
    if torch.is_grad_enabled() and any(t.requires_grad for t in (data, gamma, beta)):
        raise NotImplementedError("_contrib_GroupNorm has no backward yet: GroupNorm training is part of the FCOS "
                                  "training follow-up; run under torch.no_grad()")
    return group_norm_raw(data, gamma, beta, num_group, eps, relu)[0]


def get_proposal_single_stage(centerness_logit, cls_logit, offset_logit, img_info, pre_nms_top_n, stride,
                              pre_nms_thresh):
    """CustomOp 'get_proposal_single_stage' (models/FCOS/utils.py:7-94), arguments in its list_arguments order:
    centerness (B,1,H,W), cls_prob (B,C,H,W), offset (B,4,H,W) (post-sigmoid / post-exp), im_info (B,3)
    -> res_bbox (B, pre_nms_top_n, 6).  cls_prob may be channels_last; offset is then read in the same layout."""
    ctr, cls = _dev_any_layout(centerness_logit, "centerness"), _dev_any_layout(cls_logit, "cls_prob")
    off, im_info = _dev_any_layout(offset_logit, "offset"), _dev(img_info, "im_info")
    if cls.dim() != 4:
        raise ValueError("get_proposal_single_stage: cls_prob must be (B,C,H,W)")
    B, C, H, W = (int(v) for v in cls.shape)
    if tuple(ctr.shape) != (B, 1, H, W) or tuple(off.shape) != (B, 4, H, W) or tuple(im_info.shape) != (B, 3):
        raise ValueError("get_proposal_single_stage: centerness (B,1,H,W), offset (B,4,H,W), im_info (B,3)")
    cl = _channels_last_4d(cls)
    if not cl:
        cls = cls.contiguous()
    ctr = ctr.contiguous()
    off = off.contiguous(memory_format=torch.channels_last) if cl else off.contiguous()
    top_n = int(pre_nms_top_n)
    out = torch.empty((B, top_n, 6), device=cls.device, dtype=torch.float32)
    L = _lib.lib()
    nbytes = L.sdet_fcos_proposal_workspace(B, C, H, W)
    ws = _ws(nbytes, cls.device)
    check(L.sdet_fcos_proposal(_p(ctr), _p(cls), _p(off), _p(im_info), _p(out), B, C, H, W, top_n, int(stride),
                               float(pre_nms_thresh), int(cl), _p(ws), nbytes, _stream()))
    return out


def get_batch_proposal(bbox):
    """CustomOp 'get_batch_proposal' (models/FCOS/utils.py:97-149): bbox (B,K,6) -> (res_bbox (B,K,4),
    score (B,K,81), cls_id (B,K,1)), rows sorted by score per image."""
    bbox = _dev(bbox, "bbox")
    if bbox.dim() != 3 or bbox.shape[2] != 6:
        raise ValueError("get_batch_proposal: bbox must be (B,K,6)")
    B, K = int(bbox.shape[0]), int(bbox.shape[1])
    res = torch.empty((B, K, 4), device=bbox.device, dtype=torch.float32)
    score = torch.empty((B, K, 81), device=bbox.device, dtype=torch.float32)
    cls_id = torch.empty((B, K, 1), device=bbox.device, dtype=torch.float32)
    check(_lib.lib().sdet_fcos_batch_proposal(_p(bbox), _p(res), _p(score), _p(cls_id), B, K, _stream()))
    return res, score, cls_id


OPS = {
    "_contrib_ROIAlign_v2": ROIAlign_v2,
    "ROIPooling_v1": ROIPooling_v1,
    "fpn_roi_align": fpn_roi_align,  # fusion of assign_layer_fpn + ROIAlign_v2 x L + add_n
    "_contrib_DecodeBBox": DecodeBBox,
    "_contrib_Proposal_v3": Proposal_v3,
    "_contrib_Proposal": Proposal,
    "_contrib_ModulatedDeformableConvolution": ModulatedDeformableConvolution,
    "_contrib_GenAnchor": GenAnchor,
    "_contrib_GenProposal": GenProposal,
    "_contrib_GenProposalRetina": GenProposalRetina,
    "_contrib_Proposal_v2": Proposal_v2,
    "_contrib_NMS": NMS,
    "ProposalTarget": ProposalTarget,
    "ProposalMaskTarget": ProposalMaskTarget,
    "ProposalTarget_v2": ProposalTarget_v2,
    "_contrib_DeformableConvolution": DeformableConvolution,
    "_contrib_FocalLoss": FocalLoss,
    "_contrib_BBoxNorm": BBoxNorm,
    "_contrib_SigmoidCrossEntropy": SigmoidCrossEntropy,
    "get_top_proposal": get_top_proposal,  # mx.operator.register('get_top_proposal')
    "assign_layer_fpn": assign_layer_fpn,  # mx.operator.register('assign_layer_fpn')
    "BboxPostProcessing": BboxPostProcessing,  # mx.operator.register('BboxPostProcessing')
    "decode_retina": decode_retina,            # mx.operator.register("decode_retina")
    "bbox_target": bbox_target,                # mx.operator.register('bbox_target')
    "segm_results": segm_results,              # models/maskrcnn/utils.py:26
    "maskiou_compute": maskiou_compute,        # mx.operator.register('maskiou_compute')
    "_contrib_GroupNorm": GroupNorm,
    "get_proposal_single_stage": get_proposal_single_stage,  # mx.operator.register("get_proposal_single_stage")
    "get_batch_proposal": get_batch_proposal,                # mx.operator.register("get_batch_proposal")
    # plain callables of operator_py (same names and argument meaning)
    "gpu_nms": gpu_nms,
    "greedy_nms": greedy_nms,
    "bbox_overlaps_cython": bbox_overlaps_cython,
    "soft_nms": soft_nms,
    "cython_soft_nms_wrapper": cython_soft_nms_wrapper,
    "py_set_nms_wrapper": py_set_nms_wrapper,
    "wnms_wrapper": wnms_wrapper,
}
