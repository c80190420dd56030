"""Device time of the RoI pooling backward: the default atomic kernels against the ordered (deterministic) ones that
torch.use_deterministic_algorithms(True) selects.  Shapes of the mask_train workload: 2 images, 256 channels, the
P2-P5 levels of an 800x1333 input.

  fused FPN RoIAlign, 512 rois per image at 7x7 and 128 rois per image at 14x14
  plain RoIAlign_v2 on P2, 512 rois per image at 7x7
  ROIPooling_v1 on P2, 512 rois per image at 7x7

Each call is timed with CUDA events; the two kernels alternate call by call after a warm-up, so both see the same
clocks and neighbours.  The card's name and power limit are read in the same run.  One JSON line per case.

  python benchmarks/roi_backward_bench.py [--iters 100] [--warmup 10]"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from simpledet_b200 import _lib, ops, synth  # noqa: E402

B, C = 2, 256


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def _time(calls, iters, warmup):
    """calls: {name: fn}.  -> {name: (median us, mean us)}, the calls alternating one by one."""
    for _ in range(warmup):
        for fn in calls.values():
            fn()
    torch.cuda.synchronize()
    ev = {k: [] for k in calls}
    for _ in range(iters):
        for k, fn in calls.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            ev[k].append((s, e))
    torch.cuda.synchronize()
    out = {}
    for k, pairs in ev.items():
        t = [s.elapsed_time(e) * 1e3 for s, e in pairs]
        out[k] = (round(statistics.median(t), 1), round(statistics.fmean(t), 1))
    return out


def fused_case(dev, rng, n, pooled):
    shapes = synth.fpn_shapes()
    feats = [torch.randn((B, C, h, w), device=dev) for h, w in shapes]
    rois = torch.from_numpy(synth.random_rois(rng, B, n)).to(dev)
    _, ax, ay, lv = ops.fpn_roi_align_raw(feats, rois, synth.FPN_STRIDES, pooled)
    g = torch.randn(ax.shape, device=dev)
    grads = [torch.empty_like(f) for f in feats]
    L = len(grads)
    ptrs = (ctypes.c_void_p * L)(*[x.data_ptr() for x in grads])
    Hs = (ctypes.c_int * L)(*[s[0] for s in shapes])
    Ws = (ctypes.c_int * L)(*[s[1] for s in shapes])
    lib = _lib.lib()

    def mk(fn):
        return lambda: _lib.check(fn(_p(g), _p(ax), _p(ay), _p(lv), ptrs, Hs, Ws, L, B, n, C, pooled, pooled, 0,
                                     _stream()))

    per_level = np.bincount(lv.cpu().numpy().ravel() + 1, minlength=L + 1)[1:].tolist()
    return mk(lib.sdet_fpn_roi_align_v2_backward), mk(lib.sdet_fpn_roi_align_v2_backward_ordered), \
        {"rois_per_level": per_level}


def plain_case(dev, rng, n, pooled):
    H, W = synth.fpn_shapes()[0]
    data = torch.randn((B, C, H, W), device=dev)
    rois = torch.from_numpy(synth.random_rois(rng, B, n, max_side=224.0)).to(dev)
    _, ax, ay = ops.roi_align_v2_raw(data, rois, pooled, 0.25)
    g = torch.randn(ax.shape, device=dev)
    grad = torch.empty_like(data)
    lib = _lib.lib()

    def mk(fn):
        return lambda: _lib.check(fn(_p(g), _p(ax), _p(ay), _p(grad), None, B, n, C, H, W, pooled, pooled, 0,
                                     _stream()))

    return mk(lib.sdet_roi_align_v2_backward), mk(lib.sdet_roi_align_v2_backward_ordered), {}


def pool_case(dev, rng, n, pooled):
    H, W = synth.fpn_shapes()[0]
    data = torch.randn((B, C, H, W), device=dev)
    boxes = synth.random_rois(rng, 1, B * n, max_side=224.0)[0]
    img = np.repeat(np.arange(B, dtype=np.float32), n)[:, None]
    rois = torch.from_numpy(np.concatenate([img, boxes], 1)).to(dev)
    _, idx = ops.roi_pooling_v1_raw(data, rois, pooled, 0.25)
    g = torch.randn(idx.shape, device=dev)
    grad = torch.empty_like(data)
    R = B * n
    lib = _lib.lib()

    def mk(fn):
        return lambda: _lib.check(fn(_p(g), _p(idx), _p(rois), _p(grad), None, B, R, C, H, W, pooled, pooled, 0.25, 0,
                                     _stream()))

    return mk(lib.sdet_roi_pooling_v1_backward), mk(lib.sdet_roi_pooling_v1_backward_ordered), {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("roi_backward_bench needs a GPU")
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    print(json.dumps({"card": _card(), "iters": a.iters, "warmup": a.warmup}))
    cases = [("fpn_roi_align", fused_case, 512, 7), ("fpn_roi_align", fused_case, 128, 14),
             ("roi_align_v2_P2", plain_case, 512, 7), ("roi_pooling_v1_P2", pool_case, 512, 7)]
    for name, make, n, pooled in cases:
        atomic, ordered, info = make(dev, np.random.default_rng(0), n, pooled)
        t = _time({"atomic": atomic, "ordered": ordered}, a.iters, a.warmup)
        print(json.dumps({"case": name, "rois_per_image": n, "pooled": pooled, **info,
                          "atomic_us_median": t["atomic"][0], "atomic_us_mean": t["atomic"][1],
                          "ordered_us_median": t["ordered"][0], "ordered_us_mean": t["ordered"][1],
                          "ordered_over_atomic": round(t["ordered"][0] / t["atomic"][0], 2)}))


if __name__ == "__main__":
    main()
