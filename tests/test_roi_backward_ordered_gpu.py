"""Deterministic RoI pooling backward (csrc/roi_bwd_ordered.cu) against the serial oracle, by bit pattern.

The oracle (oracle/roi_ops.c) adds the contributions in ascending flat index, which is one of the orders the
reference's atomics can produce (pinned against the reference's own backward in test_oracle_ref_cxx.py).  Every
comparison here is on uint32 views: -0.0 and +0.0 differ, any NaN equals any NaN."""
import ctypes

import numpy as np
import pytest
import torch

import oracle
from simpledet_b200 import _lib, ops, synth

pytestmark = pytest.mark.gpu


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def assert_bits(got, ref):
    got = got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else got
    got, ref = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(ref, np.float32)
    assert got.shape == ref.shape
    gn, rn = np.isnan(got), np.isnan(ref)
    assert np.array_equal(gn, rn), f"NaN positions differ at {np.argwhere(gn != rn)[:5]}"
    gb, rb = got.view(np.uint32), ref.view(np.uint32)
    bad = (gb != rb) & ~gn
    assert not bad.any(), f"{bad.sum()} values differ, first at {np.argwhere(bad)[:5]}: {got[bad][:5]} vs {ref[bad][:5]}"


def align_bwd(dev, ograd, ax, ay, shape, init=None, grad_rois=None):
    """sdet_roi_align_v2_backward_ordered on host arrays; init given -> kAddTo into it."""
    B, N, C, ph, pw = ograd.shape
    _, _, H, W = shape
    grad = _t(init, dev) if init is not None else torch.full(shape, 3.0, device=dev)
    ograd, ax, ay = _t(ograd, dev), _t(ax, dev), _t(ay, dev)  # held until the kernel has run
    _lib.check(_lib.lib().sdet_roi_align_v2_backward_ordered(
        _p(ograd), _p(ax), _p(ay), _p(grad), _p(grad_rois), B, N, C, H, W, ph, pw,
        int(init is not None), _stream()))
    torch.cuda.synchronize()
    return grad.cpu().numpy()


def random_rois(rng, B, N, H, W, lo=2.0, hi=None):
    hi = hi or min(H, W) * 0.9
    wh = rng.uniform(lo, hi, (B, N, 2))
    xy = rng.uniform(0, 1, (B, N, 2)) * (np.array([W, H]) - wh)
    return np.concatenate([xy, xy + wh], -1).astype(np.float32)


@pytest.mark.parametrize("pooled", [(7, 7), (14, 14), (3, 5), (1, 1)])
@pytest.mark.parametrize("C", [1, 37, 256])
def test_roi_align_forward_argmax(cuda, pooled, C):
    rng = np.random.default_rng(pooled[0] * 100 + C)
    B, N, H, W = 2, 24, 23, 37
    data = rng.standard_normal((B, C, H, W)).astype(np.float32)
    rois = random_rois(rng, B, N, H * 4, W * 4, hi=60)
    _, ax, ay = ops.roi_align_v2_raw(_t(data, cuda), _t(rois, cuda), pooled, 0.25)
    ax, ay = ax.cpu().numpy(), ay.cpu().numpy()
    g = rng.standard_normal(ax.shape).astype(np.float32)
    assert_bits(align_bwd(cuda, g, ax, ay, data.shape), oracle.roi_align_v2_backward(g, ax, ay, data.shape))


def test_roi_align_pile_up_is_order_exact(cuda):
    """Hundreds of nearly identical rois on a few pixels, gradients of mixed magnitude: the sum depends on order."""
    rng = np.random.default_rng(5)
    B, N, C, ph, pw, H, W = 1, 400, 2, 2, 2, 9, 11
    shape = (B, C, H, W)
    ax = (4 + rng.uniform(0, 1.5, (B, N, C, ph, pw))).astype(np.float32)
    ay = (3 + rng.uniform(0, 1.5, (B, N, C, ph, pw))).astype(np.float32)
    g = rng.choice(np.float32([1e8, 1.0, -1e8, 3.0, -1.0, 0.5]), (B, N, C, ph, pw)).astype(np.float32)
    g *= rng.uniform(0.9, 1.1, g.shape).astype(np.float32)
    ref = oracle.roi_align_v2_backward(g, ax, ay, shape)
    rev = oracle.roi_align_v2_backward(*(a[:, ::-1, :, ::-1, ::-1] for a in (g, ax, ay)), shape)
    assert not np.array_equal(ref.view(np.uint32), rev.view(np.uint32)), "case is not sensitive to order"
    assert_bits(align_bwd(cuda, g, ax, ay, shape), ref)


def test_roi_align_hand_made_argmax(cuda):
    """Integer coordinates (four adds of one pixel at weight 0.5 x 0.5), coordinates clamped at H-1 / W-1 and
    below 0, -1 entries, on top of ordinary fractional ones."""
    rng = np.random.default_rng(6)
    B, N, C, ph, pw, H, W = 2, 40, 3, 4, 4, 13, 17
    shape = (B, C, H, W)
    sz = (B, N, C, ph, pw)
    ax = rng.uniform(0, W - 1, sz).astype(np.float32)
    ay = rng.uniform(0, H - 1, sz).astype(np.float32)
    kind = rng.integers(0, 6, sz)
    ax = np.where(kind == 1, np.floor(ax), ax)
    ay = np.where(kind == 1, np.floor(ay), ay)
    ax = np.where(kind == 2, W - 1 + rng.uniform(0, 3, sz), ax)   # clamped right
    ay = np.where(kind == 3, H - 1 + rng.uniform(0, 3, sz), ay)   # clamped bottom
    ay = np.where(kind == 4, rng.uniform(-0.99, 0, sz), ay)        # clamped top
    ax = np.where(kind == 5, -1, ax)                               # no contribution
    ay = np.where((kind == 5) & (rng.random(sz) < 0.5), -1, ay)
    ax, ay = ax.astype(np.float32), ay.astype(np.float32)
    g = rng.standard_normal(sz).astype(np.float32)
    gr = torch.full((B, N, 4), 7.0, device=cuda)
    assert_bits(align_bwd(cuda, g, ax, ay, shape, grad_rois=gr), oracle.roi_align_v2_backward(g, ax, ay, shape))
    assert torch.equal(gr, torch.zeros_like(gr))


def test_roi_align_signed_zeros(cuda):
    """kWriteTo starts from +0.0, so -0.0 contributions give +0.0; kAddTo into -0.0 keeps -0.0 where nothing or only
    -0.0 lands."""
    rng = np.random.default_rng(7)
    B, N, C, ph, pw, H, W = 1, 16, 2, 3, 3, 10, 12
    shape = (B, C, H, W)
    sz = (B, N, C, ph, pw)
    ax = rng.uniform(0, 5, sz).astype(np.float32)
    ay = rng.uniform(0, 4, sz).astype(np.float32)
    g = rng.choice(np.float32([0.0, -0.0]), sz).astype(np.float32)
    g[0, 0, 0, 0, 0] = -0.0
    ref = oracle.roi_align_v2_backward(g, ax, ay, shape)
    assert not np.signbit(ref).any()
    assert_bits(align_bwd(cuda, g, ax, ay, shape), ref)
    g = np.full(sz, -0.0, np.float32)
    init = np.full(shape, -0.0, np.float32)
    ref = oracle.roi_align_v2_backward(g, ax, ay, shape, accumulate_into=init)
    assert np.signbit(ref).all()
    assert_bits(align_bwd(cuda, g, ax, ay, shape, init=init), ref)


def test_roi_align_accumulate(cuda):
    rng = np.random.default_rng(8)
    B, C, H, W = 2, 5, 19, 29
    data = rng.standard_normal((B, C, H, W)).astype(np.float32)
    rois = random_rois(rng, B, 30, H * 2, W * 2)
    _, ax, ay = ops.roi_align_v2_raw(_t(data, cuda), _t(rois, cuda), (7, 7), 0.5)
    ax, ay = ax.cpu().numpy(), ay.cpu().numpy()
    g = rng.standard_normal(ax.shape).astype(np.float32)
    init = rng.standard_normal(data.shape).astype(np.float32)
    assert_bits(align_bwd(cuda, g, ax, ay, data.shape, init=init),
                oracle.roi_align_v2_backward(g, ax, ay, data.shape, accumulate_into=init))


def test_roi_align_banded_plane(cuda):
    """A P2-sized plane (200x334) is split into row bands: contributions on every row, so on both sides of each band
    boundary and straddling it."""
    rng = np.random.default_rng(9)
    B, N, C, ph, pw, H, W = 1, 64, 2, 7, 7, 200, 334
    shape = (B, C, H, W)
    sz = (B, N, C, ph, pw)
    ay = (rng.integers(0, H, sz) + rng.choice(np.float32([0.0, 0.5, 0.999]), sz)).astype(np.float32)
    ax = rng.uniform(0, W - 1, sz).astype(np.float32)
    g = rng.standard_normal(sz).astype(np.float32)
    init = rng.standard_normal(shape).astype(np.float32)
    assert_bits(align_bwd(cuda, g, ax, ay, shape), oracle.roi_align_v2_backward(g, ax, ay, shape))
    assert_bits(align_bwd(cuda, g, ax, ay, shape, init=init),
                oracle.roi_align_v2_backward(g, ax, ay, shape, accumulate_into=init))


def test_roi_align_nan_inf(cuda):
    rng = np.random.default_rng(10)
    B, N, C, ph, pw, H, W = 1, 20, 2, 3, 3, 8, 9
    shape = (B, C, H, W)
    sz = (B, N, C, ph, pw)
    ax = rng.uniform(0, W - 1, sz).astype(np.float32)
    ay = rng.uniform(0, H - 1, sz).astype(np.float32)
    g = rng.standard_normal(sz).astype(np.float32)
    pick = rng.random(sz)
    g[pick < 0.03] = np.nan
    g[(pick >= 0.03) & (pick < 0.06)] = np.inf
    g[(pick >= 0.06) & (pick < 0.09)] = -np.inf
    assert_bits(align_bwd(cuda, g, ax, ay, shape), oracle.roi_align_v2_backward(g, ax, ay, shape))


def _fpn_setup(cuda, rng, B=2, N=96, C=8, out=7, img=(400, 672)):
    shapes = synth.fpn_shapes(*img)
    feats = [rng.standard_normal((B, C, h, w)).astype(np.float32) for h, w in shapes]
    rois = synth.random_rois(rng, B, N, img[0], img[1], 8, 300)  # sqrt(area) < 448: no roi on P5
    _, ax, ay, lv = ops.fpn_roi_align_raw([_t(f, cuda) for f in feats], _t(rois, cuda), synth.FPN_STRIDES, out)
    return feats, ax, ay, lv


def _fpn_oracle(g, ax, ay, lv, feats, inits=None):
    refs = []
    for i, f in enumerate(feats):
        m = (lv == i)[..., None, None, None]
        refs.append(oracle.roi_align_v2_backward(np.where(m, g, 0).astype(np.float32),
                                                 np.where(m, ax, -1).astype(np.float32),
                                                 np.where(m, ay, -1).astype(np.float32), f.shape,
                                                 accumulate_into=None if inits is None else inits[i]))
    return refs


def _fpn_bwd(cuda, g, ax, ay, lv, shapes, inits=None):
    B, N, C, ph, pw = g.shape
    grads = [_t(x, cuda) for x in inits] if inits is not None else [torch.full(s, 5.0, device=cuda) for s in shapes]
    n = len(shapes)
    ptrs = (ctypes.c_void_p * n)(*[x.data_ptr() for x in grads])
    Hs = (ctypes.c_int * n)(*[s[2] for s in shapes])
    Ws = (ctypes.c_int * n)(*[s[3] for s in shapes])
    keep = [_t(g, cuda), ax, ay, _t(lv.astype(np.int32), cuda)]
    _lib.check(_lib.lib().sdet_fpn_roi_align_v2_backward_ordered(
        _p(keep[0]), _p(ax), _p(ay), _p(keep[3]), ptrs, Hs, Ws, n, B, N, C, ph, pw, int(inits is not None),
        _stream()))
    torch.cuda.synchronize()
    return grads


def test_fpn_levels_skip_and_accumulate(cuda):
    """Rois with level -1 (their argmax still valid) add nothing; P5 receives no roi; kWriteTo and kAddTo."""
    rng = np.random.default_rng(11)
    feats, ax, ay, lv = _fpn_setup(cuda, rng)
    lvn = lv.cpu().numpy()
    assert not (lvn == 3).any() and (lvn == 0).any() and (lvn == 1).any()
    lvn[:, ::7] = -1
    g = rng.standard_normal(ax.shape).astype(np.float32)
    axn, ayn = ax.cpu().numpy(), ay.cpu().numpy()
    shapes = [f.shape for f in feats]
    for got, ref in zip(_fpn_bwd(cuda, g, ax, ay, lvn, shapes), _fpn_oracle(g, axn, ayn, lvn, feats)):
        assert_bits(got, ref)
    inits = [rng.standard_normal(s).astype(np.float32) for s in shapes]
    for got, ref in zip(_fpn_bwd(cuda, g, ax, ay, lvn, shapes, inits), _fpn_oracle(g, axn, ayn, lvn, feats, inits)):
        assert_bits(got, ref)


def _pool_bwd(cuda, g, idx, rois, shape, init=None, grad_rois=None):
    R, C, ph, pw = g.shape
    B, _, H, W = shape
    grad = _t(init, cuda) if init is not None else torch.full(shape, 9.0, device=cuda)
    g, idx, rois = _t(g, cuda), _t(idx, cuda), _t(rois, cuda)  # held until the kernel has run
    _lib.check(_lib.lib().sdet_roi_pooling_v1_backward_ordered(
        _p(g), _p(idx), _p(rois), _p(grad), _p(grad_rois), B, R, C, H, W, ph, pw,
        0.25, int(init is not None), _stream()))
    torch.cuda.synchronize()
    return grad.cpu().numpy()


def test_roi_pool_interleaved_overlapping(cuda):
    """Rois of two images in an arbitrary order, heavily overlapping; an image index outside [0, B) adds nothing."""
    rng = np.random.default_rng(12)
    B, C, H, W, R = 2, 6, 21, 27, 300
    data = rng.standard_normal((B, C, H, W)).astype(np.float32)
    data = np.round(data * 4) / 4  # ties: the first maximum wins in the forward, many rois elect the same pixel
    x1 = rng.uniform(0, 30, R)
    y1 = rng.uniform(0, 20, R)
    rois = np.stack([rng.integers(0, B, R), x1, y1, x1 + rng.uniform(4, 60, R), y1 + rng.uniform(4, 50, R)],
                    1).astype(np.float32)
    _, idx = ops.roi_pooling_v1_raw(_t(data, cuda), _t(rois, cuda), (7, 7), 0.25)
    idx = idx.cpu().numpy()
    g = rng.standard_normal(idx.shape).astype(np.float32)
    gr = torch.full((R, 5), 7.0, device=cuda)
    assert_bits(_pool_bwd(cuda, g, idx, rois, data.shape, grad_rois=gr),
                oracle.roi_pool_v1_backward(g, idx, rois, data.shape))
    assert torch.equal(gr, torch.zeros_like(gr))
    init = rng.standard_normal(data.shape).astype(np.float32)
    assert_bits(_pool_bwd(cuda, g, idx, rois, data.shape, init=init),
                oracle.roi_pool_v1_backward(g, idx, rois, data.shape, accumulate_into=init))
    bad = rois.copy()
    bad[::5, 0] = np.where(rng.random(len(bad[::5])) < 0.5, B, -1)
    idx_ref = idx.copy()
    idx_ref[::5] = -1
    assert_bits(_pool_bwd(cuda, g, idx, bad, data.shape), oracle.roi_pool_v1_backward(g, idx_ref, rois, data.shape))


def test_mask_train_size_deterministic(cuda):
    """The fused operator at the mask_train size (2 images, 256 channels, P2-P5 of 800x1333, 512 rois per image at
    7x7) under torch's deterministic mode: two backward passes give identical bits and both equal the oracle."""
    rng = np.random.default_rng(13)
    B, N, C = 2, 512, 256
    shapes = synth.fpn_shapes()
    feats = [torch.randn((B, C, h, w), device=cuda).requires_grad_(True) for h, w in shapes]
    rois = _t(synth.random_rois(rng, B, N), cuda)
    g = torch.randn((B, N, C, 7, 7), device=cuda)
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        runs = []
        for _ in range(2):
            for f in feats:
                f.grad = None
            ops.fpn_roi_align(feats, rois, synth.FPN_STRIDES, 7).backward(g)
            runs.append([f.grad.clone() for f in feats])
    finally:
        torch.use_deterministic_algorithms(prev)
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    _, ax, ay, lv = ops.fpn_roi_align_raw([f.detach() for f in feats], rois, synth.FPN_STRIDES, 7)
    refs = _fpn_oracle(g.cpu().numpy(), ax.cpu().numpy(), ay.cpu().numpy(), lv.cpu().numpy(),
                       [f.detach().cpu().numpy() for f in feats])
    for got, ref in zip(runs[0], refs):
        assert_bits(got, ref)


def test_deterministic_flag_selects_ordered_entries(cuda, monkeypatch):
    L = _lib.lib()
    names = ["sdet_roi_align_v2_backward", "sdet_fpn_roi_align_v2_backward", "sdet_roi_pooling_v1_backward"]
    calls = []
    for name in names + [n + "_ordered" for n in names]:
        fn = getattr(L, name)

        def rec(*args, _fn=fn, _name=name):
            calls.append(_name)
            return _fn(*args)

        monkeypatch.setattr(L, name, rec)
    rng = np.random.default_rng(14)
    data = torch.randn((2, 4, 16, 20), device=cuda, requires_grad=True)
    rois = _t(random_rois(rng, 2, 6, 64, 80), cuda)
    feats = [torch.randn((2, 4, h, w), device=cuda, requires_grad=True) for h, w in synth.fpn_shapes(128, 160)]
    prois = _t(np.concatenate([rng.integers(0, 2, (8, 1)), random_rois(rng, 1, 8, 60, 70)[0]], 1).astype(np.float32),
               cuda)

    def run_all():
        ops.ROIAlign_v2(data, rois, 3, 0.25).sum().backward()
        ops.fpn_roi_align(feats, rois, synth.FPN_STRIDES, 3).sum().backward()
        ops.ROIPooling_v1(data, prois, 3, 0.25).sum().backward()
        torch.cuda.synchronize()

    prev = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        run_all()
        assert calls == [n + "_ordered" for n in names]
        calls.clear()
        torch.use_deterministic_algorithms(False)
        run_all()
        assert calls == names
    finally:
        torch.use_deterministic_algorithms(prev)


def test_cuda_graph_replay(cuda):
    """No allocation and no host synchronisation: the ordered backward captures into a CUDA graph, and the replay
    equals the eager call."""
    rng = np.random.default_rng(15)
    B, C, H, W = 2, 16, 50, 84
    data = rng.standard_normal((B, C, H, W)).astype(np.float32)
    rois = random_rois(rng, B, 40, H * 4, W * 4)
    _, ax, ay = ops.roi_align_v2_raw(_t(data, cuda), _t(rois, cuda), (7, 7), 0.25)
    g = torch.randn(ax.shape, device=cuda)
    eager = torch.empty((B, C, H, W), device=cuda)
    replay = torch.full((B, C, H, W), 1.0, device=cuda)
    L = _lib.lib()

    def call(out):
        _lib.check(L.sdet_roi_align_v2_backward_ordered(_p(g), _p(ax), _p(ay), _p(out), None, B, ax.shape[1], C,
                                                        H, W, 7, 7, 0, _stream()))

    call(eager)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call(replay)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(eager.view(torch.int32), replay.view(torch.int32))
    assert_bits(eager, oracle.roi_align_v2_backward(g.cpu().numpy(), ax.cpu().numpy(), ay.cpu().numpy(), data.shape))
