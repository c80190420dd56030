"""Argument checks of the deterministic RoI pooling backward entries.  Every check runs before the first CUDA call, so
they are testable without a GPU; on an error nothing is launched."""
import ctypes

import pytest


@pytest.fixture(scope="module")
def L():
    import __graft_entry__ as g

    g.build()
    from simpledet_b200 import _lib

    return _lib.lib()


def _err(L):
    return L.sdet_last_error()


def test_roi_align_ordered_checks(L):
    f = L.sdet_roi_align_v2_backward_ordered
    # ograd, argmax_x, argmax_y, grad_data, grad_rois, B, N, C, H, W, ph, pw, accumulate, stream
    assert f(None, 8, 8, 8, None, 1, 1, 1, 4, 4, 7, 7, 0, None) == 1 and b"NULL" in _err(L)
    assert f(8, 8, 8, None, None, 1, 1, 1, 4, 4, 7, 7, 0, None) == 1 and b"NULL" in _err(L)
    assert f(8, 8, 8, 8, None, 0, 1, 1, 4, 4, 7, 7, 0, None) == 1 and b"> 0" in _err(L)
    assert f(8, 8, 8, 8, None, 1, -1, 1, 4, 4, 7, 7, 0, None) == 1
    assert f(8, 8, 8, 8, None, 1, 1, 0, 4, 4, 7, 7, 0, None) == 1
    assert f(8, 8, 8, 8, None, 1, 1, 1, 0, 4, 7, 7, 0, None) == 1 and b"bad grad" in _err(L)
    assert f(8, 8, 8, 8, None, 1, 1, 1, 4, -4, 7, 7, 0, None) == 1
    assert f(8, 8, 8, 8, None, 1, 1, 1, 4, 4, 0, 7, 0, None) == 1 and b"pooled_size" in _err(L)
    assert f(8, 8, 8, 8, None, 1, 1, 1, 4, 4, 33, 7, 0, None) == 2 and b"pooled_size" in _err(L)
    assert f(8, 8, 8, 8, None, 1, 1, 1, 4, 4, 7, 33, 0, None) == 2
    # a plane row wider than one shared-memory band holds
    assert f(8, 8, 8, 8, None, 1, 1, 1, 4, 12289, 7, 7, 0, None) == 2 and b"band" in _err(L)


def test_fpn_roi_align_ordered_checks(L):
    f = L.sdet_fpn_roi_align_v2_backward_ordered
    n = 4
    ptrs = (ctypes.c_void_p * n)(8, 8, 8, 8)
    Hs = (ctypes.c_int * n)(200, 100, 50, 25)
    Ws = (ctypes.c_int * n)(334, 167, 84, 42)
    # ograd, argmax_x, argmax_y, levels, grad_feats, H, W, num_levels, B, N, C, ph, pw, accumulate, stream
    assert f(8, 8, 8, None, ptrs, Hs, Ws, n, 1, 1, 1, 7, 7, 0, None) == 1 and b"NULL" in _err(L)
    assert f(8, 8, 8, 8, None, Hs, Ws, n, 1, 1, 1, 7, 7, 0, None) == 1 and b"NULL" in _err(L)
    assert f(8, 8, 8, 8, ptrs, Hs, Ws, 0, 1, 1, 1, 7, 7, 0, None) == 1 and b"num_levels" in _err(L)
    assert f(8, 8, 8, 8, ptrs, Hs, Ws, 9, 1, 1, 1, 7, 7, 0, None) == 1 and b"num_levels" in _err(L)
    assert f(8, 8, 8, 8, ptrs, Hs, Ws, n, 1, 0, 1, 7, 7, 0, None) == 1 and b"> 0" in _err(L)
    assert f(8, 8, 8, 8, ptrs, Hs, Ws, n, 1, 1, 1, 7, 40, 0, None) == 2 and b"pooled_size" in _err(L)
    bad_ptr = (ctypes.c_void_p * n)(8, 8, None, 8)
    assert f(8, 8, 8, 8, bad_ptr, Hs, Ws, n, 1, 1, 1, 7, 7, 0, None) == 1 and b"level 2" in _err(L)
    bad_h = (ctypes.c_int * n)(200, 100, 50, 0)
    assert f(8, 8, 8, 8, ptrs, bad_h, Ws, n, 1, 1, 1, 7, 7, 0, None) == 1 and b"level 3" in _err(L)
    # the last level is too wide: refused before level 0 is launched
    wide = (ctypes.c_int * n)(334, 167, 84, 20000)
    assert f(8, 8, 8, 8, ptrs, Hs, wide, n, 1, 1, 1, 7, 7, 0, None) == 2 and b"band" in _err(L)


def test_roi_pool_ordered_checks(L):
    f = L.sdet_roi_pooling_v1_backward_ordered
    # ograd, max_idx, rois, grad_data, grad_rois, B, R, C, H, W, ph, pw, spatial_scale, accumulate, stream
    assert f(8, 8, None, 8, None, 1, 1, 1, 4, 4, 7, 7, 0.5, 0, None) == 1 and b"NULL" in _err(L)
    assert f(8, None, 8, 8, None, 1, 1, 1, 4, 4, 7, 7, 0.5, 0, None) == 1 and b"NULL" in _err(L)
    for shape in [(0, 1, 1, 4, 4, 7, 7), (1, 0, 1, 4, 4, 7, 7), (1, 1, 0, 4, 4, 7, 7), (1, 1, 1, 0, 4, 7, 7),
                  (1, 1, 1, 4, 0, 7, 7), (1, 1, 1, 4, 4, 0, 7), (1, 1, 1, 4, 4, 7, -7)]:
        assert f(8, 8, 8, 8, None, *shape, 0.5, 0, None) == 1 and b"positive" in _err(L)
    assert f(8, 8, 8, 8, None, 1, 1, 1, 4, 4, 33, 7, 0.5, 0, None) == 2 and b"pooled_size" in _err(L)
    assert f(8, 8, 8, 8, None, 1, 1, 1, 4, 12289, 7, 7, 0.5, 0, None) == 2 and b"band" in _err(L)
