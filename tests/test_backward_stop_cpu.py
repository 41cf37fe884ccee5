"""CPU: the C ABI of the fine-tuning backward with early ray termination (mvsn_render_backward_rays_stop) -- declared,
exported, bound, sized, and its argument errors returned without a device, from C and from Python."""
import ctypes
import math
import os

import pytest
import torch

from conftest import ROOT
from mvsnerf_b200 import backend, lib

NAMES = ("mvsn_render_backward_rays_stop_workspace_bytes", "mvsn_render_backward_rays_stop")
FAKE = 0x10000                                                    # 16-byte aligned, never dereferenced


@pytest.fixture(scope="module")
def built():
    from mvsnerf_b200 import build
    return build.build_library()


def test_backward_stop_is_declared_exported_and_bound(built):
    header = open(os.path.join(ROOT, "include", "mvsnerf_b200.h")).read()
    dll = ctypes.CDLL(built)
    L = lib.load()
    for name in NAMES:
        assert name + "(" in header, name
        assert name in lib.EXPORTS, name
        assert hasattr(dll, name), name
    assert L.mvsn_render_backward_rays_stop_workspace_bytes.restype is ctypes.c_size_t
    assert len(L.mvsn_render_backward_rays_stop_workspace_bytes.argtypes) == 7
    assert len(L.mvsn_render_backward_rays_stop.argtypes) == 19


def test_backward_stop_workspace_sizes(built):
    """A little more than the rays entry's (the [N] live counts and the per-CTA deferred-ray lists), growing with N."""
    L = lib.load()
    ws = L.mvsn_render_backward_rays_stop_workspace_bytes
    S, D, H, W = 128, 128, 200, 200
    for mode in (lib.MLP_FP32, lib.MLP_TC_HALF):
        for det in (0, 1):
            prev = 0
            for N in (1, 7, 130, 1024, 4096, 65536):
                plain = L.mvsn_render_backward_rays_workspace_bytes(N, S, D, H, W, mode, det)
                got = ws(N, S, D, H, W, mode, det)
                assert plain + 4 * N + 8 * N <= got <= plain + 4 * N + 8 * (N + 2 * 132 * 4) + 512, (mode, det, N)
                assert got >= prev
                prev = got
            for s in (32, 48, 64, 128):                           # fewer samples: no smaller list
                assert ws(1024, s, D, H, W, mode, det) > L.mvsn_render_backward_rays_workspace_bytes(1024, s, D, H, W, mode, det)
            assert ws(1024, S, 0, 0, 0, mode, det) > 0            # frozen volume
        for shape in ((1024, 160), (0, S), (1024, 0)):            # N_samples > 128, no rays, no samples
            assert ws(*shape, D, H, W, mode, 0) == 0 and ws(*shape, D, H, W, mode, 1) == 0
    for mode in (lib.MLP_TC_SPLIT, lib.MLP_TC_PAIR, -1, 99):      # unknown grad_mode
        assert ws(1024, S, D, H, W, mode, 0) == 0 and ws(1024, S, D, H, W, mode, 1) == 0


def _fake_scene():
    sc = lib.RenderScene()
    sc.volume_dhwc, sc.D, sc.Hp, sc.Wp = FAKE, 8, 8, 8
    sc.imgs_hwc4, sc.V, sc.H, sc.W = FAKE, 3, 32, 32
    sc.w2cs, sc.intrinsics, sc.mlp_packed, sc.mlp_mode, sc.white_bkgd = FAKE, FAKE, FAKE, lib.MLP_FP32, 0
    return sc


def _call(L, grad_mode, scene=None, rp=None, rays=None, t_steps=None, N=8, S=32, t_stop=1e-4, g=None, w=None, gw=None,
          live=None, tiles=None):
    return L.mvsn_render_backward_rays_stop(scene, w, rp, rays, t_steps, None, N, S, grad_mode, 0, t_stop, g, gw, None,
                                            live, tiles, None, 0, None)


def test_backward_stop_argument_errors_need_no_gpu(built):
    """Order: unknown grad_mode, NULL pointers, t_stop, per-sample cotangents, misaligned rays / live_samples /
    tiles_done, N_samples > 128, the weight image -- all before any CUDA call (the fake pointers are never touched)."""
    L = lib.load()
    for mode in (lib.MLP_TC_SPLIT, lib.MLP_TC_PAIR, -1, 99):
        assert _call(L, mode) == -6                               # MVSN_EUNSUPPORTED, checked first
        assert b"grad_mode" in L.mvsn_last_error()
    sc, rp, g = _fake_scene(), lib.RayParams(2.0, 6.0, 0.0, 0), lib.RenderGrads()
    g.rgb = FAKE
    w = (ctypes.c_void_p * lib.N_MLP_TENSORS)(*([FAKE] * lib.N_MLP_TENSORS))
    sref, rref, gref = ctypes.byref(sc), ctypes.byref(rp), ctypes.byref(g)
    ok = dict(g=gref, w=w, gw=w)
    for mode in (lib.MLP_FP32, lib.MLP_TC_HALF):
        assert _call(L, mode, **ok) == -4                                                  # MVSN_ENULL: scene
        assert _call(L, mode, sref, None, FAKE, FAKE, **ok) == -4                          # ray params
        assert _call(L, mode, sref, rref, FAKE, FAKE, g=None, w=w, gw=w) == -4             # gradients
        assert _call(L, mode, sref, rref, None, FAKE, **ok) == -4                          # rays
        assert b"mvsn_render_backward_rays_stop" in L.mvsn_last_error()
        for bad in (-1e-6, float("nan"), 1.5, math.inf):                                   # MVSN_EBADSHAPE
            assert _call(L, mode, sref, rref, FAKE, FAKE, t_stop=bad, **ok) == -1, bad
            assert b"t_stop" in L.mvsn_last_error()
        for field in ("weights", "alpha", "input_feat"):                                   # per-sample cotangents
            setattr(g, field, FAKE)
            assert _call(L, mode, sref, rref, FAKE, FAKE, **ok) == -6, field
            assert b"dead samples" in L.mvsn_last_error()
            setattr(g, field, None)
        assert _call(L, mode, sref, rref, FAKE + 4, FAKE, **ok) == -2                      # MVSN_EALIGN: rays
        assert _call(L, mode, sref, rref, FAKE, FAKE, live=FAKE + 2, **ok) == -2           # live_samples
        assert b"live_samples" in L.mvsn_last_error()
        assert _call(L, mode, sref, rref, FAKE, FAKE, live=FAKE + 4, tiles=FAKE + 4, **ok) == -2   # tiles_done
        assert b"tiles_done" in L.mvsn_last_error()
        assert _call(L, mode, sref, rref, FAKE, FAKE, S=160, **ok) == -6                   # N_samples > 128
        assert b"N_samples=160 > 128" in L.mvsn_last_error()
        sc.mlp_mode = lib.MLP_TC_HALF                                                      # not the fp32 image
        assert _call(L, mode, sref, rref, FAKE, FAKE, **ok) == -6
        assert b"MVSN_MLP_FP32" in L.mvsn_last_error()
        sc.mlp_mode = lib.MLP_FP32
        for t in (0.0, 1.0):                                                               # the closed range, empty batch
            assert _call(L, mode, sref, rref, FAKE, FAKE, N=0, t_stop=t, live=FAKE + 4, tiles=FAKE + 8, **ok) == 0


def test_backward_stop_python_argument_errors_need_no_gpu(built):
    """backend.render_backward_rays rejects a bad t_stop, per-sample cotangents and bad live_samples / tiles_done before
    it touches a tensor's data or the device."""
    rays = torch.zeros(4, 8)
    kw = dict(volume_feature=None, imgs=None, pose_ref=None, network_fn=None, near_far=(2.0, 6.0), pad=0.0, N_samples=32)
    for bad in (-0.5, 1.5, float("nan")):
        with pytest.raises(RuntimeError, match="t_stop"):
            backend.render_backward_rays(rays, **kw, t_stop=bad)
    for field in ("weights", "alpha", "input_feat"):
        with pytest.raises(RuntimeError, match="per-sample"):
            backend.render_backward_rays(rays, **kw, t_stop=1e-4, grads={"rgb": torch.zeros(4, 3), field: torch.zeros(1)})
    with pytest.raises(RuntimeError, match="live_samples"):
        backend.render_backward_rays(rays, **kw, t_stop=1e-4, live_samples=torch.zeros(4, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="tiles_done"):
        backend.render_backward_rays(rays, **kw, t_stop=1e-4, tiles_done=torch.zeros(3, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="need t_stop"):
        backend.render_backward_rays(rays, **kw, tiles_done=torch.zeros(3, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="grad_mode"):
        backend.render_backward_rays(rays, **kw, t_stop=1e-4, grad_mode=lib.MLP_TC_SPLIT)
