"""CPU: the C ABI of the fine-tuning backward from rays (mvsn_render_backward_rays) -- declared, exported, bound, sized,
and its argument errors returned without a device."""
import ctypes
import os

import pytest

from conftest import ROOT
from mvsnerf_b200 import lib

NAMES = ("mvsn_render_backward_rays_workspace_bytes", "mvsn_render_backward_rays")


@pytest.fixture(scope="module")
def built():
    from mvsnerf_b200 import build
    return build.build_library()


def test_backward_rays_is_declared_exported_and_bound(built):
    header = open(os.path.join(ROOT, "include", "mvsnerf_b200.h")).read()
    dll = ctypes.CDLL(built)
    L = lib.load()
    for name in NAMES:
        assert name + "(" in header, name
        assert name in lib.EXPORTS, name
        assert hasattr(dll, name), name
    assert L.mvsn_render_backward_rays_workspace_bytes.restype is ctypes.c_size_t
    assert len(L.mvsn_render_backward_rays_workspace_bytes.argtypes) == 7
    assert len(L.mvsn_render_backward_rays.argtypes) == 16


def test_backward_rays_workspace_sizes(built):
    L = lib.load()
    ws = L.mvsn_render_backward_rays_workspace_bytes
    N, S, D, H, W = 1024, 128, 128, 200, 200
    for mode, base in ((lib.MLP_FP32, L.mvsn_render_backward_workspace_bytes(N, S)),
                       (lib.MLP_TC_HALF, L.mvsn_render_backward_tc_workspace_bytes(N, S))):
        plain = ws(N, S, D, H, W, mode, 0)
        assert plain == base > 0                                  # nothing per sample: the march happens in the kernel
        assert ws(N, S, 0, 0, 0, mode, 0) == plain
        det = ws(N, S, D, H, W, mode, 1)
        assert det >= plain + D * H * W * 8 * 8                   # + the int64 accumulator
        assert det == L.mvsn_render_backward_deterministic_workspace_bytes(N, S, D, H, W, mode)
        frozen = ws(N, S, 0, 0, 0, mode, 1)
        assert plain + 4 * N <= frozen < det                      # + the per-ray loss terms only
        for shape in ((N, 160), (0, S), (N, 0)):                  # N_samples > 128, no rays, no samples
            assert ws(*shape, D, H, W, mode, 0) == 0 and ws(*shape, D, H, W, mode, 1) == 0
    for mode in (lib.MLP_TC_SPLIT, lib.MLP_TC_PAIR, -1, 99):      # unknown grad_mode
        assert ws(N, S, D, H, W, mode, 0) == 0 and ws(N, S, D, H, W, mode, 1) == 0


def _call(L, grad_mode, scene=None, rp=None, rays=None, t_steps=None, N=8, S=32, g=None, w=None, gw=None):
    return L.mvsn_render_backward_rays(scene, w, rp, rays, t_steps, None, N, S, grad_mode, 0, g, gw, None, None, 0, None)


def test_backward_rays_argument_errors_need_no_gpu(built):
    """Order: unknown grad_mode, NULL pointers, misaligned rays, N_samples > 128 -- all before any CUDA call (the
    pointers below are never dereferenced on the device, so this runs on a machine without one)."""
    L = lib.load()
    for mode in (lib.MLP_TC_SPLIT, lib.MLP_TC_PAIR, -1, 99):
        assert _call(L, mode) == -6                               # MVSN_EUNSUPPORTED, checked first
        assert b"grad_mode" in L.mvsn_last_error()
    for mode in (lib.MLP_FP32, lib.MLP_TC_HALF):
        assert _call(L, mode) == -4                               # MVSN_ENULL: scene
        assert b"NULL" in L.mvsn_last_error()

    # a scene whose buffers are fake 16-byte-aligned addresses: make_scene only looks at them
    fake = 0x10000
    sc = lib.RenderScene()
    sc.volume_dhwc, sc.D, sc.Hp, sc.Wp = fake, 8, 8, 8
    sc.imgs_hwc4, sc.V, sc.H, sc.W = fake, 3, 32, 32
    sc.w2cs, sc.intrinsics, sc.mlp_packed, sc.mlp_mode, sc.white_bkgd = fake, fake, fake, lib.MLP_FP32, 0
    rp = lib.RayParams(2.0, 6.0, 0.0, 0)
    g = lib.RenderGrads()
    g.rgb = fake
    w = (ctypes.c_void_p * lib.N_MLP_TENSORS)(*([fake] * lib.N_MLP_TENSORS))
    sref, rref, gref = ctypes.byref(sc), ctypes.byref(rp), ctypes.byref(g)
    for mode in (lib.MLP_FP32, lib.MLP_TC_HALF):
        assert _call(L, mode, sref, None, fake, fake, g=gref, w=w, gw=w) == -4             # ray params
        assert _call(L, mode, sref, rref, fake, fake, g=None, w=w, gw=w) == -4             # gradients
        assert _call(L, mode, sref, rref, None, fake, g=gref, w=w, gw=w) == -4             # rays
        assert b"rays" in L.mvsn_last_error()
        assert _call(L, mode, sref, rref, fake, None, g=gref, w=w, gw=w) == -4             # t_steps
        assert _call(L, mode, sref, rref, fake + 4, fake, g=gref, w=w, gw=w) == -2         # MVSN_EALIGN
        assert b"aligned" in L.mvsn_last_error()
        assert _call(L, mode, sref, rref, fake + 4, fake, S=160, g=gref, w=w, gw=w) == -2  # alignment before S
        assert _call(L, mode, sref, rref, fake, fake, S=160, g=gref, w=w, gw=w) == -6      # N_samples > 128
        assert b"N_samples=160 > 128" in L.mvsn_last_error()
        sc.mlp_mode = lib.MLP_TC_HALF                                                      # not the fp32 image
        assert _call(L, mode, sref, rref, fake, fake, g=gref, w=w, gw=w) == -6
        assert b"MVSN_MLP_FP32" in L.mvsn_last_error()
        sc.mlp_mode = lib.MLP_FP32
        assert _call(L, mode, sref, rref, fake, fake, N=0, g=gref, w=w, gw=w) == 0         # empty batch: nothing to do
