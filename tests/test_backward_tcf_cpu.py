"""CPU: grad_mode GRAD_TC_FULL in the C ABI and the Python entries -- accepted and sized by the rays entries, refused by
the samples entries, and every argument error returned before any CUDA call."""
import ctypes

import pytest
import torch

from mvsnerf_b200 import backend, lib


@pytest.fixture(scope="module")
def built():
    from mvsnerf_b200 import build
    return build.build_library()


def test_grad_tc_full_value():
    assert lib.GRAD_TC_FULL == 4
    assert lib.GRAD_TC_FULL not in (lib.MLP_FP32, lib.MLP_TC_HALF, lib.MLP_TC_SPLIT, lib.MLP_TC_PAIR)


def test_workspace_sizes(built):
    L = lib.load()
    N, S, D, H, W = 1024, 128, 128, 200, 200
    half = L.mvsn_render_backward_tc_workspace_bytes(N, S)
    for ws in (L.mvsn_render_backward_rays_workspace_bytes, L.mvsn_render_backward_rays_stop_workspace_bytes):
        for det in (0, 1):
            full = ws(N, S, D, H, W, lib.GRAD_TC_FULL, det)
            tch = ws(N, S, D, H, W, lib.MLP_TC_HALF, det)
            assert 0 < tch < full <= tch + 2 * 128 * 64 * 2 + 256    # + the forward's two fp16 [128][64] operands
            assert ws(N, 160, D, H, W, lib.GRAD_TC_FULL, det) == 0   # N_samples > 128
            assert ws(0, S, D, H, W, lib.GRAD_TC_FULL, det) == 0
        assert ws(N, S, 0, 0, 0, lib.GRAD_TC_FULL, 1) > 0            # frozen volume
    assert L.mvsn_render_backward_rays_workspace_bytes(N, S, D, H, W, lib.GRAD_TC_FULL, 0) == half + 2 * 128 * 64 * 2
    # the samples entries do not take the mode
    assert L.mvsn_render_backward_deterministic_workspace_bytes(N, S, D, H, W, lib.GRAD_TC_FULL) == 0
    # the other values keep their meaning
    for mode in (lib.MLP_TC_SPLIT, lib.MLP_TC_PAIR, -1, 99):
        assert L.mvsn_render_backward_rays_workspace_bytes(N, S, D, H, W, mode, 0) == 0
        assert L.mvsn_render_backward_rays_stop_workspace_bytes(N, S, D, H, W, mode, 0) == 0


FAKE = 0x10000


def _fake_args():
    sc = lib.RenderScene()
    sc.volume_dhwc, sc.D, sc.Hp, sc.Wp = FAKE, 8, 8, 8
    sc.imgs_hwc4, sc.V, sc.H, sc.W = FAKE, 3, 32, 32
    sc.w2cs, sc.intrinsics, sc.mlp_packed, sc.mlp_mode, sc.white_bkgd = FAKE, FAKE, FAKE, lib.MLP_FP32, 0
    rp = lib.RayParams(2.0, 6.0, 0.0, 0)
    g = lib.RenderGrads()
    g.rgb = FAKE
    w = (ctypes.c_void_p * lib.N_MLP_TENSORS)(*([FAKE] * lib.N_MLP_TENSORS))
    return sc, rp, g, w


def _rays(L, mode, scene=None, rp=None, rays=None, t_steps=None, N=8, S=32, g=None, w=None, det=0):
    return L.mvsn_render_backward_rays(scene, w, rp, rays, t_steps, None, N, S, mode, det, g, w, None, None, 0, None)


def _stop(L, mode, scene=None, rp=None, rays=None, t_steps=None, N=8, S=32, g=None, w=None, det=0, t_stop=1e-4,
          live=None):
    return L.mvsn_render_backward_rays_stop(scene, w, rp, rays, t_steps, None, N, S, mode, det, t_stop, g, w, None,
                                            live, None, None, 0, None)


@pytest.mark.parametrize("det", [0, 1])
def test_rays_entries_error_order(built, det):
    """The new mode passes the grad_mode check and then meets the same errors, in the same order, as MLP_TC_HALF:
    NULL pointers, misaligned rays, N_samples > 128, not the fp32 image, and an empty batch succeeds -- none of which
    touches a device (the fake addresses are never dereferenced)."""
    L = lib.load()
    sc, rp, g, w = _fake_args()
    sref, rref, gref = ctypes.byref(sc), ctypes.byref(rp), ctypes.byref(g)
    for call in (_rays, _stop):
        codes = {}
        for mode in (lib.MLP_TC_HALF, lib.GRAD_TC_FULL):
            c = [call(L, mode, det=det),                                                    # NULL scene
                 call(L, mode, sref, None, FAKE, FAKE, g=gref, w=w, det=det),               # NULL ray params
                 call(L, mode, sref, rref, None, FAKE, g=gref, w=w, det=det),               # NULL rays
                 call(L, mode, sref, rref, FAKE + 4, FAKE, g=gref, w=w, det=det),           # misaligned rays
                 call(L, mode, sref, rref, FAKE, FAKE, S=160, g=gref, w=w, det=det)]        # N_samples > 128
            sc.mlp_mode = lib.MLP_TC_HALF
            c.append(call(L, mode, sref, rref, FAKE, FAKE, g=gref, w=w, det=det))         # not the fp32 image
            sc.mlp_mode = lib.MLP_FP32
            c.append(call(L, mode, sref, rref, FAKE, FAKE, N=0, g=gref, w=w, det=det))    # empty batch
            codes[mode] = c
        assert codes[lib.GRAD_TC_FULL] == codes[lib.MLP_TC_HALF] == [-4, -4, -4, -2, -6, -6, 0], (call, codes)
    bad_t = [_stop(L, m, sref, rref, FAKE, FAKE, g=gref, w=w, det=det, t_stop=-1.0) for m in (lib.MLP_TC_HALF, lib.GRAD_TC_FULL)]
    assert bad_t[0] == bad_t[1] == -1 and b"t_stop" in L.mvsn_last_error()           # MVSN_EBADSHAPE
    for mode in (lib.MLP_TC_SPLIT, lib.MLP_TC_PAIR, -1, 99):                             # still unknown, checked first
        assert _rays(L, mode, sref, rref, FAKE, FAKE, g=gref, w=w, det=det) == -6
        assert b"grad_mode" in L.mvsn_last_error()


def test_samples_entry_refuses_the_mode(built):
    """mvsn_render_backward_deterministic returns MVSN_EUNSUPPORTED for it before any CUDA call, even with every
    other argument missing."""
    L = lib.load()
    rc = L.mvsn_render_backward_deterministic(None, None, None, None, None, None, 8, 32, lib.GRAD_TC_FULL, None, None,
                                              None, None, 0, None)
    assert rc == -6
    assert b"grad_mode 4" in L.mvsn_last_error()


class _Vol(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.feat_volume = torch.nn.Parameter(torch.zeros(1, 8, 2, 2, 2))


def test_python_samples_entries_refuse_the_mode():
    """FineTuner.step, render_backward and rendering under autograd raise before touching CUDA (every tensor here
    is on the CPU), naming the entries that take the mode."""
    fn = backend.MVSNeRF()
    with pytest.raises(RuntimeError, match="step_rays.*render_backward_rays"):
        backend.render_backward(None, torch.zeros(2, 4, 3), torch.zeros(2, 4, 3), torch.zeros(2, 4), torch.zeros(2, 3),
                                None, None, fn, grad_mode=lib.GRAD_TC_FULL)
    with pytest.raises(RuntimeError, match="step_rays.*render_backward_rays"):
        backend.rendering(None, {"w2cs": None}, torch.zeros(2, 4, 3), torch.zeros(2, 4, 3), torch.zeros(2, 4), None,
                          torch.zeros(2, 3), _Vol(), None, fn, grad_mode=lib.GRAD_TC_FULL)
    tuner = backend.FineTuner.__new__(backend.FineTuner)                 # the checks of step() run before any state
    tuner.grad_mode = lib.GRAD_TC_FULL
    with pytest.raises(RuntimeError, match="step_rays.*render_backward_rays"):
        tuner.step(None, None, None, None, None)
    for bad in (lib.MLP_TC_SPLIT, lib.MLP_TC_PAIR, -1, 99):                      # unchanged for the other values
        with pytest.raises(RuntimeError, match="MLP_FP32 \\(FFMA\\) or MLP_TC_HALF"):
            backend._check_grad_mode(bad, rays=True)
    backend._check_grad_mode(lib.GRAD_TC_FULL, rays=True)
