"""CPU: early ray termination from the samples entries (mvsn_render_samples_stop, mvsn_render_backward_stop and the
`t_stop` of rendering / render_backward / FineTuner.step / create_nerf_mvs) -- declared, exported, bound, sized, and
their argument errors returned without a device, from C and from Python."""
import ctypes
import math
import os
from types import SimpleNamespace

import pytest
import torch

from conftest import ROOT
from mvsnerf_b200 import backend, lib

NAMES = ("mvsn_render_samples_stop", "mvsn_render_backward_stop_workspace_bytes", "mvsn_render_backward_stop")
FAKE = 0x10000                                                    # 16-byte aligned, never dereferenced


@pytest.fixture(scope="module")
def built():
    from mvsnerf_b200 import build
    return build.build_library()


def test_symbols_are_declared_exported_and_bound(built):
    header = open(os.path.join(ROOT, "include", "mvsnerf_b200.h")).read()
    dll = ctypes.CDLL(built)
    L = lib.load()
    for name in NAMES:
        assert name + "(" in header, name
        assert name in lib.EXPORTS, name
        assert hasattr(dll, name), name
    assert len(L.mvsn_render_samples_stop.argtypes) == 12
    assert L.mvsn_render_backward_stop_workspace_bytes.restype is ctypes.c_size_t
    assert len(L.mvsn_render_backward_stop_workspace_bytes.argtypes) == 7
    assert len(L.mvsn_render_backward_stop.argtypes) == 19


def test_backward_stop_workspace_is_the_rays_stop_workspace(built):
    """The same layout as the rays entry's: the grad mode's workspace, the live counts and the deferred-ray lists."""
    L = lib.load()
    S, D, H, W = 128, 128, 200, 200
    for mode in (lib.MLP_FP32, lib.MLP_TC_HALF):
        for det in (0, 1):
            for N in (1, 7, 130, 1024, 65536):
                got = L.mvsn_render_backward_stop_workspace_bytes(N, S, D, H, W, mode, det)
                assert got == L.mvsn_render_backward_rays_stop_workspace_bytes(N, S, D, H, W, mode, det) > 0
            assert L.mvsn_render_backward_stop_workspace_bytes(1024, S, 0, 0, 0, mode, det) > 0      # frozen volume
        for shape in ((1024, 160), (0, S), (1024, 0)):
            assert L.mvsn_render_backward_stop_workspace_bytes(*shape, D, H, W, mode, 0) == 0
    for mode in (lib.GRAD_TC_FULL, lib.MLP_TC_SPLIT, lib.MLP_TC_PAIR, -1):                  # samples grad modes only
        assert L.mvsn_render_backward_stop_workspace_bytes(1024, S, D, H, W, mode, 0) == 0


def _scene(mode):
    sc = lib.RenderScene()
    sc.volume_dhwc, sc.D, sc.Hp, sc.Wp = FAKE, 8, 8, 8
    sc.imgs_hwc4, sc.V, sc.H, sc.W = FAKE, 3, 32, 32
    sc.w2cs, sc.intrinsics, sc.mlp_packed, sc.mlp_mode, sc.white_bkgd = FAKE, FAKE, FAKE, mode, 0
    return sc


def _render(mode, t_stop=1e-4, rgb=FAKE, pts=FAKE, tiles=None, N=16, S=8):
    L = lib.load()
    sc = _scene(mode)
    rc = L.mvsn_render_samples_stop(ctypes.byref(sc), pts, FAKE, FAKE, FAKE, N, S, t_stop, rgb, FAKE, tiles, None)
    return rc, L.mvsn_last_error().decode()


def test_render_stop_argument_errors_need_no_gpu(built):
    assert _render(lib.MLP_TC_PAIR, rgb=None)[0] == -4                              # MVSN_ENULL
    assert _render(lib.MLP_TC_PAIR, pts=None)[0] == -4
    for bad in (-1e-3, math.nan):                                                   # MVSN_EBADSHAPE
        rc, msg = _render(lib.MLP_TC_SPLIT, bad)
        assert rc == -1 and "t_stop" in msg and "mvsn_render_samples_stop" in msg
    rc, msg = _render(lib.MLP_FP32)
    assert rc == -6 and "mlp_mode 0" in msg                                         # MVSN_EUNSUPPORTED
    rc, msg = _render(lib.MLP_TC_HALF, tiles=FAKE + 4)
    assert rc == -2 and "tiles_done" in msg                                         # MVSN_EALIGN
    assert _render(lib.MLP_FP32, -1.0, rgb=None)[0] == -4                           # NULL is reported first
    assert _render(lib.MLP_TC_HALF, N=-1)[0] == -1
    for mode in (lib.MLP_TC_HALF, lib.MLP_TC_PAIR | lib.VOLUME_F16, lib.MLP_TC_SPLIT):   # empty batch: nothing to do
        assert _render(mode, 2.0, N=0, tiles=FAKE + 8)[0] == 0


def _bwd(L, grad_mode, scene=None, pts=FAKE, N=8, S=32, t_stop=1e-4, g=None, w=None, gw=None, vol=None, live=None,
         tiles=None):
    return L.mvsn_render_backward_stop(scene, w, pts, FAKE, FAKE, FAKE, N, S, grad_mode, 0, t_stop, g, gw, vol, live,
                                       tiles, None, 0, None)


def test_backward_stop_argument_errors_need_no_gpu(built):
    """Order: the grad_mode, NULL pointers, t_stop, per-sample cotangents, misaligned buffers, N_samples > 128, the
    weight image -- all before any CUDA call (the fake pointers are never touched)."""
    L = lib.load()
    for mode in (lib.GRAD_TC_FULL, lib.MLP_TC_SPLIT, lib.MLP_TC_PAIR, -1, 99):
        assert _bwd(L, mode) == -6                                                  # MVSN_EUNSUPPORTED, checked first
        assert b"grad_mode" in L.mvsn_last_error()
    sc, g = _scene(lib.MLP_FP32), lib.RenderGrads()
    g.rgb = FAKE
    w = (ctypes.c_void_p * lib.N_MLP_TENSORS)(*([FAKE] * lib.N_MLP_TENSORS))
    sref, gref = ctypes.byref(sc), ctypes.byref(g)
    ok = dict(g=gref, w=w, gw=w)
    for mode in (lib.MLP_FP32, lib.MLP_TC_HALF):
        assert _bwd(L, mode, **ok) == -4                                            # MVSN_ENULL: scene
        assert _bwd(L, mode, sref, g=None, w=w, gw=w) == -4                         # gradients
        assert _bwd(L, mode, sref, pts=None, **ok) == -4                            # samples
        assert b"mvsn_render_backward_stop" in L.mvsn_last_error()
        for bad in (-1e-6, float("nan"), 1.5, math.inf):                            # MVSN_EBADSHAPE
            assert _bwd(L, mode, sref, t_stop=bad, **ok) == -1, bad
            assert b"t_stop" in L.mvsn_last_error()
        for field in ("weights", "alpha", "input_feat"):                            # per-sample cotangents
            setattr(g, field, FAKE)
            assert _bwd(L, mode, sref, **ok) == -6, field
            assert b"dead samples" in L.mvsn_last_error()
            setattr(g, field, None)
        assert _bwd(L, mode, sref, vol=FAKE + 4, **ok) == -2                        # MVSN_EALIGN: volume gradient
        assert _bwd(L, mode, sref, live=FAKE + 2, **ok) == -2                       # live_samples
        assert b"live_samples" in L.mvsn_last_error()
        assert _bwd(L, mode, sref, live=FAKE + 4, tiles=FAKE + 4, **ok) == -2       # tiles_done
        assert b"tiles_done" in L.mvsn_last_error()
        assert _bwd(L, mode, sref, S=160, **ok) == -6                               # N_samples > 128
        assert b"N_samples=160 > 128" in L.mvsn_last_error()
        for image in (lib.MLP_TC_HALF, lib.MLP_FP32 | lib.VOLUME_F16):             # not the fp32 image
            sc.mlp_mode = image
            assert _bwd(L, mode, sref, **ok) == -6
            assert b"MVSN_MLP_FP32" in L.mvsn_last_error()
        sc.mlp_mode = lib.MLP_FP32
        for t in (0.0, 1.0):                                                        # the closed range, empty batch
            assert _bwd(L, mode, sref, N=0, t_stop=t, live=FAKE + 4, tiles=FAKE + 8, **ok) == 0


def _cpu_inputs(n=4, S=8):
    pose = {"w2cs": torch.eye(4).expand(3, 4, 4).contiguous(), "intrinsics": torch.eye(3).expand(3, 3, 3).contiguous()}
    return dict(pose_ref=pose, rays_pts=torch.zeros(n, S, 3), rays_ndc=torch.zeros(n, S, 3),
                depth_candidates=torch.zeros(n, S), rays_o=torch.zeros(n, 3), rays_dir=torch.ones(n, 3),
                volume_feature=torch.zeros(1, 8, 4, 4, 4), imgs=torch.zeros(1, 3, 3, 8, 8))


def test_rendering_rejects_bad_t_stop_and_cpu_tensors(built):
    args = SimpleNamespace()
    fn = backend.MVSNeRF()
    kw = _cpu_inputs()
    for bad in (-0.5, float("nan")):
        with pytest.raises(RuntimeError, match="t_stop"):
            backend.rendering(args, network_fn=fn, t_stop=bad, **kw)
    with pytest.raises(RuntimeError, match="tensor-core"):
        backend.rendering(args, network_fn=fn, t_stop=1e-4, mlp_mode=lib.MLP_FP32, **kw)
    with pytest.raises(RuntimeError, match="need t_stop|needs t_stop"):
        backend.rendering(args, network_fn=fn, tiles_done=torch.zeros(1, dtype=torch.int64), **kw)
    with pytest.raises(RuntimeError, match="tiles_done"):
        backend.rendering(args, network_fn=fn, t_stop=1e-4, tiles_done=torch.zeros(1, dtype=torch.int64), **kw)
    with pytest.raises(RuntimeError, match=r"\[0, 1\]"):                            # under autograd (the MLP trains)
        backend.rendering(args, network_fn=fn, t_stop=2.0, **kw)
    with pytest.raises(RuntimeError, match="CUDA"):                                  # training step
        backend.rendering(args, network_fn=fn, t_stop=1e-4, **kw)
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA"):                 # inference
        backend.rendering(args, network_fn=fn, t_stop=1e-4, **kw)


def test_render_backward_and_step_reject_bad_t_stop_and_cpu_tensors(built):
    kw = _cpu_inputs()
    pos = (kw["pose_ref"], kw["rays_pts"], kw["rays_ndc"], kw["depth_candidates"], kw["rays_dir"], kw["volume_feature"],
           kw["imgs"], backend.MVSNeRF())
    for bad in (-0.5, 1.5, float("nan")):
        with pytest.raises(RuntimeError, match="t_stop"):
            backend.render_backward(*pos, t_stop=bad)
    for field in ("weights", "alpha", "input_feat"):
        with pytest.raises(RuntimeError, match="per-sample"):
            backend.render_backward(*pos, t_stop=1e-4, grads={"rgb": torch.zeros(4, 3), field: torch.zeros(1)})
    with pytest.raises(RuntimeError, match="live_samples"):
        backend.render_backward(*pos, t_stop=1e-4, live_samples=torch.zeros(4, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="tiles_done"):
        backend.render_backward(*pos, t_stop=1e-4, tiles_done=torch.zeros(3, dtype=torch.int64))
    with pytest.raises(RuntimeError, match="need t_stop"):
        backend.render_backward(*pos, live_samples=torch.zeros(4, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="GRAD_TC_FULL"):
        backend.render_backward(*pos, t_stop=1e-4, grad_mode=lib.GRAD_TC_FULL)
    with pytest.raises(RuntimeError, match="CUDA"):
        backend.render_backward(*pos, t_stop=1e-4, target_rgb=torch.zeros(4, 3))
    # FineTuner: a CPU volume is refused at construction, and a step on CPU samples before any launch
    with pytest.raises(RuntimeError, match="CUDA"):
        backend.FineTuner(pos[7], backend.RefVolume(kw["volume_feature"]), kw["imgs"], kw["pose_ref"])
    tuner = object.__new__(backend.FineTuner)
    tuner.grad_mode, tuner.lr, tuner.step_count, tuner.loss = lib.MLP_FP32, 5e-4, 0, torch.zeros(1)
    tuner.pose_ref, tuner.volume, tuner.imgs, tuner.network_fn = kw["pose_ref"], kw["volume_feature"], kw["imgs"], pos[7]
    tuner.white_bkgd, tuner.vol_g, tuner.g = False, None, None
    with pytest.raises(RuntimeError, match="CUDA"):
        tuner.step(*pos[1:5], torch.zeros(4, 3), t_stop=1e-4)
    with pytest.raises(RuntimeError, match="t_stop"):
        tuner.step(*pos[1:5], torch.zeros(4, 3), t_stop=-1.0)


def _args(**extra):
    return SimpleNamespace(multires=10, i_embed=0, pts_dim=3, multires_views=4, dir_dim=3, netdepth=6, netwidth=128,
                           feat_dim=20, net_type="v0", N_importance=0, netchunk=1024, ckpt=None, perturb=1.0,
                           N_samples=128, use_viewdirs=True, white_bkgd=False, raw_noise_std=0.0, **extra)


def test_create_nerf_mvs_adds_t_stop_only_when_args_has_one():
    keys = {"network_query_fn", "perturb", "N_importance", "network_fine", "N_samples", "network_fn", "network_mvs",
            "use_viewdirs", "white_bkgd", "raw_noise_std"}
    cpu = torch.device("cpu")
    for args in (_args(), _args(t_stop=None)):
        train, test, _, _ = backend.create_nerf_mvs(args, dir_embedder=False, device=cpu)
        assert set(train) == keys and set(test) == keys
    train, test, _, _ = backend.create_nerf_mvs(_args(t_stop=1e-4), dir_embedder=False, device=cpu)
    assert set(train) == keys | {"t_stop"} and set(test) == keys | {"t_stop"}
    assert train["t_stop"] == test["t_stop"] == 1e-4 and test["perturb"] is False
    train, _, _, _ = backend.create_nerf_mvs(_args(t_stop=0), dir_embedder=False, device=cpu)
    assert train["t_stop"] == 0.0
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="CUDA"):
            backend.create_nerf_mvs(_args(t_stop=1e-4), dir_embedder=False)
