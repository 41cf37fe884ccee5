"""Importance sampling without a GPU: the restatement in tests/importance_oracle.py against the reference's own
sample_pdf / ray_marcher_fine (the committed fixture, and the live reference where its source tree is present), the
new entries exported and declared, their argument errors returned before any CUDA call, from C and from Python, and
create_nerf_mvs with N_importance > 0."""
import ctypes as C
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from mvsnerf_b200 import backend, lib
import importance_oracle as io_orc

NEW = ["mvsn_build_density_workspace_bytes", "mvsn_build_density", "mvsn_sample_importance"]


def _fixture():
    z = np.load(os.path.join(GOLDEN, "importance_16x12x10.npz"))
    return {k: torch.from_numpy(z[k]) for k in z.files}


def test_oracle_matches_the_reference_fixture():
    f = _fixture()
    xyz, z, _ = io_orc.ray_marcher_fine(f["rays"], f["grid"], f["z_vals"], f["pts_ndc"], f["u"], ref_mapping=True)
    assert (z - f["z_fine"]).abs().max() <= 1e-6 * f["z_fine"].abs().max()
    assert (xyz - f["xyz"]).abs().max() <= 1e-6 * f["xyz"].abs().max()
    det, _ = io_orc.sample_pdf(f["bins"], f["weights"], io_orc.linspace_u(*f["det_samples"].shape))
    assert (det - f["det_samples"]).abs().max() <= 1e-6 * f["det_samples"].abs().max()
    # the default mapping differs from the reference's only through the lookup coordinate: fed 2 ndc - 1 (which it maps
    # to the reference's 4 ndc - 3), it reproduces the reference
    xyz2, z2, _ = io_orc.ray_marcher_fine(f["rays"], f["grid"], f["z_vals"], f["pts_ndc"] * 2 - 1.0, f["u"])
    assert torch.equal(z2, z) and torch.equal(xyz2, xyz)
    _, z3, _ = io_orc.ray_marcher_fine(f["rays"], f["grid"], f["z_vals"], f["pts_ndc"], f["u"])
    assert not torch.equal(z3, z)
    # float64 against float32: the same samples to fp32 rounding almost everywhere
    _, z64, _ = io_orc.ray_marcher_fine(f["rays"].double(), f["grid"].double(), f["z_vals"].double(),
                                        f["pts_ndc"].double(), f["u"].double(), ref_mapping=True)
    assert ((z64 - f["z_fine"].double()).abs() <= 1e-5).double().mean() > 0.999


def test_oracle_matches_the_live_reference():
    from oracle import ref_shim
    if not ref_shim.reference_available():
        pytest.skip("reference source tree not present")
    ref = ref_shim.load_reference()
    f = _fixture()
    torch.manual_seed(31)
    xyz, _, _, z = ref.ray_utils.ray_marcher_fine(f["rays"], f["grid"], f["z_vals"], f["pts_ndc"], N_importance=17)
    torch.manual_seed(31)
    u = torch.rand(f["rays"].shape[0], 17)
    xyz_o, z_o, _ = io_orc.ray_marcher_fine(f["rays"], f["grid"], f["z_vals"], f["pts_ndc"], u, ref_mapping=True)
    assert (z_o - z).abs().max() <= 1e-6 * z.abs().max()
    assert (xyz_o - xyz).abs().max() <= 1e-6 * xyz.abs().max()


def test_symbols_exported_and_declared():
    L = lib.load()
    with open(os.path.join(ROOT, "include", "mvsnerf_b200.h")) as fh:
        header = fh.read()
    for name in NEW:
        assert name in lib.EXPORTS and hasattr(L, name)
        assert f" {name}(" in header, name
    assert "typedef struct mvsn_density" in header
    assert L.mvsn_abi_version() == 2


class Buf:
    def __init__(self):
        self.mem = (C.c_float * 4096)()
        self.addr = (C.addressof(self.mem) + 15) & ~15


def _scene(b, mode, dims=(8, 8, 8)):
    return lib.RenderScene(b.addr, *dims, b.addr, 3, 8, 8, b.addr, b.addr, b.addr, mode, 0)


def _sample(S=8, K=8, N=4, grid_dims=(8, 8, 8), scene=True, rays_off=0, sigma_off=0, source="march", jitter=False,
            ndc_out=True, density=True):
    L, b = lib.load(), Buf()
    sc = _scene(b, lib.MLP_TC_SPLIT)
    rp = lib.RayParams(2.0, 6.0, 0.0, 0)
    grid = lib.DensityGrid(b.addr + sigma_off, *grid_dims)
    a = b.addr
    t_steps, z, ndc = (a, None, None) if source == "march" else (None, a, a) if source == "given" else \
        (None, a, None) if source == "no_ndc" else (a, a, a)
    rc = L.mvsn_sample_importance(C.byref(sc) if scene else None, C.byref(rp) if scene else None,
                                  C.byref(grid) if density else None, a + rays_off, t_steps, a if jitter else None, z,
                                  ndc, None, N, S, K, a, a, a if ndc_out else None, None)
    return rc, L.mvsn_last_error().decode()


def test_sampler_argument_errors():
    assert _sample(S=2)[0] == -1                                                    # MVSN_EBADSHAPE
    assert _sample(K=0)[0] == -1
    assert _sample(N=-1)[0] == -1
    rc, msg = _sample(S=1000, K=25)
    assert rc == -6 and "1024" in msg                                               # MVSN_EUNSUPPORTED
    assert _sample(density=False)[0] == -4                                          # MVSN_ENULL
    assert _sample(source="both")[0] == -4
    assert _sample(source="no_ndc")[0] == -4
    assert _sample(source="given", jitter=True)[0] == -6
    assert _sample(scene=False)[0] == -4                                            # the march needs the cameras
    assert _sample(scene=False, source="given")[0] == -4                            # and so does ndc_out
    assert _sample(rays_off=4)[0] == -2                                             # MVSN_EALIGN
    assert _sample(sigma_off=2)[0] == -2
    for dims in ((8, 8, 16), (4, 8, 8), (8, 16, 8)):
        rc, msg = _sample(grid_dims=dims)
        assert rc == -1 and "does not match" in msg, dims
    assert _sample(grid_dims=(1, 8, 8), scene=False, source="given", ndc_out=False)[0] == -1
    # the caller's samples without ndc_out need no scene, and N = 0 returns before any CUDA call
    assert _sample(N=0, scene=False, source="given", ndc_out=False)[0] == 0
    assert _sample(N=0)[0] == 0


def _density(mode=lib.MLP_FP32, sigma_off=0, ws_off=0, ws_bytes=1 << 30, dims=(8, 8, 8)):
    L, b = lib.load(), Buf()
    sc = _scene(b, mode, dims)
    rp = lib.RayParams(2.0, 6.0, 0.0, 0)
    rc = L.mvsn_build_density(C.byref(sc), C.byref(rp), b.addr + sigma_off, b.addr + ws_off, ws_bytes, None)
    return rc, L.mvsn_last_error().decode()


def test_density_sizes_and_argument_errors():
    L = lib.load()
    assert L.mvsn_build_density_workspace_bytes(1, 8, 8) == 0
    assert L.mvsn_build_density_workspace_bytes(8, 8, 8) >= 8 * 8 * 8 * 28
    rc, msg = _density(mode=lib.MLP_TC_SPLIT)
    assert rc == -6 and "MVSN_MLP_FP32" in msg
    assert _density(dims=(1, 8, 8))[0] == -1
    rc, msg = _density(sigma_off=2)
    assert rc == -2 and "sigma" in msg
    rc, msg = _density(ws_off=4)
    assert rc == -2 and "workspace" in msg
    assert _density(ws_bytes=16)[0] == -5


def test_python_rejections_without_a_device():
    occ = backend.Occupancy(torch.zeros(16, dtype=torch.int32), 8, 8, 8, (2.0, 6.0), 0.0, False, 1)
    den = backend.Density(torch.zeros(8, 8, 8), (2.0, 6.0), 0.0, False)
    for kw in ({"occupancy": occ}, {"sink": object()}):
        with pytest.raises(RuntimeError, match="occupancy or sink"):
            backend.render_rays(torch.zeros(4, 8), None, None, None, None, (2.0, 6.0), 0.0, density=den,
                                N_importance=8, **kw)
    with pytest.raises(RuntimeError, match="needs density"):
        backend.render_rays(torch.zeros(4, 8), None, None, None, None, (2.0, 6.0), 0.0, N_importance=8)
    with pytest.raises(RuntimeError, match="N_importance"):
        backend.render_rays(torch.zeros(4, 8), None, None, None, None, (2.0, 6.0), 0.0, density=den, N_importance=0)
    with pytest.raises(RuntimeError, match="1024"):
        backend.render_rays(torch.zeros(4, 8), None, None, None, None, (2.0, 6.0), 0.0, N_samples=1000, density=den,
                            N_importance=25)
    with pytest.raises(RuntimeError, match="near_far"):
        backend.render_rays(torch.zeros(4, 8), None, None, None, None, (2.0, 7.0), 0.0, density=den, N_importance=8)
    with pytest.raises(RuntimeError, match="Density"):
        backend.render_rays(torch.zeros(4, 8), None, None, None, None, (2.0, 6.0), 0.0, density=torch.zeros(8, 8, 8),
                            N_importance=8)
    with pytest.raises(RuntimeError, match="N_samples >= 3"):
        backend.ray_marcher_fine(torch.zeros(4, 8), den, torch.zeros(4, 2), torch.zeros(4, 2, 3), N_importance=4)
    tuner = object.__new__(backend.FineTuner)
    tuner.lr, tuner.grad_mode = 1e-3, lib.MLP_FP32
    with pytest.raises(RuntimeError, match="128"):
        tuner.step_rays(torch.zeros(4, 8), None, (2.0, 6.0), 0.0, N_samples=128, density=den, N_importance=64)
    with pytest.raises(RuntimeError, match="needs density"):
        tuner.step_rays(torch.zeros(4, 8), None, (2.0, 6.0), 0.0, N_samples=64, N_importance=64)
    tuner.grad_mode = lib.GRAD_TC_FULL
    with pytest.raises(RuntimeError, match="GRAD_TC_FULL"):
        tuner.step_rays(torch.zeros(4, 8), None, (2.0, 6.0), 0.0, N_samples=64, density=den, N_importance=64)


def _args(**extra):
    return SimpleNamespace(multires=10, i_embed=0, pts_dim=3, multires_views=4, dir_dim=3, netdepth=6, netwidth=128,
                           feat_dim=20, net_type="v0", netchunk=1024, ckpt=None, perturb=1.0, N_samples=128,
                           use_viewdirs=True, white_bkgd=False, raw_noise_std=0.0, **extra)


def test_create_nerf_mvs_with_n_importance():
    keys = {"network_query_fn", "perturb", "N_importance", "network_fine", "N_samples", "network_fn", "network_mvs",
            "use_viewdirs", "white_bkgd", "raw_noise_std"}
    cpu = torch.device("cpu")
    train, test, _, grad_vars = backend.create_nerf_mvs(_args(N_importance=64), dir_embedder=False, device=cpu)
    assert set(train) == keys and set(test) == keys
    assert isinstance(train["network_fine"], backend.MVSNeRF) and test["network_fine"] is train["network_fine"]
    n_fn = len(list(train["network_fn"].parameters()))
    assert len(grad_vars) == 2 * n_fn
    assert all(a is b for a, b in zip(grad_vars[n_fn:], train["network_fine"].parameters()))
    train, _, _, grad_vars = backend.create_nerf_mvs(_args(N_importance=0), dir_embedder=False, device=cpu)
    assert train["network_fine"] is None and len(grad_vars) == n_fn


def test_render_density_is_the_reference_loop():
    fn = backend.MVSNeRF()
    pts, feats = torch.rand(700, 3), torch.rand(700, 20)
    calls = []

    def query(p, viewdirs, f, net):
        calls.append(p.shape[0])
        assert viewdirs is None and net is fn
        return p[:, :1] + f[:, :1]
    out = backend.render_density(fn, pts, feats, query, chunk=256)
    assert calls == [256, 256, 188]
    assert torch.equal(out, pts[:, :1] + feats[:, :1])
