"""CPU: the C-ABI library builds/loads and exports every declared symbol; host-side mirror logic
(state_dict compatibility with the reference checkpoint, loud failures without a GPU)."""
import ctypes
import os
import re

import pytest
import torch

from conftest import GOLDEN, ROOT
from mvsnerf_b200 import backend, lib, synthetic


@pytest.fixture(scope="module")
def built():
    from mvsnerf_b200 import build
    return build.build_library()


def test_abi2_library_exports_every_declared_symbol(built):
    header = open(os.path.join(ROOT, "include", "mvsnerf_b200.h")).read()
    declared = sorted(set(re.findall(r"\b(mvsn_[a-z0-9_]+)\s*\(", header)))
    assert declared == sorted(lib.EXPORTS)
    dll = ctypes.CDLL(built)
    for name in declared:
        assert hasattr(dll, name), name
    L = lib.load()
    assert L.mvsn_abi_version() == 2
    assert L.mvsn_mlp_packed_bytes(lib.MLP_FP32) > 126788 * 4
    assert L.mvsn_costreg_workspace_bytes(128, 176, 208) > 400e6
    assert L.mvsn_cost_volume_workspace_bytes(3, 128, 160) == 3 * 128 * 160 * (4 + 32) * 4
    assert L.mvsn_featurenet_workspace_bytes(3, 512, 640) == 4096 + 2 * 3 * 8 * 512 * 640 * 4


def test_argument_errors_do_not_need_a_gpu(built):
    L = lib.load()
    rc = L.mvsn_pack_images(None, 3, 4, 4, None, None)
    assert rc == -4 and b"NULL" in L.mvsn_last_error()
    rc = L.mvsn_costreg_forward(None, None, 128, 20, 24, None, None, 0, None)
    assert rc == -4
    rc = L.mvsn_featurenet_forward(None, None, 3, 32, 32, None, None, 0, None)
    assert rc == -4 and b"featurenet" in L.mvsn_last_error()
    assert L.mvsn_mlp_packed_bytes(99) == 0


def test_state_dict_keys_match_reference_checkpoint():
    import numpy as np
    z = np.load(os.path.join(GOLDEN, "mvsnerf_v0_weights.npz"))
    fn, mvs = backend.MVSNeRF(), backend.MVSNet()
    assert sorted(fn.state_dict().keys()) == sorted(k[4:] for k in z.files if k.startswith("mlp/"))
    assert sorted(mvs.state_dict().keys()) == sorted(k[4:] for k in z.files if k.startswith("mvs/"))
    backend.load_weights_npz(fn, mvs, os.path.join(GOLDEN, "mvsnerf_v0_weights.npz"))   # strict load
    assert len(fn.ordered_params()) == lib.N_MLP_TENSORS
    assert len(mvs.cost_reg_2.weight_list()) == lib.N_COSTREG_TENSORS
    assert len(mvs.feature.weight_list()) == lib.N_FEATURENET_TENSORS
    assert mvs.feature.weight_list()[6].shape == (16, 8, 5, 5) and mvs.feature.weight_list()[24].shape == (32, 32, 1, 1)
    assert sum(p.numel() for p in fn.parameters()) == 126788


def test_pytorch_mirror_of_mlp_matches_oracle(weights):
    """MVSNeRF.forward (kept for the alpha-only callers) is the same function as the oracle MLP."""
    from oracle import mvsnerf_oracle as orc
    fn = backend.MVSNeRF()
    backend.load_weights_npz(fn, None, os.path.join(GOLDEN, "mvsnerf_v0_weights.npz"))
    x = torch.rand(50, 7, 86, generator=torch.Generator().manual_seed(0))
    with torch.no_grad():
        assert (fn(x) - orc.mlp(x, weights)).abs().max() < 1e-6


def test_no_silent_cpu_fallback():
    fn, mvs = backend.MVSNeRF(), backend.MVSNet().train()
    sc = synthetic.make_scene(32, 32, pad=4, seed=0)
    with pytest.raises(RuntimeError):
        mvs(sc.imgs_norm, sc.proj_mats, sc.near_far, pad=4)
    with pytest.raises(RuntimeError):
        fn.packed()
    with pytest.raises(RuntimeError):
        backend.render_rays(synthetic.scene_rays(sc), torch.zeros(1, 8, 128, 16, 16), sc.imgs_raw, sc.pose_source,
                            fn, sc.near_far, 4.0)
    with pytest.raises(RuntimeError):
        backend.MVSNet().eval()(sc.imgs_norm, sc.proj_mats, sc.near_far)       # eval mode exists, but not on the CPU


def test_synthetic_scene_contract():
    sc = synthetic.make_scene(64, 96, pad=4, seed=3)
    assert sc.imgs_norm.shape == (1, 3, 3, 64, 96) and sc.proj_mats.shape == (1, 3, 3, 4)
    assert torch.allclose(sc.proj_mats[0, 0], torch.eye(4)[:3])
    rays = synthetic.scene_rays(sc)
    assert rays.shape == (64 * 96, 8) and float(rays[0, 6]) == pytest.approx(sc.near_far[0])
    sc2 = synthetic.make_scene(64, 96, pad=4, seed=3)
    assert torch.equal(sc.imgs_raw, sc2.imgs_raw)


def test_backward_recompute_is_the_oracle_function(weights):
    """The PyTorch statement that _RenderSamplesFn.backward differentiates is the same function as the
    oracle's render_samples (values and gradients), checked on the CPU where no kernel is involved."""
    from oracle import mvsnerf_oracle as orc
    sc = synthetic.make_scene(32, 32, pad=4, seed=1)
    vol = torch.randn(1, 8, 16, 16, 16, generator=torch.Generator().manual_seed(2))
    rays = synthetic.scene_rays(sc)[::37][:24]
    pts, z = orc.march_rays(rays, 8)
    ndc = orc.ndc_coords(sc.pose_source["w2cs"][0], sc.pose_source["intrinsics"][0], pts, sc.H, sc.W,
                         sc.near_far[0], sc.near_far[1], 4.0)
    fn = backend.MVSNeRF()
    backend.load_weights_npz(fn, None, os.path.join(GOLDEN, "mvsnerf_v0_weights.npz"))
    v1 = vol.clone().requires_grad_(True)
    a = backend._render_samples_torch(pts, ndc, z, rays[:, 3:6], v1, sc.imgs_raw, sc.pose_source["w2cs"],
                                      sc.pose_source["intrinsics"], fn, True)
    wt = {k: v.clone().requires_grad_(k.startswith("mlp/")) for k, v in weights.items()}
    v2 = vol.clone().requires_grad_(True)
    b = orc.render_samples(pts, ndc, z, rays[:, 3:6], v2, sc.imgs_raw, sc.pose_source, wt, white_bkgd=True)
    for x, y in zip(a, b):
        assert (x - y).abs().max() < 1e-5
    (a[0].sum() + a[3].sum()).backward()
    (b[0].sum() + b[3].sum()).backward()
    assert (v1.grad - v2.grad).abs().max() <= 1e-5 * v2.grad.abs().max() + 1e-8
    for name, p in fn.named_parameters():
        g = wt["mlp/" + name].grad
        assert (p.grad - g).abs().max() <= 1e-4 * g.abs().max() + 1e-8, name
    assert [n for n, _ in backend._ordered_named_params(fn)][:2] == ["nerf.pts_linears.0.weight", "nerf.pts_linears.0.bias"]


def test_autograd_plumbing_of_rendering(monkeypatch):
    """rendering() under autograd: argument/gradient routing of _RenderSamplesFn, exercised on the CPU with the
    kernel launch stubbed out (the GPU test checks the same against the real kernel and the oracle)."""
    from oracle import mvsnerf_oracle as orc
    sc = synthetic.make_scene(32, 32, pad=4, seed=1)
    rays = synthetic.scene_rays(sc)[::41][:16]
    pts, z = orc.march_rays(rays, 6)
    ndc = orc.ndc_coords(sc.pose_source["w2cs"][0], sc.pose_source["intrinsics"][0], pts, sc.H, sc.W,
                         sc.near_far[0], sc.near_far[1], 4.0)
    fn = backend.MVSNeRF()
    backend.load_weights_npz(fn, None, os.path.join(GOLDEN, "mvsnerf_v0_weights.npz"))
    volume = backend.RefVolume(torch.randn(1, 8, 16, 16, 16, generator=torch.Generator().manual_seed(2)))

    def fake_kernel(pose_ref, rays_pts, rays_ndc, zz, rays_dir, volume_feature, imgs, network_fn, white_bkgd, mode,
                    want_aux=True):
        assert not torch.is_grad_enabled()
        return backend._render_samples_torch(rays_pts, rays_ndc, zz, rays_dir, volume_feature.feat_volume, imgs,
                                             pose_ref["w2cs"], pose_ref["intrinsics"], network_fn, white_bkgd)

    monkeypatch.setattr(backend, "_render_samples_kernel", fake_kernel)
    monkeypatch.setattr(backend, "BACKWARD_IMPL", "torch")       # the kernel backward needs a GPU (tests/test_gpu_backward.py)

    class A:
        use_color_volume = False
    out = backend.rendering(A(), sc.pose_source, pts, ndc, z, rays[:, :3], rays[:, 3:6], volume_feature=volume,
                            imgs=sc.imgs_raw, network_fn=fn, white_bkgd=False, perturb=0, N_importance=0)
    assert len(out) == 6 and out[0].requires_grad and out[5] == {}
    (out[0].sum() + 0.5 * out[3].sum() + 0.1 * out[2].sum()).backward()
    got = {n: p.grad.clone() for n, p in fn.named_parameters()}
    gv = volume.feat_volume.grad.clone()
    fn.zero_grad(); volume.zero_grad()
    ref = backend._render_samples_torch(pts, ndc, z, rays[:, 3:6], volume.feat_volume, sc.imgs_raw, sc.pose_source["w2cs"],
                                        sc.pose_source["intrinsics"], fn, False)
    (ref[0].sum() + 0.5 * ref[3].sum() + 0.1 * ref[2].sum()).backward()
    for n, p in fn.named_parameters():
        assert torch.allclose(got[n], p.grad, rtol=1e-5, atol=1e-8), n
    assert torch.allclose(gv, volume.feat_volume.grad, rtol=1e-5, atol=1e-9)
    # only the volume trainable
    for p in fn.parameters():
        p.requires_grad_(False)
    fn.zero_grad(set_to_none=True)
    volume.zero_grad(set_to_none=True)
    out = backend.rendering(A(), sc.pose_source, pts, ndc, z, rays[:, :3], rays[:, 3:6], volume_feature=volume,
                            imgs=sc.imgs_raw, network_fn=fn)
    out[0].sum().backward()
    assert volume.feat_volume.grad is not None and all(p.grad is None for p in fn.parameters())


def test_ray_marcher_and_ndc_mirrors_match_the_oracle():
    """backend.ray_marcher / backend.get_ndc_coordinate (the host functions the fine-tuning step calls before `rendering`,
    data/ray_utils.py:152-197, utils.py:112-146) against the oracle's restatement, bit for bit, incl. lindisp and pad."""
    from oracle import mvsnerf_oracle as orc
    sc = synthetic.make_scene(64, 96, pad=8, seed=2)
    rays = synthetic.scene_rays(sc)[::7].contiguous()
    for lindisp in (False, True):
        xyz, ro, rd, z = backend.ray_marcher(rays, N_samples=24, lindisp=lindisp, perturb=0)
        pts, z2 = orc.march_rays(rays, 24, lindisp)
        assert torch.equal(xyz, pts) and torch.equal(z, z2)
        assert torch.equal(ro, rays[:, :3]) and torch.equal(rd, rays[:, 3:6])
        for pad in (0, 8):
            ndc = backend.get_ndc_coordinate(sc.pose_source["w2cs"][0], sc.pose_source["intrinsics"][0], xyz,
                                             torch.tensor([sc.W - 1.0, sc.H - 1.0]), near=sc.near_far[0], far=sc.near_far[1],
                                             pad=pad, lindisp=lindisp)
            ref = orc.ndc_coords(sc.pose_source["w2cs"][0], sc.pose_source["intrinsics"][0], xyz, sc.H, sc.W, sc.near_far[0],
                                 sc.near_far[1], float(pad), lindisp)
            assert torch.equal(ndc, ref)
    # perturb > 0: stratified samples stay inside their bins and are reproducible under a seed
    torch.manual_seed(0)
    _, _, _, za = backend.ray_marcher(rays, N_samples=24, perturb=1.0)
    torch.manual_seed(0)
    _, _, _, zb = backend.ray_marcher(rays, N_samples=24, perturb=1.0)
    _, _, _, z0 = backend.ray_marcher(rays, N_samples=24, perturb=0)
    assert torch.equal(za, zb) and not torch.equal(za, z0)
    mid = 0.5 * (z0[:, 1:] + z0[:, :-1])
    assert bool((za[:, 1:-1] >= mid[:, :-1] - 1e-6).all()) and bool((za[:, 1:-1] <= mid[:, 1:] + 1e-6).all())


def test_finetuner_and_backward_refuse_cpu_tensors():
    fn = backend.MVSNeRF()
    vol = backend.RefVolume(torch.zeros(1, 8, 8, 8, 8))
    sc = synthetic.make_scene(32, 32, pad=0, seed=0)
    with pytest.raises(RuntimeError):
        backend.FineTuner(fn, vol, sc.imgs_raw, sc.pose_source)
    with pytest.raises(RuntimeError):
        backend.render_backward(sc.pose_source, torch.zeros(4, 8, 3), torch.zeros(4, 8, 3), torch.zeros(4, 8), torch.zeros(4, 3),
                                vol, sc.imgs_raw, fn, grads={"rgb": torch.zeros(4, 3)})


def test_pack_pixels_layout():
    from mvsnerf_b200.distributed import pack_pixels
    rgb, depth = torch.arange(12.0).view(4, 3), torch.arange(4.0) + 100
    px = pack_pixels(rgb, depth)
    assert px.shape == (4, 4) and torch.equal(px[:, :3], rgb) and torch.equal(px[:, 3], depth)
