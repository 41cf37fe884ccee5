"""GPU: the fine-tuning step kernels (csrc/render_bwd.cu, SURVEY.md 8(f) row 2) against three independent statements:

  * the oracle's autograd on the CPU (reference semantics: train_mvs_nerf_finetuning_pl.py:140-189 differentiates
    renderer.rendering; tests/test_gpu_parity.py::test_rendering_gradients_vs_oracle_autograd covers the loss the script
    uses; here EVERY output of `rendering` carries a random cotangent),
  * the PyTorch-recompute backward (backend.BACKWARD_IMPL = "torch") on the same GPU,
  * torch.optim.Adam for the fused Adam kernels.
"""
import os

import pytest
import torch

from conftest import GOLDEN
from oracle import mvsnerf_oracle as orc
from mvsnerf_b200 import backend, lib, synthetic

pytestmark = pytest.mark.gpu
DEV = "cuda"
WPATH = os.path.join(GOLDEN, "mvsnerf_v0_weights.npz")


class Args:
    use_color_volume = False


@pytest.fixture(scope="module")
def scene(weights):
    sc = synthetic.make_scene(96, 128, pad=4, seed=9)
    vol = orc.encode_volume(sc.imgs_norm, sc.proj_mats, sc.near_far, sc.pad, weights)
    return sc, vol


def _samples(sc, n, S, seed, perturb=0.0):
    rays = synthetic.scene_rays(sc)
    rays = rays[torch.randperm(rays.shape[0], generator=torch.Generator().manual_seed(seed))[:n]].contiguous()
    torch.manual_seed(seed)
    pts, _, _, z = backend.ray_marcher(rays, N_samples=S, perturb=perturb)
    ndc = backend.get_ndc_coordinate(sc.pose_source["w2cs"][0], sc.pose_source["intrinsics"][0], pts,
                                     torch.tensor([sc.W - 1.0, sc.H - 1.0]), near=sc.near_far[0], far=sc.near_far[1], pad=sc.pad)
    return rays, pts.contiguous(), ndc.contiguous(), z.contiguous()


def _cotangents(n, S, seed):
    g = torch.Generator().manual_seed(seed)
    return {"rgb": torch.randn(n, 3, generator=g), "depth": 0.1 * torch.randn(n, generator=g),
            "weights": 0.05 * torch.randn(n, S, generator=g), "alpha": 0.05 * torch.randn(n, S, generator=g),
            "input_feat": 0.01 * torch.randn(n, S, 20, generator=g)}


def _assert_close(a, b, rel, what):
    scale = b.abs().max().item()
    err = (a - b).abs().max().item()
    assert err <= rel * scale + 1e-8, (what, err, scale)


@pytest.mark.parametrize("S,n,white", [(128, 37, False), (32, 130, True), (48, 21, False), (128, 300, True)])
def test_backward_kernel_vs_oracle_autograd_all_outputs(scene, weights, S, n, white):
    """Random cotangents on rgb, depth, weights, alpha and input_feat; N_samples 128 (one ray per tile), 32 (four rays
    per tile), 48 (two rays per tile + 32 idle rows); ragged ray counts; white_bkgd on and off."""
    sc, vol_ref = scene
    rays, pts, ndc, z = _samples(sc, n, S, seed=S + n, perturb=1.0)
    cot = _cotangents(n, S, seed=1)
    # oracle autograd on the CPU
    wt = {k: v.clone().requires_grad_(k.startswith("mlp/")) for k, v in weights.items()}
    vt = vol_ref.clone().requires_grad_(True)
    rgb, feat, w, depth, alpha = orc.render_samples(pts, ndc, z, rays[:, 3:6], vt, sc.imgs_raw, sc.pose_source, wt, white_bkgd=white)
    loss = (rgb * cot["rgb"]).sum() + (depth * cot["depth"]).sum() + (w * cot["weights"]).sum() + \
        (alpha * cot["alpha"]).sum() + (feat * cot["input_feat"]).sum()
    loss.backward()
    # kernel
    fn = backend.MVSNeRF().to(DEV)
    backend.load_weights_npz(fn, None, WPATH)
    d = sc.to(DEV)
    vol = vol_ref.to(DEV)
    grads = {k: v.to(DEV) for k, v in cot.items()}
    g_mlp, g_vol, rgb_k, depth_k = backend.render_backward(d.pose_source, pts.to(DEV), ndc.to(DEV), z.to(DEV), rays[:, 3:6].to(DEV),
                                                           vol, d.imgs_raw, fn, white, grads=grads, want_forward=True)
    assert (rgb_k.cpu() - rgb.detach()).abs().max() < 1e-5 and (depth_k.cpu() - depth.detach()).abs().max() < 1e-4
    for (name, p), g in zip(backend._ordered_named_params(fn), g_mlp):
        _assert_close(g.cpu(), wt["mlp/" + name].grad, 2e-4, name)
    _assert_close(g_vol.permute(3, 0, 1, 2).unsqueeze(0).cpu(), vt.grad, 2e-4, "volume")


@pytest.mark.parametrize("S,n,white", [(32, 130, True), (48, 21, False), (128, 37, False), (128, 300, True)])
def test_backward_recompute_renders_what_the_fp32_kernel_renders(scene, S, n, white):
    """The backward kernel's forward recompute and mlp_mode=MLP_FP32 rendering run the same fp32 forward tile, so the
    rgb the backward reports is bit-identical to the render kernel's on the same samples.  Depth is composed with
    different rounding in the two kernels (fmaf vs multiply-then-add), so it agrees to 1e-6 only."""
    sc, vol_ref = scene
    rays, pts, ndc, z = _samples(sc, n, S, seed=S + n, perturb=1.0)
    fn = backend.MVSNeRF().to(DEV)
    backend.load_weights_npz(fn, None, WPATH)
    d = sc.to(DEV)
    vol = vol_ref.to(DEV)
    pts, ndc, z, rd = pts.to(DEV), ndc.to(DEV), z.to(DEV), rays[:, 3:6].to(DEV)
    _, _, rgb_b, depth_b = backend.render_backward(d.pose_source, pts, ndc, z, rd, vol, d.imgs_raw, fn, white,
                                                   grads={"rgb": torch.ones(n, 3, device=DEV)}, want_forward=True)
    with torch.no_grad():
        rgb_f, _, _, depth_f, _, _ = backend.rendering(Args(), d.pose_source, pts, ndc, z, None, rd, volume_feature=vol,
                                                       imgs=d.imgs_raw, network_fn=fn, white_bkgd=white,
                                                       mlp_mode=lib.MLP_FP32)
    assert torch.equal(rgb_b, rgb_f), (rgb_b - rgb_f).abs().max().item()
    assert (depth_b - depth_f).abs().max().item() <= 1e-6


@pytest.mark.parametrize("tag,white", [("s32", False), ("s128w", True)])
def test_backward_kernel_vs_reference_gradient_fixture(golden_grad, golden_tiny, tag, white):
    """The fused-loss launch (img2mse formed in the kernel) against gradients the unmodified reference's autograd
    produced (tests/golden/make_golden_grad.py): loss, every MLP parameter, the encoding volume."""
    g = {k[len(tag) + 1:]: v for k, v in golden_grad.items() if k.startswith(tag + "/")}
    t = golden_tiny
    pose = {"w2cs": t["w2cs"].to(DEV), "c2ws": t["c2ws"].to(DEV), "intrinsics": t["intrinsics"].to(DEV)}
    fn = backend.MVSNeRF().to(DEV)
    backend.load_weights_npz(fn, None, WPATH)
    loss = torch.zeros(1, device=DEV)
    g_mlp, g_vol, rgb, _ = backend.render_backward(pose, g["xyz"].to(DEV), g["ndc"].to(DEV), g["z"].to(DEV),
                                                   g["rays"][:, 3:6].to(DEV), t["volume"].to(DEV), t["imgs_raw"].to(DEV), fn,
                                                   white, target_rgb=g["target"].to(DEV), want_forward=True, loss_out=loss)
    assert (rgb.cpu() - g["rgb"]).abs().max() < 1e-5
    assert abs(loss.item() - float(g["loss"])) < 1e-5 * max(1.0, float(g["loss"]))
    for (name, p), gk in zip(backend._ordered_named_params(fn), g_mlp):
        _assert_close(gk.cpu(), g["grad_mlp/" + name], 2e-4, name)
    ref_v = torch.zeros(t["volume"].numel())
    ref_v[g["grad_volume_idx"]] = g["grad_volume_val"]
    _assert_close(g_vol.permute(3, 0, 1, 2).reshape(-1).cpu(), ref_v, 2e-4, "volume")


def test_autograd_function_kernel_vs_torch_recompute(scene):
    """backend.rendering under autograd: the kernel backward and the PyTorch-recompute backward agree (planar AND
    channels-last RefVolume parameters), and gradients land with the parameter's own layout."""
    sc, vol_ref = scene
    n, S = 200, 64
    rays, pts, ndc, z = _samples(sc, n, S, seed=5)
    d = sc.to(DEV)
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    results = {}
    for impl in ("kernel", "torch"):
        for layout in ("planar", "channels_last"):
            fn = backend.MVSNeRF().to(DEV)
            backend.load_weights_npz(fn, None, WPATH)
            v = vol_ref.clone().to(DEV)
            if layout == "channels_last":
                v = v[0].permute(1, 2, 3, 0).contiguous().permute(3, 0, 1, 2).unsqueeze(0)
            volume = backend.RefVolume(v)
            old = backend.BACKWARD_IMPL
            backend.BACKWARD_IMPL = impl
            try:
                rgb, _, w, depth, _, _ = backend.rendering(Args(), d.pose_source, pts.to(DEV), ndc.to(DEV), z.to(DEV), None,
                                                           rays[:, 3:6].to(DEV), volume_feature=volume, imgs=d.imgs_raw,
                                                           network_fn=fn, mlp_mode=lib.MLP_FP32)
                (((rgb - target) ** 2).mean() + 0.1 * depth.mean() + 0.01 * w.sum(-1).mean()).backward()
            finally:
                backend.BACKWARD_IMPL = old
            assert volume.feat_volume.grad.shape == volume.feat_volume.shape
            results[(impl, layout)] = ([p.grad.clone() for p in fn.ordered_params()], volume.feat_volume.grad.clone())
    ref_p, ref_v = results[("torch", "planar")]
    for key, (gp, gv) in results.items():
        for a, b in zip(gp, ref_p):
            _assert_close(a, b, 2e-4, key)
        _assert_close(gv, ref_v, 2e-4, key)


def test_fused_loss_mode_equals_explicit_gradient(scene):
    sc, vol_ref = scene
    n, S = 96, 128
    rays, pts, ndc, z = _samples(sc, n, S, seed=11)
    d = sc.to(DEV)
    fn = backend.MVSNeRF().to(DEV)
    backend.load_weights_npz(fn, None, WPATH)
    vol = vol_ref.to(DEV)
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(3)).to(DEV)
    args = (d.pose_source, pts.to(DEV), ndc.to(DEV), z.to(DEV), rays[:, 3:6].to(DEV), vol, d.imgs_raw, fn, True)
    loss = torch.zeros(1, device=DEV)
    g1, v1, rgb, _ = backend.render_backward(*args, target_rgb=target, want_forward=True, loss_out=loss)
    assert abs(loss.item() - ((rgb - target) ** 2).mean().item()) < 1e-6
    g2, v2, _, _ = backend.render_backward(*args, grads={"rgb": 2.0 * (rgb - target) / (3 * n)})
    for a, b in zip(g1, g2):
        _assert_close(a, b, 1e-5, "fused loss")
    _assert_close(v1, v2, 1e-5, "fused loss volume")
    # n_total: a batch split into two calls accumulates the same volume gradient and loss
    loss2 = torch.zeros(1, device=DEV)
    half = n // 2
    va = torch.zeros_like(v1)
    parts = []
    for lo, hi in ((0, half), (half, n)):
        a2 = (d.pose_source, pts[lo:hi].to(DEV), ndc[lo:hi].to(DEV), z[lo:hi].to(DEV), rays[lo:hi, 3:6].to(DEV), vol, d.imgs_raw, fn, True)
        gp, _, _, _ = backend.render_backward(*a2, target_rgb=target[lo:hi], n_total=n, grad_volume=va, loss_out=loss2)
        parts.append([g.clone() for g in gp])
    assert abs(loss2.item() - loss.item()) < 1e-6
    _assert_close(va, v1, 1e-4, "split batch volume")
    for a, b, c in zip(parts[0], parts[1], g1):
        _assert_close(a + b, c, 1e-4, "split batch mlp")


def test_backward_rejects_long_rays_and_wrong_image(scene):
    sc, vol_ref = scene
    rays, pts, ndc, z = _samples(sc, 8, 160, seed=1)
    d = sc.to(DEV)
    fn = backend.MVSNeRF().to(DEV)
    backend.load_weights_npz(fn, None, WPATH)
    with pytest.raises(RuntimeError):
        backend.render_backward(d.pose_source, pts.to(DEV), ndc.to(DEV), z.to(DEV), rays[:, 3:6].to(DEV), vol_ref.to(DEV),
                                d.imgs_raw, fn, False, grads={"rgb": torch.ones(8, 3, device=DEV)})
    # N_samples > 128 under autograd falls back to the PyTorch-recompute backward and still trains
    volume = backend.RefVolume(vol_ref.clone().to(DEV))
    rgb = backend.rendering(Args(), d.pose_source, pts.to(DEV), ndc.to(DEV), z.to(DEV), None, rays[:, 3:6].to(DEV),
                            volume_feature=volume, imgs=d.imgs_raw, network_fn=fn)[0]
    rgb.sum().backward()
    assert volume.feat_volume.grad is not None and fn.nerf.rgb_linear.weight.grad is not None


@pytest.mark.parametrize("planar", [True, False])
def test_fused_adam_kernels_vs_torch_adam(planar):
    """mvsn_adam_step / mvsn_adam_step_volume against torch.optim.Adam on identical gradients, 3 steps."""
    L = lib.load()
    g = torch.Generator(device=DEV).manual_seed(0)
    shapes = [(128, 63), (128,), (3, 64), (1,)]
    params = [torch.randn(s, device=DEV, generator=g) for s in shapes]
    ref = [p.clone().requires_grad_(True) for p in params]
    D, Hp, Wp = 8, 6, 10
    nvox = D * Hp * Wp
    vol = torch.randn(1, 8, D, Hp, Wp, device=DEV, generator=g)
    if not planar:
        vol = vol[0].permute(1, 2, 3, 0).contiguous().permute(3, 0, 1, 2).unsqueeze(0)
    vol_ref = vol.clone().requires_grad_(True)
    opt = torch.optim.Adam(ref + [vol_ref], lr=3e-3, betas=(0.9, 0.999), eps=1e-8)
    m = [torch.zeros_like(p) for p in params]; v = [torch.zeros_like(p) for p in params]
    vm, vv = torch.zeros_like(vol), torch.zeros_like(vol)
    import ctypes as C
    numel = (C.c_int * len(params))(*[p.numel() for p in params])
    for step in range(1, 4):
        grads = [torch.randn(p.shape, device=DEV, generator=g) * (10.0 ** -step) for p in params]
        gvol_cl = torch.randn(D, Hp, Wp, 8, device=DEV, generator=g)
        gvol_cl[0] = 0.0                                        # untouched voxels still decay their moments
        for r, gg in zip(ref, grads):
            r.grad = gg.clone()
        vol_ref.grad = gvol_cl.permute(3, 0, 1, 2).unsqueeze(0).clone()
        opt.step()
        lib.check(L.mvsn_adam_step(lib.ptr_array(params), lib.ptr_array(grads), lib.ptr_array(m), lib.ptr_array(v), numel,
                                   len(params), 3e-3, 0.9, 0.999, 1e-8, step, lib.stream_ptr()), "mvsn_adam_step")
        lib.check(L.mvsn_adam_step_volume(lib.ptr(vol), lib.ptr(gvol_cl), lib.ptr(vm), lib.ptr(vv), nvox, int(planar),
                                          3e-3, 0.9, 0.999, 1e-8, step, lib.stream_ptr()), "mvsn_adam_step_volume")
        assert float(gvol_cl.abs().max()) == 0.0                 # gradient buffer handed back zeroed
        for p, r in zip(params, ref):
            assert (p - r.detach()).abs().max().item() <= 2e-6 * max(1.0, r.abs().max().item())
        assert (vol - vol_ref.detach()).abs().max().item() <= 2e-6 * vol_ref.abs().max().item()


def test_finetuner_trains_and_tracks_torch_adam(scene):
    """FineTuner.step (no autograd) vs `rendering` under autograd + torch.optim.Adam on the same batches: the loss
    sequences agree, the loss goes down, and caches notice the in-place updates (version counters)."""
    sc, vol_ref = scene
    d = sc.to(DEV)
    n, S = 256, 128
    fn_a, fn_b = backend.MVSNeRF().to(DEV), backend.MVSNeRF().to(DEV)
    backend.load_weights_npz(fn_a, None, WPATH); backend.load_weights_npz(fn_b, None, WPATH)
    vol_a = backend.RefVolume(vol_ref.clone().to(DEV))
    vol_b = backend.RefVolume(vol_ref.clone().to(DEV))
    tuner = backend.FineTuner(fn_a, vol_a, d.imgs_raw, d.pose_source, lr=5e-4, white_bkgd=False)
    opt = torch.optim.Adam(list(fn_b.parameters()) + list(vol_b.parameters()), lr=5e-4, betas=(0.9, 0.999))
    la, lb = [], []
    for it in range(8):
        rays, pts, ndc, z = _samples(sc, n, S, seed=100 + it % 2, perturb=1.0)
        target = torch.full((n, 3), 0.3, device=DEV)
        pts, ndc, z, rd = pts.to(DEV), ndc.to(DEV), z.to(DEV), rays[:, 3:6].to(DEV)
        v0 = fn_a.nerf.rgb_linear.weight._version
        loss, (rgb, _) = tuner.step(pts, ndc, z, rd, target, want_forward=True)
        assert fn_a.nerf.rgb_linear.weight._version > v0
        la.append(loss.item())
        out = backend.rendering(Args(), d.pose_source, pts, ndc, z, None, rd, volume_feature=vol_b, imgs=d.imgs_raw,
                                network_fn=fn_b, mlp_mode=lib.MLP_FP32)[0]
        l2 = ((out - target) ** 2).mean()
        opt.zero_grad(); l2.backward(); opt.step()
        lb.append(l2.item())
    assert la[-1] < 0.8 * la[0], la
    for a, b in zip(la, lb):
        assert abs(a - b) <= 2e-3 * max(a, b) + 1e-6, (la, lb)      # Adam amplifies rounding noise on near-zero gradients
    # the render entry points see the updated parameters
    with torch.no_grad():
        r1 = backend.render_rays(synthetic.scene_rays(sc)[:512].to(DEV), vol_a, d.imgs_raw, d.pose_source, fn_a, sc.near_far,
                                 float(sc.pad), N_samples=32)[0]
        r0 = backend.render_rays(synthetic.scene_rays(sc)[:512].to(DEV), vol_ref.to(DEV), d.imgs_raw, d.pose_source,
                                 backend.MVSNeRF().to(DEV), sc.near_far, float(sc.pad), N_samples=32)[0]
    assert not torch.equal(r0, r1)
