"""GPU: the fine-tuning backward straight from rays (mvsn_render_backward_rays: backend.render_backward_rays and
FineTuner.step_rays), whose kernel also does ray_marcher (stratified by a given jitter) and get_ndc_coordinate.

  * no jitter: the forward it reports is the fp32 render kernel's (render_rays, MLP_FP32);
  * jitter: against the samples-entry backward and the oracle's autograd on the same jitter marched on the host with
    ray_marcher's ops and get_ndc_coordinate (which uses torch.matmul, so its NDC differs in the last bits);
  * the deterministic variant, a frozen volume, the `grads` path, rejected arguments;
  * training: step_rays tracks step(*ray_marcher(...)) on the same random stream, and repeats bit for bit under
    torch.use_deterministic_algorithms(True).
"""
import ctypes as C
import os

import pytest
import torch

from conftest import GOLDEN
from oracle import mvsnerf_oracle as orc
from mvsnerf_b200 import backend, lib, synthetic

pytestmark = pytest.mark.gpu
DEV = "cuda"
WPATH = os.path.join(GOLDEN, "mvsnerf_v0_weights.npz")
MODES = [lib.MLP_FP32, lib.MLP_TC_HALF]
GATE = {lib.MLP_FP32: 2e-4, lib.MLP_TC_HALF: 3e-3}      # vs the oracle's fp32 autograd, as the samples-entry tests


@pytest.fixture(scope="module")
def scene(weights):
    sc = synthetic.make_scene(96, 128, pad=4, seed=9)
    vol = orc.encode_volume(sc.imgs_norm, sc.proj_mats, sc.near_far, sc.pad, weights)
    return sc, vol


@pytest.fixture
def deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn)


def _net():
    fn = backend.MVSNeRF().to(DEV)
    backend.load_weights_npz(fn, None, WPATH)
    return fn


def _rays(sc, n, seed):
    rays = synthetic.scene_rays(sc)
    return rays[torch.randperm(rays.shape[0], generator=torch.Generator().manual_seed(seed))[:n]].contiguous().to(DEV)


def _jitter(n, S, seed):
    return torch.rand(n, S, generator=torch.Generator().manual_seed(seed)).to(DEV)


def _host_march(sc, rays, S, j, lindisp=False):
    """ray_marcher (data/ray_utils.py:152-197) with the uniform draw replaced by `j`, then get_ndc_coordinate, on the
    device: the samples the kernel marches itself."""
    near, far = rays[:, 6:7], rays[:, 7:8]
    t = torch.linspace(0, 1, S, device=DEV)
    z = near * (1 - t) + far * t if not lindisp else 1 / (1 / near * (1 - t) + 1 / far * t)
    z = z.expand(rays.shape[0], S)
    if j is not None:
        mid = 0.5 * (z[:, :-1] + z[:, 1:])
        upper = torch.cat([mid, z[:, -1:]], -1)
        lower = torch.cat([z[:, :1], mid], -1)
        z = lower + (upper - lower) * j
    pts = rays[:, None, 0:3] + rays[:, None, 3:6] * z[..., None]
    d = sc.to(DEV)
    ndc = backend.get_ndc_coordinate(d.pose_source["w2cs"][0], d.pose_source["intrinsics"][0], pts,
                                     torch.tensor([sc.W - 1.0, sc.H - 1.0], device=DEV), near=sc.near_far[0],
                                     far=sc.near_far[1], pad=sc.pad, lindisp=lindisp)
    return pts.contiguous(), ndc.contiguous(), z.contiguous()


def _kernel_order_ndc(sc, pts):
    """get_ndc_coordinate (no lindisp) in the kernel's operation order (ndc_of_point / project_view): fmaf chains,
    each fma formed exactly in float64 (the product of two floats is exact there) and rounded once to float32, then
    IEEE float32 divisions.  get_ndc_coordinate's torch.matmul rounds differently, and the positional encoding
    multiplies an NDC difference by up to 2^9 (sin(2^9 x)), so its last-bit differences reach the gradients at ~1e-4
    of max|g|; against this NDC they do not."""
    f32 = lambda t: t.to(torch.float32)                           # noqa: E731
    fma = lambda a, b, c: f32(a.double() * b.double() + c.double())  # noqa: E731
    p = pts.reshape(-1, 3).cpu()
    w = sc.pose_source["w2cs"][0].float().reshape(-1)
    K = sc.pose_source["intrinsics"][0].float().reshape(-1)
    px, py, pz = p[:, 0], p[:, 1], p[:, 2]
    cam = [fma(pz, w[4 * r + 2], fma(py, w[4 * r + 1], px * w[4 * r])) + w[4 * r + 3] for r in range(3)]
    q = [fma(cam[2], K[3 * r + 2], fma(cam[1], K[3 * r + 1], cam[0] * K[3 * r])) for r in range(3)]
    u = (q[0] / q[2]) / torch.tensor(sc.W - 1.0)
    v = (q[1] / q[2]) / torch.tensor(sc.H - 1.0)
    near, far = (torch.tensor(float(x), dtype=torch.float32) for x in sc.near_far)   # as mvsn_ray_params carries them
    nz = (q[2] - near) / f32(far.double() - near.double())
    if sc.pad > 0:
        hf, wf, pad = torch.tensor(sc.H / 4.0), torch.tensor(sc.W / 4.0), torch.tensor(float(sc.pad))
        dh, dw = hf + pad * 2, wf + pad * 2
        v = (v * hf) / dh + pad / dh
        u = (u * wf) / dw + pad / dw
    return torch.stack([u, v, nz], -1).reshape(pts.shape).contiguous().to(DEV)


def _cotangents(n, S, seed):
    g = torch.Generator().manual_seed(seed)
    c = {"rgb": torch.randn(n, 3, generator=g), "depth": 0.1 * torch.randn(n, generator=g),
         "weights": 0.05 * torch.randn(n, S, generator=g), "alpha": 0.05 * torch.randn(n, S, generator=g),
         "input_feat": 0.01 * torch.randn(n, S, 20, generator=g)}
    return {k: v.to(DEV) for k, v in c.items()}


def _rel(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def _bwd_rays(sc, vol, fn, rays, S, white, grad_mode, j=None, lindisp=False, **kw):
    d = sc.to(DEV)
    return backend.render_backward_rays(rays, vol.to(DEV), d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad),
                                        N_samples=S, lindisp=lindisp, jitter=j, white_bkgd=white, want_forward=True,
                                        grad_mode=grad_mode, **kw)


def _bwd_samples(sc, vol, fn, rays, samples, white, grad_mode, **kw):
    d = sc.to(DEV)
    pts, ndc, z = samples
    return backend.render_backward(d.pose_source, pts, ndc, z, rays[:, 3:6], vol.to(DEV), d.imgs_raw, fn, white,
                                   want_forward=True, grad_mode=grad_mode, **kw)


@pytest.mark.parametrize("pad,lindisp", [(0, False), (0, True), (24, False)])
@pytest.mark.parametrize("S,n,white", [(32, 130, True), (48, 21, False), (128, 37, False), (128, 300, True)])
def test_no_jitter_forward_is_the_fp32_render(S, n, white, pad, lindisp):
    """jitter=None marches render_rays' depths, and the recompute is the fp32 render kernel's forward tile: rgb is
    bit-identical to render_rays(mlp_mode=MLP_FP32).  Depth is composed with different rounding in the two kernels
    (fmaf vs multiply-then-add), so it agrees to 1e-6 only."""
    sc = synthetic.make_scene(64, 96, pad=pad, seed=2)
    vol = 0.5 * torch.randn(1, 8, 128, 16 + 2 * pad, 24 + 2 * pad, generator=torch.Generator().manual_seed(pad))
    d = sc.to(DEV)
    fn = _net()
    rays = _rays(sc, n, seed=S + n)
    with torch.no_grad():
        rgb_f, depth_f = backend.render_rays(rays, vol.to(DEV), d.imgs_raw, d.pose_source, fn, sc.near_far, float(pad),
                                             N_samples=S, white_bkgd=white, lindisp=lindisp, mlp_mode=lib.MLP_FP32)
    for mode in MODES:
        _, _, rgb_b, depth_b = _bwd_rays(sc, vol, fn, rays, S, white, mode, lindisp=lindisp,
                                         grads={"rgb": torch.ones(n, 3, device=DEV)})
        assert torch.equal(rgb_b, rgb_f), (mode, (rgb_b - rgb_f).abs().max().item())
        assert (depth_b - depth_f).abs().max().item() <= 1e-6
    # FineTuner.step_rays reports the same forward (before its update)
    tuner = backend.FineTuner(fn, backend.RefVolume(vol.clone().to(DEV)), d.imgs_raw, d.pose_source, white_bkgd=white)
    _, (rgb_s, _) = tuner.step_rays(rays, torch.zeros(n, 3, device=DEV), sc.near_far, float(pad), N_samples=S,
                                    lindisp=lindisp, perturb=0.0, want_forward=True)
    assert torch.equal(rgb_s, rgb_f)


@pytest.mark.parametrize("grad_mode", MODES)
@pytest.mark.parametrize("S,n,white", [(32, 130, True), (48, 21, False), (128, 300, True)])
def test_jittered_backward_matches_host_marched_samples(scene, S, n, white, grad_mode):
    """The same jitter marched on the host with ray_marcher's ops (points and depths bit-identical to the kernel's).
    With the NDC in the kernel's operation order: loss to 1e-6 relative, MLP and volume gradients to 1e-6 of max|g| of
    the samples-entry backward.  With get_ndc_coordinate's NDC (torch.matmul, see _kernel_order_ndc): to 1e-3."""
    sc, vol = scene
    rays = _rays(sc, n, seed=S + n)
    j = _jitter(n, S, seed=S)
    samples = _host_march(sc, rays, S, j)
    exact = (samples[0], _kernel_order_ndc(sc, samples[0]), samples[2])
    fn = _net()
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(1)).to(DEV)
    loss_r = torch.zeros(1, device=DEV)
    g_r, v_r, rgb_r, depth_r = _bwd_rays(sc, vol, fn, rays, S, white, grad_mode, j, target_rgb=target, loss_out=loss_r)
    for name, smp, gate in (("kernel-order ndc", exact, 1e-6), ("get_ndc_coordinate", samples, 1e-3)):
        loss_s = torch.zeros(1, device=DEV)
        g_s, v_s, rgb_s, depth_s = _bwd_samples(sc, vol, fn, rays, smp, white, grad_mode, target_rgb=target, loss_out=loss_s)
        e_l = abs(loss_r.item() - loss_s.item()) / loss_s.item()
        worst = max(_rel(a, b) for a, b in zip(g_r, g_s))
        e_v = _rel(v_r, v_s)
        print(f"\n[rays vs samples, {name}, {grad_mode} S={S}] loss {e_l:.3e} rgb {(rgb_r - rgb_s).abs().max().item():.3e} "
              f"mlp {worst:.3e} vol {e_v:.3e}")
        assert e_l <= max(gate, 1e-6) and worst < gate and e_v < gate
        assert (rgb_r - rgb_s).abs().max().item() < 1e-5 and (depth_r - depth_s).abs().max().item() < 1e-4


@pytest.mark.parametrize("grad_mode", MODES)
@pytest.mark.parametrize("S,n,white", [(128, 37, False), (32, 130, True), (48, 21, False), (128, 300, True)])
def test_jittered_backward_vs_oracle_autograd(scene, weights, S, n, white, grad_mode):
    """The cases of test_backward_kernel_vs_oracle_autograd_all_outputs (same rays, same seed): its samples were
    marched by ray_marcher on the CPU after torch.manual_seed(S + n), so the same torch.rand draw is the jitter here.
    Random cotangents on every output; the oracle's fp32 autograd at the samples-entry gates."""
    sc, vol = scene
    rays = synthetic.scene_rays(sc)
    rays = rays[torch.randperm(rays.shape[0], generator=torch.Generator().manual_seed(S + n))[:n]].contiguous()
    torch.manual_seed(S + n)
    pts, _, _, z = backend.ray_marcher(rays, N_samples=S, perturb=1.0)
    torch.manual_seed(S + n)
    j = torch.rand(n, S).to(DEV)
    ndc = backend.get_ndc_coordinate(sc.pose_source["w2cs"][0], sc.pose_source["intrinsics"][0], pts,
                                     torch.tensor([sc.W - 1.0, sc.H - 1.0]), near=sc.near_far[0], far=sc.near_far[1], pad=sc.pad)
    fn = _net()
    g = torch.Generator().manual_seed(1)
    cot = {"rgb": torch.randn(n, 3, generator=g), "depth": 0.1 * torch.randn(n, generator=g),
           "weights": 0.05 * torch.randn(n, S, generator=g), "alpha": 0.05 * torch.randn(n, S, generator=g),
           "input_feat": 0.01 * torch.randn(n, S, 20, generator=g)}
    g_k, v_k, _, _ = _bwd_rays(sc, vol, fn, rays.to(DEV), S, white, grad_mode, j,
                               grads={k: v.to(DEV) for k, v in cot.items()})
    wt = {k: v.clone().requires_grad_(k.startswith("mlp/")) for k, v in weights.items()}
    vt = vol.clone().requires_grad_(True)
    rgb, feat, w, depth, alpha = orc.render_samples(pts, ndc, z, rays[:, 3:6], vt, sc.imgs_raw, sc.pose_source, wt,
                                                    white_bkgd=white)
    c = cot
    ((rgb * c["rgb"]).sum() + (depth * c["depth"]).sum() + (w * c["weights"]).sum() + (alpha * c["alpha"]).sum() +
     (feat * c["input_feat"]).sum()).backward()
    # per tensor, err <= gate * max|g| + 1e-8 as test_backward_kernel_vs_oracle_autograd_all_outputs checks it
    pairs = [(g.cpu(), wt["mlp/" + name].grad) for (name, _), g in zip(backend._ordered_named_params(fn), g_k)]
    pairs.append((v_k.permute(3, 0, 1, 2).unsqueeze(0).cpu(), vt.grad))
    excess = max((a - b).abs().max().item() - GATE[grad_mode] * b.abs().max().item() - 1e-8 for a, b in pairs)
    print(f"[rays vs oracle {grad_mode} S={S}] mlp {max(_rel(a, b) for a, b in pairs[:-1]):.3e} "
          f"vol {_rel(*pairs[-1]):.3e}")
    assert excess <= 0, excess


@pytest.mark.parametrize("grad_mode", MODES)
@pytest.mark.parametrize("tag,white", [("s32", False), ("s128w", True)])
def test_rays_backward_vs_reference_gradient_fixture(golden_grad, golden_tiny, tag, white, grad_mode):
    """The fused loss from the fixture's rays against the gradients the unmodified reference's autograd produced
    (tests/golden/make_golden_grad.py: ray_marcher without perturbation on make_scene(32, 32, pad=4, seed=1)), at the
    samples-entry gates: the in-kernel march reproduces the reference's samples."""
    g = {k[len(tag) + 1:]: v for k, v in golden_grad.items() if k.startswith(tag + "/")}
    t = golden_tiny
    sc = synthetic.make_scene(32, 32, pad=4, seed=1)
    rays = g["rays"].to(DEV).contiguous()
    S = g["z"].shape[1]
    pose = {"w2cs": t["w2cs"].to(DEV), "c2ws": t["c2ws"].to(DEV), "intrinsics": t["intrinsics"].to(DEV)}
    fn = _net()
    loss = torch.zeros(1, device=DEV)
    g_mlp, g_vol, rgb, _ = backend.render_backward_rays(rays, t["volume"].to(DEV), t["imgs_raw"].to(DEV), pose, fn,
                                                        sc.near_far, float(sc.pad), N_samples=S, white_bkgd=white,
                                                        target_rgb=g["target"].to(DEV), want_forward=True, loss_out=loss,
                                                        grad_mode=grad_mode)
    assert (rgb.cpu() - g["rgb"]).abs().max() < 1e-5
    assert abs(loss.item() - float(g["loss"])) < 1e-5 * max(1.0, float(g["loss"]))
    worst = max(_rel(gk.cpu(), g["grad_mlp/" + name]) for (name, _), gk in zip(backend._ordered_named_params(fn), g_mlp))
    ref_v = torch.zeros(t["volume"].numel())
    ref_v[g["grad_volume_idx"]] = g["grad_volume_val"]
    e_v = _rel(g_vol.permute(3, 0, 1, 2).reshape(-1).cpu(), ref_v)
    print(f"\n[rays vs fixture {grad_mode}] mlp {worst:.3e} vol {e_v:.3e}")
    assert worst < GATE[grad_mode] and e_v < GATE[grad_mode]


def _assert_same(a, b):
    for x, y in zip(a[0], b[0]):
        assert torch.equal(x, y)
    for x, y in zip(a[1:], b[1:]):
        assert (x is None and y is None) or torch.equal(x, y)


@pytest.mark.parametrize("grad_mode", MODES)
def test_deterministic_rays_backward_repeats_and_agrees_with_atomics(scene, grad_mode):
    sc, vol = scene
    n, S = 1023, 128
    rays = _rays(sc, n, seed=4)
    j = _jitter(n, S, seed=5)
    fn = _net()
    cot = _cotangents(n, S, seed=6)
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(7)).to(DEV)
    atomic = _bwd_rays(sc, vol, fn, rays, S, True, grad_mode, j, grads=cot)
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        a = _bwd_rays(sc, vol, fn, rays, S, True, grad_mode, j, grads=cot)
        b = _bwd_rays(sc, vol, fn, rays, S, True, grad_mode, j, grads=cot)
        la, lb = torch.zeros(1, device=DEV), torch.zeros(1, device=DEV)
        fa = _bwd_rays(sc, vol, fn, rays, S, True, grad_mode, j, target_rgb=target, loss_out=la)
        fb = _bwd_rays(sc, vol, fn, rays, S, True, grad_mode, j, target_rgb=target, loss_out=lb)
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)
    assert torch.isfinite(a[1]).all() and a[1].abs().max() > 0
    _assert_same(a, b)
    _assert_same(fa, fb)
    assert torch.equal(la, lb) and abs(la.item() - ((fa[2] - target) ** 2).mean().item()) < 1e-6
    for x, y in zip(atomic[0], a[0]):                             # MLP gradients: private accumulators in both
        assert torch.equal(x, y)
    assert torch.equal(atomic[2], a[2]) and torch.equal(atomic[3], a[3])
    e = _rel(a[1], atomic[1])
    print(f"\n[rays det {grad_mode}] vs atomic vol {e:.3e}")
    assert e < 1e-6


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("grad_mode", MODES)
def test_rays_backward_with_frozen_volume(scene, grad_mode, det):
    sc, vol = scene
    n, S = 130, 32
    rays = _rays(sc, n, seed=9)
    j = _jitter(n, S, seed=9)
    fn = _net()
    cot = _cotangents(n, S, seed=4)
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(det, warn_only=True)
    try:
        with_vol = _bwd_rays(sc, vol, fn, rays, S, False, grad_mode, j, grads=cot)
        frozen = _bwd_rays(sc, vol, fn, rays, S, False, grad_mode, j, grads=cot, want_volume_grad=False)
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)
    assert frozen[1] is None
    for a, b in zip(with_vol[0], frozen[0]):
        assert torch.equal(a, b)
    assert torch.equal(with_vol[2], frozen[2]) and torch.equal(with_vol[3], frozen[3])


@pytest.mark.parametrize("grad_mode", MODES)
def test_rays_backward_grads_dict_rgb_and_depth(scene, grad_mode):
    """d rgb + d depth (no fused loss): the depth differentiated is the jittered one."""
    sc, vol = scene
    n, S = 200, 64
    rays = _rays(sc, n, seed=12)
    j = _jitter(n, S, seed=12)
    fn = _net()
    g = torch.Generator().manual_seed(2)
    grads = {"rgb": torch.randn(n, 3, generator=g).to(DEV), "depth": 0.1 * torch.randn(n, generator=g).to(DEV)}
    pts, _, z = _host_march(sc, rays, S, j)
    g_r, v_r, _, _ = _bwd_rays(sc, vol, fn, rays, S, False, grad_mode, j, grads=grads)
    g_s, v_s, _, _ = _bwd_samples(sc, vol, fn, rays, (pts, _kernel_order_ndc(sc, pts), z), False, grad_mode, grads=grads)
    worst = max(_rel(a, b) for a, b in zip(g_r, g_s))
    e_v = _rel(v_r, v_s)
    assert worst < 1e-6 and e_v < 1e-6, (worst, e_v)


def test_rays_backward_rejects_long_rays_wrong_image_and_misaligned_rays(scene):
    sc, vol = scene
    d = sc.to(DEV)
    fn = _net()
    rays = _rays(sc, 8, seed=1)
    with pytest.raises(RuntimeError, match="128"):
        _bwd_rays(sc, vol, fn, rays, 160, False, lib.MLP_FP32, grads={"rgb": torch.ones(8, 3, device=DEV)})
    with pytest.raises(RuntimeError, match="128"):
        _bwd_rays(sc, vol, fn, rays, 160, False, lib.MLP_TC_HALF, grads={"rgb": torch.ones(8, 3, device=DEV)})
    with pytest.raises(RuntimeError, match="aligned"):
        buf = torch.empty(8 * 8 + 1, device=DEV)
        bad = buf[1:].view(8, 8)
        bad.copy_(rays)
        _bwd_rays(sc, vol, fn, bad, 32, False, lib.MLP_FP32, grads={"rgb": torch.ones(8, 3, device=DEV)})
    # the C entry with a non-FP32 weight image
    L = lib.load()
    sc_c, keep = backend._make_scene(d.pose_source, vol.to(DEV), d.imgs_raw, fn, False, lib.MLP_TC_HALF)
    params = [p.detach() for p in fn.ordered_params()]
    grads = [torch.empty_like(p) for p in params]
    g = lib.RenderGrads()
    g_rgb = torch.ones(8, 3, device=DEV)
    g.rgb = g_rgb.data_ptr()
    rp = lib.RayParams(float(sc.near_far[0]), float(sc.near_far[1]), float(sc.pad), 0)
    t_steps = torch.linspace(0, 1, 32, device=DEV)
    for mode in MODES:
        need = L.mvsn_render_backward_rays_workspace_bytes(8, 32, 0, 0, 0, mode, 0)
        ws = torch.empty(need, dtype=torch.uint8, device=DEV)
        rc = L.mvsn_render_backward_rays(C.byref(sc_c), lib.ptr_array(params), C.byref(rp), lib.ptr(rays), lib.ptr(t_steps),
                                         None, 8, 32, mode, 0, C.byref(g), lib.ptr_array(grads), None, lib.ptr(ws), need,
                                         lib.stream_ptr())
        assert rc == -6 and b"MVSN_MLP_FP32" in L.mvsn_last_error()
    del keep


def _train(sc, vol, grad_mode, steps, use_rays, n=256, S=128, seed=0):
    """`steps` FineTuner steps on batches of the reference camera's rays; the batch indices come from their own
    generator and the jitter from the default one, seeded once, so both forms of the step see the same draws.  The
    host form marches with ray_marcher (its own torch.rand draw) and converts with the kernel's NDC operation order, so
    the two runs differ only by the order of the float atomics (see _kernel_order_ndc)."""
    d = sc.to(DEV)
    fn = _net()
    volume = backend.RefVolume(vol.clone().to(DEV))
    tuner = backend.FineTuner(fn, volume, d.imgs_raw, d.pose_source, lr=5e-4, grad_mode=grad_mode)
    rays_all = synthetic.scene_rays(sc).to(DEV)
    tgt_all = d.imgs_raw[0, 0].permute(1, 2, 0).reshape(-1, 3).contiguous()
    gen = torch.Generator(device=DEV).manual_seed(seed)
    torch.manual_seed(seed)
    losses = []
    for _ in range(steps):
        idx = torch.randint(0, rays_all.shape[0], (n,), device=DEV, generator=gen)
        rays, tgt = rays_all[idx], tgt_all[idx]
        if use_rays:
            loss = tuner.step_rays(rays, tgt, sc.near_far, float(sc.pad), N_samples=S, perturb=1.0)[0]
        else:
            xyz, _, rd, z = backend.ray_marcher(rays, N_samples=S, perturb=1.0)
            loss = tuner.step(xyz, _kernel_order_ndc(sc, xyz), z, rd, tgt)[0]
        losses.append(loss.clone())
    return [p.detach().clone() for p in fn.ordered_params()], volume.feat_volume.detach().clone(), torch.cat(losses)


@pytest.mark.parametrize("grad_mode", MODES)
def test_step_rays_tracks_step_on_the_same_random_stream(scene, deterministic, grad_mode):
    """Same seed, 50 steps each: step_rays draws the jitter ray_marcher draws.  The volume gradient is summed in a fixed
    order here, so the runs differ only in how the samples were prepared (with float atomics, TC_HALF runs drift apart
    by ~1e-4 over 50 steps from the summation order alone); a different random stream would differ by percents."""
    sc, vol = scene
    _, _, la = _train(sc, vol, grad_mode, 50, use_rays=False)
    _, _, lb = _train(sc, vol, grad_mode, 50, use_rays=True)
    rel = ((la - lb).abs() / la.abs()).max().item()
    print(f"\n[step_rays vs step {grad_mode}] first {la[0].item():.6e} / {lb[0].item():.6e} last {la[-1].item():.6e} / "
          f"{lb[-1].item():.6e} ; max rel {rel:.3e}")
    assert rel < 1e-4
    assert lb[-10:].mean() < lb[:10].mean()


@pytest.mark.parametrize("grad_mode", MODES)
def test_step_rays_repeats_bit_for_bit_when_deterministic(scene, deterministic, grad_mode):
    sc, vol = scene
    pa, va, la = _train(sc, vol, grad_mode, 50, use_rays=True)
    pb, vb, lb = _train(sc, vol, grad_mode, 50, use_rays=True)
    for x, y in zip(pa, pb):
        assert torch.equal(x, y)
    assert torch.equal(va, vb) and torch.equal(la, lb)
