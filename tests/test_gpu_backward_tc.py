"""GPU: the fine-tuning backward with grad_mode MLP_TC_HALF (csrc/render_bwd.cu, render_bwd_tc_kernel: dgrad / wgrad
GEMMs on wgmma with fp16 operands and per-tile power-of-two scales, fp32 accumulation).

  * the forward it reports (rgb, depth, the fused loss) is bit-identical to the fp32 backward's: same fp32 tile;
  * its gradients are held against the emulation of its arithmetic (tests/grad_emulation.py, 2e-4 of max|g|) and
    against fp32 autograd of the oracle (3e-3 of max|g|), over ray layouts, white_bkgd, and ranges well beyond fp16:
    a tiny loss scale (dpre ~ 1e-10), cotangents x1e4, the encoding volume x3 (activations ~1e5), trunk weights x1.5;
  * it reaches users through render_backward, rendering under autograd and FineTuner.
"""
import os

import pytest
import torch

from conftest import GOLDEN
from grad_emulation import mlp_grad_emulated
from oracle import mvsnerf_oracle as orc
from mvsnerf_b200 import backend, lib, synthetic

pytestmark = pytest.mark.gpu
DEV = "cuda"
WPATH = os.path.join(GOLDEN, "mvsnerf_v0_weights.npz")
TC = lib.MLP_TC_HALF
GATE_EMU, GATE_FP32 = 2e-4, 3e-3


class Args:
    use_color_volume = False


@pytest.fixture(scope="module")
def scene(weights):
    sc = synthetic.make_scene(96, 128, pad=4, seed=9)
    vol = orc.encode_volume(sc.imgs_norm, sc.proj_mats, sc.near_far, sc.pad, weights)
    return sc, vol


def _samples(sc, n, S, seed, perturb=1.0):
    rays = synthetic.scene_rays(sc)
    rays = rays[torch.randperm(rays.shape[0], generator=torch.Generator().manual_seed(seed))[:n]].contiguous()
    torch.manual_seed(seed)
    pts, _, _, z = backend.ray_marcher(rays, N_samples=S, perturb=perturb)
    ndc = backend.get_ndc_coordinate(sc.pose_source["w2cs"][0], sc.pose_source["intrinsics"][0], pts,
                                     torch.tensor([sc.W - 1.0, sc.H - 1.0]), near=sc.near_far[0], far=sc.near_far[1], pad=sc.pad)
    return rays, pts.contiguous(), ndc.contiguous(), z.contiguous()


def _cotangents(n, S, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    c = {"rgb": torch.randn(n, 3, generator=g), "depth": 0.1 * torch.randn(n, generator=g),
         "weights": 0.05 * torch.randn(n, S, generator=g), "alpha": 0.05 * torch.randn(n, S, generator=g),
         "input_feat": 0.01 * torch.randn(n, S, 20, generator=g)}
    return {k: v * scale for k, v in c.items()}


def _oracle_grads(sc, vol, weights, pts, ndc, z, rd, cot=None, target=None, n_total=None, white=False, mlp_fn=None):
    """(MLP gradients by name, volume gradient [1,8,D,H,W]) of the oracle on the CPU."""
    wt = {k: v.clone().requires_grad_(k.startswith("mlp/")) for k, v in weights.items()}
    vt = vol.clone().requires_grad_(True)
    rgb, feat, w, depth, alpha = orc.render_samples(pts, ndc, z, rd, vt, sc.imgs_raw, sc.pose_source, wt,
                                                    white_bkgd=white, mlp_fn=mlp_fn)
    if target is not None:
        loss = ((rgb - target) ** 2).sum() / (3.0 * n_total)
    else:
        loss = (rgb * cot["rgb"]).sum() + (depth * cot["depth"]).sum() + (w * cot["weights"]).sum() + \
            (alpha * cot["alpha"]).sum() + (feat * cot["input_feat"]).sum()
    loss.backward()
    return {k[len("mlp/"):]: v.grad for k, v in wt.items() if v.grad is not None}, vt.grad


def _net(weights=None):
    fn = backend.MVSNeRF().to(DEV)
    backend.load_weights_npz(fn, None, WPATH)
    if weights is not None:                                     # modified weights (range tests)
        with torch.no_grad():
            for name, p in backend._ordered_named_params(fn):
                p.copy_(weights["mlp/" + name])
    return fn


def _rel(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def _check(g_mlp, g_vol, fn, ref, what):
    """Worst relative error of the kernel's gradients against a (by-name MLP, volume) reference."""
    ref_p, ref_v = ref
    worst = 0.0
    for (name, _), g in zip(backend._ordered_named_params(fn), g_mlp):
        assert torch.isfinite(g).all(), (what, name)
        worst = max(worst, _rel(g.cpu(), ref_p[name]))
    assert torch.isfinite(g_vol).all(), what
    e_v = _rel(g_vol.permute(3, 0, 1, 2).unsqueeze(0).cpu(), ref_v)
    return worst, e_v


def _run(sc, vol, fn, pts, ndc, z, rd, white, grad_mode, **kw):
    d = sc.to(DEV)
    return backend.render_backward(d.pose_source, pts.to(DEV), ndc.to(DEV), z.to(DEV), rd.to(DEV), vol.to(DEV), d.imgs_raw, fn,
                                   white, want_forward=True, grad_mode=grad_mode, **kw)


CASES = [(128, 37, False), (32, 130, True), (48, 21, False), (128, 300, True)]


@pytest.mark.parametrize("S,n,white", CASES)
def test_tc_backward_same_forward_and_gradients(scene, weights, S, n, white):
    """Random cotangents on all five outputs; S = 128 (one ray per tile), 32 (four), 48 (two + 32 idle rows); ragged
    ray counts; white_bkgd on and off."""
    sc, vol = scene
    rays, pts, ndc, z = _samples(sc, n, S, seed=S + n)
    rd = rays[:, 3:6]
    cot = _cotangents(n, S, seed=1)
    fn = _net()
    grads = {k: v.to(DEV) for k, v in cot.items()}
    g32, v32, rgb32, dep32 = _run(sc, vol, fn, pts, ndc, z, rd, white, lib.MLP_FP32, grads=grads)
    gtc, vtc, rgbtc, deptc = _run(sc, vol, fn, pts, ndc, z, rd, white, TC, grads=grads)
    assert torch.equal(rgb32, rgbtc) and torch.equal(dep32, deptc)
    e_emu = _check(gtc, vtc, fn, _oracle_grads(sc, vol, weights, pts, ndc, z, rd, cot, white=white, mlp_fn=mlp_grad_emulated), "emu")
    e_f32 = _check(gtc, vtc, fn, _oracle_grads(sc, vol, weights, pts, ndc, z, rd, cot, white=white), "fp32")
    print(f"\n[tc backward S={S} n={n} white={white}] vs emulator mlp {e_emu[0]:.3e} vol {e_emu[1]:.3e} ; "
          f"vs fp32 mlp {e_f32[0]:.3e} vol {e_f32[1]:.3e}")
    assert max(e_emu) < GATE_EMU, e_emu
    assert max(e_f32) < GATE_FP32, e_f32


@pytest.mark.parametrize("white", [False, True])
def test_tc_backward_fused_loss_is_the_fp32_loss(scene, white):
    """rgb and depth are bit-identical.  Each ray's loss term is too, but the terms are summed with float atomics
    across CTAs (in either mode), so the total agrees within their reordering."""
    sc, vol = scene
    n, S = 200, 64
    rays, pts, ndc, z = _samples(sc, n, S, seed=7)
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(3)).to(DEV)
    fn = _net()
    out = {}
    for mode in (lib.MLP_FP32, TC):
        loss = torch.zeros(1, device=DEV)
        _, _, rgb, depth = _run(sc, vol, fn, pts, ndc, z, rays[:, 3:6], white, mode, target_rgb=target, loss_out=loss)
        out[mode] = (rgb, depth, loss)
    assert torch.equal(out[lib.MLP_FP32][0], out[TC][0]) and torch.equal(out[lib.MLP_FP32][1], out[TC][1])
    assert _rel(out[TC][2], out[lib.MLP_FP32][2]) < 1e-6
    assert abs(out[TC][2].item() - ((out[TC][0] - target) ** 2).mean().item()) < 1e-6


@pytest.mark.parametrize("tag,white", [("s32", False), ("s128w", True)])
def test_tc_backward_vs_reference_gradient_fixture(golden_grad, golden_tiny, tag, white):
    """Gradients the unmodified reference's autograd produced (tests/golden/make_golden_grad.py), at the fp16 gate."""
    g = {k[len(tag) + 1:]: v for k, v in golden_grad.items() if k.startswith(tag + "/")}
    t = golden_tiny
    pose = {"w2cs": t["w2cs"].to(DEV), "c2ws": t["c2ws"].to(DEV), "intrinsics": t["intrinsics"].to(DEV)}
    fn = _net()
    loss = torch.zeros(1, device=DEV)
    g_mlp, g_vol, rgb, _ = backend.render_backward(pose, g["xyz"].to(DEV), g["ndc"].to(DEV), g["z"].to(DEV),
                                                   g["rays"][:, 3:6].to(DEV), t["volume"].to(DEV), t["imgs_raw"].to(DEV), fn,
                                                   white, target_rgb=g["target"].to(DEV), want_forward=True, loss_out=loss,
                                                   grad_mode=TC)
    assert (rgb.cpu() - g["rgb"]).abs().max() < 1e-5
    assert abs(loss.item() - float(g["loss"])) < 1e-5 * max(1.0, float(g["loss"]))
    worst = 0.0
    for (name, _), gk in zip(backend._ordered_named_params(fn), g_mlp):
        worst = max(worst, _rel(gk.cpu(), g["grad_mlp/" + name]))
    ref_v = torch.zeros(t["volume"].numel())
    ref_v[g["grad_volume_idx"]] = g["grad_volume_val"]
    e_v = _rel(g_vol.permute(3, 0, 1, 2).reshape(-1).cpu(), ref_v)
    print(f"\n[tc backward fixture {tag}] mlp {worst:.3e} vol {e_v:.3e}")
    assert worst < GATE_FP32 and e_v < GATE_FP32


@pytest.mark.parametrize("case", ["tiny_loss_scale", "cotangent_x1e4", "volume_x3", "trunk_x1.5"])
def test_tc_backward_range(scene, weights, case):
    """Operands far outside fp16's range stay finite and within the gates: the per-tile scales absorb them.
    tiny_loss_scale: the fused img2mse loss normalised by n_total = 1e7, so dpre ~ 1e-10 -- unscaled fp16 would flush
    almost all of it to zero."""
    sc, vol = scene
    n, S = 64, 128
    rays, pts, ndc, z = _samples(sc, n, S, seed=21)
    rd = rays[:, 3:6]
    w = dict(weights)
    if case == "volume_x3":
        vol = vol * 3.0
    if case == "trunk_x1.5":
        w = {k: (v * 1.5 if "pts_linears" in k and k.endswith("weight") else v) for k, v in weights.items()}
    fn = _net(w)
    if case == "tiny_loss_scale":
        target = torch.rand(n, 3, generator=torch.Generator().manual_seed(4))
        kw = dict(target_rgb=target.to(DEV), n_total=10_000_000)
        okw = dict(target=target, n_total=10_000_000)
    else:
        cot = _cotangents(n, S, seed=2, scale=1e4 if case == "cotangent_x1e4" else 1.0)
        kw = dict(grads={k: v.to(DEV) for k, v in cot.items()})
        okw = dict(cot=cot)
    g_mlp, g_vol, _, _ = _run(sc, vol, fn, pts, ndc, z, rd, False, TC, **kw)
    e_emu = _check(g_mlp, g_vol, fn, _oracle_grads(sc, vol, w, pts, ndc, z, rd, mlp_fn=mlp_grad_emulated, **okw), "emu")
    e_f32 = _check(g_mlp, g_vol, fn, _oracle_grads(sc, vol, w, pts, ndc, z, rd, **okw), "fp32")
    print(f"\n[tc backward range {case}] vs emulator mlp {e_emu[0]:.3e} vol {e_emu[1]:.3e} ; "
          f"vs fp32 mlp {e_f32[0]:.3e} vol {e_f32[1]:.3e}")
    assert max(e_emu) < GATE_EMU, e_emu
    assert max(e_f32) < GATE_FP32, e_f32


def test_tc_backward_is_deterministic(scene):
    """MLP gradients go through per-CTA private accumulators (no atomics): bit-identical across launches.  The volume
    gradient is scattered with float atomics and agrees within their reordering."""
    sc, vol = scene
    rays, pts, ndc, z = _samples(sc, 300, 128, seed=8)
    fn = _net()
    cot = {k: v.to(DEV) for k, v in _cotangents(300, 128, seed=3).items()}
    a = _run(sc, vol, fn, pts, ndc, z, rays[:, 3:6], True, TC, grads=cot)
    b = _run(sc, vol, fn, pts, ndc, z, rays[:, 3:6], True, TC, grads=cot)
    for x, y in zip(a[0], b[0]):
        assert torch.equal(x, y)
    assert _rel(a[1], b[1]) < 1e-6


def test_tc_backward_with_frozen_volume(scene):
    """want_volume_grad=False skips the pts_bias dgrad and the scatter; the MLP gradients do not depend on them, so they
    are bit-identical to those of the launch that also produces the volume gradient."""
    sc, vol = scene
    rays, pts, ndc, z = _samples(sc, 130, 32, seed=9)
    fn = _net()
    cot = {k: v.to(DEV) for k, v in _cotangents(130, 32, seed=4).items()}
    with_vol = _run(sc, vol, fn, pts, ndc, z, rays[:, 3:6], False, TC, grads=cot)
    frozen = _run(sc, vol, fn, pts, ndc, z, rays[:, 3:6], False, TC, grads=cot, want_volume_grad=False)
    assert frozen[1] is None
    for a, b in zip(with_vol[0], frozen[0]):
        assert torch.equal(a, b)
    assert torch.equal(with_vol[2], frozen[2]) and torch.equal(with_vol[3], frozen[3])


def test_tc_rendering_under_autograd_uses_the_tc_backward(scene):
    sc, vol = scene
    n, S = 200, 64
    rays, pts, ndc, z = _samples(sc, n, S, seed=5)
    d = sc.to(DEV)
    pts, ndc, z, rd = pts.to(DEV), ndc.to(DEV), z.to(DEV), rays[:, 3:6].to(DEV)
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    fn = _net()
    volume = backend.RefVolume(vol.clone().to(DEV))
    rgb = backend.rendering(Args(), d.pose_source, pts, ndc, z, None, rd, volume_feature=volume, imgs=d.imgs_raw,
                            network_fn=fn, mlp_mode=lib.MLP_FP32, grad_mode=TC)[0]
    ((rgb - target) ** 2).mean().backward()
    g_mlp, g_vol, _, _ = backend.render_backward(d.pose_source, pts, ndc, z, rd, vol.to(DEV), d.imgs_raw, _net(), False,
                                                 grads={"rgb": 2.0 * (rgb.detach() - target) / (3 * n)}, grad_mode=TC)
    for p, g in zip(fn.ordered_params(), g_mlp):
        assert torch.equal(p.grad, g)
    assert _rel(volume.feat_volume.grad, g_vol.permute(3, 0, 1, 2).unsqueeze(0)) < 1e-6
    with pytest.raises(RuntimeError):
        backend.rendering(Args(), d.pose_source, pts, ndc, z, None, rd, volume_feature=volume, imgs=d.imgs_raw,
                          network_fn=fn, grad_mode=lib.MLP_TC_SPLIT)


def test_tc_finetuner_tracks_the_fp32_finetuner(scene):
    """Same start, same batches: the first loss is the same (same forward; its per-ray terms are summed with float
    atomics, so within their reordering), then the two runs track each other (H100 80GB HBM3: 4e-6 relative over the 8
    steps) and both train."""
    sc, vol = scene
    d = sc.to(DEV)
    n, S = 256, 128
    runs = {}
    for mode in (lib.MLP_FP32, TC):
        fn = _net()
        volume = backend.RefVolume(vol.clone().to(DEV))
        tuner = backend.FineTuner(fn, volume, d.imgs_raw, d.pose_source, lr=5e-4, grad_mode=mode)
        losses = []
        for it in range(8):
            rays, pts, ndc, z = _samples(sc, n, S, seed=100 + it % 2)
            target = torch.full((n, 3), 0.3, device=DEV)
            losses.append(tuner.step(pts.to(DEV), ndc.to(DEV), z.to(DEV), rays[:, 3:6].to(DEV), target)[0].item())
        runs[mode] = losses
    a, b = runs[lib.MLP_FP32], runs[TC]
    print(f"\n[tc finetuner] fp32 {a}\n[tc finetuner] tc   {b}")
    assert abs(a[0] - b[0]) <= 1e-6 * a[0], (a, b)
    assert b[-1] < 0.8 * b[0], b
    for x, y in zip(a, b):
        assert abs(x - y) <= 1e-4 * max(x, y), (a, b)
    with pytest.raises(RuntimeError):
        backend.FineTuner(_net(), backend.RefVolume(vol.clone().to(DEV)), d.imgs_raw, d.pose_source, grad_mode=lib.MLP_TC_PAIR)


def test_tc_backward_rejects_long_rays_and_wrong_image(scene):
    sc, vol = scene
    rays, pts, ndc, z = _samples(sc, 8, 160, seed=1)
    d = sc.to(DEV)
    fn = _net()
    with pytest.raises(RuntimeError):
        backend.render_backward(d.pose_source, pts.to(DEV), ndc.to(DEV), z.to(DEV), rays[:, 3:6].to(DEV), vol.to(DEV),
                                d.imgs_raw, fn, False, grads={"rgb": torch.ones(8, 3, device=DEV)}, grad_mode=TC)
    # the C entry with a non-FP32 weight image
    L = lib.load()
    rays, pts, ndc, z = _samples(sc, 8, 32, seed=1)
    sc_c, keep = backend._make_scene(d.pose_source, vol.to(DEV), d.imgs_raw, fn, False, lib.MLP_TC_HALF)
    params = [p.detach() for p in fn.ordered_params()]
    grads = [torch.empty_like(p) for p in params]
    g = lib.RenderGrads()
    g_rgb = torch.ones(8, 3, device=DEV)
    g.rgb = g_rgb.data_ptr()
    need = L.mvsn_render_backward_tc_workspace_bytes(8, 32)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    dev_t = [t.to(DEV).contiguous() for t in (pts, ndc, z, rays[:, 3:6])]
    import ctypes as C
    rc = L.mvsn_render_backward_tc(C.byref(sc_c), lib.ptr_array(params), *[lib.ptr(t) for t in dev_t], 8, 32, C.byref(g),
                                   lib.ptr_array(grads), None, lib.ptr(ws), need, lib.stream_ptr())
    assert rc != 0 and b"MVSN_MLP_FP32" in L.mvsn_last_error()
    del keep
