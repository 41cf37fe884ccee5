"""GPU: the deterministic fine-tuning backward (mvsn_render_backward_deterministic), which render_backward, FineTuner and
`rendering` under autograd take while torch.use_deterministic_algorithms(True) is in effect.

  * repeat: identical inputs give bit-identical volume gradient, MLP gradients, rgb, depth and loss, in both grad modes;
  * exactness: a pure trilinear scatter equals the fp64 sum of the same fp32 products within 1 ulp plus half a
    fixed-point quantum per contribution, and is bit-equal almost everywhere;
  * agreement with the float-atomic path and the oracle's autograd; permutation invariance in MLP_FP32; NaN;
  * training: FineTuner and rendering + torch.optim.Adam runs repeat bit for bit.
"""
import math
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
GATE = {lib.MLP_FP32: 2e-4, lib.MLP_TC_HALF: 3e-3}


class Args:
    use_color_volume = False


@pytest.fixture
def deterministic():
    """torch.use_deterministic_algorithms(True, warn_only=True) for the test, the previous setting restored after."""
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn)


@pytest.fixture(scope="module")
def scene(weights):
    sc = synthetic.make_scene(96, 128, pad=4, seed=9)
    vol = orc.encode_volume(sc.imgs_norm, sc.proj_mats, sc.near_far, sc.pad, weights)
    return sc, vol


def _samples(sc, n, S, seed, perturb=1.0):
    """n rays of the reference camera (so many rays cross the same voxels), marched with S samples."""
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


def _net():
    fn = backend.MVSNeRF().to(DEV)
    backend.load_weights_npz(fn, None, WPATH)
    return fn


def _rel(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def _run(sc, vol, fn, pts, ndc, z, rd, white, grad_mode, **kw):
    d = sc.to(DEV)
    return backend.render_backward(d.pose_source, pts.to(DEV), ndc.to(DEV), z.to(DEV), rd.to(DEV), vol.to(DEV), d.imgs_raw, fn,
                                   white, want_forward=True, grad_mode=grad_mode, **kw)


def _fused(sc, vol, fn, pts, ndc, z, rd, white, grad_mode, target):
    loss = torch.zeros(1, device=DEV)
    g_mlp, g_vol, rgb, depth = _run(sc, vol, fn, pts, ndc, z, rd, white, grad_mode, target_rgb=target, loss_out=loss)
    return g_mlp, g_vol, rgb, depth, loss


def _assert_same(a, b):
    g_a, v_a, *rest_a = a
    g_b, v_b, *rest_b = b
    for x, y in zip(g_a, g_b):
        assert torch.equal(x, y)
    assert torch.equal(v_a, v_b)
    for x, y in zip(rest_a, rest_b):
        assert torch.equal(x, y)


@pytest.mark.parametrize("grad_mode", MODES)
@pytest.mark.parametrize("S,white", [(32, False), (48, True), (128, False), (128, True)])
def test_deterministic_backward_repeats_bit_for_bit(scene, deterministic, S, white, grad_mode):
    """2 047 rays of one camera (ragged for S = 32 and 48), cotangents on all five outputs, then the fused loss."""
    sc, vol = scene
    n = 2047
    rays, pts, ndc, z = _samples(sc, n, S, seed=S)
    rd = rays[:, 3:6]
    fn = _net()
    cot = {k: v.to(DEV) for k, v in _cotangents(n, S, seed=11).items()}
    a = _run(sc, vol, fn, pts, ndc, z, rd, white, grad_mode, grads=cot)
    b = _run(sc, vol, fn, pts, ndc, z, rd, white, grad_mode, grads=cot)
    assert torch.isfinite(a[1]).all() and a[1].abs().max() > 0
    _assert_same(a, b)
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(5)).to(DEV)
    fa = _fused(sc, vol, fn, pts, ndc, z, rd, white, grad_mode, target)
    fb = _fused(sc, vol, fn, pts, ndc, z, rd, white, grad_mode, target)
    _assert_same(fa, fb)
    assert abs(fa[4].item() - ((fa[2] - target) ** 2).mean().item()) < 1e-6


def _pure_scatter(vol, ndc, g8):
    """On the CPU: the fp64 index_add of the fp32 products g * ((wx * wy) * wz) the kernel forms (trilinear_corners,
    zeros padding, channels-last [D,Hp,Wp,8]), and the number of contributions each entry receives."""
    D, Hp, Wp = vol.shape[2:]
    nd = ndc.reshape(-1, 3)
    g = g8.reshape(-1, 8)
    i = [((nd[:, a] * 2.0 - 1.0 + 1.0) * 0.5) * float(s - 1) for a, s in ((0, Wp), (1, Hp), (2, D))]
    i0 = [torch.floor(t) for t in i]
    w = [((f + 1.0) - t, t - f) for f, t in zip(i0, i)]
    o = [f.to(torch.int64) for f in i0]
    ref = torch.zeros(D * Hp * Wp * 8, dtype=torch.float64)
    cnt = torch.zeros(D * Hp * Wp * 8, dtype=torch.float64)
    for c in range(8):
        bx, by, bz = c & 1, (c >> 1) & 1, c >> 2
        x, y, zz = o[0] + bx, o[1] + by, o[2] + bz
        ok = (x >= 0) & (x < Wp) & (y >= 0) & (y < Hp) & (zz >= 0) & (zz < D)
        wgt = (w[0][bx] * w[1][by]) * w[2][bz]
        p = (g * wgt.unsqueeze(1))[ok]                          # fp32 products
        idx = ((((zz * Hp + y) * Wp + x) * 8)[ok]).unsqueeze(1) + torch.arange(8)
        ref.index_add_(0, idx.reshape(-1), p.reshape(-1).double())
        cnt.index_add_(0, idx.reshape(-1), torch.ones(idx.numel(), dtype=torch.float64))
    return ref.reshape(D, Hp, Wp, 8).to(DEV), cnt.reshape(D, Hp, Wp, 8).to(DEV)


@pytest.mark.parametrize("grad_mode", MODES)
def test_deterministic_scatter_is_the_exact_sum(scene, deterministic, grad_mode):
    """Only an input_feat cotangent: the volume gradient is a pure trilinear scatter of it.  Against the fp64 sum of the
    same fp32 products: within 1 ulp plus half a quantum per contribution, and >= 99.9 % of entries bit-equal."""
    sc, vol = scene
    n, S = 2048, 128
    rays, pts, ndc, z = _samples(sc, n, S, seed=3)
    fn = _net()
    gf = 0.01 * torch.randn(n, S, 20, generator=torch.Generator().manual_seed(6))
    _, g_vol, _, _ = _run(sc, vol, fn, pts, ndc, z, rays[:, 3:6], False, grad_mode, grads={"input_feat": gf.to(DEV)})
    ref, cnt = _pure_scatter(vol, ndc, gf[..., :8].contiguous())
    em = math.frexp(gf[..., :8].abs().max().item())[1] - 1
    e = 61 - (n * S - 1).bit_length() - em
    quantum = 2.0 ** -e
    ref32 = ref.float()
    ulp = (torch.nextafter(ref32.abs(), torch.tensor(float("inf"), device=DEV)) - ref32.abs()).double()
    err = (g_vol.double() - ref).abs()
    assert (err <= ulp + 0.5 * quantum * cnt).all(), (err - ulp - 0.5 * quantum * cnt).max().item()
    equal = (g_vol == ref32).double().mean().item()
    touched = cnt > 0
    equal_touched = (g_vol[touched] == ref32[touched]).double().mean().item()
    print(f"\n[det scatter {grad_mode}] quantum {quantum:.3e} max|g| {gf[..., :8].abs().max().item():.3e} "
          f"bit-equal {equal:.6f} (touched entries {equal_touched:.6f}, {touched.double().mean().item():.3f} touched)")
    assert equal >= 0.999


@pytest.mark.parametrize("grad_mode", MODES)
def test_deterministic_backward_agrees_with_atomic_path_and_oracle(scene, weights, grad_mode):
    sc, vol = scene
    n, S, white = 200, 64, True
    rays, pts, ndc, z = _samples(sc, n, S, seed=17)
    rd = rays[:, 3:6]
    fn = _net()
    cot = _cotangents(n, S, seed=12)
    grads = {k: v.to(DEV) for k, v in cot.items()}
    atomic = _run(sc, vol, fn, pts, ndc, z, rd, white, grad_mode, grads=grads)
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        det = _run(sc, vol, fn, pts, ndc, z, rd, white, grad_mode, grads=grads)
    finally:
        torch.use_deterministic_algorithms(was)
    for x, y in zip(atomic[0], det[0]):                         # MLP gradients: same kernel code, private accumulators
        assert torch.equal(x, y)
    assert torch.equal(atomic[2], det[2]) and torch.equal(atomic[3], det[3])
    e_atomic = (det[1] - atomic[1]).abs().max().item() / atomic[1].abs().max().item()
    assert e_atomic < 1e-6, e_atomic
    # the oracle's fp32 autograd on the CPU
    wt = {k: v.clone().requires_grad_(k.startswith("mlp/")) for k, v in weights.items()}
    vt = vol.clone().requires_grad_(True)
    rgb, feat, w, depth, alpha = orc.render_samples(pts, ndc, z, rd, vt, sc.imgs_raw, sc.pose_source, wt, white_bkgd=white)
    loss = (rgb * cot["rgb"]).sum() + (depth * cot["depth"]).sum() + (w * cot["weights"]).sum() + \
        (alpha * cot["alpha"]).sum() + (feat * cot["input_feat"]).sum()
    loss.backward()
    worst = 0.0
    for (name, _), g in zip(backend._ordered_named_params(fn), det[0]):
        worst = max(worst, _rel(g.cpu(), wt["mlp/" + name].grad))
    e_v = _rel(det[1].permute(3, 0, 1, 2).unsqueeze(0).cpu(), vt.grad)
    print(f"\n[det agreement {grad_mode}] vs atomic vol {e_atomic:.3e} ; vs oracle mlp {worst:.3e} vol {e_v:.3e}")
    assert worst < GATE[grad_mode] and e_v < GATE[grad_mode]


@pytest.mark.parametrize("S", [32, 128])
def test_deterministic_volume_gradient_is_permutation_invariant_in_fp32(scene, deterministic, S):
    """MLP_FP32 computes every row independently, so shuffling the rays (and their cotangents) moves each sample's 8
    gradients, not their values, and the integer sum does not depend on the order."""
    sc, vol = scene
    n = 1021
    rays, pts, ndc, z = _samples(sc, n, S, seed=23)
    fn = _net()
    cot = _cotangents(n, S, seed=13)
    a = _run(sc, vol, fn, pts, ndc, z, rays[:, 3:6], False, lib.MLP_FP32, grads={k: v.to(DEV) for k, v in cot.items()})
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(1))
    b = _run(sc, vol, fn, pts[perm], ndc[perm], z[perm], rays[perm, 3:6], False, lib.MLP_FP32,
             grads={k: v[perm].to(DEV) for k, v in cot.items()})
    assert torch.equal(a[1], b[1])
    assert torch.equal(a[2][perm.to(DEV)], b[2])


@pytest.mark.parametrize("grad_mode", MODES)
def test_deterministic_backward_propagates_nan_like_the_atomics(scene, grad_mode):
    sc, vol = scene
    n, S = 300, 64
    rays, pts, ndc, z = _samples(sc, n, S, seed=29)
    fn = _net()
    cot = _cotangents(n, S, seed=14)
    inside = ((ndc > 0.05) & (ndc < 0.95)).all(-1).nonzero()
    r, s = inside[len(inside) // 2].tolist()
    cot["input_feat"][r, s, 2] = float("nan")
    grads = {k: v.to(DEV) for k, v in cot.items()}
    atomic = _run(sc, vol, fn, pts, ndc, z, rays[:, 3:6], False, grad_mode, grads=grads)[1]
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        det = _run(sc, vol, fn, pts, ndc, z, rays[:, 3:6], False, grad_mode, grads=grads)[1]
    finally:
        torch.use_deterministic_algorithms(was)
    assert atomic.isnan().any()
    assert torch.equal(atomic.isnan(), det.isnan())
    ok = ~det.isnan()
    assert (det[ok] - atomic[ok]).abs().max() <= 1e-6 * atomic[ok].abs().max()


def _finetune(sc, vol, grad_mode, steps, n=256, S=128):
    d = sc.to(DEV)
    fn = _net()
    volume = backend.RefVolume(vol.clone().to(DEV))
    tuner = backend.FineTuner(fn, volume, d.imgs_raw, d.pose_source, lr=5e-4, grad_mode=grad_mode)
    losses = []
    for it in range(steps):
        rays, pts, ndc, z = _samples(sc, n, S, seed=200 + it % 5)
        target = torch.full((n, 3), 0.3, device=DEV)
        losses.append(tuner.step(pts.to(DEV), ndc.to(DEV), z.to(DEV), rays[:, 3:6].to(DEV), target)[0].clone())
    return [p.detach().clone() for p in fn.ordered_params()], volume.feat_volume.detach().clone(), torch.cat(losses)


@pytest.mark.parametrize("grad_mode", MODES)
def test_deterministic_finetuner_runs_repeat_bit_for_bit(scene, deterministic, grad_mode):
    sc, vol = scene
    pa, va, la = _finetune(sc, vol, grad_mode, 50)
    pb, vb, lb = _finetune(sc, vol, grad_mode, 50)
    for x, y in zip(pa, pb):
        assert torch.equal(x, y)
    assert torch.equal(va, vb) and torch.equal(la, lb)
    assert lb[-1] < lb[0]


def _autograd_adam(sc, vol, grad_mode, steps, n=200, S=64):
    d = sc.to(DEV)
    fn = _net()
    volume = backend.RefVolume(vol.clone().to(DEV))
    opt = torch.optim.Adam(list(fn.parameters()) + list(volume.parameters()), lr=5e-4)
    for it in range(steps):
        rays, pts, ndc, z = _samples(sc, n, S, seed=300 + it)
        target = torch.rand(n, 3, generator=torch.Generator().manual_seed(it)).to(DEV)
        rgb = backend.rendering(Args(), d.pose_source, pts.to(DEV), ndc.to(DEV), z.to(DEV), None, rays[:, 3:6].to(DEV),
                                volume_feature=volume, imgs=d.imgs_raw, network_fn=fn, mlp_mode=lib.MLP_FP32,
                                grad_mode=grad_mode)[0]
        opt.zero_grad(set_to_none=True)
        ((rgb - target) ** 2).mean().backward()
        opt.step()
    return [p.detach().clone() for p in fn.ordered_params()], volume.feat_volume.detach().clone()


@pytest.mark.parametrize("grad_mode", MODES)
def test_deterministic_rendering_under_autograd_with_adam_repeats(scene, deterministic, grad_mode):
    sc, vol = scene
    pa, va = _autograd_adam(sc, vol, grad_mode, 10)
    pb, vb = _autograd_adam(sc, vol, grad_mode, 10)
    for x, y in zip(pa, pb):
        assert torch.equal(x, y)
    assert torch.equal(va, vb)


@pytest.mark.parametrize("grad_mode", MODES)
def test_deterministic_backward_with_frozen_volume(scene, deterministic, grad_mode):
    sc, vol = scene
    n, S = 130, 32
    rays, pts, ndc, z = _samples(sc, n, S, seed=9)
    fn = _net()
    cot = {k: v.to(DEV) for k, v in _cotangents(n, S, seed=4).items()}
    with_vol = _run(sc, vol, fn, pts, ndc, z, rays[:, 3:6], False, grad_mode, grads=cot)
    frozen = _run(sc, vol, fn, pts, ndc, z, rays[:, 3:6], False, grad_mode, grads=cot, want_volume_grad=False)
    assert frozen[1] is None
    for a, b in zip(with_vol[0], frozen[0]):
        assert torch.equal(a, b)
    assert torch.equal(with_vol[2], frozen[2]) and torch.equal(with_vol[3], frozen[3])
