"""GPU: grad_mode GRAD_TC_FULL -- the rays fine-tuning backward with its forward recompute on tensor cores
(render_bwd_tc_kernel<.., FULL = true>, tile_mlp_tc).

  * parity: rgb, depth, the fused loss and every gradient against tests/grad_emulation_full on the same samples, and
    against MLP_FP32 / the oracle's fp32 autograd within the band tests/test_oracle_grad_emulation_full.py pins;
  * invariants: t_stop = 0 is the non-stop call bit for bit; a ray's outputs do not depend on the batch (per-row
    scales); the early-termination paths (immediate, deferred, packed); the deterministic variant repeats bit for bit;
  * range: a scaled volume and scaled weights, and a tiny loss scale, stay finite and within the gates.
"""
import pytest
import torch

from grad_emulation_full import mlp_full_emulated
from oracle import mvsnerf_oracle as orc
from mvsnerf_b200 import backend, lib, synthetic
from test_gpu_backward_rays import _bwd_rays, _host_march, _jitter, _kernel_order_ndc, _net, _rays, _rel
from test_oracle_grad_emulation_full import BAND

pytestmark = pytest.mark.gpu
DEV = "cuda"
FULL = lib.GRAD_TC_FULL
# Kernel against the emulation on the same samples.  The kernel accumulates in fp32 (wgmma, FFMA heads), the
# emulation exactly, so the forward differs by ~1e-5 (rgb 3.6e-5 measured) and an fp16 operand rounds the other way
# now and then.  The gradients amplify such differences: d mod = d g * h / mod (pre = h / mod) is large where mod is
# near 0, and a ReLU gate can flip -- the same sensitivity that puts the fp16 forward ~0.1 of max|g| from fp32 autograd
# (test_oracle_grad_emulation_full.BAND).  Measured on an H100 80GB HBM3 over CASES: rgb <= 3.7e-5, depth <= 1.7e-5 of
# far, loss <= 1.6e-6, gradients <= 7.7e-3 (MLP, S 128 n 300) and <= 7.6e-4 (volume) of max|g|; so the gradient gate
# is 2e-2 of max|g| per tensor, not the 2e-4 MLP_TC_HALF's backward-only rounding holds to.  With activations of
# 1e4 - 1e5 (test_range) the fp32 accumulation rounds coarser: rgb 2.5e-4 (volume x3) and 4.4e-4 (weights x1.5).
EMU = {"rgb": 2e-4, "depth": 2e-4, "loss": 2e-4, "grad": 2e-2}
EMU_RANGE = {"rgb": 1e-3, "depth": 1e-3, "loss": 2e-4, "grad": 2e-2}


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


def _cot(n, S, seed=1):
    g = torch.Generator().manual_seed(seed)
    c = {"target": torch.rand(n, 3, generator=g), "depth": 0.1 * torch.randn(n, generator=g),
         "weights": 0.05 * torch.randn(n, S, generator=g), "alpha": 0.05 * torch.randn(n, S, generator=g),
         "input_feat": 0.01 * torch.randn(n, S, 20, generator=g)}
    return {k: v.to(DEV) for k, v in c.items()}


def _kernel(sc, vol, fn, rays, S, white, mode, j, cot, n_total=None):
    loss = torch.zeros(1, device=DEV)
    grads = {k: cot[k] for k in ("depth", "weights", "alpha", "input_feat")}
    g, v, rgb, depth = _bwd_rays(sc, vol, fn, rays, S, white, mode, j, target_rgb=cot["target"], grads=grads,
                                 loss_out=loss, n_total=n_total)
    return {"rgb": rgb, "depth": depth, "loss": loss[0], "mlp": [t.clone() for t in g], "vol": v.permute(3, 0, 1, 2)}


def _oracle(sc, vol, weights, rays, S, white, j, cot, mlp_fn, n_total=None):
    """the oracle's render_samples on the kernel's own samples (host march, NDC in the kernel's order), on the GPU"""
    pts, _, z = _host_march(sc, rays, S, j)
    ndc = _kernel_order_ndc(sc, pts)
    d = sc.to(DEV)
    wt = {k: v.to(DEV).clone().requires_grad_(k.startswith("mlp/")) for k, v in weights.items()}
    vt = vol.to(DEV).clone().requires_grad_(True)
    rgb, feat, w, depth, alpha = orc.render_samples(pts, ndc, z, rays[:, 3:6], vt, d.imgs_raw, d.pose_source, wt,
                                                    white_bkgd=white, mlp_fn=mlp_fn)
    n = rays.shape[0]
    loss = ((rgb - cot["target"]) ** 2).sum() / (3.0 * (n if n_total is None else n_total))
    (loss + (depth * cot["depth"]).sum() + (w * cot["weights"]).sum() + (alpha * cot["alpha"]).sum()
     + (feat * cot["input_feat"]).sum()).backward()
    return {"rgb": rgb.detach(), "depth": depth.detach(), "loss": loss.detach(), "vol": vt.grad[0], "mlp": wt}


def _errors(k, ref, fn, far):
    mlp = [_rel(g, ref["mlp"]["mlp/" + name].grad) for (name, _), g in zip(backend._ordered_named_params(fn), k["mlp"])]
    return {"rgb": (k["rgb"] - ref["rgb"]).abs().max().item(), "depth": (k["depth"] - ref["depth"]).abs().max().item() / far,
            "loss": abs(k["loss"].item() - ref["loss"].item()) / ref["loss"].item(), "mlp": max(mlp),
            "vol": _rel(k["vol"], ref["vol"])}


CASES = [(32, 130, True, True), (48, 21, False, True), (128, 37, False, False), (128, 300, True, True),
         (48, 77, True, False)]


@pytest.mark.parametrize("S,n,white,jit", CASES)
def test_parity_with_emulation_and_fp32(scene, weights, S, n, white, jit):
    sc, vol = scene
    fn = _net()
    rays = _rays(sc, n, seed=S + n)
    j = _jitter(n, S, seed=S) if jit else None
    cot = _cot(n, S)
    far = sc.near_far[1]
    k = _kernel(sc, vol, fn, rays, S, white, FULL, j, cot)
    emu = _oracle(sc, vol, weights, rays, S, white, j, cot, mlp_full_emulated)
    ref = _oracle(sc, vol, weights, rays, S, white, j, cot, None)
    e_emu, e_ref = _errors(k, emu, fn, far), _errors(k, ref, fn, far)
    k32 = _kernel(sc, vol, fn, rays, S, white, lib.MLP_FP32, j, cot)
    e_rgb32 = (k["rgb"] - k32["rgb"]).abs().max().item()
    print(f"\n[TC_FULL S={S} n={n} white={white} jitter={jit}] vs emulation: "
          + " ".join(f"{a} {b:.2e}" for a, b in e_emu.items()) + " | vs fp32 autograd: "
          + " ".join(f"{a} {b:.2e}" for a, b in e_ref.items()) + f" | rgb vs MLP_FP32 kernel {e_rgb32:.2e}")
    for key in ("rgb", "depth", "loss"):
        assert e_emu[key] < EMU[key], (key, e_emu[key])
    assert e_emu["mlp"] < EMU["grad"] and e_emu["vol"] < EMU["grad"], e_emu
    for key in BAND:
        assert e_ref[key] < BAND[key], (key, e_ref[key])
    assert e_rgb32 < 5e-3


def test_t_stop_zero_is_the_plain_call(scene):
    sc, vol = scene
    fn = _net()
    n, S = 300, 128
    rays, j = _rays(sc, n, seed=5), _jitter(n, S, seed=5)
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    outs = []
    for t_stop in (None, 0.0):
        loss = torch.zeros(1, device=DEV)
        g, v, rgb, depth = _bwd_rays(sc, vol, fn, rays, S, True, FULL, j, target_rgb=target, loss_out=loss, t_stop=t_stop)
        outs.append((g, v, rgb, depth, loss))
    (g0, v0, r0, d0, l0), (g1, v1, r1, d1, l1) = outs
    assert torch.equal(r0, r1) and torch.equal(d0, d1)
    for a, b in zip(g0, g1):
        assert torch.allclose(a, b, rtol=0, atol=1e-6 * b.abs().max().item())   # float atomics: summation order only
    assert torch.allclose(v0, v1, rtol=0, atol=1e-6 * v1.abs().max().item())


def test_rays_do_not_depend_on_the_batch(scene, deterministic):
    """The same rays in another order and in another batch: each ray's rgb, depth and loss term are bit-identical
    (per-row scales; a shared per-tile scale would mix the rays of a tile)."""
    sc, vol = scene
    fn = _net()
    n, S = 257, 48
    rays, j = _rays(sc, n, seed=11), _jitter(n, S, seed=11)
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(3)).to(DEV)
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(4)).to(DEV)
    _, _, r0, d0 = _bwd_rays(sc, vol, fn, rays, S, False, FULL, j, target_rgb=target)
    _, _, r1, d1 = _bwd_rays(sc, vol, fn, rays[perm].contiguous(), S, False, FULL, j[perm].contiguous(),
                             target_rgb=target[perm].contiguous())
    assert torch.equal(r1, r0[perm]) and torch.equal(d1, d0[perm])
    # a ray's loss term: one ray per call, summed by the deterministic fixed-order reduction
    for i in (0, 100, 256):
        loss = torch.zeros(1, device=DEV)
        _, _, ri, _ = _bwd_rays(sc, vol, fn, rays[i:i + 1], S, False, FULL, j[i:i + 1], target_rgb=target[i:i + 1],
                                loss_out=loss, n_total=n)
        assert torch.equal(ri[0], r0[i])
        assert abs(loss.item() - ((r0[i] - target[i]) ** 2).sum().item() / (3 * n)) <= 1e-6 * loss.item()


@pytest.mark.parametrize("det", [False, True])
def test_early_termination_paths(scene, det):
    """400 rays x 128 samples with t_stop = 0.5: tiles back-propagated at once, deferred and packed.  The recompute of
    a deferred ray repeats phase A, so the written rgb is the render truncated at each ray's live count: within
    (-t_stop, 0] of the full render per channel; the live counts do not depend on the batch."""
    sc, vol = scene
    fn = _net()
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det, warn_only=True)
    try:
        many = torch.cat([synthetic.scene_rays(sc)] * 2)[:400].contiguous().to(DEV)
        j = _jitter(400, 128, seed=7)
        target = torch.rand(400, 3, generator=torch.Generator().manual_seed(8)).to(DEV)
        tiles = torch.zeros(3, dtype=torch.int64, device=DEV)
        live = torch.empty(400, dtype=torch.int32, device=DEV)
        _, _, rgb_s, depth_s = _bwd_rays(sc, vol, fn, many, 128, False, FULL, j, target_rgb=target, t_stop=0.5,
                                         live_samples=live, tiles_done=tiles)
        _, _, rgb_f, depth_f = _bwd_rays(sc, vol, fn, many, 128, False, FULL, j, target_rgb=target)
        assert (tiles > 0).all(), tiles.tolist()
        assert (live >= 1).all() and (live <= 128).all() and (live < 128).any()
        diff = rgb_s - rgb_f
        assert (diff <= 1e-6).all() and (diff > -0.5 - 1e-6).all()
        assert torch.equal(rgb_s[live == 128], rgb_f[live == 128]) or (diff[live == 128].abs() <= 1e-6).all()
        perm = torch.randperm(400, generator=torch.Generator().manual_seed(9)).to(DEV)
        live_p = torch.empty(400, dtype=torch.int32, device=DEV)
        _, _, rgb_p, _ = _bwd_rays(sc, vol, fn, many[perm].contiguous(), 128, False, FULL, j[perm].contiguous(),
                                   target_rgb=target[perm].contiguous(), t_stop=0.5, live_samples=live_p)
        assert torch.equal(live_p, live[perm]) and torch.equal(rgb_p, rgb_s[perm])
    finally:
        torch.use_deterministic_algorithms(was, warn_only=True)


def test_deterministic_repeats(scene, deterministic):
    sc, vol = scene
    fn = _net()
    n, S = 1023, 128
    rays, j = _rays(sc, n, seed=4), _jitter(n, S, seed=4)
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(5)).to(DEV)
    runs = []
    for t_stop in (None, None, 1e-4, 1e-4):
        loss = torch.zeros(1, device=DEV)
        g, v, rgb, depth = _bwd_rays(sc, vol, fn, rays, S, False, FULL, j, target_rgb=target, loss_out=loss,
                                     t_stop=t_stop)
        runs.append(([t.clone() for t in g], v.clone(), rgb, depth, loss))
    for a, b in ((runs[0], runs[1]), (runs[2], runs[3])):
        for x, y in zip(a[0], b[0]):
            assert torch.equal(x, y)
        for x, y in zip(a[1:], b[1:]):
            assert torch.equal(x, y)


def test_step_rays_trains(scene):
    """FineTuner.step_rays in this mode, with and without t_stop: the loss falls over 30 steps."""
    sc, vol = scene
    d = sc.to(DEV)
    for t_stop in (None, 1e-4):
        fn = _net()
        tuner = backend.FineTuner(fn, backend.RefVolume(vol.clone().to(DEV)), d.imgs_raw, d.pose_source, lr=5e-4,
                                  grad_mode=FULL)
        rays = _rays(sc, 512, seed=1)
        target = torch.rand(512, 3, generator=torch.Generator().manual_seed(6)).to(DEV)
        losses = [tuner.step_rays(rays, target, sc.near_far, float(sc.pad), N_samples=64, t_stop=t_stop)[0].item()
                  for _ in range(30)]
        assert all(torch.isfinite(torch.tensor(losses))) and losses[-1] < losses[0], losses


@pytest.mark.parametrize("case", ["volume_x3", "weights_x1.5", "loss_scale"])
def test_range(scene, weights, case):
    """test_gpu_tc_range.py's cases: volume x3, trunk and pts_bias weights x1.5, loss scale 1 / (3 10^7).  Everything
    finite; against the emulation within EMU_RANGE (the forward's fp32 accumulation at activations of 1e4 - 1e5)."""
    sc, vol = scene
    n, S = 130, 32
    fn = _net()
    w = dict(weights)
    if case == "volume_x3":
        vol = vol * 3.0
    if case == "weights_x1.5":
        scaled = [f"nerf.pts_linears.{i}.weight" for i in range(6)] + ["nerf.pts_bias.weight"]
        with torch.no_grad():
            for name, p in backend._ordered_named_params(fn):
                if name in scaled:
                    p.mul_(1.5)
        w = {k: (v * 1.5 if k[len("mlp/"):] in scaled else v) for k, v in weights.items()}
    n_total = 10 ** 7 if case == "loss_scale" else None
    rays, j = _rays(sc, n, seed=S + n), _jitter(n, S, seed=S)
    cot = _cot(n, S)
    if case == "loss_scale":
        cot = {**cot, "depth": cot["depth"] * 0, "weights": cot["weights"] * 0, "alpha": cot["alpha"] * 0,
               "input_feat": cot["input_feat"] * 0}
    k = _kernel(sc, vol, fn, rays, S, True, FULL, j, cot, n_total=n_total)
    emu = _oracle(sc, vol, w, rays, S, True, j, cot, mlp_full_emulated, n_total=n_total)
    for t in [k["rgb"], k["depth"], k["vol"], *k["mlp"]]:
        assert torch.isfinite(t).all()
    e = _errors(k, emu, fn, sc.near_far[1])
    print(f"\n[TC_FULL range {case}] vs emulation: " + " ".join(f"{a} {b:.2e}" for a, b in e.items()))
    assert e["rgb"] < EMU_RANGE["rgb"] and e["depth"] < EMU_RANGE["depth"] and e["loss"] < EMU_RANGE["loss"], e
    assert e["mlp"] < EMU_RANGE["grad"] and e["vol"] < EMU_RANGE["grad"], e
