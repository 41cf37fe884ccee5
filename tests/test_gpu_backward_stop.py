"""GPU: early ray termination in the fine-tuning step (mvsn_render_backward_rays_stop: backend.render_backward_rays and
FineTuner.step_rays with t_stop).

  * t_stop = 0 is bit-identical to the entry without it, in both grad modes and both summation orders;
  * the rule: each ray's live count follows from the alpha of render_rays (MLP_FP32) and T in the kernel's fp32 order;
  * the gradients are exactly those of the truncated render (the oracle's autograd with w_j masked for j >= L);
  * the signed bounds against t_stop = 0, on batches of a scene whose rays become opaque (synthetic.make_plane_scene);
  * the tile counters follow from the live counts, and every path (immediate, deferred, packed) runs;
  * packing independence, determinism, a frozen volume, misaligned rays; FineTuner.step_rays with t_stop.
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
MODES = [lib.MLP_FP32, lib.MLP_TC_HALF]
GATE = {lib.MLP_FP32: 2e-4, lib.MLP_TC_HALF: 3e-3}
WPATH = os.path.join(GOLDEN, "mvsnerf_v0_weights.npz")


class Ctx:
    def __init__(self, sc, vol):
        self.sc, self.d, self.vol = sc, sc.to(DEV), vol.to(DEV)
        self.fn = backend.MVSNeRF().to(DEV)
        backend.load_weights_npz(self.fn, None, WPATH)
        self.rays_all = synthetic.scene_rays(sc).to(DEV).contiguous()

    def rays(self, n, seed):
        g = torch.Generator().manual_seed(seed)
        return self.rays_all[torch.randperm(self.rays_all.shape[0], generator=g)[:n].to(DEV)].contiguous()

    def bwd(self, rays, S, mode, t_stop, j=None, white=False, lindisp=False, det=False, **kw):
        """(grad_mlp, grad_volume, rgb, depth, loss, live, tiles) of one backward launch"""
        n = rays.shape[0]
        live = torch.full((n,), -1, dtype=torch.int32, device=DEV) if t_stop is not None else None
        tiles = torch.zeros(3, dtype=torch.int64, device=DEV) if t_stop is not None else None
        loss = torch.zeros(1, device=DEV)
        if "grads" not in kw:
            kw.setdefault("target_rgb", torch.rand(n, 3, generator=torch.Generator().manual_seed(n)).to(DEV))
            loss = kw.setdefault("loss_out", loss)
        was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
        torch.use_deterministic_algorithms(det, warn_only=True)
        try:
            g, v, rgb, depth = backend.render_backward_rays(
                rays, self.vol, self.d.imgs_raw, self.d.pose_source, self.fn, self.sc.near_far, float(self.sc.pad),
                N_samples=S, lindisp=lindisp, jitter=j, white_bkgd=white, want_forward=True, grad_mode=mode,
                t_stop=t_stop, live_samples=live, tiles_done=tiles, **kw)
        finally:
            torch.use_deterministic_algorithms(was, warn_only=warn)
        return g, v, rgb, depth, loss, live, (tiles.tolist() if tiles is not None else None)

    def alpha(self, rays, S, white=False):
        """alpha [N,S] of mvsn_render_rays with the MLP_FP32 image (the recompute's forward)"""
        L = lib.load()
        sc, keep = backend._make_scene(self.d.pose_source, self.vol, self.d.imgs_raw, self.fn, white, lib.MLP_FP32)
        rp = lib.RayParams(float(self.sc.near_far[0]), float(self.sc.near_far[1]), float(self.sc.pad), 0)
        n = rays.shape[0]
        rgb, depth, alpha = torch.empty(n, 3, device=DEV), torch.empty(n, device=DEV), torch.empty(n, S, device=DEV)
        lib.check(L.mvsn_render_rays(C.byref(sc), C.byref(rp), lib.ptr(rays), lib.ptr(torch.linspace(0, 1, S, device=DEV)),
                                     n, S, lib.ptr(rgb), lib.ptr(depth), None, lib.ptr(alpha), None, lib.stream_ptr()),
                  "mvsn_render_rays")
        torch.cuda.synchronize()
        del keep
        return alpha


def _volume(sc):
    mvs = backend.MVSNet().to(DEV).train()
    fn = backend.MVSNeRF().to(DEV)
    backend.load_weights_npz(fn, mvs, WPATH)
    d = sc.to(DEV)
    with torch.no_grad():
        vol, _, _ = mvs(d.imgs_norm, d.proj_mats, sc.near_far, pad=sc.pad)
    return vol.detach().clone()


@pytest.fixture(scope="module")
def plane():
    sc = synthetic.make_plane_scene(96, 128, pad=4, seed=3)
    return Ctx(sc, _volume(sc))


def _live_of(alpha, t_stop):
    """each ray's live count from alpha in the kernel's fp32 order: T_0 = 1, T_{j+1} = T_j ((1 - a_j) + 1e-10)"""
    n, S = alpha.shape
    T = torch.ones(n, dtype=torch.float32, device=alpha.device)
    live = torch.zeros(n, dtype=torch.int32, device=alpha.device)
    alive = torch.ones(n, dtype=torch.bool, device=alpha.device)
    one, tiny = torch.tensor(1.0, device=alpha.device), torch.tensor(1e-10, dtype=torch.float32, device=alpha.device)
    for j in range(S):
        alive &= T >= t_stop
        live += alive.int()
        T = T * ((one - alpha[:, j]) + tiny)
    return live


def _same(a, b, what=""):
    assert a.dtype == b.dtype and torch.equal(a, b), (what, (a.float() - b.float()).abs().max().item())


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("S,n,white,lindisp,jit", [(32, 130, True, False, True), (48, 21, False, True, False),
                                                   (128, 300, True, False, True), (128, 37, False, False, False),
                                                   (32, 1, False, False, True)])
def test_t_stop_zero_is_bit_identical(plane, S, n, white, lindisp, jit, det):
    rays = plane.rays(n, seed=S + n)
    j = torch.rand(n, S, generator=torch.Generator().manual_seed(S)).to(DEV) if jit else None
    for mode in MODES:
        a = plane.bwd(rays, S, mode, None, j, white, lindisp, det)
        b = plane.bwd(rays, S, mode, 0.0, j, white, lindisp, det)
        for x, y in zip(a[0], b[0]):
            _same(x, y, "mlp")
        _same(a[2], b[2], "rgb")
        _same(a[3], b[3], "depth")
        assert torch.all(b[5] == S)
        groups = -(-n // (128 // S))
        assert b[6] == [groups, 0, 0]                              # every tile back-propagated at once
        if det:                                                    # the float atomics are not reproducible
            _same(a[1], b[1], "volume")
            _same(a[4], b[4], "loss")
        else:
            assert (a[1] - b[1]).abs().max().item() <= 1e-6 * a[1].abs().max().item()
            assert abs(a[4].item() - b[4].item()) <= 1e-6 * a[4].item()


@pytest.mark.parametrize("S,n", [(128, 200), (64, 130), (32, 77)])
@pytest.mark.parametrize("t_stop", [1e-4, 1e-2, 0.5])
def test_live_samples_follow_the_rule(plane, S, n, t_stop):
    rays = plane.rays(n, seed=n)
    want = _live_of(plane.alpha(rays, S), t_stop)
    for mode in MODES:
        live = plane.bwd(rays, S, mode, t_stop)[5]
        _same(live, want, "live")
    assert (want >= 1).all() and (want < S).any()


def _truncated_render(pts, ndc, z, rays_d, vol, imgs_raw, pose, w, live, white):
    """orc.render_samples with w_j = 0 for j >= live (the function the stop entry differentiates)"""
    N, S = pts.shape[:2]
    dirs = orc.view_direction(rays_d, pose["w2cs"][0])
    feat = torch.cat([orc.lookup_volume(vol, ndc), orc.gather_colors(pts, pose["w2cs"], pose["intrinsics"], imgs_raw[0])], -1)
    x = torch.cat([orc.positional_encoding(ndc), feat, dirs.unsqueeze(1).expand(-1, S, -1)], -1)
    raw = orc.mlp(x, w)
    alpha = 1.0 - torch.exp(-raw[..., 3])
    trans = torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1.0 - alpha + 1e-10], -1), -1)[:, :-1]
    mask = (torch.arange(S)[None, :] < live[:, None]).float()
    weights = alpha * trans * mask
    rgb = (weights.unsqueeze(-1) * raw[..., :3]).sum(-2)
    depth = (weights * z).sum(-1)
    if white:
        rgb = rgb + (1.0 - weights.sum(-1, keepdim=True))
    return rgb, depth


@pytest.mark.parametrize("grad_mode", MODES)
@pytest.mark.parametrize("S,n,white", [(32, 130, True), (128, 60, False)])
def test_exact_gradients_of_the_truncated_render(plane, weights, grad_mode, S, n, white):
    from test_gpu_backward_rays import _host_march, _kernel_order_ndc
    sc = plane.sc
    rays = plane.rays(n, seed=7)
    j = torch.rand(n, S, generator=torch.Generator().manual_seed(5)).to(DEV)
    pts, _, z = _host_march(sc, rays, S, j)
    ndc = _kernel_order_ndc(sc, pts)
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(n)).to(DEV)
    g_k, v_k, rgb_k, depth_k, loss_k, live, _ = plane.bwd(rays, S, grad_mode, 1e-3, j, white)
    assert (live < S).any()
    wt = {k: v.clone().requires_grad_(k.startswith("mlp/")) for k, v in weights.items()}
    vt = plane.vol.detach().cpu().clone().requires_grad_(True)
    rgb, depth = _truncated_render(pts.cpu(), ndc.cpu(), z.cpu(), rays[:, 3:6].cpu(), vt, sc.imgs_raw, sc.pose_source, wt,
                                   live.long().cpu(), white)
    loss = ((rgb - target.cpu()) ** 2).mean()
    loss.backward()
    assert (rgb_k.cpu() - rgb).abs().max().item() < 1e-5 and (depth_k.cpu() - depth).abs().max().item() < 1e-4
    assert abs(loss_k.item() - loss.item()) <= 1e-5 * loss.item()
    pairs = [(g.cpu(), wt["mlp/" + name].grad) for (name, _), g in zip(backend._ordered_named_params(plane.fn), g_k)]
    pairs.append((v_k.permute(3, 0, 1, 2).unsqueeze(0).cpu(), vt.grad))
    excess = max((a - b).abs().max().item() - GATE[grad_mode] * b.abs().max().item() - 1e-8 for a, b in pairs)
    assert excess <= 0, excess


@pytest.mark.parametrize("white", [False, True])
@pytest.mark.parametrize("t_stop", [1e-4, 1e-3, 1e-2])
def test_bounds_against_the_full_step(plane, t_stop, white):
    S, n = 128, 1024
    rays = plane.rays(n, seed=11)
    far = float(rays[:, 7].max())
    for mode in MODES:
        full = plane.bwd(rays, S, mode, 0.0, white=white)
        cut = plane.bwd(rays, S, mode, t_stop, white=white)
        d = cut[2] - full[2]
        ulp = 4 * 2.0 ** -23
        if white:
            assert d.min().item() >= -ulp and d.max().item() < t_stop + ulp
        else:
            assert d.max().item() <= ulp and d.min().item() > -t_stop - ulp
        dd = full[3] - cut[3]
        assert dd.min().item() >= -ulp * far and dd.max().item() < t_stop * far + ulp * far
        assert (cut[5] < S).float().mean().item() > 0.5
        print(f"\n[bounds {mode} eps={t_stop} white={white}] live fraction {cut[5].float().mean().item() / S:.3f} "
              f"tiles {cut[6]} max|drgb| {d.abs().max().item():.2e}")


def _expected_tiles(live, S, n_sm):
    """The three counters from the live counts: phase A groups per CTA (group g on CTA g % grid), a group deferred iff
    some sample is dead and fewer than 64 rows are live, the CTA's deferred rays packed whole, in order, into 128 rows."""
    R = 128 // S
    N = live.shape[0]
    ngroups = -(-N // R)
    grid = min(ngroups, n_sm)
    imm = dfr = packed = 0
    lists = [[] for _ in range(grid)]
    for g in range(ngroups):
        ls = live[g * R:(g + 1) * R].tolist()
        tot = sum(ls)
        if tot < len(ls) * S and 2 * tot < 128:
            dfr += 1
            lists[g % grid] += ls
        else:
            imm += 1
    for lst in lists:
        rows = 0
        for x in lst:
            if rows == 0 or rows + x > 128:
                packed += 1
                rows = 0
            rows += x
    return [imm, dfr, packed]


@pytest.mark.parametrize("S,n,t_stop", [(128, 1024, 1e-2), (32, 3000, 1e-3), (64, 777, 1e-4)])
def test_tile_counters_and_every_path(plane, S, n, t_stop):
    rays = plane.rays(n, seed=S)
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    for mode in MODES:
        for det in (False, True):
            out = plane.bwd(rays, S, mode, t_stop, det=det)
            want = _expected_tiles(out[5].cpu(), S, n_sm)
            assert out[6] == want, (mode, det, out[6], want)
    print(f"\n[tiles S={S} n={n} eps={t_stop}] {out[6]}")
    if S == 128:
        assert all(c > 0 for c in out[6]), out[6]


def test_packing_independence(plane):
    """FP32: a ray's rgb, depth and loss term do not depend on the rest of the batch."""
    S, n, t_stop = 64, 600, 1e-3
    rays = plane.rays(n, seed=3)
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(1)).to(DEV)
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(2)).to(DEV)
    for det in (False, True):
        base = plane.bwd(rays, S, lib.MLP_FP32, t_stop, det=det, grads={"rgb": torch.ones(n, 3, device=DEV)})
        permuted = plane.bwd(rays[perm].contiguous(), S, lib.MLP_FP32, t_stop, det=det, grads={"rgb": torch.ones(n, 3, device=DEV)})
        _same(permuted[2], base[2][perm], "rgb")
        _same(permuted[3], base[3][perm], "depth")
        _same(permuted[5], base[5][perm], "live")
        for lo, hi in ((0, 211), (211, n)):
            part = plane.bwd(rays[lo:hi].contiguous(), S, lib.MLP_FP32, t_stop, det=det,
                             grads={"rgb": torch.ones(hi - lo, 3, device=DEV)})
            _same(part[2], base[2][lo:hi], "rgb split")
            _same(part[3], base[3][lo:hi], "depth split")
    # each ray's loss term: the fused loss of a one-ray batch, normalised as a whole batch would be
    full = plane.bwd(rays, S, lib.MLP_FP32, t_stop, det=True, target_rgb=target, n_total=n, loss_out=torch.zeros(1, device=DEV))
    terms = ((full[2] - target) ** 2).sum(-1) / (3 * n)
    for i in (0, 17, 599):
        lo = torch.zeros(1, device=DEV)
        plane.bwd(rays[i:i + 1].contiguous(), S, lib.MLP_FP32, t_stop, det=True, target_rgb=target[i:i + 1], n_total=n,
                  loss_out=lo)
        assert abs(lo.item() - terms[i].item()) <= 1e-7 * max(terms[i].item(), 1e-30)


@pytest.mark.parametrize("grad_mode", MODES)
def test_deterministic_repeats_and_agrees_with_atomics(plane, grad_mode):
    S, n, t_stop = 128, 1023, 1e-3
    rays = plane.rays(n, seed=4)
    j = torch.rand(n, S, generator=torch.Generator().manual_seed(5)).to(DEV)
    atomic = plane.bwd(rays, S, grad_mode, t_stop, j, True)
    a = plane.bwd(rays, S, grad_mode, t_stop, j, True, det=True)
    b = plane.bwd(rays, S, grad_mode, t_stop, j, True, det=True)
    for x, y in zip(a[0], b[0]):
        _same(x, y, "mlp")
    for k in (1, 2, 3, 4, 5):
        _same(a[k], b[k], k)
    assert a[6] == b[6]
    for x, y in zip(atomic[0], a[0]):
        _same(x, y, "mlp vs atomic")
    e = (a[1] - atomic[1]).abs().max().item() / a[1].abs().max().item()
    assert e < 1.3e-7, e


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("grad_mode", MODES)
def test_frozen_volume_and_misaligned_rays(plane, grad_mode, det):
    S, n = 64, 300
    rays = plane.rays(n, seed=9)
    with_vol = plane.bwd(rays, S, grad_mode, 1e-3, det=det)
    frozen = plane.bwd(rays, S, grad_mode, 1e-3, det=det, want_volume_grad=False)
    assert frozen[1] is None
    for x, y in zip(with_vol[0], frozen[0]):
        _same(x, y, "mlp")
    _same(with_vol[2], frozen[2], "rgb")
    buf = torch.empty(n * 8 + 1, device=DEV)
    bad = buf[1:].view(n, 8)
    bad.copy_(rays)
    with pytest.raises(RuntimeError, match="aligned"):
        plane.bwd(bad, S, grad_mode, 1e-3)


def _train(ctx, steps, t_stop, grad_mode=lib.MLP_FP32, n=256, S=64, every=1):
    fn = backend.MVSNeRF().to(DEV)
    backend.load_weights_npz(fn, None, WPATH)
    volume = backend.RefVolume(ctx.vol.clone())
    tuner = backend.FineTuner(fn, volume, ctx.d.imgs_raw, ctx.d.pose_source, lr=5e-4, grad_mode=grad_mode)
    tgt_all = ctx.d.imgs_raw[0, 0].permute(1, 2, 0).reshape(-1, 3).contiguous()
    gen = torch.Generator(device=DEV).manual_seed(0)
    jgen = torch.Generator(device=DEV).manual_seed(1)
    losses = []
    for i in range(steps):
        idx = torch.randint(0, ctx.rays_all.shape[0], (n,), device=DEV, generator=gen)
        loss = tuner.step_rays(ctx.rays_all[idx], tgt_all[idx], ctx.sc.near_far, float(ctx.sc.pad), N_samples=S,
                               perturb=1.0, generator=jgen, t_stop=t_stop)[0]
        if i % every == 0:
            losses.append(loss.clone())
    return torch.cat(losses)


@pytest.mark.parametrize("grad_mode", MODES)
def test_step_rays_t_stop_zero_repeats_the_full_step(plane, grad_mode):
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        a = _train(plane, 50, None, grad_mode)
        b = _train(plane, 50, 0.0, grad_mode)
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)
    _same(a, b, "losses")


def test_step_rays_t_stop_tracks_the_full_step(plane):
    a = _train(plane, 500, None, every=50)
    b = _train(plane, 500, 1e-4, every=50)
    rel = ((a - b).abs() / a.abs()).max().item()
    print(f"\n[step_rays 1e-4 vs full, 500 steps] {a.tolist()} / {b.tolist()} ; max rel {rel:.3e}")
    assert rel < 1e-2
