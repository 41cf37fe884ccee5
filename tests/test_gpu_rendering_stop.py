"""GPU: early ray termination through the reference's call surface -- `rendering(..., t_stop=)` forward and under
autograd (mvsn_render_samples_stop, mvsn_render_backward_stop), `render_backward(..., t_stop=)` and
`FineTuner.step(..., t_stop=)`.

  * t_stop = 0 is bit-identical to the call without it (render: pair / split, fp32 / fp16 volume, ragged N, a partial
    last tile, white_bkgd, lindisp; step: both grad modes, both summation orders);
  * the bounds at t_stop = 1e-4 on whole 512x640 frames against the full samples render, and tiles_done falls where
    rays become opaque;
  * the samples entries agree bit for bit with the rays entries on host samples marched in the kernel's operation order;
  * the gradients are those of the per-ray truncated render (the oracle's autograd);
  * a training step written as the reference writes it (create_nerf_mvs with args.t_stop, ray_marcher,
    get_ndc_coordinate, rendering, img2mse, backward, Adam) gets render_backward's gradients;
  * 50 deterministic steps repeat bit for bit.
"""
import os
from types import SimpleNamespace

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
ULP = 4 * 2.0 ** -23


def img2mse(x, y):
    """utils.img2mse of the reference"""
    return torch.mean((x - y) ** 2)


@pytest.fixture
def deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn)


def _set_det(on):
    torch.use_deterministic_algorithms(on, warn_only=True)


def _net():
    fn = backend.MVSNeRF().to(DEV)
    backend.load_weights_npz(fn, None, WPATH)
    return fn


def _volume(sc):
    mvs = backend.MVSNet().to(DEV).train()
    fn = backend.MVSNeRF().to(DEV)
    backend.load_weights_npz(fn, mvs, WPATH)
    d = sc.to(DEV)
    with torch.no_grad():
        vol, _, _ = mvs(d.imgs_norm, d.proj_mats, sc.near_far, pad=sc.pad)
    return vol.detach().clone()


class Ctx:
    def __init__(self, sc):
        self.sc, self.d, self.vol, self.fn = sc, sc.to(DEV), _volume(sc), _net()
        self.rays_all = synthetic.scene_rays(sc).to(DEV).contiguous()

    def rays(self, n, seed):
        g = torch.Generator().manual_seed(seed)
        return self.rays_all[torch.randperm(self.rays_all.shape[0], generator=g)[:n].to(DEV)].contiguous()

    def march(self, rays, S, j=None, lindisp=False, kernel_order=True):
        """host samples (pts, ndc, z); kernel_order: the NDC in the kernel's operation order (no lindisp)"""
        pts, ndc, z = _host_march(self.sc, rays, S, j, lindisp)
        if kernel_order:
            ndc = _kernel_order_ndc(self.sc, pts)
        return pts, ndc, z

    def render(self, rays, smp, mode=lib.MLP_TC_SPLIT, vol=None, white=False, **kw):
        """rendering() as the reference calls it, forward only: (rgb, depth)"""
        pts, ndc, z = smp
        with torch.no_grad():
            out = backend.rendering(SimpleNamespace(), self.d.pose_source, pts, ndc, z, rays[:, :3], rays[:, 3:6],
                                    volume_feature=self.vol if vol is None else vol, imgs=self.d.imgs_raw,
                                    network_fn=self.fn, white_bkgd=white, mlp_mode=mode, **kw)
        if kw.get("t_stop") is not None:
            assert out[1] is None and out[2] is None and out[4] is None
        return out[0], out[3]

    def bwd(self, rays, smp, grad_mode, t_stop, det=False, white=False, **kw):
        """render_backward on host samples: (grad_mlp, grad_volume, rgb, depth, loss, live, tiles)"""
        pts, ndc, z = smp
        n = rays.shape[0]
        live = torch.full((n,), -1, dtype=torch.int32, device=DEV) if t_stop is not None else None
        tiles = torch.zeros(3, dtype=torch.int64, device=DEV) if t_stop is not None else None
        loss = torch.zeros(1, device=DEV)
        if "grads" not in kw:
            kw.setdefault("target_rgb", torch.rand(n, 3, generator=torch.Generator().manual_seed(n)).to(DEV))
            loss = kw.setdefault("loss_out", loss)
        was = torch.are_deterministic_algorithms_enabled()
        _set_det(det)
        try:
            stop = {} if t_stop is None else dict(t_stop=t_stop, live_samples=live, tiles_done=tiles)
            g, v, rgb, depth = backend.render_backward(self.d.pose_source, pts, ndc, z, rays[:, 3:6], self.vol,
                                                       self.d.imgs_raw, self.fn, white, want_forward=True,
                                                       grad_mode=grad_mode, **stop, **kw)
        finally:
            _set_det(was)
        return g, v, rgb, depth, loss, live, (tiles.tolist() if tiles is not None else None)

    def bwd_rays(self, rays, S, grad_mode, t_stop, j=None, det=False, white=False, **kw):
        n = rays.shape[0]
        live = torch.full((n,), -1, dtype=torch.int32, device=DEV)
        tiles = torch.zeros(3, dtype=torch.int64, device=DEV)
        loss = torch.zeros(1, device=DEV)
        if "grads" not in kw:
            kw.setdefault("target_rgb", torch.rand(n, 3, generator=torch.Generator().manual_seed(n)).to(DEV))
            loss = kw.setdefault("loss_out", loss)
        was = torch.are_deterministic_algorithms_enabled()
        _set_det(det)
        try:
            g, v, rgb, depth = backend.render_backward_rays(
                rays, self.vol, self.d.imgs_raw, self.d.pose_source, self.fn, self.sc.near_far, float(self.sc.pad),
                N_samples=S, jitter=j, white_bkgd=white, want_forward=True, grad_mode=grad_mode, t_stop=t_stop,
                live_samples=live, tiles_done=tiles, **kw)
        finally:
            _set_det(was)
        return g, v, rgb, depth, loss, live, tiles.tolist()


def _host_march(sc, rays, S, j, lindisp=False):
    """ray_marcher (data/ray_utils.py:152-197) with the uniform draw replaced by `j`, then get_ndc_coordinate, on the
    device: the points and depths the kernels march themselves, bit for bit."""
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
    """get_ndc_coordinate (no lindisp) in the kernels' operation order (ndc_of_point / project_view with IEEE
    divisions): fmaf chains, each fma formed exactly in float64 and rounded once to float32, then float32 divisions.
    The split render mode and the fp32 backward recompute use these divisions; the fp16 render modes use approximate
    ones, so host samples are not bit-equal to their in-kernel march."""
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
    near, far = (torch.tensor(float(x), dtype=torch.float32) for x in sc.near_far)
    nz = (q[2] - near) / f32(far.double() - near.double())
    if sc.pad > 0:
        hf, wf, pad = torch.tensor(sc.H / 4.0), torch.tensor(sc.W / 4.0), torch.tensor(float(sc.pad))
        dh, dw = hf + pad * 2, wf + pad * 2
        v = (v * hf) / dh + pad / dh
        u = (u * wf) / dw + pad / dw
    return torch.stack([u, v, nz], -1).reshape(pts.shape).contiguous().to(DEV)


def _same(a, b, what=""):
    assert a.dtype == b.dtype and torch.equal(a, b), (what, (a.float() - b.float()).abs().max().item())


@pytest.fixture(scope="module")
def plane():
    return Ctx(synthetic.make_plane_scene(96, 128, pad=4, seed=3))


# ---- 1. t_stop = 0 is bit-identical ------------------------------------------------------------------------------
@pytest.mark.parametrize("S,n,white,lindisp", [(128, 1000, False, False), (45, 777, True, False), (100, 37, False, True),
                                               (64, 1, True, True)])
def test_render_t_stop_zero_is_bit_identical(plane, S, n, white, lindisp):
    rays = plane.rays(n, seed=S + n)
    smp = plane.march(rays, S, lindisp=lindisp, kernel_order=False)
    for vol in (plane.vol, plane.vol.half()):
        for mode in (lib.MLP_TC_PAIR, lib.MLP_TC_SPLIT):
            rgb_a, depth_a = plane.render(rays, smp, mode, vol, white)
            tiles = torch.zeros(1, dtype=torch.int64, device=DEV)
            rgb_b, depth_b = plane.render(rays, smp, mode, vol, white, t_stop=0.0, tiles_done=tiles)
            _same(rgb_a, rgb_b, ("rgb", mode, vol.dtype))
            _same(depth_a, depth_b, ("depth", mode, vol.dtype))
            assert tiles.item() > 0


def _tuner(ctx, grad_mode):
    fn = _net()
    return backend.FineTuner(fn, backend.RefVolume(ctx.vol.clone()), ctx.d.imgs_raw, ctx.d.pose_source, lr=5e-4,
                             grad_mode=grad_mode)


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("grad_mode", MODES)
def test_step_t_stop_zero_is_bit_identical(plane, grad_mode, det):
    n, S = 300, 64
    rays = plane.rays(n, seed=1)
    smp = plane.march(rays, S, j=torch.rand(n, S, generator=torch.Generator().manual_seed(2)).to(DEV))
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(3)).to(DEV)
    was = torch.are_deterministic_algorithms_enabled()
    _set_det(det)
    try:
        a, b = _tuner(plane, grad_mode), _tuner(plane, grad_mode)
        la = a.step(*smp[:3], rays[:, 3:6], target)[0].clone()
        lb = b.step(*smp[:3], rays[:, 3:6], target, t_stop=0.0)[0].clone()
    finally:
        _set_det(was)
    for x, y in zip(a.g, b.g):
        _same(x, y, "mlp grad")
    for x, y in zip(a.params, b.params):
        _same(x.detach(), y.detach(), "mlp after Adam")
    if det:                                         # the float atomics of the loss and the volume are not reproducible
        _same(la, lb, "loss")
        _same(a.volume.feat_volume.detach(), b.volume.feat_volume.detach(), "volume after Adam")
    else:
        assert abs(la.item() - lb.item()) <= 1e-6 * la.item()
    # the volume gradient itself, through render_backward
    full = plane.bwd(rays, smp, grad_mode, None, det=det, target_rgb=target)
    zero = plane.bwd(rays, smp, grad_mode, 0.0, det=det, target_rgb=target)
    assert torch.all(zero[5] == S) and zero[6] == [-(-n // (128 // S)), 0, 0]
    _same(full[2], zero[2], "rgb")
    _same(full[3], zero[3], "depth")
    if det:
        _same(full[1], zero[1], "volume grad")
    else:
        assert (full[1] - zero[1]).abs().max().item() <= 1e-6 * full[1].abs().max().item()


# ---- 2. the bounds on whole frames ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["plane", "bench"])
def test_bounds_on_512x640_frames(name):
    make = synthetic.make_plane_scene if name == "plane" else synthetic.make_scene
    ctx = Ctx(make(512, 640, seed=0))
    S, chunk, t_stop = 128, 32768, 1e-4
    rays = ctx.rays_all
    far = float(rays[:, 7].max())
    for mode in (lib.MLP_TC_PAIR, lib.MLP_TC_SPLIT):
        tiles = torch.zeros(1, dtype=torch.int64, device=DEV)
        all_tiles = 0
        worst = 0.0
        for i in range(0, rays.shape[0], chunk):
            r = rays[i:i + chunk]
            xyz, _, _, z = backend.ray_marcher(r, N_samples=S)
            smp = (xyz, _host_march(ctx.sc, r, S, None)[1], z)
            rgb_f, depth_f = ctx.render(r, smp, mode)
            rgb_c, depth_c = ctx.render(r, smp, mode, t_stop=t_stop, tiles_done=tiles)
            d = rgb_c - rgb_f
            assert d.max().item() <= ULP and d.min().item() > -t_stop - ULP, (mode, d.min().item(), d.max().item())
            dd = depth_f - depth_c
            assert dd.min().item() >= -ULP * far and dd.max().item() < (t_stop + ULP) * far
            worst = max(worst, d.abs().max().item())
            all_tiles += -(-r.shape[0] // 32) * (S // 2)                            # 32 rays x 2 samples per tile
        frac = tiles.item() / all_tiles
        print(f"\n[{name} {mode} t_stop={t_stop}] tiles {frac:.3f} max|drgb| {worst:.2e}")
        if name == "plane":
            assert frac < 0.8, frac


# ---- 3. samples entries == rays entries -------------------------------------------------------------------------
@pytest.mark.parametrize("t_stop", [1e-4, 1e-2])
@pytest.mark.parametrize("S,n", [(128, 3000), (48, 777)])
def test_rendering_equals_render_rays(plane, S, n, t_stop):
    """Split mode (IEEE divisions in the in-kernel NDC, so host samples in the kernel's order are the kernel's own)."""
    rays = plane.rays(n, seed=n)
    smp = plane.march(rays, S)
    for vol in (plane.vol, plane.vol.half()):
        ta, tb = torch.zeros(1, dtype=torch.int64, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)
        rgb_s, depth_s = plane.render(rays, smp, lib.MLP_TC_SPLIT, vol, t_stop=t_stop, tiles_done=ta)
        with torch.no_grad():
            rgb_r, depth_r = backend.render_rays(rays, vol, plane.d.imgs_raw, plane.d.pose_source, plane.fn,
                                                 plane.sc.near_far, float(plane.sc.pad), N_samples=S,
                                                 mlp_mode=lib.MLP_TC_SPLIT, t_stop=t_stop, tiles_done=tb)
        _same(rgb_s, rgb_r, "rgb")
        _same(depth_s, depth_r, "depth")
        assert ta.item() == tb.item()


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("grad_mode", MODES)
def test_step_equals_step_rays(plane, grad_mode, det):
    n, S, t_stop = 600, 128, 1e-3
    rays = plane.rays(n, seed=5)
    j = torch.rand(n, S, generator=torch.Generator().manual_seed(6)).to(DEV)
    smp = plane.march(rays, S, j)
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(7)).to(DEV)
    s = plane.bwd(rays, smp, grad_mode, t_stop, det=det, target_rgb=target)
    r = plane.bwd_rays(rays, S, grad_mode, t_stop, j, det=det, target_rgb=target)
    for x, y in zip(s[0], r[0]):
        _same(x, y, "mlp grad")
    for k, what in ((2, "rgb"), (3, "depth"), (5, "live")):
        _same(s[k], r[k], what)
    assert s[6] == r[6] and (s[5] < S).any()
    if det:
        _same(s[1], r[1], "volume grad")
        _same(s[4], r[4], "loss")
    else:                                           # float atomics: the order of the sums differs from run to run
        assert (s[1] - r[1]).abs().max().item() <= 1e-6 * r[1].abs().max().item()
        assert abs(s[4].item() - r[4].item()) <= 1e-6 * r[4].item()
    # FineTuner: one step each from the same start; step_rays draws its jitter from the generator, step gets the same
    # draw marched on the host
    jr = torch.rand((n, S), device=DEV, generator=torch.Generator(device=DEV).manual_seed(11))
    smp_r = plane.march(rays, S, jr)
    was = torch.are_deterministic_algorithms_enabled()
    _set_det(det)
    try:
        a, b = _tuner(plane, grad_mode), _tuner(plane, grad_mode)
        la = a.step(*smp_r, rays[:, 3:6], target, t_stop=t_stop)[0].clone()
        lb = b.step_rays(rays, target, plane.sc.near_far, float(plane.sc.pad), N_samples=S, perturb=1.0,
                         generator=torch.Generator(device=DEV).manual_seed(11), t_stop=t_stop)[0].clone()
    finally:
        _set_det(was)
    for x, y in zip(a.g, b.g):
        _same(x, y, "step mlp grad")
    if det:
        _same(la, lb, "step loss")
        _same(a.volume.feat_volume.detach(), b.volume.feat_volume.detach(), "volume after Adam")
    else:
        assert abs(la.item() - lb.item()) <= 1e-6 * lb.item()


# ---- 4. gradients of the truncated render -------------------------------------------------------------------------
def _truncated_render(pts, ndc, z, rays_d, vol, imgs_raw, pose, w, live, white):
    """orc.render_samples with w_j = 0 for j >= live (the function the stop entries differentiate)"""
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
def test_gradients_of_the_truncated_render(plane, weights, grad_mode, S, n, white):
    sc = plane.sc
    rays = plane.rays(n, seed=7)
    smp = plane.march(rays, S, torch.rand(n, S, generator=torch.Generator().manual_seed(5)).to(DEV))
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(n)).to(DEV)
    g_k, v_k, rgb_k, depth_k, loss_k, live, _ = plane.bwd(rays, smp, grad_mode, 1e-3, white=white, target_rgb=target)
    assert (live < S).any()
    wt = {k: v.clone().requires_grad_(k.startswith("mlp/")) for k, v in weights.items()}
    vt = plane.vol.detach().cpu().clone().requires_grad_(True)
    rgb, depth = _truncated_render(smp[0].cpu(), smp[1].cpu(), smp[2].cpu(), rays[:, 3:6].cpu(), vt, sc.imgs_raw,
                                   sc.pose_source, wt, live.long().cpu(), white)
    loss = ((rgb - target.cpu()) ** 2).mean()
    loss.backward()
    assert (rgb_k.cpu() - rgb).abs().max().item() < 1e-5 and (depth_k.cpu() - depth).abs().max().item() < 1e-4
    assert abs(loss_k.item() - loss.item()) <= 1e-5 * loss.item()
    pairs = [(g.cpu(), wt["mlp/" + name].grad) for (name, _), g in zip(backend._ordered_named_params(plane.fn), g_k)]
    pairs.append((v_k.permute(3, 0, 1, 2).unsqueeze(0).cpu(), vt.grad))
    excess = max((a - b).abs().max().item() - GATE[grad_mode] * b.abs().max().item() - 1e-8 for a, b in pairs)
    assert excess <= 0, excess


# ---- 5. the reference's own training step -------------------------------------------------------------------------
def _reference_args(t_stop):
    return SimpleNamespace(multires=10, i_embed=0, pts_dim=3, multires_views=4, dir_dim=3, netdepth=6, netwidth=128,
                           feat_dim=20, net_type="v0", N_importance=0, netchunk=1024, ckpt=None, perturb=1.0,
                           N_samples=64, use_viewdirs=True, white_bkgd=True, raw_noise_std=0.0, use_color_volume=False,
                           t_stop=t_stop)


@pytest.mark.parametrize("grad_mode", MODES)
def test_reference_training_step(plane, deterministic, grad_mode):
    """train_mvs_nerf_finetuning_pl.py's training_step: create_nerf_mvs(args) with args.t_stop, ray_marcher,
    get_ndc_coordinate, rendering(**render_kwargs_train), img2mse, backward(), Adam -- the gradients are
    render_backward(..., t_stop=args.t_stop)'s on the same batch and cotangent."""
    args = _reference_args(1e-4)
    kw_train, kw_test, _, grad_vars = backend.create_nerf_mvs(args, dir_embedder=False, pts_embedder=True)
    assert kw_train["t_stop"] == kw_test["t_stop"] == 1e-4
    fn = kw_train["network_fn"]
    backend.load_weights_npz(fn, None, WPATH)
    volume = backend.RefVolume(plane.vol.clone())
    optimizer = torch.optim.Adam(grad_vars + [volume.feat_volume], lr=5e-4)
    sc, d = plane.sc, plane.d
    rays = plane.rays(512, seed=9)
    target = d.imgs_raw[0, 0].permute(1, 2, 0).reshape(-1, 3)[:512].contiguous()
    torch.manual_seed(0)
    xyz, rays_o, rays_d, z_vals = backend.ray_marcher(rays, N_samples=args.N_samples, lindisp=False,
                                                      perturb=kw_train["perturb"])
    inv_scale = torch.tensor([sc.W - 1.0, sc.H - 1.0], device=DEV)
    ndc = backend.get_ndc_coordinate(d.pose_source["w2cs"][0], d.pose_source["intrinsics"][0], xyz, inv_scale,
                                     near=sc.near_far[0], far=sc.near_far[1], pad=sc.pad)
    extra = {} if grad_mode == lib.MLP_FP32 else {"grad_mode": grad_mode}
    rgbs, feat, weights, depth, alpha, _ = backend.rendering(args, d.pose_source, xyz, ndc, z_vals, rays_o, rays_d,
                                                             volume, d.imgs_raw, img_feat=None, **kw_train, **extra)
    assert feat is None and weights is None and alpha is None
    cot = {}
    rgbs.register_hook(lambda g: cot.setdefault("rgb", g.clone()))
    loss = img2mse(rgbs, target)
    optimizer.zero_grad()
    loss.backward()
    g_ref, v_ref, _, _ = backend.render_backward(d.pose_source, xyz, ndc, z_vals, rays_d, volume, d.imgs_raw, fn, True,
                                                 grads={"rgb": cot["rgb"], "depth": torch.zeros(512, device=DEV)},
                                                 grad_mode=grad_mode, t_stop=1e-4)
    for p, g in zip(fn.ordered_params(), g_ref):
        _same(p.grad, g, "mlp grad")
    _same(volume.feat_volume.grad, v_ref.permute(3, 0, 1, 2).unsqueeze(0), "volume grad")
    before = [p.detach().clone() for p in grad_vars]
    optimizer.step()
    assert any(not torch.equal(a, p.detach()) for a, p in zip(before, grad_vars))
    # a per-sample cotangent is refused: dead samples have none
    with pytest.raises(RuntimeError, match="per-sample"):
        backend.render_backward(d.pose_source, xyz, ndc, z_vals, rays_d, volume, d.imgs_raw, fn, True,
                                grads={"rgb": cot["rgb"], "weights": torch.ones(512, args.N_samples, device=DEV)},
                                t_stop=1e-4)


# ---- 6. determinism ---------------------------------------------------------------------------------------------
def test_fifty_deterministic_steps_repeat(plane, deterministic):
    def run():
        tuner = _tuner(plane, lib.MLP_FP32)
        tgt_all = plane.d.imgs_raw[0, 0].permute(1, 2, 0).reshape(-1, 3).contiguous()
        gen = torch.Generator(device=DEV).manual_seed(0)
        torch.manual_seed(1)
        losses = []
        for _ in range(50):
            idx = torch.randint(0, plane.rays_all.shape[0], (256,), device=DEV, generator=gen)
            rays = plane.rays_all[idx]
            xyz, _, rays_d, z = backend.ray_marcher(rays, N_samples=64, perturb=1.0)
            ndc = backend.get_ndc_coordinate(plane.d.pose_source["w2cs"][0], plane.d.pose_source["intrinsics"][0], xyz,
                                             torch.tensor([plane.sc.W - 1.0, plane.sc.H - 1.0], device=DEV),
                                             near=plane.sc.near_far[0], far=plane.sc.near_far[1], pad=plane.sc.pad)
            losses.append(tuner.step(xyz, ndc, z, rays_d, tgt_all[idx], t_stop=1e-4)[0].clone())
        return tuner, torch.cat(losses)

    a, la = run()
    b, lb = run()
    _same(la, lb, "losses")
    for x, y in zip(a.params + [a.volume.feat_volume], b.params + [b.volume.feat_volume]):
        _same(x.detach(), y.detach(), "parameters")
