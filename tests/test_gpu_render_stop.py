"""GPU: early ray termination (render_rays(..., t_stop=eps), mvsn_render_rays_stop) in the tensor-core modes.

  * eps = 0 is bit-identical to render_rays without the option, and computes every tile;
  * the signed per-pixel bounds of the omitted tail hold on whole 512x640 frames of the bench scene and of a scene whose
    rays do become opaque (synthetic.make_plane_scene), where most tiles are skipped;
  * exact prefix: the stop tile of every group follows from the alpha the full render reports, and each pixel equals
    the full render of its first (computed tiles x samples per tile) samples.  The prefix is rendered through the same
    ray entry with a prefix of t_steps rather than through render_samples with host-marched samples: the fp16 modes'
    in-kernel NDC uses approximate divisions, so host-marched samples are not bit-equal to the ray path in those
    modes, while a t_steps prefix runs the identical front end in every mode;
  * many groups per CTA at few rays per group and an odd group count, so the shared-counter hand-out and the idle
    consumer's passes run;
  * determinism, and the rejected arguments.
"""
import ctypes as C
import os

import pytest
import torch

from conftest import GOLDEN
from mvsnerf_b200 import backend, lib, synthetic

pytestmark = pytest.mark.gpu
DEV = "cuda"
MODES = [lib.MLP_TC_PAIR, lib.MLP_TC_HALF, lib.MLP_TC_SPLIT]
EPS = [1e-4, 1e-3, 1e-2]


def _net():
    fn, mvs = backend.MVSNeRF().to(DEV), backend.MVSNet().to(DEV).train()
    backend.load_weights_npz(fn, mvs, os.path.join(GOLDEN, "mvsnerf_v0_weights.npz"))
    return fn, mvs


class Ctx:
    def __init__(self, sc, fn, mvs):
        self.sc, self.fn, self.d = sc, fn, sc.to(DEV)
        with torch.no_grad():
            self.vol, _, _ = mvs(self.d.imgs_norm, self.d.proj_mats, sc.near_far, pad=sc.pad)
        self.rays = synthetic.scene_rays(sc).to(DEV).contiguous()

    def render(self, rays, mode, S=128, white=False, lindisp=False, **kw):
        with torch.no_grad():
            return backend.render_rays(rays, self.vol, self.d.imgs_raw, self.d.pose_source, self.fn, self.sc.near_far,
                                       float(self.sc.pad), N_samples=S, white_bkgd=white, lindisp=lindisp, mlp_mode=mode,
                                       **kw)

    def stop(self, rays, mode, eps, **kw):
        tiles = torch.zeros(1, dtype=torch.int64, device=DEV)
        rgb, depth = self.render(rays, mode, t_stop=eps, tiles_done=tiles, **kw)
        return rgb, depth, int(tiles.item())

    def raw(self, rays, mode, t_steps, white=False, alpha=None):
        """mvsn_render_rays with explicit t_steps (any prefix of linspace(0, 1, S)) and an optional alpha output."""
        L = lib.load()
        sc, keep = backend._make_scene(self.d.pose_source, self.vol, self.d.imgs_raw, self.fn, white, mode)
        rp = lib.RayParams(float(self.sc.near_far[0]), float(self.sc.near_far[1]), float(self.sc.pad), 0)
        n, s = rays.shape[0], t_steps.shape[0]
        rgb = torch.empty(n, 3, device=DEV)
        depth = torch.empty(n, device=DEV)
        lib.check(L.mvsn_render_rays(C.byref(sc), C.byref(rp), lib.ptr(rays), lib.ptr(t_steps), n, s, lib.ptr(rgb),
                                     lib.ptr(depth), None, lib.ptr(alpha), None, lib.stream_ptr()), "mvsn_render_rays")
        torch.cuda.synchronize()
        del keep
        return rgb, depth


def _rays_per_tile(n):
    """the launcher's rule: 32 unless the batch gives fewer than two groups per SM"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rt = 32
    while rt > 4 and (n + rt - 1) // rt < 2 * sms:
        rt //= 2
    return rt


def _all_tiles(n, S):
    rt = _rays_per_tile(n)
    sp = 64 // rt
    return ((n + rt - 1) // rt) * ((S + sp - 1) // sp)


@pytest.fixture(scope="module")
def net():
    return _net()


@pytest.fixture(scope="module")
def small(net):
    return Ctx(synthetic.make_scene(96, 128, pad=4, seed=5), *net)


@pytest.fixture(scope="module")
def bench_scene(net):
    return Ctx(synthetic.make_scene(512, 640, seed=0), *net)


@pytest.fixture(scope="module")
def plane_scene(net):
    return Ctx(synthetic.make_plane_scene(512, 640, seed=0), *net)


@pytest.mark.parametrize("S", [1, 24, 128, 192, 256])
@pytest.mark.parametrize("mode", MODES)
def test_eps0_is_bit_identical(small, mode, S):
    """ragged N at 32 rays per group, and N small enough for fewer rays per group; lindisp and white_bkgd"""
    for n, white, lindisp in ((8461, False, False), (8461, True, True), (300, True, False), (37, False, True)):
        rays = small.rays[:n].contiguous()
        rgb0, depth0 = small.render(rays, mode, S, white, lindisp)
        rgb, depth, tiles = small.stop(rays, mode, 0.0, S=S, white=white, lindisp=lindisp)
        assert torch.equal(rgb, rgb0), (n, white, lindisp, (rgb - rgb0).abs().max().item())
        assert torch.equal(depth, depth0), (n, white, lindisp)
        assert tiles == _all_tiles(n, S)


def _check_bounds(ctx, mode, white, eps_list, max_fraction=None):
    rgb0, depth0 = ctx.render(ctx.rays, mode, white=white)
    zmax = float(ctx.rays[:, 7].max())
    fractions = {}
    for eps in eps_list:
        rgb, depth, tiles = ctx.stop(ctx.rays, mode, eps, white=white)
        d = rgb - rgb0
        ulp = 4e-7                                              # a few ulps of the final fp32 additions
        if white:
            assert d.min().item() >= -ulp and d.max().item() < eps + ulp, (eps, d.min().item(), d.max().item())
        else:
            assert d.min().item() > -eps - ulp and d.max().item() <= ulp, (eps, d.min().item(), d.max().item())
        dd = depth0 - depth
        assert dd.min().item() >= -4 * ulp * zmax and dd.max().item() < eps * zmax + 4 * ulp * zmax, (eps, dd.min(), dd.max())
        fractions[eps] = tiles / _all_tiles(ctx.rays.shape[0], 128)
    return fractions


@pytest.mark.parametrize("white", [False, True])
@pytest.mark.parametrize("mode", MODES)
def test_bounds_bench_scene(bench_scene, mode, white):
    f = _check_bounds(bench_scene, mode, white, EPS)
    assert all(0 < v <= 1 for v in f.values())


@pytest.mark.parametrize("white", [False, True])
@pytest.mark.parametrize("mode", MODES)
def test_bounds_plane_scene_and_tiles_skipped(plane_scene, mode, white):
    f = _check_bounds(plane_scene, mode, white, EPS)
    assert f[1e-4] < 0.70, f
    assert f[1e-2] <= f[1e-3] <= f[1e-4], f


@pytest.mark.parametrize("white", [False, True])
@pytest.mark.parametrize("mode", MODES)
def test_exact_prefix(plane_scene, mode, white):
    """Every group's stop tile follows from the full render's alpha (the kernel's transmittance recurrence, replayed in
    fp32; a verdict after tile k leaves tiles k + 1 and k + 2 to compute); each pixel is bit-identical to the full
    render of its first samples, computed through the same ray entry with a prefix of t_steps (so the front end is the
    same in every mode)."""
    ctx, S, eps = plane_scene, 128, 1e-3
    n = 32 * 640                                               # 32 image rows through the plane, 32 rays per group
    rays = ctx.rays[200 * 640:200 * 640 + n].contiguous()
    rt = _rays_per_tile(n)
    assert rt == 32
    sp, nt = 64 // rt, (S + 64 // rt - 1) // (64 // rt)
    t_steps = backend._tsteps_of(S, torch.device(DEV))
    alpha = torch.empty(n, S, device=DEV)
    ctx.raw(rays, mode, t_steps, white, alpha=alpha)
    T = torch.ones(n, device=DEV)
    stopped = torch.zeros(n // rt, dtype=torch.bool, device=DEV)
    tiles = torch.full((n // rt,), nt, dtype=torch.int64, device=DEV)
    for k in range(nt):
        for s in range(k * sp, min((k + 1) * sp, S)):
            T = T * ((1.0 - alpha[:, s]) + 1e-10)
        verdict = (T < eps).view(-1, rt).all(1) & ~stopped
        tiles[verdict] = min(k + 3, nt)
        stopped |= verdict
    rgb, depth, done = ctx.stop(rays, mode, eps, white=white)
    assert done == int(tiles.sum().item())
    assert done < 0.8 * nt * (n // rt), "the band must stop early for this test to mean anything"
    per_ray = tiles.repeat_interleave(rt)
    for L in per_ray.unique().tolist():
        sel = (per_ray == L).nonzero().squeeze(1)
        s_l = min(L * sp, S)
        rgb_p, depth_p = ctx.raw(rays[sel].contiguous(), mode, t_steps[:s_l].contiguous(), white)
        assert torch.equal(rgb[sel], rgb_p), (L, (rgb[sel] - rgb_p).abs().max().item())
        assert torch.equal(depth[sel], depth_p), L


@pytest.mark.parametrize("mode", MODES)
def test_deterministic_and_split_invariant(plane_scene, mode):
    ctx, eps = plane_scene, 1e-3
    rgb1, depth1, t1 = ctx.stop(ctx.rays, mode, eps)
    rgb2, depth2, t2 = ctx.stop(ctx.rays, mode, eps)
    assert torch.equal(rgb1, rgb2) and torch.equal(depth1, depth2) and t1 == t2
    cut = 32 * 4000                                            # both parts keep 32 rays per group
    a = ctx.stop(ctx.rays[:cut].contiguous(), mode, eps)
    b = ctx.stop(ctx.rays[cut:].contiguous(), mode, eps)
    assert torch.equal(torch.cat([a[0], b[0]]), rgb1) and torch.equal(torch.cat([a[1], b[1]]), depth1)
    assert a[2] + b[2] == t1


@pytest.mark.parametrize("mode", MODES)
def test_many_groups_per_cta(small, mode):
    """1994 rays at 128 samples: 4 rays per group (16 samples per tile, 8 tiles), 499 groups, so most CTAs hand out
    four groups through the shared counter and one CTA three, whose second consumer runs idle passes while the first
    works.  t_stop = 2 (> any transmittance) stops every group after its first tile (three tiles computed),
    t_stop = 0.5 some of them."""
    n = 1994
    rays = torch.cat([small.rays, small.rays])[:n].contiguous()
    assert _rays_per_tile(n) == 4
    rgb0, depth0 = small.render(rays, mode)
    rgb, depth, tiles = small.stop(rays, mode, 0.0)
    assert torch.equal(rgb, rgb0) and torch.equal(depth, depth0) and tiles == _all_tiles(n, 128)
    rgb, depth, tiles = small.stop(rays, mode, 2.0)
    assert tiles == 3 * ((n + 3) // 4)
    rgb_p, depth_p = small.raw(rays, mode, backend._tsteps_of(128, torch.device(DEV))[:48].contiguous())
    assert torch.equal(rgb, rgb_p) and torch.equal(depth, depth_p)
    rgb, depth, tiles = small.stop(rays, mode, 0.5)
    assert 3 * ((n + 3) // 4) <= tiles <= _all_tiles(n, 128)
    d = rgb - rgb0
    assert d.min().item() > -0.5 - 4e-7 and d.max().item() <= 4e-7
    again = small.stop(rays, mode, 0.5)
    assert torch.equal(again[0], rgb) and torch.equal(again[1], depth) and again[2] == tiles


def test_rejections(small):
    rays = small.rays[:64].contiguous()
    with pytest.raises(RuntimeError, match="tensor-core"):
        small.render(rays, lib.MLP_FP32, t_stop=1e-4)
    with pytest.raises(RuntimeError, match="sink"):
        small.render(rays, lib.MLP_TC_SPLIT, t_stop=1e-4, sink=lib.PeerSink())
    with pytest.raises(RuntimeError, match="CUDA"):
        small.render(rays.cpu(), lib.MLP_TC_SPLIT, t_stop=1e-4)
    with pytest.raises(RuntimeError, match="t_stop"):
        small.render(rays, lib.MLP_TC_PAIR, t_stop=-1.0)
    with pytest.raises(RuntimeError, match="tiles_done"):
        small.render(rays, lib.MLP_TC_PAIR, t_stop=1e-4, tiles_done=torch.zeros(1, dtype=torch.int64))


def test_render_video_passes_t_stop(small):
    from mvsnerf_b200 import scene_io
    c2ws = synthetic.spiral_path(small.sc, n_frames=2).to(DEV)
    dirs = small.d.directions
    args = (dirs, small.vol, small.d.imgs_raw, small.d.pose_source, small.fn, small.sc.near_far, float(small.sc.pad))
    with torch.no_grad():
        full = scene_io.render_video(c2ws, *args, mlp_mode=lib.MLP_TC_PAIR)
        same = scene_io.render_video(c2ws, *args, mlp_mode=lib.MLP_TC_PAIR, t_stop=0.0)
    for (a, b), (c, d) in zip(full, same):
        assert torch.equal(a, c) and torch.equal(b, d)
