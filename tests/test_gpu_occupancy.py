"""GPU: empty-space skipping (build_occupancy, render_rays(..., occupancy=), mvsn_render_rays_occ).

  * an all-ones grid is bit-identical to render_rays(t_stop=eps) (eps in {0, 1e-4}), pair and split, fp32 and fp16
    volumes, ragged N, S of 24 and 200, lindisp and white_bkgd, with the same tile counts;
  * an all-zeros grid gives rgb 0 (1 with white_bkgd), depth 0 and no tile, on rays whose samples all lie in the volume;
  * the grid bits against the oracle's sigma at the nodes (only nodes whose pre-ReLU sigma is within rounding of 0 may
    differ), the dilation against the host restatement, and an fp16 volume against its fp32 upcast;
  * the kernel's group ranges against a host recomputation (only samples within 1e-5 of a cell face may differ), and
    the tile count they imply;
  * on the plane scene at 512x640: every pixel within the bound of the skipped samples, computed from the full render's
    alpha, and bit-identity on every pixel whose skipped samples all have alpha == 0;
  * determinism, invariance to splitting the batch at a group boundary, the cache and render_video.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from mvsnerf_b200 import backend, lib, synthetic
from oracle import mvsnerf_oracle as orc
import occupancy_host as oh

pytestmark = pytest.mark.gpu
DEV = "cuda"
PAIR, SPLIT = lib.MLP_TC_PAIR, lib.MLP_TC_SPLIT


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

    def occ(self, dilate=1, vol=None, lindisp=False):
        return backend.build_occupancy(self.vol if vol is None else vol, self.d.imgs_raw, self.d.pose_source, self.fn,
                                       self.sc.near_far, float(self.sc.pad), lindisp=lindisp, dilate=dilate)

    def render(self, rays, mode, S=128, white=False, lindisp=False, vol=None, **kw):
        with torch.no_grad():
            return backend.render_rays(rays, self.vol if vol is None else vol, self.d.imgs_raw, self.d.pose_source,
                                       self.fn, self.sc.near_far, float(self.sc.pad), N_samples=S, white_bkgd=white,
                                       lindisp=lindisp, mlp_mode=mode, **kw)

    def counted(self, rays, mode, **kw):
        tiles = torch.zeros(1, dtype=torch.int64, device=DEV)
        rgb, depth = self.render(rays, mode, tiles_done=tiles, **kw)
        return rgb, depth, int(tiles.item())

    def alpha(self, rays, mode, S=128, lindisp=False):
        """the full render's alpha [N,S] (mvsn_render_rays with the alpha output)"""
        L = lib.load()
        sc, keep = backend._make_scene(self.d.pose_source, self.vol, self.d.imgs_raw, self.fn, False, mode)
        rp = lib.RayParams(float(self.sc.near_far[0]), float(self.sc.near_far[1]), float(self.sc.pad), int(lindisp))
        n = rays.shape[0]
        rgb, depth, alpha = torch.empty(n, 3, device=DEV), torch.empty(n, device=DEV), torch.empty(n, S, device=DEV)
        lib.check(L.mvsn_render_rays(C.byref(sc), C.byref(rp), lib.ptr(rays), lib.ptr(backend._tsteps_of(S, rays.device)),
                                     n, S, lib.ptr(rgb), lib.ptr(depth), None, lib.ptr(alpha), None, lib.stream_ptr()),
                  "mvsn_render_rays")
        torch.cuda.synchronize()
        del keep
        return alpha


def _filled(occ, value):
    return backend.Occupancy(torch.full_like(occ.bits, value), occ.D, occ.Hp, occ.Wp, occ.near_far, occ.pad, occ.lindisp,
                             occ.dilate)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _kernel_ranges(n):
    """the range table the last render_rays(occupancy=) call left in its workspace"""
    rt = oh.rays_per_tile(n, _sms())
    G = (n + rt - 1) // rt
    ws = backend._occ_workspace[torch.device(DEV, torch.cuda.current_device())]
    return ws[:G * 8].view(torch.int32).view(G, 2).cpu().numpy().astype(np.int64), rt


@pytest.fixture(scope="module")
def net():
    return _net()


@pytest.fixture(scope="module")
def small(net):
    return Ctx(synthetic.make_scene(96, 128, pad=4, seed=5), *net)


@pytest.fixture(scope="module")
def plane(net):
    return Ctx(synthetic.make_plane_scene(512, 640, seed=0), *net)


# ---- the grid is a no-op when full, and skips everything when empty -------------------------------------------
@pytest.mark.parametrize("half", [False, True])
@pytest.mark.parametrize("mode", [PAIR, SPLIT])
def test_all_ones_grid_is_stop(small, mode, half):
    vol = small.vol.half() if half else small.vol
    for lindisp in (False, True):
        ones = _filled(small.occ(lindisp=lindisp), -1)
        for S in (24, 200):
            for n, white in ((8461, False), (300, True), (37, False)):
                rays = small.rays[:n].contiguous()
                for eps in (0.0, 1e-4):
                    a = small.counted(rays, mode, S=S, white=white, lindisp=lindisp, vol=vol, t_stop=eps)
                    b = small.counted(rays, mode, S=S, white=white, lindisp=lindisp, vol=vol, t_stop=eps, occupancy=ones)
                    key = (lindisp, S, n, white, eps)
                    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), key
                    assert a[2] == b[2], key
            if not half and not lindisp:                      # without t_stop: the existing entry, bit for bit
                rgb0, depth0 = small.render(small.rays, mode, S=S)
                rgb, depth = small.render(small.rays, mode, S=S, occupancy=ones)
                assert torch.equal(rgb, rgb0) and torch.equal(depth, depth0)


@pytest.mark.parametrize("mode", [PAIR, SPLIT])
def test_all_zeros_grid(small, mode):
    """rays through the middle of the frame, marched between near + 0.02 and far - 0.02 of the volume's depth range, so
    every sample lies inside [0,1]^3 and none is occupied"""
    H, W = small.sc.H, small.sc.W
    idx = torch.arange(H * W, device=DEV).view(H, W)[H // 2 - 12:H // 2 + 12, W // 2 - 16:W // 2 + 16].reshape(-1)
    rays = small.rays[idx].clone()
    rays[:, 6] += 0.02
    rays[:, 7] -= 0.02
    rays = rays.contiguous()
    xyz, _, _, _ = backend.ray_marcher(rays, N_samples=128)
    ndc = backend.get_ndc_coordinate(small.d.pose_source["w2cs"][0], small.d.pose_source["intrinsics"][0], xyz,
                                     torch.tensor([W - 1.0, H - 1.0], device=DEV), near=small.sc.near_far[0],
                                     far=small.sc.near_far[1], pad=small.sc.pad)
    assert ndc.min() > 1e-3 and ndc.max() < 1 - 1e-3
    zeros = _filled(small.occ(), 0)
    for white in (False, True):
        for eps in (None, 1e-4):
            rgb, depth, tiles = small.counted(rays, mode, white=white, t_stop=eps, occupancy=zeros)
            assert tiles == 0
            assert torch.equal(rgb, torch.full_like(rgb, 1.0 if white else 0.0)) and torch.equal(depth, torch.zeros_like(depth))


# ---- the grid ---------------------------------------------------------------------------------------------------
def _node_samples(ctx, D, Hp, Wp, lindisp=False):
    """the nodes' NDC (fp32, as the kernel forms it) and world points (fp64 inversion of get_ndc_coordinate)"""
    d, y, x = torch.meshgrid(torch.arange(D), torch.arange(Hp), torch.arange(Wp), indexing="ij")
    ndc = torch.stack([x.float() / (Wp - 1), y.float() / (Hp - 1), d.float() / (D - 1)], -1).reshape(-1, 3)
    u, v, nz = ndc[:, 0].double(), ndc[:, 1].double(), ndc[:, 2].double()
    H, W, pad = ctx.sc.H, ctx.sc.W, float(ctx.sc.pad)
    if pad > 0:
        wf, hf = np.float32(W) / np.float32(4.0), np.float32(H) / np.float32(4.0)
        u = (u * (float(wf) + 2 * pad) - pad) / float(wf)
        v = (v * (float(hf) + 2 * pad) - pad) / float(hf)
    near, far = ctx.sc.near_far
    zc = 1.0 / (1.0 / near + nz * (1.0 / far - 1.0 / near)) if lindisp else near + nz * (far - near)
    q = torch.stack([u * (W - 1) * zc, v * (H - 1) * zc, zc], -1)
    w2c = ctx.sc.pose_source["w2cs"][0].double()
    K = ctx.sc.pose_source["intrinsics"][0].double()
    M = K @ w2c[:3, :3]
    pts = torch.linalg.solve(M, (q - (K @ w2c[:3, 3])).T).T
    return ndc, pts


def _oracle_presigma(ctx, weights, ndc, pts):
    """alpha_linear(h) before the ReLU at the given samples, the oracle's MLP in fp64 on the GPU"""
    w = {k: v.to(DEV).double() for k, v in weights.items() if k.startswith("mlp/")}
    vol = ctx.vol.detach().float().contiguous().double()
    ndc_d, pts_d = ndc.to(DEV).double().view(1, -1, 3), pts.to(DEV).double().view(1, -1, 3)
    pose = {k: v.to(DEV).double() for k, v in ctx.sc.pose_source.items()}
    feat = torch.cat([orc.lookup_volume(vol, ndc_d),
                      orc.gather_colors(pts_d, pose["w2cs"], pose["intrinsics"], ctx.d.imgs_raw[0].double())], -1)[0]
    pe = orc.positional_encoding(ndc_d[0])
    p = "mlp/nerf."
    out = []
    for i in range(0, pe.shape[0], 65536):
        x_pe, x_f = pe[i:i + 65536], feat[i:i + 65536]
        mod = torch.nn.functional.linear(x_f, w[p + "pts_bias.weight"], w[p + "pts_bias.bias"])
        h = x_pe
        for k in range(6):
            h = torch.relu(torch.nn.functional.linear(h, w[p + f"pts_linears.{k}.weight"], w[p + f"pts_linears.{k}.bias"]) * mod)
            if k == 4:
                h = torch.cat([x_pe, h], -1)
        out.append(torch.nn.functional.linear(h, w[p + "alpha_linear.weight"], w[p + "alpha_linear.bias"])[:, 0])
    return torch.cat(out).cpu()


@pytest.mark.parametrize("lindisp", [False, True])
def test_grid_bits_against_oracle(small, weights, lindisp):
    occ = small.occ(dilate=0, lindisp=lindisp)
    D, Hp, Wp = occ.D, occ.Hp, occ.Wp
    assert (D, Hp, Wp) == tuple(small.vol.shape[2:])
    cells = occ.cells().cpu().numpy()
    ndc, pts = _node_samples(small, D, Hp, Wp, lindisp)
    z = _oracle_presigma(small, weights, ndc, pts).view(D, Hp, Wp).numpy()
    tol = max(1e-3, 1e-5 * float(np.abs(z).max()))             # pre-ReLU sigma within rounding of 0
    lo, hi = oh.cells_from_alpha(z > tol), oh.cells_from_alpha(z > -tol)
    assert (lo <= cells).all(), int((lo & ~cells).sum())
    assert (cells <= hi).all(), int((cells & ~hi).sum())
    frac = cells[:-1, :-1, :-1].mean()
    assert 0.01 < frac < 0.99, frac
    assert (np.abs(z) < tol).mean() < 0.01
    # dilation against the host restatement, exactly
    for r in (1, 2):
        assert np.array_equal(small.occ(dilate=r, lindisp=lindisp).cells().cpu().numpy(), oh.dilate(cells, r)), r


def test_half_volume_grid(small):
    a = small.occ(vol=small.vol.half())
    b = small.occ(vol=small.vol.half().float())
    assert torch.equal(a.bits, b.bits)


def test_cache(small):
    a = small.occ()
    assert small.occ() is a
    assert small.occ(dilate=2) is not a
    vol = small.vol.clone()
    c = small.occ(vol=vol)
    assert small.occ(vol=vol) is c
    vol.add_(0.0)                                               # a new version of the volume: rebuilt
    d = small.occ(vol=vol)
    assert d is not c and torch.equal(d.bits, c.bits)


# ---- the ranges ---------------------------------------------------------------------------------------------------
def _host_occupied(ctx, rays, cells, S, lindisp):
    """per sample (host march + NDC in fp32): occupied, and ambiguous (within 1e-5 of a cell face or the volume's
    boundary, where the kernel's NDC may round to the other side)"""
    H, W = ctx.sc.H, ctx.sc.W
    xyz, _, _, _ = backend.ray_marcher(rays, N_samples=S, lindisp=lindisp)
    ndc = backend.get_ndc_coordinate(ctx.d.pose_source["w2cs"][0], ctx.d.pose_source["intrinsics"][0], xyz,
                                     torch.tensor([W - 1.0, H - 1.0], device=DEV), near=ctx.sc.near_far[0],
                                     far=ctx.sc.near_far[1], pad=ctx.sc.pad, lindisp=lindisp).cpu().numpy()
    occupied = oh.sample_occupied(ndc, cells)
    amb = np.zeros(occupied.shape, dtype=bool)
    for axis, size in enumerate((cells.shape[2], cells.shape[1], cells.shape[0])):
        i = ndc[..., axis].astype(np.float64) * (size - 1)
        amb |= np.abs(i - np.round(i)) < 1e-5 * (size - 1)
    return occupied, amb


@pytest.mark.parametrize("lindisp", [False, True])
@pytest.mark.parametrize("mode", [PAIR, SPLIT])
def test_ranges_against_host(small, mode, lindisp):
    occ = small.occ(lindisp=lindisp)
    cells = occ.cells().cpu().numpy()
    for n, S in ((8461, 128), (8461, 24), (1994, 200)):
        rays = torch.cat([small.rays, small.rays])[:n].contiguous()
        rgb, depth, tiles = small.counted(rays, mode, S=S, lindisp=lindisp, occupancy=occ)
        got, rt = _kernel_ranges(n)
        occupied, amb = _host_occupied(small, rays, cells, S, lindisp)
        lo, hi = oh.group_ranges(occupied & ~amb, rt), oh.group_ranges(occupied | amb, rt)
        assert (hi[:, 0] <= got[:, 0]).all() and (got[:, 0] <= lo[:, 0]).all(), (n, S)
        assert (lo[:, 1] <= got[:, 1]).all() and (got[:, 1] <= hi[:, 1]).all(), (n, S)
        assert tiles == int(np.maximum(got[:, 1] - got[:, 0] + 1, 0).sum()), (n, S)


# ---- the result ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("white", [False, True])
@pytest.mark.parametrize("mode", [PAIR, SPLIT])
def test_plane_bound_and_bit_identity(plane, mode, white):
    S = 128
    occ = plane.occ(dilate=1)
    rays = plane.rays
    n = rays.shape[0]
    rgb0, depth0 = plane.render(rays, mode, S=S, white=white)
    rgb, depth, tiles = plane.counted(rays, mode, S=S, white=white, occupancy=occ)
    got, rt = _kernel_ranges(n)
    alpha = plane.alpha(rays, mode, S).double()
    sp = 64 // rt
    tile_of = torch.arange(S, device=DEV) // sp
    kf = torch.from_numpy(got[:, 0]).to(DEV).repeat_interleave(rt)[:n]
    kl = torch.from_numpy(got[:, 1]).to(DEV).repeat_interleave(rt)[:n]
    lead = tile_of[None, :] < kf[:, None]
    kept = (tile_of[None, :] >= kf[:, None]) & (tile_of[None, :] <= kl[:, None])
    A = 1.0 - torch.where(lead, 1.0 - alpha, torch.ones_like(alpha)).prod(1)
    T_after = torch.where(lead | kept, 1.0 - alpha, torch.ones_like(alpha)).prod(1)
    bound = A + torch.where(kl >= 0, T_after, torch.zeros_like(T_after)) + 1e-5
    d = (rgb - rgb0).abs().max(1).values.double()
    assert (d <= bound).all(), (d - bound).max().item()
    exact = (torch.where(kept, torch.zeros_like(alpha), alpha) == 0).all(1)
    same = (rgb == rgb0).all(1) & (depth == depth0)
    assert same[exact].all(), int((~same[exact]).sum())
    assert tiles == int(np.maximum(got[:, 1] - got[:, 0] + 1, 0).sum())
    assert tiles < ((n + rt - 1) // rt) * ((S + sp - 1) // sp)          # some tiles are skipped
    assert exact.float().mean() > 0.9
    print(f"plane {mode} white={white}: tiles {tiles}, pixels with only alpha == 0 skipped {exact.float().mean():.4f}, "
          f"bit-identical {same.float().mean():.4f}, max |drgb| {d.max():.3e}")


@pytest.mark.parametrize("mode", [PAIR, SPLIT])
def test_deterministic_and_split_invariant(plane, mode):
    occ = plane.occ()
    rgb1, depth1, t1 = plane.counted(plane.rays, mode, t_stop=1e-4, occupancy=occ)
    rgb2, depth2, t2 = plane.counted(plane.rays, mode, t_stop=1e-4, occupancy=occ)
    assert torch.equal(rgb1, rgb2) and torch.equal(depth1, depth2) and t1 == t2
    cut = 32 * 4000                                            # both parts keep 32 rays per group
    a = plane.counted(plane.rays[:cut].contiguous(), mode, t_stop=1e-4, occupancy=occ)
    b = plane.counted(plane.rays[cut:].contiguous(), mode, t_stop=1e-4, occupancy=occ)
    assert torch.equal(torch.cat([a[0], b[0]]), rgb1) and torch.equal(torch.cat([a[1], b[1]]), depth1)
    assert a[2] + b[2] == t1
    _, _, t_stop_only = plane.counted(plane.rays, mode, t_stop=1e-4)
    assert t1 < t_stop_only


def test_rejections_and_render_video(small):
    occ = small.occ()
    rays = small.rays[:64].contiguous()
    with pytest.raises(RuntimeError, match="tensor-core"):
        small.render(rays, lib.MLP_FP32, occupancy=occ)
    with pytest.raises(RuntimeError, match="sink"):
        small.render(rays, SPLIT, occupancy=occ, sink=lib.PeerSink())
    with pytest.raises(RuntimeError, match="lindisp"):
        small.render(rays, SPLIT, occupancy=occ, lindisp=True)
    from mvsnerf_b200 import scene_io
    c2ws = synthetic.spiral_path(small.sc, n_frames=2).to(DEV)
    args = (small.d.directions, small.vol, small.d.imgs_raw, small.d.pose_source, small.fn, small.sc.near_far,
            float(small.sc.pad))
    with torch.no_grad():
        full = scene_io.render_video(c2ws, *args, mlp_mode=PAIR)
        same = scene_io.render_video(c2ws, *args, mlp_mode=PAIR, occupancy=_filled(occ, -1))
        skip = scene_io.render_video(c2ws, *args, mlp_mode=PAIR, occupancy=occ)
    for (a, b), (c, d), (e, f) in zip(full, same, skip):
        assert torch.equal(a, c) and torch.equal(b, d)
        assert (a - e).abs().max() < 0.5
