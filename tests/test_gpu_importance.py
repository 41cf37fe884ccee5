"""GPU: importance sampling from a density grid (build_density, mvsn_sample_importance, render_rays(density=),
FineTuner.step_rays(density=), ray_marcher_fine).

  * the density grid against the oracle MLP's sigma at every node, fp16 volume bit-identical to its fp32 upcast, a
    sigma tensor interchangeable with its Density, the cache;
  * the sampler against the float64 restatement (tests/importance_oracle.py) on mixed-camera rays with per-ray
    near/far (near == far and NDC outside [0,1]^3 included), S in {3, 33, 64, 128}, K in {1, 32, 64, 200}, lindisp,
    jittered and unjittered, an all-zero grid and a one-slab grid: output sorted, the coarse march bit-identical to
    ray_marcher, the coarse depths present bit-exactly, pts bit-identical to o + d z, NDC against get_ndc_coordinate,
    the fine depths within 1e-3 of their bin's width on rays whose every sample lies in a bin of pdf >= 1e-3 (all but
    2e-4 of them) and within two of the widest bins everywhere;
  * ray_marcher_fine draws the reference's u from the default generator;
  * render_rays(density=) bit-identical to `rendering` on the sampler's samples in all four modes, with and without
    t_stop, chunked and not;
  * FineTuner.step_rays(density=) bit-identical to FineTuner.step on the sampler's samples from the same generator
    state, deterministic repeats, t_stop = 0.
"""
import copy
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from mvsnerf_b200 import backend, lib, synthetic
import importance_oracle as io_orc
from test_gpu_mixed_rays import mixed_rays
from test_gpu_occupancy import _node_samples, _oracle_presigma

pytestmark = pytest.mark.gpu
DEV = "cuda"
MODES = [lib.MLP_FP32, lib.MLP_TC_HALF, lib.MLP_TC_PAIR, lib.MLP_TC_SPLIT]


class Ctx:
    def __init__(self, sc, fn, mvs):
        self.sc, self.fn, self.d = sc, fn, sc.to(DEV)
        with torch.no_grad():
            self.vol, _, _ = mvs(self.d.imgs_norm, self.d.proj_mats, sc.near_far, pad=sc.pad)
        self.rays = synthetic.scene_rays(sc).to(DEV).contiguous()
        self.nf, self.pad = sc.near_far, float(sc.pad)

    def density(self, vol=None, lindisp=False):
        return backend.build_density(self.vol if vol is None else vol, self.d.imgs_raw, self.d.pose_source, self.fn,
                                     self.nf, self.pad, lindisp=lindisp)

    def sample(self, rays, density, S, K, lindisp=False, jitter=None, u=None):
        return backend.sample_importance(rays, density, self.vol, self.d.imgs_raw, self.d.pose_source, self.fn, self.nf,
                                         self.pad, N_samples=S, N_importance=K, lindisp=lindisp, jitter=jitter, u=u)

    def ndc(self, pts, lindisp=False):
        H, W = self.sc.H, self.sc.W
        n, m = pts.shape[:2]
        return backend.get_ndc_coordinate(self.d.pose_source["w2cs"][0], self.d.pose_source["intrinsics"][0], pts,
                                          torch.tensor([W - 1.0, H - 1.0], device=DEV), near=self.nf[0], far=self.nf[1],
                                          pad=self.pad, lindisp=lindisp).view(n, m, 3)


@pytest.fixture(scope="module")
def small():
    fn, mvs = backend.MVSNeRF().to(DEV), backend.MVSNet().to(DEV).train()
    backend.load_weights_npz(fn, mvs, os.path.join(GOLDEN, "mvsnerf_v0_weights.npz"))
    return Ctx(synthetic.make_scene(96, 128, pad=4, seed=5), fn, mvs)


# ---- the grid ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lindisp", [False, True])
def test_density_against_oracle(small, weights, lindisp):
    den = small.density(lindisp=lindisp)
    D, Hp, Wp = den.D, den.Hp, den.Wp
    assert (D, Hp, Wp) == tuple(small.vol.shape[2:])
    ndc, pts = _node_samples(small, D, Hp, Wp, lindisp)
    want = torch.relu(_oracle_presigma(small, weights, ndc, pts)).view(D, Hp, Wp)
    got = den.sigma.cpu().double()
    err = ((got - want).abs() / want.abs().clamp(min=1.0)).max().item()
    assert err < 1e-4, err
    assert 0.01 < (want > 0).double().mean() < 0.99


def test_density_half_volume_cache_and_tensor(small):
    a = small.density(vol=small.vol.half())
    b = small.density(vol=small.vol.half().float())
    assert torch.equal(a.sigma, b.sigma)
    c = small.density()
    assert small.density() is c
    rays = small.rays[:4096]
    z0, p0, n0 = small.sample(rays, c, 32, 32)
    z1, p1, n1 = small.sample(rays, c.sigma.clone(), 32, 32)
    assert torch.equal(z0, z1) and torch.equal(p0, p1) and torch.equal(n0, n1)


# ---- the sampler ------------------------------------------------------------------------------------------------
def _host_march(rays, S, lindisp, jitter):
    """ray_marcher (data/ray_utils.py:152-197) with the draw replaced by `jitter`"""
    near, far = rays[:, 6:7], rays[:, 7:8]
    t = torch.linspace(0, 1, S, device=rays.device)
    z = 1 / (1 / near * (1 - t) + 1 / far * t) if lindisp else near * (1 - t) + far * t
    z = z.expand(rays.shape[0], S)
    if jitter is not None:
        mid = 0.5 * (z[:, :-1] + z[:, 1:])
        upper, lower = torch.cat([mid, z[:, -1:]], -1), torch.cat([z[:, :1], mid], -1)
        z = lower + (upper - lower) * jitter
    return z.contiguous()


def _fine_of(z, zc, with_mask=False):
    """the K fine depths of the sorted output z [N,S+K]: z without one occurrence of each coarse depth zc [N,S]"""
    zs = torch.sort(zc, -1)[0].contiguous()
    occ = torch.arange(z.shape[1], device=z.device).expand_as(z) - torch.searchsorted(z, z, right=False)
    cnt = torch.searchsorted(zs, z.contiguous(), right=True) - torch.searchsorted(zs, z.contiguous(), right=False)
    fine = occ >= cnt
    assert (fine.sum(1) == z.shape[1] - zc.shape[1]).all()        # every coarse depth is present, bit-exactly
    return (z[fine].view(z.shape[0], -1), fine) if with_mask else z[fine].view(z.shape[0], -1)


def _check_sampler(ctx, rays, sigma, S, K, lindisp, jitter, u, worst):
    """u: None (linspace) or sorted per ray, so that the k-th smallest fine depth is the k-th draw's"""
    n = rays.shape[0]
    z, pts, ndc = ctx.sample(rays, sigma, S, K, lindisp=lindisp, jitter=jitter, u=u)
    zc = _host_march(rays, S, lindisp, jitter)
    assert (z[:, 1:] >= z[:, :-1]).all()
    fk, fine = _fine_of(z, zc, with_mask=True)
    fk = fk.double()
    assert torch.equal(pts, rays[:, None, 0:3] + rays[:, None, 3:6] * z[..., None])
    nd = ctx.ndc(pts, lindisp)
    fin = torch.isfinite(nd)
    assert ((ndc - nd).abs()[fin] <= 1e-5 * nd.abs()[fin].clamp(min=1.0)).all(), (ndc - nd).abs()[fin].max()
    # the float64 oracle on the host march and the kernel's NDC of those points (its output at the coarse depths: the
    # grid is steep enough that get_ndc_coordinate's last-bit differences move sigma, and so the cdf, by more than the
    # sampler's own rounding)
    u64 = (io_orc.linspace_u(n, K, device=DEV) if u is None else u).double()
    zs = torch.sort(zc, -1)[0]
    ndc_c = ndc[~fine].view(n, S, 3)
    _, _, dg = io_orc.ray_marcher_fine(rays.double(), sigma.double(), zs.double(), ndc_c.double(), u64)
    fo, order = torch.sort(dg["fine"], -1)
    below = dg["below"].gather(1, order)
    denom = dg["denom"].gather(1, order)
    above = (below + 1).clamp(max=S - 2)
    width = (dg["bins"].gather(1, above) - dg["bins"].gather(1, below)).abs()
    err = (fk - fo).abs()
    # the fp32 rounding of the bins, of the interpolation and of the coarse depths themselves (a near == far ray marches
    # depths an ulp or two apart): 16 ulp of the larger bin
    slack = 16 * 2.0 ** (torch.floor(torch.log2(torch.maximum(dg["bins"].gather(1, below).abs(),
                                                             dg["bins"].gather(1, above).abs()).clamp(min=1e-30))) - 23)
    near_thr = (denom - 1e-5).abs() < 1e-8                       # within 0.1 % of sample_pdf's 1e-5 threshold
    # the fp32 cdf near 1 carries ~5e-7 absolute error (S fp32 additions), which moves a sample in a bin of pdf p by
    # ~5e-7 / p of the bin: the 1e-3 gate holds from p = 1e-3 (the proposed 1e-4 would need an fp64 cdf)
    strict = (denom >= 1e-3) & ~near_thr
    rel = torch.where(width > 0, err / width, torch.zeros_like(err))
    # near the threshold the fp32 difference of two cdf values close to 1 (~1e-7 absolute, 1 % of 1e-5) decides
    # whether sample_pdf divides by it or by 1; those samples are counted and held to their bin.  The lists are compared
    # by rank, so a ray with one sample outside the strict gate can shift its neighbours by up to that sample's bin: the
    # 1e-3 gate applies to rays whose every fine sample lies in a bin of pdf >= 1e-4, the rest to the widest bin.
    flipped = near_thr & (err > 1e-3 * width + slack)
    ray_strict = strict.all(1)
    wmax = (dg["bins"][:, 1:] - dg["bins"][:, :-1]).abs().max(1, keepdim=True).values if S > 2 else width
    worst.append((float(rel[ray_strict].max()) if ray_strict.any() else 0.0, float((err / wmax.clamp(min=1e-30)).max()),
                  int(flipped.sum()), int((~ray_strict).sum()), int(err.numel())))
    over = ray_strict[:, None] & (err > 1e-3 * width + slack)
    worst.append(worst.pop() + (int(over.sum()),))
    # a few samples of a ray compared by rank can shift by one neighbour (measured: at most 8.8e-5 of the samples)
    if int(over.sum()) > max(1, int(2e-4 * err.numel())):
        r, c = [int(v) for v in over.nonzero()[0]]
        raise AssertionError(f"S={S} K={K} lindisp={lindisp}: {int(over.sum())} samples, e.g. ray {r}: kernel {fk[r, c]!r} "
                             f"oracle {fo[r, c]!r} width {width[r, c]!r} denom {denom[r, c]!r} ray {rays[r].tolist()}")
    # a threshold flip moves a sample across its bin, and the comparison by rank can then pair it with a neighbour in
    # the next bin: two of the widest bins
    far_off = err > 2 * wmax + slack
    if far_off.any():
        r, c = [int(v) for v in far_off.nonzero()[0]]
        raise AssertionError(f"S={S} K={K} lindisp={lindisp}: {int(far_off.sum())} samples beyond two of the widest bins, e.g. ray "
                             f"{r} sample {c}: kernel {fk[r, c]!r} oracle {fo[r, c]!r} widest {wmax[r, 0]!r} "
                             f"denom {denom[r, c]!r} ray {rays[r].tolist()} fine kernel {fk[r].tolist()} "
                             f"fine oracle {fo[r].tolist()}")
    assert int(flipped.sum()) <= max(1, int(1e-2 * err.numel())), int(flipped.sum())


@pytest.mark.parametrize("S,K", [(3, 1), (3, 200), (33, 32), (64, 64), (128, 64), (128, 200), (33, 1)])
def test_sampler_against_oracle(small, S, K):
    den = small.density()
    worst = []
    rays, _, _ = mixed_rays(small.sc, 4096, seed=S * 1000 + K)
    rays = rays.to(DEV)
    g = torch.Generator(device=DEV).manual_seed(S + K)
    for lindisp in (False, True):
        d = den.sigma if not lindisp else small.density(lindisp=True).sigma
        for jit in (False, True):
            jitter = torch.rand((rays.shape[0], S), device=DEV, generator=g) if jit else None
            for u in (None, torch.sort(torch.rand((rays.shape[0], K), device=DEV, generator=g), -1)[0]):
                _check_sampler(small, rays, d, S, K, lindisp, jitter, u, worst)
    print("IMPORTANCE worst (err / bin width on strict rays, err / widest bin; threshold flips, non-strict rays, samples, over the 1e-3 gate):",
          [max(w[i] for w in worst) for i in range(6)])


@pytest.mark.parametrize("grid", ["zeros", "slab"])
def test_sampler_special_grids(small, grid):
    den = small.density()
    sigma = torch.zeros_like(den.sigma)
    if grid == "slab":
        sigma[den.D // 2] = 50.0
    rays, _, _ = mixed_rays(small.sc, 2048, seed=7)
    rays = rays.to(DEV)
    worst = []
    for S, K in ((64, 64), (33, 200)):
        _check_sampler(small, rays, sigma, S, K, False, None, None, worst)
        _check_sampler(small, rays, sigma, S, K, False, None, torch.sort(torch.rand((2048, K), device=DEV), -1)[0], worst)
    print("IMPORTANCE", grid, "worst:", [max(w[i] for w in worst) for i in range(6)])


def test_ray_marcher_fine_mirror(small):
    den = small.density()
    rays = small.rays[:3000]
    xyz, _, _, zc = backend.ray_marcher(rays, N_samples=48, perturb=1.0)
    ndc = small.ndc(xyz)
    torch.manual_seed(5)
    got = backend.ray_marcher_fine(rays, den, zc, ndc, N_importance=40)
    after = torch.rand(4, device=DEV)
    torch.manual_seed(5)
    u = torch.rand((3000, 40), device=DEV)
    assert torch.equal(torch.rand(4, device=DEV), after)
    xyz_o, z_o, _ = io_orc.ray_marcher_fine(rays.double(), den.sigma.double(), zc.double(), ndc.double(), u.double())
    spacing = (zc[:, -1] - zc[:, 0]).double() / 47
    close = (got[3].double() - z_o).abs().max(1).values <= 1e-3 * spacing + 1e-6
    frac = close.float().mean().item()
    print("IMPORTANCE mirror: rays within 1e-3 of the spacing", frac)
    assert frac > 0.95                  # the rest: samples in bins whose pdf sits at sample_pdf's 1e-5 threshold
    assert ((got[3].double() - z_o).abs().max(1).values <= spacing * 1.01 + 1e-6).all()
    assert torch.equal(got[0], rays[:, None, 0:3] + rays[:, None, 3:6] * got[3][..., None])
    assert torch.equal(got[1], rays[:, 0:3]) and torch.equal(got[2], rays[:, 3:6])


# ---- render -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
def test_render_matches_rendering_on_samples(small, mode, monkeypatch):
    den = small.density()
    rays = small.rays
    S, K = 64, 64
    args = SimpleNamespace(use_color_volume=False)
    z, pts, ndc = small.sample(rays, den, S, K)
    stops = (None,) if mode == lib.MLP_FP32 else (None, 0.0, 1e-3)
    for t_stop in stops:
        kw = {} if t_stop is None else {"t_stop": t_stop}
        with torch.no_grad():
            rgb, depth = backend.render_rays(rays, small.vol, small.d.imgs_raw, small.d.pose_source, small.fn, small.nf,
                                             small.pad, N_samples=S, mlp_mode=mode, density=den, N_importance=K, **kw)
            ref = backend.rendering(args, small.d.pose_source, pts, ndc, z, None, rays[:, 3:6].contiguous(), small.vol,
                                    small.d.imgs_raw, network_fn=small.fn, mlp_mode=mode, want_aux=False, **kw)
        assert torch.equal(rgb, ref[0]) and torch.equal(depth, ref[3]), t_stop
    if mode != lib.MLP_FP32:
        with torch.no_grad():
            a = backend.render_rays(rays, small.vol, small.d.imgs_raw, small.d.pose_source, small.fn, small.nf, small.pad,
                                    N_samples=S, mlp_mode=mode, density=den, N_importance=K)
            monkeypatch.setattr(backend, "IMPORTANCE_CHUNK_RAYS", 4096)
            b = backend.render_rays(rays, small.vol, small.d.imgs_raw, small.d.pose_source, small.fn, small.nf, small.pad,
                                    N_samples=S, mlp_mode=mode, density=den, N_importance=K)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


# ---- fine-tuning ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,K", [(64, 64), (96, 32)])
@pytest.mark.parametrize("grad_mode", [lib.MLP_FP32, lib.MLP_TC_HALF])
def test_step_rays_matches_step(small, S, K, grad_mode):
    den = small.density()
    rays = small.rays[::7][:1024].contiguous()
    tgt = small.d.imgs_raw[0, 0].permute(1, 2, 0).reshape(-1, 3)[::7][:1024].contiguous()

    def tuner():
        fn = copy.deepcopy(small.fn)
        vol = backend.RefVolume(small.vol.detach().clone()).to(DEV)
        return backend.FineTuner(fn, vol, small.d.imgs_raw, small.d.pose_source, white_bkgd=False, grad_mode=grad_mode)

    def state(t):
        return [p.detach().clone() for p in t.params] + [t.volume.feat_volume.detach().clone()]

    torch.use_deterministic_algorithms(True)        # float atomics would make two runs differ in the last bits
    for t_stop in (None, 0.0):
        a, b = tuner(), tuner()
        ga = torch.Generator(device=DEV).manual_seed(3)
        gb = torch.Generator(device=DEV).manual_seed(3)
        la, _ = a.step_rays(rays, tgt, small.nf, small.pad, N_samples=S, perturb=1.0, generator=ga, density=den,
                            N_importance=K, t_stop=t_stop)
        jitter = torch.rand((1024, S), device=DEV, generator=gb)
        u = torch.rand((1024, K), device=DEV, generator=gb)
        z, pts, ndc = small.sample(rays, den, S, K, jitter=jitter, u=u)
        lb, _ = b.step(pts, ndc, z, rays[:, 3:6], tgt, t_stop=t_stop)
        assert torch.equal(la, lb), t_stop
        for x, y in zip(state(a), state(b)):
            assert torch.equal(x, y)
        if t_stop is None:
            base = state(a)
        else:
            for x, y in zip(state(a), base):
                assert torch.equal(x, y)
    try:
        out = []
        for _ in range(2):
            t = tuner()
            g = torch.Generator(device=DEV).manual_seed(4)
            for _ in range(3):
                t.step_rays(rays, tgt, small.nf, small.pad, N_samples=S, generator=g, density=den, N_importance=K)
            out.append(state(t))
        for x, y in zip(*out):
            assert torch.equal(x, y)
    finally:
        torch.use_deterministic_algorithms(False)


def test_step_rays_rejections(small):
    den = small.density()
    t = backend.FineTuner(copy.deepcopy(small.fn), backend.RefVolume(small.vol.detach().clone()).to(DEV),
                          small.d.imgs_raw, small.d.pose_source, grad_mode=lib.GRAD_TC_FULL)
    with pytest.raises(RuntimeError, match="GRAD_TC_FULL"):
        t.step_rays(small.rays[:64], small.rays[:64, :3], small.nf, small.pad, N_samples=64, density=den, N_importance=32)
    with pytest.raises(RuntimeError, match="128"):
        t.step_rays(small.rays[:64], small.rays[:64, :3], small.nf, small.pad, N_samples=128, density=den, N_importance=64)
