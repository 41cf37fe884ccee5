"""GPU: the render and fine-tuning entries on ray batches drawn from several cameras, each ray with its own near / far.

Training batches mix rays of several views (the reference's fine-tuning script draws them so), and the [N,8] ray format
carries a near and a far per ray.  Several kernels share state across the rays of a group or tile: the early-termination
verdict, the occupancy ranges, the fp16 modes' tile packing (RT rays x SP samples per 64-row tile), the per-tile operand
scales of the MLP_TC_HALF backward, the rays-entry backward's NDC staging.  On single-camera batches with one near / far
every ray of a group has the same depth range, so a ray's near / far or depths taken from another ray of its group
cancel out.  Here every group of 4, 8, 16 or 32 consecutive rays mixes four cameras and five kinds of depth range:

  * render_rays against independent references: MLP_FP32 and MLP_TC_SPLIT against the fp32 oracle, MLP_TC_PAIR and
    MLP_TC_HALF against the fp16 emulation (oracle.mlp_emulated "half") and against fp32; every rays-per-tile band,
    S of 24, 33, 128 and 200, pad 0 and 24, white_bkgd, lindisp, an fp16 volume and random weights;
  * the samples entry (backend.rendering, all five outputs) on per-ray stratified depths;
  * t_stop: 0 is bit-identical, and each group's stop tile follows from the full render's alpha;
  * occupancy: the range table against a host march, an all-ones grid against t_stop, the skip bound;
  * fine-tuning: render_backward_rays against the same jitter marched on the host and against the oracle's autograd,
    the t_stop backward's live counts, and FineTuner.step_rays against `rendering` under autograd + torch.optim.Adam.

The forward oracle and the fp16 emulation run on the GPU here (both follow the device of their inputs), so that whole
batches of every rays-per-tile band are checked in seconds; the gradient references run on the CPU.

Measured on an H100 80GB HBM3, largest error over the cases against each gate: render_rays FP32 / TC_SPLIT vs the
oracle rgb 3.5e-5 (1e-4), depth 2.1e-4 (1e-3 x far scale); TC_PAIR / TC_HALF vs the emulation alpha 7.9e-4 (1.6e-3),
rgb 2.1e-4 (8e-4), depth 1.0e-3 (2.4e-3 x far scale), vs the oracle rgb 2.8e-3 (5e-3), depth 1.3e-2 (2e-2 x far
scale); the rays-entry backward bit-identical to the samples entry on the host-marched jitter; its gradients vs the
oracle 2.5e-6 (FP32, 2e-4) and 1.1e-3 (TC_HALF, 3e-3), TC_HALF vs its emulation 1.1e-4 (2e-4).
"""
import contextlib
import ctypes as C
import functools
import itertools
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from grad_emulation import mlp_grad_emulated
from mvsnerf_b200 import backend, lib, synthetic
from oracle import mvsnerf_oracle as orc
import occupancy_host as oh

pytestmark = pytest.mark.gpu
DEV = "cuda"
WPATH = os.path.join(GOLDEN, "mvsnerf_v0_weights.npz")
TC_MODES = [lib.MLP_TC_PAIR, lib.MLP_TC_HALF, lib.MLP_TC_SPLIT]
GRAD_MODES = [lib.MLP_FP32, lib.MLP_TC_HALF]

# the gates of tests/test_gpu_tc_range.py; depth gates scale with the batch's largest far (they were set at far 4.525)
RGB_TOL, DEPTH_TOL = 1e-4, 1e-3          # fp32 and split modes vs the fp32 oracle
PAIR_TOL, PAIR_DEPTH_TOL = 5e-3, 2e-2    # fp16 modes vs the fp32 oracle
PAIR_EMU_TOL = 8e-4                      # fp16 modes vs their emulation
PAIR_EMU_SAMPLE_TOL = 1.6e-3             # per-sample alpha / weights
PAIR_EMU_DEPTH_TOL = 2.4e-3
MASK_COLS = [11, 15, 19]                 # input_feat: the strict in-bounds mask of each source view
HALF = functools.partial(orc.mlp_emulated, mode="half")
GRAD_GATE = {lib.MLP_FP32: 2e-4, lib.MLP_TC_HALF: 3e-3}   # vs the oracle's fp32 autograd, of max|g|
GRAD_EMU_GATE = 2e-4                                      # TC_HALF vs tests/grad_emulation.py


# ------------------------------------------------------------------------------------------------------------------
# the mixed batch
# ------------------------------------------------------------------------------------------------------------------
N_CAMS = 4
FRONT, BEYOND, WIDE, NARROW, EQUAL = range(5)           # kinds of depth range
KIND_P = [0.3, 0.3, 0.2, 0.13, 0.07]
# only NARROW and EQUAL: every sample inside the scene's depth range, so groups of an occupancy launch can skip tiles
# (a sample outside the volume counts as occupied, and most groups of KIND_P hold one at both ends)
INSIDE_P = [0.0, 0.0, 0.0, 0.8, 0.2]


def mixed_cameras(sc):
    """c2w [4,4,4]: the scene's target camera and three poses of its spiral path.  Every one is rotated against the
    reference camera: a camera that is only translated along x from it (spiral_path(sc, 6)[3]) puts its top and bottom
    pixel rows exactly on the reference view's border at every depth, where the fp16 modes' approximate projection flips
    the strict in-bounds mask of most samples of those rays"""
    return torch.stack([sc.c2w_target] + [synthetic.spiral_path(sc, 8)[i] for i in (1, 3, 5)])


def mixed_rays(sc, n, seed, kind_p=KIND_P):
    """(rays [n,8], camera [n], kind [n]).  Ray i comes from camera i % 4 (a random pixel of it), so every group of 4
    or more consecutive rays holds all four cameras.  Each ray gets its own near / far around the scene's near_far
    (n0, f0), span = f0 - n0, by kind:
      FRONT   near in n0 - [0.05, 0.35] span (NDC z < 0 at the first samples), far in f0 - [0, 0.2] span;
      BEYOND  near in n0 + [0, 0.2] span, far in f0 + [0.05, 0.45] span (past the volume);
      WIDE    near in n0 - [0, 0.25] span, far in f0 + [0, 0.25] span;
      NARROW  near in n0 + [0, 0.9] span, far = near + [0.002, 0.032] span;
      EQUAL   near == far in [n0, f0].
    `kind_p`: the probabilities of the five kinds."""
    g = torch.Generator().manual_seed(seed)
    n0, f0 = (float(x) for x in sc.near_far)
    span = f0 - n0
    cam = torch.arange(n) % N_CAMS
    rays = torch.empty(n, 8)
    for c, c2w in enumerate(mixed_cameras(sc)):
        sel = (cam == c).nonzero().squeeze(1)
        allr = synthetic.camera_rays(sc.directions, c2w, n0, f0)
        pix = torch.randperm(allr.shape[0], generator=g)[:sel.numel()]
        rays[sel] = allr[pix]
    kind = torch.multinomial(torch.tensor(kind_p, dtype=torch.float32), n, replacement=True, generator=g)
    u0, u1 = torch.rand(n, generator=g), torch.rand(n, generator=g)
    near = torch.empty(n)
    far = torch.empty(n)
    for k, (nr, fr) in {FRONT: (n0 - span * (0.05 + 0.3 * u0), f0 - 0.2 * span * u1),
                        BEYOND: (n0 + 0.2 * span * u0, f0 + span * (0.05 + 0.4 * u1)),
                        WIDE: (n0 - 0.25 * span * u0, f0 + 0.25 * span * u1),
                        NARROW: (n0 + 0.9 * span * u0, n0 + 0.9 * span * u0 + span * (0.002 + 0.03 * u1)),
                        EQUAL: (n0 + span * u0, n0 + span * u0)}.items():
        near[kind == k], far[kind == k] = nr[kind == k], fr[kind == k]
    rays[:, 6], rays[:, 7] = near, far
    return rays.contiguous(), cam, kind


NWG = 2                                   # MMA warpgroups per CTA (csrc/render_wg.cu, wg::NWG)


def rays_per_tile(n, sms):
    """The selection loop of launch_render_wg (csrc/render_wg.cu): 32 rays per tile unless that leaves a warpgroup of
    some SM without a ray group."""
    rt = 32
    while rt > 4 and (n + rt - 1) // rt < NWG * sms:
        rt >>= 1
    return rt


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def n_for(rt):
    """rt (2 sms + 1) - 1 rays: inside the band of rt rays per tile, an odd number of groups, a ragged last group"""
    n = rt * (2 * _sms() + 1) - 1
    assert rays_per_tile(n, _sms()) == rt, (rt, n)
    return n


@contextlib.contextmanager
def _deterministic(flag):
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(flag, warn_only=True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


# ------------------------------------------------------------------------------------------------------------------
# scenes
# ------------------------------------------------------------------------------------------------------------------
def _net(w=None):
    fn = backend.MVSNeRF().to(DEV)
    if w is None:
        backend.load_weights_npz(fn, None, WPATH)
    else:
        fn.load_state_dict({k[len("mlp/"):]: v for k, v in w.items() if k.startswith("mlp/")})
    return fn


def _random_weights(seed):
    """tests/test_gpu_tc_range.py's random MLP (nn.Linear default init): every hidden unit carries signal"""
    torch.manual_seed(seed)
    net = backend.MVSNeRF()
    return {"mlp/" + k: v.detach().clone() for k, v in net.state_dict().items()}


class Ctx:
    def __init__(self, sc):
        self.sc, self.d = sc, sc.to(DEV)
        self.fn = _net()
        mvs = backend.MVSNet().to(DEV).train()
        backend.load_weights_npz(None, mvs, WPATH)
        with torch.no_grad():
            vol, _, _ = mvs(self.d.imgs_norm, self.d.proj_mats, sc.near_far, pad=sc.pad)
        self.vol = vol.detach()

    def render(self, rays, mode, S, white=False, lindisp=False, vol=None, fn=None, **kw):
        with torch.no_grad():
            return backend.render_rays(rays, self.vol if vol is None else vol, self.d.imgs_raw, self.d.pose_source,
                                       self.fn if fn is None else fn, self.sc.near_far, float(self.sc.pad), N_samples=S,
                                       white_bkgd=white, lindisp=lindisp, mlp_mode=mode, **kw)

    def counted(self, rays, mode, S, **kw):
        tiles = torch.zeros(1, dtype=torch.int64, device=DEV)
        rgb, depth = self.render(rays, mode, S, tiles_done=tiles, **kw)
        return rgb, depth, int(tiles.item())

    def raw(self, rays, mode, t_steps, white=False, lindisp=False, alpha=None, feat=None, vol=None, fn=None):
        """mvsn_render_rays with explicit t_steps (any prefix of linspace(0, 1, S)) and optional alpha / input_feat
        outputs"""
        L = lib.load()
        sc, keep = backend._make_scene(self.d.pose_source, self.vol if vol is None else vol, self.d.imgs_raw,
                                       self.fn if fn is None else fn, white, mode, half_ok=True)
        rp = lib.RayParams(float(self.sc.near_far[0]), float(self.sc.near_far[1]), float(self.sc.pad), int(lindisp))
        n = rays.shape[0]
        rgb, depth = torch.empty(n, 3, device=DEV), torch.empty(n, device=DEV)
        lib.check(L.mvsn_render_rays(C.byref(sc), C.byref(rp), lib.ptr(rays), lib.ptr(t_steps), n, t_steps.shape[0],
                                     lib.ptr(rgb), lib.ptr(depth), None, lib.ptr(alpha), lib.ptr(feat), lib.stream_ptr()),
                  "mvsn_render_rays")
        torch.cuda.synchronize()
        del keep
        return rgb, depth

    def occ(self, lindisp=False):
        return backend.build_occupancy(self.vol, self.d.imgs_raw, self.d.pose_source, self.fn, self.sc.near_far,
                                       float(self.sc.pad), lindisp=lindisp, dilate=1)


@pytest.fixture(scope="module")
def scenes():
    return {pad: Ctx(synthetic.make_scene(96, 128, pad=pad, seed=5)) for pad in (0, 24)}


@pytest.fixture(scope="module")
def sparse():
    """tests/test_gpu_occupancy.py's small scene: empty space in its grid, so groups skip tiles"""
    return Ctx(synthetic.make_scene(96, 128, pad=4, seed=5))


@pytest.fixture(scope="module")
def plane():
    """rays of this scene become opaque at a textured plane (synthetic.make_plane_scene), so groups do stop"""
    return Ctx(synthetic.make_plane_scene(96, 128, pad=4, seed=3))


# ------------------------------------------------------------------------------------------------------------------
# render_rays against the oracle and the fp16 emulation
# ------------------------------------------------------------------------------------------------------------------
# (rays per tile, S, pad, white_bkgd, lindisp, fp16 volume, random weights)
RENDER_CASES = [(4, 24, 0, False, False, False, False), (8, 33, 24, True, False, False, False),
                (16, 128, 0, False, True, False, False), (32, 200, 24, False, False, True, False),
                (32, 24, 0, True, True, False, False), (4, 200, 24, False, True, True, False),
                (8, 128, 0, True, False, True, False), (16, 33, 24, False, False, False, True),
                (32, 128, 0, True, True, True, True)]


def _feat_flips(feat, want, mask, rel=0.0):
    """input_feat entries off by more than 1e-4 + rel |want|: only the strict in-bounds masks (MASK_COLS) may be (the
    fp16 front end projects with approximate reciprocals, so a sample on a view's border may flip that view's mask);
    returns the flipped entries and the rays that hold one.  `rel`: the fp16 modes' NDC is also approximate (two
    approximate divisions in a row with lindisp), which moves a volume tap by ~2.5e-5 of its value where the volume is
    steep (1.3e-4 at 4.3, lindisp, measured on an H100)."""
    err = (feat - want).abs()
    off = err > 1e-4 + rel * want.abs()
    bad = off & ~mask
    if bad.any():
        cols = bad.nonzero()[:, 2]
        raise AssertionError(f"input_feat off outside the masks: {bad.sum().item()} entries, columns {cols.unique().tolist()}, "
                             f"max {err[..., ~mask].max().item():.3e}, rays {bad.flatten(1).any(1).nonzero()[:8, 0].tolist()}, "
                             f"samples {bad.any(2).nonzero()[:8].tolist()}, got {feat[bad][:6].tolist()} want {want[bad][:6].tolist()}")
    return off, off.flatten(1).any(1)


@pytest.mark.parametrize("case", range(len(RENDER_CASES)))
def test_render_rays_vs_oracle(scenes, weights, case):
    """FP32 and TC_SPLIT against the fp32 oracle on every ray.  TC_PAIR and TC_HALF against the fp16 emulation fed the
    kernel's own input_feat (so that a flipped border mask, checked separately, is not counted twice): per-sample alpha
    on every ray, rgb and depth on the rays with near < far, and against the fp32 oracle on those of them with no
    flipped mask.  A near == far ray composites S copies of one sample, so a rounding difference in that sample's
    alpha compounds S-fold in its pixel (the emulation itself is up to ~6e-3 from fp32 there)."""
    rt, S, pad, white, lindisp, half, rnd = RENDER_CASES[case]
    ctx = scenes[pad]
    sc = ctx.sc
    n = n_for(rt)
    rays, _, kind = mixed_rays(sc, n, seed=1000 * rt + S)
    rays, kind = rays.to(DEV), kind.to(DEV)
    w = _random_weights(7) if rnd else weights
    fn = _net(w) if rnd else ctx.fn
    vol_k = ctx.vol.half() if half else ctx.vol
    vol_r = vol_k.float()                         # what the kernels read: the fp16 volume is rendered as its upcast
    w_d = {k: v.to(DEV) for k, v in w.items() if k.startswith("mlp/")}
    pose = ctx.d.pose_source
    with torch.no_grad():
        pts, z = orc.march_rays(rays, S, lindisp)
        ndc = orc.ndc_coords(pose["w2cs"][0], pose["intrinsics"][0], pts, sc.H, sc.W, sc.near_far[0], sc.near_far[1],
                             float(pad), lindisp)
        rgb_ref, feat_ref, _, depth_ref, _ = orc.render_samples(pts, ndc, z, rays[:, 3:6], vol_r, ctx.d.imgs_raw, pose,
                                                                w_d, white_bkgd=white)
    dirs = orc.view_direction(rays[:, 3:6], pose["w2cs"][0])[:, None].expand(-1, S, -1)
    t_steps = backend._tsteps_of(S, torch.device(DEV))
    mask = torch.zeros(20, dtype=torch.bool, device=DEV)
    mask[MASK_COLS] = True
    zs = max(1.0, rays[:, 7].max().item() / sc.near_far[1])
    tag = f"[render rt={rt} S={S} pad={pad} white={white} lindisp={lindisp} half_vol={half} random={rnd}]"
    for name, mode in (("fp32", lib.MLP_FP32), ("split", lib.MLP_TC_SPLIT), ("pair", lib.MLP_TC_PAIR),
                       ("half", lib.MLP_TC_HALF)):
        rgb, depth = ctx.render(rays, mode, S, white, lindisp, vol=vol_k, fn=fn)
        assert torch.isfinite(rgb).all() and torch.isfinite(depth).all(), name
        e_rgb, e_depth = (rgb - rgb_ref).abs().max(1).values, (depth - depth_ref).abs()
        if mode in (lib.MLP_FP32, lib.MLP_TC_SPLIT):
            print(f"\n{tag} {name}: vs oracle rgb {e_rgb.max():.3e} depth {e_depth.max():.3e}", end="")
            assert e_rgb.max() < RGB_TOL and e_depth.max() < DEPTH_TOL * zs, (name, e_rgb.max().item(), e_depth.max().item())
            continue
        feat, alpha = torch.empty(n, S, 20, device=DEV), torch.empty(n, S, device=DEV)
        rgb_f, depth_f = ctx.raw(rays, mode, t_steps, white, lindisp, alpha=alpha, feat=feat, vol=vol_k, fn=fn)
        assert torch.equal(rgb_f, rgb) and torch.equal(depth_f, depth), name
        off, flipped = _feat_flips(feat, feat_ref, mask, rel=1e-4)
        with torch.no_grad():
            raw = torch.cat([HALF(torch.cat([orc.positional_encoding(ndc[i:i + 1024]), feat[i:i + 1024], dirs[i:i + 1024]],
                                            -1), w_d) for i in range(0, n, 1024)])
            rgb_emu, depth_emu, _, alpha_emu = orc.composite(raw, z, white)
        m_alpha = (alpha - alpha_emu).abs().max().item()
        m_rgb, m_depth = (rgb - rgb_emu).abs().max(1).values, (depth - depth_emu).abs()
        lo = kind != EQUAL
        ok = lo & ~flipped
        print(f"\n{tag} {name}: vs emulation alpha {m_alpha:.3e} rgb {m_rgb[lo].max():.3e} depth {m_depth[lo].max():.3e} "
              f"(near == far: {m_rgb[~lo].max():.3e}, {m_depth[~lo].max():.3e}) ; vs oracle rgb {e_rgb[ok].max():.3e} "
              f"depth {e_depth[ok].max():.3e} (all rays: {e_rgb.max():.3e}, {e_depth.max():.3e}) ; "
              f"flipped masks {off.sum().item()} on {flipped.sum().item()} rays", end="")
        assert off.sum().item() <= 1e-5 * off.numel(), (name, off.sum().item())
        assert m_alpha < PAIR_EMU_SAMPLE_TOL, (name, m_alpha)
        assert m_rgb[lo].max() < PAIR_EMU_TOL and m_depth[lo].max() < PAIR_EMU_DEPTH_TOL * zs, name
        assert e_rgb[ok].max() < PAIR_TOL and e_depth[ok].max() < PAIR_DEPTH_TOL * zs, name


# (rays per tile, S, pad)
SAMPLE_CASES = [(4, 200, 24), (8, 33, 0), (32, 128, 24)]


@pytest.mark.parametrize("case", range(len(SAMPLE_CASES)))
def test_samples_entry_vs_oracle(scenes, weights, case):
    """`rendering` on per-ray stratified depths of a mixed batch: rgb, depth, weights, alpha and every row of
    input_feat.  The fp32-grade modes against the oracle, the fp16 modes against the emulation on the kernel's own
    input_feat (the fp16 front end projects with approximate reciprocals, so a sample on a view's border may flip that
    view's strict in-bounds mask, and nothing else); their pixel gates apply to the rays with near < far (see
    test_render_rays_vs_oracle), the per-sample gates to every ray."""
    class Args:
        use_color_volume = False
    rt, S, pad = SAMPLE_CASES[case]
    ctx = scenes[pad]
    sc = ctx.sc
    n = n_for(rt)
    rays, _, kind = mixed_rays(sc, n, seed=7 * rt + S)
    rays, kind = rays.to(DEV), kind.to(DEV)
    g = torch.Generator(device=DEV).manual_seed(n)
    _, z = orc.march_rays(rays, S)
    mid = 0.5 * (z[:, :-1] + z[:, 1:])
    lower, upper = torch.cat([z[:, :1], mid], -1), torch.cat([mid, z[:, -1:]], -1)
    z = (lower + (upper - lower) * torch.rand(z.shape, device=DEV, generator=g)).contiguous()
    pts = (rays[:, None, :3] + rays[:, None, 3:6] * z[..., None]).contiguous()
    pose = ctx.d.pose_source
    ndc = orc.ndc_coords(pose["w2cs"][0], pose["intrinsics"][0], pts, sc.H, sc.W, sc.near_far[0], sc.near_far[1],
                         float(pad)).contiguous()
    assert (ndc[..., 2] < 0).any() and (ndc[..., 2] > 1).any()
    w_d = {k: v.to(DEV) for k, v in weights.items() if k.startswith("mlp/")}
    vol = ctx.vol.float()
    with torch.no_grad():
        ref = orc.render_samples(pts, ndc, z, rays[:, 3:6], vol, ctx.d.imgs_raw, pose, w_d)   # rgb, feat, wts, depth, alpha
    dirs = orc.view_direction(rays[:, 3:6], pose["w2cs"][0])[:, None].expand(-1, S, -1)
    zs = max(1.0, rays[:, 7].max().item() / sc.near_far[1])
    mask = torch.zeros(20, dtype=torch.bool, device=DEV)
    mask[MASK_COLS] = True
    for mode in (lib.MLP_FP32, lib.MLP_TC_SPLIT, lib.MLP_TC_PAIR, lib.MLP_TC_HALF):
        with torch.no_grad():
            rgb, feat, wts, depth, alpha, _ = backend.rendering(Args, pose, pts, ndc, z, rays[:, :3], rays[:, 3:6], ctx.vol,
                                                                ctx.d.imgs_raw, network_fn=ctx.fn, mlp_mode=mode)
        got = [rgb, feat, wts, depth, alpha]
        assert all(torch.isfinite(t).all() for t in got), mode
        if mode in (lib.MLP_FP32, lib.MLP_TC_SPLIT):
            want, tol = ref, (RGB_TOL, RGB_TOL, DEPTH_TOL * zs)
        else:
            with torch.no_grad():
                raw = torch.cat([HALF(torch.cat([orc.positional_encoding(ndc[i:i + 1024]), feat[i:i + 1024],
                                                 dirs[i:i + 1024]], -1), w_d) for i in range(0, n, 1024)], 0)
            e_rgb, e_depth, e_wts, e_alpha = orc.composite(raw, z)
            want, tol = (e_rgb, ref[1], e_wts, e_depth, e_alpha), (PAIR_EMU_TOL, PAIR_EMU_SAMPLE_TOL, PAIR_EMU_DEPTH_TOL * zs)
        off, _ = _feat_flips(feat, want[1], mask, rel=0.0 if mode in (lib.MLP_FP32, lib.MLP_TC_SPLIT) else 1e-4)
        if mode in (lib.MLP_FP32, lib.MLP_TC_SPLIT):
            assert not off.any(), mode
        else:
            assert off.sum().item() <= 1e-5 * off.numel(), (mode, off.sum().item())
        # rgb, weights, alpha, depth (near < far), depth (near == far: S copies of one sample, see test_render_rays_vs_oracle)
        lo = kind != EQUAL
        e_rgb, e_depth = (rgb - want[0]).abs().max(1).values, (depth - want[3]).abs()
        errs = [e_rgb[lo].max().item()] + [(got[k] - want[k]).abs().max().item() for k in (2, 4)]
        errs += [e_depth[lo].max().item(), e_rgb[~lo].max().item(), e_depth[~lo].max().item()]
        print(f"\n[samples rt={rt} S={S} pad={pad}] mode {mode}: rgb {errs[0]:.3e} weights {errs[1]:.3e} "
              f"alpha {errs[2]:.3e} depth {errs[3]:.3e} (near == far {errs[4]:.3e}, {errs[5]:.3e}) "
              f"vs {'oracle' if tol[0] == RGB_TOL else 'emulation'}, flipped masks {off.sum().item()}", end="")
        assert errs[0] < tol[0] and errs[1] < tol[1] and errs[2] < tol[1] and errs[3] < tol[2], (mode, errs)
        if mode in (lib.MLP_FP32, lib.MLP_TC_SPLIT):
            assert errs[4] < tol[0] and errs[5] < tol[2], (mode, errs)


# ------------------------------------------------------------------------------------------------------------------
# early ray termination: the group verdict
# ------------------------------------------------------------------------------------------------------------------
def _n_tiles(n, S, rt):
    sp = 64 // rt
    return ((n + rt - 1) // rt) * ((S + sp - 1) // sp)


@pytest.mark.parametrize("mode", TC_MODES)
def test_t_stop_zero_is_bit_identical(plane, mode):
    for rt, S, white, lindisp in ((4, 33, False, True), (8, 200, True, False), (16, 24, True, True), (32, 128, False, False)):
        n = n_for(rt)
        rays = mixed_rays(plane.sc, n, seed=rt + S)[0].to(DEV)
        rgb0, depth0 = plane.render(rays, mode, S, white, lindisp)
        rgb, depth, tiles = plane.counted(rays, mode, S, white=white, lindisp=lindisp, t_stop=0.0)
        key = (rt, S, white, lindisp)
        assert torch.equal(rgb, rgb0), (key, (rgb - rgb0).abs().max().item())
        assert torch.equal(depth, depth0), key
        assert tiles == _n_tiles(n, S, rt), key


def _stop_tiles(alpha, rt, S, eps):
    """tiles computed per group, from the full render's alpha: the kernel's transmittance recurrence in fp32, a group
    stops after tile k once every ray of it has T < eps (rays past the batch end count as stopped), and computes tiles
    k + 1 and k + 2 still"""
    n = alpha.shape[0]
    sp, nt, G = 64 // rt, (S + 64 // rt - 1) // (64 // rt), (n + rt - 1) // rt
    T = torch.ones(n, device=alpha.device)
    stopped = torch.zeros(G, dtype=torch.bool, device=alpha.device)
    tiles = torch.full((G,), nt, dtype=torch.int64, device=alpha.device)
    for k in range(nt):
        for s in range(k * sp, min((k + 1) * sp, S)):
            T = T * ((1.0 - alpha[:, s]) + 1e-10)
        below = torch.ones(G * rt, dtype=torch.bool, device=alpha.device)
        below[:n] = T < eps
        verdict = below.view(G, rt).all(1) & ~stopped
        tiles[verdict] = min(k + 3, nt)
        stopped |= verdict
    return tiles


@pytest.mark.parametrize("white,lindisp", [(False, False), (True, True)])
@pytest.mark.parametrize("mode", TC_MODES)
def test_t_stop_follows_the_group_alpha(plane, mode, white, lindisp):
    """Each group's tile count follows from the full render's alpha, replayed on the host; each pixel is bit-identical to
    the full render of its first (computed tiles x samples per tile) samples through the same entry with a prefix of
    t_steps; the signed bounds against the full render hold.  Few groups of a mixed batch become opaque as a whole (a
    narrow or near == far ray in front of the plane keeps its group going), so t_stop = 0.5 joins 1e-4 and 1e-2 to
    make most groups stop early."""
    for rt, S in ((4, 128), (8, 200)):
        n = n_for(rt)
        rays = mixed_rays(plane.sc, n, seed=31 * rt + S)[0].to(DEV)
        sp = 64 // rt
        t_steps = backend._tsteps_of(S, torch.device(DEV))
        alpha = torch.empty(n, S, device=DEV)
        rgb0, depth0 = plane.raw(rays, mode, t_steps, white, lindisp, alpha=alpha)
        zmax = float(rays[:, 7].max())
        ulp = 4e-7
        for eps in (1e-4, 1e-2, 0.5):
            tiles = _stop_tiles(alpha, rt, S, eps)
            rgb, depth, done = plane.counted(rays, mode, S, white=white, lindisp=lindisp, t_stop=eps)
            key = (rt, S, eps)
            print(f"\n[t_stop mode {mode} white={white} lindisp={lindisp} rt={rt} S={S} eps={eps}] tiles {done} of "
                  f"{_n_tiles(n, S, rt)}", end="")
            assert done == int(tiles.sum().item()), (key, done, int(tiles.sum().item()))
            if eps == 0.5:                                               # groups do stop, for this test to mean anything
                assert done < 0.9 * _n_tiles(n, S, rt), key
            per_ray = tiles.repeat_interleave(rt)[:n]
            for L in per_ray.unique().tolist():
                sel = (per_ray == L).nonzero().squeeze(1)
                rgb_p, depth_p = plane.raw(rays[sel].contiguous(), mode, t_steps[:min(L * sp, S)].contiguous(), white,
                                           lindisp)
                assert torch.equal(rgb[sel], rgb_p), (key, L, (rgb[sel] - rgb_p).abs().max().item())
                assert torch.equal(depth[sel], depth_p), (key, L)
            d = rgb - rgb0
            if white:
                assert d.min().item() >= -ulp and d.max().item() < eps + ulp, (key, d.min().item(), d.max().item())
            else:
                assert d.min().item() > -eps - ulp and d.max().item() <= ulp, (key, d.min().item(), d.max().item())
            dd = depth0 - depth
            assert dd.min().item() >= -4 * ulp * zmax and dd.max().item() < (eps + 4 * ulp) * zmax, key


# ------------------------------------------------------------------------------------------------------------------
# empty-space skipping: the group ranges
# ------------------------------------------------------------------------------------------------------------------
def _kernel_ranges(n):
    """the range table the last render_rays(occupancy=) call left in its workspace"""
    rt = oh.rays_per_tile(n, _sms())
    G = (n + rt - 1) // rt
    ws = backend._occ_workspace[torch.device(DEV, torch.cuda.current_device())]
    return ws[:G * 8].view(torch.int32).view(G, 2).cpu().numpy().astype(np.int64), rt


def _host_occupied(ctx, rays, cells, S, lindisp):
    """per sample (host march over each ray's own near / far, NDC with the scene's near_far, fp32): occupied, and
    ambiguous (within 1e-5 of a cell face or the volume's boundary, where the kernel's NDC may round to the other side)"""
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


def _filled(occ, value):
    return backend.Occupancy(torch.full_like(occ.bits, value), occ.D, occ.Hp, occ.Wp, occ.near_far, occ.pad, occ.lindisp,
                             occ.dilate)


@pytest.mark.parametrize("lindisp", [False, True])
@pytest.mark.parametrize("mode", TC_MODES)
@pytest.mark.parametrize("scene", ["plane", "sparse"])
def test_occupancy_ranges_against_host(request, scene, mode, lindisp):
    ctx = request.getfixturevalue(scene)
    occ = ctx.occ(lindisp)
    cells = occ.cells().cpu().numpy()
    for (rt, S), kind_p in itertools.product(((4, 200), (8, 33), (16, 128), (32, 24)), (KIND_P, INSIDE_P)):
        n = n_for(rt)
        rays = mixed_rays(ctx.sc, n, seed=rt * S, kind_p=kind_p)[0].to(DEV)
        _, _, tiles = ctx.counted(rays, mode, S, lindisp=lindisp, occupancy=occ)
        got, rt_k = _kernel_ranges(n)
        assert rt_k == rt
        occupied, amb = _host_occupied(ctx, rays, cells, S, lindisp)
        lo, hi = oh.group_ranges(occupied & ~amb, rt), oh.group_ranges(occupied | amb, rt)
        key = (rt, S, kind_p)
        assert (hi[:, 0] <= got[:, 0]).all() and (got[:, 0] <= lo[:, 0]).all(), key
        assert (lo[:, 1] <= got[:, 1]).all() and (got[:, 1] <= hi[:, 1]).all(), key
        assert tiles == int(np.maximum(got[:, 1] - got[:, 0] + 1, 0).sum()), key
        print(f"\n[occupancy ranges mode {mode} lindisp={lindisp} rt={rt} S={S} kinds {kind_p}] tiles {tiles} of {_n_tiles(n, S, rt)}, "
              f"ambiguous samples {amb.mean():.2e}", end="")


@pytest.mark.parametrize("mode", TC_MODES)
def test_occupancy_all_ones_is_stop(plane, mode):
    for lindisp in (False, True):
        ones = _filled(plane.occ(lindisp), -1)
        for rt, S, white in ((4, 24, True), (16, 200, False), (32, 33, True)):
            n = n_for(rt)
            rays = mixed_rays(plane.sc, n, seed=5 * rt + S)[0].to(DEV)
            for eps in (0.0, 1e-4):
                a = plane.counted(rays, mode, S, white=white, lindisp=lindisp, t_stop=eps)
                b = plane.counted(rays, mode, S, white=white, lindisp=lindisp, t_stop=eps, occupancy=ones)
                key = (lindisp, rt, S, white, eps)
                assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), key
                assert a[2] == b[2], key


@pytest.mark.parametrize("white", [False, True])
@pytest.mark.parametrize("mode", TC_MODES)
def test_occupancy_skip_bound(sparse, mode, white):
    ctx = sparse
    """every pixel within the bound of its group's skipped samples (from the full render's alpha), and bit-identical
    wherever those samples all have alpha == 0.  Few tiles are skipped at this resolution (the grid of a 24 x 32
    feature map is mostly occupied once dilated); test_gpu_occupancy.py's 512 x 640 plane scene skips many."""
    occ = ctx.occ()
    for rt, S in ((4, 128), (8, 200)):
        n = n_for(rt)
        rays = mixed_rays(ctx.sc, n, seed=3 * rt + S, kind_p=INSIDE_P)[0].to(DEV)
        t_steps = backend._tsteps_of(S, torch.device(DEV))
        alpha = torch.empty(n, S, device=DEV)
        rgb0, depth0 = ctx.raw(rays, mode, t_steps, white, alpha=alpha)
        rgb, depth, tiles = ctx.counted(rays, mode, S, white=white, occupancy=occ)
        got, _ = _kernel_ranges(n)
        alpha = alpha.double()
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
        assert (d <= bound).all(), (rt, S, (d - bound).max().item())
        exact = (torch.where(kept, torch.zeros_like(alpha), alpha) == 0).all(1)
        same = (rgb == rgb0).all(1) & (depth == depth0)
        assert same[exact].all(), (rt, S, int((~same[exact]).sum()))
        assert tiles == int(np.maximum(got[:, 1] - got[:, 0] + 1, 0).sum())
        print(f"\n[occupancy bound mode {mode} white={white} rt={rt} S={S}] tiles {tiles} of {_n_tiles(n, S, rt)}, "
              f"exact {exact.float().mean():.3f}, bit-identical {same.float().mean():.3f}, max |drgb| {d.max():.3e}", end="")


# ------------------------------------------------------------------------------------------------------------------
# fine-tuning
# ------------------------------------------------------------------------------------------------------------------
def _host_march(sc, rays, S, j):
    """ray_marcher (data/ray_utils.py:152-197) over each ray's own near / far, with the uniform draw replaced by `j`, on
    the device: the points and depths the backward kernel marches itself"""
    near, far = rays[:, 6:7], rays[:, 7:8]
    t = torch.linspace(0, 1, S, device=DEV)
    z = (near * (1 - t) + far * t).expand(rays.shape[0], S)
    mid = 0.5 * (z[:, :-1] + z[:, 1:])
    upper = torch.cat([mid, z[:, -1:]], -1)
    lower = torch.cat([z[:, :1], mid], -1)
    z = lower + (upper - lower) * j
    pts = rays[:, None, 0:3] + rays[:, None, 3:6] * z[..., None]
    return pts.contiguous(), z.contiguous()


def _kernel_order_ndc(sc, pts):
    """get_ndc_coordinate (no lindisp, the scene's near_far) in the kernel's operation order (ndc_of_point): fmaf
    chains, each fma formed exactly in float64 and rounded once to float32, then IEEE float32 divisions (as
    tests/test_gpu_backward_rays.py states it)"""
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


def _cotangents(n, S, seed):
    g = torch.Generator().manual_seed(seed)
    return {"rgb": torch.randn(n, 3, generator=g), "depth": 0.1 * torch.randn(n, generator=g),
            "weights": 0.05 * torch.randn(n, S, generator=g), "alpha": 0.05 * torch.randn(n, S, generator=g),
            "input_feat": 0.01 * torch.randn(n, S, 20, generator=g)}


def _rel(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def _bwd_rays(ctx, rays, S, white, grad_mode, j, **kw):
    return backend.render_backward_rays(rays, ctx.vol, ctx.d.imgs_raw, ctx.d.pose_source, ctx.fn, ctx.sc.near_far,
                                        float(ctx.sc.pad), N_samples=S, jitter=j, white_bkgd=white, want_forward=True,
                                        grad_mode=grad_mode, **kw)


def _bwd_samples(ctx, rays, pts, ndc, z, white, grad_mode, **kw):
    return backend.render_backward(ctx.d.pose_source, pts, ndc, z, rays[:, 3:6].contiguous(), ctx.vol, ctx.d.imgs_raw,
                                   ctx.fn, white, want_forward=True, grad_mode=grad_mode, **kw)


# (S, n, white): 4, 2 (+ 32 idle rows) and 1 ray per backward tile
BWD_CASES = [(32, 390, True), (48, 133, False), (128, 200, True)]


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("grad_mode", GRAD_MODES)
def test_backward_rays_matches_host_march(scenes, grad_mode, det):
    """render_backward_rays with jitter against the samples-entry backward on the same jitter marched on the host (with
    the NDC in the kernel's operation order): the forward and the MLP gradients bit for bit, the loss and the volume
    gradient bit for bit when deterministic and to the float atomics' rounding otherwise"""
    ctx = scenes[24]
    for S, n, white in BWD_CASES:
        rays = mixed_rays(ctx.sc, n, seed=S + n)[0].to(DEV)
        j = torch.rand(n, S, generator=torch.Generator().manual_seed(S)).to(DEV)
        pts, z = _host_march(ctx.sc, rays, S, j)
        ndc = _kernel_order_ndc(ctx.sc, pts)
        target = torch.rand(n, 3, generator=torch.Generator().manual_seed(n)).to(DEV)
        loss_r, loss_s = torch.zeros(1, device=DEV), torch.zeros(1, device=DEV)
        with _deterministic(det):
            g_r, v_r, rgb_r, depth_r = _bwd_rays(ctx, rays, S, white, grad_mode, j, target_rgb=target, loss_out=loss_r)
            g_s, v_s, rgb_s, depth_s = _bwd_samples(ctx, rays, pts, ndc, z, white, grad_mode, target_rgb=target,
                                                    loss_out=loss_s)
        e_rgb, e_depth = (rgb_r - rgb_s).abs().max().item(), (depth_r - depth_s).abs().max().item()
        e_l = abs(loss_r.item() - loss_s.item()) / loss_s.item()
        worst = max(_rel(a, b) for a, b in zip(g_r, g_s))
        e_v = _rel(v_r, v_s)
        print(f"\n[rays vs host march {grad_mode} det={det} S={S} n={n}] rgb {e_rgb:.3e} depth {e_depth:.3e} loss {e_l:.3e} "
              f"mlp {worst:.3e} vol {e_v:.3e}", end="")
        assert torch.equal(rgb_r, rgb_s) and torch.equal(depth_r, depth_s), (S, e_rgb, e_depth)
        assert all(torch.equal(a, b) for a, b in zip(g_r, g_s)), (S, worst)        # private accumulators in both
        if det:                                                                      # the float atomics are not reproducible
            assert torch.equal(loss_r, loss_s) and torch.equal(v_r, v_s), (S, e_l, e_v)
        assert e_l <= 1e-6 and e_v < 1e-6, (S, e_l, e_v)


def _oracle_grads(ctx, weights, pts, ndc, z, rays, cot, white, mlp_fn=None):
    """(MLP gradients by name, volume gradient [1,8,D,H,W]) of the oracle's autograd on the CPU"""
    sc = ctx.sc
    wt = {k: v.clone().requires_grad_(k.startswith("mlp/")) for k, v in weights.items()}
    vt = ctx.vol.detach().cpu().contiguous().requires_grad_(True)
    rgb, feat, w, depth, alpha = orc.render_samples(pts.cpu(), ndc.cpu(), z.cpu(), rays[:, 3:6].cpu(), vt, sc.imgs_raw,
                                                    sc.pose_source, wt, white_bkgd=white, mlp_fn=mlp_fn)
    ((rgb * cot["rgb"]).sum() + (depth * cot["depth"]).sum() + (w * cot["weights"]).sum() + (alpha * cot["alpha"]).sum() +
     (feat * cot["input_feat"]).sum()).backward()
    return {k[len("mlp/"):]: v.grad for k, v in wt.items() if v.grad is not None}, vt.grad


def _excess(ctx, g_k, v_k, ref, gate):
    """max over tensors of err - gate * max|g_ref| - 1e-8 (<= 0 passes), and the worst relative error"""
    ref_p, ref_v = ref
    pairs = [(g.cpu(), ref_p[name]) for (name, _), g in zip(backend._ordered_named_params(ctx.fn), g_k)]
    pairs.append((v_k.permute(3, 0, 1, 2).unsqueeze(0).cpu(), ref_v))
    for a, _ in pairs:
        assert torch.isfinite(a).all()
    return (max((a - b).abs().max().item() - gate * b.abs().max().item() - 1e-8 for a, b in pairs),
            max(_rel(a, b) for a, b in pairs))


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("grad_mode", GRAD_MODES)
def test_backward_rays_vs_oracle_autograd(scenes, weights, grad_mode, det):
    """Random cotangents on all five outputs; the oracle's fp32 autograd on the host-marched samples (FP32 at 2e-4 of
    max|g|, TC_HALF at 3e-3) and, for TC_HALF, the emulation of its gradient arithmetic at 2e-4."""
    ctx = scenes[0]
    for S, n, white in BWD_CASES:
        rays = mixed_rays(ctx.sc, n, seed=3 * S + n)[0].to(DEV)
        j = torch.rand(n, S, generator=torch.Generator().manual_seed(S + 1)).to(DEV)
        pts, z = _host_march(ctx.sc, rays, S, j)
        ndc = _kernel_order_ndc(ctx.sc, pts)
        cot = _cotangents(n, S, seed=n)
        with _deterministic(det):
            g_k, v_k, _, _ = _bwd_rays(ctx, rays, S, white, grad_mode, j, grads={k: v.to(DEV) for k, v in cot.items()})
        x32, r32 = _excess(ctx, g_k, v_k, _oracle_grads(ctx, weights, pts, ndc, z, rays, cot, white), GRAD_GATE[grad_mode])
        msg = f"\n[rays backward {grad_mode} det={det} S={S} n={n}] vs oracle {r32:.3e}"
        if grad_mode == lib.MLP_TC_HALF:
            xe, re = _excess(ctx, g_k, v_k, _oracle_grads(ctx, weights, pts, ndc, z, rays, cot, white, mlp_grad_emulated),
                             GRAD_EMU_GATE)
            msg += f" vs emulation {re:.3e}"
            assert xe <= 0, (S, xe)
        print(msg, end="")
        assert x32 <= 0, (S, x32)


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


@pytest.mark.parametrize("t_stop", [1e-4, 1e-2])
def test_t_stop_backward_live_samples_follow_the_rule(plane, t_stop):
    """each ray's live count follows from its own alpha (render_rays, MLP_FP32), whatever the other rays of its tile"""
    for S, n in ((32, 390), (64, 131), (128, 200)):
        rays = mixed_rays(plane.sc, n, seed=S * n)[0].to(DEV)
        alpha = torch.empty(n, S, device=DEV)
        plane.raw(rays, lib.MLP_FP32, torch.linspace(0, 1, S, device=DEV), alpha=alpha)
        want = _live_of(alpha, t_stop)
        assert (want >= 1).all() and (want < S).any() and (want == S).any()
        for mode in GRAD_MODES:
            live = torch.full((n,), -1, dtype=torch.int32, device=DEV)
            tiles = torch.zeros(3, dtype=torch.int64, device=DEV)
            _bwd_rays(plane, rays, S, False, mode, None, target_rgb=torch.zeros(n, 3, device=DEV), t_stop=t_stop,
                      live_samples=live, tiles_done=tiles)
            assert torch.equal(live, want), (S, mode, int((live != want).sum()))


@pytest.mark.parametrize("grad_mode", GRAD_MODES)
def test_step_rays_tracks_autograd_adam(scenes, grad_mode):
    """20 FineTuner.step_rays steps on mixed batches against `rendering` under autograd + torch.optim.Adam on the same
    jitter marched on the host: the loss sequences agree at test_finetuner_trains_and_tracks_torch_adam's tolerance and
    go down"""
    ctx = scenes[0]
    sc, d = ctx.sc, ctx.d
    n, S = 256, 64

    class Args:
        use_color_volume = False
    fn_a, fn_b = _net(), _net()
    vol_a, vol_b = backend.RefVolume(ctx.vol.clone()), backend.RefVolume(ctx.vol.clone())
    tuner = backend.FineTuner(fn_a, vol_a, d.imgs_raw, d.pose_source, lr=5e-4, grad_mode=grad_mode)
    opt = torch.optim.Adam(list(fn_b.parameters()) + list(vol_b.parameters()), lr=5e-4, betas=(0.9, 0.999))
    gen_a, gen_b = torch.Generator(device=DEV).manual_seed(3), torch.Generator(device=DEV).manual_seed(3)
    target = torch.full((n, 3), 0.3, device=DEV)
    la, lb = [], []
    for it in range(20):
        rays = mixed_rays(sc, n, seed=500 + it)[0].to(DEV)
        la.append(tuner.step_rays(rays, target, sc.near_far, float(sc.pad), N_samples=S, perturb=1.0,
                                  generator=gen_a)[0].item())
        j = torch.rand((n, S), device=DEV, generator=gen_b)
        pts, z = _host_march(sc, rays, S, j)
        rgb = backend.rendering(Args(), d.pose_source, pts, _kernel_order_ndc(sc, pts), z, None, rays[:, 3:6].contiguous(),
                                volume_feature=vol_b, imgs=d.imgs_raw, network_fn=fn_b, mlp_mode=lib.MLP_FP32,
                                grad_mode=grad_mode)[0]
        loss = ((rgb - target) ** 2).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        lb.append(loss.item())
    rel = max(abs(a - b) / max(a, b) for a, b in zip(la, lb))
    print(f"\n[step_rays vs autograd + Adam {grad_mode}] first {la[0]:.6e} / {lb[0]:.6e} last {la[-1]:.6e} / {lb[-1]:.6e} "
          f"max rel {rel:.3e}", end="")
    for a, b in zip(la, lb):
        assert abs(a - b) <= 2e-3 * max(a, b) + 1e-6, (la, lb)
    assert np.mean(la[-5:]) < np.mean(la[:5]), la
