"""GPU: the tensor-core MLP modes (csrc/render_wg.cu) and conv0 on wgmma (csrc/conv0_tc.cu) beyond the shipped checkpoint
and the synthetic scenes' usual range: scaled encoding volumes, drifted and random weights, every tile geometry of the
render kernel, the packed weight image bit for bit, and cost volumes up to |cost| ~ 1e4.

References: the fp32 oracle (oracle.mvsnerf_oracle.mlp) for MLP_FP32 and MLP_TC_SPLIT (gate 1e-4), and
oracle.mlp_emulated(..., "half") -- the fp16 mode's own operand rounding -- for MLP_TC_PAIR, so that an error of a few
1e-4 in the fp16 kernel is not lost under the 5e-3 gate that mode has against fp32."""
import functools
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import mvsnerf_oracle as orc
from mvsnerf_b200 import backend, lib, synthetic

pytestmark = pytest.mark.gpu
DEV = "cuda"
WPATH = os.path.join(GOLDEN, "mvsnerf_v0_weights.npz")

RGB_TOL, DEPTH_TOL = 1e-4, 1e-3          # fp32 and split modes vs the fp32 oracle
PAIR_TOL, PAIR_DEPTH_TOL = 5e-3, 2e-2    # fp16 mode vs the fp32 oracle
# fp16 mode vs its emulation: the kernel's fast sin / cos / exp and fp32 accumulation order against exact arithmetic on
# the same fp16 operands.  Measured on an H100 80GB HBM3 (400 W), RGB L-inf: at most 2.1e-4 over the x1 volume, the random
# weights and every tile geometry; per-sample alpha / weights of the signature path 4.8e-4, depth 5.9e-4.  Larger activations
# amplify a flipped fp16 rounding: 8.1e-4 (volume x1.5), 8.8e-4 (x2), 3.3e-3 (x3), 5.1e-3 (trunk x1.5).  Gates are
# at most 4x the largest error seen in their group.  Rounding the activations toward zero instead of to nearest gives
# 1.2e-3 at x1, a bias read one column off for one hidden unit 6.2e-3: the first passes the 5e-3 gate against fp32.
PAIR_EMU_TOL = 8e-4
PAIR_EMU_SAMPLE_TOL = 1.6e-3             # per-sample alpha / weights
PAIR_EMU_DEPTH_TOL = 2.4e-3
MASK_COLS = [11, 15, 19]                 # input_feat: the strict in-bounds mask of each source view
HALF = functools.partial(orc.mlp_emulated, mode="half")


def _net(w):
    fn = backend.MVSNeRF().to(DEV)
    fn.load_state_dict({k[len("mlp/"):]: v for k, v in w.items() if k.startswith("mlp/")})
    return fn


@pytest.fixture(scope="module")
def scene(weights):
    sc = synthetic.make_scene(128, 160, pad=8, seed=5)
    vol = orc.encode_volume(sc.imgs_norm, sc.proj_mats, sc.near_far, sc.pad, weights)
    return sc, vol


def _rays(sc, n, seed):
    rays = synthetic.scene_rays(sc)
    g = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, rays.shape[0], (n,), generator=g) if n > rays.shape[0] else torch.randperm(rays.shape[0], generator=g)[:n]
    return rays[idx].contiguous()


def _check_modes(sc, vol, w, rays, S, pair_vs_oracle=True, emu_tol=PAIR_EMU_TOL):
    """FP32, TC_SPLIT and TC_PAIR through render_rays against the oracle and the fp16 emulation; returns the TC_PAIR
    error against the emulation."""
    args = (sc.imgs_raw, sc.pose_source, w, sc.H, sc.W, sc.near_far, float(sc.pad))
    rgb_ref, depth_ref = orc.render_rays(rays, vol, *args, n_samples=S)
    rgb_emu, _ = orc.render_rays(rays, vol, *args, n_samples=S, mlp_fn=HALF)
    fn, d = _net(w), sc.to(DEV)
    out = {}
    for name, mode in (("fp32", lib.MLP_FP32), ("split", lib.MLP_TC_SPLIT), ("pair", lib.MLP_TC_PAIR)):
        rgb, depth = backend.render_rays(rays.to(DEV), vol.to(DEV), d.imgs_raw, d.pose_source, fn, sc.near_far,
                                         float(sc.pad), N_samples=S, mlp_mode=mode)
        rgb, depth = rgb.cpu(), depth.cpu()
        assert torch.isfinite(rgb).all() and torch.isfinite(depth).all(), name
        out[name] = (rgb, depth)
    for name in ("fp32", "split"):
        rgb, depth = out[name]
        e = (rgb - rgb_ref).abs().max().item()
        assert e < RGB_TOL, (name, e)
        assert (depth - depth_ref).abs().max().item() < DEPTH_TOL, name
    rgb, depth = out["pair"]
    e_emu = (rgb - rgb_emu).abs().max().item()
    print(f"pair vs emulation {e_emu:.3e}  vs fp32 {(rgb - rgb_ref).abs().max().item():.3e}")
    assert e_emu < emu_tol, e_emu
    if pair_vs_oracle:
        assert (rgb - rgb_ref).abs().max().item() < PAIR_TOL
        assert (depth - depth_ref).abs().max().item() < PAIR_DEPTH_TOL
    return e_emu


# ------------------------------------------------------------------------------------------------------------------
# dynamic range: hidden activations from ~1e2 (x1) to ~1e5 (volume x3)
# ------------------------------------------------------------------------------------------------------------------
def _trunk_scaled(w, k):
    w = dict(w)
    for key in [f"mlp/nerf.pts_linears.{i}.weight" for i in range(6)] + ["mlp/nerf.pts_bias.weight"]:
        w[key] = w[key] * k
    return w


@pytest.mark.parametrize("vol_scale,trunk_scale,emu_tol", [(1.0, 1.0, PAIR_EMU_TOL), (1.5, 1.0, 3.5e-3), (2.0, 1.0, 3.5e-3),
                                                           (3.0, 1.0, 2e-2), (1.0, 1.5, 2e-2)])
def test_dynamic_range(scene, weights, vol_scale, trunk_scale, emu_tol):
    """Layer-5 activations peak at ~1e2, 1.3e3, 8.1e3, 1.0e5 and 1.5e4.  Beyond 4095 the split mode's old fixed x16
    activation scale overflowed fp16 into inf - inf = NaN.  The fp16 mode saturates: it stays finite and matches its
    emulation everywhere, and leaves the 5e-3 gate against fp32 at x3 and trunk x1.5 (1.1e-2, 1.6e-2: fp16 precision,
    DESIGN.md section 5)."""
    sc, vol = scene
    w = _trunk_scaled(weights, trunk_scale) if trunk_scale != 1.0 else weights
    _check_modes(sc, vol * vol_scale, w, _rays(sc, 2048, 128 * 1000 + 2048), 128,
                 pair_vs_oracle=vol_scale <= 2.0 and trunk_scale == 1.0, emu_tol=emu_tol)


# ------------------------------------------------------------------------------------------------------------------
# arbitrary weights: every input column and hidden unit carries signal
# ------------------------------------------------------------------------------------------------------------------
def _random_weights(seed, trunk_scale):
    torch.manual_seed(seed)
    net = backend.MVSNeRF()                              # nn.Linear default init
    w = {"mlp/" + k: v.detach().clone() for k, v in net.state_dict().items()}
    if trunk_scale != 1.0:
        for i in range(6):
            w[f"mlp/nerf.pts_linears.{i}.weight"] *= trunk_scale
    return w


@pytest.mark.parametrize("trunk_scale", [1.0, 3.0])
def test_random_weights(scene, trunk_scale):
    """Default init gives small activations (the fp16 subnormal end); x3 on the trunk gives large ones."""
    sc, vol = scene
    _check_modes(sc, vol, _random_weights(7, trunk_scale), _rays(sc, 1024, 77), 128)


# ------------------------------------------------------------------------------------------------------------------
# tile geometries: 4, 8, 16 or 32 rays per 64-sample tile
# ------------------------------------------------------------------------------------------------------------------
NWG = 2                                   # MMA warpgroups per CTA (csrc/render_wg.cu, wg::NWG)


def rays_per_tile(n, sms):
    """Mirrors the selection loop of launch_render_wg (csrc/render_wg.cu): 32 rays per tile unless that leaves a
    warpgroup of some SM without a ray group."""
    rt = 32
    while rt > 4 and (n + rt - 1) // rt < NWG * sms:
        rt >>= 1
    return rt


def _tile_cases():
    """(rt, N, S).  N = rt (2 sms + 1) - 1: an odd number of ray groups (one consumer idles in the last pass) and
    sms + 1 units of work, so CTA 0 makes two passes.  N = 2 rt (2 sms - 1): the top of the rt band, most CTAs make two
    passes with both consumers busy."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    odd = {rt: rt * (2 * sms + 1) - 1 for rt in (4, 8, 16, 32)}
    cases = [(rt, odd[rt], 128) for rt in (4, 8, 16, 32)]
    cases += [(rt, 2 * rt * (2 * sms - 1), 128) for rt in (8, 16)]
    cases += [(8, odd[8], 24), (16, odd[16], 200), (32, odd[32], 24), (4, odd[4], 200)]
    for rt, n, _ in cases:
        assert rays_per_tile(n, sms) == rt, (rt, n, sms)
    return cases


@pytest.fixture(scope="module")
def tile_cases():
    return _tile_cases()


@pytest.mark.parametrize("i", range(10))
def test_tile_geometry_fused(scene, weights, tile_cases, i):
    rt, n, S = tile_cases[i]
    sc, vol = scene
    _check_modes(sc, vol, weights, _rays(sc, n, 1000 * rt + S), S)


@pytest.mark.parametrize("i", [1, 2, 4, 6, 7])
def test_tile_geometry_signature_path(scene, weights, tile_cases, i):
    """`rendering` with perturb=1 z values: rgb, depth, alpha, weights and every row of input_feat."""
    class Args:
        use_color_volume = False
    rt, n, S = tile_cases[i]
    sc, vol = scene
    rays = _rays(sc, n, 1000 * rt + S + 1)
    g = torch.Generator().manual_seed(n)
    pts, z = orc.march_rays(rays, S)
    mid = 0.5 * (z[:, :-1] + z[:, 1:])
    lower, upper = torch.cat([z[:, :1], mid], -1), torch.cat([mid, z[:, -1:]], -1)
    z = lower + (upper - lower) * torch.rand(z.shape, generator=g)
    pts = rays[:, None, :3] + rays[:, None, 3:6] * z[..., None]
    ndc = orc.ndc_coords(sc.pose_source["w2cs"][0], sc.pose_source["intrinsics"][0], pts, sc.H, sc.W,
                         sc.near_far[0], sc.near_far[1], float(sc.pad))
    ref = orc.render_samples(pts, ndc, z, rays[:, 3:6], vol, sc.imgs_raw, sc.pose_source, weights)   # rgb, feat, wts, depth, alpha
    dirs = orc.view_direction(rays[:, 3:6], sc.pose_source["w2cs"][0])[:, None].expand(-1, S, -1)
    fn, d = _net(weights), sc.to(DEV)
    for mode in (lib.MLP_TC_SPLIT, lib.MLP_TC_PAIR):
        rgb, feat, wts, depth, alpha, _ = backend.rendering(
            Args, d.pose_source, pts.to(DEV), ndc.to(DEV), z.to(DEV), rays[:, :3].to(DEV), rays[:, 3:6].to(DEV),
            vol.to(DEV), d.imgs_raw, network_fn=fn, mlp_mode=mode)
        got = [t.cpu() for t in (rgb, feat, wts, depth, alpha)]
        assert all(torch.isfinite(t).all() for t in got), mode
        if mode == lib.MLP_TC_SPLIT:
            want, tol = ref, (RGB_TOL, RGB_TOL, DEPTH_TOL)
        else:
            # the fp16 emulation on the kernel's own input_feat, so that a flipped border mask (below) is not counted twice
            raw = orc.mlp_emulated(torch.cat([orc.positional_encoding(ndc), got[1], dirs], -1), weights, "half")
            e_rgb, e_depth, e_wts, e_alpha = orc.composite(raw, z)
            want, tol = (e_rgb, ref[1], e_wts, e_depth, e_alpha), (PAIR_EMU_TOL, PAIR_EMU_SAMPLE_TOL, PAIR_EMU_DEPTH_TOL)
        # input_feat, every row: the gather is fp32 in every mode.  The fp16 front end projects with MUFU reciprocals, so
        # a sample on a view's border may flip that view's strict in-bounds mask, and nothing else.
        off = (got[1] - want[1]).abs() > 1e-4
        mask = torch.zeros(20, dtype=torch.bool)
        mask[MASK_COLS] = True
        assert not (off & ~mask).any(), mode
        assert not off.any() if mode == lib.MLP_TC_SPLIT else off.sum().item() <= 1e-5 * off.numel(), mode
        errs = [(got[k] - want[k]).abs().max().item() for k in (0, 2, 4, 3)]    # rgb, weights, alpha, depth
        print(f"signature path mode {mode}: rgb {errs[0]:.3e} weights {errs[1]:.3e} alpha {errs[2]:.3e} depth {errs[3]:.3e}")
        assert errs[0] < tol[0] and errs[1] < tol[1] and errs[2] < tol[1] and errs[3] < tol[2], (mode, errs)


# ------------------------------------------------------------------------------------------------------------------
# the packed weight image, decoded on the host
# ------------------------------------------------------------------------------------------------------------------
NCHUNK, HALF_STRIDE = 17, 16384
BIAS_TRUNK, BIAS_HEAD, BIAS_RGB, BIAS_WINV, BIAS_WMAX, BIAS_FLOATS = 128, 896, 968, 1016, 1017, 1024


def chunk_rows(c):
    return 72 if 13 <= c <= 15 else 8 if c == 16 else 128


def _host_chunks(net):
    """The 17 B-operand chunks [rows, 64] fp32 and the fp32 bias tail, from the module's fp32 tensors (the layout of
    csrc/render_wg.cu: wg::chunk_rows, wg_weight, the bias tail of pack_mlp_wg_kernel)."""
    n = net.nerf
    W = [l.weight.detach().cpu().float() for l in n.pts_linears]
    V = n.views_linears[0].weight.detach().cpu().double()
    fold = (V[:, :128] @ n.feature_linear.weight.detach().cpu().double()).float()
    ch = [torch.zeros(chunk_rows(c), 64) for c in range(NCHUNK)]
    ch[0][:, :20] = n.pts_bias.weight.detach().cpu()
    ch[1][:, :63] = W[0]
    for l in range(1, 5):
        ch[2 * l][:], ch[2 * l + 1][:] = W[l][:, :64], W[l][:, 64:]
    ch[10][:, :63] = W[5][:, :63]
    ch[11][:], ch[12][:] = W[5][:, 63:127], W[5][:, 127:191]
    for kb in range(2):
        ch[13 + kb][:64] = fold[:, kb * 64:(kb + 1) * 64]
        ch[13 + kb][64] = n.alpha_linear.weight.detach().cpu()[0, kb * 64:(kb + 1) * 64]
    ch[15][:64, 32:35] = V[:, 128:].float()
    ch[16][:3] = n.rgb_linear.weight.detach().cpu()
    tail = torch.zeros(BIAS_FLOATS)
    tail[:128] = n.pts_bias.bias.detach().cpu()
    for l in range(6):
        tail[BIAS_TRUNK + 128 * l:BIAS_TRUNK + 128 * (l + 1)] = n.pts_linears[l].bias.detach().cpu()
    tail[BIAS_HEAD:BIAS_HEAD + 64] = (n.views_linears[0].bias.detach().cpu().double() +
                                      V[:, :128] @ n.feature_linear.bias.detach().cpu().double()).float()
    tail[BIAS_HEAD + 64] = n.alpha_linear.bias.detach().cpu()[0]
    tail[BIAS_RGB:BIAS_RGB + 3] = n.rgb_linear.bias.detach().cpu()
    return ch, tail


def _sw128_index(rows):
    """Element index (in fp16 units) of (r, k) in a SWIZZLE_128B tile of 64-wide fp16 rows."""
    r = np.arange(rows)[:, None]
    k = np.arange(64)[None, :]
    byte = (r >> 3) * 1024 + (r & 7) * 128 + ((((k >> 3) ^ (r & 7)) & 7) << 4) + (k & 7) * 2
    return byte // 2


def _decode(img, split):
    stride = (2 if split else 1) * HALF_STRIDE
    h = img[:NCHUNK * stride].view(np.float16)
    chunks = []
    for c in range(NCHUNK):
        base = c * stride // 2
        idx = _sw128_index(chunk_rows(c))
        hi = h[base + idx]
        lo = h[base + HALF_STRIDE // 2 + idx] if split else None
        chunks.append((hi, lo))
    tail = img[NCHUNK * stride:].view(np.float32)
    return chunks, tail


def _weight_nets():
    v0 = backend.MVSNeRF()
    backend.load_weights_npz(v0, None, WPATH)
    big = backend.MVSNeRF()
    big.load_state_dict({k[len("mlp/"):]: v for k, v in _random_weights(11, 1.0).items()})
    with torch.no_grad():
        big.nerf.pts_linears[2].weight[5, 7] = 300.0     # |w| >= 256: inf at a fixed x256 scale
        big.nerf.rgb_linear.weight[1, 3] = -1e-3
    return {"v0": v0, "random": _random_weights_net(3), "large": big}


def _random_weights_net(seed):
    net = backend.MVSNeRF()
    net.load_state_dict({k[len("mlp/"):]: v for k, v in _random_weights(seed, 1.0).items()})
    return net


@pytest.mark.parametrize("name", ["v0", "random", "large"])
@pytest.mark.parametrize("mode", [lib.MLP_TC_PAIR, lib.MLP_TC_SPLIT])
def test_weight_image_bit_exact(name, mode):
    net = _weight_nets()[name]
    ch, tail_want = _host_chunks(net)
    net = net.to(DEV)
    split = mode == lib.MLP_TC_SPLIT
    img = net.packed(mode).cpu().numpy()
    assert img.size == NCHUNK * (2 if split else 1) * HALF_STRIDE + 4 * BIAS_FLOATS
    chunks, tail = _decode(img, split)
    if split:
        wmax = max(c.abs().max().item() for c in ch)
        assert tail[BIAS_WMAX].view(np.uint32) == np.float32(wmax).view(np.uint32)
        sw = 2.0 ** min(8, 14 - (int(np.frexp(np.float32(wmax))[1]) - 1))
        assert tail[BIAS_WINV] == np.float32(1.0 / sw)
        assert (sw < 256) == (name == "large")
        tail_want[BIAS_WINV], tail_want[BIAS_WMAX] = 1.0 / sw, torch.tensor(tail[BIAS_WMAX])
    np.testing.assert_array_equal(tail, tail_want.numpy())
    for c, (hi, lo) in enumerate(chunks):
        v = ch[c]
        if not split:
            want_hi = v.half().numpy()
        else:
            a = v * sw
            want_hi = a.half()
            lo_want = (a - want_hi.float()).half().numpy()
            want_hi = want_hi.numpy()
            assert np.isfinite(lo).all(), c
            np.testing.assert_array_equal(lo.view(np.uint16), lo_want.view(np.uint16), err_msg=f"chunk {c} lo")
        assert np.isfinite(hi).all(), c
        np.testing.assert_array_equal(hi.view(np.uint16), want_hi.view(np.uint16), err_msg=f"chunk {c} hi")


def test_large_weight_renders_in_split_mode(scene):
    """The |w| = 300 image renders at fp32 grade (the split mode was inf - inf = NaN with it)."""
    sc, vol = scene
    net = _weight_nets()["large"]
    w = {"mlp/" + k: v.detach() for k, v in net.state_dict().items()}
    rays = _rays(sc, 512, 5)
    args = (sc.imgs_raw, sc.pose_source, w, sc.H, sc.W, sc.near_far, float(sc.pad))
    rgb_ref, depth_ref = orc.render_rays(rays, vol, *args, n_samples=64)
    d = sc.to(DEV)
    rgb, depth = backend.render_rays(rays.to(DEV), vol.to(DEV), d.imgs_raw, d.pose_source, net.to(DEV), sc.near_far,
                                     float(sc.pad), N_samples=64, mlp_mode=lib.MLP_TC_SPLIT)
    assert torch.isfinite(rgb).all()
    assert (rgb.cpu() - rgb_ref).abs().max().item() < RGB_TOL
    assert (depth.cpu() - depth_ref).abs().max().item() < DEPTH_TOL


# ------------------------------------------------------------------------------------------------------------------
# conv0 on wgmma at |cost| ~ 1e4
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("top", [30.0, 300.0, 3000.0])
def test_conv0_tensor_core_range(weights, top):
    """Channel scales up to `top` (|cost| up to ~4.5 top): the wgmma conv0 against the FFMA conv0 through the whole
    CostRegNet at 2e-5 of the volume's range, bit-identical from run to run, and against the oracle's cost_reg_net.
    BatchNorm after conv0 keeps the expected volume bounded, so a NaN or a wrong value shows directly."""
    L = lib.load()
    mvs = backend.MVSNet().to(DEV).train()
    backend.load_weights_npz(None, mvs, WPATH)
    D, Hp, Wp = 16, 24, 40
    g = torch.Generator().manual_seed(int(top))
    cost = (torch.randn(1, 41, D, Hp, Wp, generator=g) * torch.linspace(0.05, top, 41).view(1, 41, 1, 1, 1)).contiguous()
    cost_d = cost.to(DEV)
    wl = [w.detach().contiguous() for w in mvs.cost_reg_2.weight_list()]
    ws_bytes = L.mvsn_costreg_workspace_bytes(D, Hp, Wp)
    outs = []
    for flags in (lib.BN_BATCH, lib.BN_BATCH, lib.BN_BATCH | lib.CONV0_FFMA):
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
        vol = torch.empty(D, Hp, Wp, 8, device=DEV)
        lib.check(L.mvsn_costreg_forward_bn(lib.ptr_array(wl), None, flags, 0.0, lib.ptr(cost_d), D, Hp, Wp, lib.ptr(vol),
                                            lib.ptr(ws), ws_bytes, lib.stream_ptr()), "mvsn_costreg_forward_bn")
        outs.append(vol)
    assert cost.abs().max().item() > 4.0 * top
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0], outs[1])
    scale = outs[2].abs().max().item()
    assert (outs[0] - outs[2]).abs().max().item() <= 2e-5 * scale
    ref = orc.cost_reg_net(cost, weights)[0].permute(1, 2, 3, 0)
    e = (outs[0].cpu() - ref).abs().max().item()
    print(f"conv0 top {top}: |cost| {cost.abs().max().item():.3g}, vs oracle {e:.3e} of {ref.abs().max().item():.3g}")
    assert e <= 1e-4 * ref.abs().max().item(), e
