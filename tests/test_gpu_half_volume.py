"""GPU: rendering from an fp16 encoding volume (MVSN_VOLUME_F16) in the tensor-core modes.

  * bit-identity: every render entry and TC mode gives exactly the bits of the same render from the fp32 volume
    `vol.half().float()` -- the kernel widens each half exactly and keeps the fp32 path's FMA order -- across S,
    ragged and small N, lindisp, white_bkgd, pad 0 and 24, early ray termination, the per-sample outputs, the x3
    volume range, and values that round to inf or to fp16 subnormals (NaN compared equal to NaN);
  * layouts: a channels-last half tensor is read in place (no cache entry, no allocation), a planar one is converted
    once per tensor version, and the conversion kernel rounds exactly as Tensor.half();
  * modes that keep the fp32 upcast (MLP_FP32) are unchanged;
  * accuracy against the oracle at 512x640, pad 24, every pixel;
  * the encoder's fp16 output is .half() of its fp32 output and leaves the same BatchNorm running buffers.
"""
import copy
import ctypes as C
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
MODES = [lib.MLP_TC_PAIR, lib.MLP_TC_HALF, lib.MLP_TC_SPLIT]


class Args:
    feat_dim = 20
    img_downscale = 1.0
    use_color_volume = False
    net_type = "v0"


def same_bits(a, b):
    """bitwise equality, NaN equal to NaN (an inf in the volume can make NaN in the MLP)"""
    if a is None or b is None:
        return a is None and b is None
    assert a.dtype == b.dtype == torch.float32 and a.shape == b.shape
    eq = a.view(torch.int32) == b.view(torch.int32)
    return bool((eq | (torch.isnan(a) & torch.isnan(b))).all())


@pytest.fixture(scope="module")
def net():
    fn, mvs = backend.MVSNeRF().to(DEV), backend.MVSNet().to(DEV).train()
    backend.load_weights_npz(fn, mvs, WPATH)
    return fn, mvs


class Ctx:
    def __init__(self, sc, fn, mvs):
        self.sc, self.fn, self.d = sc, fn, sc.to(DEV)
        with torch.no_grad():
            vol, _, _ = mvs(self.d.imgs_norm, self.d.proj_mats, sc.near_far, pad=sc.pad)
        self.set_volume(vol)
        self.rays = synthetic.scene_rays(sc).to(DEV).contiguous()

    def set_volume(self, vol32):
        self.vol32 = vol32
        self.volh = vol32.half()              # channels-last, like the encoder's output
        self.volr = self.volh.float()         # the fp32 volume the half render must reproduce bit for bit

    def render(self, vol, rays, mode, S=128, white=False, lindisp=False, **kw):
        with torch.no_grad():
            return backend.render_rays(rays, vol, self.d.imgs_raw, self.d.pose_source, self.fn, self.sc.near_far,
                                       float(self.sc.pad), N_samples=S, white_bkgd=white, lindisp=lindisp, mlp_mode=mode,
                                       **kw)

    def samples(self, vol, rays, mode, S, white=False, lindisp=False):
        pts, z = orc.march_rays(rays, S, lindisp)
        ndc = orc.ndc_coords(self.d.pose_source["w2cs"][0], self.d.pose_source["intrinsics"][0], pts, self.sc.H,
                             self.sc.W, self.sc.near_far[0], self.sc.near_far[1], float(self.sc.pad), lindisp)
        with torch.no_grad():
            return backend.rendering(Args, self.d.pose_source, pts, ndc, z, rays[:, :3], rays[:, 3:6], vol,
                                     self.d.imgs_raw, network_fn=self.fn, white_bkgd=white, mlp_mode=mode)[:5]


@pytest.fixture(scope="module", params=[0, 24], ids=["pad0", "pad24"])
def small(net, request):
    return Ctx(synthetic.make_scene(96, 128, pad=request.param, seed=5), *net)


@pytest.fixture(scope="module")
def plane(net):
    return Ctx(synthetic.make_plane_scene(96, 128, pad=4, seed=1), *net)


CASES = ((8461, False, False), (8461, True, True), (300, True, False), (37, False, True))


@pytest.mark.parametrize("mode", MODES)
def test_rays_bit_identical(small, mode):
    """mvsn_render_rays: S of 24, 32, 48, 128 and 200; ragged and small N; white_bkgd and lindisp"""
    assert small.volh.dtype == torch.float16 and small.volh[0].permute(1, 2, 3, 0).is_contiguous()
    for S in (24, 32, 48, 128, 200):
        for n, white, lindisp in CASES:
            rays = small.rays[:n].contiguous()
            a = small.render(small.volh, rays, mode, S, white, lindisp)
            b = small.render(small.volr, rays, mode, S, white, lindisp)
            assert same_bits(a[0], b[0]) and same_bits(a[1], b[1]), (S, n, white, lindisp)


@pytest.mark.parametrize("mode", MODES)
def test_samples_bit_identical_all_outputs(small, mode):
    """mvsn_render_samples (rendering without grad): rgb, input_feat, weights, depth and alpha"""
    for S, (n, white, lindisp) in ((24, CASES[0]), (128, CASES[1]), (200, CASES[2]), (32, CASES[3])):
        rays = small.rays[:n].contiguous()
        a = small.samples(small.volh, rays, mode, S, white, lindisp)
        b = small.samples(small.volr, rays, mode, S, white, lindisp)
        for x, y, name in zip(a, b, ("rgb", "input_feat", "weights", "depth", "alpha")):
            assert same_bits(x, y), (S, n, name)
    # the volume features in input_feat are the fp32 volume's, exactly
    assert not same_bits(a[1], small.samples(small.vol32, rays, mode, S, white, lindisp)[1])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("eps", [0.0, 1e-4])
def test_stop_bit_identical(small, plane, mode, eps):
    """mvsn_render_rays_stop: same pixels and the same tiles_done"""
    for ctx in (small, plane):
        for n, white, lindisp in CASES[:3]:
            rays = ctx.rays[:n].contiguous()
            ta = torch.zeros(1, dtype=torch.int64, device=DEV)
            tb = torch.zeros(1, dtype=torch.int64, device=DEV)
            a = ctx.render(ctx.volh, rays, mode, 128, white, lindisp, t_stop=eps, tiles_done=ta)
            b = ctx.render(ctx.volr, rays, mode, 128, white, lindisp, t_stop=eps, tiles_done=tb)
            assert same_bits(a[0], b[0]) and same_bits(a[1], b[1]), (n, white, lindisp)
            assert int(ta.item()) == int(tb.item()) > 0
    if eps > 0:                                    # the plane scene does stop
        rays = plane.rays
        t = torch.zeros(1, dtype=torch.int64, device=DEV)
        plane.render(plane.volh, rays, mode, 128, t_stop=eps, tiles_done=t)
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        rt = 32
        while rt > 4 and (rays.shape[0] + rt - 1) // rt < 2 * sms:
            rt //= 2
        full = ((rays.shape[0] + rt - 1) // rt) * ((128 + 64 // rt - 1) // (64 // rt))
        assert int(t.item()) < full


@pytest.mark.parametrize("mode", MODES)
def test_peer_sink_bit_identical(small, mode):
    """mvsn_render_rays_to_peers: the frame texels"""
    rays = small.rays[:5000].contiguous()
    frames = []
    for vol in (small.volh, small.volr):
        f = torch.full((rays.shape[0] + 64, 4), -7.0, device=DEV)
        sink = lib.PeerSink()
        sink.frame[0], sink.n_peers, sink.first_pixel = f.data_ptr(), 1, 17
        assert small.render(vol, rays, mode, 64, sink=sink) == (None, None)
        frames.append(f)
    assert same_bits(frames[0], frames[1]) and bool((frames[0][17:17 + rays.shape[0]] != -7.0).all())


@pytest.mark.parametrize("mode", MODES)
def test_volume_range_x3(small, mode):
    """test_gpu_tc_range's x3 volume: hidden activations near 1e5"""
    base = small.vol32
    try:
        small.set_volume(base * 3.0)
        rays = small.rays[:4096].contiguous()
        a = small.render(small.volh, rays, mode, 128)
        b = small.render(small.volr, rays, mode, 128)
        assert same_bits(a[0], b[0]) and same_bits(a[1], b[1])
        a = small.samples(small.volh, rays[:700], mode, 48)
        b = small.samples(small.volr, rays[:700], mode, 48)
        assert all(same_bits(x, y) for x, y in zip(a, b))
    finally:
        small.set_volume(base)


def _extreme(vol32):
    """values above 65504 (inf in fp16, either sign) and in the fp16 subnormal range"""
    v = vol32.clone()                                     # keeps the encoder's channels-last strides
    flat = v.permute(0, 2, 3, 4, 1).view(-1)
    g = torch.Generator(device=DEV).manual_seed(3)
    idx = torch.randint(0, flat.numel(), (flat.numel() // 50,), generator=g, device=DEV)
    k = idx.numel() // 4
    flat[idx[:k]] = 7.0e4
    flat[idx[k:2 * k]] = -1.0e5
    flat[idx[2 * k:3 * k]] = 3.0e-6 * torch.sign(flat[idx[2 * k:3 * k]])
    flat[idx[3 * k:]] = 2.5e-7
    return v


@pytest.mark.parametrize("mode", MODES)
def test_inf_and_subnormal_volume(small, mode):
    base = small.vol32
    try:
        small.set_volume(_extreme(base))
        h = small.volh
        assert bool(torch.isinf(h).any()) and bool(((h != 0) & (h.abs() < 6.1035e-5)).any())
        rays = small.rays[:4096].contiguous()
        a = small.render(small.volh, rays, mode, 64)
        b = small.render(small.volr, rays, mode, 64)
        assert same_bits(a[0], b[0]) and same_bits(a[1], b[1])
        a = small.samples(small.volh, rays[:500], mode, 32)
        b = small.samples(small.volr, rays[:500], mode, 32)
        assert all(same_bits(x, y) for x, y in zip(a, b))
        t = torch.zeros(1, dtype=torch.int64, device=DEV)
        u = torch.zeros(1, dtype=torch.int64, device=DEV)
        a = small.render(small.volh, rays, mode, 64, t_stop=1e-4, tiles_done=t)
        b = small.render(small.volr, rays, mode, 64, t_stop=1e-4, tiles_done=u)
        assert same_bits(a[0], b[0]) and same_bits(a[1], b[1]) and int(t.item()) == int(u.item())
    finally:
        small.set_volume(base)


# ------------------------------------------------------------------------------------------------------------------
# layouts and the conversion kernel
# ------------------------------------------------------------------------------------------------------------------
def test_channels_last_half_is_read_in_place(small):
    rays = small.rays[:4096].contiguous()
    out = (torch.empty(4096, 3, device=DEV), torch.empty(4096, device=DEV))
    small.render(small.volh, rays, lib.MLP_TC_PAIR, 64, out=out)          # warm the image, weight and t_steps caches
    fresh = small.vol32.half()                                            # a new tensor object: no cache entry to hit
    torch.cuda.synchronize()
    before, misses = torch.cuda.memory_allocated(), backend.cache_stats["miss"]
    torch.cuda.reset_peak_memory_stats()
    small.render(fresh, rays, lib.MLP_TC_PAIR, 64, out=out)
    torch.cuda.synchronize()
    assert backend.cache_stats["miss"] == misses
    assert torch.cuda.max_memory_allocated() == before == torch.cuda.memory_allocated()
    ref = small.render(small.volr, rays, lib.MLP_TC_PAIR, 64)
    assert same_bits(out[0], ref[0]) and same_bits(out[1], ref[1])


def test_planar_half_is_converted_once_per_version(small):
    planar = small.vol32.contiguous().half()                              # [1,8,D,Hp,Wp] dense: not channels-last
    assert planar.is_contiguous() and not planar[0].permute(1, 2, 3, 0).is_contiguous()
    rays = small.rays[:2048].contiguous()
    backend.clear_cache()
    m0 = backend.cache_stats["miss"]
    a = small.render(planar, rays, lib.MLP_TC_SPLIT, 48)
    m1 = backend.cache_stats["miss"]
    b = small.render(planar, rays, lib.MLP_TC_PAIR, 48)
    assert backend.cache_stats["miss"] == m1 > m0
    img = backend._cache["volume_f16"][2]
    assert img.dtype == torch.float16 and tuple(img.shape) == tuple(small.volh[0].permute(1, 2, 3, 0).shape)
    assert torch.equal(img.view(torch.int16), small.volh[0].permute(1, 2, 3, 0).contiguous().view(torch.int16))
    assert same_bits(a[0], small.render(small.volr, rays, lib.MLP_TC_SPLIT, 48)[0])
    assert same_bits(b[0], small.render(small.volr, rays, lib.MLP_TC_PAIR, 48)[0])
    planar.mul_(1.0)                                                      # new version: converted again
    m2 = backend.cache_stats["miss"]
    small.render(planar, rays, lib.MLP_TC_PAIR, 48)
    assert backend.cache_stats["miss"] == m2 + 1


def test_conversion_kernel_rounds_as_tensor_half(small):
    """every source layout and dtype, with inf-rounding values and fp16 subnormals"""
    L = lib.load()
    v = _extreme(small.vol32)[0]                                          # [8,D,Hp,Wp] view of channels-last memory
    _, D, Hp, Wp = v.shape
    want = v.permute(1, 2, 3, 0).contiguous().half()
    for src, half, planar in ((v.contiguous(), 0, 1), (v.permute(1, 2, 3, 0).contiguous(), 0, 0),
                              (v.contiguous().half(), 1, 1), (want, 1, 0)):
        dst = torch.full((D, Hp, Wp, 8), float("nan"), dtype=torch.float16, device=DEV)
        lib.check(L.mvsn_volume_to_half(lib.ptr(src), half, planar, D, Hp, Wp, lib.ptr(dst), lib.stream_ptr()),
                  "mvsn_volume_to_half")
        torch.cuda.synchronize()
        assert torch.equal(dst.view(torch.int16), want.view(torch.int16)), (half, planar)


def test_fp32_mode_keeps_the_upcast(small):
    rays = small.rays[:3000].contiguous()
    a = small.render(small.volh, rays, lib.MLP_FP32, 48)
    b = small.render(small.volr, rays, lib.MLP_FP32, 48)
    assert same_bits(a[0], b[0]) and same_bits(a[1], b[1])
    vol = backend.RefVolume(small.volh.clone())
    a = small.samples(vol, rays[:500], lib.MLP_TC_SPLIT, 32)
    b = small.samples(small.volr, rays[:500], lib.MLP_TC_SPLIT, 32)
    assert all(same_bits(x, y) for x, y in zip(a, b))


# ------------------------------------------------------------------------------------------------------------------
# accuracy against the oracle at 512x640, pad 24, N_samples = 128 (every pixel)
# ------------------------------------------------------------------------------------------------------------------
def test_accuracy_vs_oracle_full_frame(net):
    fn, _ = net
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        w = {k: v.to(DEV) for k, v in orc.load_weights_npz(WPATH).items()}
        sc = synthetic.make_scene(512, 640, pad=24, seed=0)
        d = sc.to(DEV)
        rays = synthetic.scene_rays(sc).to(DEV)
        with torch.no_grad():
            vol = orc.encode_volume(d.imgs_norm, d.proj_mats, sc.near_far, sc.pad, w)
            volr = vol.half().float()
            args = (d.imgs_raw, d.pose_source, w, sc.H, sc.W, sc.near_far, float(sc.pad))
            ref = orc.render_rays(rays, vol, *args, n_samples=128)[0]
            ref_r = orc.render_rays(rays, volr, *args, n_samples=128)[0]
            volh = vol.permute(0, 2, 3, 4, 1).contiguous().permute(0, 4, 1, 2, 3).half()
            out = {}
            for name, mode in (("pair", lib.MLP_TC_PAIR), ("split", lib.MLP_TC_SPLIT)):
                out[name] = backend.render_rays(rays, volh, d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad),
                                                N_samples=128, mlp_mode=mode)[0]
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old
    e_pair = (out["pair"] - ref).abs().max().item()
    e_split = (out["split"] - ref).abs().max().item()
    e_split_r = (out["split"] - ref_r).abs().max().item()
    e_store = (ref_r - ref).abs().max().item()
    psnr = -10.0 * math.log10(max(float(((out["split"] - ref) ** 2).mean()), 1e-30))
    msg = (f"fp16 volume, 512x640 pad 24: pair vs oracle {e_pair:.3e}; split vs oracle {e_split:.3e} (PSNR {psnr:.1f} dB), "
           f"vs oracle on the rounded volume {e_split_r:.3e}; storage rounding alone (oracle) {e_store:.3e}")
    print("\n" + msg)
    assert e_pair <= 5e-3, e_pair
    assert e_split_r <= 1e-4, e_split_r


# ------------------------------------------------------------------------------------------------------------------
# encoder output
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("train", [True, False])
def test_encoder_f16_output(net, train):
    _, mvs = net
    sc = synthetic.make_scene(128, 160, pad=8, seed=2)
    d = sc.to(DEV)
    a, b = copy.deepcopy(mvs).train(train), copy.deepcopy(mvs).train(train)
    with torch.no_grad():
        v32, _, _ = a(d.imgs_norm, d.proj_mats, sc.near_far, pad=sc.pad)
        v16, _, _ = b(d.imgs_norm, d.proj_mats, sc.near_far, pad=sc.pad, volume_dtype=torch.float16)
    assert v16.dtype == torch.float16 and v16.shape == v32.shape and v16.stride() == v32.stride()
    assert torch.equal(v16.view(torch.int16), v32.half().view(torch.int16))
    for (na, ta), (nb, tb) in zip(a.named_buffers(), b.named_buffers()):
        assert na == nb and torch.equal(ta, tb), na
    with pytest.raises(RuntimeError, match="volume_dtype"):
        b.cost_reg_2(torch.zeros(1, 41, 8, 8, 8, device=DEV), torch.bfloat16)
