"""GPU: the plain fp16 render kernels keep part of the weight image resident in shared memory and stream the rest.

The early-termination kernels (`t_stop`) keep the schedule that streams every chunk, and at t_stop = 0 they compute
exactly what the plain kernels compute (test_gpu_render_stop pins that), so `render_rays(..., t_stop=0)` is the
reference the plain ray entry must match bit for bit:

  * the full bench frame (512x640, 128 samples, pad 24) in pair mode, from the fp32 and from the fp16 volume;
  * shapes where a consumer runs idle passes (one ray, an odd number of ray groups, several groups per CTA), sample
    counts that leave a partial last tile, white_bkgd and lindisp;
  * the samples entry (host-marched samples) against the fp32 kernel at the fp16 modes' 5e-3 gate.
"""
import os

import pytest
import torch

from conftest import GOLDEN
from oracle import mvsnerf_oracle as orc
from mvsnerf_b200 import backend, lib, synthetic

pytestmark = pytest.mark.gpu
DEV = "cuda"


class Args:
    feat_dim = 20
    img_downscale = 1.0
    use_color_volume = False
    net_type = "v0"


@pytest.fixture(scope="module")
def net():
    fn, mvs = backend.MVSNeRF().to(DEV), backend.MVSNet().to(DEV).train()
    backend.load_weights_npz(fn, mvs, os.path.join(GOLDEN, "mvsnerf_v0_weights.npz"))
    return fn, mvs


class Ctx:
    def __init__(self, sc, fn, mvs):
        self.sc, self.fn, self.d = sc, fn, sc.to(DEV)
        with torch.no_grad():
            vol, _, _ = mvs(self.d.imgs_norm, self.d.proj_mats, sc.near_far, pad=sc.pad)
        self.vols = {"fp32": vol, "fp16": vol.half()}
        self.rays = synthetic.scene_rays(sc).to(DEV).contiguous()

    def render(self, rays, vol="fp32", S=128, white=False, lindisp=False, mode=lib.MLP_TC_PAIR, **kw):
        with torch.no_grad():
            return backend.render_rays(rays, self.vols[vol], self.d.imgs_raw, self.d.pose_source, self.fn,
                                       self.sc.near_far, float(self.sc.pad), N_samples=S, white_bkgd=white,
                                       lindisp=lindisp, mlp_mode=mode, **kw)

    def check_streamed(self, rays, **kw):
        rgb, depth = self.render(rays, **kw)
        rgb0, depth0 = self.render(rays, t_stop=0.0, **kw)
        assert torch.equal(rgb, rgb0) and torch.equal(depth, depth0)


@pytest.fixture(scope="module")
def bench(net):
    return Ctx(synthetic.make_scene(512, 640, pad=24, seed=0, near_far=(2.125, 4.525)), *net)


@pytest.fixture(scope="module")
def small(net):
    return Ctx(synthetic.make_scene(96, 128, pad=8, seed=3), *net)


@pytest.mark.parametrize("vol", ["fp32", "fp16"])
def test_bench_frame_equals_streamed(bench, vol):
    bench.check_streamed(bench.rays, vol=vol)


def _rays(ctx, n):
    reps = (n + ctx.rays.shape[0] - 1) // ctx.rays.shape[0]
    return torch.cat([ctx.rays] * reps)[:n].contiguous()


# 1: one group, the second consumer idle throughout; 37: ten 4-ray groups; 993: 249 groups of 4 rays, an odd count,
# so the last CTA's second consumer runs idle passes (fewer than 2 x 4 rays x grid); 16990: 531 groups of 32 rays,
# several units on some CTAs and an idle consumer on the last one
@pytest.mark.parametrize("n", [1, 37, 993, 16990])
@pytest.mark.parametrize("vol", ["fp32", "fp16"])
def test_idle_consumers_equal_streamed(small, n, vol):
    small.check_streamed(_rays(small, n), vol=vol)


@pytest.mark.parametrize("S", [33, 48, 128])
@pytest.mark.parametrize("white,lindisp", [(False, False), (True, False), (False, True)])
def test_options_equal_streamed(small, S, white, lindisp):
    small.check_streamed(_rays(small, 2001), S=S, white=white, lindisp=lindisp)


@pytest.mark.parametrize("mode", [lib.MLP_TC_PAIR, lib.MLP_TC_HALF])
@pytest.mark.parametrize("S", [33, 128])
def test_samples_entry_against_fp32(small, mode, S):
    rays = _rays(small, 3000)
    pts, z = orc.march_rays(rays, S, False)
    ndc = orc.ndc_coords(small.d.pose_source["w2cs"][0], small.d.pose_source["intrinsics"][0], pts, small.sc.H,
                         small.sc.W, small.sc.near_far[0], small.sc.near_far[1], float(small.sc.pad), False)
    out = {}
    for m in (mode, lib.MLP_FP32):
        with torch.no_grad():
            out[m] = backend.rendering(Args, small.d.pose_source, pts, ndc, z, rays[:, :3], rays[:, 3:6],
                                       small.vols["fp32"], small.d.imgs_raw, network_fn=small.fn, mlp_mode=m)
    rgb, rgb32 = out[mode][0], out[lib.MLP_FP32][0]
    assert torch.isfinite(rgb).all()
    assert (rgb - rgb32).abs().max().item() < 5e-3
