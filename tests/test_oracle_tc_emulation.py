"""CPU: oracle.mlp_emulated -- the operand arithmetic of the tensor-core MLP modes (csrc/render_wg.cu) -- pinned against
the fp32 oracle on the mid-size synthetic scene the GPU tests render (2048 rays x 128 samples)."""
import functools

import pytest
import torch

from oracle import mvsnerf_oracle as orc
from mvsnerf_b200 import synthetic


@pytest.fixture(scope="module")
def scene(weights):
    sc = synthetic.make_scene(128, 160, pad=8, seed=5)
    vol = orc.encode_volume(sc.imgs_norm, sc.proj_mats, sc.near_far, sc.pad, weights)
    rays = synthetic.scene_rays(sc)
    g = torch.Generator().manual_seed(128 * 1000 + 2048)
    return sc, vol, rays[torch.randperm(rays.shape[0], generator=g)[:2048]]


def _render(scene, weights, scale, mlp_fn=None):
    sc, vol, rays = scene
    rgb, _ = orc.render_rays(rays, vol * scale, sc.imgs_raw, sc.pose_source, weights, sc.H, sc.W, sc.near_far,
                             float(sc.pad), n_samples=128, mlp_fn=mlp_fn)
    return rgb


def test_emulated_modes_vs_fp32_mlp(scene, weights):
    """fp16 operands cost 6.4e-4 RGB Linf on this set; the 2-term split 3e-7 (fp32 rounding)."""
    ref = _render(scene, weights, 1.0)
    half = _render(scene, weights, 1.0, functools.partial(orc.mlp_emulated, mode="half"))
    split = _render(scene, weights, 1.0, functools.partial(orc.mlp_emulated, mode="split"))
    e_half, e_split = (half - ref).abs().max().item(), (split - ref).abs().max().item()
    assert 1e-4 < e_half < 1e-3, e_half          # fp16 rounding is visible, and bounded
    assert e_split < 1e-6, e_split


def test_emulated_split_keeps_its_range(scene, weights):
    """Volume x3: hidden activations reach ~1e5, beyond fp16 (65504).  The per-row activation scale keeps the split
    mode at fp32 grade; the fp16 mode saturates and leaves its 5e-3 gate (measured 1.1e-2)."""
    ref = _render(scene, weights, 3.0)
    split = _render(scene, weights, 3.0, functools.partial(orc.mlp_emulated, mode="split"))
    assert torch.isfinite(split).all()
    assert (split - ref).abs().max().item() < 2e-5


def test_emulated_split_with_large_weights():
    """A weight of 300 would be inf at the x256 scale: the image scale drops to 2^6 and the result stays fp32 grade."""
    torch.manual_seed(0)
    from mvsnerf_b200 import backend
    fn = backend.MVSNeRF()
    w = {"mlp/" + k: v.detach() for k, v in fn.state_dict().items()}
    w["mlp/nerf.pts_linears.2.weight"][5, 7] = 300.0
    x = torch.cat([orc.positional_encoding(torch.rand(4096, 3)), torch.rand(4096, 20) * 4 - 2,
                   torch.nn.functional.normalize(torch.randn(4096, 3), dim=-1)], -1)
    ref = orc.mlp(x, w)
    split = orc.mlp_emulated(x, w, "split")
    assert torch.isfinite(split).all()
    assert (split - ref).abs().max().item() < 1e-5 * max(1.0, ref.abs().max().item())
