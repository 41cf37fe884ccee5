"""CPU: tests/grad_emulation.mlp_grad_emulated -- the gradient arithmetic of grad_mode MLP_TC_HALF -- pinned against
fp32 autograd of the oracle on the scene tests/test_gpu_backward.py uses, with random cotangents on all five outputs
of `rendering`."""
import functools

import pytest
import torch

from grad_emulation import mlp_grad_emulated, round_half_significand
from oracle import mvsnerf_oracle as orc
from mvsnerf_b200 import backend, synthetic


@pytest.fixture(scope="module")
def scene(weights):
    sc = synthetic.make_scene(96, 128, pad=4, seed=9)
    vol = orc.encode_volume(sc.imgs_norm, sc.proj_mats, sc.near_far, sc.pad, weights)
    return sc, vol


def _grads(scene, weights, n, S, mlp_fn=None, dtype=torch.float32):
    """MLP and volume gradients of the oracle's render_samples under random cotangents; `dtype` float64 runs the whole
    render (samples, volume, images, cameras, weights) in fp64"""
    sc, vol = scene
    rays = synthetic.scene_rays(sc)
    rays = rays[torch.randperm(rays.shape[0], generator=torch.Generator().manual_seed(S + n))[:n]].contiguous()
    torch.manual_seed(S + n)
    pts, _, _, z = backend.ray_marcher(rays, N_samples=S, perturb=1.0)
    ndc = backend.get_ndc_coordinate(sc.pose_source["w2cs"][0], sc.pose_source["intrinsics"][0], pts,
                                     torch.tensor([sc.W - 1.0, sc.H - 1.0]), near=sc.near_far[0], far=sc.near_far[1], pad=sc.pad)
    g = torch.Generator().manual_seed(1)
    cot = [torch.randn(n, 3, generator=g), 0.1 * torch.randn(n, generator=g), 0.05 * torch.randn(n, S, generator=g),
           0.05 * torch.randn(n, S, generator=g), 0.01 * torch.randn(n, S, 20, generator=g)]
    cot = [c.to(dtype) for c in cot]
    wt = {k: v.to(dtype, copy=True).requires_grad_(k.startswith("mlp/")) for k, v in weights.items()}
    vt = vol.to(dtype, copy=True).requires_grad_(True)
    pose = {k: v.to(dtype) for k, v in sc.pose_source.items()}
    rgb, feat, w, depth, alpha = orc.render_samples(pts.to(dtype), ndc.to(dtype), z.to(dtype), rays[:, 3:6].to(dtype), vt,
                                                    sc.imgs_raw.to(dtype), pose, wt, mlp_fn=mlp_fn)
    ((rgb * cot[0]).sum() + (depth * cot[1]).sum() + (w * cot[2]).sum() + (alpha * cot[3]).sum()
     + (feat * cot[4]).sum()).backward()
    return {k: v.grad for k, v in wt.items() if v.grad is not None}, vt.grad


def _worst(a, b):
    """max over tensors of max|a - b| / max|b|"""
    return max((a[k] - b[k]).abs().max().item() / b[k].abs().max().item() for k in b)


def test_round_half_significand_is_fp16_rounding():
    x = torch.randn(10000) * 100.0
    assert torch.equal(round_half_significand(x).float(), x.half().float())
    tiny = torch.tensor([1e-12, 3.3e-9, -7.7e-20])                     # unbounded exponent: no fp16 underflow
    r = round_half_significand(tiny)
    assert ((r - tiny.double()).abs() <= tiny.double().abs() * 2.0 ** -11).all() and (r != 0).all()


@pytest.mark.parametrize("S,n", [(128, 37), (32, 130)])
def test_emulator_without_rounding_is_autograd(scene, weights, S, n):
    """In fp64 both sides, so that the comparison measures the emulator's backward and not how the host's BLAS rounds
    fp32 autograd (which moves it by ~1.6e-6 of max|g| where the BLAS has no FMA path)."""
    ref_p, ref_v = _grads(scene, weights, n, S, dtype=torch.float64)
    p, v = _grads(scene, weights, n, S, functools.partial(mlp_grad_emulated, rounding=False), dtype=torch.float64)
    print(f"emulator without rounding vs fp64 autograd: mlp {_worst(p, ref_p):.3e}")
    assert _worst(p, ref_p) < 1e-6
    assert (v - ref_v).abs().max().item() < 1e-6 * ref_v.abs().max().item()


@pytest.mark.parametrize("S,n", [(128, 37), (32, 130)])
def test_emulator_rounding_error_is_fp16_sized(scene, weights, S, n):
    """fp16 operands move the gradients by ~1e-3 of max|g| at most: visible, and bounded."""
    ref_p, ref_v = _grads(scene, weights, n, S)
    p, v = _grads(scene, weights, n, S, mlp_grad_emulated)
    e_p = _worst(p, ref_p)
    e_v = (v - ref_v).abs().max().item() / ref_v.abs().max().item()
    assert 1e-4 < e_p < 2e-3, e_p
    assert 1e-5 < e_v < 2e-3, e_v
