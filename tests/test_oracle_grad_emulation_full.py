"""CPU: tests/grad_emulation_full.mlp_full_emulated -- the arithmetic of grad_mode GRAD_TC_FULL -- pinned against fp32
autograd of the oracle on the scene tests/test_gpu_backward.py uses: rgb, depth, the fused loss and every gradient,
with random cotangents on the other outputs of `rendering`.  The bands measured here set the GPU gates of
tests/test_gpu_backward_tcf.py."""
import pytest
import torch

from grad_emulation_full import mlp_full_emulated, row_scaled_half
from oracle import mvsnerf_oracle as orc
from mvsnerf_b200 import backend, synthetic

# Measured on this scene (S 128 / 32): rgb 2.0e-4 / 2.3e-4, depth 2.0e-4 / 3.0e-4 of far, loss 5.7e-5 / 5.0e-5
# relative, MLP gradients 7.2e-2 / 1.1e-1 of max|g| (worst tensor; alpha_linear and rgb_linear ~5e-4), volume
# gradient 1.1e-2 / 4.3e-2.  The forward's fp16 operands move h by ~5e-4 relative; through the modulation product and
# the ReLU gates that moves the trunk's gradients far more than MLP_TC_HALF's backward-only rounding (~1e-3).  The GPU
# cases of tests/test_gpu_backward_tcf.py add white_bkgd and other batches: there the kernel is up to rgb 4.3e-4, depth
# 3.0e-4, loss 7.3e-5, MLP 0.19 and volume 0.078 (S 128, 300 rays) from fp32 autograd.  The pins cover both with
# about 1.5 - 2x of headroom.
BAND = {"rgb": 1e-3, "depth": 1e-3, "loss": 2e-4, "mlp": 0.3, "vol": 0.15}


@pytest.fixture(scope="module")
def scene(weights):
    sc = synthetic.make_scene(96, 128, pad=4, seed=9)
    vol = orc.encode_volume(sc.imgs_norm, sc.proj_mats, sc.near_far, sc.pad, weights)
    return sc, vol


def run(scene, weights, n, S, mlp_fn=None):
    """rgb, depth, loss = mean((rgb - target)^2) and the MLP / volume gradients of loss + random cotangents on depth,
    weights, alpha and input_feat, through the oracle's render_samples"""
    sc, vol = scene
    rays = synthetic.scene_rays(sc)
    rays = rays[torch.randperm(rays.shape[0], generator=torch.Generator().manual_seed(S + n))[:n]].contiguous()
    torch.manual_seed(S + n)
    pts, _, _, z = backend.ray_marcher(rays, N_samples=S, perturb=1.0)
    ndc = backend.get_ndc_coordinate(sc.pose_source["w2cs"][0], sc.pose_source["intrinsics"][0], pts,
                                     torch.tensor([sc.W - 1.0, sc.H - 1.0]), near=sc.near_far[0], far=sc.near_far[1],
                                     pad=sc.pad)
    g = torch.Generator().manual_seed(1)
    target = torch.rand(n, 3, generator=g)
    cot = [0.1 * torch.randn(n, generator=g), 0.05 * torch.randn(n, S, generator=g),
           0.05 * torch.randn(n, S, generator=g), 0.01 * torch.randn(n, S, 20, generator=g)]
    wt = {k: v.clone().requires_grad_(k.startswith("mlp/")) for k, v in weights.items()}
    vt = vol.clone().requires_grad_(True)
    rgb, feat, w, depth, alpha = orc.render_samples(pts, ndc, z, rays[:, 3:6], vt, sc.imgs_raw, sc.pose_source, wt,
                                                    mlp_fn=mlp_fn)
    loss = ((rgb - target) ** 2).mean()
    (loss + (depth * cot[0]).sum() + (w * cot[1]).sum() + (alpha * cot[2]).sum() + (feat * cot[3]).sum()).backward()
    return {"rgb": rgb.detach(), "depth": depth.detach(), "loss": loss.detach(),
            "mlp": {k: v.grad for k, v in wt.items() if v.grad is not None}, "vol": vt.grad}


def band(a, b, far):
    """the errors of run() output a against b, in the units BAND uses"""
    return {"rgb": (a["rgb"] - b["rgb"]).abs().max().item(),
            "depth": (a["depth"] - b["depth"]).abs().max().item() / far,
            "loss": abs(a["loss"].item() - b["loss"].item()) / b["loss"].item(),
            "mlp": max((a["mlp"][k] - b["mlp"][k]).abs().max().item() / b["mlp"][k].abs().max().item() for k in b["mlp"]),
            "vol": (a["vol"] - b["vol"]).abs().max().item() / b["vol"].abs().max().item()}


def test_row_scaled_half_is_per_row():
    """Each row takes its own scale: a row's operand does not depend on the other rows, and a row of small values keeps
    fp16's relative precision where a shared scale would flush it."""
    v = torch.tensor([[3.0e-6, 1.7e-6, 0.0], [4.0e3, 1.0, 0.0], [0.0, 0.0, 0.0]])
    q = row_scaled_half(v)
    for r in range(3):
        assert torch.equal(row_scaled_half(v[r:r + 1]), q[r:r + 1])
    assert ((q - v.double()).abs() <= v.double().abs() * 2.0 ** -11).all()
    assert torch.equal(q[2], torch.zeros(3, dtype=torch.float64))
    big = torch.tensor([[1.0e5, 3.0]])                                  # a row max of 1e5 is scaled below 2^15
    assert torch.isfinite(row_scaled_half(big)).all()


@pytest.mark.parametrize("S,n", [(128, 37), (32, 130)])
def test_full_emulation_band_against_fp32_autograd(scene, weights, S, n):
    """fp16 operands in the forward and the backward move every output by fp16-sized amounts: visible, and bounded."""
    ref = run(scene, weights, n, S)
    emu = run(scene, weights, n, S, mlp_full_emulated)
    e = band(emu, ref, scene[0].near_far[1])
    print("\nGRAD_TC_FULL emulation vs fp32 autograd: " + " ".join(f"{k} {v:.3e}" for k, v in e.items()))
    for k, v in e.items():
        assert v < BAND[k], (k, v)
    assert e["mlp"] > 1e-3 and e["rgb"] > 1e-5                          # the rounding is really there
