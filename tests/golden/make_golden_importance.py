"""Generate tests/golden/importance_16x12x10.npz from the UNMODIFIED reference (where its source tree is present).

    python tests/golden/make_golden_importance.py

data/ray_utils.sample_pdf and ray_marcher_fine on a seeded 16 x 12 x 10 density grid (sigma in [-2, 6]) and 96 rays
with 24 coarse samples each (ray_marcher, perturb 1, seed 21), their pts_NDC spread over [-0.1, 1.1]^3 so that zero
padding is exercised:
  * ray_marcher_fine with N_importance 32 under torch.manual_seed(22) (its one draw, sample_pdf's torch.rand), and
    that draw re-made from the same seed, so the test can feed it to the oracle;
  * sample_pdf with det=True (linspace draws) on the same bins and weights.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402

N, S, K = 96, 24, 32
D, H, W = 16, 12, 10


def main():
    ref = ref_shim.load_reference()
    g = torch.Generator().manual_seed(20)
    grid = torch.rand(D, H, W, generator=g) * 8.0 - 2.0
    o = torch.rand(N, 3, generator=g) - 0.5
    d = torch.nn.functional.normalize(torch.rand(N, 3, generator=g) - 0.5 + torch.tensor([0.0, 0.0, 1.0]), dim=-1)
    near = 2.0 + torch.rand(N, 1, generator=g)
    far = near + 1.0 + 3.0 * torch.rand(N, 1, generator=g)
    rays = torch.cat([o, d, near, far], -1)
    torch.manual_seed(21)
    _, _, _, z_vals = ref.ray_utils.ray_marcher(rays, N_samples=S, perturb=1.0)
    pts_ndc = torch.rand(N, S, 3, generator=g) * 1.2 - 0.1
    torch.manual_seed(22)
    xyz, _, _, z_fine = ref.ray_utils.ray_marcher_fine(rays, grid, z_vals, pts_ndc, N_importance=K)
    torch.manual_seed(22)
    u = torch.rand(N, K)
    # sample_pdf alone, deterministic draws, on ray_marcher_fine's bins and weights (recomputed as it forms them)
    sigma = ref.utils.index_point_feature(grid[None, None], pts_ndc * 2 - 1.0)
    alpha = 1.0 - torch.exp(-torch.relu(sigma))
    weights = alpha * torch.cumprod(torch.cat([torch.ones(N, 1), 1.0 - alpha + 1e-10], -1), -1)[:, :-1]
    bins = 0.5 * (z_vals[:, :-1] + z_vals[:, 1:])
    det = ref.ray_utils.sample_pdf(bins, weights[:, 1:-1], K, det=True)
    out = os.path.join(HERE, "importance_16x12x10.npz")
    np.savez_compressed(out, grid=grid.numpy(), rays=rays.numpy(), z_vals=z_vals.numpy(), pts_ndc=pts_ndc.numpy(),
                        u=u.numpy(), xyz=xyz.numpy(), z_fine=z_fine.numpy(), bins=bins.numpy(),
                        weights=weights[:, 1:-1].numpy(), det_samples=det.numpy())
    print(out, os.path.getsize(out))


if __name__ == "__main__":
    main()
