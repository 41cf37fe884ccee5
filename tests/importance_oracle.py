"""Restatement of the reference's importance sampling (data/ray_utils.py:98-141 sample_pdf, :199-224 ray_marcher_fine)
with the uniform draws as an input, in the dtype of its inputs (float64 for the GPU comparisons, float32 to pin it
against the reference's own outputs), and the per-sample quantities the GPU tests gate on.

`ref_mapping=True` looks the grid up where the reference does, at 4 ndc - 3 (ray_marcher_fine maps pts_NDC * 2 - 1 and
index_point_feature maps it again); the default looks it up at the sample's NDC, the encoding volume's own mapping."""
import torch
import torch.nn.functional as F


def lookup_sigma(grid, ndc, ref_mapping=False):
    """grid [D,H,W], ndc [N,S,3] -> sigma [N,S]: F.grid_sample, align_corners=True, zero padding"""
    g = ndc * 2 - 1.0
    if ref_mapping:
        g = g * 2 - 1.0
    n, s = ndc.shape[:2]
    return F.grid_sample(grid[None, None].to(g.dtype), g.reshape(1, 1, n, s, 3), mode="bilinear", padding_mode="zeros",
                         align_corners=True)[0, 0, 0]


def weights_of(sigma):
    alpha = 1.0 - torch.exp(-torch.relu(sigma))
    return alpha * torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1.0 - alpha + 1e-10], -1), -1)[:, :-1]


def sample_pdf(bins, weights, u):
    """sample_pdf with the draws `u` [N,K]; returns (samples [N,K], diagnostics)"""
    weights = weights + 1e-5
    pdf = weights / torch.sum(weights, -1, keepdim=True)
    cdf = torch.cat([torch.zeros_like(pdf[:, :1]), torch.cumsum(pdf, -1)], -1)
    inds = torch.searchsorted(cdf.contiguous(), u.contiguous(), right=True)
    below = torch.clamp(inds - 1, min=0)
    above = torch.clamp(inds, max=cdf.shape[-1] - 1)
    cb, ca = cdf.gather(1, below), cdf.gather(1, above)
    denom_raw = ca - cb
    denom = torch.where(denom_raw < 1e-5, torch.ones_like(denom_raw), denom_raw)
    t = (u - cb) / denom
    bb, ba = bins.gather(1, below), bins.gather(1, above)
    return bb + t * (ba - bb), {"below": below, "denom": denom_raw, "cdf": cdf, "pdf": pdf}


def linspace_u(n, k, dtype=torch.float32, device=None):
    """the deterministic draws: torch.linspace(0, 1, k) (fp32) for every ray"""
    return torch.linspace(0, 1, k, device=device).to(dtype).expand(n, k).contiguous()


def ray_marcher_fine(rays, grid, z_vals, pts_ndc, u, ref_mapping=False):
    """(xyz [N,S+K,3], z [N,S+K], diagnostics): ray_marcher_fine with the draws `u` [N,K]"""
    sigma = lookup_sigma(grid, pts_ndc, ref_mapping)
    w = weights_of(sigma)
    bins = 0.5 * (z_vals[:, :-1] + z_vals[:, 1:])
    fine, diag = sample_pdf(bins, w[:, 1:-1], u)
    z = torch.sort(torch.cat([fine, z_vals], -1), -1)[0]
    xyz = rays[:, None, 0:3] + rays[:, None, 3:6] * z[..., None]
    diag.update(fine=fine, bins=bins, sigma=sigma)
    return xyz, z, diag
