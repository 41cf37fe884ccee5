"""Seeded synthetic scenes shaped like the reference's datasets (no datasets ship here).

What a dataset's `read_source_views()` hands the hot path (reference
data/dtu_ft.py:72-119) is: three ImageNet-normalised source images, the
plane-sweep projection matrices `src_proj @ inv(ref_proj)` in 1/4-resolution
feature space, `near_far`, and the `pose_source` dict (w2cs, c2ws, full-res
intrinsics).  This module fabricates exactly that contract from a seed, plus a
target camera and its rays `[N, 8] = (origin, direction, near, far)` as the
notebooks build them (renderer_video.ipynb "DTU video rendering" cell).

Everything is generated on the host with a seeded CPU generator so the oracle
and the CUDA path consume bit-identical inputs.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch
import torch.nn.functional as F

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


@dataclass
class Scene:
    H: int
    W: int
    pad: int
    focal: float
    imgs_norm: torch.Tensor      # [1, V, 3, H, W]  ImageNet-normalised (MVSNet input)
    imgs_raw: torch.Tensor       # [1, V, 3, H, W]  in [0, 1] (rendering input)
    proj_mats: torch.Tensor      # [1, V, 3, 4]     feature-space homographies, [0] = identity
    near_far: tuple              # (near, far)
    pose_source: dict            # w2cs [V,4,4], c2ws [V,4,4], intrinsics [V,3,3] (full res)
    c2w_target: torch.Tensor     # [4, 4]
    directions: torch.Tensor     # [H, W, 3] camera-frame ray directions of the target view

    def to(self, device):
        mv = lambda t: t.to(device)
        return Scene(self.H, self.W, self.pad, self.focal, mv(self.imgs_norm), mv(self.imgs_raw),
                     mv(self.proj_mats), self.near_far,
                     {k: mv(v) for k, v in self.pose_source.items()}, mv(self.c2w_target),
                     mv(self.directions))


def _yaw(deg: float) -> np.ndarray:
    a = math.radians(deg)
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]], dtype=np.float64)


def _w2c(R: np.ndarray, cam_center: np.ndarray) -> np.ndarray:
    m = np.eye(4)
    m[:3, :3] = R
    m[:3, 3] = -R @ cam_center
    return m


def pixel_directions(H: int, W: int, fx: float, fy: float, cx: float | None = None,
                     cy: float | None = None) -> torch.Tensor:
    """Camera-frame directions ((x-cx)/fx, (y-cy)/fy, 1), no half-pixel offset.

    Same convention as reference data/ray_utils.py:12-30 (get_ray_directions)."""
    cx = W / 2 if cx is None else cx
    cy = H / 2 if cy is None else cy
    xs = torch.linspace(0, W - 1, W)
    ys = torch.linspace(0, H - 1, H)
    gy, gx = torch.meshgrid(ys, xs, indexing="ij")
    return torch.stack([(gx - cx) / fx, (gy - cy) / fy, torch.ones_like(gx)], -1)


def camera_rays(directions: torch.Tensor, c2w: torch.Tensor, near: float, far: float) -> torch.Tensor:
    """rays [H*W, 8] = (o, d, near, far); d is NOT normalised (reference data/ray_utils.py:32-53)."""
    d = (directions.reshape(-1, 3) @ c2w[:3, :3].T).contiguous()
    o = c2w[:3, 3].expand_as(d)
    nf = torch.tensor([near, far], dtype=d.dtype, device=d.device).expand(d.shape[0], 2)
    return torch.cat([o, d, nf], 1).contiguous()


def make_scene(H: int = 512, W: int = 640, pad: int = 24, seed: int = 0,
               near_far=(2.125, 4.525), n_views: int = 3, target_shift: float = 0.1) -> Scene:
    g = torch.Generator().manual_seed(seed)
    # low-frequency texture shared by all views + a little per-view noise so the
    # feature variance volume is structured rather than white (SURVEY.md 8(d)).
    lh, lw = max(H // 8, 2), max(W // 8, 2)
    base = torch.rand(1, 3, lh, lw, generator=g)
    base = F.interpolate(base, size=(H, W), mode="bicubic", align_corners=False).clamp(0, 1)
    noise = torch.rand(n_views, 3, H, W, generator=g) * 0.02
    imgs_raw = (base + noise).clamp(0, 1).unsqueeze(0).contiguous()        # [1,V,3,H,W]
    mean = torch.tensor(IMAGENET_MEAN).view(1, 1, 3, 1, 1)
    std = torch.tensor(IMAGENET_STD).view(1, 1, 3, 1, 1)
    imgs_norm = ((imgs_raw - mean) / std).contiguous()

    focal = 1.1 * W
    K = np.array([[focal, 0, W / 2], [0, focal, H / 2], [0, 0, 1]], dtype=np.float64)
    K_feat = K.copy()
    K_feat[:2] /= 4.0                                  # feature maps are 1/4 resolution
    # reference view at the origin; sources +-0.3 on x with a 3 degree yaw toward the scene
    centers = [np.zeros(3), np.array([0.3, 0.0, 0.0]), np.array([-0.3, 0.0, 0.0])][:n_views]
    yaws = [0.0, -3.0, 3.0][:n_views]
    w2cs, c2ws, projs = [], [], []
    ref_proj_inv = None
    for i, (c, y) in enumerate(zip(centers, yaws)):
        w2c = _w2c(_yaw(y), c)
        w2cs.append(w2c)
        c2ws.append(np.linalg.inv(w2c))
        P = np.eye(4)
        P[:3, :4] = K_feat @ w2c[:3, :4]
        if i == 0:
            ref_proj_inv = np.linalg.inv(P)
            projs.append(np.eye(4))
        else:
            projs.append(P @ ref_proj_inv)
    pose_source = {
        "w2cs": torch.from_numpy(np.stack(w2cs)).float(),
        "c2ws": torch.from_numpy(np.stack(c2ws)).float(),
        "intrinsics": torch.from_numpy(np.stack([K] * n_views)).float(),
    }
    proj_mats = torch.from_numpy(np.stack(projs)[:, :3]).float().unsqueeze(0)
    c2w_t = np.linalg.inv(_w2c(_yaw(1.0), np.array([target_shift, 0.02, 0.0])))
    return Scene(H, W, pad, focal, imgs_norm, imgs_raw, proj_mats, tuple(near_far), pose_source,
                 torch.from_numpy(c2w_t).float(), pixel_directions(H, W, focal, focal))


def make_plane_scene(H: int = 512, W: int = 640, pad: int = 24, seed: int = 0, near_far=(2.125, 4.525),
                     n_views: int = 3, target_shift: float = 0.1, plane=(3.0, 0.4), tex_hw=(48, 60),
                     extent=(2.0, 1.6)) -> Scene:
    """make_scene's cameras, but multi-view-consistent source views: each is a rendering of one textured plane
    z = plane[0] + plane[1] * x (world frame = reference camera), between near and far.  The texture is seeded
    uniform noise [3, *tex_hw] resampled bicubically over x in [-extent[0], extent[0]], y in [-extent[1], extent[1]].
    The encoder recovers such geometry, so rays of the target view become opaque at the plane (make_scene's views are
    identical images, whose only consistent depth is at infinity)."""
    sc = make_scene(H, W, pad=pad, seed=seed, near_far=near_far, n_views=n_views, target_shift=target_shift)
    g = torch.Generator().manual_seed(seed + 7919)
    tex = torch.rand(1, 3, tex_hw[0], tex_hw[1], generator=g, dtype=torch.float64)
    z0, sx = plane
    dirs = sc.directions.reshape(-1, 3).double()                       # camera frame, z = 1
    views = []
    for v in range(n_views):
        w2c = sc.pose_source["w2cs"][v].double()
        R, t = w2c[:3, :3], w2c[:3, 3]
        c = -R.T @ t                                                   # camera centre
        d = dirs @ R                                                   # world directions (R^T d per row)
        s = (z0 + sx * c[0] - c[2]) / (d[:, 2] - sx * d[:, 0])
        p = c[None] + s[:, None] * d
        grid = torch.stack([p[:, 0] / extent[0], p[:, 1] / extent[1]], -1).view(1, H, W, 2)
        img = F.grid_sample(tex, grid, mode="bicubic", padding_mode="border", align_corners=True)
        views.append(img[0].clamp(0, 1).float())
    imgs_raw = torch.stack(views).unsqueeze(0).contiguous()          # [1,V,3,H,W]
    mean = torch.tensor(IMAGENET_MEAN).view(1, 1, 3, 1, 1)
    std = torch.tensor(IMAGENET_STD).view(1, 1, 3, 1, 1)
    return Scene(H, W, pad, sc.focal, ((imgs_raw - mean) / std).contiguous(), imgs_raw, sc.proj_mats, sc.near_far,
                 sc.pose_source, sc.c2w_target, sc.directions)


def scene_rays(scene: Scene, c2w: torch.Tensor | None = None) -> torch.Tensor:
    c2w = scene.c2w_target if c2w is None else c2w
    return camera_rays(scene.directions, c2w, scene.near_far[0], scene.near_far[1])


def spiral_path(scene: Scene, n_frames: int = 60, radius: float = 0.12) -> torch.Tensor:
    """A closed loop of target cameras around the reference view (free-viewpoint video shape)."""
    out = []
    for i in range(n_frames):
        t = 2 * math.pi * i / n_frames
        c = np.array([radius * math.cos(t), 0.5 * radius * math.sin(t), 0.05 * math.sin(2 * t)])
        out.append(np.linalg.inv(_w2c(_yaw(2.0 * math.sin(t)), c)))
    return torch.from_numpy(np.stack(out)).float()
