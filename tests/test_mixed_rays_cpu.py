"""CPU: the references tests/test_gpu_mixed_rays.py relies on, on its mixed batches (four cameras, a near / far per ray).

  * orc.march_rays and backend.ray_marcher march each ray over its own [near, far] (linear and lindisp, near == far),
    and agree bit for bit;
  * the NDC of both host conversions follows each sample's camera depth with the scene's near_far, also for rays that
    start in front of the scene's near (NDC z < 0) and end past its far (NDC z > 1);
  * the batch builder mixes cameras and depth ranges inside every group of 4, 8, 16 and 32 consecutive rays.
"""
import pytest
import torch

from mvsnerf_b200 import backend, synthetic
from oracle import mvsnerf_oracle as orc
from test_gpu_mixed_rays import EQUAL, FRONT, BEYOND, N_CAMS, NARROW, mixed_cameras, mixed_rays


@pytest.fixture(scope="module")
def batch():
    sc = synthetic.make_scene(96, 128, pad=24, seed=5)
    rays, cam, kind = mixed_rays(sc, 1999, seed=11)
    return sc, rays, cam, kind


def _z_f64(rays, S, lindisp):
    t = torch.linspace(0, 1, S).double()
    near, far = rays[:, 6:7].double(), rays[:, 7:8].double()
    return 1 / (1 / near * (1 - t) + 1 / far * t) if lindisp else near * (1 - t) + far * t


@pytest.mark.parametrize("lindisp", [False, True])
@pytest.mark.parametrize("S", [24, 33, 128])
def test_march_over_each_rays_own_range(batch, S, lindisp):
    sc, rays, _, kind = batch
    pts, z = orc.march_rays(rays, S, lindisp)
    xyz, o, d, z_b = backend.ray_marcher(rays, N_samples=S, lindisp=lindisp)
    assert torch.equal(z, z_b) and torch.equal(pts, xyz)
    assert torch.equal(o, rays[:, :3]) and torch.equal(d, rays[:, 3:6])
    want = _z_f64(rays, S, lindisp)
    assert ((z.double() - want).abs() <= 4e-7 * want.abs()).all()
    near, far = rays[:, 6], rays[:, 7]
    assert ((z[:, 0] - near).abs() <= 4e-7 * near).all() and ((z[:, -1] - far).abs() <= 4e-7 * far).all()
    eq = kind == EQUAL
    assert eq.any() and ((z[eq] - near[eq, None]).abs() <= 4e-7 * near[eq, None]).all()
    # monotone along every ray with near < far, and the points on the ray
    assert (z[~eq][:, 1:] >= z[~eq][:, :-1]).all()
    p64 = rays[:, None, :3].double() + rays[:, None, 3:6].double() * z[..., None].double()
    assert (pts.double() - p64).abs().max() < 1e-5


@pytest.mark.parametrize("lindisp", [False, True])
def test_ndc_of_mixed_rays(batch, lindisp):
    """NDC z is (zc - near) / (far - near) (lindisp: in 1 / depth) with the scene's near_far, zc each sample's depth in
    the reference camera; x, y its padded pixel coordinates.  FRONT rays reach NDC z < 0, BEYOND rays z > 1."""
    sc, rays, _, kind = batch
    S = 33
    pts, z = orc.march_rays(rays, S, lindisp)
    w2c, K = sc.pose_source["w2cs"][0], sc.pose_source["intrinsics"][0]
    near, far = sc.near_far
    ndc = orc.ndc_coords(w2c, K, pts, sc.H, sc.W, near, far, float(sc.pad), lindisp)
    ndc_b = backend.get_ndc_coordinate(w2c, K, pts, torch.tensor([sc.W - 1.0, sc.H - 1.0]), near=near, far=far,
                                       pad=sc.pad, lindisp=lindisp)
    cam = pts.reshape(-1, 3).double() @ w2c[:3, :3].double().t() + w2c[:3, 3].double()
    pix = cam @ K.double().t()
    zc = pix[:, 2].view(pts.shape[:2])
    nz = (1 / zc - 1 / near) / (1 / far - 1 / near) if lindisp else (zc - near) / (far - near)
    wf, hf = sc.W / 4.0, sc.H / 4.0
    u = (pix[:, 0] / pix[:, 2] / (sc.W - 1)).view(pts.shape[:2])
    v = (pix[:, 1] / pix[:, 2] / (sc.H - 1)).view(pts.shape[:2])
    x = (u * wf + sc.pad) / (wf + 2 * sc.pad)
    y = (v * hf + sc.pad) / (hf + 2 * sc.pad)
    want = torch.stack([x, y, nz], -1)
    for got in (ndc, ndc_b):
        assert (got.double() - want).abs().max() < 2e-5
    assert (ndc[kind == FRONT][:, 0, 2] < 0).all()
    assert (ndc[kind == BEYOND][:, -1, 2] > 1).all()
    eq = kind == EQUAL
    assert (ndc[eq] - ndc[eq][:, :1]).abs().max() < 1e-6          # every sample of a near == far ray: one point


@pytest.mark.parametrize("rt", [4, 8, 16, 32])
def test_every_group_mixes_cameras_and_depth_ranges(batch, rt):
    sc, rays, cam, kind = batch
    G = rays.shape[0] // rt
    c = cam[:G * rt].view(G, rt)
    assert all(len(set(row.tolist())) == N_CAMS for row in c)
    near = rays[:G * rt, 6].view(G, rt)
    far = rays[:G * rt, 7].view(G, rt)
    assert (near.amax(1) > near.amin(1)).all() and (far.amax(1) > far.amin(1)).all()
    for k in range(5):
        assert (kind == k).sum() >= 0.03 * rays.shape[0], k
    assert ((rays[kind == NARROW, 7] - rays[kind == NARROW, 6]) < 0.04 * (sc.near_far[1] - sc.near_far[0])).all()


def test_batch_builder_draws_the_camera_rays(batch):
    """each ray is a pixel ray of its camera (origin and direction of synthetic.camera_rays), so the mix is of views"""
    sc, rays, cam, _ = batch
    c2ws = mixed_cameras(sc)
    assert len(c2ws) == N_CAMS and all(not torch.equal(c2ws[0], c) for c in c2ws[1:])
    for k, c2w in enumerate(c2ws):
        allr = synthetic.camera_rays(sc.directions, c2w, *sc.near_far)
        sel = rays[cam == k]
        assert torch.equal(sel[:, :3], allr[: sel.shape[0], :3])
        d = torch.cdist(sel[:, 3:6], allr[:, 3:6], compute_mode="donot_use_mm_for_euclid_dist").min(1).values
        assert (d < 1e-5).all()                                    # pixels are 1 / focal ~ 7e-3 apart
