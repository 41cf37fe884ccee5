#!/usr/bin/env python
"""Small-shape pass through EVERY kernel of the library, for compute-sanitizer (memcheck / initcheck / racecheck):

    compute-sanitizer --tool initcheck python tools/sanitize_smoke.py

K-F FeatureNet, K-A cost volume (the F5 zero border matters for initcheck), K-B CostRegNet (train + eval BN, fp32 and
fp16 output), the K-C render kernels (both entries, fp32 and fp16 volume), the peer sink, the backward kernel + reduce +
both Adam kernels, layout helpers."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from mvsnerf_b200 import backend, lib, synthetic  # noqa: E402

dev = torch.device("cuda", 0)
fn, mvs = backend.MVSNeRF().to(dev), backend.MVSNet().to(dev).train()
backend.load_weights_npz(fn, mvs, os.path.join(ROOT, "tests", "golden", "mvsnerf_v0_weights.npz"))
sc = synthetic.make_scene(32, 32, pad=4, seed=0)
d = sc.to(dev)
only = set(sys.argv[1:])          # optionally restrict: encoder render backward
with torch.no_grad():
    vol, _, _ = mvs(d.imgs_norm, d.proj_mats, sc.near_far, pad=sc.pad, return_color=True)
    if not only or "encoder" in only:
        mvs.eval()(d.imgs_norm, d.proj_mats, sc.near_far, pad=sc.pad)
        mvs.train()
        mvs(d.imgs_norm, d.proj_mats, sc.near_far, pad=sc.pad, volume_dtype=torch.float16)   # fp16 encoder output
    rays = synthetic.scene_rays(sc)[::3].contiguous().to(dev)
    if not only or "render" in only:
        for mode in (lib.MLP_FP32, lib.MLP_TC_HALF, lib.MLP_TC_SPLIT, lib.MLP_TC_PAIR):
            frame = torch.zeros(rays.shape[0] + 8, 4, device=dev)
            sink = lib.PeerSink()
            sink.frame[0], sink.n_peers, sink.first_pixel = frame.data_ptr(), 1, 5
            backend.render_rays(rays, vol, d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad), N_samples=24, mlp_mode=mode,
                                out=(torch.empty(rays.shape[0], 3, device=dev), torch.empty(rays.shape[0], device=dev)), sink=sink)
            if mode != lib.MLP_FP32:
                # early ray termination (the STOP instantiations): 1994 rays x 128 samples = 499 groups of 4 rays, 8 tiles
                # each, so CTAs hand out up to four groups through the shared counter, one CTA three (its second consumer
                # runs idle passes), and the last group is ragged; t_stop 0 never stops, 0.5 stops some groups, 2 all
                many = torch.cat([synthetic.scene_rays(sc)] * 2)[:1994].contiguous().to(dev)
                for t_stop in (0.0, 0.5, 2.0):
                    backend.render_rays(many, vol, d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad), N_samples=128,
                                        mlp_mode=mode, t_stop=t_stop, tiles_done=torch.zeros(1, dtype=torch.int64, device=dev))
                # empty-space skipping: the grid build (node samples through the split samples entry, cell reduction,
                # dilation, packing), then the range pre-pass and the STOP kernels with a range table -- the built grid,
                # an empty one (every group stored by the pre-pass) and a full one, on the same 1994-ray shape
                occ = backend.build_occupancy(vol, d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad), dilate=1)
                empty = backend.Occupancy(torch.zeros_like(occ.bits), occ.D, occ.Hp, occ.Wp, sc.near_far, sc.pad, False, 1)
                full = backend.Occupancy(torch.full_like(occ.bits, -1), occ.D, occ.Hp, occ.Wp, sc.near_far, sc.pad, False, 1)
                for grid in (occ, empty, full):
                    backend.render_rays(many, vol, d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad), N_samples=128,
                                        mlp_mode=mode, t_stop=0.5, occupancy=grid, white_bkgd=True)
                # importance sampling: the density grid (fp32 tile over the node samples, fp32 and fp16 volumes), the
                # sampler marching the 1994 rays (S + K = 88, random draws) into the samples entry, and the sampler on
                # given samples (ray_marcher_fine, S + K = 1024: the largest sort)
                den = backend.build_density(vol, d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad))
                backend.build_density(vol.half(), d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad))
                backend.render_rays(many, vol, d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad), N_samples=64,
                                    mlp_mode=mode, t_stop=0.5, density=den, N_importance=24,
                                    importance_u=torch.rand(many.shape[0], 24, device=dev))
                xyz_i, _, _, z_i = backend.ray_marcher(many[:300], N_samples=1000)
                ndc_i = backend.get_ndc_coordinate(d.pose_source["w2cs"][0], d.pose_source["intrinsics"][0], xyz_i,
                                                   torch.tensor([sc.W - 1.0, sc.H - 1.0], device=dev),
                                                   near=sc.near_far[0], far=sc.near_far[1], pad=sc.pad)
                backend.ray_marcher_fine(many[:300], den, z_i, ndc_i, N_importance=24)
                # fp16 volume (MVSN_VOLUME_F16): channels-last in place, then planar through mvsn_volume_to_half; both
                # entries, the sink and the STOP instantiations
                for vh in (vol.half(), vol.contiguous().half()):
                    backend.render_rays(rays, vh, d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad), N_samples=24,
                                        mlp_mode=mode, out=(torch.empty(rays.shape[0], 3, device=dev),
                                                            torch.empty(rays.shape[0], device=dev)), sink=sink)
                    backend.render_rays(many, vh, d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad), N_samples=128,
                                        mlp_mode=mode, t_stop=0.5, tiles_done=torch.zeros(1, dtype=torch.int64, device=dev))
                    occ_h = backend.build_occupancy(vh, d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad))
                    backend.render_rays(many, vh, d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad), N_samples=128,
                                        mlp_mode=mode, occupancy=occ_h)
                    xyz_h, _, rd_h, z_h = backend.ray_marcher(rays[:100], N_samples=24)
                    ndc_h = backend.get_ndc_coordinate(d.pose_source["w2cs"][0], d.pose_source["intrinsics"][0], xyz_h,
                                                       torch.tensor([sc.W - 1.0, sc.H - 1.0], device=dev),
                                                       near=sc.near_far[0], far=sc.near_far[1], pad=sc.pad)

                    class AH:
                        use_color_volume = False
                    backend.rendering(AH(), d.pose_source, xyz_h, ndc_h, z_h, None, rd_h, volume_feature=vh, imgs=d.imgs_raw,
                                      network_fn=fn, mlp_mode=mode)
            xyz, _, rd, z = backend.ray_marcher(rays[:100], N_samples=24)
            ndc = backend.get_ndc_coordinate(d.pose_source["w2cs"][0], d.pose_source["intrinsics"][0], xyz,
                                             torch.tensor([sc.W - 1.0, sc.H - 1.0], device=dev), near=sc.near_far[0],
                                             far=sc.near_far[1], pad=sc.pad)

            class A:
                use_color_volume = False
            backend.rendering(A(), d.pose_source, xyz, ndc, z, None, rd, volume_feature=backend.RefVolume(vol.contiguous().clone()),
                              imgs=d.imgs_raw, network_fn=fn, mlp_mode=mode)
    if not only or "render" in only:
        dirs = torch.randn(16, 24, 3, device=dev)
        backend.get_rays(dirs, d.pose_source["c2ws"][0], sc.near_far[0], sc.near_far[1])          # mvsn_make_rays
if not only or "backward" in only:
    # channels-last volume (what MVSNet.forward returns: element-wise Adam kernel), then checkpoint layout (planar kernel)
    for volume in (backend.RefVolume(vol.detach().clone()), backend.RefVolume(vol.detach().contiguous().clone())):
        tuner = backend.FineTuner(fn, volume, d.imgs_raw, d.pose_source, lr=1e-4)
        print("sanitize_smoke: FineTuner planar =", tuner.planar)
        for S in (32, 48, 128):
            xyz, _, rd, z = backend.ray_marcher(rays[:37], N_samples=S, perturb=1.0)
            ndc = backend.get_ndc_coordinate(d.pose_source["w2cs"][0], d.pose_source["intrinsics"][0], xyz,
                                             torch.tensor([sc.W - 1.0, sc.H - 1.0], device=dev), near=sc.near_far[0],
                                             far=sc.near_far[1], pad=sc.pad)
            tuner.step(xyz, ndc, z, rd, torch.rand(37, 3, device=dev), want_forward=True)
            # the same step from rays (mvsn_render_backward_rays), with and without jitter, then deterministic
            tuner.step_rays(rays[:37], torch.rand(37, 3, device=dev), sc.near_far, float(sc.pad), N_samples=S,
                            want_forward=True)
            tuner.step_rays(rays[:37], torch.rand(37, 3, device=dev), sc.near_far, float(sc.pad), N_samples=S, perturb=0.0)
            torch.use_deterministic_algorithms(True, warn_only=True)
            tuner.step_rays(rays[:37], torch.rand(37, 3, device=dev), sc.near_far, float(sc.pad), N_samples=S)
            torch.use_deterministic_algorithms(False)
    # early ray termination (mvsn_render_backward_rays_stop): 400 rays x 128 samples = 400 one-ray groups on up to 132
    # CTAs, t_stop = 0.5 stops rays at different depths, so some tiles are back-propagated at once, others deferred, and
    # a CTA's deferred rays fill packed tiles of which the last is partial; every grad mode and summation order
    many = torch.cat([synthetic.scene_rays(sc)] * 2)[:400].contiguous().to(dev)
    for mode in (lib.MLP_FP32, lib.MLP_TC_HALF, lib.GRAD_TC_FULL):
        for det in (False, True):
            torch.use_deterministic_algorithms(det, warn_only=True)
            tiles = torch.zeros(3, dtype=torch.int64, device=dev)
            live = torch.empty(400, dtype=torch.int32, device=dev)
            backend.render_backward_rays(many, vol, d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad), N_samples=128,
                                         jitter=torch.rand(400, 128, device=dev), target_rgb=torch.rand(400, 3, device=dev),
                                         want_forward=True, grad_mode=mode, t_stop=0.5, live_samples=live, tiles_done=tiles)
            print("sanitize_smoke: backward stop", mode, det, "tiles", tiles.tolist())
            torch.use_deterministic_algorithms(False)
    # grad_mode GRAD_TC_FULL without early termination (mvsn_render_backward_rays), S 32 / 48 / 128, both orders
    tuner = backend.FineTuner(fn, backend.RefVolume(vol.detach().clone()), d.imgs_raw, d.pose_source, lr=1e-4,
                              grad_mode=lib.GRAD_TC_FULL)
    for S in (32, 48, 128):
        for det in (False, True):
            torch.use_deterministic_algorithms(det, warn_only=True)
            tuner.step_rays(rays[:37], torch.rand(37, 3, device=dev), sc.near_far, float(sc.pad), N_samples=S,
                            want_forward=True)
            torch.use_deterministic_algorithms(False)
torch.cuda.synchronize()
print("sanitize_smoke: done")
