#!/usr/bin/env python
"""Early ray termination through the reference's call surface, measured.

Render: one 512x640 frame (128 samples, samples marched on the host with ray_marcher + get_ndc_coordinate beforehand)
through `rendering` under torch.no_grad, in the reference's 5120-ray chunks and as one call, with t_stop None / 0 /
1e-4, in TC_PAIR and TC_SPLIT, on the bench scene (synthetic.make_scene) and on a scene whose rays become opaque
(synthetic.make_plane_scene).  The time is the CUDA-event time of the `rendering` calls of a frame (the host march is
not in it).  Also: tiles computed as a fraction of all 64-sample tiles, max |rgb - rgb(None)| and PSNR against it.

Training step: config 3 (1024 rays x 128 samples, 800x800 scenes, encoding volume 8x128x200x200, white_bkgd,
perturb 1) as the reference's training_step does it -- ray_marcher, get_ndc_coordinate, `rendering` under autograd,
img2mse, loss.backward(), torch.optim.Adam -- and through FineTuner.step on the same marched samples, with t_stop None
and 1e-4 (MLP_FP32 backward).  Also: the live-sample fraction and max |rgb - rgb(None)| of one fixed batch.

Variants alternate; each is run `--runs` times, each run the median of `--frames` frames / `--steps` steps.  The card's
name, SM clock and power limit are read in the same call.

    python tools/rendering_stop_check.py [--frames 5] [--steps 10] [--runs 3] [--json out.json]
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from mvsnerf_b200 import backend, lib, synthetic  # noqa: E402

CHUNK = 5120


def gpu_state():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,clocks.sm,clocks.max.sm,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "n/a"
    return out


def timed(fn, n):
    ts = []
    for _ in range(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


def march(sc, d, rays, S, perturb=0):
    xyz, rays_o, rays_d, z = backend.ray_marcher(rays, N_samples=S, perturb=perturb)
    ndc = backend.get_ndc_coordinate(d.pose_source["w2cs"][0], d.pose_source["intrinsics"][0], xyz,
                                     torch.tensor([sc.W - 1.0, sc.H - 1.0], device=rays.device), near=sc.near_far[0],
                                     far=sc.near_far[1], pad=sc.pad)
    return xyz, ndc, z, rays_o, rays_d


def render_part(a, dev, fn, mvs, report):
    S = 128
    for name, make in (("bench", synthetic.make_scene), ("plane", synthetic.make_plane_scene)):
        sc = make(512, 640, seed=0)
        d = sc.to(dev)
        with torch.no_grad():
            vol, _, _ = mvs(d.imgs_norm, d.proj_mats, sc.near_far, pad=sc.pad)
        rays = synthetic.scene_rays(sc).to(dev).contiguous()
        N = rays.shape[0]
        whole = march(sc, d, rays, S)
        chunks = [tuple(t[i:i + CHUNK] for t in whole) for i in range(0, N, CHUNK)]
        tiles = torch.zeros(1, dtype=torch.int64, device=dev)
        args = SimpleNamespace()
        for mode, mname in ((lib.MLP_TC_PAIR, "pair"), (lib.MLP_TC_SPLIT, "split")):
            def frame(eps, parts):
                out = []
                with torch.no_grad():
                    for xyz, ndc, z, ro, rd in parts:
                        kw = {} if eps is None else {"t_stop": eps, "tiles_done": tiles}
                        out.append(backend.rendering(args, d.pose_source, xyz, ndc, z, ro, rd, vol, d.imgs_raw,
                                                     network_fn=fn, mlp_mode=mode, want_aux=False, **kw)[0])
                return out

            variants = [(eps, split) for split in ("chunks", "one call") for eps in (None, 0.0, 1e-4)]
            parts = {"chunks": chunks, "one call": [whole]}
            out = {}
            for eps, split in variants:
                tiles.zero_()
                rgb = torch.cat(frame(eps, parts[split]))
                torch.cuda.synchronize()
                out[(eps, split)] = (rgb, int(tiles.item()))
            times = {v: [] for v in variants}
            for v in variants:                                  # warm-up
                frame(v[0], parts[v[1]])
            for _ in range(a.runs):
                for v in variants:                              # alternate the variants
                    times[v].append(timed(lambda: frame(v[0], parts[v[1]]), a.frames))
            for split in ("chunks", "one call"):
                rt = 32
                all_tiles = sum(-(-p[0].shape[0] // rt) for p in parts[split]) * (S // (64 // rt))
                base = statistics.median(times[(None, split)])
                for eps in (None, 0.0, 1e-4):
                    ms = statistics.median(times[(eps, split)])
                    row = {"part": "render", "scene": name, "mode": mname, "calls": split, "t_stop": eps,
                           "ms": round(ms, 3), "ms_runs": [round(x, 3) for x in times[(eps, split)]],
                           "vs_none": round(ms / base, 4)}
                    if eps is not None:
                        diff = out[(eps, split)][0] - out[(None, split)][0]
                        mse = float((diff ** 2).mean())
                        row.update(tiles_fraction=round(out[(eps, split)][1] / all_tiles, 4),
                                   max_abs_drgb=float(diff.abs().max()),
                                   psnr_vs_none=(math.inf if mse == 0 else round(10 * math.log10(1.0 / mse), 2)))
                    report["rows"].append(row)
                    print(json.dumps(row), flush=True)


def step_part(a, dev, fn0, mvs, report):
    B, S = 1024, 128
    wpath = os.path.join(ROOT, "tests", "golden", "mvsnerf_v0_weights.npz")
    for name, make in (("bench", synthetic.make_scene), ("plane", synthetic.make_plane_scene)):
        sc = make(800, 800, pad=0, seed=3, near_far=(2.0, 6.0)) if name == "bench" else make(800, 800, pad=0, seed=3)
        d = sc.to(dev)
        with torch.no_grad():
            vol, _, _ = mvs(d.imgs_norm, d.proj_mats, sc.near_far, pad=0)
        rays_all = synthetic.scene_rays(sc).to(dev)
        target_all = d.imgs_raw[0, 0].permute(1, 2, 0).reshape(-1, 3).contiguous()
        fn = backend.MVSNeRF().to(dev)
        backend.load_weights_npz(fn, None, wpath)
        volume = backend.RefVolume(vol.detach().clone())
        optimizer = torch.optim.Adam(list(fn.parameters()) + [volume.feat_volume], lr=0.0)   # every variant: same model
        tuner = backend.FineTuner(fn, volume, d.imgs_raw, d.pose_source, lr=0.0, white_bkgd=True)
        gen = torch.Generator(device=dev).manual_seed(0)
        args = SimpleNamespace()

        def batch():
            idx = torch.randint(0, rays_all.shape[0], (B,), device=dev, generator=gen)
            return rays_all[idx], target_all[idx]

        def autograd_step(eps):
            rays, tgt = batch()
            xyz, ndc, z, ro, rd = march(sc, d, rays, S, perturb=1.0)
            kw = {} if eps is None else {"t_stop": eps}
            rgb = backend.rendering(args, d.pose_source, xyz, ndc, z, ro, rd, volume, d.imgs_raw, network_fn=fn,
                                    white_bkgd=True, **kw)[0]
            loss = torch.mean((rgb - tgt) ** 2)
            optimizer.zero_grad()
            loss.backward()
            optimizer.step()

        def tuner_step(eps):
            rays, tgt = batch()
            xyz, ndc, z, _, rd = march(sc, d, rays, S, perturb=1.0)
            tuner.step(xyz, ndc, z, rd, tgt, t_stop=eps)

        rays0, tgt0 = batch()
        smp0 = march(sc, d, rays0, S, perturb=1.0)
        fixed = {}
        for eps in (None, 1e-4):
            live = torch.zeros(B, dtype=torch.int32, device=dev) if eps is not None else None
            kw = {} if eps is None else {"t_stop": eps, "live_samples": live}
            _, _, rgb, _ = backend.render_backward(d.pose_source, smp0[0], smp0[1], smp0[2], smp0[4], volume, d.imgs_raw,
                                                   fn, True, target_rgb=tgt0, want_forward=True, **kw)
            torch.cuda.synchronize()
            fixed[eps] = (rgb, None if live is None else float(live.float().mean()) / S)
        variants = [(path, eps) for path in ("rendering+backward+Adam", "FineTuner.step") for eps in (None, 1e-4)]
        run = {"rendering+backward+Adam": autograd_step, "FineTuner.step": tuner_step}
        for path, eps in variants:                              # warm-up
            for _ in range(3):
                run[path](eps)
        times = {v: [] for v in variants}
        for _ in range(a.runs):
            for v in variants:
                times[v].append(timed(lambda: run[v[0]](v[1]), a.steps))
        for path, eps in variants:
            ms = statistics.median(times[(path, eps)])
            row = {"part": "step", "scene": name, "path": path, "t_stop": eps, "step_ms": round(ms, 3),
                   "step_ms_runs": [round(x, 3) for x in times[(path, eps)]],
                   "vs_none": round(ms / statistics.median(times[(path, None)]), 4), "live_fraction": fixed[eps][1],
                   "max_abs_drgb": float((fixed[eps][0] - fixed[None][0]).abs().max())}
            report["rows"].append(row)
            print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    fn, mvs = backend.MVSNeRF().to(dev), backend.MVSNet().to(dev).train()
    backend.load_weights_npz(fn, mvs, os.path.join(ROOT, "tests", "golden", "mvsnerf_v0_weights.npz"))
    report = {"gpu_before": gpu_state(), "frames": a.frames, "steps": a.steps, "runs": a.runs, "rows": []}
    render_part(a, dev, fn, mvs, report)
    step_part(a, dev, fn, mvs, report)
    report["gpu_after"] = gpu_state()
    print("gpu (name, SM clock, max SM clock, power limit):", report["gpu_before"], "|", report["gpu_after"])
    if a.json:
        with open(a.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
