"""Importance sampling on the H100: build_density, the sampler and the frame / fine-tuning cost of N_samples + K.

    python tools/importance_check.py [--json report.json] [--psnr-steps 2000]

Reports, with the card's name and power limit read in the same run:
  * build_density ms on the plane scene at 512x640 and 960x640 (pad 24);
  * mvsn_sample_importance ms per 512x640 frame (64 + 64);
  * render_rays frame ms per mode for uniform 128, 64 + 64 and 128 + 64 (importance_u None: linspace draws);
  * the fine-tuning step (1024 rays, FineTuner.step_rays, FP32, plane scene) for uniform 128 against 64 + 64;
  * held-out PSNR of the two after --psnr-steps steps on the plane scene (every 8th pixel held out).
Median of CUDA-event timings after warm-up.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mvsnerf_b200 import backend, lib, synthetic  # noqa: E402

DEV = "cuda"


def timed(fn, reps=10, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); e.record(); e.synchronize()
        ts.append(a.elapsed_time(e))
    return sorted(ts)[len(ts) // 2]


def scene(H, W, fn, mvs):
    sc = synthetic.make_plane_scene(H, W, seed=0)
    d = sc.to(DEV)
    with torch.no_grad():
        vol, _, _ = mvs(d.imgs_norm, d.proj_mats, sc.near_far, pad=sc.pad)
    return sc, d, vol, synthetic.scene_rays(sc).to(DEV).contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None, help="also write the report to this file")
    ap.add_argument("--psnr-steps", type=int, default=2000)
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    out = {"gpu": smi}
    fn, mvs = backend.MVSNeRF().to(DEV), backend.MVSNet().to(DEV).train()
    backend.load_weights_npz(fn, mvs, os.path.join(ROOT, "tests", "golden", "mvsnerf_v0_weights.npz"))
    for H, W in ((512, 640), (960, 640)):
        sc, d, vol, _ = scene(H, W, fn, mvs)

        def build():
            backend.clear_cache()
            backend.build_density(vol, d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad))
        out[f"build_density_ms_{H}x{W}"] = timed(build, reps=5, warmup=2)
        out[f"volume_{H}x{W}"] = list(vol.shape)
    sc, d, vol, rays = scene(512, 640, fn, mvs)
    nf, pad = sc.near_far, float(sc.pad)
    den = backend.build_density(vol, d.imgs_raw, d.pose_source, fn, nf, pad)
    out["sampler_ms_64+64"] = timed(lambda: backend.sample_importance(rays, den, vol, d.imgs_raw, d.pose_source, fn, nf, pad,
                                                                      N_samples=64, N_importance=64))
    frames = {}
    with torch.no_grad():
        for name, mode in (("fp32", lib.MLP_FP32), ("half", lib.MLP_TC_HALF), ("pair", lib.MLP_TC_PAIR),
                           ("split", lib.MLP_TC_SPLIT)):
            r = {"uniform_128": timed(lambda: backend.render_rays(rays, vol, d.imgs_raw, d.pose_source, fn, nf, pad,
                                                                  N_samples=128, mlp_mode=mode), reps=5)}
            for S, K in ((64, 64), (128, 64)):
                r[f"{S}+{K}"] = timed(lambda: backend.render_rays(rays, vol, d.imgs_raw, d.pose_source, fn, nf, pad,
                                                                  N_samples=S, mlp_mode=mode, density=den,
                                                                  N_importance=K), reps=5)
            frames[name] = r
    out["frame_ms"] = frames
    target = d.imgs_raw[0, 0].permute(1, 2, 0).reshape(-1, 3).contiguous()
    idx = torch.arange(rays.shape[0], device=DEV)
    train_idx, test_idx = idx[idx % 8 != 0], idx[idx % 8 == 0]

    def run(imp, steps):
        f2 = backend.MVSNeRF().to(DEV)
        backend.load_weights_npz(f2, None, os.path.join(ROOT, "tests", "golden", "mvsnerf_v0_weights.npz"))
        v2 = backend.RefVolume(vol.detach().clone()).to(DEV)
        t = backend.FineTuner(f2, v2, d.imgs_raw, d.pose_source, lr=5e-4)
        g = torch.Generator(device=DEV).manual_seed(0)
        held = [backend.build_density(v2, d.imgs_raw, d.pose_source, f2, nf, pad)] if imp else []

        def step():
            b = train_idx[torch.randint(0, train_idx.numel(), (1024,), device=DEV, generator=g)]
            if imp:
                t.step_rays(rays[b], target[b], nf, pad, N_samples=64, generator=g, density=held[0], N_importance=64)
            else:
                t.step_rays(rays[b], target[b], nf, pad, N_samples=128, generator=g)
        ms = timed(step, reps=20, warmup=5)
        for i in range(steps):
            if imp and i % 200 == 0:                  # the reference refreshes the grid every 200 steps
                held[0] = backend.build_density(v2, d.imgs_raw, d.pose_source, f2, nf, pad)
            step()
        with torch.no_grad():
            tr = rays[test_idx]
            if imp:
                dn = backend.build_density(v2, d.imgs_raw, d.pose_source, f2, nf, pad)
                rgb, _ = backend.render_rays(tr, v2, d.imgs_raw, d.pose_source, f2, nf, pad, N_samples=64, density=dn,
                                             N_importance=64)
            else:
                rgb, _ = backend.render_rays(tr, v2, d.imgs_raw, d.pose_source, f2, nf, pad, N_samples=128)
        mse = torch.mean((rgb - target[test_idx]) ** 2).item()
        return ms, -10.0 * torch.log10(torch.tensor(mse)).item()
    for name, imp in (("uniform_128", False), ("64+64", True)):
        ms, psnr = run(imp, a.psnr_steps)
        out[f"finetune_{name}"] = {"step_ms": ms, "heldout_psnr": psnr, "steps": a.psnr_steps}
    print(json.dumps(out, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
