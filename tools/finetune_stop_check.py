#!/usr/bin/env python
"""Early ray termination in the fine-tuning step, measured: the config-3 step from rays (1024 rays x 128 samples,
encoding volume 8x128x200x200, white_bkgd, perturb 1) with FineTuner.step_rays at t_stop in {None, 0, 1e-4, 1e-3}, in
MLP_FP32 and MLP_TC_HALF, on the bench scene (synthetic.make_scene: rays stay transparent) and on a scene whose rays
become opaque (synthetic.make_plane_scene), both 800x800.  Variants alternate; each is run `--runs` times, each run the
median of `--steps` steps timed with CUDA events (batch selection + step).  The backward kernel alone is timed the same
way (render_backward_rays on a fixed batch).  Also reported: the live-sample fraction, the three tile counters
(immediate, deferred, packed), max |rgb - rgb(None)| and |loss - loss(None)| of the first step, the card's name and
power limit.

    python tools/finetune_stop_check.py [--steps 20] [--runs 3] [--json out.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from mvsnerf_b200 import backend, lib, synthetic  # noqa: E402

EPS = [None, 0.0, 1e-4, 1e-3]


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    wpath = os.path.join(ROOT, "tests", "golden", "mvsnerf_v0_weights.npz")
    fn, mvs = backend.MVSNeRF().to(dev), backend.MVSNet().to(dev).train()
    backend.load_weights_npz(fn, mvs, wpath)
    B, S = 1024, 128
    report = {"gpu_before": gpu_state(), "steps": a.steps, "runs": a.runs, "rows": []}
    for name, make in (("bench", synthetic.make_scene), ("plane", synthetic.make_plane_scene)):
        sc = make(800, 800, pad=0, seed=3, near_far=(2.0, 6.0)) if name == "bench" else make(800, 800, pad=0, seed=3)
        d = sc.to(dev)
        with torch.no_grad():
            vol, _, _ = mvs(d.imgs_norm, d.proj_mats, sc.near_far, pad=0)
        rays_all = synthetic.scene_rays(sc).to(dev)
        target_all = d.imgs_raw[0, 0].permute(1, 2, 0).reshape(-1, 3).contiguous()
        gen = torch.Generator(device=dev).manual_seed(0)
        idx0 = torch.randint(0, rays_all.shape[0], (B,), device=dev, generator=gen)
        rays0, tgt0 = rays_all[idx0].contiguous(), target_all[idx0].contiguous()
        jit0 = torch.rand(B, S, device=dev, generator=gen)
        for mode, mname in ((lib.MLP_FP32, "fp32"), (lib.MLP_TC_HALF, "tc_half")):
            tuner = backend.FineTuner(fn, backend.RefVolume(vol.detach().clone()), d.imgs_raw, d.pose_source, lr=0.0,
                                      white_bkgd=True, grad_mode=mode)        # lr 0: every variant sees the same model
            fwd = {}
            for eps in EPS:                                     # outputs of one fixed batch, counters, live fraction
                live = torch.zeros(B, dtype=torch.int32, device=dev) if eps is not None else None
                tiles = torch.zeros(3, dtype=torch.int64, device=dev) if eps is not None else None
                loss = torch.zeros(1, device=dev)
                _, _, rgb, _ = backend.render_backward_rays(rays0, tuner.volume, d.imgs_raw, d.pose_source, fn, sc.near_far,
                                                            0.0, N_samples=S, jitter=jit0, white_bkgd=True, target_rgb=tgt0,
                                                            want_forward=True, loss_out=loss, grad_mode=mode, t_stop=eps,
                                                            live_samples=live, tiles_done=tiles)
                torch.cuda.synchronize()
                fwd[eps] = (rgb, float(loss), None if live is None else float(live.float().mean()) / S,
                            None if tiles is None else tiles.tolist())

            def step(eps):
                idx = torch.randint(0, rays_all.shape[0], (B,), device=dev, generator=gen)
                tuner.step_rays(rays_all[idx], target_all[idx], sc.near_far, 0.0, N_samples=S, perturb=1.0, t_stop=eps)

            def kernel(eps):
                backend.render_backward_rays(rays0, tuner.volume, d.imgs_raw, d.pose_source, fn, sc.near_far, 0.0,
                                             N_samples=S, jitter=jit0, white_bkgd=True, target_rgb=tgt0, grad_mode=mode,
                                             t_stop=eps, want_volume_grad=True, grad_volume=tuner.vol_g, grad_mlp=tuner.g)

            for eps in EPS:                                     # warm-up
                for _ in range(3):
                    step(eps)
                    kernel(eps)
            t_step = {e: [] for e in EPS}
            t_kern = {e: [] for e in EPS}
            for _ in range(a.runs):
                for eps in EPS:                                 # alternate the variants
                    t_step[eps].append(timed(lambda: step(eps), a.steps))
                    t_kern[eps].append(timed(lambda: kernel(eps), a.steps))
            base = statistics.median(t_step[None])
            base_k = statistics.median(t_kern[None])
            for eps in EPS:
                ms, ks = statistics.median(t_step[eps]), statistics.median(t_kern[eps])
                row = {"scene": name, "grad_mode": mname, "t_stop": eps, "step_ms": round(ms, 4),
                       "step_ms_runs": [round(x, 4) for x in t_step[eps]], "step_vs_none": round(ms / base, 4),
                       "backward_ms": round(ks, 4), "backward_ms_runs": [round(x, 4) for x in t_kern[eps]],
                       "backward_vs_none": round(ks / base_k, 4), "live_fraction": fwd[eps][2], "tiles": fwd[eps][3],
                       "max_abs_drgb": float((fwd[eps][0] - fwd[None][0]).abs().max()),
                       "abs_dloss": abs(fwd[eps][1] - fwd[None][1])}
                report["rows"].append(row)
                print(json.dumps(row), flush=True)
    report["gpu_after"] = gpu_state()
    print("gpu (name, SM clock, max SM clock, power limit):", report["gpu_before"], "|", report["gpu_after"])
    if a.json:
        with open(a.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
