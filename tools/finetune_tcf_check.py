#!/usr/bin/env python
"""grad_mode GRAD_TC_FULL (the forward recompute on tensor cores) against MLP_TC_HALF in the fine-tuning step from rays,
measured in one command:

    python tools/finetune_tcf_check.py [--steps 20] [--runs 3] [--conv-steps 2000] [--json out.json]

  * timing: the config-3 step (1024 rays x 128 samples, encoding volume 8x128x200x200, white_bkgd, perturb 1) with
    FineTuner.step_rays in MLP_TC_HALF and GRAD_TC_FULL, each with t_stop None and 1e-4, on the bench scene
    (synthetic.make_scene) and the plane scene (synthetic.make_plane_scene, rays become opaque), both 800x800.  The
    variants alternate; each is run `--runs` times, each run the median of `--steps` steps timed with CUDA events.  The
    backward call alone (render_backward_rays on a fixed batch) is timed the same way;
  * convergence: FineTuner.step_rays from the same start on the same batches in MLP_FP32, MLP_TC_HALF and GRAD_TC_FULL
    on a 128x160 synthetic scene (rays of source views 1 and 2 against their images): the loss every 100 steps and the
    PSNR of the held-out reference view rendered after fine-tuning;
  * the card's name, SM clocks and power limit, read before and after.
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

WEIGHTS = os.path.join(ROOT, "tests", "golden", "mvsnerf_v0_weights.npz")
MODES = (("tc_half", lib.MLP_TC_HALF), ("tc_full", lib.GRAD_TC_FULL))
EPS = (None, 1e-4)


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


def timing(dev, fn, mvs, steps, runs, report):
    B, S = 1024, 128
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
        tuners = {m: backend.FineTuner(fn, backend.RefVolume(vol.detach().clone()), d.imgs_raw, d.pose_source, lr=0.0,
                                       white_bkgd=True, grad_mode=gm) for m, gm in MODES}   # lr 0: the same model
        variants = [(m, gm, eps) for m, gm in MODES for eps in EPS]
        fwd = {}
        for m, gm, eps in variants:                            # outputs of one fixed batch
            loss = torch.zeros(1, device=dev)
            _, _, rgb, _ = backend.render_backward_rays(rays0, tuners[m].volume, d.imgs_raw, d.pose_source, fn,
                                                        sc.near_far, 0.0, N_samples=S, jitter=jit0, white_bkgd=True,
                                                        target_rgb=tgt0, want_forward=True, loss_out=loss, grad_mode=gm,
                                                        t_stop=eps)
            fwd[(m, eps)] = (rgb, float(loss))

        def step(m, eps):
            idx = torch.randint(0, rays_all.shape[0], (B,), device=dev, generator=gen)
            tuners[m].step_rays(rays_all[idx], target_all[idx], sc.near_far, 0.0, N_samples=S, perturb=1.0, t_stop=eps)

        def kernel(m, gm, eps):
            t = tuners[m]
            backend.render_backward_rays(rays0, t.volume, d.imgs_raw, d.pose_source, fn, sc.near_far, 0.0, N_samples=S,
                                         jitter=jit0, white_bkgd=True, target_rgb=tgt0, grad_mode=gm, t_stop=eps,
                                         want_volume_grad=True, grad_volume=t.vol_g, grad_mlp=t.g)

        for m, gm, eps in variants:                            # warm-up
            for _ in range(3):
                step(m, eps)
                kernel(m, gm, eps)
        t_step = {(m, e): [] for m, _, e in variants}
        t_kern = {(m, e): [] for m, _, e in variants}
        for _ in range(runs):
            for m, gm, eps in variants:                        # alternate the variants
                t_step[(m, eps)].append(timed(lambda: step(m, eps), steps))
                t_kern[(m, eps)].append(timed(lambda: kernel(m, gm, eps), steps))
        for m, gm, eps in variants:
            ms, ks = statistics.median(t_step[(m, eps)]), statistics.median(t_kern[(m, eps)])
            ref_ms, ref_ks = statistics.median(t_step[("tc_half", eps)]), statistics.median(t_kern[("tc_half", eps)])
            row = {"scene": name, "grad_mode": m, "t_stop": eps, "step_ms": round(ms, 4),
                   "step_ms_runs": [round(x, 4) for x in t_step[(m, eps)]], "step_vs_tc_half": round(ms / ref_ms, 4),
                   "backward_ms": round(ks, 4), "backward_ms_runs": [round(x, 4) for x in t_kern[(m, eps)]],
                   "backward_vs_tc_half": round(ks / ref_ks, 4),
                   "max_abs_drgb_vs_tc_half": float((fwd[(m, eps)][0] - fwd[("tc_half", eps)][0]).abs().max()),
                   "loss": fwd[(m, eps)][1]}
            report["rows"].append(row)
            print(json.dumps(row), flush=True)


def convergence(dev, grad_mode, steps, batch=1024, S=128):
    fn, mvs = backend.MVSNeRF().to(dev), backend.MVSNet().to(dev).train()
    backend.load_weights_npz(fn, mvs, WEIGHTS)
    sc = synthetic.make_scene(128, 160, pad=8, seed=5)
    d = sc.to(dev)
    with torch.no_grad():
        vol, _, _ = mvs(d.imgs_norm, d.proj_mats, sc.near_far, pad=sc.pad)
    volume = backend.RefVolume(vol.detach().clone())
    rays, tgts = [], []
    for v in (1, 2):                                            # training views; view 0 is held out
        rays.append(synthetic.scene_rays(sc, sc.pose_source["c2ws"][v]).to(dev))
        tgts.append(d.imgs_raw[0, v].permute(1, 2, 0).reshape(-1, 3))
    rays, tgts = torch.cat(rays), torch.cat(tgts).contiguous()
    tuner = backend.FineTuner(fn, volume, d.imgs_raw, d.pose_source, lr=5e-4, grad_mode=grad_mode)
    gen = torch.Generator(device=dev).manual_seed(0)
    curve = []
    for it in range(steps):
        idx = torch.randint(0, rays.shape[0], (batch,), device=dev, generator=gen)
        loss = tuner.step_rays(rays[idx], tgts[idx], sc.near_far, float(sc.pad), N_samples=S, perturb=1.0,
                               generator=gen)[0]
        if it % 100 == 0 or it == steps - 1:
            curve.append([it, float(loss)])
    with torch.no_grad():
        held = synthetic.scene_rays(sc, sc.pose_source["c2ws"][0]).to(dev)
        rgb = backend.render_rays(held, volume, d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad), N_samples=S)[0]
        mse = ((rgb - d.imgs_raw[0, 0].permute(1, 2, 0).reshape(-1, 3)) ** 2).mean().item()
    return {"loss_every_100": curve, "heldout_psnr_db": -10.0 * torch.log10(torch.tensor(mse)).item()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--conv-steps", type=int, default=2000)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("finetune_tcf_check: no CUDA device")
    dev = torch.device("cuda", 0)
    fn, mvs = backend.MVSNeRF().to(dev), backend.MVSNet().to(dev).train()
    backend.load_weights_npz(fn, mvs, WEIGHTS)
    report = {"gpu_before": gpu_state(), "steps": a.steps, "runs": a.runs, "rows": []}
    timing(dev, fn, mvs, a.steps, a.runs, report)
    report["convergence"] = {m: convergence(dev, gm, a.conv_steps)
                             for m, gm in (("fp32", lib.MLP_FP32),) + MODES}
    for m, c in report["convergence"].items():
        print(m, "loss", c["loss_every_100"][0][1], "->", c["loss_every_100"][-1][1], "held-out PSNR",
              round(c["heldout_psnr_db"], 3), flush=True)
    report["gpu_after"] = gpu_state()
    print("gpu (name, SM clock, max SM clock, power limit):", report["gpu_before"], "|", report["gpu_after"])
    if a.json:
        with open(a.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
