#!/usr/bin/env python
"""Fine-tuning with and without torch.use_deterministic_algorithms on one GPU, in one command:

    python tools/finetune_det_check.py OUT_DIR [--steps 200]

Writes OUT_DIR/finetune_det_check.json with
  * gpu: the card's name and power limit, read in this call (and again at the end);
  * timing: the BASELINE config-3 step of backend.finetune_step_timing (800x800 Blender-shaped scene, volume
    8x128x200x200, 1024 rays x 128 samples, white_bkgd, perturb 1) with the flag off and on, in both grad modes,
    alternated, three runs each: the median CUDA-event step time of the fused FineTuner step and of the autograd path;
  * kernel_mean_ms_per_call: with the flag on, torch.profiler's mean device time per call (and call count) of the
    backward kernel and of the kernels the deterministic path adds (fixed-point scatter, conversion, loss reduction,
    the accumulator memset), in a separate run of finetune_step_timing;
  * repeat: two FineTuner runs of --steps steps from the same start on the same batches (128x160 synthetic scene),
    with the flag on and with it off, in each grad mode: the largest differences between the two runs' parameters,
    volumes and losses.  Measured, not asserted: with the flag on they are expected to be zero.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

WEIGHTS = os.path.join(ROOT, "tests", "golden", "mvsnerf_v0_weights.npz")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def set_flag(on):
    torch.use_deterministic_algorithms(on, warn_only=True)


def kernel_times(dev, grad_mode, steps=10):
    from torch.profiler import ProfilerActivity, profile
    from mvsnerf_b200 import backend
    set_flag(True)
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            backend.finetune_step_timing(dev, WEIGHTS, steps=steps, warmup=2, grad_mode=grad_mode)
            torch.cuda.synchronize()
    finally:
        set_flag(False)
    out = {}
    for e in prof.key_averages():
        for k in ("render_bwd_tc_kernel", "render_bwd_kernel", "det_scatter_kernel", "det_convert_kernel",
                  "loss_reduce_kernel", "mlp_grad_reduce_kernel", "adam_volume", "Memset"):
            if k in e.key:
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                prev = out.get(k, {"total_ms": 0.0, "calls": 0})
                out[k] = {"total_ms": prev["total_ms"] + t / 1e3, "calls": prev["calls"] + e.count}
                break
    for v in out.values():
        v["mean_ms_per_call"] = v["total_ms"] / max(v["calls"], 1)
    return out


def finetune_run(dev, grad_mode, steps, batch=1024, S=128):
    from mvsnerf_b200 import backend, synthetic
    fn, mvs = backend.MVSNeRF().to(dev), backend.MVSNet().to(dev).train()
    backend.load_weights_npz(fn, mvs, WEIGHTS)
    sc = synthetic.make_scene(128, 160, pad=8, seed=5)
    d = sc.to(dev)
    with torch.no_grad():
        vol, _, _ = mvs(d.imgs_norm, d.proj_mats, sc.near_far, pad=sc.pad)
    volume = backend.RefVolume(vol.detach().clone())
    inv_scale = torch.tensor([sc.W - 1.0, sc.H - 1.0], device=dev)
    rays = synthetic.scene_rays(sc, sc.pose_source["c2ws"][1]).to(dev)
    tgts = d.imgs_raw[0, 1].permute(1, 2, 0).reshape(-1, 3).contiguous()
    tuner = backend.FineTuner(fn, volume, d.imgs_raw, d.pose_source, lr=5e-4, grad_mode=grad_mode)
    gen = torch.Generator(device=dev).manual_seed(0)
    torch.manual_seed(0)
    losses = []
    for _ in range(steps):
        idx = torch.randint(0, rays.shape[0], (batch,), device=dev, generator=gen)
        xyz, _, rd, z = backend.ray_marcher(rays[idx], N_samples=S, perturb=1.0)
        ndc = backend.get_ndc_coordinate(d.pose_source["w2cs"][0], d.pose_source["intrinsics"][0], xyz, inv_scale,
                                         near=sc.near_far[0], far=sc.near_far[1], pad=sc.pad)
        losses.append(tuner.step(xyz, ndc, z, rd, tgts[idx])[0].clone())
    return [p.detach().clone() for p in fn.ordered_params()], volume.feat_volume.detach().clone(), torch.cat(losses)


def repeat(dev, grad_mode, steps, flag):
    set_flag(flag)
    try:
        a, b = finetune_run(dev, grad_mode, steps), finetune_run(dev, grad_mode, steps)
    finally:
        set_flag(False)
    return {"max_abs_param_diff": max((x - y).abs().max().item() for x, y in zip(a[0], b[0])),
            "max_abs_volume_diff": (a[1] - b[1]).abs().max().item(),
            "max_abs_loss_diff": (a[2] - b[2]).abs().max().item(),
            "params_equal": all(torch.equal(x, y) for x, y in zip(a[0], b[0])),
            "volume_equal": torch.equal(a[1], b[1]), "losses_equal": torch.equal(a[2], b[2]),
            "loss_first_last": [a[2][0].item(), a[2][-1].item()]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("finetune_det_check: no CUDA device")
    os.makedirs(a.out_dir, exist_ok=True)
    from mvsnerf_b200 import backend, lib
    dev = torch.device("cuda", 0)
    modes = {"fp32": lib.MLP_FP32, "tc_half": lib.MLP_TC_HALF}
    res = {"gpu": gpu_info(), "timing": {f"{m}_{f}": [] for m in modes for f in ("off", "on")}}
    for _ in range(3):                                          # alternated
        for name, m in modes.items():
            for flag in (False, True):
                set_flag(flag)
                try:
                    r = backend.finetune_step_timing(dev, WEIGHTS, grad_mode=m)
                finally:
                    set_flag(False)
                res["timing"][f"{name}_{'on' if flag else 'off'}"].append(
                    {"fused_ms": r["fused_ms"], "autograd_adam_ms": r["autograd_adam_ms"]})
    res["kernel_mean_ms_per_call"] = {name: kernel_times(dev, m) for name, m in modes.items()}
    res["repeat"] = {f"{name}_{'on' if flag else 'off'}": repeat(dev, m, a.steps, flag)
                     for name, m in modes.items() for flag in (True, False)}
    res["gpu_after"] = gpu_info()
    with open(os.path.join(a.out_dir, "finetune_det_check.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
