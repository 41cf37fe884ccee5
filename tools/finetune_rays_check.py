#!/usr/bin/env python
"""Fine-tuning from rays: FineTuner.step(*host march) against FineTuner.step_rays on one GPU, in one command:

    python tools/finetune_rays_check.py OUT_DIR [--steps 50] [--warmup 5]

The shape is BASELINE config 3 (backend.finetune_step_timing's scene: 800x800 Blender-shaped, pad 0, white_bkgd,
near_far [2, 6], encoding volume 8x128x200x200; 1024 rays x 128 samples, perturb 1).  Each timed step is what a training
loop does per step: random batch selection, sample preparation (host: ray_marcher + get_ndc_coordinate; rays: the
jitter draw inside step_rays) and the step itself, between two CUDA events.  Writes OUT_DIR/finetune_rays_check.json:
  * gpu: the card's name and power limit, read in this call (and again at the end);
  * timing: median ms per step, both forms in both grad modes, alternated, three runs each;
  * peak_mem: the peak allocated memory during each timed loop, and its excess over what was allocated before it;
  * kernels_per_step: CUDA kernel launches (and memsets / copies) per step from torch.profiler, in a separate run.
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
BATCH, S = 1024, 128


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


class Config3:
    def __init__(self, dev):
        from mvsnerf_b200 import backend, synthetic
        self.backend = backend
        self.fn, mvs = backend.MVSNeRF().to(dev), backend.MVSNet().to(dev).train()
        backend.load_weights_npz(self.fn, mvs, WEIGHTS)
        self.sc = synthetic.make_scene(800, 800, pad=0, seed=3, near_far=(2.0, 6.0))
        self.d = self.sc.to(dev)
        with torch.no_grad():
            self.vol, _, _ = mvs(self.d.imgs_norm, self.d.proj_mats, self.sc.near_far, pad=0)
        self.rays_all = synthetic.scene_rays(self.sc).to(dev)
        self.target_all = self.d.imgs_raw[0, 0].permute(1, 2, 0).reshape(-1, 3).contiguous()
        self.inv_scale = torch.tensor([self.sc.W - 1.0, self.sc.H - 1.0], device=dev)
        self.dev = dev

    def tuner(self, grad_mode):
        b = self.backend
        return b.FineTuner(self.fn, b.RefVolume(self.vol.detach().clone()), self.d.imgs_raw, self.d.pose_source, lr=5e-4,
                           white_bkgd=True, grad_mode=grad_mode)

    def step_fn(self, tuner, form, gen):
        b, d, sc = self.backend, self.d, self.sc

        def host():
            idx = torch.randint(0, self.rays_all.shape[0], (BATCH,), device=self.dev, generator=gen)
            rays, tgt = self.rays_all[idx], self.target_all[idx]
            xyz, _, rd, z = b.ray_marcher(rays, N_samples=S, perturb=1.0)
            ndc = b.get_ndc_coordinate(d.pose_source["w2cs"][0], d.pose_source["intrinsics"][0], xyz, self.inv_scale,
                                       near=sc.near_far[0], far=sc.near_far[1], pad=0)
            return tuner.step(xyz, ndc, z, rd, tgt)[0]

        def rays():
            idx = torch.randint(0, self.rays_all.shape[0], (BATCH,), device=self.dev, generator=gen)
            return tuner.step_rays(self.rays_all[idx], self.target_all[idx], sc.near_far, 0.0, N_samples=S, perturb=1.0)[0]

        return host if form == "host" else rays


def timed(cfg, grad_mode, form, steps, warmup):
    tuner = cfg.tuner(grad_mode)
    gen = torch.Generator(device=cfg.dev).manual_seed(0)
    step = cfg.step_fn(tuner, form, gen)
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ts = []
    for _ in range(steps):
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        e.record()
        e.synchronize()
        ts.append(a.elapsed_time(e))
    peak = torch.cuda.max_memory_allocated()
    ts.sort()
    return ts[len(ts) // 2], {"peak_allocated_mb": peak / 2**20, "peak_over_steady_mb": (peak - base) / 2**20}


def kernels_per_step(cfg, grad_mode, form, steps=10):
    from torch.profiler import ProfilerActivity, profile
    tuner = cfg.tuner(grad_mode)
    gen = torch.Generator(device=cfg.dev).manual_seed(0)
    step = cfg.step_fn(tuner, form, gen)
    for _ in range(2):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    kernels = other = 0
    for ev in prof.events():
        if getattr(ev, "device_type", None) is None or "CUDA" not in str(ev.device_type):
            continue
        if "Memset" in ev.name or "Memcpy" in ev.name:
            other += 1
        else:
            kernels += 1
    return {"kernels": kernels / steps, "memsets_and_copies": other / steps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("finetune_rays_check: no CUDA device")
    os.makedirs(a.out_dir, exist_ok=True)
    from mvsnerf_b200 import lib
    dev = torch.device("cuda", 0)
    cfg = Config3(dev)
    modes = {"fp32": lib.MLP_FP32, "tc_half": lib.MLP_TC_HALF}
    keys = [f"{m}_{f}" for m in modes for f in ("host", "rays")]
    res = {"gpu": gpu_info(), "shape": {"rays": BATCH, "n_samples": S, "volume": list(cfg.vol.shape), "white_bkgd": True,
                                        "perturb": 1.0},
           "timing_ms": {k: [] for k in keys}, "peak_mem": {k: [] for k in keys}}
    for _ in range(3):                                          # alternated
        for name, m in modes.items():
            for form in ("host", "rays"):
                ms, mem = timed(cfg, m, form, a.steps, a.warmup)
                res["timing_ms"][f"{name}_{form}"].append(ms)
                res["peak_mem"][f"{name}_{form}"].append(mem)
    res["kernels_per_step"] = {f"{name}_{form}": kernels_per_step(cfg, m, form) for name, m in modes.items()
                               for form in ("host", "rays")}
    res["gpu_after"] = gpu_info()
    with open(os.path.join(a.out_dir, "finetune_rays_check.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
