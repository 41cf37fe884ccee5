#!/usr/bin/env python
"""Fine-tuning with grad_mode MLP_FP32 vs MLP_TC_HALF on one GPU, in one command:

    python tools/finetune_tc_check.py OUT_DIR [--conv-steps 2000]

Writes OUT_DIR/finetune_tc_check.json with
  * gpu: the card's name and power limit, read in this call;
  * timing: the BASELINE config-3 step of backend.finetune_step_timing (800x800 Blender-shaped scene, volume
    8x128x200x200, 1024 rays x 128 samples, white_bkgd, perturb 1), the two modes alternated, three runs each: the
    median CUDA-event step time; and per kernel (the backward kernel, the weight packs, the gradient reduction, the
    Adam kernels) the mean device time per call and the number
    of calls, from torch.profiler in a separate run of finetune_step_timing (warm-up and timed steps of both its fused
    and its autograd path; every one of these kernels runs once per step in either path);
  * forward_tile_ms: the fp32 render kernel alone on a batch of the same shape -- the forward recompute both
    backward kernels run first, so a bound on what a faster dgrad / wgrad can save;
  * convergence: FineTuner from the same start on the same batches in each mode on a 128x160 synthetic scene (rays of
    source views 1 and 2 against their images), the loss every 100 steps, and the PSNR of the held-out reference view
    rendered after fine-tuning against its image.
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


def kernel_times(dev, grad_mode, steps=10):
    """Mean device ms per call and number of calls of each kernel of the step, over one finetune_step_timing run
    (torch.profiler, CUDA activities)."""
    from torch.profiler import ProfilerActivity, profile
    from mvsnerf_b200 import backend
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        backend.finetune_step_timing(dev, WEIGHTS, steps=steps, warmup=2, grad_mode=grad_mode)
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        name = e.key
        for k in ("render_bwd_tc_kernel", "render_bwd_kernel", "pack_dgrad_half_kernel", "pack_dgrad_kernel",
                  "mlp_grad_reduce_kernel", "adam_tensors_kernel", "adam_volume", "render_fp32_kernel"):
            if k in name:
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                out[k] = {"mean_ms_per_call": t / 1e3 / max(e.count, 1), "calls": e.count}
                break
    return out


def forward_tile_ms(dev, batch=1024, S=128, reps=20):
    from mvsnerf_b200 import backend, lib, synthetic
    from types import SimpleNamespace
    fn, mvs = backend.MVSNeRF().to(dev), backend.MVSNet().to(dev).train()
    backend.load_weights_npz(fn, mvs, WEIGHTS)
    sc = synthetic.make_scene(800, 800, pad=0, seed=3, near_far=(2.0, 6.0))
    d = sc.to(dev)
    with torch.no_grad():
        vol, _, _ = mvs(d.imgs_norm, d.proj_mats, sc.near_far, pad=0)
    rays = synthetic.scene_rays(sc).to(dev)[:batch]
    xyz, _, rd, z = backend.ray_marcher(rays, N_samples=S, perturb=1.0)
    ndc = backend.get_ndc_coordinate(d.pose_source["w2cs"][0], d.pose_source["intrinsics"][0], xyz,
                                     torch.tensor([sc.W - 1.0, sc.H - 1.0], device=dev), near=2.0, far=6.0, pad=0)
    args = SimpleNamespace(use_color_volume=False)

    def run():
        with torch.no_grad():
            backend.rendering(args, d.pose_source, xyz, ndc, z, None, rd, volume_feature=vol, imgs=d.imgs_raw,
                              network_fn=fn, white_bkgd=True, mlp_mode=lib.MLP_FP32)
    for _ in range(3):
        run()
    ts = []
    for _ in range(reps):
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); run(); e.record(); e.synchronize()
        ts.append(a.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def convergence(dev, grad_mode, steps, batch=1024, S=128):
    from mvsnerf_b200 import backend, synthetic
    fn, mvs = backend.MVSNeRF().to(dev), backend.MVSNet().to(dev).train()
    backend.load_weights_npz(fn, mvs, WEIGHTS)
    sc = synthetic.make_scene(128, 160, pad=8, seed=5)
    d = sc.to(dev)
    with torch.no_grad():
        vol, _, _ = mvs(d.imgs_norm, d.proj_mats, sc.near_far, pad=sc.pad)
    volume = backend.RefVolume(vol.detach().clone())
    inv_scale = torch.tensor([sc.W - 1.0, sc.H - 1.0], device=dev)
    rays, tgts = [], []
    for v in (1, 2):                                            # training views; view 0 is held out
        rays.append(synthetic.scene_rays(sc, sc.pose_source["c2ws"][v]).to(dev))
        tgts.append(d.imgs_raw[0, v].permute(1, 2, 0).reshape(-1, 3))
    rays, tgts = torch.cat(rays), torch.cat(tgts).contiguous()
    tuner = backend.FineTuner(fn, volume, d.imgs_raw, d.pose_source, lr=5e-4, grad_mode=grad_mode)
    gen = torch.Generator(device=dev).manual_seed(0)
    torch.manual_seed(0)
    curve = []
    for it in range(steps):
        idx = torch.randint(0, rays.shape[0], (batch,), device=dev, generator=gen)
        xyz, _, rd, z = backend.ray_marcher(rays[idx], N_samples=S, perturb=1.0)
        ndc = backend.get_ndc_coordinate(d.pose_source["w2cs"][0], d.pose_source["intrinsics"][0], xyz, inv_scale,
                                         near=sc.near_far[0], far=sc.near_far[1], pad=sc.pad)
        loss = tuner.step(xyz, ndc, z, rd, tgts[idx])[0]
        if it % 100 == 0 or it == steps - 1:
            curve.append([it, float(loss)])
    with torch.no_grad():
        held = synthetic.scene_rays(sc, sc.pose_source["c2ws"][0]).to(dev)
        rgb = backend.render_rays(held, volume, d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad), N_samples=S)[0]
        mse = ((rgb - d.imgs_raw[0, 0].permute(1, 2, 0).reshape(-1, 3)) ** 2).mean().item()
    return {"loss_every_100": curve, "heldout_psnr_db": -10.0 * torch.log10(torch.tensor(mse)).item()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--conv-steps", type=int, default=2000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("finetune_tc_check: no CUDA device")
    os.makedirs(a.out_dir, exist_ok=True)
    from mvsnerf_b200 import backend, lib
    dev = torch.device("cuda", 0)
    modes = {"fp32": lib.MLP_FP32, "tc_half": lib.MLP_TC_HALF}
    res = {"gpu": gpu_info(), "timing": {m: [] for m in modes}}
    for _ in range(3):                                          # alternated
        for name, m in modes.items():
            r = backend.finetune_step_timing(dev, WEIGHTS, grad_mode=m)
            res["timing"][name].append({"fused_ms": r["fused_ms"], "autograd_adam_ms": r["autograd_adam_ms"],
                                        "fused_loss_first_last": r["fused_loss_first_last"]})
    res["kernel_mean_ms_per_call"] = {name: kernel_times(dev, m) for name, m in modes.items()}
    res["forward_tile_ms"] = forward_tile_ms(dev)
    res["convergence"] = {name: convergence(dev, m, a.conv_steps) for name, m in modes.items()}
    res["gpu_after"] = gpu_info()
    with open(os.path.join(a.out_dir, "finetune_tc_check.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
