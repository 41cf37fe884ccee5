#!/usr/bin/env python
"""fp16 encoding-volume storage, measured: render-kernel time per frame (128 samples) from the fp32 volume and from its
fp16 copy (MVSN_VOLUME_F16, read in place), resident volume bytes, and max |rgb - rgb(fp32 volume)| with the PSNR
against the fp32-volume frame.  Cases: 512x640 (pad 24, config 2) and 960x640 (pad 24, config 5) frames of the bench
scene (synthetic.make_scene) and of the plane scene (synthetic.make_plane_scene), TC_PAIR and TC_SPLIT, the plain ray
entry (t_stop None) and mvsn_render_rays_stop at t_stop = 1e-4.  The two volumes alternate; each is run `--runs` times,
each run the median of `--frames` frames timed with CUDA events around the bare library call (scene packed once).  The
card's name, SM clock and power limit are read in the same process, before and after.

    python tools/half_volume_check.py [--frames 10] [--runs 3] [--json out.json]
"""
import argparse
import ctypes as C
import json
import math
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from mvsnerf_b200 import backend, lib, synthetic  # noqa: E402

SIZES = {"512x640": (512, 640), "960x640": (640, 960)}      # (H, W)


def gpu_state():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,clocks.sm,clocks.max.sm,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "n/a"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    L = lib.load()
    fn, mvs = backend.MVSNeRF().to(dev), backend.MVSNet().to(dev).train()
    backend.load_weights_npz(fn, mvs, os.path.join(ROOT, "tests", "golden", "mvsnerf_v0_weights.npz"))
    S = 128
    t_steps = backend._tsteps_of(S, dev)
    report = {"gpu_before": gpu_state(), "frames": a.frames, "runs": a.runs, "rows": []}
    for size, (H, W) in SIZES.items():
        for name, make in (("bench", synthetic.make_scene), ("plane", synthetic.make_plane_scene)):
            sc = make(H, W, pad=24, seed=0, near_far=(2.125, 4.525))
            d = sc.to(dev)
            with torch.no_grad():
                vol32, _, _ = mvs(d.imgs_norm, d.proj_mats, sc.near_far, pad=sc.pad)
            vol16 = vol32.half()                                   # channels-last: read in place
            vols = {"fp32": vol32, "fp16": vol16}
            rays = synthetic.scene_rays(sc).to(dev).contiguous()
            N = rays.shape[0]
            rp = lib.RayParams(float(sc.near_far[0]), float(sc.near_far[1]), float(sc.pad), 0)
            rgb, depth = torch.empty(N, 3, device=dev), torch.empty(N, device=dev)
            for mode, mname in ((lib.MLP_TC_PAIR, "pair"), (lib.MLP_TC_SPLIT, "split")):
                scenes = {k: backend._make_scene(d.pose_source, v, d.imgs_raw, fn, False, mode, half_ok=True)
                          for k, v in vols.items()}
                assert scenes["fp16"][0].mlp_mode == mode | lib.VOLUME_F16
                for eps in (None, 1e-4):
                    def call(k):
                        scene = scenes[k][0]
                        if eps is None:
                            return L.mvsn_render_rays(C.byref(scene), C.byref(rp), lib.ptr(rays), lib.ptr(t_steps), N, S,
                                                      lib.ptr(rgb), lib.ptr(depth), None, None, None, lib.stream_ptr())
                        return L.mvsn_render_rays_stop(C.byref(scene), C.byref(rp), lib.ptr(rays), lib.ptr(t_steps), N, S,
                                                       eps, lib.ptr(rgb), lib.ptr(depth), None, lib.stream_ptr())

                    out = {}
                    for k in vols:                                  # outputs (once)
                        lib.check(call(k), "render")
                        torch.cuda.synchronize()
                        out[k] = rgb.clone()
                    times = {k: [] for k in vols}
                    for _ in range(3):                              # warm-up
                        for k in vols:
                            lib.check(call(k), "render")
                    for _ in range(a.runs):
                        for k in vols:                              # alternate the two volumes
                            ts = []
                            for _ in range(a.frames):
                                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                                e0.record()
                                call(k)
                                e1.record()
                                e1.synchronize()
                                ts.append(e0.elapsed_time(e1))
                            times[k].append(statistics.median(ts))
                    base = statistics.median(times["fp32"])
                    for k, v in vols.items():
                        ms = statistics.median(times[k])
                        diff = out[k] - out["fp32"]
                        mse = float((diff ** 2).mean())
                        row = {"size": size, "scene": name, "mode": mname,
                               "t_stop": "none" if eps is None else f"{eps:g}", "volume": k,
                               "volume_bytes": v.numel() * v.element_size(),
                               "ms": round(ms, 4), "ms_runs": [round(x, 4) for x in times[k]],
                               "spread": round((max(times[k]) - min(times[k])) / ms, 4), "vs_fp32": round(ms / base, 4),
                               "max_abs_drgb": float(diff.abs().max()),
                               "psnr_vs_fp32": math.inf if mse == 0 else round(10 * math.log10(1.0 / mse), 2)}
                        report["rows"].append(row)
                        print(json.dumps(row), flush=True)
                del scenes
    report["gpu_after"] = gpu_state()
    print("gpu (name, SM clock, max SM clock, power limit):", report["gpu_before"], "|", report["gpu_after"])
    if a.json:
        with open(a.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
