#!/usr/bin/env python
"""Early ray termination, measured: render-kernel time per 512x640 frame (128 samples) of the existing ray entry
(mvsn_render_rays) and of mvsn_render_rays_stop at t_stop in {0, 1e-4, 1e-3, 1e-2}, in the fp16 (TC_PAIR) and split
(TC_SPLIT) modes, on the bench scene (synthetic.make_scene) and on a scene whose rays become opaque
(synthetic.make_plane_scene).  Variants alternate; each is run `--runs` times, each run the median of `--frames` frames
timed with CUDA events around the bare library call (scene packed once).  Also reported: tiles computed as a fraction
of all tiles, max |rgb - rgb(t_stop = 0)| and PSNR against the t_stop = 0 frame, the SM clock and the power limit.

    python tools/render_stop_check.py [--frames 20] [--runs 3] [--json out.json]
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

EPS = [0.0, 1e-4, 1e-3, 1e-2]
# tiles computed at t_stop = 1e-4 / 1e-3 / 1e-2, estimated on the host (fp32 oracle, shipped checkpoint, 96 random groups,
# one tile of lag where the kernel has two)
CPU_ESTIMATE = {"bench": {1e-4: 0.96, 1e-3: 0.94, 1e-2: 0.87}, "plane": {1e-4: 0.53, 1e-3: 0.50, 1e-2: 0.47}}


def gpu_state():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,clocks.sm,clocks.max.sm,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "n/a"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20)
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
    for name, make in (("bench", synthetic.make_scene), ("plane", synthetic.make_plane_scene)):
        sc = make(512, 640, seed=0)
        d = sc.to(dev)
        with torch.no_grad():
            vol, _, _ = mvs(d.imgs_norm, d.proj_mats, sc.near_far, pad=sc.pad)
        rays = synthetic.scene_rays(sc).to(dev).contiguous()
        N = rays.shape[0]
        rp = lib.RayParams(float(sc.near_far[0]), float(sc.near_far[1]), float(sc.pad), 0)
        rgb, depth = torch.empty(N, 3, device=dev), torch.empty(N, device=dev)
        tiles = torch.zeros(1, dtype=torch.int64, device=dev)
        for mode, mname in ((lib.MLP_TC_PAIR, "pair"), (lib.MLP_TC_SPLIT, "split")):
            scene, keep = backend._make_scene(d.pose_source, vol, d.imgs_raw, fn, False, mode)

            def call(eps):
                if eps is None:
                    return L.mvsn_render_rays(C.byref(scene), C.byref(rp), lib.ptr(rays), lib.ptr(t_steps), N, S,
                                              lib.ptr(rgb), lib.ptr(depth), None, None, None, lib.stream_ptr())
                return L.mvsn_render_rays_stop(C.byref(scene), C.byref(rp), lib.ptr(rays), lib.ptr(t_steps), N, S, eps,
                                               lib.ptr(rgb), lib.ptr(depth), lib.ptr(tiles), lib.stream_ptr())

            variants = [None] + EPS
            out = {}
            for v in variants:                                  # outputs and tile counts (once)
                tiles.zero_()
                lib.check(call(v), "render")
                torch.cuda.synchronize()
                out[v] = (rgb.clone(), int(tiles.item()))
            times = {v: [] for v in variants}
            for _ in range(3):                                  # warm-up
                for v in variants:
                    lib.check(call(v), "render")
            for _ in range(a.runs):
                for v in variants:                              # alternate the variants
                    ts = []
                    for _ in range(a.frames):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        call(v)
                        e1.record()
                        e1.synchronize()
                        ts.append(e0.elapsed_time(e1))
                    times[v].append(statistics.median(ts))
            rt = 32
            all_tiles = ((N + rt - 1) // rt) * ((S + 64 // rt - 1) // (64 // rt))
            base = statistics.median(times[None])
            for v in variants:
                ms = statistics.median(times[v])
                row = {"scene": name, "mode": mname, "variant": "existing" if v is None else f"t_stop={v:g}",
                       "ms": round(ms, 4), "ms_runs": [round(x, 4) for x in times[v]], "vs_existing": round(ms / base, 4)}
                if v is not None:
                    diff = (out[v][0] - out[0.0][0])
                    mse = float((diff ** 2).mean())
                    row.update(tiles_fraction=round(out[v][1] / all_tiles, 4),
                               cpu_estimate=CPU_ESTIMATE[name].get(v),
                               max_abs_drgb=float(diff.abs().max()),
                               psnr_vs_eps0=(math.inf if mse == 0 else round(10 * math.log10(1.0 / mse), 2)))
                report["rows"].append(row)
                print(json.dumps(row), flush=True)
            del keep
    report["gpu_after"] = gpu_state()
    print("gpu (name, SM clock, max SM clock, power limit):", report["gpu_before"], "|", report["gpu_after"])
    if a.json:
        with open(a.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
