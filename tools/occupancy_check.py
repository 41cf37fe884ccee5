#!/usr/bin/env python
"""Empty-space skipping, measured: render-kernel ms per frame (128 samples) at 512x640 and 960x640, on the bench scene
(synthetic.make_scene) and the plane scene (synthetic.make_plane_scene), in the fp16 (TC_PAIR) and split (TC_SPLIT)
modes, for four variants alternated in one call: the existing entry (mvsn_render_rays), t_stop = 1e-4 only
(mvsn_render_rays_stop), the occupancy grid only (mvsn_render_rays_occ at t_stop = 0, dilate 1) and both.  Each variant
is run `--runs` times, each run the median of `--frames` frames timed with CUDA events around the bare library call
(scene and grid built once; the grid variants include their range pre-pass).  Also reported: the grid build time
(mvsn_build_occupancy), the occupied fraction of its cells, tiles computed as a fraction of all tiles, max |rgb -
rgb_full|, PSNR against the full render, the fraction of bit-identical pixels, the card name and its power limit.

    python tools/occupancy_check.py [--frames 10] [--runs 3] [--json out.json]
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
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    L = lib.load()
    fn, mvs = backend.MVSNeRF().to(dev), backend.MVSNet().to(dev).train()
    backend.load_weights_npz(fn, mvs, os.path.join(ROOT, "tests", "golden", "mvsnerf_v0_weights.npz"))
    S, EPS = 128, 1e-4
    t_steps = backend._tsteps_of(S, dev)
    report = {"gpu_before": gpu_state(), "frames": a.frames, "runs": a.runs, "rows": []}
    for H, W in ((512, 640), (960, 640)):
        for name, make in (("bench", synthetic.make_scene), ("plane", synthetic.make_plane_scene)):
            sc = make(H, W, seed=0)
            d = sc.to(dev)
            with torch.no_grad():
                vol, _, _ = mvs(d.imgs_norm, d.proj_mats, sc.near_far, pad=sc.pad)
            rays = synthetic.scene_rays(sc).to(dev).contiguous()
            N = rays.shape[0]
            rp = lib.RayParams(float(sc.near_far[0]), float(sc.near_far[1]), float(sc.pad), 0)
            backend.clear_cache()
            build = lambda: backend.build_occupancy(vol, d.imgs_raw, d.pose_source, fn, sc.near_far, float(sc.pad))
            build()
            torch.cuda.synchronize()
            build_ms = []
            for _ in range(3):
                backend.clear_cache()
                build_ms.append(timed(build, 1))
            occ = build()
            grid = occ._grid()
            ws = torch.empty(L.mvsn_render_rays_occ_workspace_bytes(N, S), dtype=torch.uint8, device=dev)
            rgb, depth = torch.empty(N, 3, device=dev), torch.empty(N, device=dev)
            tiles = torch.zeros(1, dtype=torch.int64, device=dev)
            for mode, mname in ((lib.MLP_TC_PAIR, "pair"), (lib.MLP_TC_SPLIT, "split")):
                scene, keep = backend._make_scene(d.pose_source, vol, d.imgs_raw, fn, False, mode)
                base = (C.byref(scene), C.byref(rp), lib.ptr(rays), lib.ptr(t_steps), N, S)

                def call(v):
                    if v == "existing":
                        return L.mvsn_render_rays(*base, lib.ptr(rgb), lib.ptr(depth), None, None, None, lib.stream_ptr())
                    if v == "t_stop":
                        return L.mvsn_render_rays_stop(*base, EPS, lib.ptr(rgb), lib.ptr(depth), lib.ptr(tiles),
                                                       lib.stream_ptr())
                    return L.mvsn_render_rays_occ(*base, EPS if v == "both" else 0.0, C.byref(grid), lib.ptr(rgb),
                                                  lib.ptr(depth), lib.ptr(tiles), lib.ptr(ws), ws.numel(), lib.stream_ptr())

                variants = ["existing", "t_stop", "grid", "both"]
                out = {}
                for v in variants:
                    tiles.zero_()
                    lib.check(call(v), v)
                    torch.cuda.synchronize()
                    out[v] = (rgb.clone(), depth.clone(), int(tiles.item()))
                times = {v: [] for v in variants}
                for _ in range(2):
                    for v in variants:
                        lib.check(call(v), v)
                for _ in range(a.runs):
                    for v in variants:
                        times[v].append(timed(lambda: call(v), a.frames))
                rt = 32
                all_tiles = ((N + rt - 1) // rt) * ((S + 64 // rt - 1) // (64 // rt))
                t0 = statistics.median(times["existing"])
                for v in variants:
                    ms = statistics.median(times[v])
                    diff = out[v][0] - out["existing"][0]
                    mse = float((diff ** 2).mean())
                    same = ((out[v][0] == out["existing"][0]).all(1) & (out[v][1] == out["existing"][1])).float().mean()
                    row = {"frame": f"{H}x{W}", "scene": name, "mode": mname, "variant": v, "ms": round(ms, 3),
                           "ms_runs": [round(x, 3) for x in times[v]], "vs_existing": round(ms / t0, 4),
                           "grid_build_ms": round(statistics.median(build_ms), 3),
                           "grid_occupied": round(occ.fraction(), 4),
                           "tiles_fraction": None if v == "existing" else round(out[v][2] / all_tiles, 4),
                           "max_abs_drgb": float(diff.abs().max()),
                           "psnr_vs_full": math.inf if mse == 0 else round(10 * math.log10(1.0 / mse), 2),
                           "bit_identical_pixels": round(float(same), 5)}
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
