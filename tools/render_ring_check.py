#!/usr/bin/env python
"""Render-kernel time of two or more builds of the library, alternated: ms per 512x640 frame (128 samples, pad 24, the
bench scene of synthetic.make_scene) for TC_PAIR from the fp32 and from the fp16 volume, and TC_SPLIT (fp32 volume) as a
control.  Each library runs in its own subprocess (loaded through MVSN_LIB); the libraries alternate `--runs` times, and
each run reports the median of `--frames` frames timed with CUDA events around the bare library call.  The first run of
each library also saves its rgb and depth, and the frames of every library are compared with the first one's bit for
bit.  The card's name, SM clock and power limit are read before and after.

    python tools/render_ring_check.py --lib parent=/path/a.so --lib new=/path/b.so [--runs 3] [--frames 10] [--json out]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = (("pair", "fp32"), ("pair", "fp16"), ("split", "fp32"))


def gpu_state():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,clocks.sm,clocks.max.sm,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "n/a"


def worker(frames, out_dir):
    """One library (MVSN_LIB): ms per frame for each case, printed as one JSON line; frames saved under out_dir."""
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    from mvsnerf_b200 import backend, lib, synthetic
    dev = torch.device("cuda", 0)
    L = lib.load()
    fn, mvs = backend.MVSNeRF().to(dev), backend.MVSNet().to(dev).train()
    backend.load_weights_npz(fn, mvs, os.path.join(ROOT, "tests", "golden", "mvsnerf_v0_weights.npz"))
    S = 128
    t_steps = backend._tsteps_of(S, dev)
    sc = synthetic.make_scene(512, 640, pad=24, seed=0, near_far=(2.125, 4.525))
    d = sc.to(dev)
    with torch.no_grad():
        vol32, _, _ = mvs(d.imgs_norm, d.proj_mats, sc.near_far, pad=sc.pad)
    vols = {"fp32": vol32, "fp16": vol32.half()}
    rays = synthetic.scene_rays(sc).to(dev).contiguous()
    N = rays.shape[0]
    rp = lib.RayParams(float(sc.near_far[0]), float(sc.near_far[1]), float(sc.pad), 0)
    rgb, depth = torch.empty(N, 3, device=dev), torch.empty(N, device=dev)
    res = {}
    for mname, vname in CASES:
        mode = lib.MLP_TC_PAIR if mname == "pair" else lib.MLP_TC_SPLIT
        scene = backend._make_scene(d.pose_source, vols[vname], d.imgs_raw, fn, False, mode, half_ok=True)[0]

        def call():
            return L.mvsn_render_rays(C.byref(scene), C.byref(rp), lib.ptr(rays), lib.ptr(t_steps), N, S,
                                      lib.ptr(rgb), lib.ptr(depth), None, None, None, lib.stream_ptr())
        for _ in range(3):
            lib.check(call(), "render")
        torch.cuda.synchronize()
        if out_dir:
            np.save(os.path.join(out_dir, f"{mname}_{vname}_rgb.npy"), rgb.cpu().numpy())
            np.save(os.path.join(out_dir, f"{mname}_{vname}_depth.npy"), depth.cpu().numpy())
        ts = []
        for _ in range(frames):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call()
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        res[f"{mname}_{vname}"] = statistics.median(ts)
    print("RESULT " + json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], help="name=path of a libmvsnerf_b200.so (two or more)")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--json", default=None)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--out-dir", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        worker(a.frames, a.out_dir)
        return
    libs = dict(x.split("=", 1) for x in a.lib)
    if len(libs) < 2:
        raise SystemExit("give two or more --lib name=path")
    report = {"gpu_before": gpu_state(), "frames": a.frames, "runs": a.runs, "libs": libs, "times": {}}
    times = {n: {f"{m}_{v}": [] for m, v in CASES} for n in libs}
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(a.runs):
            for name, path in libs.items():                 # alternate the libraries
                out = os.path.join(tmp, name)
                os.makedirs(out, exist_ok=True)
                cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--frames", str(a.frames)]
                if r == 0:
                    cmd += ["--out-dir", out]
                p = subprocess.run(cmd, env=dict(os.environ, MVSN_LIB=os.path.abspath(path)), capture_output=True, text=True)
                line = [x for x in p.stdout.splitlines() if x.startswith("RESULT ")]
                if p.returncode != 0 or not line:
                    raise SystemExit(f"{name} failed:\n{p.stdout}\n{p.stderr}")
                for k, v in json.loads(line[0][7:]).items():
                    times[name][k].append(v)
                print(name, line[0][7:], flush=True)
        import numpy as np
        first = next(iter(libs))
        report["bit_equal_to_" + first] = {
            name: all(np.array_equal(np.load(os.path.join(tmp, name, f)), np.load(os.path.join(tmp, first, f)), equal_nan=True)
                      for f in sorted(os.listdir(os.path.join(tmp, first))))
            for name in libs}
    for name in libs:
        row = {}
        for k, v in times[name].items():
            ms = statistics.median(v)
            row[k] = {"ms": round(ms, 3), "runs": [round(x, 3) for x in v], "spread": round((max(v) - min(v)) / ms, 4),
                      "vs_" + first: round(ms / statistics.median(times[first][k]), 4)}
        report["times"][name] = row
        print(name, json.dumps(row), flush=True)
    report["gpu_after"] = gpu_state()
    print("bit-equal frames:", report["bit_equal_to_" + first])
    print("gpu (name, SM clock, max SM clock, power limit):", report["gpu_before"], "|", report["gpu_after"])
    if a.json:
        with open(a.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
