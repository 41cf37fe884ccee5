"""On-disk formats either side of the render hot path (SURVEY.md 8(f) row 4).

* Fine-tuned checkpoints in the reference's schema (train_mvs_nerf_finetuning_pl.py:279-291):
  `{'global_step', 'network_fn_state_dict', 'volume': {'feat_volume': [1,8,D,H,W]}, 'network_mvs_state_dict'}`
  -- what `renderer_video.ipynb`'s `is_finetued` branch reads back with
  `torch.load(args.ckpt)['volume']['feat_volume']` -> `RefVolume(...)`.
* The frame loop of the free-viewpoint video cells (renderer_video.ipynb "DTU video rendering": get_rays ->
  chunk loop -> `rgb.cpu()`, `depth.cpu()` -> frames list -> imageio.mimwrite) as `render_video`: one fused launch
  per frame and an asynchronous frame sink (`FrameWriter`: pinned double buffers, D2H on a side stream, a writer
  thread doing the uint8 conversion and the file write) so disk and PCIe never stall the render stream.

Host code only: device arithmetic stays in libmvsnerf_b200 (backend.render_rays).
"""
from __future__ import annotations

import os
import queue
import threading

import numpy as np
import torch

from . import backend


# --------------------------------------------------------------------------------------------
# fine-tuned checkpoints
# --------------------------------------------------------------------------------------------
def save_finetuned_ckpt(path, network_fn, volume, network_mvs=None, global_step=0, network_fine=None):
    """train_mvs_nerf_finetuning_pl.py:279-291 (`save_ckpt`).  `volume` is a RefVolume (or a raw [1,8,D,H,W]
    tensor); tensors are stored in the reference layout whatever their strides in memory are."""
    vol = volume.feat_volume if isinstance(volume, torch.nn.Module) else volume
    if vol.dim() != 5 or vol.shape[0] != 1 or vol.shape[1] != 8:
        raise RuntimeError(f"encoding volume must be [1,8,D,H,W], got {tuple(vol.shape)}")
    ckpt = {
        "global_step": int(global_step),
        "network_fn_state_dict": network_fn.state_dict(),
        "volume": {"feat_volume": vol.detach().contiguous()},
    }
    if network_mvs is not None:
        ckpt["network_mvs_state_dict"] = network_mvs.state_dict()
    if network_fine is not None:
        ckpt["network_fine_state_dict"] = network_fine.state_dict()
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    tmp = f"{path}.tmp.{os.getpid()}"
    torch.save(ckpt, tmp)
    os.replace(tmp, path)                      # a reader never sees a half-written checkpoint
    return path


def load_finetuned_ckpt(path, network_fn=None, network_mvs=None, device=None):
    """Inverse of `save_finetuned_ckpt`; also reads checkpoints written by the reference itself.
    Returns (RefVolume on `device`, global_step).  Modules that are passed get their state loaded strictly."""
    if device is None:
        if not torch.cuda.is_available():
            raise RuntimeError("load_finetuned_ckpt: no CUDA device; mvsnerf_b200 has no CPU path")
        device = torch.device("cuda", torch.cuda.current_device())
    ckpt = torch.load(path, map_location=device, weights_only=False)
    if "volume" not in ckpt or "feat_volume" not in ckpt["volume"]:
        raise RuntimeError(f"{path}: no ['volume']['feat_volume'] -- not a fine-tuned checkpoint "
                           "(pretrained checkpoints carry no per-scene volume)")
    if network_fn is not None:
        network_fn.load_state_dict(ckpt["network_fn_state_dict"])
    if network_mvs is not None and "network_mvs_state_dict" in ckpt:
        network_mvs.load_state_dict(ckpt["network_mvs_state_dict"])
    vol = ckpt["volume"]["feat_volume"].detach().to(device=device, dtype=torch.float32)
    return backend.RefVolume(vol).to(device), int(ckpt.get("global_step", 0))


# --------------------------------------------------------------------------------------------
# rays of a target camera (data/ray_utils.py:32-53, get_rays) + the notebooks' [N,8] packing
# --------------------------------------------------------------------------------------------
def camera_rays(directions, c2w, near, far):
    """directions [H,W,3] camera-frame (get_ray_directions), c2w [3|4,4] -> rays [H*W,8] = (o, d, near, far);
    d is NOT normalised, as in the reference."""
    d = directions.reshape(-1, 3) @ c2w[:3, :3].T
    o = c2w[:3, 3].expand_as(d)
    nf = torch.tensor([float(near), float(far)], dtype=d.dtype, device=d.device).expand(d.shape[0], 2)
    return torch.cat([o, d, nf], 1).contiguous()


# --------------------------------------------------------------------------------------------
# asynchronous frame sink
# --------------------------------------------------------------------------------------------
class FrameWriter:
    """Image-sequence writer for the video loops.

    `submit(index, rgb, depth)` takes DEVICE tensors ([H*W,3] in [0,1], [H*W]); it enqueues a D2H copy into one
    of `depth_q` pinned staging buffers on a side stream (ordered after the render by an event) and returns
    immediately.  A worker thread waits for the copy, converts to uint8 and writes `<dir>/rgb_00000.<fmt>`
    (+ `depth_00000.npy` when depths are kept).  Formats: 'ppm' (no dependency), 'png' (Pillow), 'npy'."""

    def __init__(self, out_dir, H, W, fmt="ppm", keep_depth=True, n_buffers=3, device=None):
        if fmt not in ("ppm", "png", "npy"):
            raise ValueError(f"FrameWriter: unknown format {fmt!r}")
        self.dir, self.H, self.W, self.fmt, self.keep_depth = out_dir, int(H), int(W), fmt, keep_depth
        os.makedirs(out_dir, exist_ok=True)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        n = self.H * self.W
        self._bufs = [(torch.empty(n, 3, dtype=torch.float32).pin_memory(),
                       torch.empty(n, dtype=torch.float32).pin_memory()) for _ in range(n_buffers)]
        self._free = queue.Queue()
        for i in range(n_buffers):
            self._free.put(i)
        self._work = queue.Queue()
        self._copy_stream = torch.cuda.Stream(device=self.device)
        self._error = None
        self.frames_written = 0
        self._thread = threading.Thread(target=self._run, name="mvsn-frame-writer", daemon=True)
        self._thread.start()

    def submit(self, index, rgb, depth=None):
        if self._error is not None:
            raise RuntimeError(f"FrameWriter worker failed: {self._error!r}")
        n = self.H * self.W
        if tuple(rgb.shape) != (n, 3) or not rgb.is_cuda:
            raise RuntimeError(f"FrameWriter.submit: rgb must be a CUDA tensor [{n}, 3]")
        slot = self._free.get()                       # back-pressure: blocks while all staging buffers are in flight
        h_rgb, h_depth = self._bufs[slot]
        rendered = torch.cuda.Event()
        rendered.record(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(rendered)
            h_rgb.copy_(rgb, non_blocking=True)
            if depth is not None and self.keep_depth:
                h_depth.copy_(depth.reshape(-1), non_blocking=True)
            done = torch.cuda.Event()
            done.record(self._copy_stream)
        # the device tensors must stay valid until the copy ran: keep references with the work item
        self._work.put((int(index), slot, done, depth is not None and self.keep_depth, rgb, depth))

    def _run(self):
        while True:
            item = self._work.get()
            if item is None:
                return
            index, slot, done, has_depth, _rgb, _depth = item
            try:
                done.synchronize()
                h_rgb, h_depth = self._bufs[slot]
                img = (h_rgb.view(self.H, self.W, 3).clamp(0, 1) * 255.0).round().to(torch.uint8).numpy()
                base = os.path.join(self.dir, f"rgb_{index:05d}")
                if self.fmt == "ppm":
                    with open(base + ".ppm", "wb") as f:
                        f.write(f"P6\n{self.W} {self.H}\n255\n".encode())
                        f.write(img.tobytes())
                elif self.fmt == "png":
                    from PIL import Image
                    Image.fromarray(img).save(base + ".png")
                else:
                    np.save(base + ".npy", img)
                if has_depth:
                    np.save(os.path.join(self.dir, f"depth_{index:05d}.npy"), h_depth.view(self.H, self.W).numpy().copy())
                self.frames_written += 1
            except Exception as e:          # surfaced by the next submit() / close()
                self._error = e
            finally:
                self._free.put(slot)

    def close(self):
        self._work.put(None)
        self._thread.join()
        if self._error is not None:
            raise RuntimeError(f"FrameWriter worker failed: {self._error!r}")

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
        return False


def render_video(c2ws, directions, volume_feature, imgs, pose_ref, network_fn, near_far, pad, writer=None,
                 N_samples=128, white_bkgd=False, lindisp=False, mlp_mode=None, t_stop=None, occupancy=None):
    """The free-viewpoint loop of renderer_video.ipynb (cell "DTU video rendering", raw lines 775-786 hold its
    settings): for every target pose build the rays (get_rays), render the whole frame with ONE fused launch and
    hand the pixels to `writer` (a FrameWriter) or collect them.  Returns the list of (rgb, depth) device tensors
    when no writer is given, else the number of frames submitted.  `t_stop`: early ray termination; `occupancy`:
    empty-space skipping with a grid from backend.build_occupancy, which serves every pose (see backend.render_rays)."""
    H, W = directions.shape[:2]
    frames = []
    for i, c2w in enumerate(c2ws):
        rays = camera_rays(directions, c2w, near_far[0], near_far[1])
        rgb, depth = backend.render_rays(rays, volume_feature, imgs, pose_ref, network_fn, near_far, pad,
                                         N_samples=N_samples, white_bkgd=white_bkgd, lindisp=lindisp, mlp_mode=mlp_mode,
                                         t_stop=t_stop, occupancy=occupancy)
        if writer is not None:
            writer.submit(i, rgb, depth)
        else:
            frames.append((rgb, depth))
    return len(c2ws) if writer is not None else frames
