"""ctypes binding of libmvsnerf_b200.so (the C ABI in include/mvsnerf_b200.h).

The library is the product: if it is missing or fails to load, importing callers get a loud
RuntimeError -- there is no CPU or PyTorch fallback behind these functions.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MVSN_LIB") or os.path.join(HERE, "libmvsnerf_b200.so")   # MVSN_LIB: debug builds only

MLP_FP32, MLP_TC_HALF, MLP_TC_SPLIT = 0, 1, 2
MLP_TC_PAIR = 3          # same fp16-operand kernel as MLP_TC_HALF (csrc/render_wg.cu)
GRAD_TC_FULL = 4         # grad_mode of the rays fine-tuning entries: TC_HALF's backward + the forward recompute on wgmma
N_MLP_TENSORS, N_COSTREG_TENSORS, N_FEATURENET_TENSORS = 22, 30, 26

# every symbol include/mvsnerf_b200.h declares (tests check the library exports all of them)
EXPORTS = [
    "mvsn_last_error", "mvsn_abi_version", "mvsn_mlp_packed_bytes", "mvsn_mlp_pack",
    "mvsn_pack_images", "mvsn_volume_to_channels_last", "mvsn_volume_from_channels_last",
    "mvsn_render_samples", "mvsn_render_rays", "mvsn_cost_volume_workspace_bytes",
    "mvsn_build_cost_volume", "mvsn_costreg_workspace_bytes", "mvsn_costreg_forward",
    "mvsn_featurenet_workspace_bytes", "mvsn_featurenet_forward",
    "mvsn_selftest_umma",
    "mvsn_peer_buffer_create", "mvsn_peer_buffer_open", "mvsn_peer_buffer_close", "mvsn_peer_buffer_destroy",
    "mvsn_render_rays_to_peers", "mvsn_make_rays",
    "mvsn_featurenet_forward_bn", "mvsn_costreg_forward_bn",
    "mvsn_render_backward_workspace_bytes", "mvsn_render_backward", "mvsn_adam_step", "mvsn_adam_step_volume",
    "mvsn_render_backward_tc_workspace_bytes", "mvsn_render_backward_tc",
    "mvsn_render_backward_deterministic_workspace_bytes", "mvsn_render_backward_deterministic",
    "mvsn_render_backward_rays_workspace_bytes", "mvsn_render_backward_rays",
    "mvsn_render_rays_stop",
    "mvsn_render_backward_rays_stop_workspace_bytes", "mvsn_render_backward_rays_stop",
    "mvsn_volume_to_half", "mvsn_costreg_forward_f16",
    "mvsn_occupancy_bytes", "mvsn_build_occupancy_workspace_bytes", "mvsn_build_occupancy",
    "mvsn_render_rays_occ_workspace_bytes", "mvsn_render_rays_occ",
    "mvsn_render_samples_stop", "mvsn_render_backward_stop_workspace_bytes", "mvsn_render_backward_stop",
    "mvsn_build_density_workspace_bytes", "mvsn_build_density", "mvsn_sample_importance",
]
VOLUME_F16 = 0x100       # OR-ed into RenderScene.mlp_mode (TC modes): volume_dhwc is an fp16 [D,Hp,Wp,8] image
MAX_PEERS, PEER_HANDLE_BYTES = 16, 64
BN_BATCH, BN_BATCH_UPDATE, BN_RUNNING = 0, 1, 2
CONV0_FFMA = 0x100


class RenderScene(C.Structure):
    _fields_ = [("volume_dhwc", C.c_void_p), ("D", C.c_int), ("Hp", C.c_int), ("Wp", C.c_int),
                ("imgs_hwc4", C.c_void_p), ("V", C.c_int), ("H", C.c_int), ("W", C.c_int),
                ("w2cs", C.c_void_p), ("intrinsics", C.c_void_p),
                ("mlp_packed", C.c_void_p), ("mlp_mode", C.c_int), ("white_bkgd", C.c_int)]


class PeerSink(C.Structure):
    _fields_ = [("frame", C.c_void_p * 16), ("n_peers", C.c_int), ("first_pixel", C.c_longlong)]


class RenderGrads(C.Structure):
    _fields_ = [("rgb", C.c_void_p), ("target_rgb", C.c_void_p), ("loss_scale", C.c_float), ("depth", C.c_void_p),
                ("weights", C.c_void_p), ("alpha", C.c_void_p), ("input_feat", C.c_void_p), ("rgb_out", C.c_void_p),
                ("depth_out", C.c_void_p), ("loss_out", C.c_void_p)]


class RayParams(C.Structure):
    _fields_ = [("ndc_near", C.c_float), ("ndc_far", C.c_float), ("pad", C.c_float), ("lindisp", C.c_int)]


class OccupancyGrid(C.Structure):
    _fields_ = [("bits", C.c_void_p), ("D", C.c_int), ("Hp", C.c_int), ("Wp", C.c_int)]


class DensityGrid(C.Structure):
    _fields_ = [("sigma", C.c_void_p), ("D", C.c_int), ("Hp", C.c_int), ("Wp", C.c_int)]


_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -m mvsnerf_b200.build` "
            "(mvsnerf_b200 has no CPU fallback; the CUDA library is the product)")
    lib = C.CDLL(LIB_PATH)
    vp, ip, fp = C.c_void_p, C.c_int, C.c_float
    lib.mvsn_last_error.restype = C.c_char_p
    lib.mvsn_abi_version.restype = ip
    lib.mvsn_mlp_packed_bytes.restype = C.c_size_t
    lib.mvsn_mlp_packed_bytes.argtypes = [ip]
    lib.mvsn_mlp_pack.argtypes = [C.POINTER(vp), ip, vp, C.c_size_t, vp]
    lib.mvsn_pack_images.argtypes = [vp, ip, ip, ip, vp, vp]
    lib.mvsn_volume_to_channels_last.argtypes = [vp, ip, ip, ip, vp, vp]
    lib.mvsn_volume_from_channels_last.argtypes = [vp, ip, ip, ip, vp, vp]
    lib.mvsn_volume_to_half.argtypes = [vp, ip, ip, ip, ip, ip, vp, vp]
    lib.mvsn_render_samples.argtypes = [C.POINTER(RenderScene), vp, vp, vp, vp, ip, ip, vp, vp, vp, vp, vp, vp]
    lib.mvsn_render_rays.argtypes = [C.POINTER(RenderScene), C.POINTER(RayParams), vp, vp, ip, ip,
                                     vp, vp, vp, vp, vp, vp]
    lib.mvsn_render_rays_stop.argtypes = [C.POINTER(RenderScene), C.POINTER(RayParams), vp, vp, ip, ip, fp,
                                          vp, vp, vp, vp]
    lib.mvsn_render_rays_stop.restype = ip
    lib.mvsn_render_samples_stop.argtypes = [C.POINTER(RenderScene), vp, vp, vp, vp, ip, ip, fp, vp, vp, vp, vp]
    for name in ("mvsn_occupancy_bytes", "mvsn_build_occupancy_workspace_bytes"):
        getattr(lib, name).restype = C.c_size_t
        getattr(lib, name).argtypes = [ip, ip, ip]
    lib.mvsn_build_occupancy.argtypes = [C.POINTER(RenderScene), C.POINTER(RayParams), ip, vp, vp, C.c_size_t, vp]
    lib.mvsn_build_density_workspace_bytes.restype = C.c_size_t
    lib.mvsn_build_density_workspace_bytes.argtypes = [ip, ip, ip]
    lib.mvsn_build_density.argtypes = [C.POINTER(RenderScene), C.POINTER(RayParams), vp, vp, C.c_size_t, vp]
    lib.mvsn_sample_importance.argtypes = [C.POINTER(RenderScene), C.POINTER(RayParams), C.POINTER(DensityGrid), vp, vp,
                                           vp, vp, vp, vp, ip, ip, ip, vp, vp, vp, vp]
    lib.mvsn_render_rays_occ_workspace_bytes.restype = C.c_size_t
    lib.mvsn_render_rays_occ_workspace_bytes.argtypes = [ip, ip]
    lib.mvsn_render_rays_occ.argtypes = [C.POINTER(RenderScene), C.POINTER(RayParams), vp, vp, ip, ip, fp,
                                         C.POINTER(OccupancyGrid), vp, vp, vp, vp, C.c_size_t, vp]
    lib.mvsn_cost_volume_workspace_bytes.restype = C.c_size_t
    lib.mvsn_cost_volume_workspace_bytes.argtypes = [ip, ip, ip]
    lib.mvsn_build_cost_volume.argtypes = [vp, vp, vp, vp, ip, ip, ip, ip, ip, vp, vp, vp, C.c_size_t, vp]
    lib.mvsn_costreg_workspace_bytes.restype = C.c_size_t
    lib.mvsn_costreg_workspace_bytes.argtypes = [ip, ip, ip]
    lib.mvsn_costreg_forward.argtypes = [C.POINTER(vp), vp, ip, ip, ip, vp, vp, C.c_size_t, vp]
    lib.mvsn_featurenet_workspace_bytes.restype = C.c_size_t
    lib.mvsn_featurenet_workspace_bytes.argtypes = [ip, ip, ip]
    lib.mvsn_featurenet_forward.argtypes = [C.POINTER(vp), vp, ip, ip, ip, vp, vp, C.c_size_t, vp]
    lib.mvsn_render_rays_to_peers.argtypes = [C.POINTER(RenderScene), C.POINTER(RayParams), vp, vp, ip, ip,
                                              C.POINTER(PeerSink), vp, vp, vp]
    lib.mvsn_peer_buffer_create.argtypes = [C.c_size_t, C.POINTER(vp), C.c_char_p]
    lib.mvsn_peer_buffer_open.argtypes = [C.c_char_p, C.POINTER(vp)]
    lib.mvsn_peer_buffer_close.argtypes = [vp]
    lib.mvsn_peer_buffer_destroy.argtypes = [vp]
    lib.mvsn_render_backward_workspace_bytes.restype = C.c_size_t
    lib.mvsn_render_backward_workspace_bytes.argtypes = [ip, ip]
    lib.mvsn_render_backward.argtypes = [C.POINTER(RenderScene), C.POINTER(vp), vp, vp, vp, vp, ip, ip,
                                         C.POINTER(RenderGrads), C.POINTER(vp), vp, vp, C.c_size_t, vp]
    lib.mvsn_render_backward_tc_workspace_bytes.restype = C.c_size_t
    lib.mvsn_render_backward_tc_workspace_bytes.argtypes = [ip, ip]
    lib.mvsn_render_backward_tc.argtypes = lib.mvsn_render_backward.argtypes
    lib.mvsn_render_backward_deterministic_workspace_bytes.restype = C.c_size_t
    lib.mvsn_render_backward_deterministic_workspace_bytes.argtypes = [ip, ip, ip, ip, ip, ip]
    lib.mvsn_render_backward_deterministic.argtypes = [C.POINTER(RenderScene), C.POINTER(vp), vp, vp, vp, vp, ip, ip, ip,
                                                       C.POINTER(RenderGrads), C.POINTER(vp), vp, vp, C.c_size_t, vp]
    lib.mvsn_render_backward_rays_workspace_bytes.restype = C.c_size_t
    lib.mvsn_render_backward_rays_workspace_bytes.argtypes = [ip, ip, ip, ip, ip, ip, ip]
    lib.mvsn_render_backward_rays.argtypes = [C.POINTER(RenderScene), C.POINTER(vp), C.POINTER(RayParams), vp, vp, vp,
                                              ip, ip, ip, ip, C.POINTER(RenderGrads), C.POINTER(vp), vp, vp, C.c_size_t,
                                              vp]
    lib.mvsn_render_backward_rays_stop_workspace_bytes.restype = C.c_size_t
    lib.mvsn_render_backward_rays_stop_workspace_bytes.argtypes = [ip, ip, ip, ip, ip, ip, ip]
    lib.mvsn_render_backward_rays_stop.argtypes = [C.POINTER(RenderScene), C.POINTER(vp), C.POINTER(RayParams), vp, vp,
                                                   vp, ip, ip, ip, ip, fp, C.POINTER(RenderGrads), C.POINTER(vp), vp,
                                                   vp, vp, vp, C.c_size_t, vp]
    lib.mvsn_render_backward_stop_workspace_bytes.restype = C.c_size_t
    lib.mvsn_render_backward_stop_workspace_bytes.argtypes = [ip, ip, ip, ip, ip, ip, ip]
    lib.mvsn_render_backward_stop.argtypes = [C.POINTER(RenderScene), C.POINTER(vp), vp, vp, vp, vp, ip, ip, ip, ip, fp,
                                              C.POINTER(RenderGrads), C.POINTER(vp), vp, vp, vp, vp, C.c_size_t, vp]
    lib.mvsn_adam_step.argtypes = [C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(ip), ip,
                                   fp, fp, fp, fp, ip, vp]
    lib.mvsn_adam_step_volume.argtypes = [vp, vp, vp, vp, C.c_longlong, ip, fp, fp, fp, fp, ip, vp]
    lib.mvsn_costreg_forward_bn.argtypes = [C.POINTER(vp), C.POINTER(vp), ip, fp, vp, ip, ip, ip, vp, vp, C.c_size_t, vp]
    lib.mvsn_costreg_forward_f16.argtypes = lib.mvsn_costreg_forward_bn.argtypes
    lib.mvsn_featurenet_forward_bn.argtypes = [C.POINTER(vp), C.POINTER(vp), ip, fp, vp, ip, ip, ip, vp, vp, C.c_size_t, vp]
    lib.mvsn_make_rays.argtypes = [vp, vp, fp, fp, ip, vp, vp]
    lib.mvsn_make_rays.restype = ip
    lib.mvsn_selftest_umma.argtypes = [vp, vp, vp, ip, ip, vp, vp]
    for name in ("mvsn_selftest_umma", "mvsn_mlp_pack", "mvsn_pack_images", "mvsn_volume_to_channels_last",
                 "mvsn_volume_from_channels_last", "mvsn_render_samples", "mvsn_render_rays",
                 "mvsn_build_cost_volume", "mvsn_costreg_forward", "mvsn_featurenet_forward",
                 "mvsn_render_rays_to_peers", "mvsn_peer_buffer_create", "mvsn_peer_buffer_open",
                 "mvsn_peer_buffer_close", "mvsn_peer_buffer_destroy", "mvsn_render_backward", "mvsn_render_backward_tc",
                 "mvsn_render_backward_deterministic", "mvsn_render_backward_rays",
                 "mvsn_render_backward_rays_stop", "mvsn_adam_step",
                 "mvsn_adam_step_volume", "mvsn_featurenet_forward_bn", "mvsn_costreg_forward_bn",
                 "mvsn_volume_to_half", "mvsn_costreg_forward_f16", "mvsn_build_occupancy", "mvsn_render_rays_occ",
                 "mvsn_render_samples_stop", "mvsn_render_backward_stop", "mvsn_build_density",
                 "mvsn_sample_importance"):
        getattr(lib, name).restype = ip
    _lib = lib
    return lib


def check(rc: int, what: str):
    """Non-zero return codes become RuntimeError (the reference's convention is Python exceptions)."""
    if rc != 0:
        msg = load().mvsn_last_error().decode(errors="replace")
        raise RuntimeError(f"{what} failed (code {rc}): {msg}")


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def dev_f32(t: torch.Tensor, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (got {t.device}); mvsnerf_b200 has no CPU path")
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def ptr_array(tensors):
    arr = (C.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = t.data_ptr()
    return arr
