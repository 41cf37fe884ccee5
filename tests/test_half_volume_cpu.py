"""fp16 volume storage without a GPU: the MVSN_VOLUME_F16 flag is rejected by MVSN_MLP_FP32 and by every backward
entry, the conversion and fp16-encoder entries report their argument errors before any CUDA call (on a machine without
a device a CUDA call would fail with MVSN_ECUDA instead), the weight packer ignores the flag, and the new symbols are
exported and declared."""
import ctypes as C
import os

import pytest
import torch

from conftest import ROOT
from mvsnerf_b200 import backend, lib

ENULL, EBADSHAPE, EALIGN, EUNSUPPORTED = -4, -1, -2, -6


@pytest.fixture(scope="module")
def mem():
    buf = (C.c_float * 4096)()
    return buf, (C.addressof(buf) + 15) & ~15


def _scene(addr, mode):
    return lib.RenderScene(addr, 8, 8, 8, addr, 3, 8, 8, addr, addr, addr, mode, 0)


def _err():
    return lib.load().mvsn_last_error().decode()


def test_abi_version_and_exports():
    L = lib.load()
    assert L.mvsn_abi_version() == 2
    with open(os.path.join(ROOT, "include", "mvsnerf_b200.h")) as f:
        header = f.read()
    for name in ("mvsn_volume_to_half", "mvsn_costreg_forward_f16"):
        assert name in lib.EXPORTS and hasattr(L, name)
        assert f"int {name}(" in header
    assert "#define MVSN_VOLUME_F16      0x100" in header and lib.VOLUME_F16 == 0x100


def test_mlp_pack_ignores_the_flag():
    L = lib.load()
    for mode in (lib.MLP_FP32, lib.MLP_TC_HALF, lib.MLP_TC_SPLIT, lib.MLP_TC_PAIR):
        assert L.mvsn_mlp_packed_bytes(mode | lib.VOLUME_F16) == L.mvsn_mlp_packed_bytes(mode) > 0
    assert L.mvsn_mlp_packed_bytes(77 | lib.VOLUME_F16) == 0


def test_fp32_mode_rejects_the_flag(mem):
    L = lib.load()
    _, a = mem
    sc = _scene(a, lib.MLP_FP32 | lib.VOLUME_F16)
    rp = lib.RayParams(2.0, 6.0, 0.0, 0)
    assert L.mvsn_render_samples(C.byref(sc), a, a, a, a, 16, 8, a, a, None, None, None, None) == EUNSUPPORTED
    assert "MVSN_VOLUME_F16" in _err()
    assert L.mvsn_render_rays(C.byref(sc), C.byref(rp), a, a, 16, 8, a, a, None, None, None, None) == EUNSUPPORTED
    assert L.mvsn_render_rays_stop(C.byref(sc), C.byref(rp), a, a, 16, 8, 1e-4, a, a, None, None) == EUNSUPPORTED
    sink = lib.PeerSink()
    sink.frame[0], sink.n_peers, sink.first_pixel = a, 1, 0
    assert L.mvsn_render_rays_to_peers(C.byref(sc), C.byref(rp), a, a, 16, 8, C.byref(sink), a, a, None) == EUNSUPPORTED
    assert "MVSN_VOLUME_F16" in _err()


@pytest.mark.parametrize("mode", [lib.MLP_FP32, lib.MLP_TC_HALF])
def test_backward_entries_reject_the_flag(mem, mode):
    L = lib.load()
    _, a = mem
    sc = _scene(a, mode | lib.VOLUME_F16)
    rp = lib.RayParams(2.0, 6.0, 0.0, 0)
    g = lib.RenderGrads()
    g.rgb = a
    ptrs = (C.c_void_p * lib.N_MLP_TENSORS)(*([a] * lib.N_MLP_TENSORS))
    common = (ptrs, a, a, a, a, 16, 8)
    assert L.mvsn_render_backward(C.byref(sc), *common, C.byref(g), ptrs, a, a, 1 << 20, None) == EUNSUPPORTED
    assert L.mvsn_render_backward_tc(C.byref(sc), *common, C.byref(g), ptrs, a, a, 1 << 20, None) == EUNSUPPORTED
    assert L.mvsn_render_backward_deterministic(C.byref(sc), *common, mode, C.byref(g), ptrs, a, a, 1 << 20,
                                                None) == EUNSUPPORTED
    assert L.mvsn_render_backward_rays(C.byref(sc), ptrs, C.byref(rp), a, a, None, 16, 8, mode, 0, C.byref(g), ptrs, a,
                                       a, 1 << 20, None) == EUNSUPPORTED
    assert L.mvsn_render_backward_rays_stop(C.byref(sc), ptrs, C.byref(rp), a, a, None, 16, 8, mode, 0, 1e-4,
                                            C.byref(g), ptrs, a, None, None, a, 1 << 20, None) == EUNSUPPORTED
    assert "mode %d" % (mode | lib.VOLUME_F16) in _err()


def test_conversion_argument_errors(mem):
    L = lib.load()
    _, a = mem
    assert L.mvsn_volume_to_half(None, 0, 1, 8, 8, 8, a, None) == ENULL
    assert L.mvsn_volume_to_half(a, 0, 1, 8, 8, 8, None, None) == ENULL
    assert L.mvsn_volume_to_half(a, 0, 1, 0, 8, 8, a, None) == EBADSHAPE
    assert L.mvsn_volume_to_half(a, 1, 0, 8, -8, 8, a, None) == EBADSHAPE
    assert L.mvsn_volume_to_half(a, 0, 1, 8, 8, 8, a + 8, None) == EALIGN
    assert L.mvsn_volume_to_half(a + 2, 0, 1, 8, 8, 8, a, None) == EALIGN       # fp32 source on a 2-byte boundary
    assert L.mvsn_volume_to_half(a + 1, 1, 0, 8, 8, 8, a, None) == EALIGN       # fp16 source on an odd address
    assert "mvsn_volume_to_half" in _err()


def test_encoder_f16_argument_errors(mem):
    L = lib.load()
    _, a = mem
    w = (C.c_void_p * 30)(*([a] * 30))
    run = (C.c_void_p * 20)(*([a] * 20))
    ws = L.mvsn_costreg_workspace_bytes(8, 8, 8)
    args = lambda bn, D, out: (w, run, bn, 0.1, a, D, 8, 8, out, a, ws)
    assert L.mvsn_costreg_forward_f16(*args(lib.BN_BATCH, 8, None), None) == ENULL
    assert L.mvsn_costreg_forward_f16(*args(lib.BN_BATCH, 12, a), None) == EBADSHAPE
    assert L.mvsn_costreg_forward_f16(*args(7, 8, a), None) == EBADSHAPE
    assert L.mvsn_costreg_forward_f16(*args(lib.BN_BATCH, 8, a + 8), None) == EALIGN
    assert L.mvsn_costreg_forward_f16(None, run, lib.BN_BATCH_UPDATE, 0.1, a, 8, 8, 8, a, a, ws, None) == ENULL


def test_python_rejections_without_a_device():
    with pytest.raises(RuntimeError, match="CUDA"):
        backend.render_rays(torch.zeros(4, 8), torch.zeros(1, 8, 8, 8, 8, dtype=torch.float16), None, None, None,
                            (2.0, 6.0), 0.0)
    with pytest.raises(RuntimeError, match="volume_dtype"):
        backend.CostRegNet(41)(torch.zeros(1, 41, 8, 8, 8), torch.bfloat16)
