"""Early ray termination without a GPU: mvsn_render_rays_stop is exported, declared for C callers, and reports its
argument errors before any CUDA call; the plane scene the GPU tests render is seeded."""
import ctypes as C
import math
import os
import shutil
import subprocess

import pytest
import torch

from conftest import ROOT
from mvsnerf_b200 import build, lib, synthetic

C_SRC = r"""
#include <math.h>
#include <stdio.h>
#include <string.h>
#include "mvsnerf_b200.h"

int main(void) {
    static float buf[64] __attribute__((aligned(16)));
    struct mvsn_render_scene sc;
    struct mvsn_ray_params rp;
    unsigned long long tiles = 0;
    memset(&sc, 0, sizeof sc);
    memset(&rp, 0, sizeof rp);
    sc.volume_dhwc = buf; sc.imgs_hwc4 = buf; sc.mlp_packed = buf; sc.w2cs = buf; sc.intrinsics = buf;
    sc.D = sc.Hp = sc.Wp = 8; sc.V = 3; sc.H = sc.W = 8; sc.mlp_mode = MVSN_MLP_TC_PAIR;
    if (mvsn_render_rays_stop(&sc, &rp, buf, buf, 16, 8, 1e-4f, 0, buf, &tiles, 0) != MVSN_ENULL) return 1;
    if (mvsn_render_rays_stop(&sc, &rp, buf, buf, 16, 8, -1.f, buf, buf, &tiles, 0) != MVSN_EBADSHAPE) return 2;
    if (mvsn_render_rays_stop(&sc, &rp, buf, buf, 16, 8, (float)NAN, buf, buf, &tiles, 0) != MVSN_EBADSHAPE) return 3;
    sc.mlp_mode = MVSN_MLP_FP32;
    if (mvsn_render_rays_stop(&sc, &rp, buf, buf, 16, 8, 1e-4f, buf, buf, &tiles, 0) != MVSN_EUNSUPPORTED) return 4;
    printf("stop ok: %s\n", mvsn_last_error());
    return 0;
}
"""


def test_symbol_is_exported():
    assert "mvsn_render_rays_stop" in lib.EXPORTS
    assert hasattr(lib.load(), "mvsn_render_rays_stop")
    with open(os.path.join(ROOT, "include", "mvsnerf_b200.h")) as f:
        assert "int mvsn_render_rays_stop(" in f.read()


@pytest.mark.skipif(shutil.which("gcc") is None, reason="no C compiler")
def test_c_program_links_and_gets_argument_errors(tmp_path):
    lib_path = build.build_library()
    src = tmp_path / "stop_check.c"
    src.write_text(C_SRC)
    exe = tmp_path / "stop_check"
    libdir = os.path.dirname(lib_path)
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src),
                        "-o", str(exe), "-L", libdir, "-lmvsnerf_b200", "-Wl,-rpath," + libdir], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "stop ok" in r.stdout and "mlp_mode 0" in r.stdout


def _call(mode, t_stop, null_rgb=False):
    L = lib.load()
    buf = (C.c_float * 64)()
    addr = (C.addressof(buf) + 15) & ~15
    sc = lib.RenderScene(addr, 8, 8, 8, addr, 3, 8, 8, addr, addr, addr, mode, 0)
    rp = lib.RayParams(2.0, 6.0, 0.0, 0)
    rc = L.mvsn_render_rays_stop(C.byref(sc), C.byref(rp), addr, addr, 16, 8, t_stop, None if null_rgb else addr, addr,
                                 None, None)
    return rc, L.mvsn_last_error().decode()


def test_argument_errors_in_order():
    assert _call(lib.MLP_TC_PAIR, 1e-4, null_rgb=True)[0] == -4                     # MVSN_ENULL
    rc, msg = _call(lib.MLP_TC_SPLIT, -1e-3)
    assert rc == -1 and "t_stop" in msg                                             # MVSN_EBADSHAPE
    rc, msg = _call(lib.MLP_TC_HALF, math.nan)
    assert rc == -1 and "t_stop" in msg
    rc, msg = _call(lib.MLP_FP32, 1e-4)
    assert rc == -6 and "mlp_mode 0" in msg                                         # MVSN_EUNSUPPORTED
    rc, msg = _call(lib.MLP_FP32, -1.0, null_rgb=True)                              # NULL is reported first
    assert rc == -4


def test_misaligned_tiles_done():
    L = lib.load()
    buf = (C.c_float * 64)()
    addr = (C.addressof(buf) + 15) & ~15
    sc = lib.RenderScene(addr, 8, 8, 8, addr, 3, 8, 8, addr, addr, addr, lib.MLP_TC_PAIR, 0)
    rp = lib.RayParams(2.0, 6.0, 0.0, 0)
    rc = L.mvsn_render_rays_stop(C.byref(sc), C.byref(rp), addr, addr, 16, 8, 1e-4, addr, addr, addr + 4, None)
    assert rc == -2 and "tiles_done" in L.mvsn_last_error().decode()                 # MVSN_EALIGN


def test_python_rejections_without_a_device():
    from mvsnerf_b200 import backend
    with pytest.raises(RuntimeError, match="CUDA"):
        backend.render_rays(torch.zeros(4, 8), None, None, None, None, (2.0, 6.0), 0.0, t_stop=1e-4)


def test_plane_scene_is_seeded():
    a = synthetic.make_plane_scene(48, 64, pad=4, seed=3)
    b = synthetic.make_plane_scene(48, 64, pad=4, seed=3)
    c = synthetic.make_plane_scene(48, 64, pad=4, seed=4)
    assert torch.equal(a.imgs_raw, b.imgs_raw) and torch.equal(a.imgs_norm, b.imgs_norm)
    assert not torch.equal(a.imgs_raw, c.imgs_raw)
    assert a.imgs_raw.shape == (1, 3, 3, 48, 64) and 0.0 <= a.imgs_raw.min() and a.imgs_raw.max() <= 1.0
    ref = synthetic.make_scene(48, 64, pad=4, seed=3)                               # same cameras as make_scene
    assert torch.equal(a.pose_source["w2cs"], ref.pose_source["w2cs"]) and torch.equal(a.proj_mats, ref.proj_mats)
