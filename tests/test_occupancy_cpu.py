"""Empty-space skipping without a GPU: the new entries are exported and declared for C callers, report their argument
errors before any CUDA call, the ABI version stays 2, and the host restatement of the cell reduction, the dilation, the
bit packing and the group ranges (tests/occupancy_host.py, which the GPU tests compare the kernels with) is pinned on
small hand-made inputs."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT
from mvsnerf_b200 import build, lib
import occupancy_host as oh

NEW = ["mvsn_occupancy_bytes", "mvsn_build_occupancy_workspace_bytes", "mvsn_build_occupancy",
       "mvsn_render_rays_occ_workspace_bytes", "mvsn_render_rays_occ"]

C_SRC = r"""
#include <stdio.h>
#include <string.h>
#include "mvsnerf_b200.h"

int main(void) {
    static float buf[64] __attribute__((aligned(16)));
    static uint32_t bits[64];
    struct mvsn_render_scene sc;
    struct mvsn_ray_params rp;
    struct mvsn_occupancy occ;
    memset(&sc, 0, sizeof sc);
    memset(&rp, 0, sizeof rp);
    sc.volume_dhwc = buf; sc.imgs_hwc4 = buf; sc.mlp_packed = buf; sc.w2cs = buf; sc.intrinsics = buf;
    sc.D = sc.Hp = sc.Wp = 8; sc.V = 3; sc.H = sc.W = 8; sc.mlp_mode = MVSN_MLP_TC_SPLIT;
    occ.bits = bits; occ.D = occ.Hp = occ.Wp = 8;
    if (mvsn_abi_version() != 2) return 1;
    if (mvsn_occupancy_bytes(8, 8, 8) != 64) return 2;
    if (mvsn_build_occupancy(&sc, &rp, -1, bits, buf, 1 << 30, 0) != MVSN_EBADSHAPE) return 3;
    if (mvsn_render_rays_occ(&sc, &rp, buf, buf, 16, 8, 0.f, 0, buf, buf, 0, buf, 256, 0) != MVSN_ENULL) return 4;
    occ.Wp = 16;
    if (mvsn_render_rays_occ(&sc, &rp, buf, buf, 16, 8, 0.f, &occ, buf, buf, 0, buf, 256, 0) != MVSN_EBADSHAPE) return 5;
    printf("occ ok: %s\n", mvsn_last_error());
    return 0;
}
"""


def test_symbols_exported_and_declared():
    L = lib.load()
    with open(os.path.join(ROOT, "include", "mvsnerf_b200.h")) as f:
        header = f.read()
    for name in NEW:
        assert name in lib.EXPORTS and hasattr(L, name)
        assert f" {name}(" in header, name
    assert "typedef struct mvsn_occupancy" in header
    assert L.mvsn_abi_version() == 2


@pytest.mark.skipif(shutil.which("gcc") is None, reason="no C compiler")
def test_c_program_links_and_gets_argument_errors(tmp_path):
    lib_path = build.build_library()
    src = tmp_path / "occ_check.c"
    src.write_text(C_SRC)
    exe = tmp_path / "occ_check"
    libdir = os.path.dirname(lib_path)
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src),
                        "-o", str(exe), "-L", libdir, "-lmvsnerf_b200", "-Wl,-rpath," + libdir], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "occ ok" in r.stdout and "does not match" in r.stdout


class Buf:
    def __init__(self):
        self.mem = (C.c_float * 4096)()
        self.addr = (C.addressof(self.mem) + 15) & ~15


def _scene(b, mode, dims=(8, 8, 8)):
    return lib.RenderScene(b.addr, *dims, b.addr, 3, 8, 8, b.addr, b.addr, b.addr, mode, 0)


def test_sizes():
    L = lib.load()
    assert L.mvsn_occupancy_bytes(128, 176, 208) == 4 * ((128 * 176 * 208 + 31) // 32)   # 586 KB at 512x640, pad 24
    assert L.mvsn_occupancy_bytes(0, 8, 8) == 0
    assert L.mvsn_build_occupancy_workspace_bytes(1, 8, 8) == 0
    assert L.mvsn_build_occupancy_workspace_bytes(8, 8, 8) > 8 * 8 * 8 * 4
    assert L.mvsn_render_rays_occ_workspace_bytes(1000, 128) >= 250 * 8
    assert L.mvsn_render_rays_occ_workspace_bytes(-1, 128) == 0 and L.mvsn_render_rays_occ_workspace_bytes(8, 0) == 0


def _build(mode=lib.MLP_TC_SPLIT, dilate=1, bits_off=0, ws_off=0, ws_bytes=1 << 30, dims=(8, 8, 8)):
    L, b = lib.load(), Buf()
    sc = _scene(b, mode, dims)
    rp = lib.RayParams(2.0, 6.0, 0.0, 0)
    rc = L.mvsn_build_occupancy(C.byref(sc), C.byref(rp), dilate, b.addr + bits_off, b.addr + ws_off, ws_bytes, None)
    return rc, L.mvsn_last_error().decode()


def test_build_argument_errors():
    rc, msg = _build(mode=lib.MLP_TC_PAIR)
    assert rc == -6 and "MVSN_MLP_TC_SPLIT" in msg                                  # MVSN_EUNSUPPORTED
    rc, msg = _build(mode=lib.MLP_FP32)
    assert rc == -6
    rc, msg = _build(dilate=-1)
    assert rc == -1 and "dilate" in msg                                             # MVSN_EBADSHAPE
    rc, msg = _build(dilate=9)
    assert rc == -1 and "dilate" in msg
    rc, msg = _build(dims=(1, 8, 8))
    assert rc == -1
    rc, msg = _build(bits_off=2)
    assert rc == -2 and "bits" in msg                                               # MVSN_EALIGN
    rc, msg = _build(ws_off=4)
    assert rc == -2 and "workspace" in msg
    rc, msg = _build(ws_bytes=16)
    assert rc == -5                                                                 # MVSN_EWORKSPACE


def _render(mode=lib.MLP_TC_PAIR, grid_dims=(8, 8, 8), occ=True, bits_off=0, ws_off=0, ws_bytes=4096, t_stop=0.0):
    L, b = lib.load(), Buf()
    sc = _scene(b, mode)
    rp = lib.RayParams(2.0, 6.0, 0.0, 0)
    grid = lib.OccupancyGrid(b.addr + bits_off, *grid_dims)
    rc = L.mvsn_render_rays_occ(C.byref(sc), C.byref(rp), b.addr, b.addr, 16, 8, t_stop, C.byref(grid) if occ else None,
                                b.addr, b.addr, None, b.addr + ws_off, ws_bytes, None)
    return rc, L.mvsn_last_error().decode()


def test_render_argument_errors():
    assert _render(occ=False)[0] == -4                                              # MVSN_ENULL
    rc, msg = _render(mode=lib.MLP_FP32)
    assert rc == -6 and "mlp_mode 0" in msg
    rc, msg = _render(t_stop=-1.0)
    assert rc == -1 and "t_stop" in msg
    for dims in ((8, 8, 16), (4, 8, 8), (8, 16, 8)):
        rc, msg = _render(grid_dims=dims)
        assert rc == -1 and "does not match" in msg, dims                          # MVSN_EBADSHAPE
    rc, msg = _render(bits_off=2)
    assert rc == -2 and "bits" in msg
    rc, msg = _render(ws_off=8)
    assert rc == -2 and "workspace" in msg
    rc, msg = _render(ws_bytes=8)
    assert rc == -5


def test_python_rejections_without_a_device():
    from mvsnerf_b200 import backend
    with pytest.raises(RuntimeError, match="Occupancy"):
        backend.render_rays(torch.zeros(4, 8), None, None, None, None, (2.0, 6.0), 0.0, occupancy=object())
    occ = backend.Occupancy(torch.zeros(16, dtype=torch.int32), 8, 8, 8, (2.0, 6.0), 0.0, False, 1)
    with pytest.raises(RuntimeError, match="sink"):
        backend.render_rays(torch.zeros(4, 8), None, None, None, None, (2.0, 6.0), 0.0, occupancy=occ, sink=object())
    with pytest.raises(RuntimeError, match="tensor-core"):
        backend.render_rays(torch.zeros(4, 8), None, None, None, None, (2.0, 6.0), 0.0, occupancy=occ, mlp_mode=lib.MLP_FP32)
    with pytest.raises(RuntimeError, match="near_far"):
        backend.render_rays(torch.zeros(4, 8), None, None, None, None, (2.0, 7.0), 0.0, occupancy=occ)
    with pytest.raises(RuntimeError, match="near_far"):
        backend.render_rays(torch.zeros(4, 8), None, None, None, None, (2.0, 6.0), 0.0, lindisp=True, occupancy=occ)
    with pytest.raises(RuntimeError, match="dilate"):
        backend.build_occupancy(None, None, None, None, (2.0, 6.0), 0.0, dilate=9)


def test_occupancy_cells_unpack():
    from mvsnerf_b200 import backend
    cells = np.zeros((3, 4, 5), dtype=bool)
    cells[1, 2, 3] = cells[0, 0, 0] = True
    occ = backend.Occupancy(torch.from_numpy(oh.pack(cells)), 3, 4, 5, (2.0, 6.0), 0.0, False, 0)
    assert np.array_equal(occ.cells().numpy(), cells)
    assert occ.fraction() == 2 / (2 * 3 * 4)


# ---- the host restatement, pinned ---------------------------------------------------------------------------------
def test_cells_from_alpha():
    a = np.zeros((3, 3, 4), dtype=np.float32)
    assert not oh.cells_from_alpha(a).any()
    a[1, 1, 2] = 0.5                                           # an interior node: the eight cells around it
    c = oh.cells_from_alpha(a)
    assert c.sum() == 8 and c[0:2, 0:2, 1:3].all()
    a[:] = 0
    a[2, 2, 3] = 1e-30                                         # the far corner node: only the last valid cell
    c = oh.cells_from_alpha(a)
    assert c.sum() == 1 and c[1, 1, 2]
    a[:] = 0
    a[0, 0, 0] = -1.0                                          # alpha > 0 only
    assert not oh.cells_from_alpha(a).any()


def test_dilate():
    c = np.zeros((5, 6, 7), dtype=bool)
    c[2, 2, 3] = True
    d1 = oh.dilate(c, 1)
    assert d1.sum() == 27 and d1[1:4, 1:4, 2:5].all()
    assert np.array_equal(oh.dilate(c, 0), c)
    d2 = oh.dilate(c, 2)                                       # clipped to the valid cells [0, n - 2]
    assert d2.sum() == 4 * 5 * 5 and d2[0:4, 0:5, 1:6].all() and not d2[4].any() and not d2[:, 5].any()
    e = np.zeros((5, 6, 7), dtype=bool)
    e[0, 0, 0] = True
    assert oh.dilate(e, 1).sum() == 8


def test_pack_round_trip():
    rng = np.random.default_rng(0)
    c = rng.random((3, 5, 7)) < 0.3
    w = oh.pack(c)
    assert w.dtype == np.int32 and w.size == (3 * 5 * 7 + 31) // 32
    assert np.array_equal(oh.unpack(w, c.shape), c)
    one = np.zeros((1, 1, 40), dtype=bool)
    one[0, 0, 33] = one[0, 0, 31] = True
    assert oh.pack(one).view(np.uint32).tolist() == [1 << 31, 2]


def test_sample_occupied():
    cells = np.zeros((3, 3, 3), dtype=bool)                    # 2 x 2 x 2 valid cells
    cells[1, 0, 1] = True
    ndc = np.array([[0.75, 0.25, 0.75],                        # cell (1, 0, 1)
                    [0.25, 0.25, 0.25],                        # cell (0, 0, 0)
                    [1.0, 0.0, 1.0],                           # the far faces clamp to the last cell: (1, 0, 1)
                    [0.5, 0.25, 0.5],                          # on the middle face: floor -> cell (1, 0, 1)
                    [-0.01, 0.5, 0.5],                         # outside: occupied
                    [0.5, 0.5, 1.01],
                    [np.nan, 0.5, 0.5]], dtype=np.float32)
    assert oh.sample_occupied(ndc, cells).tolist() == [True, False, True, True, True, True, True]


def test_group_ranges():
    occ = np.zeros((10, 9), dtype=bool)                        # rt = 4: 16 samples per tile -> NT = 1
    occ[5, 3] = True
    assert oh.group_ranges(occ, 4).tolist() == [[1, -1], [0, 0], [1, -1]]
    occ = np.zeros((6, 20), dtype=bool)                        # rt = 32: 2 samples per tile -> NT = 10, one group
    occ[0, 5] = occ[3, 16] = occ[5, 7] = True
    assert oh.group_ranges(occ, 32).tolist() == [[2, 8]]
    assert oh.group_ranges(np.zeros((6, 20), dtype=bool), 32).tolist() == [[10, -1]]
    occ = np.zeros((16, 40), dtype=bool)                       # rt = 8: 8 samples per tile -> NT = 5, two groups
    occ[2, 39] = occ[9, 8] = occ[15, 15] = True
    assert oh.group_ranges(occ, 8).tolist() == [[4, 4], [1, 1]]
    assert oh.rays_per_tile(327680, 132) == 32 and oh.rays_per_tile(1994, 132) == 4
