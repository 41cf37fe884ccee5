"""The boundary is a plain C ABI: include/mvsnerf_b200.h must compile as C (not only C++), and a C program
linked against libmvsnerf_b200.so must be able to call it without PyTorch, Python or a GPU."""
import os
import shutil
import subprocess
import sys

import pytest

from conftest import ROOT
from mvsnerf_b200 import build

C_SRC = r"""
#include <stdio.h>
#include <string.h>
#include "mvsnerf_b200.h"

int main(void) {
    struct mvsn_render_scene sc;
    struct mvsn_ray_params rp;
    memset(&sc, 0, sizeof sc);
    memset(&rp, 0, sizeof rp);
    if (mvsn_abi_version() != 2) return 1;
    if (mvsn_mlp_packed_bytes(MVSN_MLP_FP32) == 0 || mvsn_mlp_packed_bytes(MVSN_MLP_TC_HALF) == 0 ||
        mvsn_mlp_packed_bytes(MVSN_MLP_TC_SPLIT) == 0 || mvsn_mlp_packed_bytes(77) != 0) return 2;
    if (mvsn_costreg_workspace_bytes(128, 176, 208) == 0 || mvsn_featurenet_workspace_bytes(3, 512, 640) == 0 ||
        mvsn_cost_volume_workspace_bytes(3, 128, 160) == 0) return 3;
    /* argument errors are reported without touching a device */
    if (mvsn_render_samples(&sc, 0, 0, 0, 0, 16, 8, 0, 0, 0, 0, 0, 0) >= 0) return 4;
    if (strlen(mvsn_last_error()) == 0) return 5;
    if (mvsn_render_rays(0, &rp, 0, 0, 16, 8, 0, 0, 0, 0, 0, 0) >= 0) return 6;
    if (mvsn_featurenet_forward(0, 0, 3, 32, 32, 0, 0, 0, 0) != MVSN_ENULL) return 7;
    printf("abi %d ok: %s\n", mvsn_abi_version(), mvsn_last_error());
    return 0;
}
"""


@pytest.mark.skipif(shutil.which("gcc") is None, reason="no C compiler")
def test_header_is_c_and_abi2_library_links_from_c(tmp_path):
    lib_path = build.build_library()
    src = tmp_path / "abi_check.c"
    src.write_text(C_SRC)
    exe = tmp_path / "abi_check"
    inc = os.path.join(ROOT, "include")
    libdir = os.path.dirname(lib_path)
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", inc, str(src), "-o", str(exe),
                        "-L", libdir, "-lmvsnerf_b200", "-Wl,-rpath," + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "abi 2 ok" in r.stdout
