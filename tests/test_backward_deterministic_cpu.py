"""CPU: the C ABI of the deterministic fine-tuning backward (mvsn_render_backward_deterministic) -- declared, exported,
bound, sized, and its argument errors returned without a device."""
import ctypes
import os

import pytest

from conftest import ROOT
from mvsnerf_b200 import lib

NAMES = ("mvsn_render_backward_deterministic_workspace_bytes", "mvsn_render_backward_deterministic")


@pytest.fixture(scope="module")
def built():
    from mvsnerf_b200 import build
    return build.build_library()


def test_deterministic_backward_is_declared_and_exported(built):
    header = open(os.path.join(ROOT, "include", "mvsnerf_b200.h")).read()
    dll = ctypes.CDLL(built)
    for name in NAMES:
        assert name + "(" in header, name
        assert name in lib.EXPORTS, name
        assert hasattr(dll, name), name


def test_deterministic_workspace_sizes(built):
    L = lib.load()
    ws = L.mvsn_render_backward_deterministic_workspace_bytes
    N, S, D, H, W = 1024, 128, 128, 200, 200
    for mode, base in ((lib.MLP_FP32, L.mvsn_render_backward_workspace_bytes(N, S)),
                       (lib.MLP_TC_HALF, L.mvsn_render_backward_tc_workspace_bytes(N, S))):
        frozen, full = ws(N, S, 0, 0, 0, mode), ws(N, S, D, H, W, mode)
        assert frozen >= base + 4 * N                            # + the per-ray loss terms
        assert full - frozen >= D * H * W * 8 * 8 + N * S * 8 * 4  # + int64 accumulator and the [N*S][8] record
    assert ws(N, S, D, H, W, lib.MLP_TC_PAIR) == 0               # unknown grad_mode
    assert ws(N, S, D, H, W, 99) == 0
    assert ws(N, 160, D, H, W, lib.MLP_FP32) == 0                # N_samples > 128
    assert ws(0, S, D, H, W, lib.MLP_FP32) == 0
    assert ws(N, S, D, 0, W, lib.MLP_FP32) == 0                  # a partially empty volume is not "frozen"


def test_deterministic_backward_argument_errors_need_no_gpu(built):
    L = lib.load()
    f = L.mvsn_render_backward_deterministic
    args = lambda mode: (None, None, None, None, None, None, 8, 32, mode, None, None, None, None, 0, None)  # noqa: E731
    for mode in (lib.MLP_TC_SPLIT, lib.MLP_TC_PAIR, -1, 99):
        assert f(*args(mode)) == -6                              # MVSN_EUNSUPPORTED, checked first
        assert b"grad_mode" in L.mvsn_last_error()
    for mode in (lib.MLP_FP32, lib.MLP_TC_HALF):
        assert f(*args(mode)) == -4                              # MVSN_ENULL: scene
        assert b"NULL" in L.mvsn_last_error()
