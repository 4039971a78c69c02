"""Host-side check of the BA path's buffer layouts (csrc/ba_layout.h), compiled with g++: for every window size the
estimator accepts, with and without the extrinsic, td and relocalisation blocks, and with 0, 1 and the maximum number of
landmarks, each layout's regions are disjoint and inside its total, the input block's arrays are 16-byte aligned, a
frame's input and output blocks fit what the batch reserves per member at capacity, and the packed Schur complement has
the slack its bulk copy needs."""
import ctypes
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = tmp_path_factory.mktemp("balayout") / "libbalayout.so"
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wall", "-Werror",
                           os.path.join(ROOT, "tests", "hostlib", "ba_layout_host.cpp"), "-o", str(out)])
    l = ctypes.CDLL(str(out))
    l.check_ba_layouts.argtypes = [ctypes.c_int, ctypes.POINTER(ctypes.c_long), ctypes.c_char_p, ctypes.c_int]
    l.check_ba_layouts.restype = ctypes.c_long
    return l


@pytest.mark.parametrize("max_features", [8, 150, 1000])
def test_ba_layouts(lib, max_features):
    n = ctypes.c_long(0)
    msg = ctypes.create_string_buffer(256)
    failures = lib.check_ba_layouts(max_features, ctypes.byref(n), msg, len(msg))
    assert failures == 0, msg.value.decode()
    assert n.value > 10000
