"""CPU checks of the pose graph's anchor capacity (vp_config::max_anchors): the workspace and arena layouts at anchor
capacities on both sides of the one-CTA border limit (pg_layout.h, with g++), the creation-time bounds (checked before any
device is looked for), and the cross-compile of the pose-graph kernels for sm_90a with no register spills."""
import ctypes
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CSRC = os.path.join(ROOT, "vins_mono_b200", "csrc")


@pytest.mark.parametrize("cap_anchors", [88, 89, 256, 1024])
def test_pg_layouts_at_anchor_capacity(tmp_path, cap_anchors):
    out = tmp_path / "libpglayoutcap.so"
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wall", "-Werror", "-I", CSRC,
                           os.path.join(ROOT, "tests", "hostlib", "pg_layout_cap_host.cpp"), "-o", str(out)])
    lib = ctypes.CDLL(str(out))
    lib.check_pg_layouts_cap.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_long), ctypes.c_char_p, ctypes.c_int]
    lib.check_pg_layouts_cap.restype = ctypes.c_long
    for cap_n in (8, 501, 2048, 2100):
        n = ctypes.c_long(0)
        msg = ctypes.create_string_buffer(256)
        assert lib.check_pg_layouts_cap(cap_n, cap_anchors, ctypes.byref(n), msg, len(msg)) == 0, msg.value.decode()
        assert n.value > 4


@pytest.mark.parametrize("max_anchors", [-1, 1025])
def test_out_of_range_anchor_capacity_is_invalid(max_anchors):
    from vins_mono_b200 import build, load_library
    from vins_mono_b200.pose_graph import PoseGraphConfig
    build.build()
    lib = load_library()
    cfg = PoseGraphConfig(max_keyframes=64, fast_relocalization=0, device=0, max_anchors=max_anchors)
    h = ctypes.c_void_p()
    assert lib.vp_create(ctypes.byref(cfg), ctypes.byref(h)) == -1 and not h.value
    assert lib.vp_batch_create(ctypes.byref(cfg), 2, ctypes.byref(h)) == -1 and not h.value


def test_pg_kernels_compile_for_sm90a_without_spills(tmp_path):
    from vins_mono_b200 import build
    r = subprocess.run(["nvcc", *build.ARCH, "-O3", "-std=c++17", "--fmad=true", "-Xptxas", "-v", "-I", CSRC, "-I",
                        os.path.join(ROOT, "include"), "-c", os.path.join(CSRC, "pg_kernels.cu"), "-o", str(tmp_path / "pg.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    spills = {}
    kernel = None
    for line in r.stderr.splitlines():
        m = re.search(r"(?:entry function|Function properties for) '?\S*?(pg_[a-z_]+kernel)", line)
        if m:
            kernel = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and kernel:
            spills[kernel] = spills.get(kernel, 0) + int(m.group(1)) + int(m.group(2))
    for k in ("pg_chain_kernel", "pg_border_kernel", "pg_solve_kernel", "pg_tile_kernel", "pg_panel_kernel", "pg_solve_large_kernel"):
        assert k in spills, (k, sorted(spills))
    assert not any(spills.values()), spills
