"""CPU checks of loop verification: the twin's blur and FAST against cv2 on textured and random images, its BRIEF
against a per-bit restatement, the descriptor-arena layouts (lv_layout.h, with g++), the vp_ loop symbols exported, the
sm_90a compile of lv_kernels.cu without spills, and creation failing without a GPU."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import loop_verify as olv  # noqa: E402
from harness import synth  # noqa: E402

CSRC = os.path.join(ROOT, "vins_mono_b200", "csrc")


def _images():
    yield synth.value_noise_image(480, 752, 0)
    yield np.random.default_rng(1).integers(0, 256, (480, 752)).astype(np.uint8)
    yield synth.value_noise_image(97, 131, 3)


def test_twin_blur_and_fast_match_cv2():
    import cv2
    assert list(olv.gaussian_kernel_q8()) == [7, 17, 32, 46, 52, 46, 32, 17, 7]
    for img in _images():
        assert np.array_equal(olv.gaussian_blur(img), cv2.GaussianBlur(img, (9, 9), 2, 2))
        kp = cv2.FastFeatureDetector_create(20, True).detect(img)
        ref = np.array([[k.pt[0], k.pt[1]] for k in kp]).astype(np.int32)
        xy, score = olv.fast(img)
        assert np.array_equal(xy, ref)
        assert np.array_equal(score, np.array([k.response for k in kp]).astype(np.int32))


def test_twin_brief_matches_per_bit_restatement():
    pat = olv.load_pattern()
    img = synth.value_noise_image(480, 752, 2)
    im = olv.gaussian_blur(img)
    rng = np.random.default_rng(0)
    pts = np.r_[rng.uniform(-5, 757, (60, 2)), [[0.5, 0.5], [-0.5, 10.0], [751.9, 479.9]]].astype(np.float32)
    d = olv.brief(img, pts, pat)
    for p, words in zip(pts, d):
        for i, (x1, y1, x2, y2) in enumerate(pat):
            a = [int(np.float32(p[0]) + np.float32(x1)), int(np.float32(p[1]) + np.float32(y1))]
            b = [int(np.float32(p[0]) + np.float32(x2)), int(np.float32(p[1]) + np.float32(y2))]
            inside = all(0 <= v < 752 for v in (a[0], b[0])) and all(0 <= v < 480 for v in (a[1], b[1]))
            bit = inside and im[a[1], a[0]] < im[b[1], b[0]]
            assert bool((int(words[i // 64]) >> (i % 64)) & 1) == bit
    idx, dist = olv.match(d[:10], d)
    first = [int(np.nonzero((d == d[i]).all(1))[0][0]) for i in range(10)]  # equal descriptors: the first index wins
    assert np.array_equal(idx, first) and not dist.any()


def test_lv_layouts(tmp_path):
    out = tmp_path / "liblvlayout.so"
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wall", "-Werror", "-I", CSRC,
                           os.path.join(ROOT, "tests", "hostlib", "lv_layout_host.cpp"), "-o", str(out)])
    lib = ctypes.CDLL(str(out))
    lib.check_lv_layouts.argtypes = [ctypes.POINTER(ctypes.c_long), ctypes.c_char_p, ctypes.c_int]
    lib.check_lv_layouts.restype = ctypes.c_long
    n = ctypes.c_long(0)
    msg = ctypes.create_string_buffer(256)
    assert lib.check_lv_layouts(ctypes.byref(n), msg, len(msg)) == 0, msg.value.decode()
    assert n.value > 60


def test_loop_symbols_exported_and_no_gpu_fails_loudly():
    import torch
    from vins_mono_b200 import build, load_library
    build.build()
    lib = load_library()
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "vinsb200", "loop_verify.h")).read(), flags=re.S)
    names = sorted(set(re.findall(r"\b(vp_[a-z0-9_]+)\s*\(", src)))
    assert len(names) == 12 and not [n for n in names if not hasattr(lib, n)]
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from vins_mono_b200 import pose_graph as pg
    with pytest.raises(RuntimeError):
        pg.debug_fast(np.zeros((16, 16), np.uint8))
    with pytest.raises(RuntimeError):
        pg.PoseGraph()


def test_lv_kernels_compile_for_sm90a_without_spills(tmp_path):
    from vins_mono_b200 import build
    r = subprocess.run(["nvcc", *build.ARCH, "-O3", "-std=c++17", "--fmad=false", "-Xptxas", "-v", "-I", CSRC, "-I",
                        os.path.join(ROOT, "include"), "-c", os.path.join(CSRC, "lv_kernels.cu"), "-o", str(tmp_path / "lv.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    spills, kernel = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"(?:entry function|Function properties for) '?\S*?(lv_[a-z_]+kernel)", line)
        if m:
            kernel = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and kernel:
            spills[kernel] = spills.get(kernel, 0) + int(m.group(1)) + int(m.group(2))
    for k in ("lv_blur_kernel", "lv_fast_score_kernel", "lv_fast_nms_kernel", "lv_fast_compact_kernel", "lv_brief_kernel",
              "lv_match_kernel", "lv_pnp_hyp_kernel", "lv_pnp_refit_kernel"):
        assert k in spills, (k, sorted(spills))
    assert not any(spills.values()), spills
