"""Ownership of the CUDA resources behind the C ABI: every buffer, stream and event of a handle is one of the owning types of
csrc/cuda_check.h, so create paths that fail half-way and destroy paths release the same things.  The GPU tests read the
owners' live count (vb_debug_live_cuda_objects) rather than the device's free memory, which other processes change."""
import ctypes as C
import gc
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "vins_mono_b200", "csrc")
RAW_CALL = re.compile(r"\bcuda(Malloc|Free|HostAlloc|MallocHost|FreeHost|StreamCreate\w*|StreamDestroy|EventCreate\w*|EventDestroy|"
                      r"FuncSetAttribute)\s*\(")

TRACKER = dict(rows=64, cols=96, max_cnt=20, min_dist=10)
ESTIMATOR = dict(max_features=64)
VP_ERR_INVALID, VP_ERR_CUDA, VP_ERR_CAPACITY = -1, -3, -4


def test_cuda_resources_are_taken_only_through_the_owning_header():
    hits = []
    for f in sorted(os.listdir(CSRC)):
        if f == "cuda_check.h":
            continue
        for i, line in enumerate(open(os.path.join(CSRC, f)).read().splitlines(), 1):
            if RAW_CALL.search(line):
                hits.append(f"{f}:{i}: {line.strip()}")
    assert not hits, hits


def _live(lib):
    gc.collect()  # a batch and its members reference each other: release the ones earlier tests dropped without close()
    lib.vb_debug_live_cuda_objects.restype = C.c_longlong
    return lib.vb_debug_live_cuda_objects()


def _loop_config(**kw):
    from vins_mono_b200.pose_graph import loop_config
    args = dict(max_window=16, max_corners=256)
    args.update(kw)
    return loop_config(64, 96, [400.0, 400.0, 48.0, 32.0, 0, 0, 0, 0], np.eye(3), np.zeros(3), np.zeros((256, 4), np.int32), **args)


@pytest.mark.gpu
@pytest.mark.parametrize("profile", [False, True])
def test_every_handle_kind_releases_what_it_owns(profile):
    from vins_mono_b200 import Estimator, EstimatorBatch, FeatureTracker, PoseGraph, PoseGraphBatch, TrackerBatch, load_library
    lib = load_library()
    base = _live(lib)
    img = np.zeros((TRACKER["rows"], TRACKER["cols"]), np.uint8)
    for _ in range(3):
        handles = [FeatureTracker(**TRACKER), TrackerBatch(3, **TRACKER), Estimator(**ESTIMATOR), EstimatorBatch(3, **ESTIMATOR)]
        for h in handles:
            h.set_profile(profile)
        handles[0].readImage(img, 0.0, True)  # records the profile's events when they exist
        g, gb = PoseGraph(max_keyframes=16), PoseGraphBatch(3, max_keyframes=16)
        g.enable_loop(_loop_config())
        gb.enable_loop(_loop_config())
        handles += [g, gb]
        assert _live(lib) > base
        for h in handles:
            h.close()
        assert _live(lib) == base


@pytest.mark.gpu
def test_failed_creates_release_what_they_took():
    import torch
    from vins_mono_b200 import PoseGraph, PoseGraphBatch, PoseGraphError, load_library
    lib = load_library()
    total = torch.cuda.get_device_properties(0).total_memory
    base = _live(lib)

    g = PoseGraph(max_keyframes=16)
    g.enable_loop(_loop_config())
    with pytest.raises(PoseGraphError) as err:
        g.enable_loop(_loop_config())
    assert err.value.status == VP_ERR_INVALID and "already enabled" in str(err.value)
    g.close()
    assert _live(lib) == base

    # the workspace of 1024 anchors holds at least (4 x 1024)^2 doubles per member: the last allocation of the create fails,
    # after a few MB of pinned and device buffers
    n = 1024
    assert n * (4 * 1024) ** 2 * 8 > total
    with pytest.raises(RuntimeError, match=f"status {VP_ERR_CUDA}"):
        PoseGraphBatch(n, max_keyframes=2, max_anchors=1024)
    assert _live(lib) == base
    PoseGraphBatch(2, max_keyframes=16).close()

    # a descriptor arena of 60000 key frames x 65536 corners (32-byte descriptors): the first allocation of the enable fails
    g = PoseGraph(max_keyframes=60000)
    assert 60000 * 65536 * 32 > total
    with pytest.raises(PoseGraphError) as err:
        g.enable_loop(_loop_config(max_window=1, max_corners=65536))
    assert err.value.status == VP_ERR_CAPACITY and "out of memory" in str(err.value)
    g.enable_loop(_loop_config())
    g.close()
    assert _live(lib) == base
