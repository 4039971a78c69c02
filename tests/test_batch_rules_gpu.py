"""The rules every batched handle family shares (csrc/batch_host.h), on the tracker, the estimator and the pose graph: a
per-handle call on a member of an explicit batch is refused and names the batch call; a member that fails in a batch
step keeps its own text, which the estimator's batch reports as "member k: <text>" while the pose graph's batch reports
each member's status and keeps its own text; a member's last error falls back to its batch's; and every case releases
the CUDA objects it created."""
import ctypes as C

import numpy as np
import pytest

from harness import pipeline, synth
from test_cuda_owners import ESTIMATOR, TRACKER, _live, _loop_config

pytestmark = pytest.mark.gpu

INVALID, CAPACITY = -1, -4


@pytest.fixture
def lib():
    from vins_mono_b200 import load_library
    lib = load_library()
    base = _live(lib)
    yield lib
    assert _live(lib) == base


def _refused(lib, family, m):
    """Calls family's per-handle advancing call on member m."""
    if family == "vt":
        img = np.zeros((TRACKER["rows"], TRACKER["cols"]), np.uint8)
        return lib.vt_read_image(m.h, img.ctypes.data, img.strides[0], 0.0, 1)
    if family == "ve":
        return lib.ve_process_image(m.h, 0, None, None, 0.0)
    cfg = _loop_config()
    return lib.vp_loop_enable(m.h, C.byref(cfg))


@pytest.mark.parametrize("family, batch_call", [("vt", "vt_batch_read_image"), ("ve", "ve_batch_process_image"),
                                                ("vp", "vp_batch_loop_enable")])
def test_a_member_of_an_explicit_batch_is_driven_through_its_batch(lib, family, batch_call):
    from vins_mono_b200 import EstimatorBatch, PoseGraphBatch, TrackerBatch
    b = {"vt": lambda: TrackerBatch(2, **TRACKER), "ve": lambda: EstimatorBatch(2, **ESTIMATOR),
         "vp": lambda: PoseGraphBatch(2, max_keyframes=16)}[family]()
    m = b.members[1]
    assert _refused(lib, family, m) == INVALID
    assert batch_call in getattr(lib, family + "_last_error")(m.h).decode()
    assert getattr(lib, family + "_batch_last_error")(b.h) == b""
    b.close()


def test_estimator_member_failure_is_rolled_up_as_member_k(lib):
    from vins_mono_b200 import EstimatorBatch, VinsError
    seq = synth.Sequence(seed=2, duration=2.5)
    msgs = [synth.track_messages(seq, 14, max_feats=f) for f in (8, 120)]  # member 1 exceeds max_features = 40
    b = EstimatorBatch(2, max_features=40, tic=synth.TIC, ric=synth.RIC)
    feeders = []
    for m, ms in zip(b.members, msgs):
        m.set_seed(pipeline.gt_seed_rows(seq, [x[0] for x in ms]), seq.ba, seq.bg)
        feeders.append(pipeline.ImuFeeder(*seq.imu()))
    text = "feature capacity (max_features) exceeded"
    with pytest.raises(VinsError) as err:
        for i in range(14):
            for m, f, ms in zip(b.members, feeders, msgs):
                f.feed(m, ms[i][0])
            b.processImage([(ms[i][1], ms[i][2], ms[i][0]) for ms in msgs])
    assert err.value.status == CAPACITY
    assert lib.ve_batch_last_error(b.h).decode() == "member 1: " + text
    assert lib.ve_last_error(b.members[1].h).decode() == text
    b.close()


def _keyframes(g, n, loops):
    for k in range(n):
        li = [0.1, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0] if k in loops else None
        g.add_keyframe(0.1 * k, [0.3 * k, 0.0, 0.0], [1, 0, 0, 0], loops.get(k, -1), li)


def test_pose_graph_member_failure_stays_with_the_member(lib):
    from vins_mono_b200 import PoseGraphBatch
    b = PoseGraphBatch(2, max_keyframes=16, max_anchors=2)
    _keyframes(b[0], 10, {9: 1})                      # loops onto the range's first key frame: no free anchor
    _keyframes(b[1], 10, {6: 2, 7: 3, 8: 4, 9: 5})    # three free anchors, two allowed
    before = lib.vp_batch_last_error(b.h)
    status = b.optimize()
    assert list(status) == [1, CAPACITY]
    assert "3 free loop anchors in the optimised range, at most 2" in lib.vp_last_error(b[1].h).decode()
    assert lib.vp_last_error(b[0].h) == b""
    assert lib.vp_batch_last_error(b.h) == before
    b.sync()
    assert b[0].info()["optimizations"] == 1 and b[1].info()["optimizations"] == 0
    b.close()


def test_pose_graph_member_without_a_text_reads_its_batchs(lib):
    from vins_mono_b200 import PoseGraphBatch
    b = PoseGraphBatch(2, max_keyframes=16)
    bad = _loop_config(max_window=0)
    assert lib.vp_batch_loop_enable(b.h, C.byref(bad)) == INVALID
    text = lib.vp_batch_last_error(b.h)
    assert text == b"vp_loop_enable: invalid configuration"
    assert lib.vp_last_error(b[0].h) == text and lib.vp_last_error(b[1].h) == text
    img = np.zeros((64, 96), np.uint8)
    z = np.zeros(3)
    q = np.array([1.0, 0, 0, 0])
    assert lib.vp_attach_keyframe(b[1].h, 0, z.ctypes.data, q.ctypes.data, img.ctypes.data, 96, 0, None, None, None, None,
                                  None) == INVALID
    assert lib.vp_last_error(b[1].h) == b"vp_attach_keyframe: loop verification is not enabled"
    assert lib.vp_last_error(b[0].h) == text
    b.close()
