"""GPU tests of the batched back end (ve_batch_*, BASELINE configs[2]): every member of a batch must produce what a
stand-alone estimator produces on the same inputs (the batch only changes which grid dimension a sequence lives on), and
both must agree with the CPU oracle."""
import numpy as np
import pytest

import orc
from harness import synth, pipeline
from test_backend_gpu import TOL, quat_angle

pytestmark = pytest.mark.gpu


def _feed(est, feeder, stamp):
    feeder.feed(est, stamp)


def _worst(sa, sb):
    return dict(p=np.abs(sa[:, 0:3] - sb[:, 0:3]).max(), q=quat_angle(sa[:, 3:7], sb[:, 3:7]).max(),
                v=np.abs(sa[:, 7:10] - sb[:, 7:10]).max(), ba=np.abs(sa[:, 10:13] - sb[:, 10:13]).max(),
                bg=np.abs(sa[:, 13:16] - sb[:, 13:16]).max())


def test_batch_members_match_standalone_and_oracle():
    from vins_mono_b200 import Estimator, EstimatorBatch
    n, n_pub = 5, 20
    seqs = [synth.Sequence(seed=10 + k, duration=3.5) for k in range(n)]
    msgs = [synth.track_messages(s, n_pub, max_feats=70 + 15 * k) for k, s in enumerate(seqs)]
    batch = EstimatorBatch(n, tic=synth.TIC, ric=synth.RIC)
    solo = [Estimator(tic=synth.TIC, ric=synth.RIC) for _ in range(n)]
    cpu = [orc.OracleEstimator(orc.be_config()) for _ in range(n)]
    feeders = []
    for k in range(n):
        seeds = pipeline.gt_seed_rows(seqs[k], [m[0] for m in msgs[k]])
        t_imu, acc, gyr = seqs[k].imu()
        for est in (batch.members[k], solo[k], cpu[k]):
            est.set_seed(seeds, seqs[k].ba, seqs[k].bg)
        feeders.append([pipeline.ImuFeeder(t_imu, acc, gyr) for _ in range(3)])
    # member 3 starts two frames late, member 1 skips nothing but idles on frame 7 of the schedule (its message is delivered
    # one step later): the batch must cope with members in different phases
    cursor = [0] * n
    worst_cpu = dict(p=0, q=0, v=0, ba=0, bg=0)
    n_nl = 0
    for step in range(n_pub + 3):
        frame = []
        for k in range(n):
            idle = (k == 3 and step < 2) or (k == 1 and step == 7) or cursor[k] >= n_pub
            if idle:
                frame.append(None)
                continue
            stamp, ids, d = msgs[k][cursor[k]]
            cursor[k] += 1
            for est, f in zip((batch.members[k], solo[k], cpu[k]), feeders[k]):
                f.feed(est, stamp)
            solo[k].processImage(ids, d, stamp)
            cpu[k].processImage(ids, d, stamp)
            frame.append((ids, d, stamp))
        status = batch.processImage(frame)
        assert np.all(status == 0)
        if step == 15:
            t = batch.timing()
            assert t["launches"] > 0 and t["solve_ms"] > 0 and t["marg_ms"] > 0, t
        for k in range(n):
            if frame[k] is None:
                continue
            ia, ib, ic = batch.members[k].info(), solo[k].info(), cpu[k].info()
            for key in ("solver_flag", "frame_count", "marginalization_flag", "landmarks", "visual", "n_reboots", "n_solves"):
                assert ia[key] == ib[key] == ic[key], (step, k, key, ia, ib, ic)
            if ia["solver_flag"] != 1:
                continue
            n_nl += 1
            sa, sb, sc = batch.members[k].states()[0], solo[k].states()[0], cpu[k].states()[0]
            assert np.array_equal(sa, sb), (step, k)   # same code, fixed summation orders: bit-identical to the stand-alone handle
            for key, val in _worst(sa, sc).items():
                worst_cpu[key] = max(worst_cpu[key], val)
    assert n_nl >= n * (n_pub - 12)
    print("batch vs oracle", worst_cpu)
    for key in worst_cpu:
        assert worst_cpu[key] <= TOL[key], (key, worst_cpu)
    batch.close()


def test_batch_of_64_sequences_runs():
    """configs[2] shape: 64 members, one launch chain per frame; every member must equal its stand-alone twin's trajectory
    (members 0, 21, 42, 63 are checked, the rest must at least reach the same solver state)."""
    from vins_mono_b200 import Estimator, EstimatorBatch
    n, n_pub = 64, 14
    base = [synth.Sequence(seed=30 + k, duration=2.6) for k in range(4)]
    base_msgs = [synth.track_messages(s, n_pub, max_feats=100) for s in base]
    batch = EstimatorBatch(n, tic=synth.TIC, ric=synth.RIC)
    check = [0, 21, 42, 63]
    solo = {k: Estimator(tic=synth.TIC, ric=synth.RIC) for k in check}
    feeders, sfeed = [], {}
    for k in range(n):
        s, m = base[k % 4], base_msgs[k % 4]
        seeds = pipeline.gt_seed_rows(s, [x[0] for x in m])
        batch.members[k].set_seed(seeds, s.ba, s.bg)
        t_imu, acc, gyr = s.imu()
        feeders.append(pipeline.ImuFeeder(t_imu, acc, gyr))
        if k in solo:
            solo[k].set_seed(seeds, s.ba, s.bg)
            sfeed[k] = pipeline.ImuFeeder(t_imu, acc, gyr)
    launches = []
    for i in range(n_pub):
        frame = []
        for k in range(n):
            stamp, ids, d = base_msgs[k % 4][i]
            feeders[k].feed(batch.members[k], stamp)
            frame.append((ids, d, stamp))
            if k in solo:
                sfeed[k].feed(solo[k], stamp)
                solo[k].processImage(ids, d, stamp)
        assert np.all(batch.processImage(frame) == 0)
        launches.append(batch.launch_count())
    for k in range(n):
        info = batch.members[k].info()
        assert info["solver_flag"] == 1 and info["n_solves"] == batch.members[k % 4].info()["n_solves"] >= 3
    for k in check:   # the batch only changes which grid dimension a sequence lives on
        assert np.array_equal(batch.members[k].states()[0], solo[k].states()[0]), k
    # one launch chain per frame regardless of the batch size: zero + linearize + 8 x 3 + finish + 3 marginalisation + jobs
    assert max(launches) <= batch.groups() * (1 + 8 * 3 + 1 + 4 + 1), launches   # per launch group
    batch.close()


def test_member_keeps_its_batch_alive_and_fails_cleanly_after_close(monkeypatch):
    import gc
    from vins_mono_b200 import EstimatorBatch, VinsError, load_library
    m = EstimatorBatch(2, tic=synth.TIC, ric=synth.RIC).members[0]  # the batch itself is never bound to a name
    gc.collect()
    m.processIMU(0.005, [0, 0, 9.81], [0, 0, 0])
    states, _ = m.states()
    assert states.shape == (11, 16) and m.info()["frame_count"] == 0
    b = EstimatorBatch(2, tic=synth.TIC, ric=synth.RIC)
    m = b.members[1]
    b.close()
    monkeypatch.setattr(load_library(), "ve_get_states", lambda *a: pytest.fail("a closed member reached the library"))
    with pytest.raises(VinsError):
        m.states()
