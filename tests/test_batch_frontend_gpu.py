"""GPU tests of the batched front end (vt_batch_*) and of the batched replay driver (vr_open_batch): every member of a batch
must be bit-identical to a stand-alone tracker fed the same frames (the batch only changes which grid dimension a sequence
lives on), including members that restart or idle while the others keep going."""
import numpy as np
import pytest

from harness import synth, pipeline

pytestmark = pytest.mark.gpu

ROWS, COLS = 240, 376


def _frames(seed, n, dx, dy):
    tex = synth.value_noise_image(ROWS + 80, COLS + 120, seed=seed)
    out = []
    for i in range(n):
        ox, oy = 40 + int(round(dx * i)), 30 + int(round(dy * i))
        out.append(np.ascontiguousarray(tex[oy:oy + ROWS, ox:ox + COLS]))
    return out


def _same(a, b):
    return all(np.array_equal(a[k], b[k]) for k in ("ids", "track_cnt", "cur_pts", "un_pts", "velocity"))


def test_tracker_batch_members_bit_identical_to_standalone():
    from vins_mono_b200 import FeatureTracker, TrackerBatch
    n, n_img = 5, 24
    cfg = synth.tracker_config_dict(rows=ROWS, cols=COLS, max_cnt=80, min_dist=20)
    frames = [_frames(40 + k, n_img, 1.5 + 0.4 * k, 0.7 - 0.3 * k) for k in range(n)]
    batch = TrackerBatch(n, **cfg)
    solo = [FeatureTracker(**cfg) for _ in range(n)]
    cursor = [0] * n
    pubs = 0
    for step in range(n_img + 4):
        imgs, stamps = [None] * n, np.zeros(n)
        expect = [None] * n
        for k in range(n):
            # member 2 idles for two steps, member 4 sees a time jump (restart rule) in the middle
            if (k == 2 and step in (5, 6)) or cursor[k] >= n_img:
                continue
            i = cursor[k]
            cursor[k] += 1
            t = 0.05 * i + (5.0 if (k == 4 and i >= 12) else 0.0)
            imgs[k], stamps[k] = frames[k][i], t
            expect[k] = solo[k].node_image(frames[k][i], t)
        res, rst = batch.node_image(imgs, stamps)
        for k in range(n):
            if imgs[k] is None:
                continue
            assert (int(res[k]), int(rst[k])) == expect[k], (step, k, res, rst, expect[k])
            if res[k] > 0:
                assert _same(batch.members[k].result(), solo[k].result()), (step, k)
            if res[k] == 2:
                pubs += 1
                assert batch.members[k].feature_message() == solo[k].feature_message()
    assert pubs >= n * 6
    ms, launches = batch.timing()
    assert launches <= 6 + 7          # one launch per stage for the whole batch: 2 clahe + 3 pyrdown + lk, then 7 of the detector
    batch.close()
    for t in solo:
        t.close()


def test_tracker_batch_device_frames_and_read_image():
    import torch
    from vins_mono_b200 import FeatureTracker, TrackerBatch
    n = 3
    cfg = synth.tracker_config_dict(rows=ROWS, cols=COLS, max_cnt=60, min_dist=20)
    frames = [_frames(60 + k, 6, 2.0, 1.0) for k in range(n)]
    dev = [torch.from_numpy(np.stack(f)).cuda() for f in frames]
    batch = TrackerBatch(n, **cfg)
    solo = [FeatureTracker(**cfg) for _ in range(n)]
    for i in range(6):
        pub = [(i + k) % 2 == 0 for k in range(n)]
        batch.readImage([d[i].data_ptr() for d in dev], [0.05 * i] * n, pub)
        for k in range(n):
            solo[k].readImage(frames[k][i], 0.05 * i, pub[k])
            assert _same(batch.members[k].result(), solo[k].result()), (i, k)
    batch.close()


def test_replay_batch_matches_python_loop():
    from vins_mono_b200 import FeatureTracker, Estimator, TrackerBatch, EstimatorBatch, ReplaySession
    n_pub = 18
    n_img = 2 * (n_pub + 1) + 2
    seq = synth.Sequence(seed=3, duration=n_img / 20.0 + 0.5)
    ts, imgs = pipeline.cached_images(seq, n_img)
    imgs = np.ascontiguousarray(imgs)
    t_imu, acc, gyr = seq.imu()
    seed = pipeline.gt_seed_rows(seq, ts)
    trk, est = FeatureTracker(**synth.tracker_config_dict()), Estimator(tic=synth.TIC, ric=synth.RIC)
    est.set_seed(seed, seq.ba, seq.bg)
    ref = pipeline.run_vio(seq, trk, est, n_img, messages=list(pipeline.feature_messages(trk, ts, imgs))[:n_pub])
    ref_states, _ = est.states()
    trk.close()
    est.close()

    n = 4
    tb, eb = TrackerBatch(n, **synth.tracker_config_dict()), EstimatorBatch(n, tic=synth.TIC, ric=synth.RIC)
    for e in eb.members:
        e.set_seed(seed, seq.ba, seq.bg)
    ses = ReplaySession(tb, eb, [dict(images=imgs, stamps=ts, imu_t=t_imu, acc=acc, gyr=gyr) for _ in range(n)])
    assert ses.advance(7) == n * 7
    assert ses.advance(n_pub - 7) == n * (n_pub - 7)
    total_launches = sum(ses.stats(k)["launches"] for k in range(n))
    for k in range(n):
        st = ses.stats(k)
        assert st["frames"] == n_pub and st["h2d"] > n_pub * 2 * 752 * 480 * 0.9
        tt, pp = ses.trajectory(k)
        assert len(tt) == len(ref["t"]) and np.array_equal(tt, np.asarray(ref["t"]))
        assert np.array_equal(pp, np.asarray(ref["P"]))   # bit-reproducible: batch member == stand-alone handle
        assert np.array_equal(eb.members[k].states()[0], ref_states)
    # one launch chain per step for the whole batch: far fewer launches than sequences x per-sequence launches
    assert 0 < total_launches < n_pub * (2 * 13 + 32)
    ses.close()
    tb.close()
    eb.close()


def test_member_keeps_its_batch_alive_and_fails_cleanly_after_close(monkeypatch):
    import gc
    from vins_mono_b200 import TrackerBatch, VinsError, load_library
    cfg = synth.tracker_config_dict(rows=ROWS, cols=COLS, max_cnt=60, min_dist=20)
    m = TrackerBatch(2, **cfg).members[0]  # the batch itself is never bound to a name
    gc.collect()
    assert m.result()["ids"].size == 0 and m.traffic() == (0.0, 0.0)
    b = TrackerBatch(2, **cfg)
    m = b.members[1]
    b.close()
    monkeypatch.setattr(load_library(), "vt_count", lambda *a: pytest.fail("a closed member reached the library"))
    with pytest.raises(VinsError):
        m.result()
