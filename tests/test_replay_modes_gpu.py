"""The two modes of the native replay driver (include/vinsb200/replay.h) against each other.  A session of stand-alone handle
pairs (vr_open) and a session of batch members (vr_open_batch) run the same sequences through the same node loops, so every
sequence gets the same feature messages, IMU samples and relocalisation messages in both, and its trajectory is bit-identical."""
import numpy as np
import pytest

from harness import synth, pipeline

pytestmark = pytest.mark.gpu


def _sequence(seed, n_pub, n_images=None):
    """(synth.Sequence, seed rows, ReplaySession sequence dict) with images for n_pub published frames, or only the first
    n_images of them."""
    n_img = 2 * (n_pub + 1) + 2
    seq = synth.Sequence(seed=seed, duration=n_img / 20.0 + 0.5)
    ts, imgs = pipeline.cached_images(seq, n_img)
    t_imu, acc, gyr = seq.imu()
    keep = n_images or n_img
    return seq, pipeline.gt_seed_rows(seq, ts), dict(images=np.ascontiguousarray(imgs[:keep]), stamps=np.asarray(ts[:keep]),
                                                     imu_t=t_imu, acc=acc, gyr=gyr)


def _handles(batch, n):
    """(trackers, estimators, estimator mirrors) for a session of n sequences: two batches, or n stand-alone pairs."""
    from vins_mono_b200 import FeatureTracker, Estimator, TrackerBatch, EstimatorBatch
    cfg = synth.tracker_config_dict()
    if batch:
        tb, eb = TrackerBatch(n, **cfg), EstimatorBatch(n, tic=synth.TIC, ric=synth.RIC)
        return tb, eb, eb.members
    est = [Estimator(tic=synth.TIC, ric=synth.RIC) for _ in range(n)]
    return [FeatureTracker(**cfg) for _ in range(n)], est, est


def _close(trackers, estimators):
    for h in (trackers + estimators if isinstance(trackers, list) else [trackers, estimators]):
        h.close()


def test_per_sequence_and_batch_sessions_agree():
    """Three distinct sequences, the last one short of images so that it runs out while the others go on, each session
    advanced in two calls (cursors and IMU positions carry over)."""
    from vins_mono_b200 import ReplaySession
    n_pub, split = 18, 7
    inputs = [_sequence(3, n_pub), _sequence(4, n_pub), _sequence(5, n_pub, n_images=30)]
    runs = {}
    for batch in (False, True):
        trackers, estimators, members = _handles(batch, len(inputs))
        for e, (seq, seed, _) in zip(members, inputs):
            e.set_seed(seed, seq.ba, seq.bg)
        ses = ReplaySession(trackers, estimators, [sq for _, _, sq in inputs])
        done = [ses.advance(split), ses.advance(n_pub - split)]
        runs[batch] = dict(done=done, stats=[ses.stats(k) for k in range(len(inputs))],
                           traj=[ses.trajectory(k) for k in range(len(inputs))])
        ses.close()
        _close(trackers, estimators)
    solo, bat = runs[False], runs[True]
    assert solo["done"] == bat["done"] and sum(solo["done"]) == sum(st["frames"] for st in solo["stats"])
    for k in range(len(inputs)):
        assert solo["stats"][k]["frames"] == bat["stats"][k]["frames"], k
        (ts, ps), (tb, pb) = solo["traj"][k], bat["traj"][k]
        assert len(ts) > 0 and np.array_equal(ts, tb) and np.array_equal(ps, pb), k
    assert [st["frames"] for st in solo["stats"]][:2] == [n_pub, n_pub] and solo["stats"][2]["frames"] < n_pub  # the short one ran out
    # launches: each stand-alone pair counts its own; a batch's launches are not attributable to a member and count on sequence 0
    assert all(st["launches"] > 0 for st in solo["stats"])
    assert bat["stats"][0]["launches"] > 0 and all(st["launches"] == 0 for st in bat["stats"][1:])


def test_batch_session_delivers_queued_relocalisation_messages():
    """The scenario of test_replay_gpu.py's relocalisation test with the messages queued on sequence 1 of a batch of two: the
    message reaches setReloFrame at the same published frame as in a per-sequence session, and only on sequence 1."""
    from vins_mono_b200 import FeatureTracker, Estimator, ReplaySession
    n_pub = 22
    seq, seed, sq = _sequence(3, n_pub)
    trk = FeatureTracker(**synth.tracker_config_dict())
    msgs = list(pipeline.feature_messages(trk, sq["stamps"], sq["images"]))[:n_pub]
    trk.close()
    # a frame a few places back in the window when message 19 arrives (a Python-driven pass over messages 0 .. 18)
    probe = Estimator(tic=synth.TIC, ric=synth.RIC)
    probe.set_seed(seed, seq.ba, seq.bg)
    feeder = pipeline.ImuFeeder(sq["imu_t"], sq["acc"], sq["gyr"])
    for stamp, ids, d in msgs[1:19]:  # the node drops the first feature message
        feeder.feed(probe, stamp)
        probe.processImage(ids, d, stamp)
    window = probe.headers()[:-1]
    probe.close()
    j = next(k for k in range(16, 8, -1) if np.any(window == msgs[k][0]))
    stamp_j, ids_j, d_j = msgs[j]
    mp = np.c_[d_j[:, 0] + 0.01, d_j[:, 1] - 0.005, np.asarray(ids_j, float)]
    mp = mp[np.argsort(mp[:, 2])]

    def run(batch, seq_index):
        n = seq_index + 1
        trackers, estimators, members = _handles(batch, n)
        for e in members:
            e.set_seed(seed, seq.ba, seq.bg)
        ses = ReplaySession(trackers, estimators, [sq] * n)
        ses.queue_relo(seq_index, msgs[18][0] + 1e-4, 0.0, 1, mp[:3], np.zeros(3), np.eye(3))  # superseded in the same drain
        ses.queue_relo(seq_index, msgs[18][0] + 2e-4, stamp_j, 5, mp, np.array([0.1, 0.2, 0.3]), np.eye(3))
        e = members[seq_index]
        assert ses.advance(19) == 19 * n
        assert e.relo()["solves"] == 0 and not e.relo()["pending"]
        assert ses.advance(1) == n
        r = e.relo()
        assert r["solves"] == 1 and r["factors"] >= 10 and not r["pending"]
        assert ses.advance(n_pub - 20) == (n_pub - 20) * n and e.relo()["solves"] == 1
        out = dict(traj=[ses.trajectory(k) for k in range(n)], relo=[m.relo() for m in members])
        ses.close()
        _close(trackers, estimators)
        return out

    solo, bat = run(False, 0), run(True, 1)
    (ts, ps), (tb, pb) = solo["traj"][0], bat["traj"][1]
    assert len(ts) > 0 and np.array_equal(ts, tb) and np.array_equal(ps, pb)
    assert bat["relo"][0]["solves"] == 0 and not bat["relo"][0]["pending"]     # sequence 0 saw no relocalisation
