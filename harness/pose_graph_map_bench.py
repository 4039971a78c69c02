"""Measures pose-graph reuse on the device: vp_save / vp_load wall milliseconds for a map of 2000 key frames x about 500
corners (loop verification enabled, so the points go through the slots), and the device milliseconds (CUDA events) and
launches of one optimisation of the same 200-key-frame new session with 50 loops against maps of 0 (no map: the loops
land inside the session), 500 and 2000 key frames.  Each timed optimisation is triggered by one more key frame with the
session's last loop, so every repetition solves the same range.  The card's name and power limit are read in the same
run.  Records go to DIR/pose_graph_map_h100.jsonl.

    python harness/pose_graph_map_bench.py --out DIR [--reps 10] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import oracle.pose_graph as opg  # noqa: E402
import pose_graph_map_twin as tw  # noqa: E402
from harness.pose_graph_bench import card  # noqa: E402


def map_rows(n, n_pts, rng):
    rows = []
    for i in range(n):
        q = opg.R_to_quat(opg.ypr2R([0.1 * i, 1.0, -1.0]))
        P = [0.05 * i, 0.3 * np.sin(0.01 * i), 0.0]
        loop = i % 97 == 50
        rows.append(dict(index=i, stamp=0.1 * i, vio_T=P, pg_T=P, vio_Q=q, pg_Q=q, loop_index=i - 40 if loop else -1,
                         loop_info=[0.1, 0, 0, 1, 0, 0, 0, 0.5] if loop else [0] * 8,
                         kp=rng.uniform(0, 700, (n_pts, 2)).astype(np.float32), kpn=rng.uniform(-1, 1, (n_pts, 2)).astype(np.float32),
                         desc=rng.integers(0, 2**63, (n_pts, 4), dtype=np.int64).astype(np.uint64)))
    return rows


def session(n_map, n=200, n_loops=50):
    """The new session: n key frames along the map's path in another VIO frame; loops onto the map (or, with no map,
    onto the session's own first half)."""
    ev = []
    srcs = set(np.linspace(n // 4 if n_map else n // 2 + 1, n - 1, n_loops).astype(int).tolist())
    for k in range(n):
        i = 7 + 2 * k
        q = opg.R_to_quat(opg.ypr2R([0.1 * i + 20.0, 1.0, -1.0]))
        P = opg.ypr2R([20.0, 0, 0]) @ np.array([0.05 * i + 0.3, 0.2, 0.0]) + [1.0, 2.0, 0.0]
        l, li = -1, None
        if k in srcs:
            l = (i * 7) % n_map if n_map else k - n // 2 - 1
            li = np.r_[0.02, 0.01, 0.0, 1, 0, 0, 0, 0.3]
        ev.append((1000 + 0.1 * k, P, q, l, li))
    return ev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    from vins_mono_b200 import PoseGraph
    from vins_mono_b200.pose_graph import loop_config
    os.makedirs(a.out, exist_ok=True)
    name, power = card()
    recs = []
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as d:
        pre = tw.scratch_prefix(d, "map2000")
        tw.write_map(pre, map_rows(2000, 500, rng))
        cfg = loop_config(480, 752, [460, 460, 376, 240, 0, 0, 0, 0], np.eye(3), np.zeros(3), np.zeros((256, 4), np.int32), 64, 512)
        g = PoseGraph(max_keyframes=2400)
        g.enable_loop(cfg)
        t0 = time.perf_counter()
        n = g.load(pre)
        t_load = (time.perf_counter() - t0) * 1e3
        out = tw.scratch_prefix(d, "saved")
        t0 = time.perf_counter()
        g.save(out)
        t_save = (time.perf_counter() - t0) * 1e3
        same = all(open(pre + f, "rb").read() == open(out + f, "rb").read() for f in ("0_keypoints.txt", "0_briefdes.dat", "1999_briefdes.dat"))
        recs.append(dict(what="save_load", keyframes=n, corners=500, load_ms=t_load, save_ms=t_save, points_identical=same))
        g.close()
        for n_map in (0, 500, 2000):
            g = PoseGraph(max_keyframes=2600)
            if n_map:
                p = tw.scratch_prefix(d, f"m{n_map}")
                tw.write_map(p, [dict(r, kp=[], kpn=[], desc=[]) for r in map_rows(n_map, 0, rng)])
                g.load(p)
            ev = session(n_map)
            for stamp, P, q, l, li in ev:
                g.add_keyframe(stamp, P, q, l, li)
            last = [e for e in ev if e[3] >= 0][-1]
            dev, launches = [], 0
            for r in range(a.warmup + a.reps):
                if r:
                    g.add_keyframe(last[0] + 0.01 * r, last[1], last[2], last[3], last[4])
                assert g.optimize() == 1
                g.sync()
                ms, launches = g.timing()
                if r >= a.warmup:
                    dev.append(ms)
            info = g.info()
            recs.append(dict(what="optimize", map_keyframes=n_map, session_keyframes=200, loops=50, range_keyframes=info["last_n"],
                             border=info["last_border"], iterations=info["iterations"], device_ms_median=float(np.median(dev)),
                             device_ms_min=float(np.min(dev)), launches=launches, reps=a.reps))
            g.close()
    opt = {r["map_keyframes"]: r["device_ms_median"] for r in recs if r["what"] == "optimize"}
    recs.append(dict(what="bound", ratio_2000_over_500=opt[2000] / opt[500], within_20_percent=opt[2000] <= 1.2 * opt[500]))
    with open(os.path.join(a.out, "pose_graph_map_h100.jsonl"), "w") as f:
        for r in recs:
            r.update(gpu=name, power_limit=power)
            f.write(json.dumps(r) + "\n")
            print(json.dumps(r))


if __name__ == "__main__":
    main()
