"""Measures the device 4-DoF pose-graph optimisation (vp_batch_optimize): device milliseconds from CUDA events around the
launch chain, wall milliseconds from before the host-to-device copy to the collected result, and launches per
optimisation, for n key frames x loop anchors x batch members.  Each timed optimisation is triggered by one new key frame
next to the last one, with the same loop, so every member re-optimises its whole range.  The card's name and power limit are
read in the same run.  As CPU context, the numpy restatement (oracle/pose_graph.py, not Ceres) is timed on the same
problem for the smaller sizes.

    python harness/pose_graph_bench.py --out DIR [--reps 20] [--warmup 3] [--quick]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from harness import pose_graph_synth as ps  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})", "unknown"


def run_case(n, anchors, S, reps, warmup, cpu_context):
    from vins_mono_b200 import PoseGraphBatch
    ev = ps.make_chain(n, anchors, seed=n + anchors)
    b = PoseGraphBatch(S, max_keyframes=n + reps + warmup + 8)
    for k in range(S):
        ps.feed(b[k], ev, False)
    last = ev[-1]
    dev, wall, launches, info = [], [], 0, None
    for r in range(warmup + reps):
        P = np.asarray(last[2]) + np.array([0.01 * (r + 1), 0, 0])
        for k in range(S):  # the last key frame's loop again, from a key frame next to it
            b[k].add_keyframe(last[1] + 0.1 * (r + 1), P, last[3], last[4], last[5])
        st = b.optimize()
        assert np.all(st == 1), st
        b.sync()
        d, w, launches = b.timing()
        if r >= warmup:
            dev.append(d)
            wall.append(w)
    info = b[0].info()
    rec = dict(n=info["last_n"], anchors=anchors, border=info["last_border"], S=S, reps=reps, device_ms=float(np.mean(dev)),
               device_ms_std=float(np.std(dev)), wall_ms=float(np.mean(wall)), launches=launches, iterations=info["iterations"])
    if cpu_context and S == 1:
        from oracle.pose_graph import OraclePoseGraph
        o = OraclePoseGraph()
        ps.feed(o, ev, False)
        t = time.perf_counter()
        o.optimize()
        rec["cpu_numpy_restatement_ms"] = (time.perf_counter() - t) * 1e3
    b.close()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--quick", action="store_true", help="n = 250 and 500 only")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    name, power = card()
    sizes = [250, 500] if a.quick else [250, 500, 1000, 2000]
    recs = []
    for n in sizes:
        for anchors in (10, 40, 88):
            for S in (1, 64):
                rec = run_case(n, anchors, S, a.reps, a.warmup, cpu_context=n <= 500)
                rec.update(card=name, power_limit=power)
                recs.append(rec)
                print(json.dumps(rec), flush=True)
    with open(os.path.join(a.out, "pose_graph_bench.jsonl"), "w") as f:
        for r in recs:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
