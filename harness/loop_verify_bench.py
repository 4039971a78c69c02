"""Loop-verification bench: device time per stage of one key-frame attach (blur, FAST, BRIEF) and of one verification
launch chain (matching, PnP hypotheses, refit) at S = 1 and S = 64 pairs per chain, from the library's CUDA events, plus a
per-kernel split from torch.profiler (--profile).  Inputs: rendered revisit pairs of harness/loop_revisit.py, seen through
the EuRoC PINHOLE camera or (--camera) the reference's 3dm MEI or cla KANNALA_BRANDT camera; the FAST time includes the
corner lift.  Prints one JSON line per measurement; --out also writes them to a file.

    python -m harness.loop_verify_bench --reps 20 [--camera pinhole|mei|kb] [--profile] [--out profiles/loop_verify_h100.jsonl]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess

import numpy as np

from harness import loop_revisit, synth
from oracle import loop_verify as olv

INTR = [synth.FX, synth.FY, synth.CX, synth.CY, synth.K1, synth.K2, synth.P1, synth.P2]
CAMERA_FILES = {"mei": "3dm/3dm_config.yaml", "kb": "cla/cla_config.yaml"}


def _attach(g, old, cur):
    img, P, Q = old
    g.attach_keyframe(0, P, Q, img, np.zeros((0, 3)), np.zeros((0, 2)), np.zeros((0, 2)), np.zeros(0))
    img, P, Q, p3d, uv, norm, pid = cur
    return g.attach_keyframe(1, P, Q, img, p3d, uv, norm, pid)  # the corners of the attach loop_timing reports


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    ap.add_argument("--camera", choices=["pinhole", "mei", "kb"], default=None)  # named cameras also report their corner count
    a = ap.parse_args()
    from vins_mono_b200 import config
    from vins_mono_b200.pose_graph import PoseGraph, PoseGraphBatch, loop_config
    model, xi, tag = 0, 0.0, dict(camera=a.camera) if a.camera else {}
    if a.camera in (None, "pinhole"):
        seq = synth.Sequence(seed=0, duration=12.0)
        intr = INTR
    else:
        root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        kw = config.loop_kwargs(config.load(os.path.join(root, "tests", "golden", "config", CAMERA_FILES[a.camera])))
        model, xi, intr = kw["camera_model"], kw["xi"], kw["intrinsics"]
        seq = loop_revisit.CameraSequence(model, intr, xi, seed=0, duration=12.0, rows=kw["rows"], cols=kw["cols"])
    pts = loop_revisit.corner_landmarks(seq, np.arange(0.2, 12.0, 0.5))
    old, cur = loop_revisit.revisit_pair(seq, pts, 1.4, 8.9)  # a revisit of this sequence (2.3 m apart, accepted)
    cfg = loop_config(seq.rows, seq.cols, intr, synth.RIC, synth.TIC, olv.load_pattern(), 256, 16384)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    lines = []

    def emit(d):
        d.update(tag)
        d["gpu"] = gpu
        print(json.dumps(d), flush=True)
        lines.append(d)

    g = PoseGraph(max_keyframes=2)
    g.enable_loop(cfg, model, xi)
    att, ver = [], []
    for r in range(a.reps + 3):
        n_corners = _attach(g, old, cur)
        att.append(g.loop_timing()[:3].copy())
        res = g.find_connection(1, 0)
        ver.append(g.loop_timing()[3:].copy())
    att, ver = np.array(att[3:]), np.array(ver[3:])
    emit(dict(what="attach", S=1, blur_ms=float(att[:, 0].mean()), fast_ms=float(att[:, 1].mean()), brief_ms=float(att[:, 2].mean()),
              reps=a.reps, n_window=len(cur[4]), **({"n_corners": n_corners} if tag else {})))
    emit(dict(what="verify", S=1, match_ms=float(ver[:, 0].mean()), hyp_ms=float(ver[:, 1].mean()), refit_ms=float(ver[:, 2].mean()),
              reps=a.reps, n_matches=res["n_matches"], n_inliers=res["n_inliers"], accepted=res["accepted"]))
    S = 64
    b = PoseGraphBatch(S, max_keyframes=2)
    b.enable_loop(cfg, model, xi)
    for k in range(S):
        _attach(b[k], old, cur)
    ver = []
    for r in range(a.reps + 3):
        b.find_connection([1] * S, [0] * S)
        ver.append(b.loop_timing()[3:].copy())
    ver = np.array(ver[3:])
    emit(dict(what="verify", S=S, match_ms=float(ver[:, 0].mean()), hyp_ms=float(ver[:, 1].mean()), refit_ms=float(ver[:, 2].mean()),
              reps=a.reps))
    if a.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.init()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                _attach(g, old, cur)
                g.find_connection(1, 0)
                b.find_connection([1] * S, [0] * S)
        for ev in prof.key_averages():
            if ev.key.startswith("_ZN2vb") or "lv_" in ev.key:
                name = next((k for k in ev.key.split("_") if k.endswith("kernel")), ev.key)
                for part in ev.key.split("lv_")[1:]:
                    name = "lv_" + part.split("E")[0].split("Ev")[0]
                emit(dict(what="kernel", name=name, calls=ev.count, device_ms_total=ev.device_time_total / 1000.0,
                          device_ms_avg=ev.device_time_total / 1000.0 / max(ev.count, 1)))
    if a.out:
        with open(a.out, "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
