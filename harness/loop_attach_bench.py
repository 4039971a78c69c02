"""Batched key-frame attach bench: 64 key frames on one 64-member pose-graph batch, attached by one
vp_batch_attach_keyframes call against 64 vp_attach_keyframe calls, as a batch replay attaches one key frame per member
and step.  Per variant: host ms of the whole call(s) (each call ends in a stream synchronise, so this includes the copies
and the launch gaps) and device ms of the blur, FAST (with compaction and corner lift) and BRIEF stages from the
library's CUDA events; --profile adds a per-kernel split from torch.profiler in a run of its own.  The variants alternate
within each repetition after a warm-up of every shape.  Inputs: 16 rendered EuRoC-sized frames of harness/synth.py with
the window points of a revisit of harness/loop_revisit.py, used in turn.  Every line carries the card and its power
limit.

    python -m harness.loop_attach_bench --reps 20 [--profile] [--out profiles/loop_attach_h100.jsonl]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import time

import numpy as np

from harness import loop_revisit, synth
from oracle import loop_verify as olv

INTR = [synth.FX, synth.FY, synth.CX, synth.CY, synth.K1, synth.K2, synth.P1, synth.P2]
S = 64


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from vins_mono_b200.pose_graph import PoseGraphBatch, loop_config
    seq = synth.Sequence(seed=0, duration=12.0)
    pts = loop_revisit.corner_landmarks(seq, np.arange(0.2, 12.0, 0.5))
    _, (img, P, Q, p3d, uv, norm, pid) = loop_revisit.revisit_pair(seq, pts, 1.4, 8.9)
    frames = [seq.render(t) for t in np.linspace(0.5, 11.5, 16)]
    dev_frames = [torch.from_numpy(f).cuda() for f in frames]
    cfg = loop_config(seq.rows, seq.cols, INTR, synth.RIC, synth.TIC, olv.load_pattern(), 256, 16384)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip()
    lines = []

    def emit(d):
        d["gpu"] = gpu
        print(json.dumps(d), flush=True)
        lines.append(d)

    b = PoseGraphBatch(S, max_keyframes=4)
    b.enable_loop(cfg)
    n_corners = [len(olv.fast(f)[0]) for f in frames]

    def jobs(device, slot):
        src = dev_frames if device else frames
        return [(k, slot, P, Q, src[k % len(src)], p3d, uv, norm, pid) for k in range(S)]

    host_jobs, dev_jobs = jobs(False, 0), jobs(True, 1)

    def batched(js):
        t0 = time.perf_counter()
        nc, st = b.attach_keyframes(js)
        wall = (time.perf_counter() - t0) * 1e3
        assert (st == 0).all()
        return wall, float(b.loop_timing()[:3].sum()), nc

    def single():
        wall, dev, nc = 0.0, 0.0, []
        for k in range(S):
            t0 = time.perf_counter()
            nc.append(b[k].attach_keyframe(2, P, Q, frames[k % len(frames)], p3d, uv, norm, pid))
            wall += (time.perf_counter() - t0) * 1e3
            dev += float(b[k].loop_timing()[:3].sum())
        return wall, dev, np.array(nc)

    runs = {"batched_host_images": lambda: batched(host_jobs), "batched_device_images": lambda: batched(dev_jobs), "single_calls": single}
    for _ in range(a.warmup):
        for f in runs.values():
            f()
    res = {k: [] for k in runs}
    for _ in range(a.reps):
        for k, f in runs.items():
            wall, dev, nc = f()
            assert list(nc) == [n_corners[j % len(frames)] for j in range(S)]
            res[k].append((wall, dev))
    for k, v in res.items():
        v = np.array(v)
        emit(dict(what="attach", variant=k, key_frames=S, members=S, calls=1 if k.startswith("batched") else S, reps=a.reps,
                  host_ms_median=float(np.median(v[:, 0])), host_ms_min=float(v[:, 0].min()), host_ms_max=float(v[:, 0].max()),
                  device_ms_median=float(np.median(v[:, 1])), device_ms_min=float(v[:, 1].min()), device_ms_max=float(v[:, 1].max()),
                  rows=seq.rows, cols=seq.cols, n_window=len(uv), corners_min=min(n_corners), corners_max=max(n_corners)))
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        for k, f in runs.items():
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.reps):
                    f()
            for ev in prof.key_averages():
                if "lv_" not in ev.key:
                    continue
                name = "lv_" + ev.key.split("lv_", 1)[1].split("(")[0]
                emit(dict(what="kernel", variant=k, name=name, calls=ev.count, reps=a.reps,
                          device_ms_per_rep=ev.device_time_total / 1000.0 / a.reps,
                          device_ms_avg=ev.device_time_total / 1000.0 / max(ev.count, 1)))
    if a.out:
        with open(a.out, "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
