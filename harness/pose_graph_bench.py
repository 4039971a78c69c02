"""Measures the device 4-DoF pose-graph optimisation (vp_batch_optimize): device milliseconds from CUDA events around the
launch chain, wall milliseconds from before the host-to-device copy to the collected result, and launches per
optimisation, for n key frames x loop anchors x batch members.  Each timed optimisation is triggered by one new key frame
next to the last one, with the same loop, so every member re-optimises its whole range.  The card's name and power limit are
read in the same run.  As CPU context, the numpy restatement (oracle/pose_graph.py, not Ceres) is timed on the same
problem for the smaller sizes.

Anchor counts past 88 (352 border columns) take the multi-CTA border path; each such graph is created with max_anchors
set to fit.  In a run of its own, torch.profiler (CUDA activities) splits one optimisation of each size into phases by
kernel name: chain, border product (S = C - W^T W), factorisation, solves, and the rest (setup, linearise, update,
finish); on the one-CTA path the border factorisation runs inside pg_solve_kernel and is counted with the solves.  The
border product's FP64 rate is the staircase's real flop count (2 per multiply-add, over the rows of W each pair of
columns actually couples) over the product kernels' time.  Timing records go to DIR/pose_graph_bench.jsonl, and every
record of the anchor sweep, phases included, to DIR/pose_graph_border.jsonl.

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
    b = PoseGraphBatch(S, max_keyframes=n + reps + warmup + 8, max_anchors=max(anchors, 88))
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


PHASES = {  # kernel name -> phase of the split
    "pg_chain_kernel": "chain",
    "pg_border_kernel": "border_product",
    "pg_tile_kernel<false>": "border_product",
    "pg_panel_kernel": "factorisation",
    "pg_tile_kernel<true>": "factorisation",
    "pg_solve_kernel": "solves",
    "pg_solve_large_kernel": "solves",
}


def staircase_flops(ev):
    """Flops of S = C - W^T W and z = -g_b - W^T y for a make_chain run optimised over its whole range (key frame 0 is
    the earliest anchor): W has 16 ceil(n / 4) rows, column c starts at the first super-block holding a free key frame
    coupled to its anchor, and each pair of columns i <= j costs 2 flops per row from the later of the two starts."""
    kfs = [e for e in ev if e[0] == "kf"]
    n = len(kfs)
    loop = np.array([e[4] for e in kfs])
    anchors = sorted({int(l) for l in loop if l > 0})
    is_anchor = np.zeros(n, bool)
    is_anchor[anchors] = True
    chain = ~is_anchor
    chain[0] = False
    nsb = (n + 3) // 4
    start = []
    for a in anchors:
        ks = [k for k in range(max(1, a - 4), min(n, a + 5)) if chain[k]]
        ks += [k for k in np.nonzero(loop == a)[0] if chain[k]]
        if loop[a] >= 0 and chain[loop[a]]:
            ks.append(int(loop[a]))
        start += [min(ks) // 4 if ks else nsb] * 4
    start.append(int(np.nonzero(chain)[0][0]) // 4 if chain.any() else nsb)  # the right-hand side column
    s = np.array(start)
    rows = 16 * nsb - 16 * np.maximum.outer(s, s)
    iu = np.triu_indices(len(s))
    flops = 2.0 * rows[iu].sum() - 2.0 * rows[-1, -1]  # every pair i <= j except (D, D)
    return float(flops)


def profile_case(n, anchors, reps):
    """Per-phase device time of one optimisation (mean over reps) from torch.profiler's CUDA kernel records."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from vins_mono_b200 import PoseGraph
    ev = ps.make_chain(n, anchors, seed=n + anchors)
    g = PoseGraph(max_keyframes=n + reps + 8, max_anchors=max(anchors, 88))
    ps.feed(g, ev, False)
    last, added = ev[-1], []

    def step(r):
        added.append(("kf", last[1] + 0.1 * (r + 1), np.asarray(last[2]) + np.array([0.01 * (r + 1), 0, 0]), last[3], last[4], last[5]))
        g.add_keyframe(*added[-1][1:])
        assert g.optimize() == 1
        g.sync()

    step(0)  # warm-up: module load, shared-memory opt-in
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for r in range(1, reps + 1):
            step(r)
        torch.cuda.synchronize()
    us = {}
    for e in prof.key_averages():
        if "pg_" not in e.key or "kernel" not in e.key:
            continue
        phase = next((p for k, p in PHASES.items() if k in e.key), "other")
        us[phase] = us.get(phase, 0.0) + getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
    info = g.info()
    rec = dict(n=info["last_n"], anchors=anchors, border=info["last_border"], S=1, reps=reps, launches=g.timing()[1],
               phase_ms={p: us.get(p, 0.0) / reps / 1e3 for p in ("chain", "border_product", "factorisation", "solves", "other")})
    flops = staircase_flops(ev + added)  # the graph of the last profiled optimisation
    rec["border_product_gflop"] = flops * info["iterations"] / 1e9
    bp = rec["phase_ms"]["border_product"]
    rec["border_product_fp64_tflops"] = flops * info["iterations"] / (bp * 1e-3) / 1e12 if bp > 0 else None
    g.close()
    return rec


# Anchor counts of the sweep past the one-CTA limit, with their key-frame counts: make_chain spreads the anchors over
# the first half of the graph, so 1024 anchors need more than 2048 key frames.
BORDER_CASES = [(2000, 89), (2000, 128), (2000, 327), (2000, 512), (2056, 1024)]


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
    recs, border = [], []
    for n in sizes:
        for anchors in (10, 40, 88):
            for S in (1, 64):
                rec = run_case(n, anchors, S, a.reps, a.warmup, cpu_context=n <= 500)
                rec.update(card=name, power_limit=power)
                recs.append(rec)
                print(json.dumps(rec), flush=True)
    cases = [(500, 88), (500, 89)] if a.quick else [(2000, 10), (2000, 88)] + BORDER_CASES
    for n, anchors in cases:
        if anchors > 88:
            for S in (1, 8):
                rec = run_case(n, anchors, S, a.reps, a.warmup, cpu_context=False)
                rec.update(card=name, power_limit=power)
                recs.append(rec)
                border.append(rec)
                print(json.dumps(rec), flush=True)
    for n, anchors in cases:  # the profiled runs, after every timed one
        rec = profile_case(n, anchors, reps=5)
        rec.update(card=name, power_limit=power, kind="phases")
        border.append(rec)
        print(json.dumps(rec), flush=True)
    with open(os.path.join(a.out, "pose_graph_bench.jsonl"), "w") as f:
        for r in recs:
            f.write(json.dumps(r) + "\n")
    with open(os.path.join(a.out, "pose_graph_border.jsonl"), "w") as f:
        for r in border:
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
