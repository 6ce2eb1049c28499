#!/usr/bin/env python
"""Measurement aid: K2 alone against K2 beside the next run's K1, inputs resident (CUDA events inside the engine).
    python tools/k2_overlap.py [workload] [rounds]
"alone": every run is synchronised before the next is enqueued, so K2 runs after its own K1 with the GPU otherwise idle.
"overlapped": runs are enqueued back to back, so K1 of run i+1 shares the SMs with K2 of run i; durations and the period
(K1 start to next K1 start) come from Engine.timeline().  Prints one JSON line with the card and its power limit."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "rtlsdr-airband_b200", "py"))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

import bench  # noqa: E402
from airband_b200 import lib  # noqa: E402


def card() -> str:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as exc:  # the numbers still stand; say the card is unknown
        return f"unknown ({exc})"


def main():
    wname = sys.argv[1] if len(sys.argv) > 1 else "cfg2"
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 40
    cfg, _ = bench.make_workload(wname)
    nb = 4
    raws = bench.synth_streams(cfg, nb)
    eng = lib.Engine(cfg, max_batches_per_run=nb)
    for d in range(len(cfg.devices)):
        eng.resident_load(d, raws[d])
    for _ in range(10):
        eng.run_resident(nb)
    eng.sync()
    k1a, k2a = [], []
    for _ in range(rounds * 2):
        eng.run_resident(nb)
        t = eng.last_run_times()
        eng.sync()
        k1a.append(t[0])
        k2a.append(t[1])
    k1p, k2p, per = [], [], []
    t0 = time.perf_counter()
    for _ in range(rounds):
        for _ in range(8):
            eng.run_resident(nb)
        tl = eng.timeline(8)
        # runs 1..6: a K1 before and after each, so every K2 counted has a K1 beside it
        for r in range(1, 7):
            k1p.append(tl[r][1] - tl[r][0])
            k2p.append(tl[r][3] - tl[r][2])
            per.append(tl[r + 1][0] - tl[r][0])
    eng.sync()
    wall = (time.perf_counter() - t0) / (rounds * 8) * 1e3
    eng.close()
    res = {
        "workload": wname, "card": card(),
        "alone_k1_ms": float(np.median(k1a)), "alone_k2_ms": float(np.median(k2a)),
        "overlapped_k1_ms": float(np.median(k1p)), "overlapped_k2_ms": float(np.median(k2p)),
        "period_ms": float(np.median(per)), "wall_ms_per_run": wall,
    }
    res["k2_overlapped_over_alone"] = res["overlapped_k2_ms"] / res["alone_k2_ms"]
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
