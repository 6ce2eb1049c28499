#!/usr/bin/env python
"""Measurement aid: K1 / K2 durations (CUDA events inside the engine) of one workload for a list of environment-variable
variants of the tensor-core K1 (shared-memory cap, stages in the ring, digits), inputs resident.
    python tools/k1_variants.py cfg2 "" "ABG_K1_TC_STAGES=4" "ABG_K1_TC_CAP_KB=227" ..."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "rtlsdr-airband_b200", "py"))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

import bench  # noqa: E402
from airband_b200 import lib  # noqa: E402


def main():
    wname = sys.argv[1]
    variants = sys.argv[2:] or [""]
    cfg, desc = bench.make_workload(wname)
    nb = 4
    raws = bench.synth_streams(cfg, nb)
    knobs = ("ABG_K1_TC_CAP_KB", "ABG_K1_TC_STAGES", "ABG_K1_TC_DIGITS", "FFT_MODE", "ABG_K2_LPW", "ABG_K2_PRIO")
    for v in variants:
        for k in knobs:
            os.environ.pop(k, None)
        for kv in filter(None, v.split(",")):
            k, val = kv.split("=")
            os.environ[k] = val
        mode = int(os.environ.get("FFT_MODE", "3"))
        eng = lib.Engine(cfg, max_batches_per_run=nb, input_capacity_batches=nb + 1, fft_mode=mode)
        for d in range(len(cfg.devices)):
            eng.resident_load(d, raws[d])
        for _ in range(5):
            eng.run_resident(nb)
        eng.sync()
        k1, k2, tot = [], [], []
        import time
        for _ in range(20):
            eng.run_resident(nb)
            t = eng.last_run_times()
            k1.append(t[0]); k2.append(t[1]); tot.append(t[3])
        eng.sync()
        t0 = time.perf_counter()
        n = 200
        for _ in range(n):
            eng.run_resident(nb)
        eng.sync()
        dt = (time.perf_counter() - t0) / n * 1e3
        print(f"{wname} [{v or 'default'}] path={eng.fft_path(0)} K1 {np.median(k1):.4f} ms  K2 {np.median(k2):.4f} ms  run {np.median(tot):.4f} ms  pipelined step {dt:.4f} ms", flush=True)
        eng.close()


if __name__ == "__main__":
    main()
