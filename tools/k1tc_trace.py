#!/usr/bin/env python
"""Measurement aid: per-role timeline of the tensor-core K1 (clock64 stamps inside the kernel, ABG_K1_TC_TRACE) for one CTA.
    python tools/k1tc_trace.py [cfg2] [cta]"""
import os
import sys

os.environ["ABG_K1_TC_TRACE"] = "1"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "rtlsdr-airband_b200", "py"))
sys.path.insert(0, ROOT)
import ctypes as C  # noqa: E402

import numpy as np  # noqa: E402

import bench  # noqa: E402
from airband_b200 import lib  # noqa: E402

wname = sys.argv[1] if len(sys.argv) > 1 else "cfg2"
cta = int(sys.argv[2]) if len(sys.argv) > 2 else 5
cfg, _ = bench.make_workload(wname)
raws = bench.synth_streams(cfg, 4)
eng = lib.Engine(cfg, max_batches_per_run=4, input_capacity_batches=5, fft_mode=3)
for d in range(len(cfg.devices)):
    eng.resident_load(d, raws[d])
for _ in range(3):
    eng.run_resident(4)
eng.sync()
buf = np.zeros(256 * 4 * 16 * 4, np.int64)
assert eng.L.abg_debug_k1tc_trace(buf.ctypes.data_as(C.c_void_p)) == 0
t = buf.reshape(256, 4, 16, 4)[cta]
t0 = t[t > 0].min()
names = {0: ("producer", ["info seen", "-", "-", "tile copies issued"]), 1: ("epilogue", ["-", "accumulators ready", "done", "-"]),
         2: ("loader", ["tile start", "tile B issued", "-", "-"]), 3: ("mma", ["info seen", "-", "-", "-"])}
for tile in range(6):
    print(f"tile {tile}")
    for role in range(4):
        nm, ev = names[role]
        vals = [int(v - t0) if v > 0 else None for v in t[role, tile]]
        print(f"   {nm:9s} " + "  ".join(f"{e}={v}" for e, v in zip(ev, vals) if e != "-"))
st = buf.reshape(256, 4, 64)[cta]
print("stage-level stamps of tile 3, one stage = one column pair (cycles since the loader's first stamp):")
base = st[2, 32]
for k in range(16):
    lo, li, mw, mc = (int(st[2, 32 + 2 * k] - base), int(st[2, 33 + 2 * k] - base), int(st[3, 32 + 2 * k] - base), int(st[3, 33 + 2 * k] - base))
    print(f"   stage {k:2d}: loader empty ok {lo:6d} issued {li:6d} | mma full ok {mw:6d} committed {mc:6d}")
eng.close()
