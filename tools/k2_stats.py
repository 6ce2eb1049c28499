#!/usr/bin/env python
"""Measurement aid: event counters of the K2 tile paths for one workload (needs `make -C rtlsdr-airband_b200 stats`):
    ABG_LIB_PATH=rtlsdr-airband_b200/build/stats/libairband_b200.so python tools/k2_stats.py cfg3"""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.environ.setdefault("ABG_LIB_PATH", os.path.join(ROOT, "rtlsdr-airband_b200", "build", "stats", "libairband_b200.so"))
sys.path.insert(0, os.path.join(ROOT, "rtlsdr-airband_b200", "py"))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from airband_b200 import lib  # noqa: E402

NAMES = {0: "samples", 1: "general-path samples", 2: "tile attempts OPEN", 3: "tile attempts CLOSING", 4: "tile attempts OPENING", 5: "tile attempts CLOSED",
         6: "tile attempts ABORT", 7: "tile samples OPEN", 8: "tile samples CLOSING", 9: "tile samples OPENING", 10: "tile samples CLOSED", 11: "tile samples ABORT",
         12: "no room for a tile", 13: "CTCSS window ends in tile", 14: "post estimator not live", 15: "OPENING at buffer_size boundary", 16: "CLOSED recent_open pending",
         17: "tiles of 8", 18: "tiles of 16", 20: "  .. state ends within 8", 22: "tile attempts held-CLOSED", 23: "tile samples held-CLOSED", 31: "refused: held-CLOSED ends", 21: "  .. noise-floor update within 8", 24: "refused: low_signal_abort", 25: "refused: lp division range",
         26: "refused: sqrt range", 27: "refused: has_signal false", 28: "refused: CLOSED sees signal", 29: "refused: post < tail", 30: "refused: discriminator division range",
         32: "general in CLOSED", 33: "general in OPENING", 34: "general in CLOSING", 35: "general in ABORT", 36: "general in OPEN", 40: "general: transition sample",
         41: "AM tile attempts OPEN", 42: "AM tile samples OPEN", 43: "AM tile refused OPEN", 44: "AM tile attempts quiet", 45: "AM tile samples quiet",
         46: "AM tile refused quiet", 47: "AM OPEN tile fully capped", 48: "AM OPEN tile never capped", 57: "AM quiet tile never capped",
         49: "AM open_run attempts (LPW>=2)", 50: "AM open_run refused", 51: "AM quiet_run attempts (LPW>=2)", 52: "AM quiet_run refused",
         53: "AM open sample: exact division", 54: "NFM block attempts OPEN/CLOSING (LPW 2)", 55: "NFM block attempts OPENING", 56: "NFM block attempts CLOSED",
         58: "NFM block samples", 59: "NFM block refused"}


def main():
    wname = sys.argv[1] if len(sys.argv) > 1 else "cfg3"
    nruns = int(sys.argv[2]) if len(sys.argv) > 2 else 8
    cfg, _ = bench.make_workload(wname)
    nb = 4
    raws = bench.synth_streams(cfg, nb)
    eng = lib.Engine(cfg, max_batches_per_run=nb, input_capacity_batches=nb + 1)
    for d in range(len(cfg.devices)):
        eng.resident_load(d, raws[d])
    L = lib.load()
    out = (C.c_ulonglong * 64)()
    for _ in range(4):
        eng.run_resident(nb)
    eng.sync()
    assert L.abg_debug_k2_stats(out) == 0, "not a stats build"
    for _ in range(nruns):
        eng.run_resident(nb)
    eng.sync()
    assert L.abg_debug_k2_stats(out) == 0
    tot = max(1, out[0])
    print(f"{wname}: {nruns} runs of {nb} batches")
    for i in range(64):
        if out[i]:
            print(f"  [{i:2d}] {NAMES.get(i, '?'):36s} {out[i]:12d}  {100.0 * out[i] / tot:7.2f} % of samples")
    eng.close()


if __name__ == "__main__":
    main()
