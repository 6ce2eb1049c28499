"""Cost of history analysis on cfg2, streamed: all 64 devices pushed from pageable memory, runs of 4 batches, every live
output fetched, the I/Q history on every device (82 batches on device 0, 18 on the others).  Legs alternate in one
process, each measured on a window the history holds at that moment:
  (a) a 10 s spectrogram (80 rows of one batch) and a 10 s detection of device 0, at the default stride and at stride 1;
  (b) the last 2 s (16 batches) of all 64 devices in one call, spectrogram and detection, default stride;
  (c) the streamed live run period without calls, and with one (b) detection call between runs;
  (d) the live detector on all 64 devices at the default stride: its kernel time per run (4 batches) and the run period.
Per call: host time (a clock around the call, which waits for its results) and the three device times of
abg_debug_history_analysis_time (gathers, spectrum kernels, detector kernels).  Thresholds come from the spectrogram of the
same window (activity_threshold, 13 dB over the median of +-16 bins).  The card name and power limit are read in the same
call.

    python tools/history_analysis.py [--reps 5] [--runs 20] [--out DIR]

Prints one JSON line (and writes it to DIR/history_analysis.jsonl with --out)."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "rtlsdr-airband_b200", "py"), ROOT]
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from airband_b200 import lib  # noqa: E402
from airband_b200.config import AGC_EXTRA  # noqa: E402

HIST0, HIST = 82, 18  # batches: 10 s of device 0 and 2 s of every device, plus the batch whose tail they wait for


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--runs", type=int, default=20, help="timed live runs per leg of (c) and (d)")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    full, desc = bench.make_workload("cfg2")
    B, hop, N = full.wave_batch, full.hop(0), full.fft_size
    nd = len(full.devices)
    s_def = lib.default_stride(full, 0)
    e = lib.Engine(full, max_batches_per_run=4, input_capacity_batches=6)
    one = bench.synth_streams(lib.Config(fft_size=full.fft_size, wave_rate=full.wave_rate, devices=[full.devices[0]]), 4)[0]
    items = 2 * B * hop
    head, body = one[:one.size - 4 * items], one[one.size - 4 * items:]
    for d in range(nd):
        e.history_configure(d, HIST0 if d == 0 else HIST)
        e.push(d, head)

    def run_once():
        for k in range(nd):
            e.push(k, body)
        e.run(-1)
        for k in range(nd):
            while e.fetch(k) is not None:
                pass

    for _ in range(HIST0 // 4 + 2):  # fill every history
        run_once()
    e.sync()

    def spec_jobs(devs, seconds, stride):
        jobs = []
        for d in devs:
            b0, nb = lib.history_window(full, d, e.history_range(d), stride=stride, seconds=seconds)
            jobs.append(dict(dev=d, first_frame=AGC_EXTRA + b0 * B, n_rows=nb, frames_per_row=B, stride=stride))
        return jobs

    def act_jobs(sj, thr):
        return [dict(dev=j["dev"], first_batch=(j["first_frame"] - AGC_EXTRA) // B, n_batches=j["n_rows"], stride=j["stride"],
                     hang=1, min_span=2, thr=thr) for j in sj]

    thr_cache = {}

    def timed(fn, jobs):
        e.sync()
        t0 = time.perf_counter()
        r = fn(jobs)
        return r, (time.perf_counter() - t0) * 1e3, e.history_analysis_time()

    legs = {}

    def put(name, host, dev3):
        for k, v in (("host_ms", host), ("gather_ms", dev3[0]), ("spectrum_ms", dev3[1]), ("detector_ms", dev3[2])):
            legs.setdefault(f"{name}_{k}", []).append(v)

    def analysis_legs():
        for tag, devs, seconds, stride in (("a_10s_dev0_default", [0], 10.0, s_def), ("a_10s_dev0_stride1", [0], 10.0, 1),
                                            ("b_2s_64dev_default", list(range(nd)), 2.0, s_def)):
            sj = spec_jobs(devs, seconds, stride)
            assert sj[0]["n_rows"] == int(seconds * full.wave_rate / B), sj[0]
            spec, host, dev3 = timed(e.history_spectrogram, sj)
            put(tag + "_spectrogram", host, dev3)
            thr = thr_cache.setdefault(stride, lib.activity_threshold(spec[0], 13.0, 16))
            _, host, dev3 = timed(e.history_activity, act_jobs(sj, thr))
            put(tag + "_detection", host, dev3)

    def period(call):
        e.sync()
        t0 = time.perf_counter()
        for _ in range(args.runs):
            run_once()
            if call:
                e.history_activity(act_jobs(spec_jobs(range(nd), 2.0, s_def), thr_cache[s_def]))
        e.sync()
        return (time.perf_counter() - t0) * 1e3 / args.runs

    def live_detector():
        for d in range(nd):
            e.activity_configure(d, s_def, 1, 2, thr_cache[s_def])
        run_once()
        e.sync()
        t0 = time.perf_counter()
        ms = []
        for _ in range(args.runs):
            run_once()
            ms.append(e.activity_time())
            for d in range(nd):
                while e.fetch_activity(d) is not None:
                    pass
        e.sync()
        p = (time.perf_counter() - t0) * 1e3 / args.runs
        for d in range(nd):
            e.activity_configure(d, 0, 0, 0, None)
        return p, float(np.median(ms))

    analysis_legs()  # warm-up: allocates the analysis buffers, fills the threshold cache
    period(True)
    live_detector()
    for _ in range(args.reps):
        analysis_legs()
        legs.setdefault("c_period_no_calls_ms", []).append(period(False))
        legs.setdefault("c_period_one_2s_64dev_detection_per_run_ms", []).append(period(True))
        p, ms = live_detector()
        legs.setdefault("d_period_live_detector_ms", []).append(p)
        legs.setdefault("d_live_detector_kernel_ms_per_run", []).append(ms)
    e.close()
    med = {k + "_median": float(np.median(v)) for k, v in legs.items()}
    out = {"workload": "cfg2", "desc": desc, "card": card(), "runs_per_leg": args.runs, "default_stride": s_def, **med,
           "all": {k: [round(float(x), 3) for x in v] for k, v in legs.items()}}
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "history_analysis.jsonl"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
