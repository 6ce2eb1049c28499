"""Cost of transmission profiles on cfg2, streamed: all 64 devices pushed from pageable memory, runs of 4 batches, every
live output fetched, the I/Q history on every device (18 batches).  Legs alternate in one process:
  (a) one 2 s transmission of device 0 (its newest 16 batches), profile_job's default filter and the 51 standard tones;
  (b) one 2 s transmission on each of the 64 devices, in one call;
  (c) the streamed live run period without calls, and with one (b) call between runs.
Per call: host time (a clock around the call, which waits for its results) and the two device times of
abg_debug_history_profile_time (capture kernels, profile kernels).  The card's name, power limit and max SM clock are read
in the same call.

    python tools/history_profile.py [--reps 5] [--runs 20] [--out DIR]

Prints one JSON line (and writes it to DIR/history_profile.jsonl with --out)."""
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

HIST = 18  # batches: 2 s of every device, plus the batch whose tail a window waits for


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--runs", type=int, default=20, help="timed live runs per leg of (c)")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    full, desc = bench.make_workload("cfg2")
    B, hop = full.wave_batch, full.hop(0)
    nd = len(full.devices)
    e = lib.Engine(full, max_batches_per_run=4, input_capacity_batches=6)
    one = bench.synth_streams(lib.Config(fft_size=full.fft_size, wave_rate=full.wave_rate, devices=[full.devices[0]]), 4)[0]
    items = 2 * B * hop
    head, body = one[:one.size - 4 * items], one[one.size - 4 * items:]
    for d in range(nd):
        e.history_configure(d, HIST)
        e.push(d, head)

    def run_once():
        for k in range(nd):
            e.push(k, body)
        e.run(-1)
        for k in range(nd):
            while e.fetch(k) is not None:
                pass

    for _ in range(HIST // 4 + 2):  # fill every history
        run_once()
    e.sync()

    def jobs_for(devs):
        jobs = []
        for d in devs:
            b0, nb = lib.history_window(full, d, e.history_range(d), seconds=2.0)
            tx = dict(freq_hz=full.devices[d].centerfreq + 100_000.0, first_frame=AGC_EXTRA + b0 * B,
                      last_frame=AGC_EXTRA + (b0 + nb) * B - 1)
            jobs.append(lib.profile_job(tx, full, d, e.history_range(d)))
        return jobs

    legs = {}

    def timed(tag, devs):
        jobs = jobs_for(devs)
        e.sync()
        t0 = time.perf_counter()
        e.history_profile(jobs)
        host = (time.perf_counter() - t0) * 1e3
        cap, prof = e.history_profile_time()
        for k, v in (("host_ms", host), ("capture_ms", cap), ("profile_ms", prof)):
            legs.setdefault(f"{tag}_{k}", []).append(v)
        return jobs

    def period(call):
        e.sync()
        t0 = time.perf_counter()
        for _ in range(args.runs):
            run_once()
            if call:
                e.history_profile(jobs_for(range(nd)))
        e.sync()
        return (time.perf_counter() - t0) * 1e3 / args.runs

    j0 = timed("a_2s_dev0", [0])[0]  # warm-up: allocates the profile buffers
    timed("b_2s_64dev", range(nd))
    period(True)
    legs.clear()
    for _ in range(args.reps):
        timed("a_2s_dev0", [0])
        timed("b_2s_64dev", range(nd))
        legs.setdefault("c_period_no_calls_ms", []).append(period(False))
        legs.setdefault("c_period_one_64dev_call_per_run_ms", []).append(period(True))
    e.close()
    med = {k + "_median": float(np.median(v)) for k, v in legs.items()}
    out = {"workload": "cfg2", "desc": desc, "card": card(), "runs_per_leg": args.runs,
           "job": dict(decim=j0["decim"], n_coeffs=int(j0["coeffs"].size), n_out=j0["n_out"], tones=len(lib.STANDARD_TONES)),
           **med, "all": {k: [round(float(x), 4) for x in v] for k, v in legs.items()}}
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "history_profile.jsonl"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
