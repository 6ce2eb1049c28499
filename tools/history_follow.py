"""Cost of live follow on cfg2, streamed: all 64 devices pushed from pageable memory, runs of 4 batches, every live output
fetched, with the I/Q history on devices 0-3.  Three legs alternate in one process:
  (a) no sessions;
  (b) 1 session (device 0, its 8 channels);
  (c) 16 sessions, 4 on each of devices 0-3;
and in (b) and (c) abg_follow_run(-1) plus every session's fetch after each live run.  Per leg: the live run period (host
clock over the runs, ending in a synchronise), the host time of abg_follow_run, the follow engines' device time of the
latest call (abg_debug_follow_time: gathers, runs), and the lag (batches the live engine has enqueued minus the
fewest any session has enqueued, after every follow_run; 1 = one batch behind).  The card name and power limit are read
in the same call.

    python tools/history_follow.py [--reps 5] [--runs 20] [--out DIR]

Prints one JSON line (and writes it to DIR/history_follow.jsonl with --out)."""
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

HIST_DEVS, HIST_BATCHES = 4, 16


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--runs", type=int, default=20, help="timed live runs per leg")
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
        if d < HIST_DEVS:
            e.history_configure(d, HIST_BATCHES)
        e.push(d, head)
    sessions = []

    def live_last():
        end = e.history_range(0)[1]
        return (end // hop - AGC_EXTRA) // B - 1

    def runs(follow):
        ft, lag = [], []
        t0 = time.perf_counter()
        for _ in range(args.runs):
            for k in range(nd):
                e.push(k, body)
            e.run(-1)
            for k in range(nd):
                while e.fetch(k) is not None:
                    pass
            if follow:
                t1 = time.perf_counter()
                e.follow_run(-1)
                ft.append((time.perf_counter() - t1) * 1e3)
                lag.append(live_last() + 1 - min(e.follow_info(s)["next_batch"] for s in sessions))
                for s in sessions:
                    e.follow_fetch(s, want_iq=False)
        e.sync()
        period = (time.perf_counter() - t0) * 1e3 / args.runs
        g, r = e.follow_time() if follow else (0.0, 0.0)
        return period, (float(np.median(ft)) if ft else 0.0), g, r, (max(lag) if lag else 0)

    def open_sessions(n):
        for s in sessions:
            e.follow_close(s)
        sessions.clear()
        first = live_last() + 1
        for k in range(n):
            dev = k % HIST_DEVS if n > 1 else 0
            sessions.append(e.follow_open(dev, first, full.devices[dev].channels, queue_batches=8))

    legs = {}
    names = (("a_no_sessions", 0), ("b_1_session", 1), ("c_16_sessions_4_devices", 16))
    for n_s in (0, 1, 16):  # warm-up: fills the history, creates the follow engines
        open_sessions(n_s)
        runs(n_s > 0)
    for _ in range(args.reps):
        for name, n_s in names:
            open_sessions(n_s)
            runs(n_s > 0)  # the new sessions catch up to the live edge
            p, ft, g, r, lag = runs(n_s > 0)
            for k, v in (("period_ms", p), ("follow_run_host_ms", ft), ("gather_ms", g), ("follow_runs_ms", r), ("lag_batches", lag)):
                legs.setdefault(f"{name}_{k}", []).append(v)
    open_sessions(0)
    e.close()
    med = {k + "_median": float(np.median(v)) for k, v in legs.items()}
    out = {"workload": "cfg2", "desc": desc, "card": card(), "runs_per_leg": args.runs, "history_devices": HIST_DEVS, **med,
           "all": {k: [round(float(x), 3) for x in v] for k, v in legs.items()}}
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "history_follow.jsonl"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
