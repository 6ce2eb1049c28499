"""Time of the history replay on cfg2 devices, with the legs alternating in one process:
  (a) abg_history_replay of a 10 s window of one device with its 8 channels (host clock around the call, which waits
      for its results, and the call's own CUDA-event times of the gathers and of the replay engine's runs);
  (b) the host round trip the replay replaces: abg_history_raw of the same window, then a fresh engine (created and
      destroyed inside the timed region) that is pushed those bytes, run and fetched;
  (c) one call with 16 jobs, the same window of each of 16 devices;
and the live run period of all 64 cfg2 devices, streamed (pushes from pageable memory, runs of 4 batches, every output
fetched): without replays, with a one-job replay of 4 batches between runs, and with replays of 1, 2, 3, 1, 2, 3, ... such
jobs between runs (the replay engine grows to 3 devices in the warm-up and is not rebuilt after that).  The card name and
power limit are read in the same call.

    python tools/history_replay.py [--seconds 10] [--reps 5] [--runs 20] [--out DIR]

Prints one JSON line (and writes it to DIR/history_replay.jsonl with --out)."""
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def filled(cfg, nb, hist):
    """An engine over cfg's devices, each with a history of `hist` batches, after nb batches of synthetic input."""
    e = lib.Engine(cfg, max_batches_per_run=4, input_capacity_batches=6)
    B = cfg.wave_batch
    one = bench.synth_streams(lib.Config(fft_size=cfg.fft_size, wave_rate=cfg.wave_rate, devices=[cfg.devices[0]]), 4)[0]
    items = 2 * B * cfg.hop(0)
    head, body = one[:one.size - 4 * items], one[one.size - 4 * items:]
    for d in range(len(cfg.devices)):
        if hist:
            e.history_configure(d, hist)
        e.push(d, head)
    done = 0
    while done < nb:
        for d in range(len(cfg.devices)):
            e.push(d, body[:items * min(4, nb - done)])
        n = e.run(-1)
        done += n // len(cfg.devices)
        for d in range(len(cfg.devices)):
            while e.fetch(d) is not None:
                pass
    e.sync()
    return e, body, items


def window_job(e, cfg, dev, nb_win):
    B, hop = cfg.wave_batch, cfg.hop(dev)
    first, _ = e.history_range(dev)
    return dict(dev=dev, first_batch=-(-first // (B * hop)), n_batches=nb_win, channels=cfg.devices[dev].channels)


def round_trip(e, cfg, job):
    B, hop, N = cfg.wave_batch, cfg.hop(0), cfg.fft_size
    S = job["first_batch"] * B * hop
    need = (AGC_EXTRA + job["n_batches"] * B) * hop + N - hop
    raw = np.concatenate([e.history_raw(job["dev"], S, need), np.zeros(2 * hop, np.uint8)])
    f = lib.Engine(lib.Config(fft_size=N, wave_rate=cfg.wave_rate, devices=[cfg.devices[job["dev"]]]),
                   input_capacity_batches=job["n_batches"] + 2)
    f.push(0, raw)
    got = 0
    while f.run(-1) > 0:
        while f.fetch(0) is not None:
            got += 1
    f.close()
    assert got == job["n_batches"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--runs", type=int, default=20, help="timed live runs per leg")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    full, desc = bench.make_workload("cfg2")
    one = lib.Config(fft_size=full.fft_size, wave_rate=full.wave_rate, devices=[full.devices[0]])
    sixteen = lib.Config(fft_size=full.fft_size, wave_rate=full.wave_rate, devices=full.devices[:16])
    d = one.devices[0]
    B, hop = one.wave_batch, one.hop(0)
    nb_win = int(np.ceil(args.seconds * d.sample_rate / (B * hop)))
    e1, _, _ = filled(one, nb_win + 2, nb_win + 2)
    e16, _, _ = filled(sixteen, nb_win + 2, nb_win + 2)
    job = window_job(e1, one, 0, nb_win)
    jobs16 = [window_job(e16, sixteen, k, nb_win) for k in range(16)]
    legs = {"a_replay_ms": [], "a_gather_ms": [], "a_runs_ms": [], "b_round_trip_ms": [], "c_replay16_ms": [],
            "c_gather_ms": [], "c_runs_ms": []}
    for rep in range(args.reps + 1):  # the first round allocates and warms up
        t0 = time.perf_counter()
        e1.history_replay([job], want_iq=False)
        t1 = time.perf_counter()
        ga, ra = e1.replay_time()
        t2 = time.perf_counter()
        round_trip(e1, one, job)
        t3 = time.perf_counter()
        e16.history_replay(jobs16, want_iq=False)
        t4 = time.perf_counter()
        gc, rc = e16.replay_time()
        if rep:
            for k, v in (("a_replay_ms", (t1 - t0) * 1e3), ("a_gather_ms", ga), ("a_runs_ms", ra),
                         ("b_round_trip_ms", (t3 - t2) * 1e3), ("c_replay16_ms", (t4 - t3) * 1e3), ("c_gather_ms", gc),
                         ("c_runs_ms", rc)):
                legs[k].append(v)
    e1.close()
    e16.close()

    # live run period of cfg2, streamed, without and with a replay between runs
    e, body, items = filled(full, 8, 0)
    e.history_configure(0, 8)
    live = {"live_period_ms_no_replay": [], "live_period_ms_with_replay": [], "live_period_ms_with_1_2_3_jobs": []}
    nd = len(full.devices)

    def runs(replay, vary=False):
        t0 = time.perf_counter()
        for i in range(args.runs):
            for k in range(nd):
                e.push(k, body)
            e.run(-1)
            for k in range(nd):
                while e.fetch(k) is not None:
                    pass
            if replay:
                e.history_replay([window_job(e, full, 0, 4)] * (1 + i % 3 if vary else 1), want_iq=False)
        e.sync()
        return (time.perf_counter() - t0) * 1e3 / args.runs

    runs(False)  # fills the history
    runs(True, vary=True)
    for _ in range(args.reps):
        live["live_period_ms_no_replay"].append(runs(False))
        live["live_period_ms_with_replay"].append(runs(True))
        live["live_period_ms_with_1_2_3_jobs"].append(runs(True, vary=True))
    e.close()
    med = {k + "_median": float(np.median(v)) for k, v in {**legs, **live}.items()}
    out = {"workload": "cfg2", "desc": desc, "card": card(), "window_s": args.seconds, "window_batches": nb_win,
           "channels_per_job": len(d.channels), "raw_bytes_per_window": int((AGC_EXTRA + nb_win * B) * hop * 2 * d.bytes_per_sample),
           **med, "all": {k: [round(x, 3) for x in v] for k, v in {**legs, **live}.items()}}
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "history_replay.jsonl"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
