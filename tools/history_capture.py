"""Time of the I/Q history's captures on one cfg2 device: abg_history_subband over a 10 s window at decimation 32 with 255
coefficients (CUDA events around its kernels, and the host clock around the whole call, which includes the copy of the
result to host memory), and abg_history_raw of the same window (host clock; a device-to-host copy of ring bytes).  The
history is filled by streamed runs of synthetic input.  The card name and power limit are read in the same call.

    python tools/history_capture.py [--seconds 10] [--reps 5] [--out DIR]

Prints one JSON line (and writes it to DIR/history_capture.jsonl with --out)."""
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

DECIM, NTAPS = 32, 255


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    full, desc = bench.make_workload("cfg2")
    cfg = lib.Config(fft_size=full.fft_size, wave_rate=full.wave_rate, devices=[full.devices[0]])
    d = cfg.devices[0]
    sr, hop, B = d.sample_rate, cfg.hop(0), cfg.wave_batch
    nb_win = int(np.ceil(args.seconds * sr / (B * hop)))
    nb = nb_win + 2
    e = lib.Engine(cfg, max_batches_per_run=4, input_capacity_batches=6)
    e.history_configure(0, nb)
    one = bench.synth_streams(cfg, 4)[0]  # 4 batches of synthetic input, pushed over and over
    items = 2 * B * hop
    head = one[:one.size - 4 * items]  # the look-back and the first frame's tail
    body = one[one.size - 4 * items:]
    e.push(0, head)
    done = 0
    while done < nb:
        e.push(0, body[:items * min(4, nb - done)])
        done += e.run(-1)
        while e.fetch(0) is not None:
            pass
    e.sync()
    first, end = e.history_range(0)
    n_in = int(args.seconds * sr)
    h = lib.subband_lowpass(NTAPS, 0.4 * sr / DECIM, sr, 60.0)
    m0 = -(-(end - n_in) // DECIM)
    n_out = (end - 1) // DECIM - m0 + 1
    assert m0 * DECIM - (NTAPS - 1) >= first
    sub_host, sub_kernel, raw_host = [], [], []
    for rep in range(args.reps + 1):
        t0 = time.perf_counter()
        y = e.history_subband(0, 0.1 * sr, DECIM, h, m0, n_out)
        t1 = time.perf_counter()
        k = e.history_time()[1]
        t2 = time.perf_counter()
        r = e.history_raw(0, end - n_in, n_in)
        t3 = time.perf_counter()
        if rep:  # the first call of each allocates and warms up
            sub_host.append((t1 - t0) * 1e3); sub_kernel.append(k); raw_host.append((t3 - t2) * 1e3)
    assert y.size == n_out and r.size == 2 * n_in
    raw_bytes = n_in * 2 * d.bytes_per_sample
    out = {"workload": "cfg2, device 0", "desc": desc, "card": card(), "window_s": args.seconds, "input_samples": n_in,
           "raw_bytes": raw_bytes, "decim": DECIM, "n_coeffs": NTAPS, "outputs": n_out,
           "subband_kernel_ms_median": float(np.median(sub_kernel)), "subband_call_ms_median": float(np.median(sub_host)),
           "raw_call_ms_median": float(np.median(raw_host)), "subband_kernel_ms_all": [round(x, 3) for x in sub_kernel],
           "raw_call_ms_all": [round(x, 3) for x in raw_host]}
    line = json.dumps(out)
    print(line, flush=True)
    e.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "history_capture.jsonl"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
