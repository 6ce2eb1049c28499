"""Cost of the sub-band I/Q outputs on the resident pipeline: run period with no output, one output per device and four
outputs per device (decimation 32, 255 coefficients), alternating in one process, plus the sub-band kernel's own
CUDA-event time and K1 / K2.  Resident runs compute every output but write none to the host rings, so the times below
leave out the outputs' transfer to host memory.  The card name and power limit are read in the same call.

    python tools/subband_overhead.py [--workloads cfg2,cfg5] [--runs 40] [--reps 3] [--out DIR]

Prints one JSON line per workload (and writes it to DIR/subband_overhead.jsonl with --out)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "rtlsdr-airband_b200", "py"), ROOT]
import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
from airband_b200 import lib  # noqa: E402

NB = 4  # batches per run, as bench.py's resident leg
DECIM, NTAPS = 32, 255


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg2,cfg5")
    ap.add_argument("--runs", type=int, default=40, help="timed runs per leg")
    ap.add_argument("--reps", type=int, default=3, help="rounds of the alternating legs")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    stream = torch.cuda.Stream()
    lines = []
    for name in args.workloads.split(","):
        cfg, desc = bench.make_workload(name)
        D = len(cfg.devices)
        raws = bench.synth_streams(cfg, NB)
        e = lib.Engine(cfg, max_batches_per_run=NB, input_capacity_batches=NB + 1)
        e.set_stream(stream.cuda_stream)
        for d in range(D):
            e.resident_load(d, raws[d])
        legs = {"off": 0, "one": 1, "four": 4}
        res = {k: {"period_ms": [], "sb_ms": [], "k1_ms": [], "k2_ms": [], "launches_per_run": 0} for k in legs}
        for _ in range(args.reps):
            for leg, n_out in legs.items():
                for d in range(D):
                    sr = cfg.devices[d].sample_rate
                    h = lib.subband_lowpass(NTAPS, 0.4 * sr / DECIM, sr, 60.0)
                    for k in range(4):
                        if k < n_out:
                            e.subband_configure(d, k, (k - 1.5) * 0.2 * sr, DECIM, h)
                        else:
                            e.subband_configure(d, k, 0.0, 0)
                for _ in range(5):  # warm-up, and the pipeline reaches steady state
                    e.run_resident(NB)
                torch.cuda.synchronize()
                l0 = e.launch_count()
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record(stream)
                for _ in range(args.runs):
                    e.run_resident(NB)
                e.join()
                ev1.record(stream)
                torch.cuda.synchronize()
                r = res[leg]
                r["period_ms"].append(ev0.elapsed_time(ev1) / args.runs)
                r["launches_per_run"] = (e.launch_count() - l0) / args.runs
                for _ in range(5):  # kernel times of single runs
                    e.run_resident(NB)
                    t = e.last_run_times()
                    r["k1_ms"].append(t[0]); r["k2_ms"].append(t[1])
                    r["sb_ms"].append(e.subband_time())
        raw_bytes = sum(NB * cfg.wave_batch * cfg.hop(d) * 2 * dv.bytes_per_sample for d, dv in enumerate(cfg.devices))
        outputs = sum(NB * -(-(cfg.wave_batch * cfg.hop(d)) // DECIM) for d in range(D))
        out = {"workload": name, "desc": desc, "card": card(), "batches_per_run": NB, "runs_per_leg": args.runs, "reps": args.reps,
               "decim": DECIM, "n_coeffs": NTAPS, "raw_bytes_read_per_run": raw_bytes, "outputs_per_run_per_output": outputs}
        for leg in legs:
            r = res[leg]
            out[leg] = {"period_ms_median": float(np.median(r["period_ms"])), "period_ms_all": [round(x, 4) for x in r["period_ms"]],
                        "subband_ms_median": float(np.median(r["sb_ms"])), "k1_ms_median": float(np.median(r["k1_ms"])),
                        "k2_ms_median": float(np.median(r["k2_ms"])), "launches_per_run": r["launches_per_run"]}
        line = json.dumps(out)
        print(line, flush=True)
        lines.append(line)
        e.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "subband_overhead.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
