"""Cost of one batch monitor on the resident pipeline: run period in each of the monitor's legs, alternating in one
process, plus the monitor kernel's own CUDA-event time and K1 / K2.  The card name and power limit are read in the same
call.

    python tools/monitor_overhead.py --monitor {spectrum,carrier,input_meter,subband,tone_meter,activity,history} [--workloads cfg2,cfg5] [--runs 40]
                                     [--reps 3] [--out DIR]

Legs:
  spectrum     off, the default stride (ceil(fft_size / hop): non-overlapping frames), stride 1
  carrier      off, on for every device
  input_meter  off, on for every device
  subband      no output, one and four outputs per device (decimation 32, 255 coefficients).  Resident runs compute every
               output but write none to the host rings, so these times leave out the outputs' transfer to host memory.
  tone_meter   off, on for every device with the 51 standard tones.  As for the sub-band outputs, resident runs leave out
               the readings' transfer to host memory.
  activity     off, the default stride, stride 1; hang 1, min_span 1 and a uniform threshold of ACT_THR (|X|^2) for every
               bin.  Resident runs count pieces but store none, so these times leave out the records' transfer.
  history      off, on for every device with a capacity of HIST_BATCHES batches (the append only; resident runs append
               like streamed ones but leave the history empty).

Prints one JSON line per workload (and writes it to DIR/<monitor>_overhead.jsonl with --out).  It uses only public
lib.Engine methods, so ABG_LIB_PATH can point it at another build of the library."""
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
DECIM, NTAPS = 32, 255  # sub-band outputs
ACT_THR = 1.0e4  # activity detector threshold, on the band spectrum's scale
HIST_BATCHES = 8  # I/Q history capacity


def raw_bytes_per_run(cfg):
    return sum(NB * cfg.wave_batch * cfg.hop(d) * 2 * dv.bytes_per_sample for d, dv in enumerate(cfg.devices))


def activity_configure(e, cfg, d, stride):
    if stride == 0:
        e.activity_configure(d, 0)
    else:
        e.activity_configure(d, stride, 1, 1, np.full(cfg.fft_size, ACT_THR, np.float32))


def subband_configure(e, cfg, d, n_out):
    sr = cfg.devices[d].sample_rate
    h = lib.subband_lowpass(NTAPS, 0.4 * sr / DECIM, sr, 60.0)
    for k in range(4):
        if k < n_out:
            e.subband_configure(d, k, (k - 1.5) * 0.2 * sr, DECIM, h)
        else:
            e.subband_configure(d, k, 0.0, 0)


# legs(cfg) -> {leg: setting}; configure(engine, cfg, dev, setting); the kernel time method and its JSON name; extra(cfg):
# workload fields; setting_key: the name under which a leg records its setting (if it does)
MONITORS = {
    "spectrum": dict(
        legs=lambda cfg: {"off": 0, "default_stride": lib.default_stride(cfg, 0), "stride_1": 1},
        configure=lambda e, cfg, d, stride: e.spectrum_configure(d, stride),
        time="spectrum_time", time_key="spectrum_ms", setting_key="stride", extra=lambda cfg: {}),
    "carrier": dict(
        legs=lambda cfg: {"off": False, "on": True},
        configure=lambda e, cfg, d, on: e.carrier_configure(d, on),
        time="carrier_time", time_key="carrier_ms",
        extra=lambda cfg: {"iqin_bytes_read_per_run": NB * cfg.wave_batch * sum(len(d.channels) for d in cfg.devices) * 8}),
    "input_meter": dict(
        legs=lambda cfg: {"off": False, "on": True},
        configure=lambda e, cfg, d, on: e.input_meter_configure(d, on),
        time="input_meter_time", time_key="meter_ms", extra=lambda cfg: {"raw_bytes_read_per_run": raw_bytes_per_run(cfg)}),
    "subband": dict(
        legs=lambda cfg: {"off": 0, "one": 1, "four": 4},
        configure=subband_configure,
        time="subband_time", time_key="subband_ms",
        extra=lambda cfg: {"decim": DECIM, "n_coeffs": NTAPS, "raw_bytes_read_per_run": raw_bytes_per_run(cfg),
                           "outputs_per_run_per_output": sum(NB * -(-(cfg.wave_batch * cfg.hop(d)) // DECIM)
                                                             for d in range(len(cfg.devices)))}),
    "tone_meter": dict(
        legs=lambda cfg: {"off": False, "on": True},
        configure=lambda e, cfg, d, on: e.tone_meter_configure(d, on),
        time="tone_meter_time", time_key="tone_meter_ms",
        extra=lambda cfg: {"n_tones": len(lib.STANDARD_TONES),
                           "wout_bytes_read_per_run": NB * cfg.wave_batch * sum(len(d.channels) for d in cfg.devices) * 4,
                           "gemm_flop_per_run": 2 * NB * sum(len(d.channels) for d in cfg.devices) * cfg.wave_batch
                           * 2 * len(lib.STANDARD_TONES)}),
    "activity": dict(
        legs=lambda cfg: {"off": 0, "default_stride": lib.default_stride(cfg, 0), "stride_1": 1},
        configure=activity_configure,
        time="activity_time", time_key="activity_ms", setting_key="stride",
        extra=lambda cfg: {"threshold": ACT_THR, "hang": 1, "min_span": 1}),
    "history": dict(
        legs=lambda cfg: {"off": 0, "on": HIST_BATCHES},
        configure=lambda e, cfg, d, n: e.history_configure(d, n),
        time="history_time", time_key="append_ms", setting_key="n_batches",
        extra=lambda cfg: {"raw_bytes_read_and_written_per_run": raw_bytes_per_run(cfg)}),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--monitor", required=True, choices=sorted(MONITORS))
    ap.add_argument("--workloads", default="cfg2,cfg5")
    ap.add_argument("--runs", type=int, default=40, help="timed runs per leg")
    ap.add_argument("--reps", type=int, default=3, help="rounds of the alternating legs")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    mon = MONITORS[args.monitor]
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
        kernel_time = getattr(e, mon["time"])
        legs = mon["legs"](cfg)
        res = {k: {"period_ms": [], "kernel_ms": [], "k1_ms": [], "k2_ms": [], "launches_per_run": 0} for k in legs}
        for _ in range(args.reps):
            for leg, setting in legs.items():
                for d in range(D):
                    mon["configure"](e, cfg, d, setting)
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
                    t = kernel_time()
                    r["kernel_ms"].append(t[0] if isinstance(t, tuple) else t)  # history_time: (append, capture)
        out = {"workload": name, "desc": desc, "card": card(), "batches_per_run": NB, "runs_per_leg": args.runs, "reps": args.reps,
               **mon["extra"](cfg)}
        for leg, setting in legs.items():
            r = res[leg]
            out[leg] = {mon["setting_key"]: setting} if "setting_key" in mon else {}
            out[leg].update({"period_ms_median": float(np.median(r["period_ms"])), "period_ms_all": [round(x, 4) for x in r["period_ms"]],
                             mon["time_key"] + "_median": float(np.median(r["kernel_ms"])), "k1_ms_median": float(np.median(r["k1_ms"])),
                             "k2_ms_median": float(np.median(r["k2_ms"])), "launches_per_run": r["launches_per_run"]})
        line = json.dumps(out)
        print(line, flush=True)
        lines.append(line)
        e.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"{args.monitor}_overhead.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
