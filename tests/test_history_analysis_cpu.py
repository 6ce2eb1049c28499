"""History analysis on the CPU: the C ABI and the C layouts of its two job structs, history_window against a brute-force
reading of the range rule in airband_b200.h, and history_transmissions' composition of the spectrogram, the thresholds,
the detector and the grouping, on a stand-in engine with synthetic readings."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from airband_b200 import config as cm
from airband_b200 import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AGC = cm.AGC_EXTRA


# ---- ABI ----------------------------------------------------------------------------------------------------------------------
def test_header_symbols_and_argtypes():
    hdr = open(os.path.join(ROOT, "include", "airband_b200.h")).read()
    for s in ("abg_history_spectrogram", "abg_history_activity", "abg_debug_history_analysis_time"):
        assert s in lib.SYMBOLS and re.search(r"ABG_API int %s\(" % s, hdr), s
    L = lib.load()
    assert L.abg_history_spectrogram.argtypes == [C.c_void_p, C.c_int, C.POINTER(lib.CSpectrogramJob)]
    assert L.abg_history_activity.argtypes == [C.c_void_p, C.c_int, C.POINTER(lib.CActivityJob)]
    assert L.abg_debug_history_analysis_time.argtypes == [C.c_void_p, C.POINTER(C.c_float)]
    for s in ("abg_history_spectrogram", "abg_history_activity", "abg_debug_history_analysis_time"):
        assert getattr(L, s).restype == C.c_int


@pytest.mark.parametrize("ctype,cname", [(lib.CSpectrogramJob, "abg_spectrogram_job"), (lib.CActivityJob, "abg_activity_job")])
def test_job_layout_matches_the_header(tmp_path, ctype, cname):
    fields = [f for f, _ in ctype._fields_]
    prog = "#include <stdio.h>\n#include <stddef.h>\n#include \"airband_b200.h\"\nint main(void) {\n"
    prog += "".join(f'    printf("%zu\\n", offsetof({cname}, {f}));\n' for f in fields)
    prog += f'    printf("%zu\\n", sizeof({cname}));\n    return 0;\n}}\n'
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text(prog)
    subprocess.run(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [getattr(ctype, f).offset for f in fields] + [C.sizeof(ctype)]


# ---- history_window ---------------------------------------------------------------------------------------------------------------
def _cfg(sr, w, n):
    return cm.Config(fft_size=n, wave_rate=w, devices=[cm.Device(sample_rate=sr, sfmt=cm.SFMT_U8, centerfreq=120_000_000)])


def _brute(cfg, rng_, stride, frames_per_row, seconds):
    """The units (batches, or F-frame rows from frame AGC_EXTRA on) all of whose selected frames' samples lie in the range,
    newest first until `seconds` is covered."""
    B, hop, N = cfg.wave_batch, cfg.hop(0), cfg.fft_size
    step = B if frames_per_row is None else frames_per_row
    first, end = rng_
    ok = []
    for k in range(0, end // (step * hop) + 2):
        frames = [AGC + k * step + j for j in range(0, step, stride)]
        if all(f * hop >= first and f * hop + N <= end for f in frames):
            ok.append(k)
    if not ok:
        return None
    assert ok == list(range(ok[0], ok[-1] + 1))  # contiguous
    if seconds is not None:
        keep = max(1, int(np.ceil(seconds * cfg.devices[0].sample_rate / (step * hop))))
        ok = ok[-keep:]
    return (ok[0], len(ok)) if frames_per_row is None else (AGC + ok[0] * step, len(ok))


CFGS = [("2048_hop256", 2048000, 8000, 2048), ("hop313_w8008", 2506504, 8008, 2048), ("8192_hop8", 64000, 8000, 8192),
        ("256_hop320", 2560000, 8000, 256)]


@pytest.mark.parametrize("name,sr,w,n", CFGS, ids=[c[0] for c in CFGS])
def test_history_window_matches_the_range_rule(name, sr, w, n):
    cfg = _cfg(sr, w, n)
    B, hop = cfg.wave_batch, cfg.hop(0)
    rng = np.random.default_rng(len(name))
    cases = 0
    for _ in range(60):
        first = int(rng.integers(AGC * hop, (AGC + 5 * B) * hop))
        end = first + int(rng.integers(0, 7 * B * hop + n))
        for stride in sorted({1, 3, lib.default_stride(cfg, 0), B}):
            for fpr in (None, B, 77, 2 * B + 13):
                if stride > (fpr or B):
                    continue
                for seconds in (None, 0.2):
                    want = _brute(cfg, (first, end), stride, fpr, seconds)
                    if want is None:
                        with pytest.raises(ValueError):
                            lib.history_window(cfg, 0, (first, end), stride=stride, frames_per_row=fpr, seconds=seconds)
                    else:
                        assert lib.history_window(cfg, 0, (first, end), stride=stride, frames_per_row=fpr, seconds=seconds) == want
                        cases += 1
    assert cases > 100


def test_history_window_of_a_live_history_lags_one_batch():
    """A history that holds batches [a, L] (samples up to the end of batch L) can be analysed up to batch L - 1 at stride 1,
    the same one-batch lag as live follow; the first batch is a itself."""
    cfg = _cfg(2048000, 8000, 2048)
    B, hop = cfg.wave_batch, cfg.hop(0)
    a, L = 3, 11
    rng_ = ((AGC + a * B) * hop, (AGC + (L + 1) * B) * hop)
    assert lib.history_window(cfg, 0, rng_) == (a, L - a)
    assert lib.history_window(cfg, 0, rng_, frames_per_row=B) == (AGC + a * B, L - a)
    with pytest.raises(ValueError):
        lib.history_window(cfg, 0, (5, 5))


# ---- history_transmissions ------------------------------------------------------------------------------------------------------
class _FakeEngine:
    """Stand-in for Engine: a fixed history range, a spectrogram with two hot bins, and detector bursts; records the calls."""

    def __init__(self, cfg, rng_, bursts):
        self.cfg, self.rng, self.bursts, self.calls = cfg, rng_, bursts, []

    def history_range(self, dev):
        self.calls.append(("range", dev))
        return self.rng

    def history_spectrogram(self, jobs):
        self.calls.append(("spectrogram", jobs))
        N = self.cfg.fft_size
        p = np.ones((jobs[0]["n_rows"], N), np.float32)
        p[:, 100] = 50.0
        return [p]

    def history_activity(self, jobs):
        self.calls.append(("activity", jobs))
        return [dict(bursts=self.bursts, n_truncated=0)]


def test_history_transmissions_composes_the_loop():
    cfg = _cfg(2048000, 8000, 2048)
    cfg.devices[0].channels = [cm.make_channel(120_100_000, 120_000_000, 2048000, 2048, 8000)]
    B, hop = cfg.wave_batch, cfg.hop(0)
    rng_ = ((AGC + 2 * B) * hop + 5, (AGC + 12 * B) * hop)
    b = np.zeros(3, lib.BURST_DTYPE)
    b["bin"] = [40, 41, 2000]
    b["first_frame"] = [AGC + 3 * B + 10, AGC + 3 * B + 12, AGC + 5 * B]
    b["last_frame"] = [AGC + 4 * B, AGC + 4 * B + 7, AGC + 6 * B]
    b["sum"] = [3.0, 1.0, 2.0]
    b["peak"] = [1.0, 0.5, 0.7]
    b["n_active"] = 5
    e = _FakeEngine(cfg, rng_, b)
    txs = lib.history_transmissions(e, cfg, 0, margin_db=10.0, half_width=8, stride=7, hang=2, min_span=3, seconds=0.9)
    b0, nb = lib.history_window(cfg, 0, rng_, stride=7, seconds=0.9)
    assert [c[0] for c in e.calls] == ["range", "spectrogram", "activity"]
    sj, aj = e.calls[1][1][0], e.calls[2][1][0]
    assert sj == dict(dev=0, first_frame=AGC + b0 * B, n_rows=nb, frames_per_row=B, stride=7)
    assert {k: aj[k] for k in ("dev", "first_batch", "n_batches", "stride", "hang", "min_span")} == \
        dict(dev=0, first_batch=b0, n_batches=nb, stride=7, hang=2, min_span=3)
    spec = e.history_spectrogram([sj])[0]
    assert np.array_equal(aj["thr"], lib.activity_threshold(spec, 10.0, 8))
    assert txs == lib.group_transmissions(b, cfg, 0)
    assert len(txs) == 2 and txs[0]["bins"] == (40, 41) and txs[1]["bins"] == (-48, -48)
    job = lib.transmission_replay(txs[0], cfg, 0, rng_)  # directly usable by the replay
    assert job["n_batches"] >= 1
