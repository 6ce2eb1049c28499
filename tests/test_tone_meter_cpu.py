"""CPU checks of the CTCSS tone meter: its C ABI against the header, the default tone list against the engine's, lib's
tone_powers / ctcss_identify / tone_meter_frequency on readings synthesised in numpy with the header's definition, and the
kernel's `-Xptxas -v` log (sm_90a, no spills)."""
import os
import re

import numpy as np
import pytest

from airband_b200 import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "rtlsdr-airband_b200")
HDR = open(os.path.join(ROOT, "include", "airband_b200.h")).read()
TM_SYMBOLS = ["abg_tone_meter_configure", "abg_tone_meter_set_tones", "abg_fetch_tone_meter", "abg_debug_tone_meter_time"]


def test_symbols_and_tone_max_match_the_header():
    declared = set(re.findall(r"ABG_API\s+[\w\s\*]+?\b(abg_\w+)\s*\(", HDR))
    for s in TM_SYMBOLS:
        assert s in declared and s in lib.SYMBOLS, s
    assert int(re.search(r"#define ABG_TONE_MAX (\d+)", HDR).group(1)) == lib.TONE_MAX == 64


def test_standard_tones_are_the_engines():
    src = open(os.path.join(PKG, "csrc", "engine.cu")).read()
    body = re.search(r"const float kStandardTones\[51\] = \{(.*?)\};", src, re.S).group(1)
    engine = [float(x) for x in re.findall(r"[\d.]+", body)]
    assert len(engine) == 51 and tuple(engine) == lib.STANDARD_TONES


def delta(f, wave_rate):
    return int(np.floor(float(np.float32(f)) / wave_rate * 2.0 ** 32 + 0.5)) % (1 << 32)


def readings(y, tones, wave_rate, B, a0=0):
    """The definition in float64: per batch a of y[C, n] (n a multiple of B), (S[C, K], E[C], active[C], a)."""
    out = []
    d = np.array([delta(f, wave_rate) for f in tones], np.uint64)
    for b in range(y.shape[1] // B):
        a = a0 + b
        idx = (a * B + np.arange(B, dtype=np.uint64)).astype(np.uint64)
        ph = (d[None, :] * idx[:, None]) % np.uint64(1 << 32)  # exact: products stay below 2^64
        turns = ph.astype(np.float64) / 2.0 ** 32
        yb = y[:, b * B:(b + 1) * B].astype(np.float64)
        S = yb @ np.exp(-2j * np.pi * turns)
        out.append((S.astype(np.complex64), (yb ** 2).sum(1).astype(np.float32), np.count_nonzero(yb, 1).astype(np.int32), a))
    return out


def test_tone_meter_frequency():
    for wr in (8000, 16000):
        for f in lib.STANDARD_TONES:
            q = lib.tone_meter_frequency(f, wr)
            assert q == delta(f, wr) * wr / 2.0 ** 32
            assert abs(q - f) <= wr / 2.0 ** 33 + 1e-5  # half a step of the phase, plus float32 rounding of f


def test_a_pure_tone_reads_one_and_its_neighbours_little():
    wr, B = 8000, 1000
    n = 4 * B
    t = np.arange(3 * B, 3 * B + n)  # batches 3..6: the phase is that of the absolute index
    for k in (0, 1, 12, 50):
        f = lib.tone_meter_frequency(lib.STANDARD_TONES[k], wr)
        y = 0.3 * np.cos(2 * np.pi * f * t / wr + 0.7)
        r = readings(y[None, :], lib.STANDARD_TONES, wr, B, a0=3)
        share = lib.tone_powers(r)
        assert share.shape == (1, 51)
        assert abs(share[0, k] - 1.0) < 0.02, share[0, k]
        others = np.delete(share[0], k)
        assert others.max() < 0.1, others.max()  # 67.0 / 69.3 Hz: 1.15 bins of a 0.5 s window apart
        assert lib.ctcss_identify(r)[0] == (lib.STANDARD_TONES[k], pytest.approx(share[0, k]))
        # |S| = A n / 2 for the summed window
        S = sum(x[0][0, k] for x in r)
        assert abs(abs(S) - 0.3 * n / 2) < 0.01 * 0.3 * n


def test_channels_and_noise():
    wr, B = 16000, 2000
    rng = np.random.default_rng(5)
    n = 4 * B
    t = np.arange(n)
    y = np.stack([0.2 * np.sin(2 * np.pi * lib.tone_meter_frequency(100.0, wr) * t / wr) + rng.normal(0, 0.1, n),
                  rng.normal(0, 0.1, n),
                  np.zeros(n),
                  np.sin(2 * np.pi * 1000.0 * t / wr) + 0.1 * np.sin(2 * np.pi * lib.tone_meter_frequency(67.0, wr) * t / wr)])
    r = readings(y, lib.STANDARD_TONES, wr, B)
    got = lib.ctcss_identify(r, min_share=0.005)
    assert got[0][0] == 100.0 and 0.5 < got[0][1] < 0.8  # 0.02 of 0.03 in the tone
    assert got[1] is None and got[2] is None              # noise alone and silence
    assert got[3][0] == 67.0 and 0.005 < got[3][1] < 0.02
    assert np.all(lib.tone_powers(r)[2] == 0.0)
    # a tone outside the standard list, through a list of its own
    tones = [123.4, 97.4]
    y2 = np.cos(2 * np.pi * lib.tone_meter_frequency(123.4, wr) * t / wr)[None, :]
    assert lib.ctcss_identify(readings(y2, tones, wr, B), tones=tones)[0][0] == 123.4
    with pytest.raises(ValueError):
        lib.ctcss_identify(readings(y2, tones, wr, B))  # 2 tones read, 51 named


def test_squelch_gaps_do_not_dilute_the_share():
    wr, B = 8000, 1000
    t = np.arange(4 * B)
    y = np.cos(2 * np.pi * lib.tone_meter_frequency(131.8, wr) * t / wr)
    y[:1500] = 0.0  # squelch closed for the first 1.5 batches
    share = lib.tone_powers(readings(y[None, :], lib.STANDARD_TONES, wr, B))
    assert abs(share[0, lib.STANDARD_TONES.index(131.8)] - 1.0) < 0.02


def test_gaps_and_tone_count_changes_raise():
    wr, B = 8000, 1000
    y = np.random.default_rng(1).normal(0, 0.1, (2, 3 * B))
    r = readings(y, lib.STANDARD_TONES, wr, B)
    lib.tone_powers(r)
    with pytest.raises(ValueError, match="gap"):
        lib.tone_powers([r[0], r[2]])
    r2 = readings(y[:, B:2 * B], lib.STANDARD_TONES[:10], wr, B, a0=1)
    with pytest.raises(ValueError, match="tones"):
        lib.tone_powers([r[0], r2[0]])
    with pytest.raises(ValueError):
        lib.tone_powers([])


def test_kernel_build_is_sm90a_without_spills():
    path = os.path.join(PKG, "build", "tone_meter.ptxas.log")
    assert os.path.exists(path), f"{path} missing: build the library first (make -C rtlsdr-airband_b200)"
    log = open(path).read()
    entries = re.findall(r"Compiling entry function '(\w+)' for '(\w+)'", log)
    assert len(entries) == 1 and "abg_tone_meter_kernel" in entries[0][0] and entries[0][1] == "sm_90a", entries
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert spills and all(int(a) == 0 and int(b) == 0 for a, b in spills), spills
    regs = [int(r) for r in re.findall(r"Used (\d+) registers", log)]
    assert regs and max(regs) * 256 * 2 <= 65536, regs  # two 256-thread CTAs per SM
