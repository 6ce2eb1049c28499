"""Sub-band I/Q outputs on the CPU: the kernel (rtlsdr-airband_b200/csrc/subband.cu) as the compiler built it, and the
filter design and frequency helpers of lib."""
import os
import re

import numpy as np
import pytest

from airband_b200 import lib

BUILD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rtlsdr-airband_b200", "build")


def test_kernel_builds_for_sm90a_without_spills():
    path = os.path.join(BUILD, "subband.ptxas.log")
    assert os.path.exists(path), f"{path} missing: build the library first (make -C rtlsdr-airband_b200)"
    with open(path) as f:
        log = f.read()
    assert "sm_90a" in log and "abg_subband_kernel" in log
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert spills and all(int(a) == 0 and int(b) == 0 for a, b in spills), spills
    regs = [int(r) for r in re.findall(r"Used (\d+) registers", log)]
    assert regs and max(regs) <= 128, regs  # __launch_bounds__(256, 2)


def _response_db(h, f, fs):
    w = np.exp(-2j * np.pi * np.outer(f / fs, np.arange(h.size)))
    return 20 * np.log10(np.abs(w @ h.astype(np.float64)) + 1e-300)


@pytest.mark.parametrize("n,cutoff,fs,atten", [(255, 10000.0, 2560000.0, 60.0), (127, 12500.0, 2048000.0, 40.0),
                                               (1023, 3000.0, 2400000.0, 80.0), (4096, 1000.0, 2560000.0, 70.0)])
def test_lowpass_has_unit_dc_gain_and_its_stopband(n, cutoff, fs, atten):
    h = lib.subband_lowpass(n, cutoff, fs, atten)
    assert h.dtype == np.float32 and h.shape == (n,)
    assert abs(float(np.sum(h.astype(np.float64))) - 1.0) <= 1e-6
    assert np.allclose(h, h[::-1])  # linear phase
    # Kaiser's estimate of the transition width for this length and attenuation, with 10 % room
    width = (atten - 7.95) / (14.36 * (n - 1)) * fs
    stop = np.linspace(cutoff + 1.1 * width, fs / 2, 4000)
    assert _response_db(h, stop, fs).max() <= -atten + 1.0
    passband = np.linspace(0.0, max(cutoff - 1.1 * width, 0.0), 200)
    assert np.abs(_response_db(h, passband, fs)).max() <= 0.1


def test_lowpass_rejects_bad_arguments():
    for args in ((0, 1000.0, 2.56e6), (4097, 1000.0, 2.56e6), (255, 0.0, 2.56e6), (255, 1.3e6, 2.56e6)):
        with pytest.raises(ValueError):
            lib.subband_lowpass(*args)
    assert np.array_equal(lib.subband_lowpass(1, 5000.0, 2.56e6), np.ones(1, np.float32))


def test_frequency_rounds_and_folds():
    fs = 2560000
    step = fs / 2 ** 32
    assert lib.subband_frequency(0.0, fs) == 0.0
    # multiples of the step are exact, and the result is delta * fs / 2^32
    assert lib.subband_frequency(12345 * step, fs) == 12345 * step
    assert lib.subband_frequency(-12345 * step, fs) == -12345 * step
    # llround: to the nearest step, halves away from zero
    assert lib.subband_frequency(7.4 * step, fs) == 7 * step
    assert lib.subband_frequency(7.6 * step, fs) == 8 * step
    assert lib.subband_frequency(2.5 * step, fs) == 3 * step
    assert lib.subband_frequency(-2.5 * step, fs) == -3 * step
    # +-fs/2 is delta = 2^31 either way, folded to -fs/2: the interval is [-fs/2, fs/2)
    assert lib.subband_frequency(fs / 2, fs) == -fs / 2
    assert lib.subband_frequency(-fs / 2, fs) == -fs / 2
    assert lib.subband_frequency(fs / 2 - step, fs) == fs / 2 - step
    # an arbitrary offset lands within half a step
    for f in (1000.3, -250000.77, 1279999.9):
        q = lib.subband_frequency(f, fs)
        assert abs(q - f) <= step / 2 and -fs / 2 <= q < fs / 2


def test_symbols_and_limits_match_the_header():
    hdr = open(os.path.join(os.path.dirname(BUILD), "..", "include", "airband_b200.h")).read()
    assert int(re.search(r"#define ABG_SUBBAND_MAX (\d+)", hdr).group(1)) == lib.SUBBAND_MAX
    assert int(re.search(r"#define ABG_SUBBAND_MAX_COEFFS (\d+)", hdr).group(1)) == lib.SUBBAND_MAX_COEFFS
    for s in ("abg_subband_configure", "abg_fetch_subband", "abg_debug_subband_time"):
        assert s in lib.SYMBOLS
