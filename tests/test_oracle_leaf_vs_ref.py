"""Pins the restated leaf DSP (oracle/leaf_dsp.cpp) against the reference's OWN squelch.cpp / ctcss.cpp /
filters.cpp compiled in place (oracle/_ref/libairband_ref.so): identical inputs must give bit-identical traces.
Where oracle/_ref has not been built, the comparison is with the SHA-256 of the reference's outputs stored in
tests/golden/ref_leaf.npz (made from it by tests/golden/make_golden.py); where it has, with both."""
import hashlib
import os

import numpy as np
import pytest

import oracle_py as op

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_leaf.npz")
SQUELCH_CASES = [(mode, seed) for seed in (1, 2, 3) for mode in ("auto", "manual", "snr0", "snr20")]
NOTCH_CASES = [(8000, 100.0, 10.0), (16000, 100.0, 10.0), (8000, 123.0, 5.0), (16000, 254.1, 20.0)]
LOWPASS_CASES = [(8000, 2500.0), (16000, 2500.0), (16000, 6250.0), (8000, 1000.0)]
CTCSS_CASES = [(rate, tone) for tone in (67.0, 100.0, 151.4, 254.1, 88.0) for rate in (8000, 16000)]


def digest(a) -> np.ndarray:
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def assert_bit_identical_to_reference(key: str, got, compute):
    """`got` must equal, bit for bit, the reference leaf classes' output for the case: live from oracle/_ref when it is
    built, and always the SHA-256 of that output stored in tests/golden/ref_leaf.npz."""
    got = np.ascontiguousarray(got)
    if op.available("ref"):
        want = np.ascontiguousarray(compute())
        assert got.dtype == want.dtype and got.shape == want.shape and np.array_equal(got.view(np.uint8), want.view(np.uint8)), key
    assert np.array_equal(digest(got), np.load(GOLDEN)[key]), f"{key} differs from the reference's stored output"


def keyed_levels(n, seed, lo=0.05, hi=0.75, jitter=0.3):
    rng = np.random.default_rng(seed)
    x = np.empty(n, np.float32)
    i = 0
    on = False
    while i < n:
        seg = int(rng.integers(50, 3000))
        base = hi if on else lo
        x[i:i + seg] = base * (1.0 + jitter * rng.standard_normal(min(seg, n - i)))
        i += seg
        on = not on
    return np.abs(x).astype(np.float32)


def squelch_run(mode, seed, variant):
    """(levels float32, flags, counts int64[4]) of one squelch trace."""
    raw = keyed_levels(60000, seed)
    # a filtered stream that sometimes falls below the buffered pre-filter level (exercises the post-filter path)
    rng = np.random.default_rng(100 + seed)
    filt = (raw * rng.uniform(0.3, 1.2, raw.size)).astype(np.float32)
    audio = (0.2 * np.sin(2 * np.pi * 100.0 * np.arange(raw.size) / 8000.0)).astype(np.float32)
    s = op.SquelchHarness(variant)
    if mode == "manual":
        s.set_level(0.3)
    elif mode == "snr0":
        s.set_snr(0.0)
    elif mode == "snr20":
        s.set_snr(20.0)
    if seed == 2:
        s.set_ctcss(100.0, 8000.0)
    use_filt = filt if seed != 1 else None
    lv, fl = s.trace(raw, use_filt, audio)
    return lv, fl, np.array([s.open_count(), s.flappy_count(), s.ctcss_count(), s.no_ctcss_count()], np.int64)


def notch_input():
    return np.random.default_rng(5).standard_normal(20000).astype(np.float32) * 0.3


def lowpass_input():
    rng = np.random.default_rng(6)
    return (rng.standard_normal(20000) + 1j * rng.standard_normal(20000)).astype(np.complex64)


def ctcss_run(rate, tone, variant):
    """int64 [2 windows][n + 1][2]: (enough, has_tone) after every sample, then (found, not_found)."""
    n = int(rate * 0.4) * 3 + 17
    rng = np.random.default_rng(7)
    x = (0.2 * np.sin(2 * np.pi * tone * np.arange(n) / rate) + 0.02 * rng.standard_normal(n)).astype(np.float32)
    out = []
    for win in (int(rate * 0.05), int(rate * 0.4)):
        c = op.CtcssHarness(tone, rate, win, variant)
        seq = []
        for v in x:
            c.sample(float(v))
            seq.append((c.enough(), c.has_tone()))
        seq.append((int(c.L.abo_ctcss_found(c.c)), int(c.L.abo_ctcss_not_found(c.c))))
        out.append(seq)
    return np.array(out, np.int64)


def reference_outputs() -> dict:
    """Every reference output these tests compare with (tests/golden/make_golden.py stores their SHA-256)."""
    out = {}
    for mode, seed in SQUELCH_CASES:
        lv, fl, cnt = squelch_run(mode, seed, "ref")
        out[f"squelch_{mode}_{seed}_levels"], out[f"squelch_{mode}_{seed}_flags"], out[f"squelch_{mode}_{seed}_counts"] = lv, fl, cnt
    for rate, freq, q in NOTCH_CASES:
        out[f"notch_{rate}_{freq}_{q}"] = op.notch_run(freq, rate, q, notch_input(), "ref")
    for rate, freq in LOWPASS_CASES:
        out[f"lowpass_{rate}_{freq}"] = op.lowpass_run(freq, rate, lowpass_input(), "ref")
    for rate, tone in CTCSS_CASES:
        out[f"ctcss_{rate}_{tone}"] = ctcss_run(rate, tone, "ref")
    return out


@pytest.mark.parametrize("mode", ["auto", "manual", "snr0", "snr20"])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_squelch_trace_bit_identical(mode, seed):
    got = squelch_run(mode, seed, "restated")
    ref = squelch_run(mode, seed, "ref") if op.available("ref") else None
    for k, part in enumerate(("levels", "flags", "counts")):
        assert_bit_identical_to_reference(f"squelch_{mode}_{seed}_{part}", got[k], lambda: ref[k])
    assert got[1].max() > 0, "trace never opened — test signal is not exercising the state machine"


@pytest.mark.parametrize("rate,freq,q", [(8000, 100.0, 10.0), (16000, 100.0, 10.0), (8000, 123.0, 5.0), (16000, 254.1, 20.0)])
def test_notch_bit_identical(rate, freq, q):
    a = op.notch_run(freq, rate, q, notch_input(), "restated")
    assert_bit_identical_to_reference(f"notch_{rate}_{freq}_{q}", a, lambda: op.notch_run(freq, rate, q, notch_input(), "ref"))
    assert np.abs(a).max() > 0


@pytest.mark.parametrize("rate,freq", [(8000, 2500.0), (16000, 2500.0), (16000, 6250.0), (8000, 1000.0)])
def test_lowpass_bit_identical(rate, freq):
    a = op.lowpass_run(freq, rate, lowpass_input(), "restated")
    assert_bit_identical_to_reference(f"lowpass_{rate}_{freq}", a, lambda: op.lowpass_run(freq, rate, lowpass_input(), "ref"))


@pytest.mark.parametrize("rate", [8000, 16000])
@pytest.mark.parametrize("tone", [67.0, 100.0, 151.4, 254.1, 88.0])
def test_ctcss_bit_identical(rate, tone):
    a = ctcss_run(rate, tone, "restated")
    assert_bit_identical_to_reference(f"ctcss_{rate}_{tone}", a, lambda: ctcss_run(rate, tone, "ref"))
