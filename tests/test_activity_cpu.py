"""CPU checks of the band activity detector: its C ABI against the header, the abg_burst layout against a ctypes mirror, the
per-batch piece rule (flags and in-kernel drop) merged by lib.merge_bursts against the batch-independent burst definition,
lib.activity_threshold and lib.group_transmissions on synthetic input, and the kernel's `-Xptxas -v` log (sm_90a, no spills
beyond the band spectrum's at the same fft_size)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from airband_b200 import lib
from airband_b200.config import AGC_EXTRA, Channel, Config, Device, SFMT_U8

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "rtlsdr-airband_b200")
HDR = open(os.path.join(ROOT, "include", "airband_b200.h")).read()
ACT_SYMBOLS = ["abg_activity_configure", "abg_fetch_activity", "abg_debug_activity_time"]


def test_symbols_and_constants_match_the_header():
    declared = set(re.findall(r"ABG_API\s+[\w\s\*]+?\b(abg_\w+)\s*\(", HDR))
    for s in ACT_SYMBOLS:
        assert s in declared and s in lib.SYMBOLS, s
    assert int(re.search(r"#define ABG_ACTIVITY_MAX_RECORDS (\d+)", HDR).group(1)) == lib.ACTIVITY_MAX_RECORDS == 4096
    assert int(re.search(r"ABG_BURST_OPEN_START = (\d+)", HDR).group(1)) == lib.BURST_OPEN_START == 1
    assert int(re.search(r"ABG_BURST_OPEN_END = (\d+)", HDR).group(1)) == lib.BURST_OPEN_END == 2


def test_symbols_are_exported():
    so = os.path.join(PKG, "libairband_b200.so")
    if not os.path.exists(so):
        pytest.skip("library not built")
    L = C.CDLL(so)
    for s in ACT_SYMBOLS:
        assert hasattr(L, s), s


def test_burst_layout():
    # the header's struct, field by field, against the ctypes mirror and the numpy dtype fetch_activity returns
    body = re.search(r"typedef struct abg_burst \{(.*?)\} abg_burst;", HDR, re.S).group(1)
    fields = re.findall(r"(int32_t|uint64_t|float)\s+([\w\s,]+);", body)
    names = [n.strip() for _, group in fields for n in group.split(",")]
    assert names == [f for f, _ in lib.CBurst._fields_]
    assert C.sizeof(lib.CBurst) == lib.BURST_DTYPE.itemsize == 40
    offsets = dict(bin=0, flags=4, first_frame=8, last_frame=16, n_active=24, peak=28, sum=32, reserved=36)
    for f, off in offsets.items():
        assert getattr(lib.CBurst, f).offset == off == lib.BURST_DTYPE.fields[f][1], f


# ---- the piece rule, modelled in numpy ---------------------------------------------------------------------------------
def _groups(idx, h):
    """Split sorted active indices into runs whose consecutive members are at most h + 1 apart."""
    out, cur = [], []
    for i in idx:
        if cur and i - cur[-1] > h + 1:
            out.append(cur)
            cur = []
        cur.append(i)
    if cur:
        out.append(cur)
    return out


def _rec(k, frames, powers, flags=0):
    s = np.float32(0.0)
    for p in powers:
        s = np.float32(s + np.float32(p))
    return (k, flags, frames[0], frames[-1], len(frames), np.float32(np.max(powers)), s, 0)


def model_pieces(P, thr, seq, B, s, h, m):
    """What the kernel emits for batch seq: P[n, K] powers of its selected frames, in the header's piece rule."""
    n = P.shape[0]
    recs = []
    for k in range(P.shape[1]):
        for g in _groups(np.flatnonzero(P[:, k] > thr[k]), h):
            flags = (lib.BURST_OPEN_START if g[0] <= h else 0) | (lib.BURST_OPEN_END if g[-1] >= n - 1 - h else 0)
            if flags == 0 and g[-1] - g[0] + 1 < m:
                continue
            frames = [AGC_EXTRA + seq * B + i * s for i in g]
            recs.append(_rec(k, frames, P[g, k], flags))
    return np.array(recs, lib.BURST_DTYPE) if recs else np.zeros(0, lib.BURST_DTYPE)


def global_bursts(P, thr, seq0, B, s, n, h, m):
    """The definition, independent of batches: P[Q, K] over the absolute selected index q - seq0 * n."""
    recs = []
    for k in range(P.shape[1]):
        for g in _groups(np.flatnonzero(P[:, k] > thr[k]), h):
            if g[-1] - g[0] + 1 < m:
                continue
            q = np.asarray(g) + seq0 * n
            frames = [AGC_EXTRA + (x // n) * B + (x % n) * s for x in q]
            recs.append(_rec(k, frames, P[g, k]))
    return np.array(recs, lib.BURST_DTYPE) if recs else np.zeros(0, lib.BURST_DTYPE)


def readings_of(P, thr, seq0, B, s, n, h, m):
    out = []
    for b in range(P.shape[0] // n):
        pcs = model_pieces(P[b * n:(b + 1) * n], thr, seq0 + b, B, s, h, m)
        out.append(dict(pieces=pcs, n_total=len(pcs), batch_seq=seq0 + b, settings=(s, h, m), wave_batch=B))
    return out


def check_merge(P, thr, seq0, B, s, n, h, m):
    want = global_bursts(P, thr, seq0, B, s, n, h, m)
    got = lib.merge_bursts(readings_of(P, thr, seq0, B, s, n, h, m))
    assert got.size == want.size, (got, want)
    for f in ("bin", "first_frame", "last_frame", "n_active", "peak"):
        assert np.array_equal(got[f], want[f]), f
    np.testing.assert_allclose(got["sum"], want["sum"], rtol=1e-5)
    return want.size


def test_merged_pieces_are_the_global_bursts_random():
    rng = np.random.default_rng(7)
    found = 0
    for trial in range(1500):
        s = int(rng.integers(1, 5))
        n = int(rng.integers(1, 13))
        B = max(1, n * s - int(rng.integers(0, s)))
        assert -(-B // s) == n
        h = int(rng.integers(0, n))
        if trial % 5 == 0:
            h = n - 1  # the largest hang allowed
        m = int(rng.integers(1, 2 * n + 3))
        nb = int(rng.integers(1, 7))
        K = 4
        density = rng.uniform(0.05, 0.8)
        P = rng.uniform(0.1, 10.0, (nb * n, K)).astype(np.float32)
        thr = np.full(K, np.float32(10.0 * (1.0 - density)) + np.float32(0.1), np.float32)
        found += check_merge(P, thr, int(rng.integers(0, 50)), B, s, n, h, m)
    assert found > 1000


def _activity(active_q, Q, K=1):
    P = np.full((Q, K), np.float32(0.5), np.float32)
    for q in active_q:
        P[q, 0] = np.float32(2.0 + q)
    return P


@pytest.mark.parametrize("h", [0, 1, 3])
def test_gap_of_h_plus_1_joins_and_h_plus_2_does_not_across_a_boundary(h):
    n, s = 8, 2
    B = n * s
    thr = np.array([1.0], np.float32)
    for last in range(n - 1 - h, n):  # the first piece's last frame among the OPEN_END positions
        for gap in (h + 1, h + 2):
            nxt = n + last - n + gap  # q of the next active frame
            if nxt < n or nxt >= 2 * n:
                continue
            P = _activity([0, last, nxt], 2 * n)
            got = lib.merge_bursts(readings_of(P, thr, 3, B, s, n, h, 1))
            want = global_bursts(P, thr, 3, B, s, n, h, 1)
            assert [tuple(r)[:5] for r in got] == [tuple(r)[:5] for r in want]
            # gap h+1 (or less) joins the frames at `last` and `nxt`
            joined = any(r["first_frame"] <= AGC_EXTRA + 3 * B + last * s and r["last_frame"] >= AGC_EXTRA + 4 * B + (nxt - n) * s for r in got)
            assert joined == (gap <= h + 1), (last, gap, got)
    check_merge(_activity([n - 1, n], 2 * n), thr, 0, B, s, n, h, 1)


def test_pieces_touching_both_edges_chain_over_batches():
    n, s, h = 6, 1, 2
    B = n
    thr = np.array([1.0], np.float32)
    q = [1, 4, 7, 10, 13, 16, 19]  # every piece of the middle batches is OPEN_START and OPEN_END
    P = _activity(q, 4 * n)
    rd = readings_of(P, thr, 0, B, s, n, h, 1)
    flags = [int(p["flags"]) for r in rd[1:3] for p in r["pieces"]]
    assert flags == [3, 3]
    got = lib.merge_bursts(rd)
    assert got.size == 1 and got[0]["n_active"] == len(q)
    assert got[0]["first_frame"] == AGC_EXTRA + 1 and got[0]["last_frame"] == AGC_EXTRA + 19
    # with h = n - 1, a whole empty batch between two frames still separates them
    P = _activity([n - 1, 2 * n], 3 * n)
    assert check_merge(P, thr, 0, B, s, n, n - 1, 1) == 2


def test_in_kernel_drop_and_min_span_after_joining():
    n, s, h, m = 10, 1, 1, 4
    thr = np.array([1.0], np.float32)
    P = _activity([4, 5], n)  # short, far from both edges: dropped in the kernel
    assert model_pieces(P, thr, 0, n, s, h, m).size == 0
    P = _activity([8, 9, 10, 11], 2 * n)  # two short OPEN pieces that join into a span of 4
    rd = readings_of(P, thr, 0, n, s, n, h, m)
    assert [len(r["pieces"]) for r in rd] == [1, 1]
    got = lib.merge_bursts(rd)
    assert got.size == 1 and got[0]["n_active"] == 4


def test_merge_raises_on_gap_settings_change_and_truncation():
    thr = np.array([1.0], np.float32)
    rd = readings_of(_activity([1, 5], 12), thr, 0, 4, 1, 4, 0, 1)
    lib.merge_bursts(rd)
    with pytest.raises(ValueError, match="gap"):
        lib.merge_bursts([rd[0], rd[2]])
    bad = dict(rd[1], settings=(1, 1, 1))
    with pytest.raises(ValueError, match="settings"):
        lib.merge_bursts([rd[0], bad])
    trunc = dict(rd[1], n_total=len(rd[1]["pieces"]) + 1)
    with pytest.raises(ValueError, match="truncated"):
        lib.merge_bursts([rd[0], trunc])
    assert lib.merge_bursts([]).size == 0


# ---- host helpers ------------------------------------------------------------------------------------------------------
def test_activity_threshold_follows_the_floor_and_the_edges():
    N = 1024
    k = np.fft.fftfreq(N) * N  # signed bin offsets in natural order
    floor = 1e-3 * (1.0 + 9.0 * (np.abs(k) > 400))  # a raised floor near the band edges
    power = floor.copy()
    power[[10, 11, 12, 300]] = 1.0  # carriers
    thr = lib.activity_threshold(np.stack([power, power]), 6.0, 8)
    assert thr.dtype == np.float32 and thr.shape == (N,) and np.all(thr > 0)
    assert np.all(power[[10, 11, 12, 300]] > thr[[10, 11, 12, 300]])
    quiet = np.ones(N, bool)
    quiet[[10, 11, 12, 300]] = False
    assert np.all(power[quiet] < thr[quiet])  # the roll-off near the edges does not fire
    np.testing.assert_allclose(thr[100], 1e-3 * 10 ** 0.6, rtol=1e-6)
    np.testing.assert_allclose(thr[N // 2], 1e-2 * 10 ** 0.6, rtol=1e-6)
    assert np.all(lib.activity_threshold(np.zeros(N), 3.0, 2) > 0)


def _cfg():
    ch = [Channel(bin=b) for b in (100, 2048 - 300)]
    return Config(fft_size=2048, wave_rate=8000, devices=[Device(sfmt=SFMT_U8, sample_rate=2_048_000, channels=ch)])


def _burst(k, f0, f1, s):
    return (k, 0, f0, f1, f1 - f0 + 1, s, s, 0)


def test_group_transmissions():
    cfg = _cfg()
    N, hop = 2048, cfg.hop(0)
    b = np.array([_burst(99, 500, 900, 1.0), _burst(100, 480, 910, 4.0), _burst(101, 520, 880, 1.0),  # channel at bin 100
                  _burst(2048 - 40, 2000, 2100, 1.0), _burst(2048 - 39, 2010, 2090, 1.0),        # unconfigured, 39.5 bins below
                  _burst(1023, 100, 200, 1.0), _burst(1024, 100, 200, 1.0),                       # opposite band edges
                  _burst(100, 1200, 1300, 1.0), _burst(102, 1200, 1300, 1.0)],                    # two bins apart
                 lib.BURST_DTYPE)
    tx = lib.group_transmissions(b, cfg, 0, centerfreq=120_000_000)
    assert len(tx) == 6
    t = {(x["bins"], x["first_frame"]): x for x in tx}
    a = t[((99, 101), 480)]
    assert a["monitored"] and a["n_bursts"] == 3 and a["last_frame"] == 910
    assert a["freq_hz"] == pytest.approx(120_000_000 + 100 * 1000)
    assert a["start_s"] == pytest.approx(480 * hop / 2_048_000) and a["end_s"] == pytest.approx(910 * hop / 2_048_000)
    c = t[((-40, -39), 2000)]
    assert not c["monitored"] and c["freq_hz"] == pytest.approx(120_000_000 - 39.5 * 1000)
    assert ((1023, 1023), 100) in t and ((-1024, -1024), 100) in t  # not adjacent in frequency
    assert ((100, 100), 1200) in t and ((102, 102), 1200) in t
    assert len(lib.group_transmissions(b, cfg, 0, max_bin_gap=2, centerfreq=120_000_000)) == 5
    # overlapping bins that do not overlap in time stay apart
    b2 = np.array([_burst(50, 0, 10, 1.0), _burst(51, 11, 20, 1.0)], lib.BURST_DTYPE)
    assert len(lib.group_transmissions(b2, cfg, 0)) == 2


# ---- build -------------------------------------------------------------------------------------------------------------
def _spills(log):
    out = {}
    for name, body in re.findall(r"Compiling entry function '(\w+)' for 'sm_90a'\n(.*?bytes spill loads)", log, re.S):
        a, b = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", body).groups()
        out[int(re.search(r"ILi(\d+)E", name).group(1))] = (int(a), int(b))
    return out


def test_kernel_build_is_sm90a_with_no_more_spills_than_the_spectrum():
    path = os.path.join(PKG, "build", "activity.ptxas.log")
    assert os.path.exists(path), f"{path} missing: build the library first (make -C rtlsdr-airband_b200)"
    log = open(path).read()
    entries = re.findall(r"Compiling entry function '(\w+)' for '(\w+)'", log)
    assert len(entries) == 6 and all("abg_activity_kernel" in e and a == "sm_90a" for e, a in entries), entries
    act = _spills(log)
    spec = _spills(open(os.path.join(PKG, "build", "spectrum.ptxas.log")).read())
    assert sorted(act) == sorted(spec) == list(range(8, 14))
    for logn in act:
        assert act[logn][0] <= spec[logn][0] and act[logn][1] <= spec[logn][1], (logn, act[logn], spec[logn])
