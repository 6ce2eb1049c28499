"""I/Q history (abg_history_configure / _range / _raw / _subband) on the GPU (-m gpu).

Raw captures must be the pushed bytes and the range must follow the ring model of test_history_cpu, for every format,
across the ring's wrap, after evictions, for several run sizes, push patterns and input buffers small enough to compact.
Sub-band captures must be bitwise equal to the live sub-band output of the same settings wherever that output had all its
taps, and within the sub-band's float64 bound.  Switching the history on must leave every other output and monitor
bit-identical.  End to end: the transmitters the activity detector finds are captured from before their first sample."""
import numpy as np
import pytest

from airband_b200 import config as cm
from airband_b200 import lib
from test_gpu_activity import _all_monitors, make_raw, one_device_cfg, same_audio
from test_gpu_activity import drive as drive_monitors
from test_gpu_subband import EPS, _three_format_case, lowpass, one_device, random_stream, reference
from test_history_cpu import ring_model

pytestmark = pytest.mark.gpu
AGC = cm.AGC_EXTRA
FORMATS = [("u8_hop313", cm.SFMT_U8, 0.0, 2500000), ("s8", cm.SFMT_S8, 0.0, 2560000), ("s16", cm.SFMT_S16, 32766.5, 2560000),
           ("f32", cm.SFMT_F32, 1.0, 2048000)]


def fmt_cfg(sfmt, fs, sr):
    cfg = one_device(sfmt, sr=sr, fullscale=fs)
    if sr == 2500000:
        assert cfg.hop(0) == 313 and (AGC * 313 * 2) % 16 == 8  # batches are not 16-byte aligned
    return cfg


def pieces(raw, batch_items, rng, lo=0.3, hi=1.0):
    """raw cut into pushes of lo..hi batches, whole I/Q pairs."""
    out, pos = [], 0
    while pos < raw.size:
        n = int(rng.uniform(lo, hi) * batch_items) & ~1
        out.append(raw[pos:pos + max(n, 2)])
        pos += max(n, 2)
    return out


def check_raw(e, m, raw, rng):
    first, end = e.history_range(0)
    assert (first, end) == (m.first, m.end)
    if first == end:
        return 0
    wins = [(first, end - first), (first, 1), (end - 1, 1)]
    for _ in range(3):
        a = int(rng.integers(first, end))
        wins.append((a, int(rng.integers(1, end - a + 1))))
    # a window across the wrap: from just before the ring's byte 0 onwards
    b0 = first * m.bpc % m.R
    wrap = first + (m.R - b0) // m.bpc
    if wrap - 5 >= first and wrap + 5 <= end:
        wins.append((wrap - 5, 10))
    crossed = 0
    for a, n in wins:
        got = e.history_raw(0, a, n)
        assert got.dtype == raw.dtype and np.array_equal(got.view(np.uint8), raw[2 * a:2 * (a + n)].view(np.uint8)), (a, n, first, end)
        crossed += (a * m.bpc % m.R) + n * m.bpc > m.R
    return crossed


# ---- 1. raw capture ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,sfmt,fs,sr", FORMATS, ids=[f[0] for f in FORMATS])
@pytest.mark.parametrize("nbmax,cap,split", [(4, 3, False), (1, 2, True), (2, 5, True), (3, 1, False)])
def test_raw_capture_is_the_pushed_bytes(name, sfmt, fs, sr, nbmax, cap, split):
    cfg = fmt_cfg(sfmt, fs, sr)
    nb = 9
    raw = random_stream(cfg, 0, nb, seed=sfmt * 7 + nbmax)
    rng = np.random.default_rng(nbmax * 10 + cap)
    e = lib.Engine(cfg, max_batches_per_run=nbmax, input_capacity_batches=nbmax + 2)
    m = ring_model(sfmt, cfg.hop(0), cfg.wave_batch)
    assert e.history_range(0) == (0, 0)
    e.history_configure(0, cap)
    m.configure(cap)
    batch_items = 2 * cfg.wave_batch * cfg.hop(0)
    pushes = pieces(raw, batch_items, rng) if split else [raw[i:i + nbmax * batch_items] for i in range(0, raw.size, nbmax * batch_items)]
    seq, crossed = 0, 0
    for p in pushes:
        e.push(0, p)
        while (n := e.run(-1)) > 0:
            m.append(seq, n, raw.view(np.uint8))
            seq += n
            crossed += check_raw(e, m, raw, rng)  # before any sync: the captures queue behind the run's append
            while e.fetch(0) is not None:
                pass
    assert seq == nb and crossed > 0
    assert e.history_range(0) == (m.first, m.end) and m.end - m.first == min(cap, nb) * cfg.wave_batch * cfg.hop(0)
    e.close()


# ---- 2. sub-band capture ----------------------------------------------------------------------------------------------------
SHAPES = [(0.2113, 32, 255), (-0.5, 997, 4096), (0.0371, 1, 64), (0.1, 10007, 33)]


@pytest.mark.parametrize("name,sfmt,fs,sr", FORMATS, ids=[f[0] for f in FORMATS])
@pytest.mark.parametrize("frac,decim,L", SHAPES, ids=[f"off{s[0]}_D{s[1]}_L{s[2]}" for s in SHAPES])
def test_subband_capture_equals_the_live_output(name, sfmt, fs, sr, frac, decim, L):
    cfg = fmt_cfg(sfmt, fs, sr)
    nb, cap = 6, 3
    raw = random_stream(cfg, 0, nb, seed=sfmt * 5 + decim)
    h = lowpass(L, sr) if L != 64 else np.random.default_rng(2).standard_normal(64).astype(np.float32)
    off = frac * sr
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=nb + 2)
    e.subband_configure(0, 0, off, decim, h)
    e.history_configure(0, cap)
    e.push(0, raw)
    live = {}
    while e.run(-1) > 0:
        while e.fetch(0) is not None:
            pass
        while (x := e.fetch_subband(0, 0)) is not None:
            y, _, m0 = x
            live.update(zip(range(m0, m0 + y.size), y))
    first, end = e.history_range(0)
    n = cfg.wave_batch * cfg.hop(0)
    assert end - first == cap * n and first > AGC * cfg.hop(0) + L
    m_lo, m_hi = -(-(first + L - 1) // decim), -(-end // decim)
    assert m_hi > m_lo
    got = e.history_subband(0, off, decim, h, m_lo, m_hi - m_lo)
    assert e.history_time()[1] > 0.0
    want = np.array([live[m] for m in range(m_lo, m_hi)], np.complex64)
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    # the window straddles the ring's wrap; computed in two pieces split there, it is the same again
    m = ring_model(sfmt, cfg.hop(0), cfg.wave_batch)
    m.configure(cap)
    wrap = first + (m.R - first * m.bpc % m.R) // m.bpc  # the sample at the ring's byte 0
    assert first < wrap < end
    mid = min(max(m_lo + 1, wrap // decim), m_hi - 1)
    a = e.history_subband(0, off, decim, h, m_lo, mid - m_lo)
    b = e.history_subband(0, off, decim, h, mid, m_hi - mid)
    assert np.array_equal(np.concatenate([a, b]).view(np.uint64), got.view(np.uint64))
    # against float64: every tap lies in the history, so the live output's start does not matter
    conv, vmax = reference(cfg, 0, raw, off, decim, h, AGC * cfg.hop(0))
    ref = conv[np.arange(m_lo, m_hi) * decim]
    bound = 8 * L * EPS * float(np.abs(h.astype(np.float64)).sum()) * vmax
    assert np.abs(got.astype(np.complex128) - ref).max() <= bound
    e.close()


# ---- 3. range and contract ---------------------------------------------------------------------------------------------------
def test_range_starts_after_switch_on_and_capacity_changes_empty_it():
    cfg = fmt_cfg(cm.SFMT_U8, 0.0, 2560000)
    hop, B = cfg.hop(0), cfg.wave_batch
    raw = random_stream(cfg, 0, 8, seed=1)
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=10)
    e.push(0, raw)
    assert e.run(2) == 2 and e.history_range(0) == (0, 0)
    e.history_configure(0, 4)
    assert e.history_range(0) == (0, 0)
    assert e.run(1) == 1
    s2 = (AGC + 2 * B) * hop
    assert e.history_range(0) == (s2, s2 + B * hop)
    e.history_configure(0, 4)  # the same capacity: nothing changes
    assert e.history_range(0) == (s2, s2 + B * hop)
    e.history_configure(0, 2)  # another capacity: empty
    assert e.history_range(0) == (0, 0)
    assert e.run(2) == 2
    s3 = (AGC + 3 * B) * hop
    assert e.history_range(0) == (s3, s3 + 2 * B * hop)
    assert np.array_equal(e.history_raw(0, s3, 2 * B * hop), raw[2 * s3:2 * (s3 + 2 * B * hop)])
    e.history_configure(0, 0)
    assert e.history_range(0) == (0, 0)
    with pytest.raises(lib.AbgError) as ex:
        e.history_raw(0, s3, 1)
    assert ex.value.code == -5
    e.close()


def test_launches_resident_and_injected():
    cfg, raws = _three_format_case(nb=4)[:2]
    counts = {}
    for setup in ("untouched", "on_then_off", "on"):
        e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=6)
        if setup != "untouched":
            for d in range(3):
                e.history_configure(d, 3)
        if setup == "on_then_off":
            for d in range(3):
                e.history_configure(d, 0)
        for d in range(3):
            e.push(d, raws[d])
        per = []
        for _ in range(2):
            l0 = e.launch_count()
            assert e.run(2) == 6
            e.sync()
            per.append(e.launch_count() - l0)
            for d in range(3):
                while e.fetch(d) is not None:
                    pass
        counts[setup] = per
        assert (e.history_time()[0] > 0.0) == (setup == "on")
        e.close()
    assert counts["untouched"] == counts["on_then_off"]
    assert [a + 2 for a in counts["untouched"]] == counts["on"]
    # resident runs append (and take time) but leave the history empty
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=6)
    for d in range(3):
        e.history_configure(d, 3)
        e.resident_load(d, raws[d][:e.resident_bytes_needed(d) // raws[d].itemsize])
    e.run_resident(2)
    e.sync()
    assert e.history_time()[0] > 0.0
    assert all(e.history_range(d) == (0, 0) for d in range(3))
    e.close()
    # injected batches append nothing
    cfg2 = cm.Config(fft_size=cfg.fft_size, wave_rate=cfg.wave_rate, devices=[cfg.devices[0], cfg.devices[0]])
    e = lib.Engine(cfg2, max_batches_per_run=2, input_capacity_batches=6)
    e.history_configure(1, 3)
    l0 = e.launch_count()
    assert e.inject_wavein(1, np.full((1, 2 * e.B), 0.01, np.float32)) == 2
    e.sync()
    assert e.history_range(1) == (0, 0) and e.history_time()[0] == 0.0
    e.history_configure(1, 0)
    l1 = e.launch_count()
    assert e.inject_wavein(1, np.full((1, 2 * e.B), 0.01, np.float32)) == 2
    e.sync()
    assert e.launch_count() - l1 == l1 - l0  # the same launches with the history on and off
    e.close()


def test_error_codes():
    cfg = fmt_cfg(cm.SFMT_S16, 32766.5, 2560000)
    sr, hop, B = 2560000, cfg.hop(0), cfg.wave_batch
    raw = random_stream(cfg, 0, 3, seed=9)
    e = lib.Engine(cfg, max_batches_per_run=3, input_capacity_batches=5)
    h = lowpass(63, sr)

    def code(f, *a):
        with pytest.raises(lib.AbgError) as ex:
            f(*a)
        return ex.value.code

    assert code(e.history_configure, 1, 2) == -5 and code(e.history_configure, -1, 2) == -5
    assert code(e.history_configure, 0, -1) == -2
    assert code(e.history_range, 3) == -5
    assert code(e.history_raw, 0, 0, 1) == -5  # empty
    assert code(e.history_subband, 0, 0.0, 8, h, 1000, 1) == -5
    e.history_configure(0, 3)
    e.push(0, raw)
    assert e.run(-1) == 3
    first, end = e.history_range(0)
    assert (first, end) == (AGC * hop, (AGC + 3 * B) * hop)
    # raw: one sample outside either end
    assert code(e.history_raw, 0, first - 1, 1) == -5 and code(e.history_raw, 0, end - 1, 2) == -5
    assert code(e.history_raw, 0, first, -1) == -2 and code(e.history_raw, 1, first, 1) == -5
    assert e.history_raw(0, first, end - first).size == 2 * (end - first)
    # sub-band at decimation 1: the first output's oldest tap at first, the last output's newest at end - 1, then one
    # sample further on either side
    L = 63
    m0, mlast = first + L - 1, end - 1
    assert e.history_subband(0, 0.0, 1, h, m0, mlast - m0 + 1).size == mlast - m0 + 1
    assert code(e.history_subband, 0, 0.0, 1, h, m0 - 1, 1) == -5
    assert code(e.history_subband, 0, 0.0, 1, lowpass(64, sr), m0, 1) == -5  # one tap more
    assert code(e.history_subband, 0, 0.0, 1, h, mlast, 2) == -5
    D = 8
    # arguments abg_subband_configure refuses
    for args in ((0.0, 0, h), (0.0, B * hop + 1, h), (sr / 2 + 1, D, h), (float("nan"), D, h), (0.0, D, np.zeros(0, np.float32)),
                 (0.0, D, np.ones(4097, np.float32)), (0.0, D, np.array([1.0, np.inf], np.float32))):
        assert code(e.history_subband, 0, *args, m0, 1) == -2, args
    assert code(e.history_subband, 0, 0.0, D, h, m0, 0) == -2
    assert code(e.history_subband, 5, 0.0, D, h, m0, 1) == -5
    e.close()


# ---- 4. nothing else changes -------------------------------------------------------------------------------------------------
def test_outputs_and_monitors_unchanged_with_history_on():
    cfg, raws, _ = _three_format_case(nb=4)
    thr = np.full(cfg.fft_size, 40.0, np.float32)

    def monitors(e):
        for d in range(3):
            _all_monitors(e, cfg, d)
            e.activity_configure(d, lib.default_stride(cfg, d), 1, 2, thr)

    def with_history(e):
        monitors(e)
        e.history_configure(0, 2)
        e.history_configure(2, 5)

    for nbmax in (4, 1):
        off, e = drive_monitors(cfg, raws, monitors, nbmax=nbmax)
        e.close()
        on, e = drive_monitors(cfg, raws, with_history, nbmax=nbmax, pushes=None)
        assert e.history_range(1) == (0, 0) and e.history_range(0)[1] > e.history_range(0)[0]
        first, end = e.history_range(2)
        assert np.array_equal(e.history_raw(2, first, end - first).view(np.uint8), raws[2][2 * first:2 * end].view(np.uint8))
        e.close()
        same_audio(off, on)
        assert off["mon"] == on["mon"] and all(len(m) > 0 for m in on["mon"])
        # a truncated reading stores an unspecified subset of its pieces (airband_b200.h): compare its count only
        key = lambda act: [[(r["batch_seq"], r["n_total"], r["pieces"].tobytes() if r["n_total"] <= len(r["pieces"]) else None)  # noqa: E731
                            for r in a] for a in act]
        assert key(off["act"]) == key(on["act"])
        assert any(r["n_total"] <= len(r["pieces"]) and len(r["pieces"]) > 0 for a in on["act"] for r in a)


# ---- 5. end to end ---------------------------------------------------------------------------------------------------------------
def test_detect_then_capture_unconfigured_transmitters_from_before_their_onset():
    SR, W, n, cf = 2048000, 8000, 2048, 120_000_000
    bw = SR // n
    chan_off = [-600, -450, -300, -150, 150, 300, 450, 600]
    chans = [cm.make_channel(cf + k * bw + bw // 2, cf, SR, n, W) for k in chan_off]
    cfg = one_device_cfg(n, cm.SFMT_U8, chans, centerfreq=cf)
    B, hop, nb = cfg.wave_batch, cfg.hop(0), 6
    n_samples = (AGC + nb * B) * hop + n
    f2s = lambda f: int(f * hop)  # noqa: E731
    extra = [(-222, AGC + 3 * B + 300, AGC + 3 * B + 460), (77, AGC + B + 100, AGC + 4 * B + 100), (512, AGC + 4 * B + 900, AGC + 5 * B + 200)]
    A = 0.04
    tones = [(k * bw + bw / 2, A, [(0, n_samples)]) for k in chan_off]
    tones += [(k * bw, A, [(f2s(a), f2s(b))]) for k, a, b in extra]
    raw = make_raw(cfg, 0, n_samples, tones, noise=0.01, seed=1)
    s = lib.default_stride(cfg, 0)

    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=nb + 2)
    e.history_configure(0, 8)
    e.push(0, raw)
    e.spectrum_configure(0, s)
    assert e.run(1) == 1
    thr = lib.activity_threshold(e.fetch_spectrum(0)[0], 13.0, 16)
    e.spectrum_configure(0, 0)
    e.activity_configure(0, s, 1, 2, thr)
    rd = []
    while True:
        while e.fetch(0) is not None:
            pass
        while (r := e.fetch_activity(0)) is not None:
            rd.append(r)
        if e.run(-1) == 0:
            break
    hist = e.history_range(0)
    assert hist == (AGC * hop, (AGC + nb * B) * hop)
    tx = lib.group_transmissions(lib.merge_bursts(rd), cfg, 0)
    D, L = 32, 255
    h = lib.subband_lowpass(L, 5000.0, SR, 60.0)
    gain = float(np.sum(h.astype(np.float64)))
    for k, a, b in extra:
        hit = [t for t in tx if abs(t["freq_hz"] - (cf + k * bw)) <= bw and not t["monitored"]]
        assert len(hit) == 1, k
        off, m0, cnt = lib.transmission_capture(hit[0], cfg, 0, hist, D, L, pad_s=0.05)
        onset = f2s(a)
        # 50 ms before the onset, up to the detector's frame resolution (one stride of frames)
        assert m0 * D <= onset - 0.05 * SR + s * hop, (k, m0 * D, onset)
        y = e.history_subband(0, off, D, h, m0, cnt)
        env = np.abs(y)
        mm = m0 + np.arange(cnt)
        assert env[mm * D < onset].max() < 0.25 * A * gain  # nothing of it before its first sample
        rise = m0 + int(np.argmax(env > 0.5 * A * gain))
        assert abs(rise * D - onset) <= L + D, (k, rise * D, onset)
        steady = y[rise - m0 + L // D + 1:rise - m0 + L // D + 801]
        f = np.median(np.angle(steady[1:] * np.conj(steady[:-1]))) * (SR / D) / (2 * np.pi)
        assert abs(f) <= bw, (k, f)
    e.close()
