"""Band activity detector (abg_activity_configure / abg_fetch_activity) on the GPU (-m gpu).

Reference: the powers of every selected frame in float64 (test_tc_dft_math.reference_frame and numpy's FFT), thresholds
chosen so that no frame lies near its threshold, and the numpy piece model of test_activity_cpu on that float64 active set.
Switching the detector on must leave every other output and monitor bit-identical, and readings must not depend on how
batches are grouped into runs."""
import numpy as np
import pytest

from airband_b200 import config as cm
from airband_b200 import lib
from test_activity_cpu import model_pieces
from test_tc_dft_math import reference_frame

pytestmark = pytest.mark.gpu
AGC = cm.AGC_EXTRA
SR, W = 2048000, 8000
STAT_FIELDS = [f for f, _ in cm.CSquelchStats._fields_]


def quantize(x, sfmt, fullscale):
    v = np.empty(2 * x.size, np.float64)
    v[0::2], v[1::2] = x.real, x.imag
    if sfmt == cm.SFMT_U8:
        return np.clip(np.round(v * 127.5 + 127.5), 0, 255).astype(np.uint8)
    if sfmt == cm.SFMT_S8:
        return np.clip(np.round(v * 128.0), -128, 127).astype(np.int8)
    if sfmt == cm.SFMT_S16:
        return np.clip(np.round(v * fullscale), -32768, 32767).astype(np.int16)
    return (v * fullscale).astype(np.float32)


def make_raw(cfg, dev, n_samples, tones, noise=0.02, seed=0):
    """Complex noise plus gated tones: tones = [(offset_hz, amplitude, [(first sample, end sample), ...])]."""
    d = cfg.devices[dev]
    rng = np.random.default_rng(seed)
    x = rng.normal(0, noise, n_samples) + 1j * rng.normal(0, noise, n_samples)
    t = np.arange(n_samples)
    for f, a, gates in tones:
        for s0, s1 in gates:
            x[s0:s1] += a * np.exp(2j * np.pi * f * t[s0:s1] / d.sample_rate)
    return quantize(x, d.sfmt, d.fullscale)


def frame_powers(cfg, dev, raw, batch, stride):
    """float64 p[n, N] of the selected frames of one batch."""
    d = cfg.devices[dev]
    N, B, hop = cfg.fft_size, cfg.wave_batch, cfg.hop(dev)
    by = raw.view(np.uint8)
    bpc = 2 * d.bytes_per_sample
    rows = np.stack([by[(AGC + batch * B + j) * hop * bpc:((AGC + batch * B + j) * hop + N) * bpc] for j in range(0, B, stride)])
    out = np.empty((rows.shape[0], N))
    for i in range(0, rows.shape[0], 128):
        out[i:i + 128] = np.abs(np.fft.fft(reference_frame(rows[i:i + 128], d.sfmt, N, d.fullscale), axis=1)) ** 2
    return out


def margin_ok(P, thr, pmax):
    return np.abs(P - thr) > 1e-3 * thr + 2e-5 * pmax


def pick_thresholds(P, pmax, tone_bins):
    """Per bin: the log-midpoint of the widest gap between its sorted powers that keeps every frame clear of it (tone bins:
    any gap; other bins: gaps in the top 1 %, so that the noise gives a few short bursts)."""
    N = P.shape[1]
    thr = np.empty(N, np.float32)
    for k in range(N):
        v = np.sort(P[:, k])
        lo = 0 if k in tone_bins else min(int(0.99 * v.size), max(v.size - 2, 0))
        lv = np.log(v[lo:])
        gaps = np.argsort(np.diff(lv))[::-1]
        cands = [np.float32(np.exp(0.5 * (lv[g] + lv[g + 1]))) for g in gaps[:8]] + [np.float32(4.0 * v[-1] + 1e-4 * pmax)]
        for t in cands:  # the last resort, above every frame, leaves the bin quiet
            if np.all(margin_ok(P[:, k], float(t), pmax)):
                thr[k] = t
                break
        else:
            raise AssertionError(f"no clear threshold for bin {k}")
    return thr


def drive(cfg, raws, setup, nbmax=2, fft_mode=0, pushes=None):
    """Push every stream (whole, or in `pushes` pieces with runs between), run to exhaustion, fetch everything."""
    total = max(r.size // (2 * cfg.hop(d)) // cfg.wave_batch for d, r in enumerate(raws)) + 2
    e = lib.Engine(cfg, max_batches_per_run=nbmax, input_capacity_batches=total, fft_mode=fft_mode)
    setup(e)
    D = len(cfg.devices)
    out = dict(audio=[[] for _ in range(D)], act=[[] for _ in range(D)], mon=[[] for _ in range(D)])

    def drain():
        for d in range(D):
            while (g := e.fetch(d)) is not None:
                out["audio"][d].append(g)
            while (a := e.fetch_activity(d)) is not None:
                out["act"][d].append(a)
            out["mon"][d].extend(fetch_monitors(e, d))

    if pushes is None:
        for d, r in enumerate(raws):
            e.push(d, r)
    else:
        cut = lambda r, x: (x * r.size // pushes[-1][1]) & ~1  # noqa: E731  (whole I/Q pairs)
        for lo, hi in pushes:
            for d, r in enumerate(raws):
                e.push(d, r[cut(r, lo):cut(r, hi)])
            e.run(-1)
            drain()
    while e.run(-1) > 0:
        drain()
    drain()
    out["stats"] = [[tuple(getattr(e.stats(d, c), f) for f in STAT_FIELDS) for c in range(len(cfg.devices[d].channels))] for d in range(D)]
    return out, e


def fetch_monitors(e, d):
    got = []
    while (s := e.fetch_spectrum(d)) is not None:
        got.append(("spec", s[1], s[0].tobytes()))
    while (c := e.fetch_carrier(d)) is not None:
        got.append(("car", c[2], c[0].tobytes() + c[1].tobytes()))
    while (x := e.fetch_input_levels(d)) is not None:
        got.append(("inm", x["batch_seq"], repr({k: (v.tobytes() if hasattr(v, "tobytes") else v) for k, v in x.items()})))
    for k in range(2):
        while (x := e.fetch_subband(d, k)) is not None:
            got.append(("sb%d" % k, x[1], x[0].tobytes()))
    while (t := e.fetch_tone_meter(d)) is not None:
        got.append(("tm", t[3], t[0].tobytes() + t[1].tobytes() + t[2].tobytes()))
    return got


def act_key(readings):
    return [(r["batch_seq"], r["n_total"], r["settings"], r["pieces"].tobytes()) for r in readings]


def same_audio(a, b):
    for d in range(len(a["audio"])):
        assert len(a["audio"][d]) == len(b["audio"][d]) > 0
        for (w1, i1, x1), (w2, i2, x2) in zip(a["audio"][d], b["audio"][d]):
            assert np.array_equal(w1.view(np.uint32), w2.view(np.uint32))
            assert np.array_equal(i1.view(np.uint64), i2.view(np.uint64))
            assert np.array_equal(x1, x2)
    assert a["stats"] == b["stats"]


def one_device_cfg(n, sfmt, channels=None, centerfreq=0):
    ch = channels if channels is not None else [cm.make_channel(96060, 0, SR, n, W)]
    return cm.Config(fft_size=n, wave_rate=W, devices=[cm.Device(sample_rate=SR, sfmt=sfmt, centerfreq=centerfreq, channels=ch)])


def bursty_stream(cfg, nb, seed):
    """Gated tones in frame units: across the batch boundary 0|1 and the run boundary 1|2 (runs of 2 batches), a short one,
    two with gaps of 1 and of 40 frames, a 1-hop blip, and one tone that is on all the time."""
    N, B, hop = cfg.fft_size, cfg.wave_batch, cfg.hop(0)
    n_samples = (AGC + nb * B) * hop + N
    bw = SR / N
    fr = lambda f: int(f * hop)  # noqa: E731
    tones = [
        (7 * bw, 0.08, [(fr(AGC + B - 120), fr(AGC + B + 150))]),
        (-50 * bw, 0.08, [(fr(AGC + 2 * B - 60), fr(AGC + 2 * B + 300))]),
        (21 * bw, 0.08, [(fr(AGC + B + 400), fr(AGC + B + 403))]),
        (-90 * bw, 0.08, [(fr(AGC + 300), fr(AGC + 340)), (fr(AGC + 341), fr(AGC + 400)), (fr(AGC + 440), fr(AGC + 500))]),
        (33 * bw, 0.5, [(fr(AGC + 2 * B + 500) + N // 2, fr(AGC + 2 * B + 501) + N // 2)]),
        (-3 * bw, 0.05, [(0, n_samples)]),
    ]
    tone_bins = {int(round(f / bw)) % N for f, _, _ in tones}
    return make_raw(cfg, 0, n_samples, tones, seed=seed), tone_bins


def compare(readings, Ps, thr, pmax, B, stride, h, m):
    for b, (r, P) in enumerate(zip(readings, Ps)):
        assert np.all(margin_ok(P, thr[None, :].astype(np.float64), pmax))
        want = model_pieces(P, thr, b, B, stride, h, m)
        got = r["pieces"]
        assert r["n_total"] == got.size == want.size, (b, r["n_total"], want.size)
        assert r["settings"] == (stride, h, m)
        for f in ("bin", "flags", "first_frame", "last_frame", "n_active"):
            assert np.array_equal(got[f], want[f]), (b, f)
        n_act = want["n_active"].astype(np.float64)
        tol_p = 1e-4 * want["peak"] + 2e-5 * pmax
        assert np.all(np.abs(got["peak"] - want["peak"].astype(np.float64)) <= tol_p)
        assert np.all(np.abs(got["sum"] - want["sum"].astype(np.float64)) <= n_act * (1e-4 * want["peak"] + 2e-5 * pmax) + n_act * 2.0 ** -23 * want["sum"])


# ---- 1. float64 exactness ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [256, 512, 1024, 2048, 4096, 8192])
@pytest.mark.parametrize("sfmt", [cm.SFMT_U8, cm.SFMT_S8, cm.SFMT_S16, cm.SFMT_F32])
def test_pieces_match_the_float64_model(n, sfmt):
    cfg = one_device_cfg(n, sfmt)
    B, nb = cfg.wave_batch, 3
    raw, tone_bins = bursty_stream(cfg, nb, seed=n + sfmt)
    strides = {lib.default_stride(cfg, 0), B} | ({1} if n <= 2048 else set())
    pieces_seen = 0
    for stride in sorted(strides):
        n_sel = -(-B // stride)
        h = min(2, n_sel - 1)
        m = min(4, n_sel)
        Ps = [frame_powers(cfg, 0, raw, b, stride) for b in range(nb)]
        pmax = max(P.max() for P in Ps)
        thr = pick_thresholds(np.concatenate(Ps), pmax, tone_bins)
        out, e = drive(cfg, [raw], lambda e: e.activity_configure(0, stride, h, m, thr))
        e.close()
        rd = out["act"][0]
        assert [r["batch_seq"] for r in rd] == list(range(nb))
        compare(rd, Ps, thr, pmax, B, stride, h, m)
        pieces_seen += sum(r["n_total"] for r in rd)
    assert pieces_seen > 0


# ---- 2. reproducibility ------------------------------------------------------------------------------------------------
def _repro_case():
    cfg = one_device_cfg(2048, cm.SFMT_U8)
    raw, tone_bins = bursty_stream(cfg, 5, seed=3)
    thr = np.full(cfg.fft_size, 40.0, np.float32)
    return cfg, raw, thr


def _all_monitors(e, cfg, d=0):
    e.spectrum_configure(d, lib.default_stride(cfg, d))
    e.carrier_configure(d, True)
    e.input_meter_configure(d, True)
    e.subband_configure(d, 0, 10000.0, 32, lib.subband_lowpass(63, 5000.0, cfg.devices[d].sample_rate, 60.0))
    e.tone_meter_configure(d, True)


def test_readings_do_not_depend_on_grouping_pushes_fft_mode_or_other_monitors():
    cfg, raw, thr = _repro_case()
    s = lib.default_stride(cfg, 0)
    on = lambda e: e.activity_configure(0, s, 1, 2, thr)  # noqa: E731
    base, e = drive(cfg, [raw], on, nbmax=4)
    e.close()
    ref = act_key(base["act"][0])
    assert len(ref) == 5 and sum(r[1] for r in ref) > 0
    for nbmax in (1, 2, 3):
        got, e = drive(cfg, [raw], on, nbmax=nbmax)
        e.close()
        assert act_key(got["act"][0]) == ref, nbmax
    got, e = drive(cfg, [raw], on, nbmax=3, pushes=[(0, 3), (3, 4), (4, 9), (9, 10)])
    e.close()
    assert act_key(got["act"][0]) == ref
    for mode in (1, 2, 3):
        got, e = drive(cfg, [raw], on, fft_mode=mode)
        e.close()
        assert act_key(got["act"][0]) == ref, mode
    got, e = drive(cfg, [raw], lambda e: (_all_monitors(e, cfg), on(e)))
    e.close()
    assert act_key(got["act"][0]) == ref


# ---- 3. contract ---------------------------------------------------------------------------------------------------------
def test_outputs_and_other_monitors_unchanged():
    cfg, raw, thr = _repro_case()
    s = lib.default_stride(cfg, 0)
    on = lambda e: e.activity_configure(0, s, 1, 2, thr)  # noqa: E731
    off, e = drive(cfg, [raw], lambda e: None)
    e.close()
    got, e = drive(cfg, [raw], on)
    e.close()
    same_audio(off, got)
    all_off, e = drive(cfg, [raw], lambda e: _all_monitors(e, cfg))
    e.close()
    all_on, e = drive(cfg, [raw], lambda e: (_all_monitors(e, cfg), on(e)))
    e.close()
    same_audio(all_off, all_on)
    assert all_off["mon"] == all_on["mon"] and len(all_on["mon"][0]) > 0
    singles = [lambda e: e.spectrum_configure(0, s), lambda e: e.carrier_configure(0, True),
               lambda e: e.input_meter_configure(0, True),
               lambda e: e.subband_configure(0, 0, 10000.0, 32, lib.subband_lowpass(63, 5000.0, SR, 60.0)),
               lambda e: e.tone_meter_configure(0, True)]
    for one in singles:
        a, e = drive(cfg, [raw], one)
        e.close()
        b, e = drive(cfg, [raw], lambda e: (one(e), on(e)))
        e.close()
        assert a["mon"] == b["mon"] and len(a["mon"][0]) > 0
        same_audio(a, b)


def test_launches_resident_and_injected():
    cfg, raw, thr = _repro_case()
    e = lib.Engine(cfg, max_batches_per_run=4, input_capacity_batches=6)
    raw_res = raw[:e.resident_bytes_needed(0) // raw.itemsize]
    e.resident_load(0, raw_res)

    def per_run():
        e.run_resident(4)
        e.sync()
        l0 = e.launch_count()
        for _ in range(3):
            e.run_resident(4)
        e.sync()
        return (e.launch_count() - l0) / 3

    base = per_run()
    e.activity_configure(0, 0)  # off while off: nothing
    assert per_run() == base
    e.activity_configure(0, 4, 1, 1, thr)
    assert per_run() == base + 2  # one upload and one kernel
    assert e.activity_time() > 0.0
    assert e.fetch_activity(0) is None  # resident runs queue nothing
    e.activity_configure(0, 0)
    assert per_run() == base and e.activity_time() == 0.0
    e.close()
    # injected batches launch nothing and produce nothing
    e = lib.Engine(cfg, max_batches_per_run=4)
    e.activity_configure(0, 4, 1, 1, thr)
    l0 = e.launch_count()
    e.inject_wavein(0, np.zeros((1, 2 * cfg.wave_batch), np.float32))
    e.run(-1)
    e.sync()
    assert e.fetch_activity(0) is None and e.activity_time() == 0.0
    e.close()


def test_lossy_queue_switch_off_and_settings_mid_stream():
    cfg, raw, thr = _repro_case()
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=8)
    e.activity_configure(0, 4, 1, 2, thr)
    e.push(0, raw)
    assert e.run(1) == 1
    e.activity_configure(0, 8, 0, 1, thr)  # applies to the next runs only
    while e.run(-1) > 0:
        pass
    e.activity_configure(0, 0)  # queued readings stay fetchable
    rd = []
    while (r := e.fetch_activity(0)) is not None:
        rd.append(r)
    seqs = [r["batch_seq"] for r in rd]
    assert len(rd) == 4 and seqs == [1, 2, 3, 4]  # 5 batches, ring of max_batches_per_run + 2: batch 0 overwritten
    assert all(r["settings"] == (8, 0, 1) for r in rd)
    with pytest.raises(ValueError, match="gap"):
        lib.merge_bursts([rd[0], rd[2]])
    e.close()


def test_error_codes():
    cfg, raw, thr = _repro_case()
    e = lib.Engine(cfg, max_batches_per_run=2)
    B = cfg.wave_batch

    def code(*a):
        with pytest.raises(lib.AbgError) as x:
            e.activity_configure(*a)
        return x.value.code

    assert code(1, 4, 1, 1, thr) == -5
    assert code(-1, 4, 1, 1, thr) == -5
    assert code(0, -1, 1, 1, thr) == -2
    assert code(0, 4, -1, 1, thr) == -2
    assert code(0, 4, 1, -1, thr) == -2
    assert code(0, 4, 1, 1, None) == -2
    assert code(0, 4, 1, 0, thr) == -2
    assert code(0, B + 1, 0, 1, thr) == -2
    assert code(0, 4, -(-B // 4), 1, thr) == -2
    e.activity_configure(0, 4, -(-B // 4) - 1, 1, thr)  # the largest hang
    e.activity_configure(0, B, 0, 1, thr)
    for bad in (0.0, -1.0, np.inf, np.nan):
        t = thr.copy()
        t[17] = bad
        assert code(0, 4, 1, 1, t) == -2
    with pytest.raises(lib.AbgError) as x:
        e.fetch_activity(3)
    assert x.value.code == -5
    assert e.L.abg_fetch_activity(e.h, 0, None, -1, None, None, None, None) == -2
    e.close()


# ---- 4. truncation -------------------------------------------------------------------------------------------------------
def test_truncation_counts_every_piece():
    n = 8192
    cfg = one_device_cfg(n, cm.SFMT_F32)
    raw, _ = bursty_stream(cfg, 1, seed=11)
    s = lib.default_stride(cfg, 0)
    P = frame_powers(cfg, 0, raw, 0, s)
    thr = np.full(n, np.float32(P.min() * 1e-3), np.float32)  # far below the noise floor: every bin active in every frame
    out, e = drive(cfg, [raw], lambda e: e.activity_configure(0, s, 0, 1, thr))
    e.close()
    r = out["act"][0][0]
    want = model_pieces(P, thr, 0, cfg.wave_batch, s, 0, 1)
    assert r["n_total"] == want.size == n > lib.ACTIVITY_MAX_RECORDS
    assert r["pieces"].size == lib.ACTIVITY_MAX_RECORDS < r["n_total"]
    with pytest.raises(ValueError, match="truncated"):
        lib.merge_bursts([r])


# ---- 5. end to end -------------------------------------------------------------------------------------------------------
def test_spectrum_threshold_detector_merge_group_find_unconfigured_transmitters():
    n, cf = 2048, 120_000_000
    bw = SR // n
    chan_off = [-600, -450, -300, -150, 150, 300, 450, 600]  # bins of the 8 configured AM channels
    chans = [cm.make_channel(cf + k * bw + bw // 2, cf, SR, n, W) for k in chan_off]
    cfg = one_device_cfg(n, cm.SFMT_U8, chans, centerfreq=cf)
    B, hop, nb = cfg.wave_batch, cfg.hop(0), 6
    n_samples = (AGC + nb * B) * hop + n
    f2s = lambda f: int(f * hop)  # noqa: E731
    # (offset in bins, first frame, end frame): 20 ms = 160 frames inside batch 3; 1 s over batches 1..3; one across 4|5
    extra = [(-222, AGC + 3 * B + 300, AGC + 3 * B + 460), (77, AGC + B + 100, AGC + 4 * B + 100), (512, AGC + 4 * B + 900, AGC + 5 * B + 200)]
    tones = [(k * bw + bw / 2, 0.04, [(0, n_samples)]) for k in chan_off]
    tones += [(k * bw, 0.04, [(f2s(a), f2s(b))]) for k, a, b in extra]
    raw = make_raw(cfg, 0, n_samples, tones, noise=0.01, seed=1)
    s = lib.default_stride(cfg, 0)
    h, m = 1, 2

    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=nb + 2)
    e.push(0, raw)
    e.spectrum_configure(0, s)
    assert e.run(1) == 1
    spec = e.fetch_spectrum(0)[0]
    thr = lib.activity_threshold(spec, 13.0, 16)
    e.spectrum_configure(0, 0)
    e.activity_configure(0, s, h, m, thr)
    rd = []
    while True:
        while e.fetch(0) is not None:  # the audio holds result slots
            pass
        while (r := e.fetch_activity(0)) is not None:
            rd.append(r)
        if e.run(-1) == 0:
            break
    e.close()
    assert [r["batch_seq"] for r in rd] == list(range(1, nb))
    tx = lib.group_transmissions(lib.merge_bursts(rd), cfg, 0)
    tol = (h + 1) * s
    for k, a, b in extra:
        hit = [t for t in tx if abs(t["freq_hz"] - (cf + k * bw)) <= bw and abs(t["last_frame"] - (b - 1)) <= tol]
        assert len(hit) == 1, (k, [(t["freq_hz"] - cf, t["first_frame"], t["last_frame"]) for t in tx])
        t = hit[0]
        assert not t["monitored"]
        first = max(a, AGC + B)  # the detector starts with batch 1
        assert abs(t["first_frame"] - first) <= tol, (k, t["first_frame"], first)
        assert t["start_s"] == pytest.approx(t["first_frame"] * hop / SR)
    for k in chan_off:
        hit = [t for t in tx if t["bins"][0] <= k <= t["bins"][1]]
        assert hit and all(t["monitored"] for t in hit), k
