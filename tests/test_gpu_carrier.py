"""Carrier frequency meter (abg_carrier_configure / abg_fetch_carrier) on the GPU (-m gpu).

Reference: float64 numpy FFTs of the oracle's own float32 fftin (op.Oracle.debug_frame) for every frame of a batch, so the
check is independent of the engine's K1 and of the oracle's FFT.  Known carrier offsets must be recovered through
lib.carrier_offset_hz; switching the meter on must leave every other output bit-identical, and readings must not depend
on how batches are grouped into runs."""
import numpy as np
import pytest

import oracle_py as op
from airband_b200 import config as cm
from airband_b200 import lib
from airband_b200 import workloads as wl
from cases import CASES

pytestmark = pytest.mark.gpu
AGC_EXTRA = 100
STAT_FIELDS = [f for f, _ in cm.CSquelchStats._fields_]
DELTAS = [-3500.0, -1200.0, -310.5, 0.0, 47.25, 900.0, 3100.0]


def ref_carrier(cfg, dev, raw, batch, bins):
    """(R[C] complex128, E[C] float64) of one batch from the oracle's float32 converted + windowed frames."""
    d = cfg.devices[dev]
    one = cm.Config(fft_size=cfg.fft_size, wave_rate=cfg.wave_rate, fm_demod=cfg.fm_demod, devices=[d])
    o = op.Oracle(one)
    N, B, hop = cfg.fft_size, cfg.wave_batch, cfg.hop(dev)
    X = np.empty((B, len(bins)), np.complex128)
    step = max(1, (1 << 21) // N)
    for j0 in range(0, B, step):
        js = range(j0, min(B, j0 + step))
        fins = []
        for j in js:
            s0 = (AGC_EXTRA + batch * B + j) * hop
            fins.append(o.debug_frame(0, raw[2 * s0:2 * (s0 + N)])[0])
        X[js.start:js.stop] = np.fft.fft(np.stack(fins).astype(np.complex128), axis=1)[:, bins]
    o.close()
    return np.sum(X[1:] * np.conj(X[:-1]), 0), np.sum(np.abs(X) ** 2, 0)


def window(n):
    """The engine's 7-term Blackman-Harris window (float32 values, reference src/rtl_airband.cpp:335-351)."""
    a = [0.27105140069342, 0.43329793923448, 0.21812299954311, 0.06592544638803, 0.01081174209837, 0.00077658482522, 0.00001388721735]
    i = np.arange(n)
    w = sum((-1) ** k * np.float64(np.float32(ak)) * np.cos(2.0 * k * np.pi * i / (n - 1)) for k, ak in enumerate(a))
    return w.astype(np.float32).astype(np.float64)


def rho_w(n, hop):
    """|R| / E of white noise: sum w[n] w[n + hop] / sum w[n]^2."""
    w = window(n)
    return float(np.sum(w[:-hop] * w[hop:]) / np.sum(w * w)) if hop < n else 0.0


def drive(cfg, raws, meter=(), spectrum=None, nbmax=4, fetch_readings=True, mixers=None, scan=None, **kw):
    """Push every stream, run to exhaustion and fetch everything: audio, I/Q, flags, mixers, spectra and meter readings.
    meter = devices to meter; spectrum = {dev: stride}; scan = (dev, chan, freqs, [freq_idx per run])."""
    total = max(r.size // (2 * cfg.hop(d)) // cfg.wave_batch for d, r in enumerate(raws)) + 2
    e = lib.Engine(cfg, max_batches_per_run=nbmax, input_capacity_batches=total, **kw)
    for d in meter:
        e.carrier_configure(d, True)
    for d, s in (spectrum or {}).items():
        e.spectrum_configure(d, s)
    if mixers:
        e.configure_mixers(mixers)
    if scan:
        e.scan_configure(scan[0], scan[1], scan[2])
    for d, r in enumerate(raws):
        e.push(d, r)
    D = len(cfg.devices)
    audio = [[] for _ in range(D)]
    spectra = [[] for _ in range(D)]
    readings = [[] for _ in range(D)]
    bins = [[] for _ in range(D)]  # per batch: the bins its channels used (AFC moves them between runs)
    mix = [[] for _ in range(len(mixers or []))]
    runs = 0
    while True:
        if scan:
            e.scan_select(scan[0], scan[1], scan[3][runs % len(scan[3])])
        cur = [[e.stats(d, c).bin for c in range(len(cfg.devices[d].channels))] for d in range(D)]
        n = e.run(-1)
        if n == 0:
            break
        runs += 1
        for d in range(D):
            while (got := e.fetch(d)) is not None:
                audio[d].append(got)
                bins[d].append(cur[d])
            while (s := e.fetch_spectrum(d)) is not None:
                spectra[d].append(s)
            while fetch_readings and (r := e.fetch_carrier(d)) is not None:
                readings[d].append(r)
        for m in range(len(mix)):
            while (got := e.fetch_mixer(m)) is not None:
                mix[m].append(got)
    stats = [[tuple(getattr(e.stats(d, c), f) for f in STAT_FIELDS) for c in range(len(cfg.devices[d].channels))] for d in range(D)]
    return dict(audio=audio, spectra=spectra, readings=readings, bins=bins, mix=mix, stats=stats,
                paths=[e.fft_path(d) for d in range(D)], runs=runs), e


def same_outputs(a, b):
    assert a["paths"] == b["paths"]
    for d in range(len(a["audio"])):
        assert len(a["audio"][d]) == len(b["audio"][d]) > 0
        for (w1, i1, x1), (w2, i2, x2) in zip(a["audio"][d], b["audio"][d]):
            assert np.array_equal(w1.view(np.uint32), w2.view(np.uint32))
            assert np.array_equal(i1.view(np.uint64), i2.view(np.uint64))
            assert np.array_equal(x1, x2)
        assert len(a["spectra"][d]) == len(b["spectra"][d])
        for (p1, s1, n1), (p2, s2, n2) in zip(a["spectra"][d], b["spectra"][d]):
            assert np.array_equal(p1.view(np.uint32), p2.view(np.uint32)) and s1 == s2 and n1 == n2
    assert a["stats"] == b["stats"]
    assert len(a["mix"]) == len(b["mix"])
    for m1, m2 in zip(a["mix"], b["mix"]):
        assert len(m1) == len(m2) > 0
        for (l1, r1, s1), (l2, r2, s2) in zip(m1, m2):
            assert np.array_equal(l1.view(np.uint32), l2.view(np.uint32)) and np.array_equal(r1.view(np.uint32), r2.view(np.uint32)) and s1 == s2


def by_seq(readings):
    return {seq: (lag1, en) for lag1, en, seq in readings}


def check_against_float64(cfg, dev, raw, readings, n_batches):
    assert [s for _, _, s in readings] == list(range(n_batches))
    bins = [ch.bin for ch in cfg.devices[dev].channels]
    for lag1, en, seq in readings:
        R, E = ref_carrier(cfg, dev, raw, seq, bins)
        assert np.all(E > 0)
        errR = np.abs(lag1.astype(np.complex128) - R) / E
        errE = np.abs(en.astype(np.float64) - E) / E
        assert np.all(errR <= 1e-4) and np.all(errE <= 1e-4), (seq, float(errR.max()), float(errE.max()))
        assert np.all(np.abs(lag1) <= en * (1 + 1e-5))


# ---- 1. against float64, every K1 path ---------------------------------------------------------------------------------
def _accuracy_case(n, sfmt, sr=2048000):
    """Two keyed carriers plus a channel that only sees noise; the carriers sit 0.0075..0.24 bins above a bin centre."""
    w = 8000
    bw = sr / n
    chans = [cm.make_channel(96060, 0, sr, n, w), cm.make_channel(int(-40 * bw) + 1500, 0, sr, n, w)]
    quiet = cm.make_channel(int(25 * bw) + 700, 0, sr, n, w)
    synth = cm.Config(fft_size=n, wave_rate=w, devices=[cm.Device(sample_rate=sr, sfmt=sfmt, centerfreq=0, channels=chans)])
    cfg = cm.Config(fft_size=n, wave_rate=w, devices=[cm.Device(sample_rate=sr, sfmt=sfmt, centerfreq=0, channels=chans + [quiet])])
    nb = 2
    raw = wl.synth_iq(synth, 0, wl.samples_for_batches(cfg, 0, nb), key_on_s=0.2, key_off_s=0.05, seed=n + sfmt, amplitude=0.2,
                      noise_sigma=0.05)
    return cfg, raw, nb


@pytest.mark.parametrize("n", [256, 512, 1024, 2048, 4096, 8192])
@pytest.mark.parametrize("sfmt", [cm.SFMT_U8, cm.SFMT_S8, cm.SFMT_S16, cm.SFMT_F32])
def test_readings_match_float64_every_size_and_format(n, sfmt):
    cfg, raw, nb = _accuracy_case(n, sfmt)
    out, e = drive(cfg, [raw], meter=[0])
    assert e.fft_path(0) == (3 if sfmt in (cm.SFMT_U8, cm.SFMT_S8) else 2)
    check_against_float64(cfg, 0, raw, out["readings"][0], nb)
    e.close()


@pytest.mark.parametrize("kind", ["full_spectrum_k1", "u8_2500k"])
def test_readings_match_float64_full_k1_and_uneven_hop(kind):
    if kind == "full_spectrum_k1":
        cfg, raw, nb = _accuracy_case(1024, cm.SFMT_U8)
        kw, path = dict(fft_mode=1), 1
    else:  # hop 313: not a multiple of 16 (the pruned K1), and the frame rate is not WAVE_RATE
        cfg, raw, nb = _accuracy_case(2048, cm.SFMT_U8, sr=2500000)
        kw, path = {}, 2
        assert cfg.hop(0) == 313
    out, e = drive(cfg, [raw], meter=[0], **kw)
    assert e.fft_path(0) == path
    check_against_float64(cfg, 0, raw, out["readings"][0], nb)
    e.close()


# ---- 2. known offsets are recovered -------------------------------------------------------------------------------------
def key_state(cfg_synth, dev, ci, batch, key_on_s, key_off_s):
    """The synthesizer's key gate (workloads.synth_iq) over every sample of every frame of the batch: 1 on throughout,
    0 off throughout, -1 keyed or unkeyed inside the batch."""
    d = cfg_synth.devices[dev]
    sr, N, B, hop = d.sample_rate, cfg_synth.fft_size, cfg_synth.wave_batch, cfg_synth.hop(dev)
    s0 = (AGC_EXTRA + batch * B) * hop
    t = np.arange(s0, s0 + (B - 1) * hop + N, dtype=np.float64) / sr
    period = key_on_s + key_off_s
    on = np.mod(t + ci * 0.37 * period / max(1, len(d.channels)), period) >= key_off_s
    return 1 if on.all() else 0 if not on.any() else -1


def steady_keyed(cfg_synth, dev, ci, batch, key):
    """Channel ci's carrier is keyed for the whole batch, and no other carrier of the device is keyed or unkeyed during
    it: a key edge splatters over the whole band (the gate is a step), and a few frames of that leaking into another
    channel's bin move its reading by about a hertz."""
    st = [key_state(cfg_synth, dev, c, batch, *key) for c in range(len(cfg_synth.devices[dev].channels))]
    return st[ci] == 1 and min(st) >= 0


def _offset_device(sr, n, sfmt, deltas, modulation=cm.MOD_AM, afc=0, spacing_bins=16, squelch_dbfs=-50.0, nfm_delta=None):
    """Channels on bin centres (+1 Hz, so that calc_bin's ceil(...) - 1 picks that bin) `spacing_bins` apart, none on the
    DC bin (AFC does not search below bin 0); the synthesized carrier of channel i sits deltas[i] Hz above its channel.  An optional NFM channel (modulation index 2.5
    at 1 kHz) carries nfm_delta.  Returns (cfg the engine runs, cfg the synthesizer uses, deltas per channel)."""
    w = 8000
    bw = sr / n
    kinds = [(modulation, dl) for dl in deltas] + ([(cm.MOD_NFM, nfm_delta)] if nfm_delta is not None else [])
    chans, synth_chans = [], []
    for i, (mod, dl) in enumerate(kinds):
        f = int(round(bw * (spacing_bins * (i - len(kinds) // 2) + 4))) + 1
        kw = dict(modulation=mod, squelch_dbfs=squelch_dbfs, afc=afc)
        if mod == cm.MOD_NFM:
            kw["bandwidth"] = 12000
        ch = cm.make_channel(f, 0, sr, n, w, **kw)
        chans.append(ch)
        sc = cm.make_channel(f, 0, sr, n, w, **kw)
        sc.offset_hz = f + dl
        synth_chans.append(sc)
    dev = cm.Device(sample_rate=sr, sfmt=sfmt, centerfreq=0, channels=chans)
    sdev = cm.Device(sample_rate=sr, sfmt=sfmt, centerfreq=0, channels=synth_chans)
    return (cm.Config(fft_size=n, wave_rate=w, devices=[dev]), cm.Config(fft_size=n, wave_rate=w, devices=[sdev]),
            [dl for _, dl in kinds])


def _check_offsets(cfg, synth, deltas, out, key, tol_hz=1.0, min_batches=2):
    sr, hop = cfg.devices[0].sample_rate, cfg.hop(0)
    chans = cfg.devices[0].channels
    readings = out["readings"][0]
    assert len(readings) == len(out["audio"][0])
    counted = [0] * len(deltas)
    for (lag1, en, seq), (_, _, axc) in zip(readings, out["audio"][0]):
        off = lib.carrier_offset_hz(lag1, [ch.offset_hz for ch in chans], sr, hop)
        for c, dl in enumerate(deltas):
            if axc[c] == ord(' ') or not steady_keyed(synth, 0, c, seq, key):
                continue
            counted[c] += 1
            assert abs(off[c] - dl) <= tol_hz, (c, seq, dl, float(off[c]), chr(axc[c]))
    assert min(counted) >= min_batches, counted


@pytest.mark.parametrize("kind", ["cfg2_shape", "2500k", "afc"])
def test_known_offsets_of_keyed_carriers_are_recovered(kind):
    """Steady keyed carriers in noise at cfg2's fft_size 2048 (1250 Hz bins at 2.56 Msps), up to 2.9 bins off their
    channel: |R| / E is about 1 and the offset is exact up to noise.  S16 input keeps the noise floor low enough for 1 Hz
    with the -16 dB the window leaves of a carrier 2.8 bins away.  The noise-only channel reads rho_w(hop)."""
    key = (1.0, 0.25)
    sr = 2500000 if kind == "2500k" else 2560000
    deltas = [3100.0, -3500.0] if kind == "afc" else DELTAS
    cfg, synth, deltas = _offset_device(sr, 2048, cm.SFMT_S16, deltas, afc=2 if kind == "afc" else 0, spacing_bins=32)
    n = cfg.fft_size
    # a noise-only channel far from every carrier (the synthesizer does not know it)
    cfg.devices[0].channels.append(cm.make_channel(int(round(sr / n * 300)) + 1, 0, sr, n, 8000, squelch_dbfs=-50.0))
    nb = 10
    raw = wl.synth_iq(synth, 0, wl.samples_for_batches(cfg, 0, nb), key_on_s=key[0], key_off_s=key[1], am_depth=0.0,
                      amplitude=0.1, noise_sigma=0.0005, seed=7)
    out, e = drive(cfg, [raw], meter=[0], nbmax=4)
    _check_offsets(cfg, synth, deltas, out, key)
    q = len(deltas)
    rho = rho_w(n, cfg.hop(0))
    for lag1, en, _ in out["readings"][0]:
        assert abs(abs(lag1[q]) / en[q] - rho) <= 0.1, (abs(lag1[q]) / en[q], rho)
    if kind == "afc":  # the carriers are more than one bin off: AFC moved the bins, and the readings followed
        moved = [any(b[c] != cfg.devices[0].channels[c].bin for b in out["bins"][0]) for c in range(2)]
        assert all(moved), out["bins"][0]
    e.close()


def test_known_offsets_of_modulated_carriers():
    """AM 60 % at 1 kHz and NFM with a peak deviation of 2.5 kHz at 1 kHz.  The window weighs a modulated carrier's
    sidebands unequally once the carrier is off its bin centre, which biases the reading (airband_b200.h): with bins much
    wider than the offsets (10 Msps, fft 256: 39 kHz) AM reads within 1 Hz.  NFM's wider sidebands leave up to 25 Hz of
    bias at +-3.5 kHz; there the engine's reading must match the float64 one from the oracle's frames within 1 Hz."""
    key = (1.0, 0.25)
    sr, n = 10000000, 256
    cfg, synth, deltas = _offset_device(sr, n, cm.SFMT_S16, DELTAS, nfm_delta=-1200.0, spacing_bins=8)
    nb = 10
    raw = wl.synth_iq(synth, 0, wl.samples_for_batches(cfg, 0, nb), key_on_s=key[0], key_off_s=key[1], amplitude=0.05,
                      noise_sigma=0.0005, seed=11)
    out, e = drive(cfg, [raw], meter=[0], nbmax=4)
    am = len(DELTAS)
    _check_offsets(cfg, synth, deltas[:am], out, key)
    chans = cfg.devices[0].channels
    hop = cfg.hop(0)
    checked = 0
    for (lag1, en, seq), (_, _, axc) in zip(out["readings"][0], out["audio"][0]):
        if axc[am] == ord(' ') or not steady_keyed(synth, 0, am, seq, key):
            continue
        R, _ = ref_carrier(cfg, 0, raw, seq, [chans[am].bin])
        got = lib.carrier_offset_hz(lag1[am], chans[am].offset_hz, sr, hop)
        ref = lib.carrier_offset_hz(R[0], chans[am].offset_hz, sr, hop)
        assert abs(got - ref) <= 1.0 and abs(ref - deltas[am]) <= 25.0, (seq, float(got), float(ref))
        checked += 1
    assert checked >= 2
    e.close()


def test_carrier_offset_hz_wraps_and_uses_hop():
    sr, hop = 2500000, 313
    frame_rate = sr / hop
    for off_hz, true_hz in ((100000.0, 100000.0 + 47.25), (-250000.0, -250000.0 - 3500.0), (0.0, 0.4999 * frame_rate)):
        lag1 = np.exp(2j * np.pi * true_hz * hop / sr) * 3.0
        assert abs(float(lib.carrier_offset_hz(lag1, off_hz, sr, hop)) - (true_hz - off_hz)) < 1e-6
    got = lib.carrier_offset_hz(np.array([1j, -1j]), np.array([0.0, 0.0]), sr, hop)
    assert np.allclose(got, [0.25 * frame_rate, -0.25 * frame_rate])
    assert float(lib.carrier_offset_hz(-1.0, 0.0, sr, hop)) == -0.5 * frame_rate


# ---- 3. no other output changes -----------------------------------------------------------------------------------------
def _afc_case():
    sr, n, w, cf = 2560000, 512, 8000, 120000000
    ch = cm.make_channel(cf + 100000, cf, sr, n, w, squelch_dbfs=-40.0, afc=2)
    ch.offset_hz = 100000.0 + 3 * (sr / n)
    cfg = cm.Config(fft_size=n, wave_rate=w, devices=[cm.Device(sample_rate=sr, sfmt=cm.SFMT_U8, centerfreq=cf, channels=[ch])])
    return cfg, [wl.synth_iq(cfg, 0, wl.samples_for_batches(cfg, 0, 5), key_on_s=0.25, key_off_s=0.15, amplitude=0.3)]


def _scan_case():
    sr, n, w, cf = 2560000, 1024, 16000, 120000000
    f0 = cf + 250000
    base = cm.make_channel(f0, cf, sr, n, w, modulation=cm.MOD_NFM, bandwidth=6000, squelch_dbfs=-35.0)
    freqs = [cm.make_channel(f0, cf, sr, n, w, modulation=cm.MOD_AM, bandwidth=6000, squelch_dbfs=-35.0),
             cm.make_channel(f0, cf, sr, n, w, modulation=cm.MOD_NFM, bandwidth=6000, squelch_dbfs=-35.0, ctcss_hz=100.0)]
    base.synth_ctcss_hz = 100.0
    cfg = cm.Config(fft_size=n, wave_rate=w, devices=[cm.Device(sample_rate=sr, sfmt=cm.SFMT_S16, centerfreq=cf, channels=[base])])
    raw = wl.synth_iq(cfg, 0, wl.samples_for_batches(cfg, 0, 6), key_on_s=0.6, key_off_s=0.2, amplitude=0.2)
    return cfg, [raw], (0, 0, freqs, [0, 1, 1, 0])


@pytest.mark.parametrize("name", ["am_u8", "nfm_s16", "am_bw_f32", "s8_two_devices", "full_k1", "afc", "scan", "cfg4_mixers",
                                  "with_spectrum"])
def test_meter_changes_no_other_output(name):
    kw, scan, mixers, spectrum = {}, None, None, None
    if name == "afc":
        cfg, raws = _afc_case()
        kw["nbmax"] = 1
    elif name == "scan":
        cfg, raws, scan = _scan_case()
        kw["nbmax"] = 2
    elif name == "cfg4_mixers":
        cfg = wl.cfg4()
        raws = [wl.synth_iq(cfg, d, wl.samples_for_batches(cfg, d, 3), key_on_s=0.2, key_off_s=0.1) for d in range(len(cfg.devices))]
        mixers = [[(d, m, 1.0 + 0.25 * d, (-0.5 if (m == 1 and d == 0) else 0.0)) for d in range(len(cfg.devices))] for m in range(4)]
        kw["nbmax"] = 2
    elif name == "full_k1":
        cfg, raws = CASES["s8_two_devices"]()
        kw["fft_mode"] = 1
    elif name == "with_spectrum":
        cfg, raws = CASES["s8_two_devices"](n_batches=3)
        spectrum = {0: 1, 1: lib.default_stride(cfg, 1)}
    else:
        cfg, raws = CASES[name]()
    off, e0 = drive(cfg, raws, (), spectrum=spectrum, mixers=mixers, scan=scan, **kw)
    on, e1 = drive(cfg, raws, range(len(cfg.devices)), spectrum=spectrum, mixers=mixers, scan=scan, **kw)
    same_outputs(off, on)
    if name == "full_k1":
        assert set(on["paths"]) == {1}
    assert all(len(on["readings"][d]) == len(on["audio"][d]) for d in range(len(cfg.devices)))
    assert all(not r for r in off["readings"])
    e0.close(); e1.close()


def test_no_behaviour_change_cases_cover_every_k1_path():
    paths = set()
    for name in ("am_u8", "nfm_s16", "am_bw_f32", "s8_two_devices"):
        cfg, _ = CASES[name]()
        e = lib.Engine(cfg)
        paths.update(e.fft_path(d) for d in range(len(cfg.devices)))
        e.close()
    cfg, _ = _afc_case()
    e = lib.Engine(cfg)
    paths.add(e.fft_path(0))
    e.close()
    assert paths == {1, 2, 3}


# ---- 4. segmentation independence ---------------------------------------------------------------------------------------
def test_readings_do_not_depend_on_run_grouping_or_pushes():
    cfg, raws = CASES["am_u8"](n_batches=4)
    ref = None
    for nbmax in (1, 4):
        out, e = drive(cfg, raws, [0], nbmax=nbmax)
        got = by_seq(out["readings"][0])
        assert sorted(got) == [0, 1, 2, 3]
        if ref is None:
            ref = got
        for s in ref:
            assert np.array_equal(got[s][0].view(np.uint64), ref[s][0].view(np.uint64)), (nbmax, s)
            assert np.array_equal(got[s][1].view(np.uint32), ref[s][1].view(np.uint32)), (nbmax, s)
        e.close()
    # pushes of odd sizes
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=3)
    e.carrier_configure(0, True)
    rng = np.random.default_rng(5)
    pos, got = 0, {}
    r = raws[0]
    while pos < r.size or e.batches_available(0) > 0:
        if pos < r.size:
            step = 2 * int(rng.integers(1, 90000))
            e.push(0, r[pos:pos + step])
            pos += step
        e.run(-1)
        while e.fetch(0) is not None:
            pass
        while (x := e.fetch_carrier(0)) is not None:
            got[x[2]] = x[:2]
    assert sorted(got) == [0, 1, 2, 3]
    for s in ref:
        assert np.array_equal(got[s][0].view(np.uint64), ref[s][0].view(np.uint64)), s
        assert np.array_equal(got[s][1].view(np.uint32), ref[s][1].view(np.uint32)), s
    e.close()


# ---- 5. control ---------------------------------------------------------------------------------------------------------
def test_only_metered_devices_produce_readings():
    cfg, raws = CASES["s8_two_devices"](n_batches=3)
    out, e = drive(cfg, raws, [1], nbmax=2)
    assert [s for _, _, s in out["readings"][1]] == [0, 1, 2]
    assert all(lag.shape == (3,) and en.shape == (3,) for lag, en, _ in out["readings"][1])
    assert out["readings"][0] == [] and e.fetch_carrier(0) is None
    e.close()


def test_switching_affects_exactly_the_later_runs():
    cfg, raws = CASES["am_u8"](n_batches=6)
    always, e_all = drive(cfg, raws, [0], nbmax=2)
    ref = by_seq(always["readings"][0])
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=8)
    e.push(0, raws[0])
    seen = []
    for on in (False, True, False):
        e.carrier_configure(0, on)
        assert e.run(2) == 2
        while e.fetch(0) is not None:
            pass
        while (x := e.fetch_carrier(0)) is not None:
            seen.append(x)
    assert [s for _, _, s in seen] == [2, 3]
    for lag1, en, s in seen:
        assert np.array_equal(lag1.view(np.uint64), ref[s][0].view(np.uint64)) and np.array_equal(en.view(np.uint32), ref[s][1].view(np.uint32))
    e.close(); e_all.close()


def test_launch_count_unchanged_while_off_and_error_codes():
    cfg, raws = CASES["am_u8"](n_batches=2)
    counts = []
    for setup in ("untouched", "explicit_off", "on_then_off", "on"):
        e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=4)
        if setup == "explicit_off":
            e.carrier_configure(0, False)
        elif setup == "on_then_off":
            e.carrier_configure(0, True)
            e.carrier_configure(0, False)
        elif setup == "on":
            e.carrier_configure(0, True)
        e.push(0, raws[0])
        l0 = e.launch_count()
        assert e.run(-1) == 2
        e.sync()
        counts.append(e.launch_count() - l0)
        if setup != "on":
            assert e.fetch_carrier(0) is None and e.carrier_time() == 0.0
        else:
            assert e.carrier_time() > 0.0
        if setup == "untouched":
            for args, code in (((5, 1), -5), ((-1, 1), -5), ((0, 2), -2), ((0, -1), -2)):
                with pytest.raises(lib.AbgError) as ei:
                    e._chk(e.L.abg_carrier_configure(e.h, *args))
                assert ei.value.code == code
            with pytest.raises(lib.AbgError) as ei:
                e.fetch_carrier(5)
            assert ei.value.code == -5
        e.close()
    assert counts[0] == counts[1] == counts[2] < counts[3]


def test_injected_batches_and_resident_runs_queue_nothing():
    cfg = wl.cfg1()
    e = lib.Engine(cfg, max_batches_per_run=2)
    e.carrier_configure(0, True)
    assert e.inject_wavein(0, np.full((1, 2 * cfg.wave_batch), 5.0, np.float32)) == 2
    assert e.fetch(0) is not None and e.fetch_carrier(0) is None
    e.close()
    e = lib.Engine(cfg, max_batches_per_run=2)
    raw = wl.synth_iq(cfg, 0, wl.samples_for_batches(cfg, 0, 2), key_off_s=0.0)
    e.resident_load(0, raw)
    e.carrier_configure(0, True)
    l0 = e.launch_count()
    e.run_resident(2)
    e.sync()
    assert e.carrier_time() > 0.0 and e.launch_count() > l0  # computed ...
    assert e.fetch_carrier(0) is None                         # ... but not queued
    e.close()


def test_unfetched_readings_are_overwritten_oldest_first():
    cfg, raws = CASES["am_u8"](n_batches=10)
    nbmax = 4
    off, e0 = drive(cfg, raws, (), nbmax=nbmax)
    each, e1 = drive(cfg, raws, [0], nbmax=nbmax)
    lazy, e2 = drive(cfg, raws, [0], nbmax=nbmax, fetch_readings=False)
    assert lazy["runs"] == 3
    same_outputs(off, lazy)
    assert len(lazy["audio"][0]) == 10
    got = []
    while (x := e2.fetch_carrier(0)) is not None:
        got.append(x)
    assert [s for _, _, s in got] == list(range(10 - (nbmax + 2), 10))
    ref = by_seq(each["readings"][0])
    for lag1, en, s in got:
        assert np.array_equal(lag1.view(np.uint64), ref[s][0].view(np.uint64)) and np.array_equal(en.view(np.uint32), ref[s][1].view(np.uint32))
    for e in (e0, e1, e2):
        e.close()


# ---- 6. full size -------------------------------------------------------------------------------------------------------
def test_full_size_cfg2_every_device_metered():
    import bench
    cfg, _ = bench.make_workload("cfg2")
    nb = 4
    raws = bench.synth_streams(cfg, nb, n_unique=4)
    D = len(cfg.devices)
    off, e0 = drive(cfg, raws, (), nbmax=nb)
    on, e1 = drive(cfg, raws, range(D), nbmax=nb)
    same_outputs(off, on)
    for d in range(D):
        assert [s for _, _, s in on["readings"][d]] == list(range(nb))
        for b in range(nb):  # identical streams give bit-identical readings wherever the device sits in the launch
            assert np.array_equal(on["readings"][d][b][0].view(np.uint64), on["readings"][d % 4][b][0].view(np.uint64))
            assert np.array_equal(on["readings"][d][b][1].view(np.uint32), on["readings"][d % 4][b][1].view(np.uint32))
    for d in range(4):  # one device per distinct stream
        check_against_float64(cfg, d, raws[d], on["readings"][d], nb)
    e0.close(); e1.close()
