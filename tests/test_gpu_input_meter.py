"""Input level meter (abg_input_meter_configure / abg_fetch_input_levels) on the GPU (-m gpu).

Reference: numpy over the raw samples of each batch, s in [(AGC_EXTRA + b*B) * hop, + B*hop): the float32 levels and
bins of the definition in airband_b200.h, and float64 sums of the exact levels.  Known impairments must be recovered
through lib.input_levels; switching the meter on must leave every other output bit-identical, and readings must not
depend on how batches are grouped into runs or on push sizes."""
import math

import numpy as np
import pytest

from airband_b200 import config as cm
from airband_b200 import lib
from airband_b200 import workloads as wl
from cases import CASES

pytestmark = pytest.mark.gpu
AGC_EXTRA = 100
STAT_FIELDS = [f for f, _ in cm.CSquelchStats._fields_]
f32 = np.float32


def batch_samples(cfg, dev, raw, batch):
    """[n, 2] raw codes of one batch."""
    hop, B = cfg.hop(dev), cfg.wave_batch
    s0 = (AGC_EXTRA + batch * B) * hop
    return raw[2 * s0:2 * (s0 + B * hop)].reshape(-1, 2)


def ref_levels(cfg, dev, raw, batch):
    d = cfg.devices[dev]
    x = batch_samples(cfg, dev, raw, batch)
    sc = f32(1.0) / f32(d.fullscale)
    if d.sfmt == cm.SFMT_U8:
        v = (x.astype(f32) - f32(127.5)) / f32(127.5)
        exact = (2.0 * x.astype(np.float64) - 255.0) / 255.0
    elif d.sfmt == cm.SFMT_S8:
        v = x.astype(f32) / f32(128.0)
        exact = x.astype(np.float64) / 128.0
    elif d.sfmt == cm.SFMT_S16:
        v = sc * x.astype(f32)
        exact = x.astype(np.float64) * np.float64(sc)
    else:
        v = sc * x.astype(f32)
        exact = v.astype(np.float64)
    assert v.dtype == np.float32
    bins = np.clip(np.floor((v + f32(1.0)) * f32(128.0)), 0, 255).astype(np.int64)
    hist = np.stack([np.bincount(bins[:, k], minlength=256) for k in range(2)])
    return dict(n=x.shape[0], hist=hist, peak=np.abs(v).max(0), exact=exact, codes=x)


def check_exact(cfg, dev, raw, r):
    d = cfg.devices[dev]
    ref = ref_levels(cfg, dev, raw, r["batch_seq"])
    assert r["n_samples"] == ref["n"]
    assert np.array_equal(r["hist"], ref["hist"]), r["batch_seq"]
    if d.sfmt in (cm.SFMT_U8, cm.SFMT_S8):
        off = 0 if d.sfmt == cm.SFMT_U8 else 128
        for k in range(2):
            codes = ref["codes"][:, k].astype(np.int64) + off
            assert np.array_equal(r["hist"][k], np.bincount(codes, minlength=256))
    assert np.array_equal(r["peak"], ref["peak"].astype(np.float32)), (r["peak"], ref["peak"])
    # float64 references, summed with math.fsum: a plain float64 sum of 10^5..10^6 terms is itself off by more than
    # 1e-12 relative, while the engine's integer sums are exact
    tol = 1e-10 if d.sfmt == cm.SFMT_F32 else 1e-12
    e = ref["exact"]
    terms = ((r["sum"][0], e[:, 0]), (r["sum"][1], e[:, 1]), (r["sum_sq"][0], e[:, 0] ** 2), (r["sum_sq"][1], e[:, 1] ** 2),
             (r["sum_iq"], e[:, 0] * e[:, 1]))
    for q, (got, t) in enumerate(terms):
        want, scale = math.fsum(t), math.fsum(np.abs(t))
        assert abs(got - want) <= tol * max(scale, 1e-300), (q, got, want)


def same_reading(a, b):
    assert a["batch_seq"] == b["batch_seq"] and a["n_samples"] == b["n_samples"]
    assert np.array_equal(a["hist"], b["hist"]) and np.array_equal(a["peak"].view(np.uint32), b["peak"].view(np.uint32))
    for k in ("sum", "sum_sq"):
        assert np.array_equal(a[k].view(np.uint64), b[k].view(np.uint64)), k
    assert np.float64(a["sum_iq"]).view(np.uint64) == np.float64(b["sum_iq"]).view(np.uint64)


def drive(cfg, raws, meter=(), spectrum=None, carrier=(), nbmax=4, fetch_readings=True, mixers=None, scan=None, **kw):
    """Push every stream, run to exhaustion and fetch everything: audio, I/Q, flags, mixers, spectra, carrier readings
    and input levels.  meter = devices to meter; spectrum = {dev: stride}; scan = (dev, chan, freqs, [freq_idx per run])."""
    total = max(r.size // (2 * cfg.hop(d)) // cfg.wave_batch for d, r in enumerate(raws)) + 2
    e = lib.Engine(cfg, max_batches_per_run=nbmax, input_capacity_batches=total, **kw)
    for d in meter:
        e.input_meter_configure(d, True)
    for d in carrier:
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
    audio, spectra, car, levels = ([[] for _ in range(D)] for _ in range(4))
    mix = [[] for _ in range(len(mixers or []))]
    runs = 0
    while True:
        if scan:
            e.scan_select(scan[0], scan[1], scan[3][runs % len(scan[3])])
        n = e.run(-1)
        if n == 0:
            break
        runs += 1
        for d in range(D):
            while (got := e.fetch(d)) is not None:
                audio[d].append(got)
            while (s := e.fetch_spectrum(d)) is not None:
                spectra[d].append(s)
            while (c := e.fetch_carrier(d)) is not None:
                car[d].append(c)
            while fetch_readings and (r := e.fetch_input_levels(d)) is not None:
                levels[d].append(r)
        for m in range(len(mix)):
            while (got := e.fetch_mixer(m)) is not None:
                mix[m].append(got)
    stats = [[tuple(getattr(e.stats(d, c), f) for f in STAT_FIELDS) for c in range(len(cfg.devices[d].channels))] for d in range(D)]
    return dict(audio=audio, spectra=spectra, car=car, levels=levels, mix=mix, stats=stats,
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
        assert len(a["car"][d]) == len(b["car"][d])
        for (l1, e1, s1), (l2, e2, s2) in zip(a["car"][d], b["car"][d]):
            assert np.array_equal(l1.view(np.uint64), l2.view(np.uint64)) and np.array_equal(e1.view(np.uint32), e2.view(np.uint32)) and s1 == s2
    assert a["stats"] == b["stats"]
    assert len(a["mix"]) == len(b["mix"])
    for m1, m2 in zip(a["mix"], b["mix"]):
        assert len(m1) == len(m2) > 0
        for (l1, r1, s1), (l2, r2, s2) in zip(m1, m2):
            assert np.array_equal(l1.view(np.uint32), l2.view(np.uint32)) and np.array_equal(r1.view(np.uint32), r2.view(np.uint32)) and s1 == s2


def one_device(sfmt, sr=2560000, n=2048, fullscale=0.0):
    w = 8000
    ch = cm.make_channel(100000, 0, sr, n, w)
    return cm.Config(fft_size=n, wave_rate=w, devices=[cm.Device(sample_rate=sr, sfmt=sfmt, centerfreq=0, channels=[ch], fullscale=fullscale)])


def random_stream(cfg, dev, nb, seed):
    """Every code of the format (S16: every code in +-2.2 full scales; F32: levels out to +-1.6 full scale, exact zeros)."""
    d = cfg.devices[dev]
    m = 2 * wl.samples_for_batches(cfg, dev, nb)
    rng = np.random.default_rng(seed)
    if d.sfmt == cm.SFMT_U8:
        return rng.integers(0, 256, m).astype(np.uint8)
    if d.sfmt == cm.SFMT_S8:
        return rng.integers(-128, 128, m).astype(np.int8)
    if d.sfmt == cm.SFMT_S16:
        lim = min(32767, int(2.2 * d.fullscale))
        return rng.integers(-lim - 1, lim + 1, m).astype(np.int16)
    x = (rng.standard_normal(m) * 0.5 * d.fullscale).astype(np.float32)
    x[::97] = 0.0
    x[1::89] = f32(1.6 * d.fullscale)
    return x


# ---- 1. exact against numpy, every format ------------------------------------------------------------------------------
FORMATS = [("u8", cm.SFMT_U8, 0.0), ("s8", cm.SFMT_S8, 0.0), ("s16", cm.SFMT_S16, 32766.5), ("s16_fs2048", cm.SFMT_S16, 2048.0),
           ("f32", cm.SFMT_F32, 1.0), ("f32_fs3", cm.SFMT_F32, 3.0)]


@pytest.mark.parametrize("name,sfmt,fs", FORMATS, ids=[f[0] for f in FORMATS])
@pytest.mark.parametrize("sr", [2560000, 2500000])
def test_exact_against_numpy_every_format(name, sfmt, fs, sr):
    cfg = one_device(sfmt, sr=sr, fullscale=fs)
    nb = 3
    raw = random_stream(cfg, 0, nb, seed=sfmt * 7 + sr % 1000)
    out, e = drive(cfg, [raw], meter=[0], nbmax=2)
    got = out["levels"][0]
    assert [r["batch_seq"] for r in got] == list(range(nb))
    for r in got:
        check_exact(cfg, 0, raw, r)
    if sfmt in (cm.SFMT_S16, cm.SFMT_F32):  # levels beyond full scale land in the end bins, and the peak shows them
        assert all(r["peak"].min() > 1.0 and r["hist"][:, 0].min() > 0 and r["hist"][:, 255].min() > 0 for r in got)
    e.close()


def test_hand_built_extremes():
    """Every U8 code once per batch position pattern, constant streams, and S8 -128 / 127."""
    for sfmt, codes in ((cm.SFMT_U8, np.arange(256, dtype=np.uint8)), (cm.SFMT_S8, np.array([-128, 127, 0, -1], np.int8)),
                        (cm.SFMT_S16, np.array([-32768, 32767, 0, 1, -1], np.int16))):
        cfg = one_device(sfmt)
        m = 2 * wl.samples_for_batches(cfg, 0, 2)
        raw = np.resize(codes, m)
        out, e = drive(cfg, [raw], meter=[0], nbmax=1)
        assert len(out["levels"][0]) == 2
        for r in out["levels"][0]:
            check_exact(cfg, 0, raw, r)
        e.close()


# ---- 2. batch mapping --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sr", [2560000, 2500000])
@pytest.mark.parametrize("sfmt", [cm.SFMT_U8, cm.SFMT_S16])
def test_each_batch_covers_exactly_its_samples(sr, sfmt):
    """Batch b's samples carry code pattern b, the AGC look-back another and the unread tail a third: an error of one
    sample, one hop or AGC_EXTRA frames shows as a stray bin."""
    cfg = one_device(sfmt, sr=sr)
    hop, B, nb = cfg.hop(0), cfg.wave_batch, 5
    if sr == 2500000:
        assert hop == 313  # the batches' byte ranges are not 16-byte aligned
    m = wl.samples_for_batches(cfg, 0, nb)
    dt = np.uint8 if sfmt == cm.SFMT_U8 else np.int16
    raw = np.full((m, 2), 250 if sfmt == cm.SFMT_U8 else 32000, dt)
    raw[:AGC_EXTRA * hop] = 3 if sfmt == cm.SFMT_U8 else -32000
    for b in range(nb):
        s0 = (AGC_EXTRA + b * B) * hop
        raw[s0:s0 + B * hop, 0] = 10 + 20 * b if sfmt == cm.SFMT_U8 else 1000 * (b + 1)
        raw[s0:s0 + B * hop, 1] = 200 - 20 * b if sfmt == cm.SFMT_U8 else -1000 * (b + 1)
        raw[s0, 1] = 0 if sfmt == cm.SFMT_U8 else -32768           # first sample of the batch
        raw[s0 + B * hop - 1, 0] = 255 if sfmt == cm.SFMT_U8 else 32767  # last sample of the batch
    raw = raw.reshape(-1)
    out, e = drive(cfg, [raw], meter=[0], nbmax=2)
    got = out["levels"][0]
    assert [r["batch_seq"] for r in got] == list(range(nb))
    for r in got:
        check_exact(cfg, 0, raw, r)
        assert r["n_samples"] == B * hop
        assert [np.count_nonzero(r["hist"][k]) for k in range(2)] == [2, 2]
        assert r["hist"][0].sum() == r["hist"][1].sum() == B * hop
    e.close()


# ---- 3. known impairments ----------------------------------------------------------------------------------------------
def _u8_stream(cfg, nb, i_of_t, q_of_t, dither=1.5):
    """Levels i_of_t(t), q_of_t(t) in full scale, quantised like an ADC with `dither` codes of Gaussian noise: without
    it the rounding error of a tone has a mean of its own, a few hundredths of a code."""
    m = wl.samples_for_batches(cfg, 0, nb)
    t = np.arange(m, dtype=np.float64)
    rng = np.random.default_rng(17)
    x = np.empty((m, 2), np.uint8)
    x[:, 0] = np.clip(np.round(127.5 + 127.5 * i_of_t(t) + dither * rng.standard_normal(m)), 0, 255)
    x[:, 1] = np.clip(np.round(127.5 + 127.5 * q_of_t(t) + dither * rng.standard_normal(m)), 0, 255)
    return x.reshape(-1)


def _readings(cfg, raw, nb):
    out, e = drive(cfg, [raw], meter=[0], nbmax=4)
    e.close()
    got = out["levels"][0]
    assert [r["batch_seq"] for r in got] == list(range(nb))
    return got


def test_known_impairments_are_recovered():
    cfg = one_device(cm.SFMT_U8)
    nb = 3
    w = 2 * np.pi * 3951 / (cfg.wave_batch * cfg.hop(0))  # whole cycles in every batch: the tone's own means are zero
    a = 0.6
    # DC offset
    dc = (0.0213, -0.0377)
    for r in _readings(cfg, _u8_stream(cfg, nb, lambda t: dc[0] + a * np.cos(w * t), lambda t: dc[1] + a * np.sin(w * t)), nb):
        lv = lib.input_levels(r)
        assert np.all(np.abs(lv["dc_offset"] - dc) <= 1e-4), lv["dc_offset"]
        assert abs(lv["imbalance_db"]) <= 0.01 and abs(lv["phase_skew_deg"]) <= 0.05
    # 1 dB amplitude imbalance, then 3 degrees of phase skew
    g = 10 ** (-1.0 / 20)
    for r in _readings(cfg, _u8_stream(cfg, nb, lambda t: a * np.cos(w * t), lambda t: a * g * np.sin(w * t)), nb):
        assert abs(lib.input_levels(r)["imbalance_db"] - 1.0) <= 0.01
    phi = np.radians(3.0)
    for r in _readings(cfg, _u8_stream(cfg, nb, lambda t: a * np.cos(w * t), lambda t: a * np.sin(w * t + phi)), nb):
        lv = lib.input_levels(r)
        assert abs(lv["phase_skew_deg"] - 3.0) <= 0.05 and abs(lv["imbalance_db"]) <= 0.01, lv
    # a tone overdriven to 1.5 full scale, clipped by the generator
    raw = _u8_stream(cfg, nb, lambda t: 1.5 * np.cos(w * t), lambda t: 1.5 * np.sin(w * t), dither=0.0)
    for r in _readings(cfg, raw, nb):
        x = batch_samples(cfg, 0, raw, r["batch_seq"])
        clipped = np.count_nonzero((x == 0) | (x == 255), axis=0)
        assert np.all(clipped > 0.3 * r["n_samples"])
        assert np.array_equal(np.round(lib.input_levels(r)["full_scale_fraction"] * r["n_samples"]).astype(np.int64), clipped)
        assert np.array_equal(r["peak"], np.ones(2, np.float32))
    # low-gain noise: sigma = 2 codes
    rng = np.random.default_rng(3)
    m = wl.samples_for_batches(cfg, 0, nb)
    raw = np.clip(np.round(127.5 + 2.0 * rng.standard_normal(2 * m)), 0, 255).astype(np.uint8)
    for r in _readings(cfg, raw, nb):
        x = batch_samples(cfg, 0, raw, r["batch_seq"])
        lv = lib.input_levels(r)
        assert list(lv["codes_in_use"]) == [len(np.unique(x[:, k])) for k in range(2)]
        assert max(lv["codes_in_use"]) <= 24
        check_exact(cfg, 0, raw, r)


# ---- 4. segmentation independence --------------------------------------------------------------------------------------
@pytest.mark.parametrize("sfmt,sr", [(cm.SFMT_U8, 2500000), (cm.SFMT_F32, 2560000), (cm.SFMT_S16, 2500000)])
def test_readings_do_not_depend_on_run_grouping_or_pushes(sfmt, sr):
    cfg = one_device(sfmt, sr=sr)
    nb = 5
    raw = random_stream(cfg, 0, nb, seed=11)
    ref = None
    for nbmax in (1, 2, 4):
        out, e = drive(cfg, [raw], meter=[0], nbmax=nbmax)
        got = out["levels"][0]
        assert [r["batch_seq"] for r in got] == list(range(nb))
        if ref is None:
            ref = got
        for a, b in zip(got, ref):
            same_reading(a, b)
        e.close()
    # pushes of odd sizes into a small input buffer: abg_push compacts while the meter reads raw[]
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=3)
    e.input_meter_configure(0, True)
    rng = np.random.default_rng(5)
    pos, got = 0, {}
    while pos < raw.size or e.batches_available(0) > 0:
        if pos < raw.size:
            step = 2 * int(rng.integers(1, 90000))
            e.push(0, raw[pos:pos + step])
            pos += step
        e.run(-1)
        while e.fetch(0) is not None:
            pass
        while (x := e.fetch_input_levels(0)) is not None:
            got[x["batch_seq"]] = x
    assert sorted(got) == list(range(nb))
    for s in range(nb):
        same_reading(got[s], ref[s])
        check_exact(cfg, 0, raw, got[s])
    e.close()


# ---- 5. no other output changes ----------------------------------------------------------------------------------------
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
                                  "with_spectrum_and_carrier"])
def test_meter_changes_no_other_output(name):
    kw, scan, mixers, spectrum, carrier = {}, None, None, None, ()
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
    elif name == "with_spectrum_and_carrier":
        cfg, raws = CASES["s8_two_devices"](n_batches=3)
        spectrum = {0: 1, 1: lib.default_stride(cfg, 1)}
        carrier = (0, 1)
    else:
        cfg, raws = CASES[name]()
    D = len(cfg.devices)
    off, e0 = drive(cfg, raws, (), spectrum=spectrum, carrier=carrier, mixers=mixers, scan=scan, **kw)
    on, e1 = drive(cfg, raws, range(D), spectrum=spectrum, carrier=carrier, mixers=mixers, scan=scan, **kw)
    same_outputs(off, on)
    if name == "full_k1":
        assert set(on["paths"]) == {1}
    assert all(len(on["levels"][d]) == len(on["audio"][d]) for d in range(D))
    assert all(not r for r in off["levels"])
    for d in range(D):
        for r in on["levels"][d]:
            check_exact(cfg, d, raws[d], r)
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


# ---- 6. control and error paths ----------------------------------------------------------------------------------------
def test_only_metered_devices_produce_readings():
    cfg, raws = CASES["s8_two_devices"](n_batches=3)
    out, e = drive(cfg, raws, [1], nbmax=2)
    assert [r["batch_seq"] for r in out["levels"][1]] == [0, 1, 2]
    assert out["levels"][0] == [] and e.fetch_input_levels(0) is None
    e.close()


def test_switching_affects_exactly_the_later_runs():
    cfg, raws = CASES["am_u8"](n_batches=6)
    always, e_all = drive(cfg, raws, [0], nbmax=2)
    ref = {r["batch_seq"]: r for r in always["levels"][0]}
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=8)
    e.push(0, raws[0])
    seen = []
    for on in (False, True, False):
        e.input_meter_configure(0, on)
        assert e.run(2) == 2
        while e.fetch(0) is not None:
            pass
        while (x := e.fetch_input_levels(0)) is not None:
            seen.append(x)
    assert [r["batch_seq"] for r in seen] == [2, 3]
    for r in seen:
        same_reading(r, ref[r["batch_seq"]])
    e.close(); e_all.close()


def test_launch_count_unchanged_while_off_and_error_codes():
    cfg, raws = CASES["am_u8"](n_batches=2)
    counts = []
    for setup in ("untouched", "explicit_off", "on_then_off", "on"):
        e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=4)
        if setup == "explicit_off":
            e.input_meter_configure(0, False)
        elif setup == "on_then_off":
            e.input_meter_configure(0, True)
            e.input_meter_configure(0, False)
        elif setup == "on":
            e.input_meter_configure(0, True)
        e.push(0, raws[0])
        l0 = e.launch_count()
        assert e.run(-1) == 2
        e.sync()
        counts.append(e.launch_count() - l0)
        if setup != "on":
            assert e.fetch_input_levels(0) is None and e.input_meter_time() == 0.0
        else:
            assert e.input_meter_time() > 0.0
        if setup == "untouched":
            for args, code in (((5, 1), -5), ((-1, 1), -5), ((0, 2), -2), ((0, -1), -2)):
                with pytest.raises(lib.AbgError) as ei:
                    e._chk(e.L.abg_input_meter_configure(e.h, *args))
                assert ei.value.code == code
            with pytest.raises(lib.AbgError) as ei:
                e.fetch_input_levels(5)
            assert ei.value.code == -5
        e.close()
    assert counts[0] == counts[1] == counts[2] < counts[3]


def test_injected_batches_and_resident_runs_queue_nothing():
    cfg = wl.cfg1()
    e = lib.Engine(cfg, max_batches_per_run=2)
    e.input_meter_configure(0, True)
    assert e.inject_wavein(0, np.full((1, 2 * cfg.wave_batch), 5.0, np.float32)) == 2
    assert e.fetch(0) is not None and e.fetch_input_levels(0) is None and e.input_meter_time() == 0.0
    e.close()
    e = lib.Engine(cfg, max_batches_per_run=2)
    raw = wl.synth_iq(cfg, 0, wl.samples_for_batches(cfg, 0, 2), key_off_s=0.0)
    e.resident_load(0, raw)
    e.input_meter_configure(0, True)
    l0 = e.launch_count()
    e.run_resident(2)
    e.sync()
    assert e.input_meter_time() > 0.0 and e.launch_count() > l0  # computed ...
    assert e.fetch_input_levels(0) is None                       # ... but not queued
    e.close()


def test_streamed_readings_exact_after_resident_runs():
    """Resident runs leave the meter's work buffers clean: a streamed run after them is exact."""
    cfg = wl.cfg1()
    raw = wl.synth_iq(cfg, 0, wl.samples_for_batches(cfg, 0, 2), key_off_s=0.0)
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=4)
    e.resident_load(0, raw)
    e.input_meter_configure(0, True)
    for _ in range(3):
        e.run_resident(2)
    e.push(0, raw)
    assert e.run(-1) == 2
    got = []
    while (x := e.fetch_input_levels(0)) is not None:
        got.append(x)
    assert [r["batch_seq"] for r in got] == [0, 1]
    for r in got:
        check_exact(cfg, 0, raw, r)
    e.close()


def test_unfetched_readings_are_overwritten_oldest_first():
    cfg, raws = CASES["am_u8"](n_batches=10)
    nbmax = 4
    off, e0 = drive(cfg, raws, (), nbmax=nbmax)
    each, e1 = drive(cfg, raws, [0], nbmax=nbmax)
    lazy, e2 = drive(cfg, raws, [0], nbmax=nbmax, fetch_readings=False)
    assert lazy["runs"] == 3
    same_outputs(off, lazy)
    got = []
    while (x := e2.fetch_input_levels(0)) is not None:
        got.append(x)
    assert [r["batch_seq"] for r in got] == list(range(10 - (nbmax + 2), 10))
    ref = {r["batch_seq"]: r for r in each["levels"][0]}
    for r in got:
        same_reading(r, ref[r["batch_seq"]])
    for e in (e0, e1, e2):
        e.close()


# ---- 7. full size ------------------------------------------------------------------------------------------------------
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
        assert [r["batch_seq"] for r in on["levels"][d]] == list(range(nb))
        if np.array_equal(raws[d], raws[d % 4]):  # identical streams give bit-identical readings wherever the device sits
            for a, b in zip(on["levels"][d], on["levels"][d % 4]):
                same_reading(a, b)
    for d in (0, 1, 2, 3, D - 1):
        for r in on["levels"][d]:
            check_exact(cfg, d, raws[d], r)
    e0.close(); e1.close()


# ---- 8. hop > fft_size: a batch's samples reach past its last frame -------------------------------------------------------
@pytest.mark.parametrize("sfmt,sr,fs", [(cm.SFMT_U8, 3200000, 0.0), (cm.SFMT_F32, 2560000, 1.0), (cm.SFMT_S16, 10000000, 2048.0)],
                         ids=["u8_hop400", "f32_hop320", "s16_hop1250"])
def test_hop_longer_than_the_frame(sfmt, sr, fs):
    """With hop > fft_size the meter reads the samples between frames, past the end of the last frame of a batch: streamed
    readings stay exact, and resident runs (whose buffer holds exactly the bytes the frames need) stay inside their
    allocation and leave the meter's work buffers clean."""
    cfg = one_device(sfmt, sr=sr, n=256, fullscale=fs)
    hop, B, nb = cfg.hop(0), cfg.wave_batch, 2
    assert hop > cfg.fft_size
    raw = random_stream(cfg, 0, nb, seed=hop)
    out, e = drive(cfg, [raw], meter=[0], nbmax=nb)
    got = out["levels"][0]
    assert [r["batch_seq"] for r in got] == list(range(nb))
    for r in got:
        check_exact(cfg, 0, raw, r)
    e.close()
    e = lib.Engine(cfg, max_batches_per_run=nb, input_capacity_batches=nb + 2)
    need = e.resident_bytes_needed(0)
    bpc = 2 * cfg.devices[0].bytes_per_sample
    if sfmt == cm.SFMT_S16:  # the meter's resident range ends well past the bytes the frames need (and past any pad)
        assert (AGC_EXTRA + nb * B) * hop * bpc > need + 256
    e.resident_load(0, raw[:need // cfg.devices[0].bytes_per_sample])
    e.input_meter_configure(0, True)
    for _ in range(3):
        e.run_resident(nb)
    e.sync()
    assert e.input_meter_time() > 0.0 and e.fetch_input_levels(0) is None
    e.push(0, raw)
    assert e.run(-1) == nb
    got = []
    while e.fetch(0) is not None:
        pass
    while (x := e.fetch_input_levels(0)) is not None:
        got.append(x)
    assert [r["batch_seq"] for r in got] == list(range(nb))
    for r in got:
        check_exact(cfg, 0, raw, r)
    e.close()
