"""Band spectrum monitor (abg_spectrum_configure / abg_fetch_spectrum) on the GPU (-m gpu).

Reference: float64 numpy FFTs of the oracle's own float32 fftin (op.Oracle.debug_frame) for every selected frame, so the
check is independent of both the engine's and the oracle's FFT.  Switching the monitor on must leave every other output
bit-identical, and spectra must not depend on how batches are grouped into runs."""
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


def ref_spectrum(cfg, dev, raw, batch, stride):
    """P[k] of one batch of one device in float64, from the oracle's float32 conversion + window of each selected frame."""
    d = cfg.devices[dev]
    one = cm.Config(fft_size=cfg.fft_size, wave_rate=cfg.wave_rate, fm_demod=cfg.fm_demod, devices=[d])
    o = op.Oracle(one)
    N, B, hop = cfg.fft_size, cfg.wave_batch, cfg.hop(dev)
    acc = np.zeros(N)
    js = range(0, B, stride)
    for j in js:
        s0 = (AGC_EXTRA + batch * B + j) * hop
        fin, _ = o.debug_frame(0, raw[2 * s0:2 * (s0 + N)])
        acc += np.abs(np.fft.fft(fin.astype(np.complex128))) ** 2
    o.close()
    return acc / len(js)


def drive(cfg, raws, strides=None, nbmax=4, fetch_spectra=True, mixers=None, scan=None, **kw):
    """Push every stream, run to exhaustion and fetch everything: audio, I/Q, flags, mixers and (per run) spectra.
    scan = (dev, chan, freqs, [freq_idx per run]).  Returns a dict of outputs and the engine."""
    total = max(r.size // (2 * cfg.hop(d)) // cfg.wave_batch for d, r in enumerate(raws)) + 2
    e = lib.Engine(cfg, max_batches_per_run=nbmax, input_capacity_batches=total, **kw)
    for d, s in (strides or {}).items():
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
            while fetch_spectra and (s := e.fetch_spectrum(d)) is not None:
                spectra[d].append(s)
        for m in range(len(mix)):
            while (got := e.fetch_mixer(m)) is not None:
                mix[m].append(got)
    stats = [[tuple(getattr(e.stats(d, c), f) for f in STAT_FIELDS) for c in range(len(cfg.devices[d].channels))] for d in range(D)]
    return dict(audio=audio, spectra=spectra, mix=mix, stats=stats, paths=[e.fft_path(d) for d in range(D)], runs=runs), e


def same_outputs(a, b):
    assert a["paths"] == b["paths"]
    for d in range(len(a["audio"])):
        assert len(a["audio"][d]) == len(b["audio"][d]) > 0
        for (w1, i1, x1), (w2, i2, x2) in zip(a["audio"][d], b["audio"][d]):
            assert np.array_equal(w1.view(np.uint32), w2.view(np.uint32))
            assert np.array_equal(i1.view(np.uint64), i2.view(np.uint64))
            assert np.array_equal(x1, x2)
    assert a["stats"] == b["stats"]
    assert len(a["mix"]) == len(b["mix"])
    for m1, m2 in zip(a["mix"], b["mix"]):
        assert len(m1) == len(m2) > 0
        for (l1, r1, s1), (l2, r2, s2) in zip(m1, m2):
            assert np.array_equal(l1.view(np.uint32), l2.view(np.uint32)) and np.array_equal(r1.view(np.uint32), r2.view(np.uint32)) and s1 == s2


def by_seq(spectra):
    return {seq: (p, nf) for p, seq, nf in spectra}


# ---- 1. accuracy ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [256, 512, 1024, 2048, 4096, 8192])
@pytest.mark.parametrize("sfmt", [cm.SFMT_U8, cm.SFMT_S8, cm.SFMT_S16, cm.SFMT_F32])
def test_spectrum_matches_float64_every_size_and_format(n, sfmt):
    # 2.048 Msps divides every fft_size, and the carrier sits 0.0075..0.24 bins above a bin centre, so the configured bin
    # (the reference's ceil(...) - 1 rule, config.calc_bin) is the bin nearest the carrier
    sr, w = 2048000, 8000
    ch = cm.make_channel(96060, 0, sr, n, w)
    cfg = cm.Config(fft_size=n, wave_rate=w, devices=[cm.Device(sample_rate=sr, sfmt=sfmt, centerfreq=0, channels=[ch])])
    nb = 2
    raw = wl.synth_iq(cfg, 0, wl.samples_for_batches(cfg, 0, nb), key_off_s=0.0, seed=n + sfmt, amplitude=0.3, noise_sigma=0.05)
    for stride in sorted({1, lib.default_stride(cfg, 0)}):
        out, e = drive(cfg, [raw], {0: stride}, nbmax=4)
        got = out["spectra"][0]
        assert [s for _, s, _ in got] == list(range(nb))
        for p, seq, nf in got:
            assert nf == len(range(0, cfg.wave_batch, stride))
            ref = ref_spectrum(cfg, 0, raw, seq, stride)
            err = np.abs(p.astype(np.float64) - ref)
            assert np.all(err <= 1e-5 * ref + 1e-6 * ref.max()), (stride, seq, float((err / ref.max()).max()))
            assert int(np.argmax(p)) == ch.bin
        e.close()


# ---- 2. no behaviour change ----------------------------------------------------------------------------------------
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


@pytest.mark.parametrize("name", ["am_u8", "nfm_s16", "am_bw_f32", "s8_two_devices", "afc", "scan", "cfg4_mixers"])
def test_monitor_changes_no_other_output(name):
    kw, scan, mixers = {}, None, None
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
    else:
        cfg, raws = CASES[name]()
    off, e0 = drive(cfg, raws, None, mixers=mixers, scan=scan, **kw)
    strides = {d: (1 if d % 2 else lib.default_stride(cfg, d)) for d in range(len(cfg.devices))}
    on, e1 = drive(cfg, raws, strides, mixers=mixers, scan=scan, **kw)
    same_outputs(off, on)
    assert all(len(on["spectra"][d]) == len(on["audio"][d]) for d in range(len(cfg.devices)))
    assert all(not s for s in off["spectra"])
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


# ---- 3. segmentation independence -------------------------------------------------------------------------------------
def test_spectra_do_not_depend_on_run_grouping_or_pushes():
    cfg, raws = CASES["am_u8"](n_batches=4)
    strides = {0: 1}
    ref = None
    for nbmax in (1, 2, 4):
        out, e = drive(cfg, raws, strides, nbmax=nbmax)
        got = by_seq(out["spectra"][0])
        assert sorted(got) == [0, 1, 2, 3]
        if ref is None:
            ref = got
        for s in ref:
            assert np.array_equal(got[s][0].view(np.uint32), ref[s][0].view(np.uint32)), (nbmax, s)
        e.close()
    # pushes of odd sizes (as test_streaming_pushes_of_odd_sizes)
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=3)
    e.spectrum_configure(0, 1)
    rng = np.random.default_rng(3)
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
        while (s := e.fetch_spectrum(0)) is not None:
            got[s[1]] = s[0]
    assert sorted(got) == [0, 1, 2, 3]
    for s in ref:
        assert np.array_equal(got[s].view(np.uint32), ref[s][0].view(np.uint32)), s
    e.close()


# ---- 4. control ------------------------------------------------------------------------------------------------------
def test_only_monitored_devices_produce_spectra():
    cfg, raws = CASES["s8_two_devices"](n_batches=3)
    out, e = drive(cfg, raws, {0: lib.default_stride(cfg, 0)}, nbmax=2)
    assert [s for _, s, _ in out["spectra"][0]] == [0, 1, 2]
    assert out["spectra"][1] == [] and e.fetch_spectrum(1) is None
    e.close()


def test_switching_affects_exactly_the_later_runs():
    cfg, raws = CASES["am_u8"](n_batches=6)
    always, e_all = drive(cfg, raws, {0: 3}, nbmax=2)
    ref = by_seq(always["spectra"][0])
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=8)
    e.push(0, raws[0])
    seen = []
    for stride in (0, 3, 0):
        e.spectrum_configure(0, stride)
        assert e.run(2) == 2
        while e.fetch(0) is not None:
            pass
        while (s := e.fetch_spectrum(0)) is not None:
            seen.append(s)
    assert [s for _, s, _ in seen] == [2, 3]
    for p, s, nf in seen:
        assert np.array_equal(p.view(np.uint32), ref[s][0].view(np.uint32)) and nf == ref[s][1]
    e.close(); e_all.close()


def test_launch_count_unchanged_while_off_and_error_codes():
    cfg, raws = CASES["am_u8"](n_batches=2)
    counts = []
    for setup in ("untouched", "explicit_off", "on_then_off", "on"):
        e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=4)
        if setup == "explicit_off":
            e.spectrum_configure(0, 0)
        elif setup == "on_then_off":
            e.spectrum_configure(0, 1)
            e.spectrum_configure(0, 0)
        elif setup == "on":
            e.spectrum_configure(0, 1)
        e.push(0, raws[0])
        l0 = e.launch_count()
        assert e.run(-1) == 2
        e.sync()
        counts.append(e.launch_count() - l0)
        if setup != "on":
            assert e.fetch_spectrum(0) is None and e.spectrum_time() == 0.0
        else:
            assert e.spectrum_time() > 0.0
        if setup == "untouched":
            for args, code in (((5, 1), -5), ((-1, 1), -5), ((0, -1), -2)):
                with pytest.raises(lib.AbgError) as ei:
                    e.spectrum_configure(*args)
                assert ei.value.code == code
            with pytest.raises(lib.AbgError) as ei:
                e.fetch_spectrum(5)
            assert ei.value.code == -5
        e.close()
    assert counts[0] == counts[1] == counts[2] < counts[3]


def test_injected_batches_produce_no_spectrum():
    cfg = wl.cfg1()
    e = lib.Engine(cfg, max_batches_per_run=2)
    e.spectrum_configure(0, 1)
    assert e.inject_wavein(0, np.full((1, 2 * cfg.wave_batch), 5.0, np.float32)) == 2
    assert e.fetch(0) is not None and e.fetch_spectrum(0) is None
    e.close()


# ---- 5. lossy queue -------------------------------------------------------------------------------------------------
def test_unfetched_spectra_are_overwritten_oldest_first():
    cfg, raws = CASES["am_u8"](n_batches=10)
    nbmax = 4
    off, e0 = drive(cfg, raws, None, nbmax=nbmax)
    each, e1 = drive(cfg, raws, {0: 2}, nbmax=nbmax)
    lazy, e2 = drive(cfg, raws, {0: 2}, nbmax=nbmax, fetch_spectra=False)
    assert lazy["runs"] == 3
    same_outputs(off, lazy)
    assert len(lazy["audio"][0]) == 10
    got = []
    while (s := e2.fetch_spectrum(0)) is not None:
        got.append(s)
    assert [s for _, s, _ in got] == list(range(10 - (nbmax + 2), 10))
    ref = by_seq(each["spectra"][0])
    for p, s, _ in got:
        assert np.array_equal(p.view(np.uint32), ref[s][0].view(np.uint32))
    for e in (e0, e1, e2):
        e.close()


# ---- 6. full size --------------------------------------------------------------------------------------------------
def test_full_size_cfg2_every_device_monitored():
    import bench
    cfg, _ = bench.make_workload("cfg2")
    nb = 4
    raws = bench.synth_streams(cfg, nb, n_unique=4)
    D = len(cfg.devices)
    stride = lib.default_stride(cfg, 0)
    off, e0 = drive(cfg, raws, None, nbmax=nb)
    on, e1 = drive(cfg, raws, {d: stride for d in range(D)}, nbmax=nb)
    same_outputs(off, on)
    for d in range(D):
        assert [s for _, s, _ in on["spectra"][d]] == list(range(nb))
        for b in range(nb):  # identical streams give bit-identical spectra wherever the device sits in the launch
            assert np.array_equal(on["spectra"][d][b][0].view(np.uint32), on["spectra"][d % 4][b][0].view(np.uint32))
    for d in (0, 21, 42, 63):
        for p, seq, nf in on["spectra"][d]:
            ref = ref_spectrum(cfg, d, raws[d], seq, stride)
            assert nf == len(range(0, cfg.wave_batch, stride))
            assert np.all(np.abs(p - ref) <= 1e-5 * ref + 1e-6 * ref.max()), (d, seq)
    e0.close(); e1.close()


def test_spectrum_dbfs_restates_level_to_dbfs():
    """spectrum_dbfs(P) == the engine's level_to_dBFS on sqrt(P): the squelch levels' dBFS scale."""
    cfg, raws = CASES["am_u8"](n_batches=2)
    out, e = drive(cfg, raws, {0: 1}, nbmax=2)
    p = out["spectra"][0][-1][0]
    db = lib.spectrum_dbfs(p, cfg.fft_size)
    assert db.dtype == np.float32 and np.all(db <= 0.0)
    s = e.stats(0, 0)
    assert abs(float(lib.spectrum_dbfs(np.float32(s.noise_level) ** 2, cfg.fft_size)) - s.noise_level_dbfs) <= 1e-4
    e.close()
