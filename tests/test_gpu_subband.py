"""Sub-band I/Q outputs (abg_subband_configure / abg_fetch_subband) on the GPU (-m gpu).

Reference: numpy float64 over the pushed stream, from the definition in airband_b200.h: float32 levels v[s], the
exact integer phase, y[m] = sum_j h[j] v[mD - j] exp(-2 pi i (delta (mD - j) mod 2^32) / 2^32), samples before the
output's first batch taken as zero.  Each output is checked against the worst-case float32 bound
8 L 2^-24 sum|h| max|v|, and the rms error against a much tighter figure.  Outputs must be bitwise independent of run
grouping, push sizes, compaction, fft_mode and the other outputs in the launch, and must leave every other output of the
engine bit-identical."""
import numpy as np
import pytest
from scipy.signal import fftconvolve

from airband_b200 import config as cm
from airband_b200 import lib
from airband_b200 import workloads as wl
from cases import CASES

pytestmark = pytest.mark.gpu
AGC_EXTRA = 100
EPS = 2.0 ** -24
STAT_FIELDS = [f for f, _ in cm.CSquelchStats._fields_]
f32 = np.float32


# ---- fixtures ----------------------------------------------------------------------------------------------------------
def one_device(sfmt, sr=2560000, n=2048, fullscale=0.0, afc=0):
    w, cf = 8000, 120000000
    ch = cm.make_channel(cf + 100000, cf, sr, n, w, afc=afc) if afc else cm.make_channel(100000, 0, sr, n, w)
    return cm.Config(fft_size=n, wave_rate=w, devices=[cm.Device(sample_rate=sr, sfmt=sfmt, centerfreq=cf if afc else 0,
                                                                  channels=[ch], fullscale=fullscale)])


def random_stream(cfg, dev, nb, seed):
    d = cfg.devices[dev]
    m = 2 * wl.samples_for_batches(cfg, dev, nb)
    rng = np.random.default_rng(seed)
    if d.sfmt == cm.SFMT_U8:
        return rng.integers(0, 256, m).astype(np.uint8)
    if d.sfmt == cm.SFMT_S8:
        return rng.integers(-128, 128, m).astype(np.int8)
    if d.sfmt == cm.SFMT_S16:
        return rng.integers(-32768, 32768, m).astype(np.int16)
    return (rng.standard_normal(m) * 0.5 * d.fullscale).astype(np.float32)


def levels(cfg, dev, raw):
    """complex128 of the float32 levels v[s] of the whole stream."""
    d = cfg.devices[dev]
    x = raw.reshape(-1, 2)
    if d.sfmt == cm.SFMT_U8:
        v = (x.astype(f32) - f32(127.5)) / f32(127.5)
    elif d.sfmt == cm.SFMT_S8:
        v = x.astype(f32) / f32(128.0)
    else:
        v = (f32(1.0) / f32(d.fullscale)) * x.astype(f32)
    assert v.dtype == np.float32
    return v[:, 0].astype(np.float64) + 1j * v[:, 1].astype(np.float64)


def delta_of(offset_hz, sr):
    x = offset_hz / sr * 2.0 ** 32
    return (int(np.floor(abs(x) + 0.5)) * (1 if x >= 0 else -1)) % (1 << 32)


def reference(cfg, dev, raw, offset_hz, decim, h, start):
    """y[m] for every m with mD inside the stream, float64; samples before `start` are zero."""
    v = levels(cfg, dev, raw)
    s = np.arange(v.size, dtype=np.uint64)
    ph = (np.uint64(delta_of(offset_hz, cfg.devices[dev].sample_rate)) * s) % np.uint64(1 << 32)
    w = v * np.exp(-2j * np.pi * ph.astype(np.float64) / 2.0 ** 32)
    w[:start] = 0.0
    conv = fftconvolve(w, np.asarray(h, np.float64))[:v.size]
    return conv, float(np.abs(v).max())


def batch_range(cfg, dev, seq, decim):
    hop, B = cfg.hop(dev), cfg.wave_batch
    s0 = (AGC_EXTRA + seq * B) * hop
    return -(-s0 // decim), -(-(s0 + B * hop) // decim)


def check_against_reference(cfg, dev, raw, got, offset_hz, decim, h, start, c=8.0, rms_c=4.0):
    conv, vmax = reference(cfg, dev, raw, offset_hz, decim, h, start)
    L = len(h)
    scale = EPS * float(np.abs(np.asarray(h, np.float64)).sum()) * max(vmax, 1e-30)
    errs = []
    for y, seq, first in got:
        m0, m1 = batch_range(cfg, dev, seq, decim)
        assert first == m0 and y.size == m1 - m0, (seq, first, m0, y.size, m1 - m0)
        want = conv[np.arange(m0, m1) * decim]
        err = np.abs(y.astype(np.complex128) - want)
        assert err.max() <= c * L * scale, (seq, err.max() / scale, L)
        errs.append(err)
    e = np.concatenate(errs)
    assert np.sqrt(np.mean(e ** 2)) <= rms_c * np.sqrt(L + 32) * scale, (np.sqrt(np.mean(e ** 2)) / scale, L)


def drive(cfg, raws, outputs, nbmax=4, capacity=None, fetch_subband=True, **kw):
    """Push every stream, run to exhaustion, fetch everything.  outputs = {(dev, k): (offset_hz, decim, h)}."""
    total = max(r.size // (2 * cfg.hop(d)) // cfg.wave_batch for d, r in enumerate(raws)) + 2
    e = lib.Engine(cfg, max_batches_per_run=nbmax, input_capacity_batches=capacity or total, **kw)
    for (d, k), (off, dec, h) in outputs.items():
        e.subband_configure(d, k, off, dec, h)
    for d, r in enumerate(raws):
        e.push(d, r)
    D = len(cfg.devices)
    audio = [[] for _ in range(D)]
    sb = {key: [] for key in outputs}
    runs = 0
    while True:
        n = e.run(-1)
        if n == 0:
            break
        runs += 1
        for d in range(D):
            while (got := e.fetch(d)) is not None:
                audio[d].append(got)
        for (d, k) in outputs:
            while fetch_subband and (x := e.fetch_subband(d, k)) is not None:
                sb[(d, k)].append(x)
    stats = [[tuple(getattr(e.stats(d, c), f) for f in STAT_FIELDS) for c in range(len(cfg.devices[d].channels))] for d in range(D)]
    return dict(audio=audio, sb=sb, stats=stats, runs=runs), e


def same_batches(a, b):
    assert len(a) == len(b) > 0
    for (y1, s1, f1), (y2, s2, f2) in zip(a, b):
        assert s1 == s2 and f1 == f2 and np.array_equal(y1.view(np.uint64), y2.view(np.uint64)), s1


def lowpass(L, fs, cutoff=20000.0):
    return lib.subband_lowpass(L, cutoff, fs, 60.0) if L > 1 else np.array([0.75], np.float32)


# ---- 1. against float64 ------------------------------------------------------------------------------------------------
FORMATS = [("u8", cm.SFMT_U8, 0.0), ("s8", cm.SFMT_S8, 0.0), ("s16", cm.SFMT_S16, 32766.5), ("f32", cm.SFMT_F32, 1.0)]
SHAPES = [  # (offset as a fraction of fs, decimation, L): D dividing WAVE_BATCH * hop = 320000 or not, L = 1 and 4096
    (0.0, 32, 255), (-0.0371, 7, 1), (0.5, 997, 4096), (-0.5, 40, 33), (0.2113, 1, 64)]


@pytest.mark.parametrize("name,sfmt,fs", FORMATS, ids=[f[0] for f in FORMATS])
@pytest.mark.parametrize("frac,decim,L", SHAPES, ids=[f"off{s[0]}_D{s[1]}_L{s[2]}" for s in SHAPES])
def test_against_float64(name, sfmt, fs, frac, decim, L):
    cfg = one_device(sfmt, fullscale=fs)
    sr = cfg.devices[0].sample_rate
    assert (cfg.wave_batch * cfg.hop(0)) % 32 == 0 and (cfg.wave_batch * cfg.hop(0)) % 7 != 0
    nb = 3
    raw = random_stream(cfg, 0, nb, seed=sfmt * 13 + decim)
    h = lowpass(L, sr) if L != 64 else np.random.default_rng(1).standard_normal(64).astype(np.float32)
    off = frac * sr
    out, e = drive(cfg, [raw], {(0, 0): (off, decim, h)}, nbmax=2)
    got = out["sb"][(0, 0)]
    assert [s for _, s, _ in got] == list(range(nb))
    check_against_reference(cfg, 0, raw, got, off, decim, h, start=AGC_EXTRA * cfg.hop(0))
    e.close()


# ---- 2. semantics: a carrier at f through an output at f - 1 kHz is a +1 kHz tone ----------------------------------------
@pytest.mark.parametrize("f", [310000.0, -505000.0])
def test_carrier_appears_at_plus_one_khz(f):
    cfg = one_device(cm.SFMT_F32, fullscale=1.0)
    sr = cfg.devices[0].sample_rate
    m = wl.samples_for_batches(cfg, 0, 2)
    A = 0.3
    t = np.arange(m, dtype=np.float64)
    x = A * np.exp(2j * np.pi * f * t / sr)
    raw = np.stack([x.real, x.imag], 1).astype(np.float32).reshape(-1)
    h = lib.subband_lowpass(2047, 20000.0, sr, 70.0)  # 1 kHz lies in the flat passband
    decim = 32
    out, e = drive(cfg, [raw], {(0, 3): (f - 1000.0, decim, h)}, nbmax=2)
    y = np.concatenate([b[0] for b in out["sb"][(0, 3)]])[len(h):]  # past the start-up transient
    rate = sr / decim
    step = np.angle(y[1:] * np.conj(y[:-1]))
    assert np.all(step > 0)  # positive frequency: the sign convention
    fout = np.median(step) * rate / (2 * np.pi)
    want = f - lib.subband_frequency(f - 1000.0, sr)
    assert abs(fout - want) <= 0.01 and abs(want - 1000.0) <= 0.01, (fout, want)
    amp = A * float(np.sum(h.astype(np.float64)))
    assert np.all(np.abs(np.abs(y) - amp) <= 1e-3 * amp), (np.abs(y).min(), np.abs(y).max(), amp)
    e.close()


# ---- 3. reproducibility ------------------------------------------------------------------------------------------------
def _three_format_case(nb=4):
    sr, n, w = 2560000, 2048, 8000
    devs = [cm.Device(sample_rate=sr, sfmt=s, centerfreq=0, channels=[cm.make_channel(100000, 0, sr, n, w)], fullscale=fs)
            for s, fs in ((cm.SFMT_U8, 0.0), (cm.SFMT_S16, 2048.0), (cm.SFMT_F32, 3.0))]
    cfg = cm.Config(fft_size=n, wave_rate=w, devices=devs)
    raws = [random_stream(cfg, d, nb, seed=40 + d) for d in range(3)]
    outs = {(0, 0): (-100000.0, 32, lowpass(255, sr)), (0, 5): (640000.0, 13, lowpass(1000, sr, 5000.0)),
            (1, 2): (1280000.0, 64, lowpass(4096, sr, 2000.0)), (2, 0): (12345.6, 1, lowpass(17, sr)),
            (2, 7): (-1279000.0, 320000, lowpass(255, sr))}
    return cfg, raws, outs


def test_bitwise_across_grouping_pushes_fft_modes_and_launch_composition():
    cfg, raws, outs = _three_format_case()
    ref, e = drive(cfg, raws, outs, nbmax=4)
    e.close()
    for key, (off, dec, h) in outs.items():
        d = key[0]
        assert [s for _, s, _ in ref["sb"][key]] == list(range(4))
        check_against_reference(cfg, d, raws[d], ref["sb"][key], off, dec, h, start=AGC_EXTRA * cfg.hop(d))
    for nbmax in (1, 2):
        got, e = drive(cfg, raws, outs, nbmax=nbmax)
        for key in outs:
            same_batches(got["sb"][key], ref["sb"][key])
        e.close()
    for mode in (1, 2, 3):
        got, e = drive(cfg, raws, outs, nbmax=4, fft_mode=mode)
        for key in outs:
            same_batches(got["sb"][key], ref["sb"][key])
        e.close()
    # each output alone on its device, the device alone in the launch
    for key, spec in outs.items():
        d = key[0]
        solo_cfg = cm.Config(fft_size=cfg.fft_size, wave_rate=cfg.wave_rate, devices=[cfg.devices[d]])
        got, e = drive(solo_cfg, [raws[d]], {(0, key[1]): spec}, nbmax=2)
        same_batches(got["sb"][(0, key[1])], ref["sb"][key])
        e.close()
    # odd pushes into a small input buffer: every run compacts, and the filters' history must survive it
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=3)
    for (d, k), (off, dec, h) in outs.items():
        e.subband_configure(d, k, off, dec, h)
    rng = np.random.default_rng(5)
    pos = [0] * 3
    got = {key: {} for key in outs}
    runs = 0
    while any(pos[d] < raws[d].size for d in range(3)) or any(e.batches_available(d) for d in range(3)):
        for d in range(3):
            if pos[d] < raws[d].size:
                step = 2 * int(rng.integers(1, 90000))
                e.push(d, raws[d][pos[d]:pos[d] + step])
                pos[d] += step
        if e.run(-1) > 0:
            runs += 1
        for d in range(3):
            while e.fetch(d) is not None:
                pass
        for key in outs:
            while (x := e.fetch_subband(*key)) is not None:
                got[key][x[1]] = x
    assert runs >= 3
    for key in outs:
        assert sorted(got[key]) == list(range(4))
        same_batches([got[key][s] for s in range(4)], ref["sb"][key])
    e.close()


def test_afc_device_one_batch_per_run_is_bitwise_equal():
    cfg = one_device(cm.SFMT_U8, n=512, afc=2)
    plain = one_device(cm.SFMT_U8, n=512)
    raw = random_stream(cfg, 0, 5, seed=9)
    outs = {(0, 1): (-250000.0, 40, lowpass(255, 2560000))}
    a, e1 = drive(cfg, [raw], outs, nbmax=4)
    b, e2 = drive(plain, [raw], outs, nbmax=4)
    assert a["runs"] == 5 and b["runs"] == 2
    same_batches(a["sb"][(0, 1)], b["sb"][(0, 1)])
    e1.close(); e2.close()


# ---- 4. lifecycle ------------------------------------------------------------------------------------------------------
def test_switch_on_mid_stream_reconfigure_and_switch_off():
    cfg = one_device(cm.SFMT_S8)
    sr, hop, B = 2560000, cfg.hop(0), cfg.wave_batch
    raw = random_stream(cfg, 0, 8, seed=21)
    h = lowpass(255, sr)
    spec = (300000.0, 32, h)
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=10)
    e.push(0, raw)

    def run2():
        assert e.run(2) == 2
        while e.fetch(0) is not None:
            pass

    run2()                                     # batches 0, 1: off
    e.subband_configure(0, 0, *spec)
    run2()                                     # batches 2, 3: on from batch 2
    e.subband_configure(0, 0, *spec)           # the same configuration again restarts the output
    run2()                                     # batches 4, 5
    e.subband_configure(0, 0, 0.0, 0)          # off: batches 6, 7 produce nothing
    run2()
    got = []
    while (x := e.fetch_subband(0, 0)) is not None:  # queued entries stay fetchable after switch-off
        got.append(x)
    assert [s for _, s, _ in got] == [2, 3, 4, 5]
    check_against_reference(cfg, 0, raw, got[:2], *spec, start=(AGC_EXTRA + 2 * B) * hop)
    check_against_reference(cfg, 0, raw, got[2:], *spec, start=(AGC_EXTRA + 4 * B) * hop)
    # the restart shows: batch 4's first outputs differ from a run that never restarted
    cont, e2 = drive(cfg, [raw], {(0, 0): spec}, nbmax=2)
    ref = {s: y for y, s, _ in cont["sb"][(0, 0)]}
    assert not np.array_equal(got[2][0][:4], ref[4][:4]) and np.array_equal(got[2][0][-4:], ref[4][-4:])
    e.close(); e2.close()


def test_lossy_queue_drops_the_oldest_and_never_overflows():
    cfg, raws = CASES["am_u8"](n_batches=10)
    nbmax = 4
    outs = {(0, 0): (50000.0, 100, lowpass(63, 2560000))}
    each, e1 = drive(cfg, raws, outs, nbmax=nbmax)
    lazy, e2 = drive(cfg, raws, outs, nbmax=nbmax, fetch_subband=False)
    assert lazy["runs"] == 3
    got = []
    while (x := e2.fetch_subband(0, 0)) is not None:
        got.append(x)
    assert [s for _, s, _ in got] == list(range(10 - (nbmax + 2), 10))
    ref = {s: (y, s, f) for y, s, f in each["sb"][(0, 0)]}
    same_batches(got, [ref[s] for _, s, _ in got])
    # gaps show in first_index too: consecutive batches continue each other's output index
    firsts = [f + y.size for y, _, f in each["sb"][(0, 0)]]
    assert [f for _, _, f in each["sb"][(0, 0)]][1:] == firsts[:-1]
    assert got[0][2] > firsts[0]
    e1.close(); e2.close()


def test_resident_runs_and_injected_batches_queue_nothing():
    cfg = wl.cfg1()
    e = lib.Engine(cfg, max_batches_per_run=2)
    l_off = []
    for on in (False, True):
        if on:
            e.subband_configure(0, 0, 1000.0, 16, lowpass(31, cfg.devices[0].sample_rate))
        l0 = e.launch_count()
        assert e.inject_wavein(0, np.full((1, 2 * cfg.wave_batch), 5.0, np.float32)) == 2
        e.sync()
        l_off.append(e.launch_count() - l0)
        assert e.fetch(0) is not None and e.fetch(0) is not None
    assert l_off[0] == l_off[1] and e.fetch_subband(0, 0) is None and e.subband_time() == 0.0
    e.close()
    e = lib.Engine(cfg, max_batches_per_run=2)
    raw = wl.synth_iq(cfg, 0, wl.samples_for_batches(cfg, 0, 2), key_off_s=0.0)
    e.resident_load(0, raw)
    e.subband_configure(0, 0, 1000.0, 16, lowpass(4096, cfg.devices[0].sample_rate))
    for _ in range(3):
        e.run_resident(2)
    e.sync()
    assert e.subband_time() > 0.0 and e.fetch_subband(0, 0) is None
    # a streamed run afterwards starts the output at its first batch and is exact
    e.push(0, raw)
    assert e.run(-1) == 2
    got = []
    while (x := e.fetch_subband(0, 0)) is not None:
        got.append(x)
    assert [s for _, s, _ in got] == [0, 1]
    check_against_reference(cfg, 0, raw, got, 1000.0, 16, lowpass(4096, cfg.devices[0].sample_rate), start=AGC_EXTRA * cfg.hop(0))
    e.close()


def test_error_codes():
    cfg = wl.cfg1()
    e = lib.Engine(cfg, max_batches_per_run=2)
    sr, n = cfg.devices[0].sample_rate, cfg.wave_batch * cfg.hop(0)
    h = np.ones(4, np.float32)

    def code(dev, k, off, dec, nc, coeffs):
        with pytest.raises(lib.AbgError) as ei:
            e._chk(e.L.abg_subband_configure(e.h, dev, k, off, dec, nc, lib._ptr(coeffs)))
        return ei.value.code

    assert code(1, 0, 0.0, 4, 4, h) == -5 and code(-1, 0, 0.0, 4, 4, h) == -5
    assert code(0, 8, 0.0, 4, 4, h) == -5 and code(0, -1, 0.0, 4, 4, h) == -5
    assert code(0, 0, sr / 2 + 1, 4, 4, h) == -2 and code(0, 0, -sr / 2 - 1, 4, 4, h) == -2
    assert code(0, 0, float("nan"), 4, 4, h) == -2
    assert code(0, 0, 0.0, -1, 4, h) == -2 and code(0, 0, 0.0, n + 1, 4, h) == -2
    assert code(0, 0, 0.0, 4, 0, h) == -2 and code(0, 0, 0.0, 4, 4097, np.ones(4097, np.float32)) == -2
    assert code(0, 0, 0.0, 4, 4, None) == -2
    for bad in (np.inf, -np.inf, np.nan):
        hb = h.copy()
        hb[2] = bad
        assert code(0, 0, 0.0, 4, 4, hb) == -2
    # the limits themselves are accepted
    e.subband_configure(0, 0, sr / 2, n, np.ones(4096, np.float32))
    e.subband_configure(0, 1, -sr / 2, 1, np.ones(1, np.float32))
    for dev, k in ((1, 0), (0, 8), (-1, 0), (0, -1)):
        with pytest.raises(lib.AbgError) as ei:
            e._chk(e.L.abg_fetch_subband(e.h, dev, k, None, None, None, None))
        assert ei.value.code == -5
    with pytest.raises(lib.AbgError) as ei:
        e._chk(e.L.abg_debug_subband_time(e.h, None))
    assert ei.value.code == -2
    e.close()


# ---- 5. no effect on the rest ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["am_u8", "nfm_s16", "am_bw_f32", "s8_two_devices", "with_monitors"])
def test_outputs_change_nothing_else(name):
    if name == "with_monitors":
        cfg, raws = CASES["s8_two_devices"](n_batches=3)
    else:
        cfg, raws = CASES[name]()
    D = len(cfg.devices)
    outs = {(d, k): ((-0.3 + 0.25 * k) * cfg.devices[d].sample_rate, 32 + k,
                     lowpass(255 if k else 4096, cfg.devices[d].sample_rate, 0.01 * cfg.devices[d].sample_rate))
            for d in range(D) for k in range(3)}

    def run(with_outputs):
        e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=3)
        if name == "with_monitors":
            for d in range(D):
                e.spectrum_configure(d, 1)
                e.carrier_configure(d, True)
                e.input_meter_configure(d, True)
        if with_outputs:
            for (d, k), spec in outs.items():
                e.subband_configure(d, k, *spec)
        pos = [0] * D
        res = dict(audio=[], spec=[], car=[], inm=[], sb=0)
        while any(pos[d] < raws[d].size for d in range(D)) or any(e.batches_available(d) for d in range(D)):
            for d in range(D):
                if pos[d] < raws[d].size:
                    step = 2 * (cfg.wave_batch * cfg.hop(d) // 3 + 1)
                    e.push(d, raws[d][pos[d]:pos[d] + step])
                    pos[d] += step
            e.run(-1)
            for d in range(D):
                while (g := e.fetch(d)) is not None:
                    res["audio"].append((d, g[0].view(np.uint32).copy(), g[1].view(np.uint64).copy(), g[2].copy()))
                while (s := e.fetch_spectrum(d)) is not None:
                    res["spec"].append((d, s[0].view(np.uint32).copy(), s[1], s[2]))
                while (c := e.fetch_carrier(d)) is not None:
                    res["car"].append((d, c[0].view(np.uint64).copy(), c[1].view(np.uint32).copy(), c[2]))
                while (r := e.fetch_input_levels(d)) is not None:
                    res["inm"].append((d, r["batch_seq"], r["hist"].copy(), r["peak"].view(np.uint32).copy(),
                                       r["sum"].view(np.uint64).copy(), r["sum_sq"].view(np.uint64).copy(), r["sum_iq"]))
                for k in range(lib.SUBBAND_MAX):
                    while e.fetch_subband(d, k) is not None:
                        res["sb"] += 1
        res["stats"] = [[tuple(getattr(e.stats(d, c), f) for f in STAT_FIELDS) for c in range(len(cfg.devices[d].channels))]
                        for d in range(D)]
        e.close()
        return res

    off, on = run(False), run(True)
    assert off["sb"] == 0 and on["sb"] == 3 * len(on["audio"])  # three outputs per device, one entry per batch
    assert len(off["audio"]) == len(on["audio"]) > 0
    for a, b in zip(off["audio"], on["audio"]):
        assert a[0] == b[0] and all(np.array_equal(x, y) for x, y in zip(a[1:], b[1:]))
    for key in ("spec", "car", "inm"):
        assert len(off[key]) == len(on[key])
        for a, b in zip(off[key], on[key]):
            assert all(np.array_equal(x, y) for x, y in zip(a, b)), key
    assert off["stats"] == on["stats"]
    if name == "with_monitors":
        assert off["spec"] and off["car"] and off["inm"]


def test_launch_count_unchanged_while_off_and_one_upload_one_launch_when_on():
    cfg, raws = CASES["am_u8"](n_batches=2)
    counts = []
    for setup in ("untouched", "explicit_off", "on_then_off", "on", "two_on"):
        e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=4)
        sr = cfg.devices[0].sample_rate
        if setup == "explicit_off":
            e.subband_configure(0, 0, 0.0, 0)
        elif setup == "on_then_off":
            e.subband_configure(0, 0, 1000.0, 32, lowpass(255, sr))
            e.subband_configure(0, 0, 0.0, 0)
        elif setup in ("on", "two_on"):
            e.subband_configure(0, 0, 1000.0, 32, lowpass(255, sr))
            if setup == "two_on":
                e.subband_configure(0, 4, -1000.0, 8, lowpass(4096, sr))
        e.push(0, raws[0])
        l0 = e.launch_count()
        assert e.run(-1) == 2
        e.sync()
        counts.append(e.launch_count() - l0)
        if setup in ("on", "two_on"):
            assert e.subband_time() > 0.0 and e.fetch_subband(0, 0) is not None
        else:
            assert e.subband_time() == 0.0 and e.fetch_subband(0, 0) is None
        e.close()
    assert counts[0] == counts[1] == counts[2] and counts[3] == counts[4] == counts[0] + 2
