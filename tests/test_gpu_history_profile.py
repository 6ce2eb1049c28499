"""Transmission profiles (abg_history_profile) on the GPU (-m gpu).

Every field must match float64 sums of the same outputs (Engine.history_subband) within the header's bound, for every
format, hop 313 at wave_rate 8008, decimation 1 and one above the capture's per-item limit, 1 and 4096 coefficients,
windows across the ring's wrap, n = 2 and a window longer than one chunk.  Readings must be bitwise the same for a job
alone or among many, in another order and between live runs; calls between runs must leave the live engine as a twin that
never calls them has it; every refusal has its code.  Through the engine, pushed streams must be classified by the CPU
model's rules, and end to end three unconfigured transmitters are found, profiled and replayed from the history alone."""
import numpy as np
import pytest

from airband_b200 import config as cm
from airband_b200 import lib
from test_gpu_activity import _all_monitors, fetch_monitors, quantize
from test_gpu_history_replay import parent_cfg
from test_history_profile_cpu import synth

pytestmark = pytest.mark.gpu
AGC = cm.AGC_EXTRA
W, CF = 8000, 120_000_000
U = 2.0 ** -24


def noise_raw(cfg, n_samples, txs, noise, seed):
    """Complex noise plus transmitters txs = [(offset_hz, amplitude, first sample, end sample, kind, x, voice, ctcss)],
    kind and x as in test_history_profile_cpu.synth (without its noise)."""
    d = cfg.devices[0]
    rng = np.random.default_rng(seed)
    x = rng.normal(0, noise, n_samples) + 1j * rng.normal(0, noise, n_samples)
    for f, a, s0, s1, kind, mx, voice, ctcss in txs:
        y = synth(kind, mx, voice, ctcss, f, d.sample_rate, s1 - s0, 200.0, np.ones(1), rng)
        x[s0:s1] += a * y
    return quantize(x, d.sfmt, d.fullscale)


def fill(cfg, raw, hist, nbmax=2, piece_batches=1.0, between=None, setup=None):
    e = lib.Engine(cfg, max_batches_per_run=nbmax)
    e.history_configure(0, hist)
    if setup:
        setup(e)
    step = int(piece_batches * cfg.wave_batch * cfg.hop(0)) * 2
    pos, out = 0, []
    while True:
        if pos < raw.size:
            e.push(0, raw[pos:pos + step])
            pos += step
        n = e.run(-1)
        while (g := e.fetch(0)) is not None:
            out.append(("batch", g[0].tobytes(), g[1].tobytes(), g[2].tobytes()))
        out += fetch_monitors(e, 0)
        if n and between:
            between(e)
        if n == 0 and pos >= raw.size:
            return e, out


def ref_sums(y, m0, fs_out, tones):
    """float64 sums of the definition's float32 terms with the exact phase, and the sums of their magnitudes."""
    y = np.asarray(y)
    u, v = y[:-1], y[1:]
    p = np.abs(y.astype(np.complex128)) ** 2
    a = np.sqrt(p)
    z = v.astype(np.complex128) * np.conj(u.astype(np.complex128))
    phi = np.angle(z)
    d = np.array([int(np.floor(float(np.float32(f)) / fs_out * 4294967296.0 + 0.5)) % (1 << 32) for f in tones], np.uint64)
    fm = np.zeros(len(tones), np.complex128)
    am = np.zeros(len(tones), np.complex128)
    phi0 = np.concatenate([phi, [0.0]])
    for c in range(0, y.size, 1 << 18):
        m = (np.uint64(m0) + np.arange(c, min(c + (1 << 18), y.size), dtype=np.uint64)) % np.uint64(1 << 32)
        ph = (d[:, None] * m[None, :]) % np.uint64(1 << 32)
        E = np.exp(-2j * np.pi * ph.astype(np.float64) / 4294967296.0)
        fm += E @ phi0[c:c + m.size]
        am += E @ a[c:c + m.size]
    uv = np.abs(u.astype(np.complex128)) * np.abs(v.astype(np.complex128))
    val = dict(p1=p.sum(), p2=(p * p).sum(), a1=a.sum(), z=z.sum(), f1=phi.sum(), f2=(phi * phi).sum(), tone_fm=fm, tone_am=am)
    mag = dict(p1=p.sum(), p2=(p * p).sum(), a1=a.sum(), z=uv.sum(), f1=np.abs(phi).sum(), f2=(phi * phi).sum(),
               tone_fm=np.abs(phi).sum(), tone_am=a.sum())
    return val, mag


def check_fields(got, y, m0, fs_out, tones):
    val, mag = ref_sums(y, m0, fs_out, tones)
    n = y.size
    assert got["n"] == n and got["tone_fm"].size == len(tones)
    # the header's bound plus the terms' own float32 error (p, a, z: a few ulp relative; phi: atan2f's ulps plus z's
    # rounding, 1e-6 rad at most)
    for k in ("p1", "p2", "a1", "z"):
        tol = (16 + 8) * U * mag[k]
        assert np.all(np.abs(np.asarray(got[k]) - val[k]) <= tol), (k, got[k], val[k], tol)
    assert abs(got["f1"] - val["f1"]) <= 24 * U * mag["f1"] + 1e-6 * n
    assert abs(got["f2"] - val["f2"]) <= 24 * U * mag["f2"] + 2 * np.pi * 1e-6 * n
    for k, slop in (("tone_fm", 1e-6 * n), ("tone_am", 0.0)):
        tol = (40 + 8) * U * mag[k] + slop
        dv = got[k] - val[k]
        assert np.all(np.abs(dv.real) <= tol) and np.all(np.abs(dv.imag) <= tol), (k, np.abs(dv).max(), tol)


# (name, format, sample rate, full scale, fft_size, wave_rate)
FORMATS = [("u8", cm.SFMT_U8, 2048000, 0.0, 2048, W), ("s8", cm.SFMT_S8, 2560000, 0.0, 2048, W),
           ("s16", cm.SFMT_S16, 2560000, 32766.5, 2048, W), ("f32", cm.SFMT_F32, 2048000, 1.0, 2048, W),
           ("u8_hop313", cm.SFMT_U8, 2506504, 0.0, 2048, 8008)]
NB, HIST = 14, 6


# ---- 1. every field against float64 ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,sfmt,sr,fs,n,w", FORMATS, ids=[c[0] for c in FORMATS])
def test_fields_match_float64(name, sfmt, sr, fs, n, w):
    cfg = parent_cfg(sfmt, sr, n, fs=fs, w=w)
    B, hop = cfg.wave_batch, cfg.hop(0)
    ns = (AGC + NB * B) * hop + n
    raw = noise_raw(cfg, ns, [(31_000.0, 0.3, 0, ns, "nfm", 2500.0, [900.0], 127.3), (-52_000.0, 0.2, 0, ns, "am", 0.6, [700.0], 88.5)],
                    0.02, seed=sfmt)
    e, _ = fill(cfg, raw, HIST)
    first, end = e.history_range(0)
    R = (HIST * B * hop * 2 * cfg.devices[0].bytes_per_sample + 15) & ~15
    D0, c0, L0 = lib.profile_filter(cfg, 0)
    cases = [(31_000.0, D0, lib.subband_lowpass(L0, c0, sr), None),                  # the default filter, standard tones
             (-52_000.0, 1, lib.subband_lowpass(4096, 20_000.0, sr), [88.5, 1000.0]),  # D = 1, L = 4096
             (0.0, 9001, np.ones(1, np.float32), [11.0, 50.0]),                       # above the per-item limit, L = 1
             (31_000.0, 77, np.array([0.25, 0.5, 0.25], np.float32), None)]
    jobs = []
    for off, D, h, tones in cases:
        L = h.size
        m_lo = -(-(first + L - 1) // D)
        m_hi = (end - 1) // D  # inclusive
        jobs.append(dict(dev=0, offset_hz=off, decim=D, coeffs=h, first_m=m_lo, n_out=m_hi - m_lo + 1, tones=tones))
        jobs.append(dict(jobs[-1], first_m=m_lo + (m_hi - m_lo) // 3, n_out=2))  # n = 2
    # the ring wraps inside the windows
    assert first * 2 * cfg.devices[0].bytes_per_sample // R != (end - 1) * 2 * cfg.devices[0].bytes_per_sample // R
    got = e.history_profile(jobs)
    for j, g in zip(jobs, got):
        y = e.history_subband(0, j["offset_hz"], j["decim"], j["coeffs"], j["first_m"], j["n_out"])
        tones = lib.STANDARD_TONES if j["tones"] is None else j["tones"]
        check_fields(g, y, j["first_m"], sr / j["decim"], tones)
    cap_ms, prof_ms = e.history_profile_time()
    assert cap_ms > 0 and prof_ms > 0
    e.close()


def test_window_longer_than_a_chunk():
    """10.5 s at D = 1: 21.5 M outputs, three chunks of the 8 M output scratch."""
    SR = 2048000
    cfg = parent_cfg(cm.SFMT_U8, SR, 2048)
    B, hop = cfg.wave_batch, cfg.hop(0)
    nb = 90
    ns = (AGC + nb * B) * hop + 2048
    raw = noise_raw(cfg, ns, [(1000.0, 0.3, 0, ns, "nfm", 2500.0, [900.0], 127.3)], 0.02, seed=4)
    e, _ = fill(cfg, raw, nb + 2, nbmax=8, piece_batches=8.0)
    first, end = e.history_range(0)
    n_out = end - first - 10
    assert n_out > 2 * (8 << 20) + 1000
    job = dict(dev=0, offset_hz=1000.0, decim=1, coeffs=np.ones(1, np.float32), first_m=first + 3, n_out=n_out, tones=[127.3, 200.0])
    g = e.history_profile([job])[0]
    y = e.history_subband(0, 1000.0, 1, job["coeffs"], job["first_m"], n_out)
    check_fields(g, y, job["first_m"], SR, job["tones"])
    e.close()


# ---- 2. bitwise reproducibility, 3. the live engine untouched ---------------------------------------------------------------------
def _key(r):
    return tuple(np.asarray(r[k]).tobytes() for k in ("n", "p1", "p2", "a1", "z", "f1", "f2", "tone_fm", "tone_am"))


def test_readings_are_reproducible_and_the_live_engine_untouched():
    cfg = parent_cfg(cm.SFMT_U8, 2048000, 2048)
    B, hop = cfg.wave_batch, cfg.hop(0)
    ns = (AGC + NB * B) * hop + 2048
    raw = noise_raw(cfg, ns, [(300_000.0, 0.3, 0, ns, "am", 0.6, [700.0], 88.5), (-100_000.0, 0.3, 0, ns, "nfm", 2500.0, [900.0], 127.3)],
                    0.02, seed=9)
    D, c, L = lib.profile_filter(cfg, 0)
    h = lib.subband_lowpass(L, c, 2048000)
    base = dict(dev=0, decim=D, coeffs=h, tones=None)

    def jobs_for(e):
        first, end = e.history_range(0)
        m_lo, m_hi = -(-(first + L - 1) // D), (end - 1) // D
        n = m_hi - m_lo + 1
        return [dict(base, offset_hz=300_000.0, first_m=m_lo, n_out=n), dict(base, offset_hz=-100_000.0, first_m=m_lo + 5, n_out=n - 5),
                dict(base, offset_hz=0.0, first_m=m_lo + n // 2, n_out=2), dict(base, offset_hz=-100_000.0, first_m=m_lo + 7, n_out=n // 3)]

    calls, counts = [], []

    def between(e):
        js = jobs_for(e)
        alone = [_key(e.history_profile([j])[0]) for j in js]
        together = [_key(r) for r in e.history_profile(js)]
        reverse = [_key(r) for r in e.history_profile(js[::-1])][::-1]
        assert alone == together == reverse
        calls.append(alone)

    setup = lambda e: _all_monitors(e, cfg)  # noqa: E731
    twin, out_twin = fill(cfg, raw, HIST, setup=setup)
    n_twin = twin.launch_count()
    e, out = fill(cfg, raw, HIST, setup=setup, between=between)
    assert len(calls) >= 4
    assert out == out_twin
    assert e.history_range(0) == twin.history_range(0)
    js, rng_final = jobs_for(e), e.history_range(0)
    final = [_key(r) for r in e.history_profile(js)]
    # per-run launches: the same in the last run, whatever the calls added
    n0 = e.launch_count()
    for x in (e, twin):
        x.push(0, raw[: 2 * B * hop * 2])
    e.run(-1)
    twin.run(-1)
    assert e.launch_count() - n0 == twin.launch_count() - n_twin
    # the same windows in another engine, pushed in other pieces with another max_batches_per_run
    e2, _ = fill(cfg, raw, HIST, nbmax=3, piece_batches=1.7)
    assert e2.history_range(0) == rng_final
    assert final == [_key(r) for r in e2.history_profile(js)]
    for x in (e, twin, e2):
        x.close()


# ---- 4. error codes ---------------------------------------------------------------------------------------------------------------
def test_error_codes():
    cfg = parent_cfg(cm.SFMT_U8, 2048000, 2048)
    B, hop = cfg.wave_batch, cfg.hop(0)
    ns = (AGC + 8 * B) * hop + 2048
    raw = noise_raw(cfg, ns, [], 0.02, seed=1)
    e, _ = fill(cfg, raw, 4)
    first, end = e.history_range(0)
    h = np.ones(5, np.float32)
    ok = dict(dev=0, offset_hz=0.0, decim=10, coeffs=h, first_m=-(-(first + 4) // 10), n_out=100, tones=None)

    def code(**kw):
        try:
            e.history_profile([dict(ok, **kw)])
            return 0
        except lib.AbgError as x:
            return x.code

    assert code() == 0
    assert code(dev=1) == -5 and code(dev=-1) == -5
    assert code(first_m=ok["first_m"] - 1) == -5                      # a tap before the history
    assert code(n_out=(end - 1) // 10 - ok["first_m"] + 2) == -5      # an output at the end
    assert code(n_out=(end - 1) // 10 - ok["first_m"] + 1) == 0
    assert code(n_out=1) == -2 and code(n_out=0) == -2
    assert code(decim=0) == -2 and code(decim=B * hop + 1) == -2
    assert code(coeffs=np.ones(4097, np.float32)) == -2 and code(coeffs=np.array([np.nan], np.float32)) == -2
    assert code(offset_hz=2048000.0) == -2
    assert code(tones=[0.0]) == -2 and code(tones=[np.inf]) == -2 and code(tones=[102400.0]) == -2
    assert code(tones=[100.0] * 65) == -2
    assert code(decim=5000) == -2  # fs_out 409.6 Hz: the standard tones above 204.8 Hz are refused
    L = e.L
    arr = (lib.CProfileJob * 1)()
    assert L.abg_history_profile(e.h, 0, arr) == -2 and L.abg_history_profile(e.h, 65536, arr) == -2
    assert L.abg_history_profile(e.h, 1, None) == -2
    arr[0] = lib.CProfileJob(0, 10, 0.0, 5, 0, h.ctypes.data, ok["first_m"], 100, None, None)
    assert L.abg_history_profile(e.h, 1, arr) == -2  # null out
    e.history_configure(0, 0)  # frees the profile buffers; the next call finds no history
    assert code() == -5
    e.close()


# ---- 5. classification through the engine -----------------------------------------------------------------------------------------
CLASSES = [("am", 0.6, [1000.0], 127.3, cm.MOD_AM), ("am", 0.3, [700.0, 1500.0, 2300.0], None, cm.MOD_AM),
           ("nfm", 2500.0, [1000.0], 67.0, cm.MOD_NFM), ("nfm", 5000.0, [450.0, 1200.0, 2700.0], 254.1, cm.MOD_NFM),
           ("carrier", 0.0, [], None, cm.MOD_AM)]
ENGINES = [(512, cm.SFMT_U8, 0.0), (2048, cm.SFMT_S16, 32766.5), (8192, cm.SFMT_U8, 0.0)]


@pytest.mark.parametrize("n,sfmt,fs", ENGINES, ids=["512_u8", "2048_s16", "8192_u8"])
def test_classification_through_the_engine(n, sfmt, fs):
    SR = 2048000
    cfg = parent_cfg(sfmt, SR, n, fs=fs)
    B, hop = cfg.wave_batch, cfg.hop(0)
    nb = 12
    ns = (AGC + nb * B) * hop + n
    bin_hz = SR // n
    spacing = 60_000.0
    A = 0.08
    txs = [(-150_000.0 + i * spacing, A, 0, ns, k, x, v, c) for i, (k, x, v, c, _) in enumerate(CLASSES)]
    # 20 dB in the profile filter's passband: white noise of 2 sigma^2 over the band puts 2 sigma^2 * 2 cutoff / SR there
    D, cutoff, L = lib.profile_filter(cfg, 0)
    sigma = A * np.sqrt(SR / (400.0 * cutoff))
    raw = noise_raw(cfg, ns, txs, sigma, seed=n)
    e, _ = fill(cfg, raw, nb + 2)
    hist = e.history_range(0)
    rng = np.random.default_rng(n)
    window = [dict(first_frame=AGC + 2 * B, last_frame=AGC + 10 * B)]
    tx_list = [dict(window[0], freq_hz=CF + f + float(rng.uniform(-bin_hz / 2, bin_hz / 2))) for f, *_ in txs]
    summaries = lib.history_profiles(e, cfg, 0, tx_list)
    for (f, _, _, _, kind, x, v, ctcss), (_, _, _, _, want), s in zip(txs, CLASSES, summaries):
        assert s["modulation"] == want, (kind, x, s)
        assert s["ctcss_hz"] == ctcss, (kind, x, s)
        tol = 20.0 if kind == "nfm" else 2.0
        assert abs(s["freq_hz"] - (CF + f)) <= tol, (kind, x, s["freq_hz"] - CF - f)
    e.close()


# ---- 6. end to end, nothing configured but the history ------------------------------------------------------------------------------
def test_find_profile_and_replay_three_unconfigured_transmitters():
    SR, n = 2048000, 2048
    bw = SR // n
    cfg = parent_cfg(cm.SFMT_U8, SR, n, channels=[cm.make_channel(CF + 700_000, CF, SR, n, W)])
    B, hop, nb = cfg.wave_batch, cfg.hop(0), 16
    ns = (AGC + nb * B) * hop + n
    f2s = lambda f: int(f * hop)  # noqa: E731
    extra = [(-222 * bw, AGC + 5 * B + 300, AGC + 10 * B + 460, "am", 0.6, 700.0, None, cm.MOD_AM),
             (77 * bw + 310.0, AGC + 6 * B + 100, AGC + 11 * B + 600, "nfm", 2500.0, 400.0, 88.5, cm.MOD_NFM),
             (512 * bw - 200.0, AGC + 8 * B + 900, AGC + 13 * B + 200, "nfm", 2500.0, 1100.0, None, cm.MOD_NFM)]
    raw = noise_raw(cfg, ns, [(f, 0.05, f2s(a), f2s(b), k, x, [fm], c) for f, a, b, k, x, fm, c, _ in extra], 0.01, seed=2)
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=nb + 2)
    e.history_configure(0, nb + 1)
    e.push(0, raw)
    while e.run(-1) > 0:
        while e.fetch(0) is not None:
            pass
    hist = e.history_range(0)
    txs = lib.history_transmissions(e, cfg, 0, margin_db=13.0, half_width=16, stride=lib.default_stride(cfg, 0), hang=1, min_span=2)
    hits = []
    for f, a, b, *_ in extra:
        hit = [t for t in txs if abs(t["freq_hz"] - (CF + f)) <= 3 * bw and not t["monitored"]]
        assert len(hit) == 1, (f, [(t["freq_hz"] - CF) / bw for t in txs])
        hits.append(hit[0])
    profs = lib.history_profiles(e, cfg, 0, hits)
    jobs = []
    for (f, a, b, kind, x, fm, ctcss, want), s, t in zip(extra, profs, hits):
        assert s["modulation"] == want and s["ctcss_hz"] == ctcss, (kind, s)
        assert abs(s["freq_hz"] - (CF + f)) <= 20.0, (kind, s["freq_hz"] - CF - f)
        jobs.append(lib.transmission_replay(dict(t, freq_hz=s["freq_hz"]), cfg, 0, hist, **s["channel_kw"]))
    # the same NFM job with a wrong tone stays closed
    jobs.append(lib.transmission_replay(dict(hits[1], freq_hz=profs[1]["freq_hz"]), cfg, 0, hist, modulation=cm.MOD_NFM, ctcss_hz=127.3))
    res = e.history_replay(jobs)
    for (f, a, b, kind, x, fm, ctcss, want), job, r in zip(extra, jobs, res):
        f0 = AGC + job["first_batch"] * B
        lo, hi = f0 + B * np.arange(job["n_batches"]), f0 + B * (np.arange(job["n_batches"]) + 1)
        on = r["axc"][:, 0] == ord("*")
        inside = (lo >= a) & (hi <= b)
        assert inside.any() and on[inside].any(), (kind, on, inside)
        audio = r["waveout"][inside & on, 0, :].reshape(-1).astype(np.float64)
        spec = np.abs(np.fft.rfft((audio - audio.mean()) * np.hanning(audio.size)))
        lo_bin = int(300 * audio.size / W)  # above the CTCSS band, which NFM's audio filter keeps out anyway
        peak = (lo_bin + np.argmax(spec[lo_bin:])) * W / audio.size
        assert abs(peak - fm) <= 10.0, (kind, peak, fm)
    assert not (res[3]["axc"][:, 0] == ord("*")).any()
    e.close()
