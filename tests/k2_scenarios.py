"""Seeded scenario sets for the exact K2-against-oracle tests (tests/test_gpu_k2_exact.py): per channel a piecewise |X[bin]|
series and the matching X[bin] series, fed to the GPU demodulation kernel and to the CPU oracle through the stage tap
abg_debug_inject_wavein / abo_debug_inject_wavein, so that both sides see identical inputs and must agree bit for bit.

Each scenario set is one configuration plus, per device, wavein[C, n] and iq[C, n].  The channels of a device run different
scenarios: squelch histories (noise-floor settling, key-up, fades to CLOSING, bursts that end in LOW_SIGNAL_ABORT,
flapping, long CLOSED stretches, signal outside the low-pass that holds the squelch CLOSED), segment lengths drawn so
that state changes land at every residue mod 16, and arithmetic edges: a carrier whose AM quotient sits in and around
the guard band of the |w| > 0.8 clip, series scaled by 2^k across the ranges of the kernel's division and square-root
sequences (up to I/Q magnitudes whose squares overflow), exact zeros, subnormals and levels equal to the squelch level and
to the cap."""
from __future__ import annotations

import math

import numpy as np

import oracle_py as op
from airband_b200 import config as cm

F = np.float32
NOISE, SIGNAL = 0.05, 0.75
DELTAS = (-3e-5, -1.6e-5, -1.25e-5, -1e-5, 0.0, 1e-5, 1.25e-5, 1.6e-5, 3e-5)  # relative offsets of the AM quotient from 0.8


def _len(rng, lo, hi, residues):
    """A segment length in [lo, hi) with the next residue mod 16 from the channel's cycle."""
    r = residues.pop(0)
    residues.append(r)
    q = int(rng.integers(lo // 16, max(lo // 16 + 1, hi // 16)))
    return 16 * q + r


def history(rng, n, inband=True, outband=False, ctcss=False):
    """Squelch history: (magnitude level per sample, kind per sample) with kind 0 noise, 1 in-band signal, 2 signal outside
    the low-pass (held CLOSED), 3 signal with the wrong CTCSS tone."""
    res = list(rng.permutation(16))
    lv = np.empty(0, np.float64)
    kind = np.empty(0, np.int8)

    def add(level, k, m):
        nonlocal lv, kind
        lv = np.concatenate([lv, np.broadcast_to(level, (m,)).astype(np.float64) if np.ndim(level) == 0 else level[:m]])
        kind = np.concatenate([kind, np.full(m, k, np.int8)])

    add(NOISE, 0, _len(rng, 1500, 3000, res))                      # noise floor settles, CLOSED > 1000 samples
    while lv.size < n:
        what = rng.integers(0, 7)
        if what <= 1:                                               # key-up to OPEN, then an abrupt drop (LOW_SIGNAL_ABORT)
            add(SIGNAL, 1, _len(rng, 300, 2500, res))
            add(NOISE, 0, _len(rng, 300, 1400, res))
        elif what == 2:                                             # slow fade: pre-filter level lost, raw samples still at the level
            add(SIGNAL, 1, _len(rng, 400, 1500, res))
            m = _len(rng, 250, 600, res)
            fade = np.where(np.arange(m) % 2 == 0, 0.17, 0.01)
            add(fade, 1, m)
            add(NOISE, 0, _len(rng, 200, 1200, res))
        elif what == 3:                                             # flapping: short bursts, closed < 1000 samples in between
            for _ in range(int(rng.integers(3, 6))):
                add(SIGNAL, 1, _len(rng, 230, 420, res))
                add(NOISE, 0, _len(rng, 100, 400, res))
            add(NOISE, 0, _len(rng, 1100, 1600, res))
        elif what == 4:                                             # burst shorter than the opening delay
            add(SIGNAL, 1, _len(rng, 60, 190, res))
            add(NOISE, 0, _len(rng, 200, 800, res))
        elif what == 5 and outband:                                 # energy outside the low-pass: pre-filter opens, post-filter holds it
            add(SIGNAL, 2, _len(rng, 400, 1500, res))
            add(NOISE, 0, _len(rng, 300, 900, res))
        elif what == 6 and ctcss:                                   # wrong sub-tone
            add(SIGNAL, 3, _len(rng, 800, 2500, res))
            add(NOISE, 0, _len(rng, 300, 900, res))
        else:                                                       # dead spot inside a transmission
            add(SIGNAL, 1, _len(rng, 400, 900, res))
            add(NOISE, 0, _len(rng, 20, 60, res))
            add(SIGNAL, 1, _len(rng, 400, 900, res))
            add(NOISE, 0, _len(rng, 300, 700, res))
    return lv[:n], kind[:n]


def iq_for(rng, lv, kind, wave_rate, dm_dphi, am=True, tone=1000.0, ctcss_hz=0.0, wrong_hz=0.0):
    """X[bin] whose magnitude follows `lv` (AM: with 50 % modulation on signal samples) and whose phase, after the channel's
    derotation (dm_dphi per sample), is baseband FM (NFM) or slowly drifting (AM); kind 2 sits 0.3 cycles / sample off."""
    n = lv.size
    t = np.arange(n, dtype=np.float64)
    rot = 2 * math.pi * (dm_dphi / float(1 << 24)) * t
    if am:
        mag = lv * np.where(kind > 0, 1.0 + 0.5 * np.cos(2 * math.pi * tone * t / wave_rate), 1.0)
        ph = 0.001 * t
    else:
        mag = lv.copy()
        sub = np.where(kind == 3, wrong_hz, ctcss_hz)
        f = 2500.0 * np.cos(2 * math.pi * tone * t / wave_rate) + (250.0 * np.cos(2 * math.pi * sub * t / wave_rate) if ctcss_hz else 0.0)
        ph = 2 * math.pi * np.cumsum(f) / wave_rate
    ph = ph + np.where(kind == 2, 2 * math.pi * 0.3 * t, 0.0)
    noise = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 0.01
    x = mag * np.exp(1j * (ph + rot)) + noise * np.where(kind == 0, 1.0, 0.0)
    return x


def magnitude(iq):
    """|X| rounded once to float32 (what a K1 would store); finite wherever the complex value is."""
    return np.abs(iq.astype(np.complex128)).astype(F)


def guard_band_series(n, delta, scale=1.0, p=5):
    """A carrier of period p with one peak per period whose AM quotient (wavein[j-100] - agc) / (1.5 agc) settles at
    0.8 * (1 + delta) on every peak (rtl_airband.cpp:553-562): the periodic steady state of the AGC is solved for the peak
    height.  With delta > 0 the clip fires, the AGC jumps and creeps back, so the peaks cross the guard band in tiny steps."""
    g = 0.995
    ones = sum(g ** k for k in range(p - 1))                       # contribution of the p-1 samples of height 1 after the peak
    # a before the peak (steady state): a (1 - g^p) = 0.005 (P g^(p-1) + ones)
    den = 1.0 - g ** p
    w = 0.8 * (1.0 + delta)
    alpha = g * 0.005 * ones / den                                  # a2 at the peak = alpha + beta P
    beta = g * 0.005 * g ** (p - 1) / den + 0.005
    P = alpha * (1 + 1.5 * w) / (1.0 - beta * (1 + 1.5 * w))
    x = np.ones(n)
    x[::p] = P
    return (x * scale).astype(F)


# --------------------------------------------------------------------------------------------------------------------------
def _dev(sr, cf, channels):
    return cm.Device(sample_rate=sr, sfmt=cm.SFMT_S16, centerfreq=cf, channels=channels)


def am_set(n_batches=30, seed=11):
    """wave_rate 8000 (WAVE_BATCH 1000), one device: the AM channel kinds, the guard-band carriers, scaled series."""
    sr, fft, w, cf = 2560000, 512, 8000, 120000000
    B = w // 8
    n = n_batches * B
    rng = np.random.default_rng(seed)
    mk = lambda off, **kw: cm.make_channel(cf + off, cf, sr, fft, w, **kw)  # noqa: E731
    chans, waves, iqs = [], [], []

    def add(ch, wave, iq=None):
        chans.append(ch)
        waves.append(np.asarray(wave, F))
        iqs.append(np.zeros(n, np.complex64) if iq is None else np.asarray(iq, np.complex64))

    # squelch histories through the plain-AM fast loop: manual, SNR and default squelch
    for kw in (dict(squelch_dbfs=-41.5), dict(squelch_snr_db=9.0), dict()):
        ch = mk(25000 * (len(chans) + 1), **kw)
        lv, kind = history(rng, n)
        x = iq_for(rng, lv, kind, w, 0)
        add(ch, magnitude(x))
    # AM with `bandwidth` (derotation + low-pass + post-filter estimator), with signal outside the filter too; rawfile
    for kw in (dict(bandwidth=6000, squelch_snr_db=9.0), dict(bandwidth=6000, rawfile=True, squelch_dbfs=-41.5, ampfactor=2.0),
               dict(rawfile=True, squelch_dbfs=-41.5), dict(bandwidth=6000, notch_hz=1000.0, squelch_dbfs=-41.5)):
        ch = mk(25000 * (len(chans) + 1), **kw)
        lv, kind = history(rng, n, outband=True)
        x = iq_for(rng, lv, kind, w, ch.dm_dphi)
        add(ch, magnitude(x), x)
    # guard band of the clip: manual level at half the carrier, so every sample is above it and the squelch stays OPEN
    for d in DELTAS:
        ch = mk(25000 * (len(chans) + 1), squelch_dbfs=-41.5)
        ch.squelch_level = 0.5
        x = np.concatenate([np.full(300, NOISE, F), np.full(500, 1.0, F), guard_band_series(n - 800, d)])
        add(ch, x)
    # the same scaled by 2^k: quotient operands across 2^-62 and 2^62, subnormal magnitudes
    for k in (-140, -128, -63, -62, -61, 61, 62, 63):
        ch = mk(25000 * (len(chans) + 1), squelch_dbfs=-41.5)
        s = 2.0 ** k
        ch.squelch_level = float(F(0.5 * s))
        x = np.concatenate([np.zeros(300, F), np.full(500, s, F), guard_band_series(n - 800, DELTAS[len(chans) % len(DELTAS)], s)])
        add(ch, x)
    # probes where only the exact quotient decides the clip (AGC state after the warm-up read off the oracle)
    for seed in (5, 6):
        ch = mk(25000 * (len(chans) + 1), squelch_dbfs=-41.5)
        ch.squelch_level = 0.5
        warm = np.concatenate([np.full(300, NOISE, F), np.full(2700, 0.7, F)])
        o = op.Oracle(cm.Config(fft_size=fft, wave_rate=w, devices=[_dev(sr, cf, [ch])]))
        o.inject_wavein(0, warm[None, :])
        a0 = o.stats(0, 0).agcavgfast
        o.close()
        x, _ = clip_probe_series(a0, 0.5, n - warm.size, seed=seed)
        add(ch, np.concatenate([warm, x]))
    # exact zeros, samples exactly at the level and at the cap (the >= ties), and a wandering carrier
    ch = mk(25000 * (len(chans) + 1), squelch_dbfs=-41.5)
    ch.squelch_level = 0.25
    pieces, res = [], list(rng.permutation(16))
    while sum(p.size for p in pieces) < n:
        m = _len(rng, 100, 900, res)
        v = [0.0, 0.25, 0.375, 0.75, NOISE, 0.5][int(rng.integers(0, 6))]
        pieces.append(np.full(m, v, F))
        if rng.random() < 0.3:
            pieces.append(np.where(np.arange(m) % 3 == 0, F(0.25), F(0.375)).astype(F))
    add(ch, np.concatenate(pieces)[:n])
    # AM with bandwidth, I/Q scaled across the square-root range [2^-100, 2^125] and up to squares that overflow
    for k in (-52, -50, -49, 61, 62, 63, 64):
        ch = mk(25000 * (len(chans) + 1), bandwidth=6000, rawfile=True)
        s = 2.0 ** k
        ch.squelch_level = float(F(0.1 * s))
        lv, kind = history(rng, n)
        x = iq_for(rng, lv, kind, w, ch.dm_dphi) * s
        add(ch, magnitude(x), x)
    cfg = cm.Config(fft_size=fft, wave_rate=w, devices=[_dev(sr, cf, chans)])
    return dict(name="am", cfg=cfg, wave=[np.stack(waves)], iq=[np.stack(iqs)], scan=None)


def nfm_set(fm_demod, n_batches=16, seed=23):
    """wave_rate 16000 (WAVE_BATCH 2000): NFM with / without de-emphasis, notch, ampfactor, CTCSS, with and without the
    low-pass, scaled I/Q; a second device holds one scan channel that switches frequency-list entries between injections."""
    sr, fft, w, cf = 2560000, 512, 16000, 162000000
    B = w // 8
    n = n_batches * B
    rng = np.random.default_rng(seed + fm_demod)
    mk = lambda off, **kw: cm.make_channel(cf + off, cf, sr, fft, w, modulation=cm.MOD_NFM, **kw)  # noqa: E731
    chans, waves, iqs = [], [], []

    def add(ch, lv, kind, ctcss=0.0, wrong=0.0, scale=1.0):
        x = iq_for(rng, lv, kind, w, ch.dm_dphi, am=False, ctcss_hz=ctcss, wrong_hz=wrong) * scale
        chans.append(ch)
        waves.append(magnitude(x))
        iqs.append(x.astype(np.complex64))

    kinds = [dict(bandwidth=5000, squelch_dbfs=-41.5), dict(bandwidth=5000, squelch_dbfs=-41.5, tau_us=0),
             dict(bandwidth=5000, squelch_dbfs=-41.5, notch_hz=100.0), dict(bandwidth=5000, squelch_snr_db=9.0, ampfactor=2.5),
             dict(squelch_dbfs=-41.5), dict(squelch_snr_db=6.0, tau_us=0)]
    for kw in kinds:
        lv, kind = history(rng, n, outband=kw.get("bandwidth", 0) > 0)
        add(mk(25000 * (len(chans) + 1), **kw), lv, kind)
    for tone, wrong in ((100.0, 67.0), (123.0, 0.0)):
        lv, kind = history(rng, n, ctcss=True)
        add(mk(25000 * (len(chans) + 1), bandwidth=5000, squelch_dbfs=-41.5, ctcss_hz=tone, notch_hz=tone), lv, kind, tone, wrong)
    for k in (-52, -50, -49, 61, 62, 63, 64):
        ch = mk(25000 * (len(chans) + 1), bandwidth=5000)
        ch.squelch_level = float(F(0.1 * 2.0 ** k))
        lv, kind = history(rng, n)
        add(ch, lv, kind, scale=2.0 ** k)
    # scan: one channel, three entries (AM with bandwidth, AM with notch and SNR squelch, NFM with CTCSS)
    f0 = cf + 250000
    base = mk(250000, bandwidth=6000, squelch_dbfs=-41.5)
    entries = [cm.make_channel(f0, cf, sr, fft, w, bandwidth=6000, squelch_dbfs=-41.5),
               cm.make_channel(f0, cf, sr, fft, w, bandwidth=6000, ampfactor=2.5, notch_hz=1000.0, squelch_snr_db=6.0),
               cm.make_channel(f0, cf, sr, fft, w, modulation=cm.MOD_NFM, bandwidth=6000, squelch_dbfs=-41.5, ctcss_hz=100.0, ampfactor=1.5)]
    lv, kind = history(rng, n)
    xs = iq_for(rng, lv, kind, w, base.dm_dphi, am=False, ctcss_hz=100.0)
    cfg = cm.Config(fft_size=fft, wave_rate=w, fm_demod=fm_demod, devices=[_dev(sr, cf, chans), _dev(sr, cf, [base])])
    return dict(name=f"nfm{fm_demod}", cfg=cfg, wave=[np.stack(waves), magnitude(xs)[None, :]],
                iq=[np.stack(iqs), xs.astype(np.complex64)[None, :]], scan=(1, 0, entries))


def scenario_sets():
    return [am_set(), nfm_set(cm.FM_FAST_ATAN2), nfm_set(cm.FM_QUADRI_DEMOD)]


def calls(n_batches):
    """Batches per injection: 1, 2, 3, 4, 1, 2, ... (runs of up to max_batches_per_run = 4, batch and run boundaries move)."""
    out, k = [], 0
    while sum(out) < n_batches:
        out.append(min(1 + k % 4, n_batches - sum(out)))
        k += 1
    return out


def _disagreeing_pairs(lo, hi, want_big):
    """(agc, numerator) pairs with agc in [lo, hi] (float32) where comparing the numerator with fl(1.2 agc) and rounding the
    quotient n / fl(1.5 agc) give different answers about |w| > 0.8f."""
    a2 = np.arange(np.float32(lo).view(np.int32), np.float32(hi).view(np.int32), dtype=np.int32).view(np.float32)
    d = (a2 * F(1.5)).astype(F)
    prod = (a2 * F(1.2)).astype(F)
    out = []
    for s in (-2, -1, 1, 2):
        n = (prod.view(np.int32) + np.int32(s)).view(np.float32)
        big = np.abs((n / d).astype(F)) > F(0.8)
        hit = (big & (n < prod)) if want_big else (~big & (n > prod))
        out += list(zip(a2[hit], n[hit]))
    return out


def clip_probe_series(a0, lvl, n, base_level=0.7, spacing=600, seed=5):
    """A steady OPEN plain-AM channel (manual level `lvl`, every sample above it) that starts with AGC value a0 and carries
    probes: at a probe j the numerator wavein[j-100] - agc sits within two ulps of fl(1.2 agc), on whichever side makes the
    product and the rounded quotient fl(n / fl(1.5 agc)) disagree about |w| > 0.8f.  Those are the samples a guard band of
    the wrong width decides wrongly.  Built by walking the AGC recurrence of rtl_airband.cpp:553-562 in float32: the peak
    100 samples ahead carries numerator + agc for an (agc, numerator) pair the probe can reach, and the probe's own sample
    (which moves the AGC by 0.5 % of its offset) is chosen so that the AGC lands on exactly that value."""
    rng = np.random.default_rng(seed)
    x = np.full(n, base_level, F)
    lv = F(lvl)

    def step(a, xj, xlag):
        a2 = F(F(a * F(0.995)) + F(xj * F(0.005))) if xj > lv else a
        w = F(F(xlag - a2) / F(a2 * F(1.5)))
        return F(a2 * F(1.15)) if abs(w) > F(0.8) else a2

    def walk(a, j0, j1):
        for j in range(j0, j1):
            a = step(a, x[j], x[j - 100] if j >= 100 else F(base_level))
        return a

    probes, a, t = [], F(a0), 0
    for j in range(200, n - 1, spacing + int(rng.integers(0, 16))):
        a = walk(a, t, j - 100)
        t = j - 100
        x[t] = F(2.2 * float(walk(a, t, j)))                        # a first aim, then the AGC the probe starts from
        base = walk(a, t, j)
        c = float(F(base * F(0.995)))
        lo, hi = c + 0.005 * (lvl + 0.1 * base_level), c + 0.005 * 1.4 * base_level     # reachable with x[j] above the level
        pairs = _disagreeing_pairs(lo, hi, len(probes) % 2 == 0)
        if not pairs:
            continue
        a2t, nt = pairs[len(pairs) // 2]
        x[t] = F(float(nt) + float(a2t))
        a = walk(a, t, j)
        t = j
        ca = F(a * F(0.995))
        xj0 = (float(a2t) - float(ca)) / 0.005
        for k in range(-64, 65):
            xj = F(xj0 * (1.0 + k * 2e-8))
            if xj > lv and F(ca + F(xj * F(0.005))) == a2t and F(x[j - 100] - a2t) == nt:
                x[j] = xj
                probes.append(j)
                break
    return x, probes
