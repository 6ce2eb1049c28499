"""The CTCSS tone meter on the GPU (-m gpu): every reading against float64 sums of the fetched audio with the exact integer
phase, bitwise reproducibility across run grouping and push sizes, identification of every standard tone in injected
audio and in a pushed NFM stream, and the lossy queue and its errors."""
import numpy as np
import pytest

from airband_b200 import config as cm
from airband_b200 import lib
from airband_b200 import workloads as wl
from cases import CASES

pytestmark = pytest.mark.gpu
TONES_64 = lib.STANDARD_TONES + tuple(float(f) for f in np.linspace(260.0, 3000.0, 13))
TONE_LISTS = {1: (100.0,), 51: None, 64: TONES_64}


def definition(y, tones, wave_rate, a):
    """S[C, K] (complex128), E[C], active[C] of one batch y[C, B] with audio batch number a, in float64."""
    B = y.shape[1]
    d = np.array([int(np.floor(float(np.float32(f)) / wave_rate * 2.0 ** 32 + 0.5)) % (1 << 32) for f in tones], np.uint64)
    idx = np.uint64(a * B) + np.arange(B, dtype=np.uint64)
    turns = ((d[None, :] * idx[:, None]) % np.uint64(1 << 32)).astype(np.float64) / 2.0 ** 32
    yd = y.astype(np.float64)
    return yd @ np.exp(-2j * np.pi * turns), (yd ** 2).sum(1), np.count_nonzero(y, 1)


def stream(cfg, raws, e, push_items=None, max_batches=-1):
    """Push every device's stream (in pieces of push_items array items, default: all at once) and run to the end; returns
    per device the fetched audio [(waveout, axc)] and tone meter readings, in order."""
    audio = [[] for _ in raws]
    tm = [[] for _ in raws]
    pos = [0] * len(raws)
    while True:
        pushed = False
        for d, r in enumerate(raws):
            if pos[d] < r.size:
                n = push_items or r.size
                e.push(d, r[pos[d]:pos[d] + n])
                pos[d] += n
                pushed = True
        ran = e.run(max_batches)
        for d in range(len(raws)):
            while (g := e.fetch(d, want_iq=False)) is not None:
                audio[d].append((g[0].copy(), g[2].copy()))
            while (x := e.fetch_tone_meter(d)) is not None:
                tm[d].append(x)
        if ran == 0 and not pushed:
            return audio, tm


# ---------------------------------------------------------------------------------------------------------- definition
@pytest.mark.parametrize("K", sorted(TONE_LISTS))
@pytest.mark.parametrize("case", ["am_u8", "nfm_s16", "s8_two_devices"])
def test_readings_match_the_definition(case, K):
    cfg, raws = CASES[case]()
    e = lib.Engine(cfg, max_batches_per_run=4, input_capacity_batches=10)
    e.tone_meter_set_tones(TONE_LISTS[K])
    tones = TONE_LISTS[K] or lib.STANDARD_TONES
    for d in range(len(cfg.devices)):
        e.tone_meter_configure(d, True)
    audio, tm = stream(cfg, raws, e)
    B, wr = e.B, cfg.wave_rate
    assert B == wr // 8
    worst = 0.0
    for d in range(len(cfg.devices)):
        assert len(tm[d]) == len(audio[d]) > 0
        assert [r[3] for r in tm[d]] == list(range(len(audio[d])))
        for a, ((y, _), (S, E, act, seq)) in enumerate(zip(audio[d], tm[d])):
            assert S.shape == (len(cfg.devices[d].channels), K)
            S64, E64, act64 = definition(y, tones, wr, a)
            assert np.array_equal(act, act64)
            l1 = np.abs(y.astype(np.float64)).sum(1)[:, None]
            bound = (B + 8) * 2.0 ** -23 * l1
            err = np.maximum(np.abs(S.real - S64.real), np.abs(S.imag - S64.imag))
            assert np.all(err <= bound), (d, a, float((err / np.maximum(bound, 1e-300)).max()))
            assert np.all(np.abs(E - E64) <= (B + 1) * 2.0 ** -24 * E64)
            if l1.max() > 0:
                worst = max(worst, float((err / np.maximum(bound, 1e-300)).max()))
    assert any(np.any(y != 0) for d in range(len(cfg.devices)) for y, _ in audio[d])  # some audio was metered
    print(f"{case} K={K}: worst error / bound {worst:.3g}")
    e.close()


# -------------------------------------------------------------------------------------------------- reproducibility
def test_bitwise_reproducible_across_run_grouping_and_pushes():
    cfg, raws = CASES["am_u8"](n_batches=6)
    third = 2 * (cfg.wave_batch * cfg.hop(0) // 3)
    ref = None
    for nbmax, push in [(1, None), (2, None), (4, None), (4, third), (2, third)]:
        e = lib.Engine(cfg, max_batches_per_run=nbmax, input_capacity_batches=8)
        e.tone_meter_configure(0, True)
        audio, tm = stream(cfg, raws, e, push_items=push)
        e.close()
        got = ([y.view(np.uint32) for y, _ in audio[0]],
               [(S.view(np.uint64), E.view(np.uint32), act, seq) for S, E, act, seq in tm[0]])
        assert len(got[0]) == len(got[1]) == 6
        if ref is None:
            ref = got
            continue
        assert all(np.array_equal(x, y) for x, y in zip(got[0], ref[0])), (nbmax, push)  # the audio is the same bits
        for r, s in zip(got[1], ref[1]):
            assert all(np.array_equal(x, y) for x, y in zip(r, s)), (nbmax, push)


# ------------------------------------------------------------------------------------------- identification, injected
RAW_NO_SIGNAL, RAW_SIGNAL = 0.05, 0.75  # test_squelch.cpp:33-34, as test_gpu_upstream_fsm.py


def tone_audio(freq, n, ampl=0.2, noise=0.0, seed=0):
    """test_gpu_upstream_fsm.tone_audio: a sine at float32(freq) / 8000 from sample 1, plus noise * normal(0, 0.1)."""
    k = np.arange(1, n + 1, dtype=np.float64)
    x = np.float32(ampl) * np.sin(2 * np.pi * k * float(np.float32(freq)) / 8000.0) if freq else np.zeros(n)
    if noise:
        x = x + noise * np.random.default_rng(seed).normal(0.0, 0.1, n)
    return x


def injected_readings(audios, tones=None):
    """One AM channel without CTCSS per audio series (8 batches at 8000/s), injected as the |X| series that demodulates to
    it after the noise floor settled; returns per channel the readings of the last 4 batches."""
    C = len(audios)
    cfg = cm.Config(fft_size=512, wave_rate=8000, devices=[cm.Device(sample_rate=2560000, sfmt=cm.SFMT_U8, centerfreq=0, channels=[
        cm.make_channel(100000, 0, 2560000, 512, 8000) for _ in range(C)])])
    e = lib.Engine(cfg, max_batches_per_run=4)
    B = e.B
    if tones is not None:
        e.tone_meter_set_tones(tones)
    for _ in range(10):  # send_samples_for_noise_floor (test_squelch.cpp:39-45): the meter is still off
        assert e.inject_wavein(0, np.full((C, 4 * B), RAW_NO_SIGNAL, np.float32)) == 4
        while e.fetch(0, want_iq=False) is not None:
            pass
    e.tone_meter_configure(0, True)
    w = np.stack([(RAW_SIGNAL * (1.0 + 1.5 * a)).astype(np.float32) for a in audios])
    reads, axc = [], []
    for b0 in range(0, 8 * B, 4 * B):
        assert e.inject_wavein(0, w[:, b0:b0 + 4 * B]) == 4
        while (g := e.fetch(0, want_iq=False)) is not None:
            axc.append(g[2].copy())
        while (x := e.fetch_tone_meter(0)) is not None:
            reads.append(x)
    e.close()
    assert len(reads) == 8 and [r[3] for r in reads] == list(range(40, 48))  # injected batches count
    assert all(np.all(a == ord('*')) for a in axc[4:])
    return reads[4:]


def test_identifies_every_standard_tone_injected():
    T = lib.STANDARD_TONES
    n = 8 * 1000
    audios = [tone_audio(f, n) for f in T] + [tone_audio(f, n, noise=1.0, seed=7 + k) for k, f in enumerate(T)]
    audios.append(tone_audio(0, n, noise=1.0, seed=99))  # no tone
    got = lib.ctcss_identify(injected_readings(audios), min_share=0.005)
    for k, f in enumerate(T):
        assert got[k] is not None and got[k][0] == f and got[k][1] > 0.9, (f, got[k])
        assert got[len(T) + k] is not None and got[len(T) + k][0] == f and got[len(T) + k][1] > 0.5, (f, got[len(T) + k])
    assert got[-1] is None, got[-1]


def test_identifies_a_tone_outside_the_standard_list():
    f = (lib.STANDARD_TONES[3] + lib.STANDARD_TONES[4]) / 2  # 75.7 Hz, as test_ctcss.cpp's non-standard tone
    tones = lib.STANDARD_TONES + (f,)
    audios = [tone_audio(f, 8000, noise=1.0, seed=3), tone_audio(0, 8000, noise=1.0, seed=4)]
    r = injected_readings(audios, tones=tones)
    assert r[0][0].shape == (2, 52)
    got = lib.ctcss_identify(r, min_share=0.005, tones=tones)
    assert got[0] is not None and got[0][0] == f, got[0]
    assert got[1] is None, got[1]


# --------------------------------------------------------------------------------------- identification, end to end
def test_identifies_subaudible_tones_in_a_pushed_nfm_stream():
    """synth_iq's NFM channels carry a 1 kHz tone at 2.5 kHz deviation plus the sub-audible tone at a tenth of that; the
    channels have no ctcss, so their squelch opens on the carrier alone."""
    sr, n, w, cf = 400000, 256, 16000, 162000000
    subs = (100.0, 67.0, 69.3)
    chans = [cm.make_channel(cf + o, cf, sr, n, w, modulation=cm.MOD_NFM, bandwidth=5000, squelch_dbfs=-30.0)
             for o in (-125000, 50000, 100000)]
    for ch, s in zip(chans, subs):
        ch.synth_ctcss_hz = s
    cfg = cm.Config(fft_size=n, wave_rate=w, devices=[cm.Device(sample_rate=sr, sfmt=cm.SFMT_S16, centerfreq=cf, channels=chans)])
    raw = wl.synth_iq(cfg, 0, wl.samples_for_batches(cfg, 0, 16), key_on_s=1.4, key_off_s=0.3, amplitude=0.2)
    e = lib.Engine(cfg, max_batches_per_run=4, input_capacity_batches=20)
    e.tone_meter_configure(0, True)
    audio, tm = stream(cfg, [raw], e)
    e.close()
    assert len(tm[0]) == len(audio[0]) == 16
    for c, f in enumerate(subs):
        sig = [bool(ax[c] == ord('*')) for _, ax in audio[0]]
        starts = [b for b in range(len(sig) - 3) if all(sig[b:b + 4])]
        assert starts, (c, sig)
        r = [(S[c:c + 1], E[c:c + 1], act[c:c + 1], seq) for S, E, act, seq in tm[0][starts[0]:starts[0] + 4]]
        share = lib.tone_powers(r)[0]
        got = lib.ctcss_identify(r, min_share=0.002)[0]
        print(f"channel {c}: {f} Hz share {share[lib.STANDARD_TONES.index(f)]:.4f}, identified {got}")
        assert got is not None and got[0] == f, (f, got)
        if f in (67.0, 69.3):  # the neighbour 2.3 Hz away (1.15 bins of the 0.5 s window) reads at most half of it
            other = 69.3 if f == 67.0 else 67.0
            assert share[lib.STANDARD_TONES.index(other)] < 0.5 * got[1]


# --------------------------------------------------------------------------------------------------- queue and errors
def test_lossy_queue_tone_list_changes_and_errors():
    cfg, raws = CASES["am_u8"](n_batches=9)
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=12)

    def drain():
        while e.fetch(0, want_iq=False) is not None:
            pass

    # off: nothing launched beyond the pipeline itself, nothing queued
    e.push(0, raws[0])
    l0 = e.launch_count()
    assert e.run(2) == 2
    base = e.launch_count() - l0
    drain()
    assert e.fetch_tone_meter(0) is None and e.tone_meter_time() == 0.0
    e.tone_meter_configure(0, True)
    # lossy: 3 runs of 2 batches, ring of max_batches_per_run + 2 = 4 readings; the oldest two are gone
    for _ in range(3):
        l0 = e.launch_count()
        assert e.run(2) == 2
        assert e.launch_count() - l0 == base + 2
        drain()
    seqs = []
    while (x := e.fetch_tone_meter(0)) is not None:
        seqs.append(x[3])
        assert x[0].shape == (2, 51)
    assert seqs == [4, 5, 6, 7]
    # a new list applies to later runs; queued entries keep their K and stay fetchable after switching off
    assert e.run(1) == 1
    drain()
    e.tone_meter_set_tones([100.0, 200.0])
    e.push(0, wl.synth_iq(cfg, 0, 3 * cfg.wave_batch * cfg.hop(0)))
    assert e.run(1) == 1
    drain()
    e.tone_meter_configure(0, False)
    assert e.run(1) == 1
    drain()
    got = []
    while (x := e.fetch_tone_meter(0)) is not None:
        got.append((x[3], x[0].shape[1]))
    assert got == [(8, 51), (9, 2)]
    e.tone_meter_set_tones(None)
    # errors
    for call, code in [(lambda: e.tone_meter_configure(1, True), -5), (lambda: e.tone_meter_configure(-1, False), -5),
                       (lambda: e.L.abg_tone_meter_configure(e.h, 0, 2), -2),
                       (lambda: e.tone_meter_set_tones(np.full(65, 100.0)), -2),
                       (lambda: e.tone_meter_set_tones([100.0, 0.0]), -2), (lambda: e.tone_meter_set_tones([4000.0]), -2),
                       (lambda: e.tone_meter_set_tones([float("nan")]), -2), (lambda: e.tone_meter_set_tones([-67.0]), -2),
                       (lambda: e.fetch_tone_meter(1), -5)]:
        try:
            rc = call()
        except lib.AbgError as x:
            rc = x.code
        assert rc == code
    e.tone_meter_set_tones([3999.0] + [67.0] * 63)  # 64 tones, the highest just below wave_rate / 2
    e.close()
