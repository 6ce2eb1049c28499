"""History replay (abg_history_replay) on the GPU (-m gpu).

Every job's outputs must be bitwise those of a fresh engine fed the history's bytes, for every format (hop 313 gathers
across a misalignment), every K1 path, AM and NFM channels with CTCSS, notch, bandwidth and I/Q outputs, windows across
the ring's wrap and longer than max_batches_per_run.  They must not depend on how jobs share a call, on the parent's
max_batches_per_run or on earlier calls, and must pass the oracle's strict gate.  Replays between runs must leave every
live output, monitor reading, history range and per-run launch count as a twin engine that never replays has them.  End
to end: three unconfigured transmitters are detected, grouped and replayed in one call, and each channel hears its own."""
import ctypes as C

import numpy as np
import pytest

import oracle_py as op
import parity
from airband_b200 import config as cm
from airband_b200 import lib
from test_gpu_activity import _all_monitors, fetch_monitors, quantize

pytestmark = pytest.mark.gpu
AGC = cm.AGC_EXTRA
W, CF = 8000, 120_000_000


def tx_raw(cfg, n_samples, txs, noise, seed):
    """Complex noise plus transmitters txs = [(offset_hz, amplitude, first sample, end sample, kind, f_mod)]: kind "am" is
    60 % AM by a tone at f_mod, "nfm" FM with 2.5 kHz peak deviation by it."""
    d = cfg.devices[0]
    rng = np.random.default_rng(seed)
    x = rng.normal(0, noise, n_samples) + 1j * rng.normal(0, noise, n_samples)
    for f, a, s0, s1, kind, fm in txs:
        t = np.arange(s0, s1) / d.sample_rate
        if kind == "am":
            x[s0:s1] += a * (1 + 0.6 * np.cos(2 * np.pi * fm * t)) * np.exp(2j * np.pi * f * t)
        else:
            x[s0:s1] += a * np.exp(1j * (2 * np.pi * f * t + 2500.0 / fm * np.sin(2 * np.pi * fm * t)))
    return quantize(x, d.sfmt, d.fullscale)


def parent_cfg(sfmt, sr, n=2048, fs=0.0, channels=None, w=W):
    ch = channels or [cm.make_channel(CF + 300_000, CF, sr, n, w)]
    return cm.Config(fft_size=n, wave_rate=w, devices=[cm.Device(sample_rate=sr, sfmt=sfmt, fullscale=fs, centerfreq=CF, channels=ch)])


def drive(cfg, raw, nbmax, hist, fft_mode=0, piece_batches=1.0, between=None, setup=None, out=None):
    """A parent engine with the history of `hist` batches on device 0, fed raw in pieces with runs in between; every run's
    outputs are drained (into out, as bytes, if given).  between(e) is called after every run that demodulated something."""
    e = lib.Engine(cfg, max_batches_per_run=nbmax, fft_mode=fft_mode)
    e.history_configure(0, hist)
    if setup:
        setup(e)
    step = int(piece_batches * cfg.wave_batch * cfg.hop(0)) * 2
    pos = 0
    while True:
        if pos < raw.size:
            e.push(0, raw[pos:pos + step])
            pos += step
        n = e.run(-1)
        while (g := e.fetch(0)) is not None:
            if out is not None:
                out.append(("batch", g[0].tobytes(), g[1].tobytes(), g[2].tobytes()))
        if n and between:
            between(e)
        if n == 0 and pos >= raw.size:
            return e


def fresh(parent, cfg, raw, job, fft_mode=0):
    """The definition's fresh engine on the history's bytes: (waveout[n, C, B], iq[n, C, B], axc[n, C], stats bytes)."""
    d = cfg.devices[0]
    B, hop, N, n = cfg.wave_batch, cfg.hop(0), cfg.fft_size, job["n_batches"]
    S = job["first_batch"] * B * hop
    need = (AGC + n * B) * hop + N - hop
    data = np.concatenate([parent.history_raw(0, S, need), raw[2 * (S + need):2 * (S + need + hop)]])
    assert data.size == 2 * (need + hop)
    c = cm.Config(fft_size=N, wave_rate=cfg.wave_rate, fm_demod=cfg.fm_demod,
                  devices=[cm.Device(sample_rate=d.sample_rate, sfmt=d.sfmt, fullscale=d.fullscale, centerfreq=d.centerfreq,
                                     channels=job["channels"])])
    e = lib.Engine(c, fft_mode=fft_mode, input_capacity_batches=n + 2)
    e.push(0, data)
    got = []
    while e.run(-1) > 0:
        while (r := e.fetch(0)) is not None:
            got.append(r)
    assert len(got) == n
    st = [bytes(e.stats(0, k)) for k in range(len(job["channels"]))]
    e.close()
    return np.stack([g[0] for g in got]), np.stack([g[1] for g in got]), np.stack([g[2] for g in got]), st


def same(r, f):
    assert np.array_equal(r["waveout"].view(np.uint32), f[0].view(np.uint32))
    assert np.array_equal(r["iq"].view(np.uint64), f[1].view(np.uint64))
    assert np.array_equal(r["axc"], f[2])
    assert [bytes(s) for s in r["stats"]] == f[3]


def same_results(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        same(x, (y["waveout"], y["iq"], y["axc"], [bytes(s) for s in y["stats"]]))


# ---- the scenario: a parent with a 5-batch history after 12 batches, three transmitters -----------------------------------
NB, HIST = 12, 5


def scenario(sfmt, sr, fs=0.0, n=2048, afc=False, w=W):
    bw = sr // n
    f1, f2, f3 = 120 * bw, -333 * bw, 41 * bw + bw // 3
    cfg = parent_cfg(sfmt, sr, n, fs, w=w)
    B, hop = cfg.wave_batch, cfg.hop(0)
    ns = (AGC + NB * B) * hop + n + hop
    s = lambda fr: int(fr * hop)  # noqa: E731
    txs = [(f1, 0.2, s(AGC + 7 * B + 300), s(AGC + 11 * B + 500), "am", 700.0),
           (f2, 0.2, s(AGC + 8 * B + 200), ns, "nfm", 900.0),
           (f3, 0.15, 0, s(AGC + 9 * B + 900), "am", 400.0)]
    raw = tx_raw(cfg, ns, txs, 0.01, seed=sfmt)
    ch = lambda f, **kw: cm.make_channel(CF + int(f), CF, sr, n, w, **kw)  # noqa: E731
    jobs = [dict(dev=0, first_batch=8, n_batches=3, channels=[ch(f1, notch_hz=1500.0), ch(f1, ctcss_hz=100.0), ch(f3)]),
            dict(dev=0, first_batch=9, n_batches=2, channels=[ch(f2, modulation=cm.MOD_NFM, bandwidth=12000),
                                                           ch(f2, modulation=cm.MOD_NFM, rawfile=True)]),
            dict(dev=0, first_batch=8, n_batches=1, channels=[ch(f3, squelch_snr_db=6.0, rawfile=True)])]
    if afc:
        jobs.append(dict(dev=0, first_batch=8, n_batches=3, channels=[ch(f1 + bw, afc=2), ch(f3)]))
    return cfg, raw, jobs


# (name, format, sample rate, full scale, fft_mode, AFC job, wave_rate).  At wave_rate 8000 a batch is 1000 frames, so every
# window starts on a 16-byte boundary of the ring; at 8008 (1001 frames) with hop 313 the odd ones do not, and the gather
# shifts every vector.
CASES = [("u8_hop313", cm.SFMT_U8, 2500000, 0.0, 0, False, W), ("s8", cm.SFMT_S8, 2560000, 0.0, 0, False, W),
         ("s16", cm.SFMT_S16, 2560000, 32766.5, 0, False, W), ("f32", cm.SFMT_F32, 2048000, 1.0, 0, False, W),
         ("u8_misaligned", cm.SFMT_U8, 2506504, 0.0, 0, False, 8008), ("s16_misaligned", cm.SFMT_S16, 2506504, 32766.5, 0, False, 8008),
         ("u8_pruned", cm.SFMT_U8, 2560000, 0.0, 2, False, W), ("u8_tensor", cm.SFMT_U8, 2560000, 0.0, 3, False, W),
         ("s8_afc", cm.SFMT_S8, 2560000, 0.0, 0, True, W)]


# ---- 1. fresh-engine equivalence -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,sfmt,sr,fs,fft_mode,afc,w", CASES, ids=[c[0] for c in CASES])
def test_replay_is_bitwise_a_fresh_engine_on_the_history(name, sfmt, sr, fs, fft_mode, afc, w):
    cfg, raw, jobs = scenario(sfmt, sr, fs, afc=afc, w=w)
    B, hop = cfg.wave_batch, cfg.hop(0)
    e = drive(cfg, raw, nbmax=2, hist=HIST, fft_mode=fft_mode)
    first, end = e.history_range(0)
    assert (first, end) == ((AGC + (NB - HIST) * B) * hop, (AGC + NB * B) * hop)
    bpc = {cm.SFMT_U8: 2, cm.SFMT_S8: 2, cm.SFMT_S16: 4, cm.SFMT_F32: 8}[sfmt]
    if w == 8008:
        assert (9 * B * hop * bpc) % 16 != 0  # job 1 starts off a 16-byte boundary of the ring
    # job 0 crosses the ring's wrap and is longer than max_batches_per_run
    R = (HIST * B * hop * bpc + 15) // 16 * 16
    assert 8 * B * hop * bpc // R != (AGC + 11 * B) * hop * bpc // R
    res = e.history_replay(jobs)
    for job, r in zip(jobs, res):
        same(r, fresh(e, cfg, raw, job, fft_mode))
    assert any((r["axc"] != ord(" ")).any() for r in res)  # something opened
    g, k = e.replay_time()
    assert g > 0 and k > 0
    e.close()


# ---- 2. oracle parity ---------------------------------------------------------------------------------------------------
def test_replay_passes_the_oracle_strict_gate():
    cfg, raw, jobs = scenario(cm.SFMT_U8, 2500000)
    e = drive(cfg, raw, nbmax=2, hist=HIST)
    res = e.history_replay(jobs[:2])  # AM and NFM
    B, hop, N = cfg.wave_batch, cfg.hop(0), cfg.fft_size
    for job, r in zip(jobs[:2], res):
        S = job["first_batch"] * B * hop
        need = (AGC + job["n_batches"] * B) * hop + N - hop
        data = np.concatenate([e.history_raw(0, S, need), raw[2 * (S + need):2 * (S + need + hop)]])
        d = cfg.devices[0]
        oc = cm.Config(fft_size=N, wave_rate=W, devices=[cm.Device(sample_rate=d.sample_rate, sfmt=d.sfmt, centerfreq=CF,
                                                                   channels=job["channels"])])
        res_o, o = op.run_oracle(oc, [data])
        ow, _, oa = res_o[0]
        o.close()
        Cn = len(job["channels"])
        gw = r["waveout"].transpose(1, 0, 2).reshape(Cn, -1)
        rep = parity.strict((gw, None, r["axc"]), (ow, None, oa))
        assert rep["ok"], rep
    e.close()


# ---- 3. independence --------------------------------------------------------------------------------------------------------
def test_results_do_not_depend_on_sharing_order_parent_batches_or_earlier_calls():
    cfg, raw, jobs = scenario(cm.SFMT_U8, 2500000)
    e = drive(cfg, raw, nbmax=2, hist=HIST)
    together = e.history_replay(jobs)
    again = e.history_replay(jobs)
    same_results(together, again)  # fresh state on every call
    same_results(e.history_replay(jobs[::-1])[::-1], together)
    for k, j in enumerate(jobs):
        same_results(e.history_replay([j]), [together[k]])
    same_results(e.history_replay([jobs[0], jobs[0]]), [together[0], together[0]])
    e.close()
    for nbmax in (1, 4):
        p = drive(cfg, raw, nbmax=nbmax, hist=HIST, piece_batches=0.37 * nbmax)
        same_results(p.history_replay(jobs), together)
        p.close()


# ---- 4. the live path -------------------------------------------------------------------------------------------------------
def test_live_runs_are_unchanged_by_replays_between_them():
    cfg, raw, jobs = scenario(cm.SFMT_S8, 2560000)
    thr = np.full(cfg.fft_size, 40.0, np.float32)
    B = cfg.wave_batch

    def setup(e):
        _all_monitors(e, cfg, 0)
        e.activity_configure(0, lib.default_stride(cfg, 0), 1, 2, thr)

    def trace(replay):
        log = []

        def between(e):
            log.append((e.history_range(0), fetch_monitors(e, 0), e.launch_count() - log_count[0]))
            while (a := e.fetch_activity(0)) is not None:
                log.append(("act", a["batch_seq"], a["n_total"], a["pieces"].tobytes()))
            first, end = e.history_range(0)
            if replay and end - first >= (AGC + 2 * B) * cfg.hop(0):
                # 1, 2 or 3 jobs of two shapes: the replay engine grows between runs
                b0 = -(-first // (B * cfg.hop(0)))
                sel = [jobs[0], jobs[1], jobs[0]][:1 + len(replays) % 3]
                r = e.history_replay([dict(j, first_batch=b0, n_batches=1) for j in sel])
                replays.append(r[0]["axc"].tobytes())
            log_count[0] = e.launch_count()  # a replay's own launches are not a run's

        log_count = [0]
        e = drive(cfg, raw, nbmax=2, hist=4, between=between, setup=setup, out=log)
        e.close()
        return log

    replays = []
    with_replays, without = trace(True), trace(False)
    assert sum(x[0] == "batch" for x in without) == NB
    assert with_replays == without
    assert len(replays) >= 3


# ---- the replay engine: allocated by the first replay, grown only when a call needs more ------------------------------------
def test_nothing_is_allocated_before_the_first_replay_and_the_pool_only_grows():
    torch = pytest.importorskip("torch")
    cfg, raw, jobs = scenario(cm.SFMT_U8, 2560000)
    B, hop = cfg.wave_batch, cfg.hop(0)

    def free():
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info()[0]

    e = drive(cfg, raw, nbmax=2, hist=HIST)
    f0 = free()
    e.history_raw(0, e.history_range(0)[0], 1000)
    e.sync()
    assert abs(free() - f0) < 2 << 20  # a streamed engine with its history on: no replay engine yet
    full = e.history_replay(jobs)
    f1 = free()
    raw_bytes = 2 * (2 + 2) * B * hop * 2  # the two input buffers of one replay device, at least
    assert f0 - f1 >= len(jobs) * raw_bytes, (f0, f1)
    # calls that fit the pool allocate nothing and give what the full call gave
    for sel in ([0], [1, 2], [2, 1, 0], [1]):
        same_results(e.history_replay([jobs[k] for k in sel]), [full[k] for k in sel])
        assert abs(free() - f1) < 2 << 20, sel
    # two jobs of one shape need a second device of it: the pool grows, keeping what it had
    two = e.history_replay([jobs[2], jobs[2]])
    same_results(two, [full[2], full[2]])
    f2 = free()
    assert f1 - f2 >= raw_bytes
    same_results(e.history_replay(jobs + [jobs[2]]), full + [full[2]])
    same_results(e.history_replay(jobs), full)
    assert abs(free() - f2) < 2 << 20
    e.history_configure(0, 0)  # the last history off frees the replay engine
    assert free() - f2 >= len(jobs) * raw_bytes
    e.close()


# ---- 5. errors ------------------------------------------------------------------------------------------------------------------
def test_error_codes():
    cfg, raw, jobs = scenario(cm.SFMT_U8, 2560000)
    B, hop, N = cfg.wave_batch, cfg.hop(0), cfg.fft_size
    e = lib.Engine(cfg, max_batches_per_run=2)

    def code(*a):
        with pytest.raises(lib.AbgError) as ex:
            e.history_replay(*a)
        return ex.value.code, str(ex.value)

    job = dict(dev=0, first_batch=8, n_batches=1, channels=jobs[0]["channels"])
    assert code([job])[0] == -5  # history off
    e.history_configure(0, HIST)
    step = B * hop * 2
    for p in range(0, raw.size, step):
        e.push(0, raw[p:p + step])
        while e.run(-1):
            while e.fetch(0) is not None:
                pass
    first, end = e.history_range(0)
    assert (first, end) == ((AGC + (NB - HIST) * B) * hop, (AGC + NB * B) * hop)
    b_lo = -(-first // (B * hop))
    assert code([dict(job, first_batch=b_lo - 1)])[0] == -5  # before first
    assert code([dict(job, dev=1)])[0] == -5
    # the last frame's tail, fft_size - hop samples into the batch after the last one, must be in the history: a window
    # that ends with batch NB - 1 reads fft_size - hop samples past end
    rc, msg = code([dict(job, first_batch=NB - 1, n_batches=1)])
    assert rc == -5 and f"[{(NB - 1) * B * hop}, {(AGC + NB * B) * hop + N - hop})" in msg, msg
    assert code([dict(job, first_batch=NB - 2, n_batches=2)])[0] == -5
    assert code([dict(job, first_batch=NB, n_batches=1)])[0] == -5  # past end
    ok = e.history_replay([dict(job, first_batch=NB - 2, n_batches=1)])[0]  # the last window that fits
    assert ok["waveout"].shape == (1, 3, B)
    # what abg_create refuses, n_batches 0, null outputs
    bad = cm.Channel(bin=N)
    assert code([dict(job, first_batch=b_lo, channels=[bad])])[0] == -2
    assert code([dict(job, first_batch=b_lo, channels=[cm.Channel(bin=5, modulation=7)])])[0] == -2
    assert code([dict(job, first_batch=b_lo, n_batches=0)])[0] == -2
    assert code([])[0] == -2
    chans = cm.channels_to_c(job["channels"])
    wo = np.zeros((1, 3, B), np.float32)
    ax = np.zeros((1, 3), np.uint8)
    for w, a in ((None, ax), (wo, None)):
        j = lib.CReplayJob(0, 1, b_lo, 3, C.cast(chans, C.POINTER(cm.CChannelCfg)), lib._ptr(w), None, lib._ptr(a), None)
        assert e.L.abg_history_replay(e.h, 1, C.byref(j)) == -2
    # a failed call leaves the engine usable
    same(e.history_replay([dict(job, first_batch=b_lo)])[0], fresh(e, cfg, raw, dict(job, first_batch=b_lo)))
    e.history_configure(0, 0)  # frees the replay engine; the next replay finds no history
    assert code([dict(job, first_batch=b_lo)])[0] == -5
    e.close()


# ---- 6. end to end --------------------------------------------------------------------------------------------------------------
def test_detect_group_and_replay_three_unconfigured_transmitters_in_one_call():
    SR, n = 2048000, 2048
    bw = SR // n
    chan_off = [-600, -450, -300, -150, 150, 300, 450, 600]
    chans = [cm.make_channel(CF + k * bw + bw // 2, CF, SR, n, W) for k in chan_off]
    cfg = parent_cfg(cm.SFMT_U8, SR, n, channels=chans)
    B, hop, nb = cfg.wave_batch, cfg.hop(0), 15
    n_samples = (AGC + nb * B) * hop + n
    f2s = lambda f: int(f * hop)  # noqa: E731
    # (bin offset, first frame, end frame, modulation tone): 2.5 to 3.5 batches each, from batch 7 on
    extra = [(-222, AGC + 7 * B + 300, AGC + 10 * B + 460, 700.0), (77, AGC + 8 * B + 100, AGC + 11 * B + 600, 400.0),
             (512, AGC + 10 * B + 900, AGC + 13 * B + 200, 1100.0)]
    A = 0.04
    # the configured channels' carriers, unmodulated, all the time; the three others 60 % AM
    raw = tx_raw(cfg, n_samples, [(k * bw + bw / 2, A, 0, n_samples, "am", 0.0) for k in chan_off] +
                 [(k * bw, A, f2s(a), f2s(b), "am", fm) for k, a, b, fm in extra], 0.01, seed=1)
    s = lib.default_stride(cfg, 0)

    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=nb + 2)
    e.history_configure(0, nb + 1)
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
    tx = lib.group_transmissions(lib.merge_bursts(rd), cfg, 0)
    hits, jobs = [], []
    for k, a, b, fm in extra:
        hit = [t for t in tx if abs(t["freq_hz"] - (CF + k * bw)) <= bw and not t["monitored"]]
        assert len(hit) == 1, k
        job = lib.transmission_replay(hit[0], cfg, 0, hist)
        lead = (AGC + job["first_batch"] * B)
        assert hit[0]["first_frame"] - lead >= lib.REPLAY_SETTLE_BATCHES * B  # the default lead-in
        hits.append((k, a, b, fm))
        jobs.append(job)
    res = e.history_replay(jobs)  # all three in one call
    for (k, a, b, fm), job, r in zip(hits, jobs, res):
        f0 = AGC + job["first_batch"] * B  # frame of the replay's first audio sample
        batch_lo, batch_hi = f0 + B * np.arange(job["n_batches"]), f0 + B * (np.arange(job["n_batches"]) + 1)
        on = r["axc"][:, 0] == ord("*")
        inside = (batch_lo >= a) & (batch_hi <= b)
        assert inside.any() and on[inside].all(), (k, on, inside)
        assert not on[batch_hi < a - B // 2].any(), (k, on)  # not well before it
        audio = r["waveout"][inside, 0, :].reshape(-1).astype(np.float64)
        spec = np.abs(np.fft.rfft((audio - audio.mean()) * np.hanning(audio.size)))
        peak = np.argmax(spec) * W / audio.size
        assert abs(peak - fm) <= 10.0, (k, peak, fm)
    e.close()
