"""History analysis (abg_history_spectrogram / abg_history_activity) on the GPU (-m gpu).

Spectrogram rows of F = wave_batch frames on batch boundaries must be bitwise the live band spectrum of the same batches,
for every format (hop 313 at wave_rate 8008 gathers across a misalignment), fft_size 256, 2048 and 8192, strides 1, the
default and wave_batch, windows across the ring's wrap and calls of many chunks; other F and unaligned rows must match
float64.  Detector jobs must give merge_bursts of the live detector's readings over the same batches, with the window's
edge bursts flagged and kept, and report truncated batches.  Results must not depend on how jobs share calls, on
max_batches_per_run or on the live monitors; calls between runs must leave the live engine as a twin that never calls
them has it.  End to end: with the detector off, three unconfigured transmitters are found in the history alone and each
replay hears its own."""
import numpy as np
import pytest

from airband_b200 import config as cm
from airband_b200 import lib
from test_gpu_activity import _all_monitors, fetch_monitors, frame_powers, make_raw
from test_gpu_history_replay import parent_cfg, tx_raw
from test_tc_dft_math import reference_frame

pytestmark = pytest.mark.gpu
AGC = cm.AGC_EXTRA
W, CF = 8000, 120_000_000


def three_dev_cfg(sfmt, sr, fs, n, w):
    ch = cm.make_channel(CF + 300_000, CF, sr, n, w)
    return cm.Config(fft_size=n, wave_rate=w, devices=[cm.Device(sample_rate=sr, sfmt=sfmt, fullscale=fs, centerfreq=CF, channels=[ch])
                                                       for _ in range(3)])


def raws_for(cfg, nb, seed):
    """Per device noise plus gated tones: one on from the start, one across batch boundaries, short pulses."""
    B, N = cfg.wave_batch, cfg.fft_size
    out = []
    for d in range(len(cfg.devices)):
        hop, sr = cfg.hop(d), cfg.devices[d].sample_rate
        ns = (AGC + nb * B) * hop + N + hop
        s = lambda fr: int(fr * hop)  # noqa: E731
        bw = sr / N
        # pulses of 24 frames at the start of batch NB - HIST and the end of batch NB - 2: short bursts at the edges of the
        # detector's window in the tests below
        tones = [(37 * bw, 0.15, [(0, ns)]), (-211 * bw, 0.12, [(s(AGC + 6 * B + 500), s(AGC + 9 * B + 100))]),
                 (402 * bw, 0.2, [(s(AGC + 8 * B + k), s(AGC + 8 * B + k + 20)) for k in range(0, B, 150)]),
                 (-77 * bw, 0.2, [(s(AGC + (NB - HIST) * B), s(AGC + (NB - HIST) * B + 24)),
                                  (s(AGC + (NB - 1) * B - 24), s(AGC + (NB - 1) * B))])]
        out.append(make_raw(cfg, d, ns, tones, noise=0.02, seed=seed + d))
    return out


def live(cfg, raws, hist, nbmax=2, spec=None, act=None, piece_batches=1.0, between=None, setup=None):
    """An engine with the history of `hist` batches on every device, fed the streams in pieces with runs in between, its
    live spectra ({batch: power}), detector readings and audio drained after every run."""
    D = len(cfg.devices)
    e = lib.Engine(cfg, max_batches_per_run=nbmax)
    for d in range(D):
        e.history_configure(d, hist)
    for d, s in (spec or {}).items():
        e.spectrum_configure(d, s)
    for d, (s, h, m, thr) in (act or {}).items():
        e.activity_configure(d, s, h, m, thr)
    if setup:
        setup(e)
    out = dict(spec=[{} for _ in range(D)], act=[[] for _ in range(D)], audio=[[] for _ in range(D)])
    pos = [0] * D
    while True:
        pushed = False
        for d, r in enumerate(raws):
            step = int(piece_batches * cfg.wave_batch * cfg.hop(d)) * 2
            if pos[d] < r.size:
                e.push(d, r[pos[d]:pos[d] + step])
                pos[d] += step
                pushed = True
        n = e.run(-1)
        for d in range(D):
            while (g := e.fetch(d)) is not None:
                out["audio"][d].append(g)
            while (s := e.fetch_spectrum(d)) is not None:
                out["spec"][d][s[1]] = s[0]
            while (a := e.fetch_activity(d)) is not None:
                out["act"][d].append(a)
        if n and between:
            between(e)
        if n == 0 and not pushed:
            return e, out


# (name, format, sample rate, full scale, fft_size, wave_rate).  At wave_rate 8008 a batch is 1001 frames of hop 313, so
# the windows of odd batches start off a 16-byte boundary of the ring and the gather shifts every vector.
FORMATS = [("u8", cm.SFMT_U8, 2048000, 0.0, 2048, W), ("s8", cm.SFMT_S8, 2560000, 0.0, 2048, W),
           ("s16", cm.SFMT_S16, 2560000, 32766.5, 2048, W), ("f32", cm.SFMT_F32, 2048000, 1.0, 2048, W),
           ("u8_misaligned", cm.SFMT_U8, 2506504, 0.0, 2048, 8008), ("s16_misaligned", cm.SFMT_S16, 2506504, 32766.5, 2048, 8008),
           ("u8_256", cm.SFMT_U8, 2048000, 0.0, 256, W), ("s8_8192", cm.SFMT_S8, 2048000, 0.0, 8192, W)]
NB, HIST = 12, 5


# ---- 1. spectrogram = live spectrum ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,sfmt,sr,fs,n,w", FORMATS, ids=[c[0] for c in FORMATS])
def test_spectrogram_rows_are_the_live_spectra(name, sfmt, sr, fs, n, w):
    cfg = three_dev_cfg(sfmt, sr, fs, n, w)
    B = cfg.wave_batch
    strides = [1, lib.default_stride(cfg, 0), B]
    strides = [min(s, B) for s in strides]
    e, out = live(cfg, raws_for(cfg, NB, sfmt), HIST, spec={d: s for d, s in enumerate(strides)})
    jobs = []
    for d, s in enumerate(strides):
        f0, nr = lib.history_window(cfg, d, e.history_range(d), stride=s, frames_per_row=B)
        assert nr >= 3 and (f0 - AGC) % B == 0
        jobs.append(dict(dev=d, first_frame=f0, n_rows=nr, frames_per_row=B, stride=s))
    # the window crosses the ring's wrap: the ring holds HIST batches, and NB of them were appended
    hop, bpc = cfg.hop(0), 2 * cfg.devices[0].bytes_per_sample
    R = (HIST * B * hop * bpc + 15) & ~15
    lo = jobs[0]["first_frame"] * hop * bpc
    hi = ((jobs[0]["first_frame"] + jobs[0]["n_rows"] * B - 1) * hop + n) * bpc
    assert lo // R != (hi - 1) // R
    got = e.history_spectrogram(jobs)
    for d, (j, p) in enumerate(zip(jobs, got)):
        b0 = (j["first_frame"] - AGC) // B
        for r in range(j["n_rows"]):
            assert np.array_equal(p[r].view(np.uint32), out["spec"][d][b0 + r].view(np.uint32)), (d, r)
    gather_ms, spec_ms, act_ms = e.history_analysis_time()
    assert gather_ms > 0 and spec_ms > 0 and act_ms == 0
    e.close()


def _ref_rows(cfg, dev, raw, job):
    """float64 P[k] of every row of a spectrogram job."""
    d = cfg.devices[dev]
    N, hop, F, s = cfg.fft_size, cfg.hop(dev), job["frames_per_row"], job["stride"]
    by = raw.view(np.uint8)
    bpc = 2 * d.bytes_per_sample
    out = []
    for r in range(job["n_rows"]):
        fr = [job["first_frame"] + r * F + j for j in range(0, F, s)]
        rows = np.stack([by[f * hop * bpc:(f * hop + N) * bpc] for f in fr])
        out.append((np.abs(np.fft.fft(reference_frame(rows, d.sfmt, N, d.fullscale), axis=1)) ** 2).mean(axis=0))
    return np.array(out)


@pytest.mark.parametrize("name,sfmt,sr,fs,n,w", [FORMATS[0], FORMATS[3], FORMATS[4], FORMATS[6]], ids=["u8", "f32", "u8_misaligned", "u8_256"])
def test_spectrogram_of_other_rows_matches_float64(name, sfmt, sr, fs, n, w):
    cfg = three_dev_cfg(sfmt, sr, fs, n, w)
    cfg.devices = cfg.devices[:1]
    B = cfg.wave_batch
    raw = raws_for(cfg, NB, 7)[0]
    e, _ = live(cfg, [raw], NB + 1)
    first, end = e.history_range(0)
    jobs = []
    for F, s, off in ((77, 1, 37), (2 * B + 13, 5, 511), (333, 333, 1), (B // 8, 3, 0)):
        f0, nr = lib.history_window(cfg, 0, (first, end), stride=s, frames_per_row=F)
        jobs.append(dict(dev=0, first_frame=f0 + off, n_rows=min(nr - 1, 6), frames_per_row=F, stride=s))
    for j, p in zip(jobs, e.history_spectrogram(jobs)):
        ref = _ref_rows(cfg, 0, raw, j)
        err = np.abs(p.astype(np.float64) - ref)
        assert np.all(err <= 1e-5 * ref + 1e-6 * ref.max(axis=1, keepdims=True)), (j, float((err / ref.max()).max()))
    e.close()


# ---- 2. detector = merged live readings ----------------------------------------------------------------------------------------
def _q(frame, B, s):
    n = -(-B // s)
    f = int(frame) - AGC
    return (f // B) * n + (f % B) // s


def _check_against_live(cfg, got, readings, b0, nb, settings):
    """got (a history_activity result over batches [b0, b0 + nb)) against the live readings of the same batches."""
    s, h, m = settings
    B = cfg.wave_batch
    n_sel = -(-B // s)
    rd = [r for r in readings if b0 <= r["batch_seq"] < b0 + nb]
    assert [r["batch_seq"] for r in rd] == list(range(b0, b0 + nb))
    b = got["bursts"]
    assert got["n_truncated"] == 0
    assert np.array_equal(b, np.sort(b, order=["bin", "first_frame"]))
    span = np.array([_q(x["last_frame"], B, s) - _q(x["first_frame"], B, s) + 1 for x in b], np.int64)
    # the edge flags: the first member in the window's first batch within hang of its start, the last in its last batch
    # within hang of its end; the pieces of the first and last readings say the same
    i_first = [(int(x["first_frame"]) - AGC - b0 * B) // s for x in b]
    i_last = [(int(x["last_frame"]) - AGC - (b0 + nb - 1) * B) // s for x in b]
    starts = {(int(p["bin"]), int(p["first_frame"])) for p in rd[0]["pieces"] if p["flags"] & lib.BURST_OPEN_START}
    ends = {(int(p["bin"]), int(p["last_frame"])) for p in rd[-1]["pieces"] if p["flags"] & lib.BURST_OPEN_END}
    for x, a, z in zip(b, i_first, i_last):
        fs = bool(x["flags"] & lib.BURST_OPEN_START)
        fe = bool(x["flags"] & lib.BURST_OPEN_END)
        assert fs == (0 <= a <= h) == ((int(x["bin"]), int(x["first_frame"])) in starts)
        assert fe == (z >= n_sel - 1 - h) == ((int(x["bin"]), int(x["last_frame"])) in ends)
        assert x["flags"] & ~3 == 0
    # without the flags, and with the short edge bursts dropped, it is merge_bursts of the live readings
    kept = b[(b["flags"] == 0) | (span >= m)].copy()
    kept["flags"] = 0
    want = lib.merge_bursts(rd)
    assert np.array_equal(kept, want), (kept.size, want.size)
    assert np.all(span[b["flags"] == 0] >= m)
    return int(((b["flags"] != 0) & (span < m)).sum())


DET = [FORMATS[0], FORMATS[1], FORMATS[2], FORMATS[3], FORMATS[4], FORMATS[7]]


@pytest.mark.parametrize("name,sfmt,sr,fs,n,w", DET, ids=[c[0] for c in DET])
def test_detector_jobs_are_the_merged_live_readings(name, sfmt, sr, fs, n, w):
    cfg = three_dev_cfg(sfmt, sr, fs, n, w)
    B = cfg.wave_batch
    raws = raws_for(cfg, NB, 3 * sfmt)
    # three settings: stride 1 with hang n - 1; the default stride with min_span 3; stride 3 with a min_span edge bursts miss
    ds = min(lib.default_stride(cfg, 0), B)
    settings = [(1, B - 1, 1), (ds, 1, 3), (3, 2, 40)]
    act = {}
    for d, (s, h, m) in enumerate(settings):
        P = frame_powers(cfg, d, raws[d], 0, s)
        act[d] = (s, h, m, lib.activity_threshold(P.mean(axis=0), 12.0, 16))
    e, out = live(cfg, raws, HIST, act=act)
    jobs, wins = [], []
    for d, (s, h, m) in enumerate(settings):
        b0, nb = lib.history_window(cfg, d, e.history_range(d), stride=s)
        assert nb >= 3
        wins.append((b0, nb))
        jobs.append(dict(dev=d, first_batch=b0, n_batches=nb, stride=s, hang=h, min_span=m, thr=act[d][3]))
    got = e.history_activity(jobs)
    short_edges = 0
    for d in range(3):
        assert got[d]["bursts"].size > 3
        short_edges += _check_against_live(cfg, got[d], out["act"][d], *wins[d], settings[d])
    assert short_edges > 0  # an edge burst below min_span was kept
    assert e.history_analysis_time()[1] == 0 and e.history_analysis_time()[2] > 0
    e.close()


def test_truncated_batches_are_reported():
    cfg = three_dev_cfg(cm.SFMT_U8, 2048000, 0.0, 2048, W)
    cfg.devices = cfg.devices[:1]
    raws = raws_for(cfg, 6, 1)
    P = frame_powers(cfg, 0, raws[0], 0, 1)
    thr = np.median(P, axis=0).astype(np.float32)  # half of all frames active, in short runs: far more than 4096 pieces
    e, out = live(cfg, raws, 7, act={0: (1, 0, 1, thr)})
    b0, nb = lib.history_window(cfg, 0, e.history_range(0))
    got = e.history_activity([dict(dev=0, first_batch=b0, n_batches=nb, stride=1, thr=thr)])[0]
    live_trunc = sum(r["n_total"] > len(r["pieces"]) for r in out["act"][0] if b0 <= r["batch_seq"] < b0 + nb)
    assert got["n_truncated"] == live_trunc == nb
    e.close()


# ---- 3. independence and many chunks --------------------------------------------------------------------------------------------
def test_results_do_not_depend_on_calls_runs_or_live_monitors_and_span_chunks():
    cfg = three_dev_cfg(cm.SFMT_U8, 2048000, 0.0, 2048, W)
    cfg.devices = cfg.devices[:2]
    B = cfg.wave_batch
    nb_all = 24
    raws = raws_for(cfg, nb_all, 11)
    s = lib.default_stride(cfg, 0)
    thr = lib.activity_threshold(frame_powers(cfg, 0, raws[0], 0, s).mean(axis=0), 12.0, 16)
    # A: max_batches_per_run 1, the live spectrum and detector on, pushes of 0.7 batches; B: 4, both off, 2.3 batches
    ea, oa = live(cfg, raws, nb_all - 2, nbmax=1, spec={0: s, 1: 1}, act={0: (s, 1, 2, thr)}, piece_batches=0.7)
    eb, _ = live(cfg, raws, nb_all - 2, nbmax=4, piece_batches=2.3)
    assert ea.history_range(0) == eb.history_range(0)
    b0, nb = lib.history_window(cfg, 0, ea.history_range(0), stride=1)  # the window every stride below fits
    assert nb >= 18
    # 64 jobs over both devices: 8 MB of raw bytes each, so the calls take several chunks and cut jobs between them
    sj = [dict(dev=k % 2, first_frame=AGC + (b0 + k % 3) * B, n_rows=nb - 2, frames_per_row=B, stride=[s, 1, 7][k % 3]) for k in range(64)]
    aj = [dict(dev=k % 2, first_batch=b0 + k % 3, n_batches=nb - 2, stride=s, hang=k % 3, min_span=1 + k % 4, thr=thr) for k in range(64)]
    spec_a, act_a = ea.history_spectrogram(sj), ea.history_activity(aj)
    late = eb.history_spectrogram(sj[40:][::-1])[::-1]  # split over two calls, the first in reverse order
    spec_b = eb.history_spectrogram(sj[:40]) + late
    act_b = [eb.history_activity([j])[0] for j in aj[:6]] + eb.history_activity(aj[6:])
    for k in range(64):
        assert np.array_equal(spec_a[k].view(np.uint32), spec_b[k].view(np.uint32)), k
        assert np.array_equal(act_a[k]["bursts"], act_b[k]["bursts"]) and act_a[k]["n_truncated"] == act_b[k]["n_truncated"] == 0, k
    # and they are the live monitors' results where those ran with the same settings
    for k in range(0, 64, 6):  # device 0, stride s
        j = sj[k]
        fb = (j["first_frame"] - AGC) // B
        for r in range(j["n_rows"]):
            assert np.array_equal(spec_a[k][r].view(np.uint32), oa["spec"][0][fb + r].view(np.uint32))
    _check_against_live(cfg, ea.history_activity([dict(aj[0], hang=1, min_span=2)])[0], oa["act"][0], b0, nb - 2, (s, 1, 2))
    ea.close()
    eb.close()


# ---- 4. the live path --------------------------------------------------------------------------------------------------------------
def test_live_runs_are_unchanged_by_calls_between_them():
    cfg = three_dev_cfg(cm.SFMT_S8, 2560000, 0.0, 2048, W)
    cfg.devices = cfg.devices[:1]
    B = cfg.wave_batch
    raws = raws_for(cfg, NB, 5)
    s = lib.default_stride(cfg, 0)
    thr = np.full(cfg.fft_size, 40.0, np.float32)

    def setup(e):
        _all_monitors(e, cfg, 0)
        e.activity_configure(0, s, 1, 2, thr)

    def trace(call):
        log, count, calls = [], [0], []

        def between(e):
            log.append((e.history_range(0), fetch_monitors(e, 0), e.launch_count() - count[0]))
            try:
                b0, nb = lib.history_window(cfg, 0, e.history_range(0), stride=s)
            except ValueError:
                b0 = None
            if call and b0 is not None:
                calls.append(e.history_spectrogram([dict(dev=0, first_frame=AGC + b0 * B, n_rows=nb, stride=s)])[0].tobytes())
                calls.append(e.history_activity([dict(dev=0, first_batch=b0, n_batches=nb, stride=1, hang=3, thr=thr)])[0]["bursts"].tobytes())
            count[0] = e.launch_count()  # the calls' own launches are not a run's

        e, out = live(cfg, raws, 4, setup=setup, between=between)
        log.append([(g[0].tobytes(), g[1].tobytes(), g[2].tobytes()) for g in out["audio"][0]])
        log.append([(r["batch_seq"], r["n_total"], r["pieces"].tobytes()) for r in out["act"][0]])
        log.append(sorted((k, v.tobytes()) for k, v in out["spec"][0].items()))
        e.close()
        return log, calls

    (with_calls, calls), (without, _) = trace(True), trace(False)
    assert len(without[-3]) == NB
    assert with_calls == without
    assert len(calls) >= 6


# ---- 5. errors ----------------------------------------------------------------------------------------------------------------------
def test_error_codes():
    cfg = three_dev_cfg(cm.SFMT_U8, 2048000, 0.0, 2048, W)
    cfg.devices = cfg.devices[:1]
    B, hop, N = cfg.wave_batch, cfg.hop(0), cfg.fft_size
    raws = raws_for(cfg, NB, 2)
    thr = np.full(N, 40.0, np.float32)
    e = lib.Engine(cfg, max_batches_per_run=2)

    def code(fn, jobs):
        with pytest.raises(lib.AbgError) as ex:
            fn(jobs)
        return ex.value.code, str(ex.value)

    spec = lambda **kw: dict(dict(dev=0, first_frame=AGC + 8 * B, n_rows=1, frames_per_row=B, stride=1), **kw)  # noqa: E731
    act = lambda **kw: dict(dict(dev=0, first_batch=8, n_batches=1, stride=1, hang=0, min_span=1, thr=thr), **kw)  # noqa: E731
    assert code(e.history_spectrogram, [spec()])[0] == -5  # history off
    assert code(e.history_activity, [act()])[0] == -5
    e.close()
    e, _ = live(cfg, raws, HIST)
    first, end = e.history_range(0)
    assert (first, end) == ((AGC + (NB - HIST) * B) * hop, (AGC + NB * B) * hop)
    b_lo, b_hi = NB - HIST, NB - 2  # batches whose every frame the history holds: the last batch's tail is not there yet
    assert lib.history_window(cfg, 0, (first, end)) == (b_lo, b_hi - b_lo + 1)
    ok = e.history_activity([act(first_batch=b_lo, n_batches=b_hi - b_lo + 1)])[0]
    ok_s = e.history_spectrogram([spec(first_frame=AGC + b_lo * B, n_rows=b_hi - b_lo + 1)])[0]
    assert ok_s.shape == (b_hi - b_lo + 1, N)
    # one frame too early (hop samples before first); one frame too late: the last frame after f_max, the last one whose
    # samples all lie before end
    rc, msg = code(e.history_spectrogram, [spec(first_frame=AGC + b_lo * B - 1, n_rows=1)])
    assert rc == -5 and f"[{first - hop}, {first - hop + (B - 1) * hop + N})" in msg and f"[{first}, {end})" in msg, msg
    f_max = (end - N) // hop
    assert e.history_spectrogram([spec(first_frame=f_max - (B - 1), n_rows=1)])[0].shape == (1, N)
    rc, msg = code(e.history_spectrogram, [spec(first_frame=f_max + 1 - (B - 1), n_rows=1)])
    assert rc == -5 and f"[{(f_max + 2 - B) * hop}, {(f_max + 1) * hop + N})" in msg, msg
    assert code(e.history_activity, [act(first_batch=b_lo - 1)])[0] == -5
    rc, msg = code(e.history_activity, [act(first_batch=b_hi + 1)])
    assert rc == -5 and f"{end + N - hop})" in msg, msg
    assert code(e.history_activity, [act(first_batch=b_lo, n_batches=b_hi - b_lo + 2)])[0] == -5
    assert code(e.history_activity, [act(dev=1)])[0] == -5
    # what abg_activity_configure refuses, stride 0, n_batches 0; bad rows; job counts
    bad_thr = thr.copy()
    bad_thr[17] = np.nan
    for kw in (dict(stride=0), dict(stride=B + 1), dict(hang=B), dict(min_span=0), dict(hang=-1), dict(thr=bad_thr),
               dict(thr=np.zeros(N, np.float32)), dict(n_batches=0)):
        assert code(e.history_activity, [act(first_batch=b_lo, **kw)])[0] == -2, kw
    for kw in (dict(stride=0), dict(stride=B + 1), dict(n_rows=0), dict(frames_per_row=0), dict(frames_per_row=5, stride=6)):
        assert code(e.history_spectrogram, [spec(first_frame=AGC + b_lo * B, **kw)])[0] == -2, kw
    assert code(e.history_spectrogram, [])[0] == -2
    assert code(e.history_activity, [])[0] == -2
    # a failed call changes nothing
    assert np.array_equal(e.history_activity([act(first_batch=b_lo, n_batches=b_hi - b_lo + 1)])[0]["bursts"], ok["bursts"])
    assert np.array_equal(e.history_spectrogram([spec(first_frame=AGC + b_lo * B, n_rows=b_hi - b_lo + 1)])[0], ok_s)
    e.history_configure(0, 0)  # frees the analysis buffers; the next call finds no history
    assert code(e.history_activity, [act(first_batch=b_lo)])[0] == -5
    e.close()


# ---- 6. end to end, nothing configured but the history ----------------------------------------------------------------------------
def test_find_and_replay_three_unconfigured_transmitters_from_the_history_alone():
    SR, n = 2048000, 2048
    bw = SR // n
    chan_off = [-600, -450, -300, -150, 150, 300, 450, 600]
    chans = [cm.make_channel(CF + k * bw + bw // 2, CF, SR, n, W) for k in chan_off]
    cfg = parent_cfg(cm.SFMT_U8, SR, n, channels=chans)
    B, hop, nb = cfg.wave_batch, cfg.hop(0), 15
    n_samples = (AGC + nb * B) * hop + n
    f2s = lambda f: int(f * hop)  # noqa: E731
    extra = [(-222, AGC + 7 * B + 300, AGC + 10 * B + 460, 700.0), (77, AGC + 8 * B + 100, AGC + 11 * B + 600, 400.0),
             (512, AGC + 10 * B + 900, AGC + 13 * B + 200, 1100.0)]
    A = 0.04
    raw = tx_raw(cfg, n_samples, [(k * bw + bw / 2, A, 0, n_samples, "am", 0.0) for k in chan_off] +
                 [(k * bw, A, f2s(a), f2s(b), "am", fm) for k, a, b, fm in extra], 0.01, seed=1)
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=nb + 2)
    e.history_configure(0, nb + 1)  # the detector and the spectrum stay off
    e.push(0, raw)
    while e.run(-1) > 0:
        while e.fetch(0) is not None:
            pass
        assert e.fetch_activity(0) is None and e.fetch_spectrum(0) is None
    hist = e.history_range(0)
    tx = lib.history_transmissions(e, cfg, 0, margin_db=13.0, half_width=16, stride=lib.default_stride(cfg, 0), hang=1, min_span=2)
    jobs = []
    for k, a, b, fm in extra:
        hit = [t for t in tx if abs(t["freq_hz"] - (CF + k * bw)) <= bw and not t["monitored"]]
        assert len(hit) == 1, (k, [(t["freq_hz"] - CF) / bw for t in tx])
        tol = 2 * (n // hop + lib.default_stride(cfg, 0))  # frames that overlap its edges may be active too
        assert abs(hit[0]["first_frame"] - a) <= tol and abs(hit[0]["last_frame"] - b) <= tol, (k, hit[0])
        jobs.append(lib.transmission_replay(hit[0], cfg, 0, hist))
    res = e.history_replay(jobs)
    for (k, a, b, fm), job, r in zip(extra, jobs, res):
        f0 = AGC + job["first_batch"] * B
        batch_lo, batch_hi = f0 + B * np.arange(job["n_batches"]), f0 + B * (np.arange(job["n_batches"]) + 1)
        on = r["axc"][:, 0] == ord("*")
        inside = (batch_lo >= a) & (batch_hi <= b)
        assert inside.any() and on[inside].all(), (k, on, inside)
        assert not on[batch_hi < a - B // 2].any(), (k, on)
        audio = r["waveout"][inside, 0, :].reshape(-1).astype(np.float64)
        spec = np.abs(np.fft.rfft((audio - audio.mean()) * np.hanning(audio.size)))
        peak = np.argmax(spec) * W / audio.size
        assert abs(peak - fm) <= 10.0, (k, peak, fm)
    e.close()
