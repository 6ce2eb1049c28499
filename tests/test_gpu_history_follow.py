"""Live follow (abg_follow_open ...) on the GPU (-m gpu).

Every session's batches must be bitwise those of one long abg_history_replay of the same window, for every format
(hop 313 and wave_rate 8008 gather across misalignments), every K1 path and an AFC session, AM and NFM channels with
CTCSS, notch, bandwidth and I/Q outputs, however follow_run calls split the batches, whatever other sessions do, and with
replays in between.  After every live run and follow_run(-1) a session is one batch behind the live engine.  An unfetched
session stops at its queue and continues bitwise; one left behind the history is lost, with its queued batches still
fetchable.  The live engine's outputs, monitors, history and launches stay those of a twin without sessions.  End to
end: a transmitter that keys up mid-stream is detected, followed across the live edge, and heard until it stops."""
import ctypes as C

import numpy as np
import pytest

import oracle_py as op
import parity
from airband_b200 import config as cm
from airband_b200 import lib
from test_gpu_activity import _all_monitors, fetch_monitors
from test_gpu_history_replay import CASES, CF, NB, W, parent_cfg, scenario, tx_raw
from test_history_follow_cpu import available_end

pytestmark = pytest.mark.gpu
AGC = cm.AGC_EXTRA
BIG = NB + 2  # a history that keeps the whole stream, so that one replay can cover every followed batch


def stream(cfg, raws, nbmax, hist, fft_mode=0, after=None, setup=None):
    """A parent engine with a history of `hist` batches on every device, fed one batch of each device per run; every
    run's live outputs are drained.  after(e, k) is called after run k, and once more after the last one (with the
    stream exhausted)."""
    e = lib.Engine(cfg, max_batches_per_run=nbmax, fft_mode=fft_mode)
    for d in range(len(cfg.devices)):
        e.history_configure(d, hist)
    if setup:
        setup(e)
    steps = [cfg.wave_batch * cfg.hop(d) * 2 for d in range(len(cfg.devices))]
    pos, k = 0, 0
    while True:
        for d, raw in enumerate(raws):
            if pos * steps[d] < raw.size:
                e.push(d, raw[pos * steps[d]:(pos + 1) * steps[d]])
        pos += 1
        n = e.run(-1)
        for d in range(len(cfg.devices)):
            while e.fetch(d) is not None:
                pass
        if after:
            after(e, k)
        k += 1
        if n == 0 and all(pos * s >= r.size for s, r in zip(steps, raws)):
            return e


def live_batches(e, cfg, d=0):
    """Batches of device d the live engine has enqueued (its last batch is this minus one)."""
    end = e.history_range(d)[1]
    return 0 if end == 0 else (end // cfg.hop(d) - AGC) // cfg.wave_batch


class Sink:
    """Every batch fetched from each session, checked to be contiguous."""

    def __init__(self):
        self.got = {}

    def fetch(self, e, sid, max_batches=None):
        r = e.follow_fetch(sid, max_batches)
        if r["first_batch"] is None:
            return 0
        lst = self.got.setdefault(sid, [])
        if lst:
            assert r["first_batch"] == lst[-1][0] + len(lst[-1][1]), sid
        lst.append((r["first_batch"], r["waveout"], r["iq"], r["axc"]))
        return len(r["waveout"])

    def result(self, sid):
        lst = self.got[sid]
        return dict(first_batch=lst[0][0], waveout=np.concatenate([x[1] for x in lst]), iq=np.concatenate([x[2] for x in lst]),
                    axc=np.concatenate([x[3] for x in lst]))


def finish(e, sink, sids):
    """Catch every session up with what the history holds and fetch everything."""
    while e.follow_run(-1) > 0:
        pass
    for s in sids:
        while sink.fetch(e, s):
            pass


def same_as_replay(ref, r, job, stats=None):
    """r (a Sink result) is bitwise batches [0, n) of one replay of job from its first batch, on the reference parent."""
    n = len(r["waveout"])
    assert n >= 1 and r["first_batch"] == job["first_batch"]
    rep = ref.history_replay([dict(dev=job["dev"], first_batch=job["first_batch"], n_batches=n, channels=job["channels"])])[0]
    assert np.array_equal(r["waveout"].view(np.uint32), rep["waveout"].view(np.uint32))
    assert np.array_equal(r["iq"].view(np.uint64), rep["iq"].view(np.uint64))
    assert np.array_equal(r["axc"], rep["axc"])
    if stats is not None:
        assert [bytes(s) for s in stats] == [bytes(s) for s in rep["stats"]]
    return rep


def jobs_for(jobs):
    """The scenario's replay jobs as sessions that start earlier: (job, when to open: "start" = before the first run,
    an int k = after run k, "edge" = at the live edge after run 6)."""
    out = [(dict(dev=0, first_batch=1, channels=jobs[0]["channels"]), "start"),
           (dict(dev=0, first_batch=3, channels=jobs[1]["channels"]), 7),  # opened 4 batches back: catches up
           (dict(dev=0, first_batch=None, channels=jobs[2]["channels"]), "edge")]
    if len(jobs) > 3:
        out.append((dict(dev=0, first_batch=2, channels=jobs[3]["channels"]), "start"))  # AFC
    return out


def follow_scenario(cfg, raw, jobs, nbmax, fft_mode, policy, queue=16, stall=None):
    """Stream the scenario with its sessions; policy "each" = follow_run(1) after every run, "lazy" = follow_run(-1)
    every third run, "once" = nothing until the stream ends.  stall = (session index, run): that session is not fetched
    before that run.  Returns (parent, sink, [(sid, job)])."""
    sink, opened = Sink(), []

    def open_(e, job):
        sid = e.follow_open(**job, queue_batches=queue)
        opened.append((sid, job))

    def after(e, k):
        for job, when in jobs_for(jobs):
            if when == k:
                open_(e, job)
            elif when == "edge" and k == 6:
                open_(e, dict(job, first_batch=live_batches(e, cfg)))
        if policy == "each":
            e.follow_run(1)
        elif policy == "lazy" and k % 3 == 2:
            e.follow_run(-1)
        if policy != "once":
            for i, (sid, _) in enumerate(opened):
                if stall and stall[0] == i and k < stall[1]:
                    info = e.follow_info(sid)
                    assert info["queued"] <= queue
                    if k == stall[1] - 1:
                        assert info["queued"] == queue and info["next_batch"] == opened[i][1]["first_batch"] + queue
                    continue
                sink.fetch(e, sid)

    def setup(e):
        for job, when in jobs_for(jobs):
            if when == "start":
                open_(e, job)

    e = stream(cfg, [raw], nbmax, BIG, fft_mode, after=after, setup=setup)
    finish(e, sink, [s for s, _ in opened])
    return e, sink, opened


# ---- 1. one long replay, every format and K1 path ----------------------------------------------------------------------------
@pytest.mark.parametrize("name,sfmt,sr,fs,fft_mode,afc,w", CASES, ids=[c[0] for c in CASES])
def test_follow_is_bitwise_one_long_replay(name, sfmt, sr, fs, fft_mode, afc, w):
    cfg, raw, jobs = scenario(sfmt, sr, fs, afc=afc, w=w)
    e, sink, opened = follow_scenario(cfg, raw, jobs, nbmax=2, fft_mode=fft_mode, policy="each")
    assert len(opened) == len(jobs_for(jobs))
    for sid, job in opened:
        r = sink.result(sid)
        assert r["first_batch"] + len(r["waveout"]) == NB - 1  # every batch the history holds all samples of
        same_as_replay(e, r, job, [e.follow_stats(sid, c) for c in range(len(job["channels"]))])
    assert any((sink.result(s)["axc"] != ord(" ")).any() for s, _ in opened)  # something opened
    g, k = e.follow_time()
    assert g == 0 and k == 0  # the last follow_run enqueued nothing
    e.close()


def test_follow_passes_the_oracle_strict_gate():
    cfg, raw, jobs = scenario(cm.SFMT_U8, 2500000)
    e, sink, opened = follow_scenario(cfg, raw, jobs, nbmax=2, fft_mode=0, policy="lazy")
    B, hop, N = cfg.wave_batch, cfg.hop(0), cfg.fft_size
    for sid, job in opened[:2]:  # AM and NFM
        r = sink.result(sid)
        n = len(r["waveout"])
        S = job["first_batch"] * B * hop
        need = (AGC + n * B) * hop + N - hop
        data = np.concatenate([e.history_raw(0, S, need), raw[2 * (S + need):2 * (S + need + hop)]])
        d = cfg.devices[0]
        oc = cm.Config(fft_size=N, wave_rate=W, devices=[cm.Device(sample_rate=d.sample_rate, sfmt=d.sfmt, centerfreq=CF,
                                                                   channels=job["channels"])])
        res_o, o = op.run_oracle(oc, [data])
        ow, _, oa = res_o[0]
        o.close()
        gw = r["waveout"].transpose(1, 0, 2).reshape(len(job["channels"]), -1)
        rep = parity.strict((gw, None, r["axc"]), (ow, None, oa))
        assert rep["ok"], rep
    e.close()


# ---- 2. however follow_run splits the batches -----------------------------------------------------------------------------
def test_three_ways_of_driving_a_session_and_a_stalled_queue_give_the_same_batches():
    cfg, raw, jobs = scenario(cm.SFMT_S8, 2560000, afc=True)
    results = []
    for policy, nbmax, stall in (("each", 2, None), ("lazy", 4, None), ("once", 1, None), ("each", 3, (0, 8))):
        e, sink, opened = follow_scenario(cfg, raw, jobs, nbmax=nbmax, fft_mode=0, policy=policy, queue=3 if stall else 16,
                                          stall=stall)
        results.append([sink.result(s) for s, _ in opened])
        if policy == "once":
            ref = e
            ref_jobs = [j for _, j in opened]
        else:
            e.close()
    for res in results[1:]:
        for a, b in zip(results[0], res):
            assert a["first_batch"] == b["first_batch"]
            for k in ("waveout", "iq", "axc"):
                assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k
    for r, job in zip(results[0], ref_jobs):
        same_as_replay(ref, r, job)
    ref.close()


# ---- 3. lag ----------------------------------------------------------------------------------------------------------------------
def test_a_session_trails_the_live_engine_by_one_batch():
    cfg, raw, jobs = scenario(cm.SFMT_U8, 2560000)
    B, hop, N = cfg.wave_batch, cfg.hop(0), cfg.fft_size
    assert B * hop >= N - hop
    big = tx_raw(cfg, (AGC + 24 * B) * hop + N + hop, [], 0.01, seed=5)
    e = lib.Engine(cfg, max_batches_per_run=4)
    e.history_configure(0, 12)
    sink, sids = Sink(), []
    step, pos, k = 4 * B * hop * 2, 0, 0
    while True:
        if pos < big.size:
            e.push(0, big[pos:pos + step])
            pos += step
        n = e.run(-1)
        while e.fetch(0) is not None:
            pass
        L = live_batches(e, cfg)
        if k == 0:
            sids.append((e.follow_open(0, 1, jobs[0]["channels"]), 1))
        if k == 2:  # at the live edge: it starts there
            sids.append((e.follow_open(0, L, jobs[1]["channels"]), L))
        if k == 3:  # 6 batches back while the live engine runs 4 per run: one call catches it up
            sids.append((e.follow_open(0, L - 6, jobs[2]["channels"]), L - 6))
        if e.follow_run(-1) > 0:
            g, t = e.follow_time()
            assert g > 0 and t > 0
        for s, fb in sids:
            info = e.follow_info(s)
            assert info["next_batch"] == max(L - 1, fb) == max(available_end(e.history_range(0), B, hop, N), fb), (k, info)
            assert not info["lost"]
            sink.fetch(e, s)
        k += 1
        if n == 0 and pos >= big.size:
            break
    assert live_batches(e, cfg) == 24 and len(sids) == 3
    assert all(e.follow_info(s)["next_batch"] == 23 for s, _ in sids)
    e.close()


# ---- 4. sessions opening, closing, sharing devices and engines, with replays in between ----------------------------------------
def test_sessions_open_close_reuse_grow_and_share_with_replays_in_between():
    torch = pytest.importorskip("torch")
    cfg0, raw0, jobs0 = scenario(cm.SFMT_U8, 2500000)
    cfg1, raw1, jobs1 = scenario(cm.SFMT_S8, 2560000)
    cfg = cm.Config(fft_size=cfg0.fft_size, wave_rate=W, devices=[cfg0.devices[0], cfg1.devices[0]])
    X = jobs0[0]["channels"]  # one shape: 3 AM channels, no AFC, no I/Q output
    X2 = [X[2], X[0], X[1]]   # same shape, other list
    sink, opened, mem = Sink(), {}, {}

    def free():
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info()[0]

    def op_(e, name, dev, fb, chans):
        opened[name] = (e.follow_open(dev, fb, chans), dict(dev=dev, first_batch=fb, channels=chans))

    def after(e, k):
        if k == 0:
            op_(e, "A", 0, 1, X)
            mem["a"] = free()
            op_(e, "B", 0, 1, X2)  # two sessions on one device; a second engine
            mem["b"] = free()
            op_(e, "E", 0, 2, X)   # a third engine, with two devices of the shape
            op_(e, "C", 1, 1, jobs1[1]["channels"])  # the other device
        if k == 2:
            f = free()
            op_(e, "F", 0, 2, X2)  # the free device next to E
            assert abs(free() - f) < 2 << 20
        if k == 4:
            e.follow_close(opened.pop("E")[0])
            f = free()
            op_(e, "G", 0, 3, X)  # E's device again, reset while F keeps running beside it
            assert abs(free() - f) < 2 << 20
        if k == 5:
            e.follow_close(opened.pop("B")[0])
        if k % 2 == 1 and k >= 3:  # replays in between
            first = e.history_range(0)[0]
            b0 = -(-first // (cfg.wave_batch * cfg.hop(0)))
            e.history_replay([dict(dev=0, first_batch=b0, n_batches=1, channels=X)])
        e.follow_run(-1 if k % 2 else 1)
        for s, _ in opened.values():
            sink.fetch(e, s)

    e = stream(cfg, [raw0, raw1], nbmax=2, hist=BIG, after=after)
    assert mem["a"] - mem["b"] >= 2 * 4 * cfg.wave_batch * cfg.hop(0) * 2  # a new engine's input buffers, at least
    finish(e, sink, [s for s, _ in opened.values()])
    assert set(opened) == {"A", "C", "F", "G"}
    for name, (sid, job) in opened.items():
        same_as_replay(e, sink.result(sid), job)
    for s, _ in opened.values():
        e.follow_close(s)
    e.history_configure(0, 0)
    e.history_configure(1, 0)  # the last history off frees the follow engines
    with pytest.raises(lib.AbgError):
        e.follow_open(0, 1, X)
    e.close()


# ---- 5. queue and loss --------------------------------------------------------------------------------------------------------
def test_a_session_left_behind_is_lost_and_the_others_are_unaffected():
    cfg, raw, jobs = scenario(cm.SFMT_U8, 2500000)
    sink, sids = Sink(), {}

    def setup(e):
        sids["lazy"] = e.follow_open(0, 1, jobs[0]["channels"], queue_batches=2)
        sids["ok"] = e.follow_open(0, 1, jobs[1]["channels"])
        sids["ok2"] = e.follow_open(0, 1, jobs[0]["channels"])

    def after(e, k):
        e.follow_run(-1)
        sink.fetch(e, sids["ok"])
        sink.fetch(e, sids["ok2"])
        info = e.follow_info(sids["lazy"])
        assert info["queued"] <= 2
        # lost once the history (4 batches) has overwritten its next sample: batch 3's first frame
        B, hop = cfg.wave_batch, cfg.hop(0)
        assert info["lost"] == (e.history_range(0)[0] > (AGC + 3 * B) * hop + cfg.fft_size), (k, info, e.history_range(0))

    e = stream(cfg, [raw], nbmax=2, hist=4, after=after, setup=setup)
    info = e.follow_info(sids["lazy"])
    assert info["lost"] and info["queued"] == 2 and info["next_batch"] == 3
    got = e.follow_fetch(sids["lazy"])
    assert got["first_batch"] == 1 and len(got["waveout"]) == 2
    with pytest.raises(lib.AbgError) as ex:
        e.follow_fetch(sids["lazy"])
    assert ex.value.code == -5 and "lost" in str(ex.value)
    finish(e, sink, [sids["ok"], sids["ok2"]])
    ref = stream(cfg, [raw], nbmax=2, hist=BIG)
    for name, ch in (("ok", jobs[1]["channels"]), ("ok2", jobs[0]["channels"])):
        same_as_replay(ref, sink.result(sids[name]), dict(dev=0, first_batch=1, channels=ch))
    # the lost session's two batches too
    rep = ref.history_replay([dict(dev=0, first_batch=1, n_batches=2, channels=jobs[0]["channels"])])[0]
    assert np.array_equal(got["waveout"].view(np.uint32), rep["waveout"].view(np.uint32))
    e.follow_close(sids["lazy"])
    ref.close()
    e.close()


# ---- 6. the live path -------------------------------------------------------------------------------------------------------------
def test_live_runs_are_unchanged_by_sessions():
    cfg, raw, jobs = scenario(cm.SFMT_S8, 2560000, afc=True)
    thr = np.full(cfg.fft_size, 40.0, np.float32)

    def trace(follow):
        log, sids, count = [], [], [0]

        def setup(e):
            _all_monitors(e, cfg, 0)
            e.activity_configure(0, lib.default_stride(cfg, 0), 1, 2, thr)
            count[0] = e.launch_count()

        def after(e, k):
            log.append((e.history_range(0), fetch_monitors(e, 0), e.launch_count() - count[0]))
            while (a := e.fetch_activity(0)) is not None:
                log.append(("act", a["batch_seq"], a["n_total"], a["pieces"].tobytes()))
            if follow:
                if k in (0, 3):
                    sids.append(e.follow_open(0, 1 + k, jobs[k % 4]["channels"], queue_batches=4))
                if k == 5:
                    e.follow_close(sids.pop(0))
                e.follow_run(-1)
                for s in sids[:-1]:  # the newest one is never fetched: it stops at its queue
                    e.follow_fetch(s)
            count[0] = e.launch_count()  # a session's own launches are not a run's

        e = stream(cfg, [raw], nbmax=2, hist=4, setup=setup, after=after)
        e.close()
        return log

    assert trace(True) == trace(False)


# ---- 7. errors ------------------------------------------------------------------------------------------------------------------
def test_error_codes():
    cfg, raw, jobs = scenario(cm.SFMT_U8, 2560000)
    B, hop = cfg.wave_batch, cfg.hop(0)
    ch = jobs[0]["channels"]
    e = lib.Engine(cfg, max_batches_per_run=2)

    def code(f, *a, **kw):
        with pytest.raises(lib.AbgError) as ex:
            f(*a, **kw)
        return ex.value.code, str(ex.value)

    assert code(e.follow_open, 0, 1, ch)[0] == -5  # history off
    e.history_configure(0, 4)
    step = B * hop * 2
    for p in range(0, raw.size, step):
        e.push(0, raw[p:p + step])
        while e.run(-1):
            while e.fetch(0) is not None:
                pass
    first, end = e.history_range(0)
    b_lo = -(-first // (B * hop))
    rc, msg = code(e.follow_open, 0, b_lo - 1, ch)
    assert rc == -5 and f"[{first}, {end})" in msg, msg
    assert code(e.follow_open, 1, b_lo, ch)[0] == -5
    assert code(e.follow_open, -1, b_lo, ch)[0] == -5
    assert code(e.follow_open, 0, b_lo, [cm.Channel(bin=cfg.fft_size)])[0] == -2
    assert code(e.follow_open, 0, b_lo, [cm.Channel(bin=5, modulation=7)])[0] == -2
    assert code(e.follow_open, 0, b_lo, ch, queue_batches=0)[0] == -2
    chans = cm.channels_to_c(ch)
    assert e.L.abg_follow_open(e.h, 0, b_lo, len(ch), C.cast(chans, C.POINTER(cm.CChannelCfg)), 4, None) == -2
    s = e.follow_open(0, b_lo, ch, queue_batches=4)
    far = e.follow_open(0, b_lo + 1000, ch)  # beyond the live edge: waits
    assert e.follow_run(-1) >= 1 and e.follow_info(far)["next_batch"] == b_lo + 1000
    assert code(e.follow_stats, s, 3)[0] == -5 and code(e.follow_stats, s, -1)[0] == -5
    assert e.L.abg_follow_stats(e.h, s, 0, None) == -2
    wo = np.zeros((1, 3, B), np.float32)
    assert e.L.abg_follow_fetch(e.h, s, 1, None, None, lib._ptr(np.zeros(3, np.uint8)), None) == -2
    assert e.L.abg_follow_fetch(e.h, s, 1, lib._ptr(wo), None, None, None) == -2
    assert e.L.abg_follow_fetch(e.h, s, -1, lib._ptr(wo), None, lib._ptr(np.zeros(3, np.uint8)), None) == -2
    assert e.L.abg_follow_info(e.h, s, None) == -2
    assert e.L.abg_debug_follow_time(e.h, None) == -2
    # a change of the history under a session is refused and changes nothing
    rng = e.history_range(0)
    rc, msg = code(e.history_configure, 0, 8)
    assert rc == -2 and "follow" in msg
    assert e.history_range(0) == rng and e.follow_info(s)["queued"] >= 1
    e.history_configure(0, 4)  # no change: fine
    # closed and unknown ids
    e.follow_close(s)
    for f, a in ((e.follow_close, (s,)), (e.follow_fetch, (s,)), (e.follow_info, (s,)), (e.follow_stats, (s, 0)),
                 (e.follow_close, (12345,))):
        assert code(f, *a)[0] == -5
    # ids are not reused
    s2 = e.follow_open(0, b_lo, ch)
    assert s2 not in (s, far)
    e.follow_close(s2)
    e.follow_close(far)
    e.history_configure(0, 0)
    assert code(e.follow_open, 0, 1, ch)[0] == -5
    e.close()


# ---- 8. end to end ------------------------------------------------------------------------------------------------------------
def test_detect_and_follow_a_transmitter_that_keys_up_mid_stream():
    SR, n = 2048000, 2048
    bw = SR // n
    chan_off = [-600, -300, 300, 600]
    chans = [cm.make_channel(CF + k * bw + bw // 2, CF, SR, n, W) for k in chan_off]
    cfg = parent_cfg(cm.SFMT_U8, SR, n, channels=chans)
    B, hop, nb = cfg.wave_batch, cfg.hop(0), 20
    n_samples = (AGC + nb * B) * hop + n + hop
    k_tx, fm = 177, 700.0
    a, b = AGC + 6 * B + 400, AGC + 15 * B + 300  # keys up in batch 6, stops in batch 15
    raw = tx_raw(cfg, n_samples, [(k * bw + bw / 2, 0.04, 0, n_samples, "am", 0.0) for k in chan_off] +
                 [(k_tx * bw, 0.04, a * hop, b * hop, "am", fm)], 0.01, seed=2)
    s = lib.default_stride(cfg, 0)
    state = dict(readings=[], sid=None, opened_at=None)
    sink = Sink()

    def setup(e):
        e.spectrum_configure(0, s)

    def after(e, k):
        if "thr" not in state:  # thresholds from the first batch's spectrum
            sp = e.fetch_spectrum(0)
            if sp is None:
                return
            state["thr"] = lib.activity_threshold(sp[0], 13.0, 16)
            e.spectrum_configure(0, 0)
            e.activity_configure(0, s, 1, 2, state["thr"])
            return
        while (r := e.fetch_activity(0)) is not None:
            state["readings"].append(r)
        if state["sid"] is None and state["readings"]:
            tx = [t for t in lib.group_transmissions(lib.merge_bursts(state["readings"]), cfg, 0)
                  if abs(t["freq_hz"] - (CF + k_tx * bw)) <= bw and not t["monitored"]]
            if tx:
                job = lib.transmission_follow(tx[0], cfg, 0, e.history_range(0))
                state["sid"] = e.follow_open(**job)
                state["job"] = job
                state["opened_at"] = live_batches(e, cfg)
        if state["sid"] is not None:
            e.follow_run(-1)
            sink.fetch(e, state["sid"])

    e = stream(cfg, [raw], nbmax=2, hist=nb + 2, setup=setup, after=after)
    finish(e, sink, [state["sid"]])
    assert state["sid"] is not None and state["opened_at"] <= 9  # found while still transmitting
    r = sink.result(state["sid"])
    f0 = AGC + r["first_batch"] * B
    lo, hi = f0 + B * np.arange(len(r["axc"])), f0 + B * (np.arange(len(r["axc"])) + 1)
    on = r["axc"][:, 0] == ord("*")
    inside = (lo >= a) & (hi <= b)
    after_edge = (np.arange(len(r["axc"])) + r["first_batch"]) >= state["opened_at"]
    assert (inside & after_edge).sum() >= 4  # heard across the live edge
    assert on[inside].all(), on
    assert not on[hi < a - B // 2].any() and not on[lo > b + B].any(), on  # not before it, nor after it stopped
    audio = r["waveout"][inside, 0, :].reshape(-1).astype(np.float64)
    spec = np.abs(np.fft.rfft((audio - audio.mean()) * np.hanning(audio.size)))
    assert abs(np.argmax(spec) * W / audio.size - fm) <= 10.0
    same_as_replay(e, r, state["job"])
    e.close()
