"""Live follow on the CPU: the C ABI and its ctypes mirror (abg_follow_status included), transmission_follow's start rule,
and a numpy model of which batches one abg_follow_run may advance a session by, given the history's range, the session's
queue and the next sample it has not read, checked against the definition in airband_b200.h.  The GPU tests use the
same model to predict every session's next_batch and lost flag."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from airband_b200 import config as cm
from airband_b200 import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AGC = cm.AGC_EXTRA
FOLLOW = ("abg_follow_open", "abg_follow_close", "abg_follow_run", "abg_follow_fetch", "abg_follow_info", "abg_follow_stats",
          "abg_debug_follow_time")


# ---- the model ------------------------------------------------------------------------------------------------------------------
def batch_reads(b, B, hop, N):
    """Samples [lo, hi) the replay of batch b reads: from its first frame to the end of its last one."""
    return (AGC + b * B) * hop, (AGC + (b + 1) * B) * hop + N - hop


def available_end(history_range, B, hop, N):
    """Batches b < available_end(...) have every sample up to their last frame's end in the history (its first sample
    is checked by the loss rule)."""
    first, end = history_range
    if end <= first:
        return 0
    fl = (end + hop - N) // hop if end + hop >= N else 0
    return (fl - AGC) // B if fl >= AGC else 0


def follow_step(history_range, B, hop, N, first_batch, next_batch, next_unread, queued, queue_batches, chunk, budget):
    """One chunk of abg_follow_run for one session: (batches it advances, lost).  next_unread = the session's first sample
    not yet gathered; queued = its unfetched batches; chunk = max_batches_per_run (1 with AFC)."""
    first, end = history_range
    if end <= first:
        return 0, False
    if first > next_unread:
        return 0, True
    n = min(max(available_end(history_range, B, hop, N) - next_batch, 0), queue_batches - queued, chunk, budget)
    return max(n, 0), False


def next_unread(first_batch, next_batch, history_range, B, hop, N):
    """The session's first sample not yet gathered after it enqueued batches [first_batch, next_batch): the fill rule's
    bytes for them, clipped to the history's end (the rest is gathered again later)."""
    S = first_batch * B * hop
    if next_batch == first_batch:
        return S
    return min(S + (AGC + (next_batch - first_batch) * B) * hop + N, history_range[1])


# ---- ABI ----------------------------------------------------------------------------------------------------------------------
def test_header_symbols_and_argtypes():
    hdr = open(os.path.join(ROOT, "include", "airband_b200.h")).read()
    for s in FOLLOW:
        assert s in lib.SYMBOLS and re.search(r"ABG_API int %s\(" % s, hdr), s
    L = lib.load()
    for s in FOLLOW:
        assert hasattr(L, s), s
    vp, i = C.c_void_p, C.c_int
    assert L.abg_follow_open.argtypes == [vp, i, C.c_uint64, i, C.POINTER(cm.CChannelCfg), i, C.POINTER(C.c_int32)]
    assert L.abg_follow_close.argtypes == [vp, C.c_int32]
    assert L.abg_follow_run.argtypes == [vp, i]
    assert L.abg_follow_fetch.argtypes == [vp, C.c_int32, i, vp, vp, vp, C.POINTER(C.c_uint64)]
    assert L.abg_follow_info.argtypes == [vp, C.c_int32, C.POINTER(lib.CFollowStatus)]
    assert L.abg_follow_stats.argtypes == [vp, C.c_int32, i, C.POINTER(cm.CSquelchStats)]
    assert L.abg_debug_follow_time.argtypes == [vp, C.POINTER(C.c_float)]
    # the availability condition is stated where the definition is
    assert "WAVE_BATCH*hop >= fft_size - hop" in hdr


def test_follow_status_layout_matches_the_header(tmp_path):
    fields = [f for f, _ in lib.CFollowStatus._fields_]
    prog = "#include <stdio.h>\n#include <stddef.h>\n#include \"airband_b200.h\"\nint main(void) {\n"
    prog += "".join(f'    printf("%zu\\n", offsetof(abg_follow_status, {f}));\n' for f in fields)
    prog += '    printf("%zu\\n", sizeof(abg_follow_status));\n    return 0;\n}\n'
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text(prog)
    subprocess.run(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [getattr(lib.CFollowStatus, f).offset for f in fields] + [C.sizeof(lib.CFollowStatus)]
    assert got == [0, 4, 8, 16, 20, 24]


# ---- transmission_follow --------------------------------------------------------------------------------------------------------
def _cfg():
    ch = cm.make_channel(120_100_000, 120_000_000, 2048000, 2048, 8000)
    return cm.Config(fft_size=2048, wave_rate=8000, devices=[cm.Device(sample_rate=2048000, sfmt=cm.SFMT_U8, centerfreq=120_000_000,
                                                                       channels=[ch])])


def test_transmission_follow_starts_where_transmission_replay_does_and_has_no_end():
    cfg = _cfg()
    B, hop = cfg.wave_batch, cfg.hop(0)
    tx = dict(freq_hz=120_033_000.0, first_frame=AGC + 20 * B + 300, last_frame=AGC + 23 * B + 10)
    for hist, lead in (((0, 10 ** 12), 0.5), ((0, 10 ** 12), None), ((0, 10 ** 12), 0.0), ((18 * B * hop - 1, 10 ** 12), 0.5)):
        job = lib.transmission_follow(tx, cfg, 0, hist, lead_s=lead)
        rep = lib.transmission_replay(tx, cfg, 0, hist, lead_s=lead)
        assert set(job) == {"dev", "first_batch", "channels"}
        assert job["first_batch"] == rep["first_batch"] and job["dev"] == 0
        assert [bytes(cm.channels_to_c(job["channels"]))] == [bytes(cm.channels_to_c(rep["channels"]))]
    assert lib.transmission_follow(tx, cfg, 0, (0, 10 ** 12))["first_batch"] == 20 - lib.REPLAY_SETTLE_BATCHES
    assert lib.transmission_follow(tx, cfg, 0, (0, 10 ** 12), lead_s=0.5)["first_batch"] == 16
    # clipped to the history's start
    assert lib.transmission_follow(tx, cfg, 0, (18 * B * hop - 1, 10 ** 12), lead_s=0.5)["first_batch"] == 18
    # no end: a history that ends before the transmission (reported ahead of it) still gives a session, which waits
    early = lib.transmission_follow(tx, cfg, 0, (0, (AGC + 10 * B) * hop), lead_s=0.0)
    assert early["first_batch"] == 20
    with pytest.raises(ValueError):
        lib.transmission_follow(tx, cfg, 0, (0, 10 ** 12), lead_s=-1.0)
    nfm = lib.transmission_follow(tx, cfg, 0, (0, 10 ** 12), modulation=cm.MOD_NFM)["channels"][0]
    assert nfm.modulation == cm.MOD_NFM and nfm.dm_dphi == cm.calc_dm_dphi(120_033_000, 120_000_000, 2048000, 8000)


# ---- availability, queue and loss ----------------------------------------------------------------------------------------------
def test_available_end_is_the_definition():
    rng = np.random.default_rng(3)
    for _ in range(2000):
        B = int(rng.choice([100, 125, 1000, 1001, 2000]))
        hop = int(rng.integers(1, 400))
        N = int(rng.choice([256, 512, 2048, 8192]))
        first = int(rng.integers(0, 50 * B * hop))
        end = first + int(rng.integers(0, 20 * B * hop))
        be = available_end((first, end), B, hop, N)
        # brute force over batches: every b < be fits, be does not
        if end > first:
            assert be == 0 or batch_reads(be - 1, B, hop, N)[1] <= end
            assert batch_reads(be, B, hop, N)[1] > end
        else:
            assert be == 0


def test_lag_is_one_batch_exactly_where_the_header_says():
    """History batch L ends at (AGC + (L+1)B) hop.  Batch L - 1 is then available iff B*hop >= fft_size - hop, and batch L
    iff fft_size <= hop.  abg_create accepts configurations on both sides."""
    seen = {True: 0, False: 0}
    for wave_rate in (800, 8000, 8008, 16000):
        B = wave_rate // 8
        for N in (256, 512, 1024, 2048, 4096, 8192):
            for sr in (wave_rate + 8, 4 * wave_rate, 8 * wave_rate + 1, 2048000, 2500000, 2560000, 10_000_000):
                if sr <= wave_rate:
                    continue
                hop = int(round(sr / wave_rate))
                for L in (0, 5, 37):
                    end = (AGC + (L + 1) * B) * hop
                    be = available_end((0, end), B, hop, N)
                    cond = B * hop >= N - hop
                    seen[cond] += 1
                    if N <= hop:
                        assert be == L + 1
                    elif cond:
                        assert be == L  # next_batch == L: one batch behind
                    else:
                        assert be == max(L + 1 - -(-(N - hop) // (B * hop)), 0)
    assert seen[True] and seen[False]


def test_one_follow_run_advances_into_history_queue_room_and_budget_and_detects_loss():
    B, hop, N = 1000, 256, 2048
    fb = 10
    # history holds batches 8..15 (capacity 8): batches 10..14 are available
    hr = ((AGC + 8 * B) * hop, (AGC + 16 * B) * hop)
    assert available_end(hr, B, hop, N) == 15
    u = next_unread(fb, fb, hr, B, hop, N)
    assert follow_step(hr, B, hop, N, fb, fb, u, 0, 16, 4, 10 ** 9) == (4, False)  # one chunk of max_batches_per_run
    assert follow_step(hr, B, hop, N, fb, fb, u, 0, 16, 1, 10 ** 9) == (1, False)  # AFC: one batch
    assert follow_step(hr, B, hop, N, fb, fb, u, 0, 3, 4, 10 ** 9) == (3, False)   # queue room
    assert follow_step(hr, B, hop, N, fb, fb, u, 3, 3, 4, 10 ** 9) == (0, False)   # full queue: stops
    assert follow_step(hr, B, hop, N, fb, fb, u, 0, 16, 4, 2) == (2, False)        # max_batches
    # a whole call: chunks until nothing is left
    nb, q = fb, 0
    while True:
        n, lost = follow_step(hr, B, hop, N, fb, nb, next_unread(fb, nb, hr, B, hop, N), q, 16, 4, 10 ** 9)
        if n == 0:
            break
        nb, q = nb + n, q + n
    assert nb == 15 and q == 5 and not lost  # next_batch = the live engine's last batch
    # the gather took the fill rule's bytes for batches 10..14, fft_size past batch 15's first frame
    assert next_unread(fb, nb, hr, B, hop, N) == (AGC + 15 * B) * hop + N < hr[1]
    # with the fill rule reaching past the history's end only what it holds counts as read: the rest comes again later
    assert next_unread(fb, nb, (hr[0], (AGC + 15 * B) * hop + N - hop), B, hop, N) == (AGC + 15 * B) * hop + N - hop
    # the history (8 batches) moves on by 8 batches while the session is full: its next unread sample is overwritten -> lost
    hr2 = ((AGC + 16 * B) * hop, (AGC + 24 * B) * hop)
    assert follow_step(hr2, B, hop, N, fb, nb, next_unread(fb, nb, hr, B, hop, N), q, 16, 4, 10 ** 9) == (0, True)
    # but not while the sample is still held
    hr3 = ((AGC + 15 * B) * hop, (AGC + 23 * B) * hop)
    assert follow_step(hr3, B, hop, N, fb, nb, next_unread(fb, nb, hr, B, hop, N), q, 16, 4, 10 ** 9)[1] is False
    # a session opened at the live edge waits, then starts there
    edge = 16
    assert follow_step(hr, B, hop, N, edge, edge, next_unread(edge, edge, hr, B, hop, N), 0, 16, 4, 10 ** 9) == (0, False)
    hr4 = (hr[0] + B * hop, hr[1] + 2 * B * hop)  # two more live batches
    assert follow_step(hr4, B, hop, N, edge, edge, next_unread(edge, edge, hr4, B, hop, N), 0, 16, 4, 10 ** 9) == (1, False)
