"""I/Q history on the CPU: the kernels (rtlsdr-airband_b200/csrc/history.cu) as the compiler built them, the sub-band
kernel they share their arithmetic with, the ABI, a numpy model of the ring and its range bookkeeping, and
lib.transmission_capture's window arithmetic."""
import os
import re

import numpy as np
import pytest

from airband_b200 import config as cm
from airband_b200 import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "rtlsdr-airband_b200", "build")
AGC = cm.AGC_EXTRA
BPC = {cm.SFMT_U8: 2, cm.SFMT_S8: 2, cm.SFMT_S16: 4, cm.SFMT_F32: 8}


class RingModel:
    """The history of one device as airband_b200.h defines it: a ring of R bytes (R = capacity * bpc rounded up to 16),
    sample s at byte (s * bpc) mod R, holding one contiguous range [first, end) of at most `capacity` samples."""

    def __init__(self, bpc, hop, wave_batch):
        self.bpc, self.hop, self.B = bpc, hop, wave_batch
        self.n = wave_batch * hop  # samples per batch
        self.batches = 0
        self.cap = self.R = 0
        self.ring = None
        self.first = self.end = 0

    def configure(self, n_batches):
        if n_batches == self.batches:
            return
        self.batches = n_batches
        self.cap = n_batches * self.n
        self.R = (self.cap * self.bpc + 15) // 16 * 16
        self.ring = np.zeros(self.R, np.uint8) if n_batches else None
        self.first = self.end = 0

    def append(self, seq, n_batches, stream):
        """Batches seq .. seq + n_batches - 1 of a streamed run; stream = the device's bytes from sample 0."""
        if not self.batches or n_batches == 0:
            return
        s0 = (AGC + seq * self.B) * self.hop
        b0, nb = s0 * self.bpc, n_batches * self.n * self.bpc
        skip = max(nb - self.R, 0)
        pos = (b0 + skip + np.arange(nb - skip)) % self.R
        self.ring[pos] = stream[b0 + skip:b0 + nb]
        if self.first == self.end or s0 != self.end:
            self.first = s0
        self.end = s0 + n_batches * self.n
        self.first = max(self.first, self.end - self.cap)

    def resident(self):
        if self.batches:
            self.first = self.end = 0

    def raw(self, first, n):
        assert self.first < self.end and self.first <= first and first + n <= self.end
        return self.ring[(first * self.bpc + np.arange(n * self.bpc)) % self.R]


def ring_model(sfmt, hop, wave_batch):
    return RingModel(BPC[sfmt], hop, wave_batch)


# ---- the build ------------------------------------------------------------------------------------------------------------
def _log(name):
    path = os.path.join(BUILD, name)
    assert os.path.exists(path), f"{path} missing: build the library first (make -C rtlsdr-airband_b200)"
    with open(path) as f:
        return f.read()


def test_history_kernels_build_for_sm90a_without_spills():
    log = _log("history.ptxas.log")
    assert "sm_90a" in log and "abg_history_append_kernel" in log and "abg_history_capture_kernel" in log
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(spills) == 2 and all(int(a) == 0 and int(b) == 0 for a, b in spills), spills
    stack = re.findall(r"(\d+) bytes stack frame", log)
    assert stack and all(int(x) == 0 for x in stack), stack


def test_subband_kernel_keeps_its_registers():
    log = _log("subband.ptxas.log")
    assert re.findall(r"Used (\d+) registers", log) == ["92"]
    assert re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log) == [("0", "0")]


def test_header_symbols_match_lib():
    hdr = open(os.path.join(ROOT, "include", "airband_b200.h")).read()
    for s in ("abg_history_configure", "abg_history_range", "abg_history_raw", "abg_history_subband", "abg_debug_history_time"):
        assert s in lib.SYMBOLS and re.search(r"ABG_API int %s\(" % s, hdr), s
    assert int(re.search(r"#define ABG_SUBBAND_MAX_COEFFS (\d+)", hdr).group(1)) == lib.SUBBAND_MAX_COEFFS


# ---- the ring model -----------------------------------------------------------------------------------------------------------
def test_ring_positions_keep_stream_offsets_modulo_16():
    # 2.5 Msps at 8000 frames/s: hop 313, a batch of 1000 frames is 313000 samples; batch starts are not 16-byte aligned
    hop, B = 313, 1000
    assert (AGC * hop * 2) % 16 == 8
    for sfmt, bpc in BPC.items():
        for n_batches in (1, 3, 8):
            m = ring_model(sfmt, hop, B)
            m.configure(n_batches)
            assert m.R % 16 == 0 and m.R >= m.cap * bpc and m.R - m.cap * bpc < 16
            s = np.arange(0, 10 * B * hop, 997, dtype=np.int64)
            assert np.array_equal((s * bpc) % m.R % 16, (s * bpc) % 16)
            # a 16-byte vector of the stream never straddles the wrap
            v = s[(s * bpc) % 16 == 0] * bpc % m.R
            assert np.all(v + 16 <= m.R)


def test_ring_model_range_eviction_and_reconfiguration():
    hop, B = 16, 10
    n = B * hop
    stream = (np.arange(2 * (AGC + 40 * B) * hop + 64) % 251).astype(np.uint8)
    m = ring_model(cm.SFMT_U8, hop, B)
    m.append(0, 2, stream)  # off: nothing
    assert (m.first, m.end) == (0, 0)
    m.configure(3)
    assert (m.first, m.end) == (0, 0)
    m.append(2, 2, stream)  # starts at the first batch after it was switched on
    s0 = (AGC + 2 * B) * hop
    assert (m.first, m.end) == (s0, s0 + 2 * n)
    m.append(4, 4, stream)  # a run longer than the capacity keeps its last 3 batches
    assert (m.first, m.end) == (s0 + 3 * n, s0 + 6 * n)
    for seq in range(8, 20):  # evictions wrap the ring many times
        m.append(seq, 1, stream)
        assert m.end - m.first == 3 * n
        assert np.array_equal(m.raw(m.first, 3 * n), stream[2 * m.first:2 * m.end])
    e0 = (m.first, m.end)
    m.configure(3)  # the same capacity changes nothing
    assert (m.first, m.end) == e0
    m.configure(5)  # another capacity empties it
    assert (m.first, m.end) == (0, 0)
    m.append(20, 1, stream)
    assert (m.first, m.end) == ((AGC + 20 * B) * hop, (AGC + 21 * B) * hop)
    m.resident()  # resident runs leave it empty
    assert (m.first, m.end) == (0, 0)
    m.configure(0)
    assert m.ring is None and (m.first, m.end) == (0, 0)


# ---- transmission_capture ------------------------------------------------------------------------------------------------------
def _cfg():
    ch = cm.make_channel(120_100_000, 120_000_000, 2048000, 2048, 8000)
    return cm.Config(fft_size=2048, wave_rate=8000, devices=[cm.Device(sample_rate=2048000, sfmt=cm.SFMT_U8, centerfreq=120_000_000,
                                                                       channels=[ch])])


def test_transmission_capture_window_and_clipping():
    cfg = _cfg()
    hop = cfg.hop(0)
    assert hop == 256
    tx = dict(freq_hz=120_033_000.0, first_frame=3000, last_frame=3500)
    D, L = 32, 255
    big = (0, 10 ** 9)
    off, m0, n = lib.transmission_capture(tx, cfg, 0, big, D, L)
    assert off == 33000.0
    lo, hi = 3000 * hop, 3500 * hop + 2048
    assert m0 == -(-lo // D) and (m0 + n - 1) * D < hi <= (m0 + n) * D
    # padding widens both sides by pad_s * sample_rate samples
    off, m1, n1 = lib.transmission_capture(tx, cfg, 0, big, D, L, pad_s=0.05)
    pad = round(0.05 * 2048000)
    assert m1 == -(-(lo - pad) // D) and (m1 + n1 - 1) * D < hi + pad <= (m1 + n1) * D
    # clipped at the history's start: the first output's oldest tap is the history's first sample or later
    first = lo - pad + 1000
    _, m2, n2 = lib.transmission_capture(tx, cfg, 0, (first, 10 ** 9), D, L, pad_s=0.05)
    assert m2 * D - (L - 1) >= first and (m2 - 1) * D - (L - 1) < first and m2 + n2 == m1 + n1
    # clipped at its end: the last output's newest sample lies before end
    end = hi - 5000
    _, m3, n3 = lib.transmission_capture(tx, cfg, 0, (0, end), D, L, pad_s=0.05)
    assert m3 == m1 and (m3 + n3 - 1) * D < end <= (m3 + n3) * D
    # the padded window may start before sample 0
    _, m4, _ = lib.transmission_capture(dict(tx, first_frame=10), cfg, 0, (0, 10 ** 9), D, 1, pad_s=0.05)
    assert m4 == 0


def test_transmission_capture_raises_when_nothing_is_left():
    cfg = _cfg()
    tx = dict(freq_hz=120_000_000.0, first_frame=3000, last_frame=3500)
    hi = 3500 * 256 + 2048
    with pytest.raises(ValueError, match="nothing"):
        lib.transmission_capture(tx, cfg, 0, (hi + 10, hi + 10 ** 6), 32, 255)  # history starts after the window
    with pytest.raises(ValueError, match="nothing"):
        lib.transmission_capture(tx, cfg, 0, (0, 3000 * 256), 32, 1)  # history ends before it
    with pytest.raises(ValueError, match="nothing"):
        lib.transmission_capture(tx, cfg, 0, (0, 0), 32, 1)  # empty history
    with pytest.raises(ValueError):
        lib.transmission_capture(tx, cfg, 0, (0, 10 ** 9), 0, 255)
