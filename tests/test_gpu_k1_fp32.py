"""GPU tests of the two FP32 K1 kernels frame by frame against float64: the output-pruned kernel (fft_mode 2,
rtlsdr-airband_b200/csrc/k1_pruned.cu) over every class of its plan space (test_pruned_dft_math.PRUNED_CASES), and the
full-spectrum kernel (fft_mode 1, k1_fft.cu) over every size and format, AFC spectra included (Engine.k1_spectra).

What K1 stored (Engine.k1_outputs: win = |X[bin]|, iqin = X[bin], every frame, before any squelch decision) is compared for
every row of every device with the float64 DFT of the reference's float32 frame (test_tc_dft_math.reference_frame), per frame:

    |X_gpu - X_f64| <= K * 2^-24 * sum_n |x_n w_n|

where x_n w_n is the reference's windowed float32 frame and K counts the roundings on the longest path from a sample to an
output (pruned_k, full_k below).  Each rounding of a partial value v adds at most 2^-24 |v| per component, and |v| is at most
the l1 sum of the samples feeding it, so a path with k roundings contributes at most k 2^-24 sum|x w| per component; the
final factor 2 turns the two components' bounds into one on the complex modulus (sqrt 2) and covers the twiddle factors'
|re| + |im| <= sqrt 2.  The rms of the per-frame ratio is held to 1/8 of that bound per device.  On top: win is the correctly
rounded float32 magnitude of iqin, bit for bit; rows past a device's last frame stay unwritten; and a device's rows are
bitwise the same wherever its frames sit (tile, run grouping, push pattern, group position, neighbouring groups, channel
position within R1)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from airband_b200 import config as cm
from airband_b200 import lib
from test_gpu_tc_geometry import AGC, Group, assert_win_is_magnitude, make_stream
from test_pruned_dft_math import PRUNED_CASES, pruned_constants, pruned_plan, reduction_class
from test_tc_dft_math import reference_frame

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
RMS_FRACTION = 1 / 8
CHUNK = 256  # frames per float64 chunk
U8, S8, S16, F32 = cm.SFMT_U8, cm.SFMT_S8, cm.SFMT_S16, cm.SFMT_F32
SIZES = (256, 512, 1024, 2048, 4096, 8192)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the worst observed ratios to each bound, printed at the end of each test (run with -s to see them)
RATIOS = {}


def log2(x):
    return int(x).bit_length() - 1


def pruned_k(n, max_channels, gelem):
    """Roundings on the longest path through k1_pruned_kernel (times 2, see the module docstring):
       4  sample conversion: the kernel multiplies by fl(fl(window) * fl(1/fullscale)), the reference rounds its level
          (or scale * x) and then the product with the window: four roundings apart, plus the kernel's product, less one
          that both share (window itself);  (U8: x - 127.5 is exact, S8/S16: the integer is exact)
       1  the window fold into the first radix-2 stage: fma(xb, wb, xa * wa) (xa * wa counted above)
       3 (log2 R1 - 1)  the remaining radix-2 stages: compile-time twiddle, two fmas per component
       2  the float tables W_N^m behind the warp-uniform factor s_U and the per-lane factor s_base
       2 NCOL  the column terms a lane adds in sequence: two fmas per column and component, over every group
       NGRP - 1  the group partials added through shared memory
       2  the per-lane factor: a product and an fma
       NVP - 1 + log2(32 / NVP) <= 31  the lane reduction: a lane adds NVP partials in sequence, then the shuffle tree."""
    p = pruned_plan(n, max_channels, gelem)
    k = 4 + 1 + 3 * (log2(p["R1"]) - 1) + 2 + 2 * p["NCOL"] + (p["NGRP"] - 1) + 2 + 31
    return 2 * k


# k1_fft.cuh Plan<LOGN>: (R1, R2, R3, T, BLOCK)
FFT_PLAN = {256: (16, 16, 0, 16, 128), 512: (32, 16, 0, 16, 128), 1024: (32, 32, 0, 32, 128), 2048: (64, 32, 0, 32, 128),
            4096: (64, 64, 0, 64, 128), 8192: (32, 16, 16, 256, 256)}


def full_k(n):
    """Roundings on the longest path through fft_frame (times 2): the conversion (4, as above) and the window product (1),
    3 per radix-2 stage of every pass (log2 N stages in all), and 3 per inter-pass twiddle (table entry, product, fma)."""
    passes = 3 if FFT_PLAN[n][2] else 2
    return 2 * (4 + 1 + 3 * log2(n) + 3 * (passes - 1))


def fft_tile_frames(n, bpc, hop_bytes):
    """abg_k1_tile_frames and the frame slots S of the full-spectrum kernel (k1_fft.cu), mirrored to know which tiles end in a
    partial iteration."""
    r1, r2, r3, t, block = FFT_PLAN[n]
    rl = r3 or r2
    s = block // t
    fixed = 16 + 8 * (n // rl) + 8 * s * (n + n // rl)
    frame = n * bpc
    budget = 112 * 1024 - fixed if 112 * 1024 > fixed + frame + 64 else frame + 64
    budget = min(budget, 220 * 1024 - fixed)
    tf = 1 + (budget - frame - 64) // hop_bytes if budget > frame + 64 else 1
    return max(1, min(tf, 64)), s


def bin_lists(n, counts, r1, seed):
    """Channel lists: devices cycle through (a) bins 0, 1, N/2, N-1, a duplicate of 0, a bin on N/2's row, then distinct
    others; (b) every channel on one row (bins = 5 mod 16); (c) seeded random bins.  Lists with more than 32 channels repeat
    channel 5's bin at 37, and devices with a tone get the F32 stream's weak tone (tone + N/4) as channel 1."""
    rng = np.random.default_rng(seed)
    out = []
    for d, c in enumerate(counts):
        if d % 3 == 0:
            b = [0, 1, n // 2, n - 1, 0, n // 2 + r1] + [(n // 3 + 37 * i) % n for i in range(max(0, c - 6))]
        elif d % 3 == 1:
            b = [(5 + 16 * (3 * i + 1)) % n for i in range(c)]
        else:
            b = [int(x) for x in rng.integers(0, n, c)]
        b = b[:c]
        if d % 3 and c >= 2:
            b[1] = (b[0] + n // 4) % n
        if c > 37:
            b[37] = b[5]
        out.append(b)
    return out


def case_group(n, hop, sfmt, fullscale, counts, wave_rate=8000, seed=0, afc=()):
    bpc = 2 * cm.BYTES_PER_SAMPLE[sfmt]
    counts = list(counts) * 2  # every list twice: a device with many channels between shorter ones, batches 2, 1, 3, 1, 2, 3
    r1 = pruned_plan(n, max(counts), 64)["R1"]
    return Group(n, hop * bpc, sfmt, bin_lists(n, counts, r1, seed + n), [2, 1, 3, 1, 2, 3][:len(counts)], wave_rate,
                 seed0=seed + n + hop + sfmt, fullscale=fullscale, rails=True, afc=afc)


def run_engine(g, fft_mode, nbmax=4, runs=1, path=None, between=None, **kw):
    """Push every stream whole, run `runs` times, return [(win, iqin)] of each run.  Every device must take K1 path `path`."""
    e = lib.Engine(g.cfg, max_batches_per_run=nbmax, input_capacity_batches=max(g.batches) + 2, fft_mode=fft_mode, **kw)
    try:
        for d, r in enumerate(g.raws):
            assert e.fft_path(d) == (path or fft_mode), f"device {d} takes K1 path {e.fft_path(d)}"
            e.push(d, r)
        outs = []
        for k in range(runs):
            if between:
                between(e, k)
            e.run(-1)
            outs.append(e.k1_outputs())
        return outs
    finally:
        e.close()


def check_device(g, d, win, iq, first_frame, rows, K, bins=None):
    """Rows [0, rows) of device d (stream frames first_frame + row) against float64; returns (worst ratio, rms ratio)."""
    cols = slice(g.g0[d], g.g0[d + 1])
    b = np.asarray(g.bin_lists[d] if bins is None else bins, np.int64)
    tw = np.exp(-2j * np.pi * ((np.arange(g.n, dtype=np.int64)[:, None] * b[None, :]) % g.n) / g.n)
    worst, sq, cnt = 0.0, 0.0, 0
    for r0 in range(0, rows, CHUNK):
        r = np.arange(r0, min(rows, r0 + CHUNK))
        fin = reference_frame(g.frame_bytes(d, first_frame + r), g.sfmt, g.n, g.fullscale)
        ratio = np.abs(iq[r, cols].astype(np.complex128) - fin @ tw) / (K * U * np.abs(fin).sum(1))[:, None]
        worst, sq, cnt = max(worst, float(ratio.max())), sq + float((ratio ** 2).sum()), cnt + ratio.size
        assert worst <= 1.0, f"device {d} (bins {list(b)}): X off float64 by {worst:.3g} of the bound, rows {r0}.., " \
                             f"first bad (row, channel) {np.unravel_index(np.argmax(ratio), ratio.shape)}"
        assert_win_is_magnitude(win[r, cols], iq[r, cols])
    rms = (sq / cnt) ** 0.5
    assert rms <= RMS_FRACTION, f"device {d}: rms ratio {rms:.3g} to the bound"
    return worst, rms


def check_group_run(g, win, iq, K, first_batch=0, nb=None, key=None):
    """Every device's rows of one run against float64, the rows past its batches unwritten (first run: zeros)."""
    worst = rms = 0.0
    for d in range(len(g.bin_lists)):
        n_b = min(g.batches[d] - first_batch, win.shape[0] // g.B) if nb is None else nb[d]
        if n_b <= 0:
            continue
        w, r = check_device(g, d, win, iq, AGC + first_batch * g.B, n_b * g.B, K)
        worst, rms = max(worst, w), max(rms, r)
        if first_batch == 0:
            cols = slice(g.g0[d], g.g0[d + 1])
            assert not win[n_b * g.B:, cols].any() and not iq[n_b * g.B:, cols].any(), f"device {d}: stores past its last frame"
    if key:
        RATIOS[key] = (worst, rms)
        print(f"\nRATIO {key}: worst {worst:.4g} rms {rms:.4g} of K = {K}")
    return worst


def assert_duplicates_equal(g, iq, maxch, pruned):
    """Channels of a device on the same bin hold the same bits: always in the full-spectrum kernel (the same registers), and in
    the pruned kernel whenever the lane reduction has the same width in the two channels' passes."""
    for d, bins in enumerate(g.bin_lists):
        rows = min(g.batches[d], iq.shape[0] // g.B) * g.B
        nvp = [reduction_class(min(maxch, len(bins) - (c // maxch) * maxch))[0] for c in range(len(bins))]
        for c1, b in enumerate(bins):
            for c2 in range(c1 + 1, len(bins)):
                if bins[c2] == b and (not pruned or nvp[c1] == nvp[c2]):
                    a1, a2 = iq[:rows, g.g0[d] + c1], iq[:rows, g.g0[d] + c2]
                    assert np.array_equal(a1.view(np.uint64), a2.view(np.uint64)), (d, c1, c2, b)


# ---- the output-pruned kernel over its plan space ------------------------------------------------------------------------
def _pruned_case(name):
    n, hop, sfmt, fs, counts, ge, _ = PRUNED_CASES[name]
    g = case_group(n, hop, sfmt, fs, counts)
    (win, iq), = run_engine(g, 2)
    check_group_run(g, win, iq, pruned_k(n, max(counts), ge), key=f"pruned {name}")
    assert_duplicates_equal(g, iq, pruned_constants()["maxch"], True)
    # every device of the group has its own channel count: the R1 and CM of the launch are the group's
    assert len({len(b) for b in g.bin_lists}) == len(set(counts))


@pytest.mark.parametrize("name", [k for k, v in PRUNED_CASES.items() if v[5] == 64])
def test_pruned_plan_class_against_float64(name):
    _pruned_case(name)


def _gelem32_child():
    for name in [k for k, v in PRUNED_CASES.items() if v[5] == 32]:
        _pruned_case(name)
    print("GELEM32 OK " + " ".join(f"{k}={v[0]:.4g}/{v[1]:.4g}" for k, v in RATIOS.items()))


def test_pruned_gelem32_against_float64():
    """ABG_K1_GELEM is read once per process, so the GELEM = 32 cases run in a child process."""
    env = dict(os.environ, ABG_K1_GELEM="32")
    code = "import sys; sys.path[:0] = %r; import test_gpu_k1_fp32 as t; t._gelem32_child()" % ([os.path.dirname(os.path.abspath(__file__))] + sys.path,)
    p = subprocess.Popen([sys.executable, "-c", code], env=env, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        out, _ = p.communicate(timeout=600)
    finally:
        if p.poll() is None:
            p.kill()
            p.communicate()
    assert p.returncode == 0, out[-4000:]
    print("\n" + [x for x in out.splitlines() if x.startswith("GELEM32 OK")][-1])


# ---- the full-spectrum kernel ----------------------------------------------------------------------------------------------
FULL_CASES = [(n, sfmt) for n in SIZES for sfmt in (U8, S8, S16, F32)]
FULL_FULLSCALE = {U8: 0.0, S8: 0.0, S16: 3000.0, F32: 2048.0}


@pytest.mark.parametrize("n,sfmt", FULL_CASES, ids=[f"{n}-{['', 'u8', 's8', 's16', 'f32'][s]}" for n, s in FULL_CASES])
def test_full_spectrum_against_float64(n, sfmt):
    """Every size (frame slots S = 8, 4, 2, 1; three passes at 8192) and format; an odd hop for 8-bit formats; a 70-channel
    device (more than the 64-bit wanted mask of one butterfly) at three sizes; duplicate bins; and tiles that end in a
    partial iteration of the frame slots."""
    hop = 313 if sfmt in (U8, S8) else 320
    counts = (3, 70, 1) if n in (256, 1024, 8192) else (3, 9, 1)
    g = case_group(n, hop, sfmt, FULL_FULLSCALE[sfmt], counts, wave_rate=8008)  # WAVE_BATCH 1001: odd device lengths
    tf, s = fft_tile_frames(n, g.bpc, g.hop_bytes)
    assert any((g.frames(d) % tf) % s or tf % s for d in range(len(g.bin_lists))) or s == 1
    (win, iq), = run_engine(g, 1)
    check_group_run(g, win, iq, full_k(n), key=f"full {n} {sfmt}")
    assert_duplicates_equal(g, iq, 1 << 30, False)


# ---- bitwise invariance ---------------------------------------------------------------------------------------------------
PROBE_N = 1024


def probe_group(others, at, sfmt=U8, hop=313, cmax=49):
    """A probe device (49 channels: R1 = 16, two passes, channel 37 on channel 5's bin) at position `at` of a group with the
    other devices' channel lists; returns (group, probe index)."""
    n = PROBE_N
    probe_bins = bin_lists(n, [cmax], 16, 7)[0]
    bpc = 2 * cm.BYTES_PER_SAMPLE[sfmt]
    probe_raw = make_stream(4242, n, hop * bpc, sfmt, AGC + 3 * 1000, probe_bins[0], cm.DEFAULT_FULLSCALE[sfmt], True)
    bl = [b for b in others[:at]] + [probe_bins] + others[at:]
    nbs = [2, 1, 3, 1][:at] + [3] + [1, 3, 2, 1][:len(others) - at]
    streams = [make_stream(11 + d, n, hop * bpc, sfmt, AGC + nbs[d] * 1000, None, cm.DEFAULT_FULLSCALE[sfmt], True) for d in range(len(bl))]
    streams[at] = probe_raw
    return Group(n, hop * bpc, sfmt, bl, nbs, streams=streams), at


@pytest.mark.parametrize("fft_mode", [2, 1])
def test_rows_do_not_depend_on_where_the_frames_sit(fft_mode, monkeypatch):
    """The probe's rows, bit for bit: first, in the middle or last of its group; in runs of 4 batches and of 1; under three
    frames-per-tile settings (ABG_K1_CTA_KB, pruned kernel); and with groups of other formats and hops in the same engine."""
    others = bin_lists(PROBE_N, [3, 17, 1, 9], 16, 3)
    g0, at0 = probe_group(others, 0)
    (win, iq), = run_engine(g0, fft_mode)
    cols0 = slice(g0.g0[at0], g0.g0[at0 + 1])
    want = (win[:3000, cols0].copy(), iq[:3000, cols0].copy())
    K = pruned_k(PROBE_N, 49, 64) if fft_mode == 2 else full_k(PROBE_N)
    check_device(g0, at0, win, iq, AGC, 3000, K)
    if fft_mode == 2:
        assert np.array_equal(iq[:3000, g0.g0[at0] + 5].view(np.uint64), iq[:3000, g0.g0[at0] + 37].view(np.uint64))

    def same(w, i, g, at, rows=slice(0, 3000)):
        cols = slice(g.g0[at], g.g0[at + 1])
        assert np.array_equal(w[rows, cols].view(np.uint32), want[0][rows].view(np.uint32))
        assert np.array_equal(i[rows, cols].view(np.uint64), want[1][rows].view(np.uint64))

    for at in (2, 4):
        g, a = probe_group(others, at)
        (w, i), = run_engine(g, fft_mode)
        same(w, i, g, a)
    outs = run_engine(g0, fft_mode, nbmax=1, runs=3)
    for k, (w, i) in enumerate(outs):
        cols = slice(g0.g0[at0], g0.g0[at0 + 1])
        assert np.array_equal(w[:1000, cols].view(np.uint32), want[0][k * 1000:(k + 1) * 1000].view(np.uint32)), k
        assert np.array_equal(i[:1000, cols].view(np.uint64), want[1][k * 1000:(k + 1) * 1000].view(np.uint64)), k
    if fft_mode == 2:
        for kb in ("24", "96", "160"):
            monkeypatch.setenv("ABG_K1_CTA_KB", kb)
            (w, i), = run_engine(g0, fft_mode)
            same(w, i, g0, at0)
        monkeypatch.delenv("ABG_K1_CTA_KB")
    # neighbouring groups: an S16 and an F32 device and a U8 device of another hop in the same engine
    extra = [case_group(PROBE_N, h, f, fs, (5,)) for h, f, fs in ((320, S16, 32768.0), (320, F32, 1.0), (320, U8, 0.0))]
    devs = g0.cfg.devices + [x.cfg.devices[0] for x in extra]
    cfg = cm.Config(fft_size=PROBE_N, wave_rate=8000, devices=devs)
    e = lib.Engine(cfg, max_batches_per_run=4, input_capacity_batches=5, fft_mode=fft_mode)
    try:
        for d, r in enumerate(g0.raws + [x.raws[0] for x in extra]):
            assert e.fft_path(d) == fft_mode
            e.push(d, r)
        e.run(-1)
        w, i = e.k1_outputs()
        same(w, i, g0, at0)
    finally:
        e.close()


def test_pruned_push_patterns_and_compaction():
    """Pushed in uneven pieces into a buffer that compacts, one batch per run, with WAVE_BATCH = 1001 so that consumed % 16
    takes every residue the format allows (U8: every even one, S16: multiples of 4, F32: 0 and 8): rows bitwise equal to a
    whole push run four batches at a time, and against float64."""
    wave_rate, B, nb = 8008, 1001, 8
    groups = [case_group(1024, 313, f, fs, (9,), wave_rate=wave_rate) for f, fs in ((U8, 0.0), (S16, 32768.0), (F32, 1.0))]
    for x in groups:
        x.batches = [nb]
        x.raws = [make_stream(77 + x.sfmt, 1024, x.hop_bytes, x.sfmt, AGC + nb * B, x.bin_lists[0][0], x.fullscale, True)]
        residues = {((AGC + k * B) * x.hop_bytes) % 16 for k in range(nb)}
        assert residues == set(range(0, 16, x.bpc if x.bpc < 16 else 8)), (x.sfmt, residues)
    devs = [x.cfg.devices[0] for x in groups]
    cfg = cm.Config(fft_size=1024, wave_rate=wave_rate, devices=devs)
    rng = np.random.default_rng(5)

    def engine(cap, nbmax):
        e = lib.Engine(cfg, max_batches_per_run=nbmax, input_capacity_batches=cap, fft_mode=2)
        for d in range(len(devs)):
            assert e.fft_path(d) == 2
        return e

    whole = []
    e = engine(nb + 2, 4)
    try:
        for d, x in enumerate(groups):
            e.push(d, x.raws[0])
        for _ in range(2):
            e.run(-1)
            whole.append(e.k1_outputs())
    finally:
        e.close()
    K = pruned_k(1024, 9, 64)
    for d, x in enumerate(groups):
        cols = slice(9 * d, 9 * d + 9)
        for k, (w, i) in enumerate(whole):
            check_device(x, 0, w[:, cols], i[:, cols], AGC + 4 * k * B, 4 * B, K)
    e = engine(3, 1)
    got = [[] for _ in groups]
    try:
        pos = [0] * len(groups)
        for _ in range(4000):
            for d, x in enumerate(groups):
                step = min(int(rng.integers(1, 2 * B * x.hop_bytes // x.bpc)) * x.bpc, len(x.raws[0]) - pos[d])
                if step > 0 and e.batches_available(d) < 1:
                    e.push(d, x.raws[0][pos[d]:pos[d] + step])
                    pos[d] += step
            if all(e.batches_available(d) >= 1 for d in range(len(groups))):
                assert e.run(1) == len(groups)
                for d in range(len(groups)):
                    e.fetch_all(d)
                w, i = e.k1_outputs()
                for d in range(len(groups)):
                    got[d].append((w[:B, 9 * d:9 * d + 9].copy(), i[:B, 9 * d:9 * d + 9].copy()))
                if len(got[0]) == nb:
                    break
    finally:
        e.close()
    assert len(got[0]) == nb
    for d in range(len(groups)):
        cols = slice(9 * d, 9 * d + 9)
        w_all = np.concatenate([w[:4 * B, cols] for w, _ in whole])
        i_all = np.concatenate([i[:4 * B, cols] for _, i in whole])
        assert np.array_equal(np.concatenate([w for w, _ in got[d]]).view(np.uint32), w_all.view(np.uint32)), d
        assert np.array_equal(np.concatenate([i for _, i in got[d]]).view(np.uint64), i_all.view(np.uint64)), d


@pytest.mark.parametrize("fft_mode", [2, 1])
def test_set_bin_and_scan_select_between_runs(fft_mode):
    """Both kernels read bins[] at launch: after set_bin between runs, the next run's rows match float64 at the new bins.
    scan_select swaps a channel's frequency-level state (modulation, filters, squelch) but not its bin, as the reference
    retunes the device rather than the FFT bin: the next run's rows stay at the old bin, though the new entry lists another."""
    n = 2048
    g = case_group(n, 320, S16, 32768.0, (5, 2))
    g.batches = [2] * len(g.batches)
    g.raws = [make_stream(90 + d, n, g.hop_bytes, S16, AGC + 2 * g.B, None if d == 0 else g.bin_lists[d][0], g.fullscale, True)
              for d in range(len(g.bin_lists))]
    new = [n // 2 + 3, 0]

    def between(e, k):
        if k == 1:
            e.set_bin(0, 1, new[0])
            e.set_bin(1, 0, new[1])
            e.scan_select(2, 0, 1)

    e_scan = [cm.Channel(bin=g.bin_lists[2][0]), cm.Channel(bin=(g.bin_lists[2][0] + 7) % n)]
    outs = []
    e = lib.Engine(g.cfg, max_batches_per_run=1, input_capacity_batches=4, fft_mode=fft_mode)
    try:
        e.scan_configure(2, 0, e_scan)
        for d, r in enumerate(g.raws):
            assert e.fft_path(d) == fft_mode
            e.push(d, r)
        for k in range(2):
            between(e, k)
            e.run(-1)
            for d in range(len(g.raws)):
                e.fetch_all(d)
            outs.append(e.k1_outputs())
    finally:
        e.close()
    K = pruned_k(n, 5, 64) if fft_mode == 2 else full_k(n)
    for d in range(len(g.bin_lists)):
        check_device(g, d, *outs[0], AGC, g.B, K)
    after = [list(b) for b in g.bin_lists]
    after[0][1], after[1][0] = new
    for d in range(len(g.bin_lists)):
        check_device(g, d, *outs[1], AGC + g.B, g.B, K, bins=after[d])


# ---- AFC spectra -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", SIZES)
def test_afc_spectra_against_float64(n):
    """Engine.k1_spectra: each row is the full float64 spectrum of its batch-final frame under the per-frame bound, on the
    unprimed first run and on primed later runs; the batch-final row of iqin at each channel's bin (read before the run: AFC
    moves bins) is the spectrum row's value there, bit for bit.  The AFC device shares its format and hop with a device
    without AFC, so the whole group takes the full-spectrum kernel; that device's rows are checked too."""
    sfmt = (U8, S8, S16, F32, U8, S16)[SIZES.index(n)]
    hop = 313 if sfmt in (U8, S8) else 320
    g = case_group(n, hop, sfmt, FULL_FULLSCALE[sfmt], (3,), afc=(0,))
    g.batches = [3, 3]
    g.raws = [make_stream(30 + d, n, g.hop_bytes, sfmt, AGC + 3 * g.B, g.bin_lists[d][0] if d else n // 5, g.fullscale, True)
              for d in range(2)]
    K = full_k(n)
    e = lib.Engine(g.cfg, max_batches_per_run=4, input_capacity_batches=5, fft_mode=0)
    worst = 0.0
    try:
        with pytest.raises(lib.AbgError):
            e.k1_spectra(0)
        for d, r in enumerate(g.raws):
            assert e.fft_path(d) == 1
            e.push(d, r)
        for k in range(3):
            bins = [e.stats(0, c).bin for c in range(len(g.bin_lists[0]))]
            e.run(-1)
            spec = e.k1_spectra(0)
            win, iq = e.k1_outputs()
            assert spec.shape == (1, n)
            frame = AGC + (k + 1) * g.B - 1
            fin = reference_frame(g.frame_bytes(0, [frame]), sfmt, n, g.fullscale)
            ratio = np.abs(spec.astype(np.complex128) - np.fft.fft(fin, axis=1)) / (K * U * np.abs(fin).sum())
            assert ratio.max() <= 1.0, (k, float(ratio.max()), int(np.argmax(ratio)))
            assert (ratio ** 2).mean() ** 0.5 <= RMS_FRACTION
            worst = max(worst, float(ratio.max()))
            got = iq[g.B - 1, :len(bins)]
            assert np.array_equal(got.view(np.uint64), spec[0, bins].view(np.uint64)), (k, bins)
            check_device(g, 0, win, iq, AGC + k * g.B, g.B, K, bins=bins)
            if k == 0:
                check_device(g, 1, win, iq, AGC, 3 * g.B, K)
        with pytest.raises(lib.AbgError):
            e.k1_spectra(1)
    finally:
        e.close()
    RATIOS[f"afc {n}"] = (worst, 0.0)
    print(f"\nRATIO afc spectra {n}: worst {worst:.4g} of K = {K}")


def test_afc_spectra_of_several_batches():
    """Resident runs advance AFC devices by several batches: row b of k1_spectra is the frame that ends batch b."""
    n, sfmt = 2048, S16
    g = case_group(n, 320, sfmt, 32768.0, (3,), afc=(0, 1))
    nbmax = 4
    e = lib.Engine(g.cfg, max_batches_per_run=nbmax, input_capacity_batches=5, fft_mode=0)
    try:
        raws = []
        for d in range(2):
            need = e.resident_bytes_needed(d)
            raw = make_stream(60 + d, n, g.hop_bytes, sfmt, need // g.hop_bytes + 1, g.bin_lists[d][0], g.fullscale, True)[:need]
            raws.append(raw)
            e.resident_load(d, raw)
        g.raws = raws
        for rep in range(2):  # unprimed, then primed: the same frames
            e.run_resident(nbmax)
            for d in range(2):
                spec = e.k1_spectra(d)
                assert spec.shape == (nbmax, n)
                frames = [AGC + (b + 1) * g.B - 1 for b in range(nbmax)]
                fin = reference_frame(g.frame_bytes(d, frames), sfmt, n, g.fullscale)
                ratio = np.abs(spec.astype(np.complex128) - np.fft.fft(fin, axis=1)) / (full_k(n) * U * np.abs(fin).sum(1))[:, None]
                assert ratio.max() <= 1.0, (rep, d, float(ratio.max()))
    finally:
        e.close()
