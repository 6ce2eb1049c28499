"""GPU tests of the tensor-core K1's scheduling and geometry space (fft_mode 3, rtlsdr-airband_b200/csrc/k1_tc.cu): what K1
itself stored (Engine.k1_outputs: win = |X[bin]| and iqin = X[bin] per frame, before any squelch decision) for launches
in which every persistent CTA takes many tiles, several coefficient tables alternate, devices differ in channel count and
some run out of frames early - under every class of stage geometry the planner produces.

References.  (a) float64: the reference's float32 frame (level LUT x window) times a complex128 DFT matrix at the configured
bins (test_tc_dft_math.reference_bins), bound 3e-7 of the device's largest |X| at 4 digits and 1e-6 at 3, plus one float32
rounding for win.  (b) the output-pruned FP32 kernel (fft_mode 2) through the same tap, bound 3e-6.  Every output row of
every device is compared with (b); (a) is computed for the first and last two frames of every 128-frame tile and a seeded
sample of 8 more frames per device - all frames for the short streams of the smaller tests."""
import numpy as np
import pytest
import torch

from airband_b200 import config as cm
from airband_b200 import lib
from test_tc_dft_math import KNOBS, PLAN_CLASSES, adversarial_frame, overflow_bins, plan_class, reference_bins

pytestmark = pytest.mark.gpu

AGC = cm.AGC_EXTRA
TILE = 128  # frames per tile of k1_tc.cu


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Group:
    """Devices of one sample format, hop and fullscale (one K1 launch group) with different channel lists, streams and
    lengths.  hop_bytes counts bytes between frames; `afc` lists devices whose channels use AFC."""

    def __init__(self, n, hop_bytes, sfmt, bin_lists, batches, wave_rate=8000, seed0=0, streams=None, fullscale=0.0, rails=False,
                 afc=()):
        self.n, self.hop_bytes, self.sfmt, self.bin_lists, self.batches = n, hop_bytes, sfmt, [list(b) for b in bin_lists], list(batches)
        self.B = wave_rate // 8
        self.bpc = 2 * cm.BYTES_PER_SAMPLE[sfmt]
        sr = (hop_bytes // self.bpc) * wave_rate
        devs = [cm.Device(sample_rate=sr, sfmt=sfmt, fullscale=fullscale,
                          channels=[cm.Channel(bin=b, afc=4 if d in afc else 0) for b in bl]) for d, bl in enumerate(self.bin_lists)]
        self.fullscale = devs[0].fullscale
        self.cfg = cm.Config(fft_size=n, wave_rate=wave_rate, devices=devs)
        assert all(self.cfg.hop(d) * self.bpc == hop_bytes for d in range(len(devs)))
        self.g0 = np.concatenate([[0], np.cumsum([len(b) for b in self.bin_lists])]).astype(int)
        self.raws = streams or [make_stream(seed0 + d, n, hop_bytes, sfmt, self.frames(d), self.bin_lists[d][0] if d % 3 else None,
                                            self.fullscale, rails) for d in range(len(devs))]

    def frames(self, d):
        return AGC + self.batches[d] * self.B

    def tiles(self, d):
        return -(-self.frames(d) // TILE)

    def tables(self):
        return len({tuple(b) for b in self.bin_lists})

    def frame_bytes(self, d, frames):
        """raw bytes [len(frames), n * bytes per complex sample] of device d's stream frames `frames`."""
        start = np.asarray(frames, np.int64) * self.hop_bytes
        return self.raws[d][start[:, None] + np.arange(self.n * self.bpc)[None, :]]


def make_stream(seed, n, hop_bytes, sfmt, frames, tone_bin, fullscale=None, rails=False):
    """frames * hop_bytes + one frame of raw bytes.  8-bit: noise of +-44 codes around mid-scale, plus (tone_bin not None) a
    carrier of 70 codes on the centre of that bin, and with `rails` every 13th sample component at a rail code.  S16: the same
    shape at 256 times the amplitude, with rails at +-32767 and -32768.  F32: noise at 1e-2 of fullscale, or (tone_bin not
    None) a carrier at 0.5 of fullscale on that bin, one 100 dB weaker on bin tone_bin + n/4, and noise 140 dB below the
    carrier.  A third of the devices get noise alone, where no bin dominates the error bound's scale."""
    rng = np.random.default_rng(seed)
    bps = cm.BYTES_PER_SAMPLE[sfmt]
    nvals = (frames * hop_bytes) // bps + 2 * n
    t = np.arange(n)

    def tone(b, amp, phase):
        z = amp * np.exp(2j * np.pi * b * t / n + 1j * phase)
        one = np.empty(2 * n)
        one[0::2], one[1::2] = z.real, z.imag
        return np.resize(one, nvals)

    if sfmt == cm.SFMT_F32:
        if tone_bin is None:
            x = 1e-2 * fullscale * rng.standard_normal(nvals)
        else:
            x = fullscale * (tone(tone_bin, 0.5, seed) + tone(tone_bin + n // 4, 0.5e-5, 2 * seed) + 0.5e-7 * rng.standard_normal(nvals))
        return x.astype(np.float32).view(np.uint8)
    x = rng.integers(-44, 45, nvals, dtype=np.int16).astype(np.int64)
    if tone_bin is not None:
        x += np.rint(tone(tone_bin, 70, seed)).astype(np.int64)
    if sfmt == cm.SFMT_S16:
        x *= 256
        if rails:
            x[::13] = rng.choice([32767, -32767, -32768], x[::13].size)
        return x.astype(np.int16).view(np.uint8)
    if rails:
        x[::13] = rng.choice([-128, 127], x[::13].size)
    if sfmt == cm.SFMT_U8:
        return (np.clip(x, -128, 127) + 128).astype(np.uint8)
    return np.clip(x, -128, 127).astype(np.int8).view(np.uint8)


def k1_run(group, fft_mode, nbmax=4, runs=1):
    """Push every stream whole, run `runs` times, and return what K1 stored in each run: [(win [rows, G], iqin [rows, G])],
    or the pair itself for one run."""
    e = lib.Engine(group.cfg, max_batches_per_run=nbmax, input_capacity_batches=max(group.batches) + 2, fft_mode=fft_mode)
    try:
        for d, r in enumerate(group.raws):
            assert (e.fft_path(d) == 3) == (fft_mode == 3), f"device {d} takes K1 path {e.fft_path(d)}"
            e.push(d, r)
        outs = []
        for k in range(runs):
            assert e.run(-1) == sum(min(nbmax, max(0, b - k * nbmax)) for b in group.batches)
            outs.append(e.k1_outputs())
        return outs[0] if runs == 1 else outs
    finally:
        e.close()


def float64_frames(group, d, first_row, rows, rng):
    """Rows of device d checked against float64: the first and last two frames of every tile that has rows in
    [first_row, first_row + rows), and 8 seeded others; every row when there are at most 600."""
    if rows <= 600:
        return np.arange(rows)
    f = np.arange(first_row, first_row + rows) + AGC         # frame numbers of the rows (tiles start at frame 0 of the stream)
    edge = np.isin(f % TILE, (0, 1, TILE - 2, TILE - 1))
    edge[[0, 1, -2, -1]] = True
    return np.union1d(np.nonzero(edge)[0], rng.integers(0, rows, 8))


def check_against_float64(group, win, iq, digits=4, first_batch=0, n_batches=None):
    """win / iq rows [0, n_batches * B) of every device against the float64 DFT of frames AGC + first_batch * B + row."""
    rng = np.random.default_rng(99)
    bound = 3e-7 if digits == 4 else 1e-6
    worst = 0.0
    for d, bins in enumerate(group.bin_lists):
        nb = min(group.batches[d] - first_batch, win.shape[0] // group.B) if n_batches is None else n_batches[d]
        if nb <= 0:
            continue
        rows = float64_frames(group, d, first_batch * group.B, nb * group.B, rng)
        raw = group.frame_bytes(d, AGC + first_batch * group.B + rows)
        ref = reference_bins(raw, group.sfmt, group.n, bins)
        cols = slice(group.g0[d], group.g0[d + 1])
        assert_win_is_magnitude(win[rows, cols], iq[rows, cols])
        scale = np.abs(ref).max()
        err = np.abs(iq[rows, cols] - ref).max() / scale
        assert err < bound, f"device {d} (bins {bins}): X differs from float64 by {err:.3e} of {scale:.4g}, first bad row {rows[np.argmax(np.abs(iq[rows, cols] - ref).max(1))]}"
        werr = np.abs(win[rows, cols] - np.abs(ref)) - 2.0 ** -23 * np.abs(ref)
        assert werr.max() / scale < bound, f"device {d}: |X| differs from float64 by {werr.max() / scale:.3e}"
        worst = max(worst, err)
    return worst


def assert_win_is_magnitude(win, iq):
    """win is the correctly rounded float32 sqrtf(fl(fl(re*re) + fl(im*im))) of the stored iqin, the reference's association
    (rtl_airband.cpp:484); numpy's float32 square root is correctly rounded too."""
    re, im = np.real(iq).astype(np.float32), np.imag(iq).astype(np.float32)
    want = np.sqrt((re * re) + (im * im))
    assert np.array_equal(win.view(np.uint32), want.view(np.uint32)), f"win differs from |iqin| at {np.argwhere(win != want)[:4].tolist()}"


def check_every_row_against_fp32_kernel(group, win, iq, fwin, fiq):
    for d in range(len(group.bin_lists)):
        rows, cols = slice(0, group.batches[d] * group.B), slice(group.g0[d], group.g0[d + 1])
        scale = np.abs(fiq[rows, cols]).max()
        assert scale > 0
        err = np.abs(iq[rows, cols] - fiq[rows, cols]).max() / scale
        assert err < 3e-6, f"device {d}: X differs from the FP32 kernel by {err:.3e}"
        assert np.abs(win[rows, cols] - fwin[rows, cols]).max() / scale < 3e-6, f"device {d}: |X| differs from the FP32 kernel"
        # rows past the device's last frame were never written (buffers start zeroed): the tile's frame-count mask
        assert not win[rows.stop:, cols].any() and not iq[rows.stop:, cols].any(), f"device {d}: stores past its last frame"


def bin_pool(n):
    return [n // 2, n // 2 + 1, n // 2 - 1, 1, n - 1, 5, n // 4, n // 3 | 1, 44 % n, n - 7, 2, 3, n // 8, n // 2 + 9, 17, 99 % n]


def mixed_group(n, hop_bytes, sfmt, cmax, wave_rate=8000, min_tiles=None):
    """As many devices as give every CTA 16 tiles with frames in them (min_tiles = 16 x SMs), cycling through channel lists of
    1, 3, min(8, cmax) and cmax bins cut from rotations of one pool (so neighbouring devices share bins at different channel
    positions, and N/2 and adjacent bins occur), and through batch counts 4, 4, 2, 4, 1, 3 so that devices which have run out
    of frames sit between busy ones in the tile order."""
    pool = (bin_pool(n) * 2)[:max(cmax, 8)] if cmax <= 16 else [(n // 2 + 37 * i) % n for i in range(cmax)]
    lens, nbs = (1, 3, min(8, cmax), cmax), (4, 4, 2, 4, 1, 3)
    min_tiles = 16 * sm_count() if min_tiles is None else min_tiles
    B = wave_rate // 8
    bin_lists, batches, tiles = [], [], 0
    while tiles < min_tiles or len(bin_lists) < 12:
        d = len(bin_lists)
        rot = d % 5
        bin_lists.append((pool[rot:] + pool[:rot])[:lens[d % 4]])
        batches.append(nbs[d % 6])
        tiles += -(-(AGC + batches[-1] * B) // TILE)
    g = Group(n, hop_bytes, sfmt, bin_lists, batches, wave_rate, seed0=n + hop_bytes)
    assert sum(g.tiles(d) for d in range(len(bin_lists))) >= min_tiles and g.tables() >= 3
    assert len({len(b) for b in bin_lists}) >= 3 and min(batches) < max(batches) == 4
    return g


# (fft_size, hop_bytes, format, most channels per device, digits, wave_rate)
U8, S8 = cm.SFMT_U8, cm.SFMT_S8
GEOMETRIES = {
    "2048_hop640_whole_pairs": (2048, 640, U8, 8, 4, 8000),
    "8192_hop640_cut_pairs": (8192, 640, U8, 8, 4, 8000),
    "4096_hop512": (4096, 512, U8, 8, 4, 8000),
    "512_hop640_grouped": (512, 640, U8, 8, 4, 8000),
    "256_hop640_pairs_without_ksteps": (256, 640, U8, 8, 4, 8000),
    "512_hop1280_pairs_without_ksteps": (512, 1280, U8, 8, 4, 8000),
    "512_hop1280_17ch_5_pairs_per_stage": (512, 1280, U8, 17, 4, 8000),
    "512_hop800_grouped_3_digits": (512, 800, U8, 5, 3, 8000),
    "1024_hop128_deep_halo": (1024, 128, U8, 8, 4, 8000),
    "256_hop32_one_pair": (256, 32, U8, 8, 4, 8000),
    "512_hop32_17ch_cut": (512, 32, U8, 17, 4, 8000),
    "2048_hop64_s8_cut": (2048, 64, S8, 4, 4, 8000),
    "2048_hop320_wave_rate_16000": (2048, 320, U8, 8, 4, 16000),
    "4096_hop256_s8_cut": (4096, 256, S8, 8, 4, 8000),
    "1024_hop640_32ch_256_columns": (1024, 640, U8, 32, 4, 8000),
    "1024_hop640_17ch": (1024, 640, U8, 17, 4, 8000),
    "2048_hop640_3_digits": (2048, 640, U8, 8, 3, 8000),
    "2048_hop256_s8_3_digits": (2048, 256, S8, 12, 3, 8000),
}


def test_the_geometries_cover_every_plan_class():
    """Host-only: the cases of the next test fall, between them, into every class of stage geometry the planner produces
    over its whole space under default knobs, with 2..5 and more pairs per stage among the grouped ones."""
    plans = {k: lib.tc_plan(n, sfmt, hop, cmax, dg) for k, (n, hop, sfmt, cmax, dg, _) in GEOMETRIES.items()}
    assert all(p["eligible"] for p in plans.values())
    assert {plan_class(p, GEOMETRIES[k][1]) for k, p in plans.items()} == PLAN_CLASSES
    pps = {p["pps"] for p in plans.values()}
    assert pps & {2, 3, 4, 5} and pps & {6, 7, 8, 9} and 1 in pps
    assert {p["C2p"] for p in plans.values()} >= {8, 16, 24, 40, 64} and {p["NC"] for p in plans.values()} >= {32, 64, 160, 256}


@pytest.mark.parametrize("name", list(GEOMETRIES))
def test_many_tiles_per_cta_every_geometry_class(name, monkeypatch):
    n, hop_bytes, sfmt, cmax, digits, wave_rate = GEOMETRIES[name]
    monkeypatch.setenv("ABG_K1_TC_DIGITS", str(digits))
    g = mixed_group(n, hop_bytes, sfmt, cmax, wave_rate)
    # one launch: tiles_per_dev of the longest device for every device, the frameless ones skipped by the scheduler
    assert len(g.bin_lists) * max(g.tiles(d) for d in range(len(g.bin_lists))) >= 16 * sm_count()
    win, iq = k1_run(g, 3)
    fwin, fiq = k1_run(g, 2)
    check_every_row_against_fp32_kernel(g, win, iq, fwin, fiq)
    check_against_float64(g, win, iq, digits)


def _knob_id(k):
    return "-".join(f"{a[10:]}{b}" for a, b in k.items())


def test_outputs_do_not_depend_on_ring_geometry(monkeypatch):
    """Exact integer sums make the k order free: the same mixed groups under the default ring and under every knob setting
    (ring depth 2 and 3, stage budgets of 64, 100 and 227 KB, which also change k-steps and pairs per stage) give
    bit-identical win and iqin.  One group whose default plan cuts pairs, one whose default plan groups them."""
    for (n, hop_bytes, sfmt, cmax) in ((4096, 640, U8, 8), (256, 640, U8, 8)):
        g = mixed_group(n, hop_bytes, sfmt, cmax)
        plans, outs = [], []
        for knobs in KNOBS:
            with monkeypatch.context() as m:
                for k, v in knobs.items():
                    m.setenv(k, v)
                p = lib.tc_plan(n, sfmt, hop_bytes, cmax)
                plans.append((p["pps"], p["KBS"], p["NSTB"]))
                outs.append(k1_run(g, 3))
        assert len(set(plans)) == len(KNOBS), plans
        check_against_float64(g, *outs[0])
        for knobs, (win, iq) in zip(KNOBS[1:], outs[1:]):
            assert np.array_equal(win.view(np.uint32), outs[0][0].view(np.uint32)), (n, _knob_id(knobs))
            assert np.array_equal(iq.view(np.uint64), outs[0][1].view(np.uint64)), (n, _knob_id(knobs))


def test_outputs_do_not_depend_on_tile_placement():
    """One device (stream + bin list) first, in the middle and last of a group whose other devices have other bin lists,
    channel counts and lengths (a table switch on both sides of it), in runs of 4 batches and of 1: the same bits every time,
    and stores never leave the device's own rows and columns.  The one-batch engine runs three times, so its third run
    refills the buffer of the first: a device with no third batch must find its first batch's rows untouched there."""
    n, hop_bytes = 2048, 640
    g = mixed_group(n, hop_bytes, U8, 8, min_tiles=4 * sm_count())
    probe_bins, probe_nb = [n // 2, 9, n // 2 + 1, n - 9, 77], 3
    probe_raw = make_stream(4242, n, hop_bytes, U8, AGC + probe_nb * g.B, 9)
    D = len(g.bin_lists)
    seen = []
    for at in (0, D // 2, D):
        bl = g.bin_lists[:at] + [probe_bins] + g.bin_lists[at:]
        nbs = g.batches[:at] + [probe_nb] + g.batches[at:]
        gp = Group(n, hop_bytes, U8, bl, nbs, streams=g.raws[:at] + [probe_raw] + g.raws[at:])
        cols = slice(gp.g0[at], gp.g0[at + 1])
        win4, iq4 = k1_run(gp, 3, nbmax=4)
        seen.append((win4[:probe_nb * g.B, cols], iq4[:probe_nb * g.B, cols]))
        for k, (w1, i1) in enumerate(k1_run(gp, 3, nbmax=1, runs=3)):
            for d, nb in enumerate(nbs):
                c = slice(gp.g0[d], gp.g0[d + 1])
                # run k holds batch k of the devices that have one; the others keep what the buffer held: run k-2's
                # batch (the buffers alternate), or zeros
                src = k if nb > k else k - 2 if k >= 2 and nb > k - 2 else None
                want_w, want_i = (win4[src * g.B:(src + 1) * g.B, c], iq4[src * g.B:(src + 1) * g.B, c]) if src is not None else (0, 0)
                assert np.array_equal(w1[:, c], want_w + np.zeros_like(w1[:, c])), (at, k, d)
                assert np.array_equal(i1[:, c], want_i + np.zeros_like(i1[:, c])), (at, k, d)
        if at == 0:
            check_against_float64(gp, win4, iq4)
    for w, i in seen[1:]:
        assert np.array_equal(w.view(np.uint32), seen[0][0].view(np.uint32)) and np.array_equal(i.view(np.uint64), seen[0][1].view(np.uint64))


@pytest.mark.parametrize("sfmt", [U8, S8], ids=["u8", "s8"])
def test_adversarial_bytes_do_not_wrap_the_accumulators(sfmt):
    """N = 8192: the frame that drives the worst column's S32 accumulator to its bound (test_tc_dft_math.adversarial_frame),
    placed at several frame positions of an otherwise random stream, and the all-rails streams, against float64."""
    n, hop_bytes, bins = 8192, 640, overflow_bins(8192)
    frame, bound = adversarial_frame(n, sfmt, bins)
    assert 2 ** 26 < bound < 2 ** 31
    B = 1000
    raw = make_stream(7, n, hop_bytes, sfmt, AGC + B, None)
    # 26 or more frames apart (a frame spans 25.6 hops): rows 100, 9, 63, 127 and 44 of their tiles, i.e. both warpgroups'
    # halves and their last rows, and the stream's last frame
    at = [AGC, 137, 191, 255, 300, AGC + B - 1]
    for f in at:
        raw[f * hop_bytes:f * hop_bytes + 2 * n] = frame
    rails = [np.full_like(raw, v) for v in ((0, 255) if sfmt == U8 else (0x80, 0x7F))]
    g = Group(n, hop_bytes, sfmt, [bins] * 3, [1] * 3, streams=[raw] + rails)
    win, iq = k1_run(g, 3)
    check_against_float64(g, win, iq)
    ref = reference_bins(frame[None, :], sfmt, n, bins)
    for f in at:
        assert np.abs(iq[f - AGC, :len(bins)] - ref[0]).max() / np.abs(ref).max() < 3e-7
