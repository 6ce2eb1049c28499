"""CPU checks of the algebra behind the tensor-core K1 (rtlsdr-airband_b200/csrc/k1_tc.cu): the coefficient table the
library builds on the host (window * twiddle quantised to signed 8-bit digits, laid out as the MMA's shared-memory image)
is run through an exact integer contraction in numpy, recombined as the kernel's epilogue does, and compared with a
float64 DFT of the reference's float32 frame (reference src/rtl_airband.cpp:402-455,460,483-489).  No GPU involved:
the table builder and the plan are host code behind the C ABI (abg_debug_tc_table)."""
import numpy as np
import pytest

from airband_b200 import config as cm
from airband_b200 import lib


def window_f32(n):
    a = [np.float32(x) for x in (0.27105140069342, 0.43329793923448, 0.21812299954311, 0.06592544638803, 0.01081174209837,
                                 0.00077658482522, 0.00001388721735)]
    i = np.arange(n, dtype=np.float64)
    x = np.zeros(n)
    for k, ak in enumerate(a):
        x += (-1) ** k * float(ak) * np.cos(2.0 * np.pi * k * i / (n - 1))
    return x.astype(np.float32)


def emulate(tab, sq, cscale, plan, raw_rows, sfmt):
    """raw_rows [frames, K] bytes -> complex [frames, C] exactly as the MMA + epilogue compute it."""
    K, NC, ND, C2p = plan["K"], plan["NC"], plan["ND"], plan["C2p"]
    B = tab.transpose(0, 1, 3, 2).reshape(K, NC).astype(np.int64)          # [k byte][column]
    A = raw_rows.astype(np.int64)
    if sfmt == cm.SFMT_S8:
        A = raw_rows.view(np.int8).astype(np.int64)
    acc = A @ B                                                              # S32 accumulators (exact)
    assert np.abs(acc).max() < 2 ** 31
    v = np.zeros((A.shape[0], C2p), np.int64)
    for d in range(ND):
        v = v * 256 + acc[:, d * C2p:(d + 1) * C2p]
    mul, off = (2, 255) if sfmt == cm.SFMT_U8 else (1, 0)
    x = ((mul * v - off * sq[None, :]).astype(np.float64) * cscale).astype(np.float32)
    return x[:, 0::2] + 1j * x[:, 1::2]


@pytest.mark.parametrize("n,hop,digits", [(512, 320, 4), (2048, 320, 4), (2048, 320, 3), (256, 64, 4), (1024, 128, 4)])
@pytest.mark.parametrize("sfmt", [cm.SFMT_U8, cm.SFMT_S8])
def test_integer_dft_matches_float64(n, hop, digits, sfmt):
    rng = np.random.default_rng(n + digits)
    bins = [5, n // 3, n - 7, n // 2 + 1, 1, n - 1, 44, 411 % n][: (8 if n >= 512 else 3)]
    plan, tab, sq, cs = lib.tc_table(n, sfmt, hop * 2, bins, digits)
    assert plan["eligible"] and plan["K"] == 2 * n and plan["NC"] % 32 == 0 and plan["smem_bytes"] <= 227 * 1024
    assert np.all(tab[:, :, plan["ND"] * plan["C2p"]:, :] == 0)
    frames = 16
    # a strong carrier on one of the bins plus noise, quantised like the synthetic input
    t = np.arange(n)
    raws = []
    for f in range(frames):
        x = 0.6 * np.exp(2j * np.pi * (bins[1] + 0.1) * t / n + 1j * f) + 0.02 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
        iq = np.empty(2 * n)
        iq[0::2], iq[1::2] = x.real, x.imag
        if sfmt == cm.SFMT_U8:
            raws.append(np.clip(np.rint(127.5 * iq + 127.5), 0, 255).astype(np.uint8))
        else:
            raws.append(np.clip(np.rint(127.5 * iq - 0.5), -127, 127).astype(np.int8).view(np.uint8))
    raw = np.stack(raws)
    got = emulate(tab, sq, cs, plan, raw, sfmt)
    # the reference's float32 frame: levels LUT * window (rtl_airband.cpp:319-324,414-418), then a float64 DFT
    w = window_f32(n)
    if sfmt == cm.SFMT_U8:
        lev = ((raw.astype(np.float32) - np.float32(127.5)) / np.float32(127.5)).astype(np.float32)
    else:
        lev = (raw.view(np.int8).astype(np.float32) / np.float32(128.0)).astype(np.float32)
    fin = (lev[:, 0::2] * w).astype(np.float32) + 1j * (lev[:, 1::2] * w).astype(np.float32)
    ref = np.fft.fft(fin.astype(np.complex128), axis=1)[:, bins]
    scale = np.abs(ref).max()
    err = np.abs(got[:, :len(bins)] - ref).max() / scale
    assert err < (3e-7 if digits == 4 else 1e-6), err


def test_plan_rejects_what_the_kernel_cannot_do():
    assert not lib.tc_table(4096, cm.SFMT_S16, 2500, [1])[0]["eligible"]     # 16-bit samples
    assert not lib.tc_table(2048, cm.SFMT_U8, 600, [1])[0]["eligible"]       # hop 300 samples: 600 bytes, not a multiple of 32
    assert not lib.tc_table(2048, cm.SFMT_U8, 640, list(range(1, 40)))[0]["eligible"]  # 39 channels x 4 digits > 256 columns
    p = lib.tc_table(2048, cm.SFMT_U8, 640, list(range(1, 9)))[0]
    assert p["eligible"] and p["HC"] == 40 and p["halo"] == 6 and p["NC"] == 64 and (p["S"] // 16) % 2 == 1
    assert p["consumer_warpgroups"] == 2 and p["acc_regs"] == 32 and p["smem_bytes"] <= 200 * 1024
    p32 = lib.tc_table(1024, cm.SFMT_U8, 640, list(range(1, 33)))[0]
    assert p32["NC"] == 256 and p32["acc_regs"] == 128                       # 32 channels: the widest wgmma (N = 256)


# ---- the plan space ---------------------------------------------------------------------------------------------------
# Settings of the two geometry knobs (environment variables read by the planner) the tests run under; {} = the defaults.
KNOBS = ({}, {"ABG_K1_TC_STAGES": "2"}, {"ABG_K1_TC_STAGES": "3"}, {"ABG_K1_TC_CAP_KB": "64"}, {"ABG_K1_TC_CAP_KB": "100"},
         {"ABG_K1_TC_CAP_KB": "227"})
PLAN_FFT_SIZES = (256, 512, 1024, 2048, 4096, 8192)
PLAN_HOP_BYTES = (32, 64, 128, 256, 320, 512, 640, 800, 1280)
PLAN_CHANNELS = (1, 2, 4, 5, 8, 12, 16, 17, 32)
TC_CTRL_BYTES = 1024  # k1_tc.cu: barriers + tile-info ring in front of the stage ring


def tile_stages(plan, hop_bytes):
    """The stages of one tile as every warp role of k1_tc.cu walks them (StageSeq): (first pair, pairs, first k-step,
    k-steps per pair)."""
    K, KBS, pps = plan["K"], plan["KBS"], plan["pps"]
    npairs = min(plan["HC"] // 2, K // 32)
    out, p = [], 0
    while p < npairs:
        nk = -(-(K - 32 * p) // hop_bytes)
        np_ = min(pps, npairs - p, ((K - (nk - 1) * hop_bytes + 31) >> 5) - p)
        for q0 in range(0, nk, KBS):
            out.append((p, np_, q0, min(KBS, nk - q0)))
        p += np_
    return out


def plan_class(plan, hop_bytes):
    """(stages hold several column pairs, a pair's k-steps are cut into several stages, how the ring meets the tile:
    'deeper' = more ring stages than a tile has, so the ring never wraps inside a tile; 'divides' = every tile starts at ring
    stage 0 again; 'uneven' = tiles start at changing ring stages and barrier phases)."""
    n = len(tile_stages(plan, hop_bytes))
    ring = "deeper" if plan["NSTB"] > n else "divides" if n % plan["NSTB"] == 0 else "uneven"
    return plan["pps"] > 1, plan["KBS"] < -(-plan["K"] // hop_bytes), ring


# Every class the planner produces over the space below under its default knobs (checked by test_plan_space); the GPU tests
# of the kernel's scheduling (test_gpu_tc_geometry.py) assert that between them they ran each one.  A cut pair is never
# grouped: grouping needs at most 2 k-steps per pair, cutting at least 3.
PLAN_CLASSES = frozenset((g, c, r) for g, c in ((False, False), (False, True), (True, False)) for r in ("deeper", "divides", "uneven"))
PLAN_GROUPED_PPS = frozenset({2, 3, 4, 5, 6, 7, 8, 9})  # column pairs per stage of the grouped plans, default knobs


@pytest.mark.parametrize("knobs", KNOBS, ids=lambda k: "-".join(f"{a[10:]}{b}" for a, b in k.items()) or "default")
def test_plan_space(knobs, monkeypatch):
    """What k1_tc.cu takes for granted about every plan the host hands it, over fft sizes x hops x channel counts x digits x
    formats, under the default geometry and under each knob setting."""
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)
    classes, pps_seen, n = set(), set(), 0
    for N in PLAN_FFT_SIZES:
        for hop in PLAN_HOP_BYTES:
            for ch in PLAN_CHANNELS:
                for digits in (3, 4):
                    for sfmt in (cm.SFMT_U8, cm.SFMT_S8):
                        p = lib.tc_plan(N, sfmt, hop, ch, digits)
                        what = (N, hop, ch, digits, sfmt, p)
                        assert p["eligible"] == (digits * ((2 * ch + 7) & ~7) <= 256), what
                        if not p["eligible"]:
                            continue
                        n += 1
                        K, S, NC, KBS, NSTB, pps = p["K"], p["S"], p["NC"], p["KBS"], p["NSTB"], p["pps"]
                        kq = -(-K // hop)
                        assert K == 2 * N and p["HC"] * 16 == hop and p["ND"] == digits and p["C2p"] == (2 * ch + 7) & ~7, what
                        stage = ((2 * pps * S + 127) & ~127) + pps * KBS * NC * 32
                        assert p["smem_bytes"] == TC_CTRL_BYTES + NSTB * stage and p["smem_bytes"] <= 227 * 1024, what
                        assert 2 <= NSTB <= 32, what
                        assert p["halo"] == (K - 32) // hop and S % 16 == 0 and (S // 16) % 2 == 1 and S // 16 >= 128 + p["halo"], what
                        assert NC % 32 == 0 and digits * p["C2p"] <= NC <= 256 and p["acc_regs"] == NC // 2, what
                        assert 1 <= KBS <= kq and pps >= 1 and (pps == 1 or kq <= 2), what
                        assert 127 + KBS <= S // 16, what  # the A rows a stage's last k-step reads exist in the stage
                        # the stages of a tile cover every (column pair, k-step) with 32 p + q hop_bytes < K exactly once,
                        # and none holds more than the stage has room for
                        st = tile_stages(p, hop)
                        seen = set()
                        for (p0, np_, q0, nq) in st:
                            assert 1 <= np_ <= pps and 1 <= nq <= KBS and (np_ == 1 or q0 == 0), what
                            for g in range(p0, p0 + np_):
                                for q in range(q0, q0 + nq):
                                    assert (g, q) not in seen and 32 * g + q * hop < K, what
                                    seen.add((g, q))
                        assert len(seen) == sum(-(-(K - 32 * g) // hop) for g in range(min(hop // 32, K // 32))), what
                        classes.add(plan_class(p, hop))
                        if pps > 1:
                            pps_seen.add(pps)
    assert n > 1500
    if not knobs:
        assert classes == PLAN_CLASSES and pps_seen == PLAN_GROUPED_PPS, (sorted(classes), sorted(pps_seen))
    if "ABG_K1_TC_STAGES" in knobs:
        assert pps_seen == set() and {c[2] for c in classes} == {"divides" if knobs["ABG_K1_TC_STAGES"] == "2" else "uneven"}


# ---- the S32 accumulators cannot wrap ------------------------------------------------------------------------------------
def _flat(tab, plan):
    return tab.transpose(0, 1, 3, 2).reshape(plan["K"], plan["NC"]).astype(np.int64)  # [k byte][column]


def reference_frame(raw_rows, sfmt, n, fullscale=None):
    """The reference's float32 frame of each row of raw bytes [frames, n * bytes per complex sample], as complex128
    [frames, n]: 8-bit levels LUT x window (rtl_airband.cpp:319-324,414-418); S16 and F32 (1/fullscale * x) * window
    (:402-436), each product rounded to float32."""
    w = window_f32(n)
    if sfmt == cm.SFMT_U8:
        lev = ((raw_rows.astype(np.float32) - np.float32(127.5)) / np.float32(127.5)).astype(np.float32)
    elif sfmt == cm.SFMT_S8:
        lev = (raw_rows.view(np.int8).astype(np.float32) / np.float32(128.0)).astype(np.float32)
    else:
        x = np.ascontiguousarray(raw_rows).view(np.int16 if sfmt == cm.SFMT_S16 else np.float32).astype(np.float32)
        lev = (np.float32(1.0) / np.float32(fullscale)) * x
    fin = (lev[:, 0::2] * w).astype(np.float32) + 1j * (lev[:, 1::2] * w).astype(np.float32)
    return fin.astype(np.complex128)


def reference_bins(raw_rows, sfmt, n, bins, fullscale=None):
    """reference_frame transformed by a float64 DFT at `bins`: complex128 [frames, len(bins)]."""
    b = np.asarray(bins, np.int64) % n
    tw = np.exp(-2j * np.pi * ((np.arange(n, dtype=np.int64)[:, None] * b[None, :]) % n) / n)
    return reference_frame(raw_rows, sfmt, n, fullscale) @ tw


def reference_spectrum(raw_rows, sfmt, n, fullscale=None):
    """reference_frame's full float64 spectrum in natural bin order: complex128 [frames, n]."""
    return np.fft.fft(reference_frame(raw_rows, sfmt, n, fullscale), axis=1)


def adversarial_frame(n, sfmt, bins, digits=4):
    """The one frame of raw bytes that drives an S32 accumulator of the MMA furthest: in the table's column with the largest
    sum of |digit|, the code of largest magnitude with the digit's sign at every k (U8: 255 or 0, S8: 127 or -128).
    Returns (bytes uint8[2n], that column's bound amax * sum |digit|)."""
    plan, tab, _, _ = lib.tc_table(n, sfmt, 640, bins, digits)
    B = _flat(tab, plan)
    sums = np.abs(B).sum(0)
    col = int(np.argmax(sums))
    if sfmt == cm.SFMT_U8:
        return np.where(B[:, col] > 0, 255, 0).astype(np.uint8), 255 * int(sums[col])
    return np.where(B[:, col] < 0, -128, 127).astype(np.int8).view(np.uint8), 128 * int(sums[col])


def overflow_bins(n):
    return [n // 2, n // 4, 1, n // 3 | 1, n - 1, 0]


@pytest.mark.parametrize("digits", [3, 4])
@pytest.mark.parametrize("sfmt", [cm.SFMT_U8, cm.SFMT_S8])
@pytest.mark.parametrize("n", PLAN_FFT_SIZES)
def test_no_byte_stream_can_wrap_an_accumulator(n, sfmt, digits):
    """wgmma's S32 accumulation wraps silently, so 'exact' needs a bound over ANY input: per column, the largest sample
    magnitude times the sum over k of |digit| stays below 2^31 (at worst 16384 bytes x 128 x 255 = 2^29).  The stream that
    reaches the bound of the worst column still matches the float64 DFT."""
    bins = overflow_bins(n)
    plan, tab, sq, cs = lib.tc_table(n, sfmt, 640, bins, digits)
    B = _flat(tab, plan)
    amax = 255 if sfmt == cm.SFMT_U8 else 128
    assert plan["K"] * 128 * 255 < 2 ** 31 and np.abs(B).max() <= 128
    assert amax * int(np.abs(B).sum(0).max()) < 2 ** 31
    frame, bound = adversarial_frame(n, sfmt, bins, digits)
    A = frame.astype(np.int64) if sfmt == cm.SFMT_U8 else frame.view(np.int8).astype(np.int64)
    acc = A @ B
    # the adversarial frame reaches the worst column's bound, up to the k where the digit is 0 or the code range is lopsided
    assert bound * 0.49 <= np.abs(acc).max() <= bound < 2 ** 31
    got = emulate(tab, sq, cs, plan, frame[None, :], sfmt)
    ref = reference_bins(frame[None, :], sfmt, n, bins)
    assert np.abs(got[:, :len(bins)] - ref).max() / np.abs(ref).max() < (3e-7 if digits == 4 else 1e-6)


# ---- the table under several bin lists -----------------------------------------------------------------------------------
@pytest.mark.parametrize("digits", [3, 4])
@pytest.mark.parametrize("sfmt", [cm.SFMT_U8, cm.SFMT_S8])
def test_table_invariants_under_several_bin_lists(sfmt, digits):
    n = 1024
    lists = ([n // 2], [n // 2, n // 2 + 1, n // 2 - 1], [7, n // 2, 1, n - 1, 333], [333, 7, n - 1, 1, n // 2], list(range(1, 18)))
    tabs = []
    for bins in lists:
        plan, tab, sq, cs = lib.tc_table(n, sfmt, 640, bins, digits)
        ND, C2p, NC = plan["ND"], plan["C2p"], plan["NC"]
        B = _flat(tab, plan)
        assert not B[:, ND * C2p:].any()                                   # padding columns of the MMA
        v = np.zeros((plan["K"], C2p), np.int64)
        for d in range(ND):
            v = v * 256 + B[:, d * C2p:(d + 1) * C2p]
            assert not B[:, d * C2p + 2 * len(bins):(d + 1) * C2p].any()   # padding channels, in every digit
        assert np.array_equal(sq, v.sum(0)) and not sq[2 * len(bins):].any()
        # the de-digitised table is window x twiddle to half a unit of the last digit
        w = (window_f32(n) * (np.float32(1.0) / np.float32(127.5 if sfmt == cm.SFMT_U8 else 128.0))).astype(np.float64)
        Q = 2.0 ** (8 * ND - 2)
        th = 2.0 * np.pi * ((np.arange(n)[:, None] * (np.asarray(bins) % n)[None, :]) % n) / n
        re_i = np.cos(th) * w[:, None] / w.max() * Q                       # Re output, I input
        assert np.abs(v[0::2, 0:2 * len(bins):2] - re_i).max() <= 0.5 + 1e-6
        tabs.append((bins, plan, B, sq))
    # the same bins in another order: another table, namely the same columns in the other order
    (b3, p3, B3, sq3), (b4, p4, B4, sq4) = tabs[2], tabs[3]
    assert sorted(b3) == sorted(b4) and not np.array_equal(B3, B4) and not np.array_equal(sq3, sq4)
    for c4, b in enumerate(b4):
        c3 = b3.index(b)
        for d in range(p3["ND"]):
            for e in range(2):
                assert np.array_equal(B4[:, d * p4["C2p"] + 2 * c4 + e], B3[:, d * p3["C2p"] + 2 * c3 + e])
