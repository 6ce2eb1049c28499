"""CPU checks of the identities the lane-parallel K2 tiles rely on (rtlsdr-airband_b200/csrc/k2_demod.cu: k2_am_tile,
k2_nfm_tile).  A tile computes, once per 8 / 16 samples and across the lanes, what the reference loop computes sample by sample
(reference src/squelch.cpp:195-276,501-514, src/filters.cpp:49-64, src/rtl_airband.cpp:510-518); it may only do so where the
re-arranged form gives the SAME IEEE single-precision value.  Each test walks the sequential form and the tile's form in numpy
float32 / integer arithmetic (one rounding per operation, like the -fmad=false build) and demands bit equality."""
import numpy as np
import pytest

F = np.float32
RNG = np.random.default_rng(20260923)


def bits(a):
    return np.asarray(a, dtype=np.float32).view(np.uint32)


@pytest.mark.parametrize("n", [8, 16])
def test_low_signal_counter_from_a_ballot(n):
    """low_signal_count_ after sample k = samples since the last one at or above the level: bit arithmetic on the ballot of
    (x >= level), as in both tiles, against the sequential counter (squelch.cpp:234-245)."""
    for _ in range(500):
        x = RNG.random(n).astype(F)
        lvl = F(RNG.choice([0.05, 0.5, 0.95]))
        low_in = int(RNG.integers(0, 90))
        seq, low = [], low_in
        for k in range(n):
            low = 0 if x[k] >= lvl else low + 1
            seq.append(low)
        ballot = sum(1 << k for k in range(n) if x[k] >= lvl)
        for k in range(n):
            z = ballot & ((2 << k) - 1)
            tile = (k - (z.bit_length() - 1)) if z else (low_in + k + 1)   # 31 - clz(z) == bit_length - 1
            assert tile == seq[k]


def test_capped_average_as_one_compare_against_plus_infinity():
    """capped = (capped >= cap && sample >= cap) ? cap : min(cap, 0.99 capped + t)  (squelch.cpp:506-513) with the two
    conditions folded into capped >= xc, xc = cap where the sample reaches the cap and +inf elsewhere."""
    cap = F(0.37)
    for _ in range(2000):
        c = F(RNG.choice([0.1, 0.37, 0.3699999, 0.5]))
        x = F(RNG.choice([0.2, 0.37, 0.9]))
        t = F(x * F(0.01))
        c2 = min(cap, F(F(c * F(0.99)) + t))
        ref = cap if (c >= cap and x >= cap) else c2
        xc = cap if x >= cap else F(np.inf)
        tile = cap if c >= xc else c2
        assert bits(ref) == bits(tile)


@pytest.mark.parametrize("n", [8, 16])
def test_shortcuts_for_fully_capped_and_never_capped_tiles(n):
    """k2_am_tile: with every sample at or above the cap and the average capped on entry the average stays at the cap; with no
    sample at or above the cap it is min(cap, 0.99 avg + t) - both bit-identical to the general recurrence."""
    cap = F(0.4)

    def general(c, xs):
        out = []
        for x in xs:
            t = F(x * F(0.01))
            c2 = min(cap, F(F(c * F(0.99)) + t))
            c = cap if (c >= cap and x >= cap) else c2
            out.append(c)
        return out
    for _ in range(300):
        hi = (cap + RNG.random(n).astype(F)).astype(F)            # all >= cap
        for c0 in (cap, F(0.47)):                                  # capped (or above a cap that just dropped) on entry
            assert all(bits(v) == bits(cap) for v in general(c0, hi))
        lo = (RNG.random(n).astype(F) * F(0.399)).astype(F)        # all < cap
        c, short = F(RNG.random() * 0.5), []
        c_in = c
        for x in lo:
            c = min(cap, F(F(c * F(0.99)) + F(x * F(0.01))))
            short.append(c)
        assert [int(bits(v)) for v in general(c_in, lo)] == [int(bits(v)) for v in short]


def test_derotation_phase_of_lane_k():
    """dm_phi advances by dm_dphi and is masked to 24 bits every sample (rtl_airband.cpp:516); lane k of a tile uses
    (phi0 + k * dphi) & 0xffffff computed in 32-bit unsigned arithmetic."""
    for _ in range(2000):
        phi0 = int(RNG.integers(0, 1 << 24))
        dphi = int(RNG.integers(0, 1 << 24))
        phi = phi0
        for k in range(17):
            assert ((phi0 + k * dphi) & 0xffffffff) & 0xffffff == phi
            phi = (phi + dphi) & 0xffffff


@pytest.mark.parametrize("n", [8, 16])
def test_notch_feed_forward_half_per_lane_recursive_half_serial(n):
    """NotchFilter::apply (filters.cpp:49-64): y = d0*x[k] - d1*x[k-1] + d0*x[k-2] + d1*y[k-1] - d2*y[k-2], evaluated left to
    right.  The tile computes A[k] = (d0*x[k] - d1*x[k-1]) + d0*x[k-2] per lane and walks y = (A[k] + d1*y1) - d2*y0."""
    d0, d1, d2 = F(0.9893), F(1.9771), F(0.9786)
    for _ in range(300):
        x = (RNG.standard_normal(n) * 0.3).astype(F)
        x1, x2, y1, y2 = (F(v) for v in RNG.standard_normal(4) * 0.3)   # nx1 (older), nx2, ny1 (older), ny2
        # sequential, as the reference writes it
        sx1, sx2, sy1, sy2, seq = x1, x2, y1, y2, []
        for k in range(n):
            x0 = sx1
            sx1, sx2 = sx2, x[k]
            y0 = sy1
            sy1 = sy2
            sy2 = F(F(F(F(F(d0 * sx2) - F(d1 * sx1)) + F(d0 * x0)) + F(d1 * sy1)) - F(d2 * y0))
            seq.append(sy2)
        # tile
        xm1 = np.concatenate(([x2], x[:-1])).astype(F)
        xm2 = np.concatenate(([x1, x2], x[:-2])).astype(F)
        A = [F(F(F(d0 * x[k]) - F(d1 * xm1[k])) + F(d0 * xm2[k])) for k in range(n)]
        ty1, ty2, tile = y1, y2, []
        for k in range(n):
            y0 = ty1
            ty1 = ty2
            ty2 = F(F(A[k] + F(d1 * ty1)) - F(d2 * y0))
            tile.append(ty2)
        assert [int(bits(v)) for v in seq] == [int(bits(v)) for v in tile]


@pytest.mark.parametrize("n", [8, 16])
def test_lowpass_real_and_imaginary_parts_are_independent_recurrences(n):
    """LowpassFilter::apply (filters.cpp:146-163) filters the complex sample with real coefficients: the real and the imaginary
    part never mix, so the tile walks them in the two half-warps at once; each is the same scalar recurrence."""
    c0, c1, gain = F(-0.6413), F(1.5610), F(49.8)
    z = (RNG.standard_normal(n) + 1j * RNG.standard_normal(n)).astype(np.complex64)

    def scalar(xs, st):
        x1, x2, y1, y2 = st
        out = []
        for v in xs:
            x0 = x1
            x1, x2 = x2, F(v / gain)
            y0 = y1
            y1 = y2
            y2 = F(F(F(F(x0 + x2) + F(F(2.0) * x1)) + F(c0 * y0)) + F(c1 * y1))
            out.append(y2)
        return out
    st_r = tuple(F(v) for v in RNG.standard_normal(4))
    st_i = tuple(F(v) for v in RNG.standard_normal(4))
    # complex form as the reference writes it (std::complex<float> * float and + act per component)
    x1, x2 = complex(st_r[0], st_i[0]), complex(st_r[1], st_i[1])
    y1, y2 = complex(st_r[2], st_i[2]), complex(st_r[3], st_i[3])
    ref = []
    for v in z:
        x0 = x1
        x1 = x2
        x2 = complex(F(v.real / gain), F(v.imag / gain))
        y0 = y1
        y1 = y2

        def comp(part):
            g = (lambda c: F(c.real)) if part == 0 else (lambda c: F(c.imag))
            return F(F(F(F(g(x0) + g(x2)) + F(F(2.0) * g(x1))) + F(c0 * g(y0))) + F(c1 * g(y1)))
        y2 = complex(comp(0), comp(1))
        ref.append(y2)
    re, im = scalar(z.real, st_r), scalar(z.imag, st_i)
    assert [int(bits(v.real)) for v in ref] == [int(bits(v)) for v in re]
    assert [int(bits(v.imag)) for v in ref] == [int(bits(v)) for v in im]


def test_am_agc_recurrence_without_the_clip_inside_a_committed_tile():
    """rtl_airband.cpp:553-562: agc = 0.995 agc + 0.005 x where x > level, then waveout = (wavein[j-100] - agc) / (1.5 agc) and
    the |waveout| > 0.8 clip (waveout *= 0.85, agc *= 1.15).  k2_am_tile walks the AGC without the clip and commits only when
    every sample's |n| < 1.199985 * agc (n = numerator), i.e. |n / (1.5 agc)| < 0.79999: then no sample clipped."""
    for _ in range(300):
        n = 16
        lvl = F(0.1)
        x = (0.5 + 0.2 * RNG.standard_normal(n)).astype(F)
        lag = (0.5 + 0.2 * RNG.standard_normal(n)).astype(F)
        a_seq, a_tile, clipped, calm = F(0.5), F(0.5), False, True
        for k in range(n):
            if x[k] > lvl:
                a_seq = F(F(a_seq * F(0.995)) + F(x[k] * F(0.005)))
                a_tile = F(F(a_tile * F(0.995)) + F(x[k] * F(0.005)))
            w = F(F(lag[k] - a_seq) / F(a_seq * F(1.5)))
            if abs(w) > F(0.8):
                clipped = True
                a_seq = F(a_seq * F(1.15))
            calm = calm and abs(F(lag[k] - a_tile)) < F(a_tile * F(1.199985))
        if calm:
            assert not clipped and bits(a_seq) == bits(a_tile)


# ---- the guard bands and range tests of k2_demod.cu, read from the source so that the checks below test the kernel's own
# constants.  The reference decides the AM clip from the rounded quotient, |fl(n / d)| > 0.8f with d = fl(1.5 agc)
# (rtl_airband.cpp:556-562); the kernel decides it without the division wherever |n| is far enough from 0.8 d, and falls
# back (refuses the tile / block, or divides exactly) elsewhere.  A "decided" outcome must therefore equal the reference's.
import os
import re

K2_SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rtlsdr-airband_b200", "csrc", "k2_demod.cu")


def _k2_source():
    with open(K2_SRC) as f:
        return f.read()


def _body(src, start):
    """Source from `start` to the end of that definition (a function body or a macro)."""
    i = src.index(start)
    j = src.find("\n}\n", i)
    k = src.find("#undef", i)
    return src[i:min(x for x in (j, k) if x > 0)]


def _hexf(s):
    return float.fromhex(s.rstrip("f"))


def _band_constants():
    src = _k2_source()
    run = _body(src, "__device__ __forceinline__ bool k2_open_run(")
    tile = _body(src, "__device__ __forceinline__ bool k2_am_tile(")
    samp = _body(src, "#define K2_OPEN_SAMPLE(")
    c = {
        "run_hi": re.search(r"an > a2 \* ([0-9.]+)f", run).group(1),
        "run_lo": re.search(r"an < a2 \* ([0-9.]+)f", run).group(1),
        "tile_lo": re.search(r"calm = an < a2k \* ([0-9.]+)f", tile).group(1),
        "samp_hi": re.search(r"an > dd \* ([0-9.]+)f", samp).group(1),
        "samp_lo": re.search(r"an < dd \* ([0-9.]+)f", samp).group(1),
    }
    rng = {}
    for name, body, d in (("run", run, "d_"), ("tile", tile, "d_"), ("samp", samp, "dd")):
        m = re.search(r"%s >= (0x1p-?\d+)f && %s <= (0x1p-?\d+)f && an >= (0x1p-?\d+)f && an <= (0x1p-?\d+)f" % (d, d), body)
        rng[name] = tuple(_hexf(x) for x in m.groups())
    return {k: F(float(v)) for k, v in c.items()}, rng


def _operands(rng, n):
    """(an, a2): agc values over the whole positive float32 range (subnormals included); |numerator| mostly within +-4e-5
    (relative) of 1.2 agc = 0.8 * 1.5 agc, where the guard bands sit, some ulp steps either side of 0.8 * fl(1.5 agc), and
    some anywhere."""
    e = rng.integers(0, 255, n, dtype=np.uint32)
    m = rng.integers(0, 1 << 23, n, dtype=np.uint32)
    a2 = ((e << 23) | m).view(np.float32)
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        d = (a2 * F(1.5)).astype(F)
        kind = rng.integers(0, 8, n)
        rel = np.where(kind < 5, rng.uniform(-4e-5, 4e-5, n), rng.uniform(-1.6e-5, -1.4e-5, n) * rng.choice([-1, 1], n))
        an = (a2.astype(np.float64) * 1.2 * (1.0 + rel)).astype(F)
        steps = rng.integers(-64, 65, n)
        near = (d.astype(np.float64) * np.float64(F(0.8))).astype(F)
        near = (near.view(np.int32) + steps.astype(np.int32)).view(np.float32)
        an = np.where(kind == 6, np.abs(near), an)
        wild = ((rng.integers(0, 255, n, dtype=np.uint32) << 23) | rng.integers(0, 1 << 23, n, dtype=np.uint32)).view(np.float32)
        an = np.where(kind == 7, wild, an)
    ok = np.isfinite(an) & np.isfinite(a2) & (a2 > 0)
    return an[ok].astype(F), a2[ok].astype(F)


def test_agc_clip_guard_bands_decide_like_the_rounded_quotient():
    """About 10^7 operand pairs through the three division-free forms of the |n / d| > 0.8f decision: k2_open_run (big /
    not big outside a band around 1.2 agc), k2_am_tile (`calm`: certainly not big) and K2_OPEN_SAMPLE (big / not big outside a
    band around 0.8 d).  Wherever a form counts as decided, its answer equals |fl(n / d)| > 0.8f."""
    c, rngs = _band_constants()
    rng = np.random.default_rng(62)
    inside = {"run": 0, "tile": 0, "samp": 0}
    decided = {"run": 0, "tile": 0, "samp": 0}
    total = 0
    for _ in range(10):
        an, a2 = _operands(rng, 1_000_000)
        total += an.size
        with np.errstate(over="ignore", under="ignore", invalid="ignore", divide="ignore"):
            d = (a2 * F(1.5)).astype(F)
            q = (an / d).astype(F)
            truth = np.abs(q) > F(0.8)
            inside_band = np.abs(an.astype(np.float64) / (1.2 * a2.astype(np.float64)) - 1.0) < 1e-5

            def in_range(name):
                dl, dh, nl, nh = rngs[name]
                return (d >= F(dl)) & (d <= F(dh)) & (an >= F(nl)) & (an <= F(nh))
            big = an > (a2 * c["run_hi"]).astype(F)
            ok = (big | (an < (a2 * c["run_lo"]).astype(F))) & in_range("run")
            assert np.array_equal(big[ok], truth[ok]), "k2_open_run decides the clip wrongly"
            decided["run"] += int(ok.sum()); inside["run"] += int((ok & inside_band).sum())
            calm = (an < (a2 * c["tile_lo"]).astype(F)) & in_range("tile")
            assert not truth[calm].any(), "k2_am_tile commits a tile in which a sample clips"
            decided["tile"] += int(calm.sum()); inside["tile"] += int((calm & inside_band).sum())
            bigs = an > (d * c["samp_hi"]).astype(F)
            sure = (bigs | (an < (d * c["samp_lo"]).astype(F))) & in_range("samp")
            assert np.array_equal(bigs[sure], truth[sure]), "K2_OPEN_SAMPLE decides the clip wrongly"
            decided["samp"] += int(sure.sum()); inside["samp"] += int((sure & inside_band).sum())
    assert total > 9_000_000
    # the operands really straddle the bands: most pairs are decided, and the undecided ones are the ones near 1.2 agc
    for k in decided:
        assert 0.1 * total < decided[k] < total, (k, decided[k], total)
        assert inside[k] == 0, (k, inside[k])


def _range_predicates():
    src = _k2_source()
    sq = re.search(r"bool k2_sqrt_ordinary_ok\(float x\) \{ return x >= (0x1p-?\d+)f && x <= (0x1p-?\d+)f; \}", src)
    dv = re.search(r"return ad >= (0x1p-?\d+)f && ad <= (0x1p-?\d+)f && an <= (0x1p-?\d+)f && \(an >= (0x1p-?\d+)f \|\| an == 0\.0f\);", src)
    assert sq and dv, "k2_sqrt_ordinary_ok / k2_div_ok changed shape: update this test"
    slo, shi = (F(_hexf(x)) for x in sq.groups())
    dlo, dhi, nhi, nlo = (F(_hexf(x)) for x in dv.groups())

    def sqrt_ok(x):
        return (x >= slo) & (x <= shi)

    def div_ok(n, d):
        an, ad = np.abs(n), np.abs(d)
        return (ad >= dlo) & (ad <= dhi) & (an <= nhi) & ((an >= nlo) | (an == F(0.0)))
    return sqrt_ok, div_ok


def _every_exponent():
    """Both signs, every exponent field (subnormals and inf / NaN included), mantissas 0, 1, a middle one and all ones."""
    e = np.arange(256, dtype=np.uint32)
    m = np.array([0, 1, 0x2aaaab, 0x7fffff], np.uint32)
    u = ((e[:, None] << 23) | m[None, :]).ravel()
    return np.concatenate([u, u | np.uint32(0x80000000)]).view(np.float32)


def test_sqrt_and_division_range_tests_admit_nothing_outside_the_documented_ranges():
    """k2_sqrt_ordinary (rsqrt.approx + one correction) equals sqrt.rn only on [2^-100, 2^125]; k2_div_ordinary (rcp.approx +
    Newton + remainder correction) equals div.rn only for |d| in [2^-62, 2^62] and |n| in [2^-62, 2^62] or n == 0.  The range
    tests must admit nothing outside, and everything inside."""
    sqrt_ok, div_ok = _range_predicates()
    x = _every_exponent()
    with np.errstate(invalid="ignore"):
        inside = (x >= F(2.0 ** -100)) & (x <= F(2.0 ** 125))
        got = sqrt_ok(x)
    assert not (got & ~inside).any(), x[got & ~inside][:8]
    assert got[inside].all()
    # the boundaries themselves and their neighbours
    for b in (2.0 ** -100, 2.0 ** 125):
        b = F(b)
        lo, hi = np.nextafter(b, F(0)), np.nextafter(b, F(np.inf))
        assert sqrt_ok(np.array([b]))[0]
        assert not sqrt_ok(np.array([lo if b < 1 else hi]))[0]
    n = np.repeat(x, x.size)
    d = np.tile(x, x.size)
    with np.errstate(invalid="ignore"):
        an, ad = np.abs(n), np.abs(d)
        r = F(2.0 ** 62)
        ok_doc = (ad >= F(1) / r) & (ad <= r) & (((an >= F(1) / r) & (an <= r)) | (an == 0))
        got = div_ok(n, d)
    assert not (got & ~ok_doc).any(), (n[got & ~ok_doc][:4], d[got & ~ok_doc][:4])
    assert got[ok_doc].all()
