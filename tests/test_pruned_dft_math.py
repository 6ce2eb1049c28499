"""The algebra behind the output-pruned K1 (rtlsdr-airband_b200/csrc/k1_pruned.cu), checked with numpy: with N = R1*M1,
X[b] = sum_{c<M1} W_N^(c*b) * Y_c[b mod R1], Y_c = R1-point DFT of the column x[c + M1*n1]; the coefficient of column
c = PAIR*l + 64*m + p factors into a per-lane part W^(PAIR*l*b) and a warp-uniform part W^((64*m+p)*b); and the window can be
folded into the first radix-2 stage of the column FFT.  The CUDA kernel itself is tested frame by frame against float64 on
the GPU (tests/test_gpu_k1_fp32.py), over every plan class the last test here enumerates."""
import os
import re

import numpy as np
import pytest


@pytest.mark.parametrize("n,r1", [(2048, 8), (2048, 16), (512, 8), (8192, 16), (256, 8)])
def test_column_split_reproduces_selected_bins(n, r1):
    rng = np.random.default_rng(n + r1)
    x = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    m1 = n // r1
    ref = np.fft.fft(x)
    cols = x.reshape(r1, m1)                 # cols[n1, c] = x[c + M1*n1]
    y = np.fft.fft(cols, axis=0)             # y[k1, c] = Y_c[k1]
    w = np.exp(-2j * np.pi * np.arange(n) / n)
    for b in rng.integers(0, n, 12):
        c = np.arange(m1)
        got = np.sum(w[(c * b) % n] * y[b % r1, c])
        assert abs(got - ref[b]) <= 1e-9 * max(1.0, abs(ref[b]))


def test_lane_and_warp_uniform_factors():
    n, r1 = 2048, 8
    m1, ncol, pair = n // r1, (n // 32) // r1, 2
    w = np.exp(-2j * np.pi * np.arange(n) / n)
    for b in (0, 1, 205, 1023, 2047):
        for lane in (0, 1, 17, 31):
            for j in range(ncol):
                col = pair * lane + (pair * 32) * (j // pair) + (j % pair)       # column owned by (lane, j)
                assert col < m1
                coff = (pair * 32) * (j // pair) + (j % pair)                     # part that does not depend on the lane
                lhs = w[(col * b) % n]
                rhs = w[((pair * lane) * b) % n] * w[(coff * b) % n]
                assert abs(lhs - rhs) < 1e-12
    # every column is owned exactly once
    owned = sorted(pair * l + (pair * 32) * (j // pair) + (j % pair) for l in range(32) for j in range(ncol))
    assert owned == list(range(m1))


def test_window_folds_into_the_first_radix2_stage():
    r1 = 8
    rng = np.random.default_rng(1)
    x = rng.standard_normal(r1) + 1j * rng.standard_normal(r1)
    win = rng.random(r1)
    ref = np.fft.fft(x * win)
    # first DIT stage pairs sample n1 with n1 + R1/2: a' = xa*wa + xb*wb, b' = xa*wa - xb*wb; then an R1/2-point DFT of
    # the sums gives the even bins and one of the (twiddled) differences the odd bins
    h = r1 // 2
    s = x[:h] * win[:h] + x[h:] * win[h:]
    d = (x[:h] * win[:h] - x[h:] * win[h:]) * np.exp(-2j * np.pi * np.arange(h) / r1)
    assert np.allclose(np.fft.fft(s), ref[0::2]) and np.allclose(np.fft.fft(d), ref[1::2])


# ---- the kernel's plan space -------------------------------------------------------------------------------------------
# k1_pruned_kernel<LOGN, SFMT, R1, GELEM> picks its code paths from template arithmetic on N, R1 and GELEM, and the launcher
# from the group's largest channel count.  The constants are read from the kernel source, so that moving a boundary there
# fails here until the GPU cases below (tests/test_gpu_k1_fp32.py) follow it.
PR_SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rtlsdr-airband_b200", "csrc", "k1_pruned.cu")


def pruned_constants():
    with open(PR_SRC) as f:
        src = f.read()
    maxch = int(re.search(r"constexpr int PR_MAXCH = (\d+);", src).group(1))
    small_n, small_r1, thresh, hi_r1, lo_r1 = (int(x) for x in re.search(
        r"if \(fft_size <= (\d+)\) return (\d+);\s*return max_channels > (\d+) \? (\d+) : (\d+);", src).groups())
    ge_env, ge_alt, ge_default = (int(x) for x in re.search(r"ge = \(e && atoi\(e\) == (\d+)\) \? (\d+) : (\d+);", src).groups())
    assert ge_env == ge_alt
    return dict(maxch=maxch, small_n=small_n, small_r1=small_r1, thresh=thresh, hi_r1=hi_r1, lo_r1=lo_r1,
                gelem=(ge_default, ge_alt))


def pruned_plan(n, max_channels, gelem):
    """The kernel's template constants and the launcher's pass count for one launch group, as k1_pruned.cu computes them."""
    k = pruned_constants()
    r1 = k["small_r1"] if n <= k["small_n"] else (k["hi_r1"] if max_channels > k["thresh"] else k["lo_r1"])   # pr_radix
    e = n // 32
    ncol = e // r1
    pair = 2 if ncol >= 2 else 1
    gcol = (gelem // r1 if gelem // r1 >= pair else pair) if ncol * r1 > gelem else ncol
    cm = max(4, min(k["maxch"], (max_channels + 3) & ~3))                                                    # pr_cm
    passes = -(-max_channels // k["maxch"])
    return dict(R1=r1, E=e, NCOL=ncol, PAIR=pair, GCOL=gcol, NGRP=ncol // gcol, CM=cm, passes=passes)


def plan_class(n, max_channels, gelem):
    """(R1, columns per lane pair or single, several register groups, channel passes): one code path of the kernel each."""
    p = pruned_plan(n, max_channels, gelem)
    return p["R1"], p["PAIR"], p["NGRP"] > 1, p["passes"]


def reduction_class(nch):
    """(NVP, reduction rounds) of the lane reduction for a device with nch channels in one pass."""
    nv = 2 * nch
    nvp = 32 if nv > 16 else 16 if nv > 8 else 8 if nv > 4 else 4 if nv > 2 else 2
    return nvp, -(-nv // nvp)


def device_reductions(counts, maxch):
    return {reduction_class(min(maxch, c - ch0)) for c in counts for ch0 in range(0, c, maxch)}


# The GPU cases of the pruned kernel: name -> (fft_size, hop in samples, format, fullscale (0 = default), channel counts of the
# group's devices, GELEM, the class they must fall into).  Odd hops put 8-bit frames on the unaligned load every other frame.
U8, S8, S16, F32 = 1, 2, 3, 4
PRUNED_CASES = {
    "256_u8_odd_hop": (256, 313, U8, 0, (1, 2, 3), 64, (8, 1, False, 1)),
    "256_s16_two_passes": (256, 320, S16, 32768.0, (33, 5), 64, (8, 1, False, 2)),
    "256_f32_three_passes": (256, 320, F32, 1.0, (70, 9, 1), 64, (8, 1, False, 3)),
    "512_u8_12ch": (512, 320, U8, 0, (1, 5, 12), 64, (8, 2, False, 1)),
    "512_s8_13ch": (512, 320, S8, 0, (13, 2), 64, (16, 1, False, 1)),
    "512_s16_49ch": (512, 320, S16, 3000.0, (49, 3), 64, (16, 1, False, 2)),
    "512_u8_odd_hop_70ch": (512, 313, U8, 0, (70, 17), 64, (16, 1, False, 3)),
    "1024_f32_12ch": (1024, 320, F32, 2048.0, (12, 1), 64, (8, 2, False, 1)),
    "1024_u8_odd_hop_32ch": (1024, 313, U8, 0, (17, 32, 5), 64, (16, 2, False, 1)),
    "2048_s16_33ch": (2048, 320, S16, 32768.0, (33, 9), 64, (16, 2, False, 2)),
    "2048_u8_70ch": (2048, 320, U8, 0, (70, 2), 64, (16, 2, False, 3)),
    "4096_u8_odd_hop_9ch": (4096, 313, U8, 0, (1, 3, 9), 64, (8, 2, True, 1)),
    "4096_s8_32ch": (4096, 320, S8, 0, (32, 1), 64, (16, 2, True, 1)),
    "8192_f32_49ch": (8192, 320, F32, 1.0, (49, 17), 64, (16, 2, True, 2)),
    "8192_s16_70ch": (8192, 320, S16, 3000.0, (70, 5), 64, (16, 2, True, 3)),
    "2048_u8_gelem32": (2048, 320, U8, 0, (2, 9), 32, (8, 2, True, 1)),
    "2048_s16_gelem32_33ch": (2048, 320, S16, 32768.0, (33, 17), 32, (16, 2, True, 2)),
}
PLAN_SIZES = (256, 512, 1024, 2048, 4096, 8192)


def test_pruned_cases_cover_the_plan_space():
    """Every (R1, PAIR, register groups, passes) class and every lane-reduction width the kernel has over N 256..8192, 1..70
    channels and both GELEM settings is run by one of the GPU cases, each case falls into the class it names, and the
    GELEM = 32 cases reach a group count that GELEM = 64 does not give at the same size."""
    k = pruned_constants()
    assert k["gelem"] == (64, 32)
    space, reductions = set(), set()
    for n in PLAN_SIZES:
        for ch in range(1, 71):
            for ge in k["gelem"]:
                p = pruned_plan(n, ch, ge)
                assert p["E"] >= p["R1"] and p["NCOL"] % p["GCOL"] == 0 and p["GCOL"] % p["PAIR"] == 0, (n, ch, ge, p)
                assert p["GCOL"] * p["R1"] <= max(ge, p["PAIR"] * p["R1"]) and p["CM"] % 4 == 0, (n, ch, ge, p)
                space.add(plan_class(n, ch, ge))
                reductions |= device_reductions([ch], k["maxch"])
    covered, reached = set(), set()
    for name, (n, hop, sfmt, fs, counts, ge, cls) in PRUNED_CASES.items():
        assert plan_class(n, max(counts), ge) == cls, (name, plan_class(n, max(counts), ge))
        covered.add(cls)
        reached |= device_reductions(counts, k["maxch"])
    assert covered == space, sorted(space - covered)
    assert reached == reductions, sorted(reductions - reached)
    assert {c[3] for c in space} == {1, 2, 3} and {r[0] for r in reductions} == {2, 4, 8, 16, 32}
    g32 = [(n, max(c)) for n, _, _, _, c, ge, _ in PRUNED_CASES.values() if ge == 32]
    assert g32 and all(pruned_plan(n, ch, 32)["NGRP"] != pruned_plan(n, ch, 64)["NGRP"] for n, ch in g32)
    # the boundaries themselves: the largest channel count on R1 = 8 and the smallest on R1 = 16, one and two passes
    assert {max(c[4]) for c in PRUNED_CASES.values() if c[0] > k["small_n"]} >= {k["thresh"], k["thresh"] + 1, k["maxch"], k["maxch"] + 1}
    assert {c[2] for c in PRUNED_CASES.values()} == {U8, S8, S16, F32}
    assert {c[1] % 2 for c in PRUNED_CASES.values() if c[2] == U8} == {0, 1}
