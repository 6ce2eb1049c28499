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
