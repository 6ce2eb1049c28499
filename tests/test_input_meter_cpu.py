"""CPU checks of the input level meter: the ctypes mirror of abg_input_levels against the header, lib.input_levels on
hand-built readings, the level-to-bin arithmetic the kernel relies on for 8-bit formats, and the kernel's `-Xptxas -v`
log (no spills)."""
import ctypes as C
import os
import re

import numpy as np

from airband_b200 import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "rtlsdr-airband_b200", "build")
f32 = np.float32


def test_struct_mirrors_the_header():
    hdr = open(os.path.join(ROOT, "include", "airband_b200.h")).read()
    body = re.search(r"typedef struct abg_input_levels \{(.*?)\} abg_input_levels;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    decls = [d.strip() for d in body.split(";") if d.strip()]
    names = [re.sub(r"\[.*?\]", "", d.split()[-1]) for d in decls]
    assert names == [f for f, _ in lib.CInputLevels._fields_]
    types = {"uint64_t": 8, "double": 8, "float": 4, "uint32_t": 4}
    size = 0
    for d, (name, ct) in zip(decls, lib.CInputLevels._fields_):
        n = int(np.prod([int(x) for x in re.findall(r"\[(\d+)\]", d)] or [1]))
        assert types[d.split()[0]] * n == C.sizeof(ct), name
        assert getattr(lib.CInputLevels, name).offset == size, name  # naturally aligned: no padding anywhere
        size += C.sizeof(ct)
    assert C.sizeof(lib.CInputLevels) == size == 2112


def test_8bit_codes_have_bins_of_their_own():
    """The kernel counts U8 code c in bin c and S8 code c in bin c + 128: the definition's float32 arithmetic agrees."""
    c = np.arange(256, dtype=np.float32)
    u8 = (c - f32(127.5)) / f32(127.5)
    s8 = (c - f32(128)) / f32(128)
    for v in (u8, s8):
        assert np.array_equal(np.clip(np.floor((v + f32(1)) * f32(128)), 0, 255).astype(int), np.arange(256))
    # the U8 peak: (c - 127.5f) is exactly u / 2 with u = |2c - 255|
    u = np.abs(2 * np.arange(256) - 255).astype(np.float32)
    assert np.array_equal(np.abs(u8), (f32(0.5) * u) / f32(127.5))


def _reading(vi, vq, hist=None):
    vi, vq = np.asarray(vi, np.float64), np.asarray(vq, np.float64)
    if hist is None:
        hist = np.zeros((2, 256), np.uint32)
    return dict(batch_seq=0, n_samples=vi.size, sum=np.array([vi.sum(), vq.sum()]), sum_sq=np.array([(vi * vi).sum(), (vq * vq).sum()]),
                sum_iq=float((vi * vq).sum()), peak=np.array([np.abs(vi).max(), np.abs(vq).max()], np.float32), hist=hist)


def test_input_levels_formulas():
    n = 4096
    t = 2 * np.pi * 17 * np.arange(n) / n  # whole cycles: exact means
    a, dc, g_db, phi = 0.5, (0.01, -0.02), 1.0, 3.0
    vi = dc[0] + a * np.cos(t)
    vq = dc[1] + a * 10 ** (-g_db / 20) * np.sin(t + np.radians(phi))
    hist = np.zeros((2, 256), np.uint32)
    hist[0, [0, 5, 255]] = [3, n - 10, 7]
    hist[1, 128] = n
    lv = lib.input_levels(_reading(vi, vq, hist))
    assert np.allclose(lv["dc_offset"], dc, atol=1e-12)
    assert abs(lv["imbalance_db"] - g_db) < 1e-9
    assert abs(lv["phase_skew_deg"] - phi) < 1e-9
    assert np.allclose(lv["mean_square_dbfs"], 10 * np.log10([np.mean(vi ** 2), np.mean(vq ** 2)]))
    assert np.array_equal(lv["full_scale_fraction"], [10 / n, 0.0])
    assert list(lv["codes_in_use"]) == [3, 1]
    # a full-scale sine reads -3.01 dBFS
    full = lib.input_levels(_reading(np.cos(t), np.sin(t)))
    assert np.allclose(full["mean_square_dbfs"], 10 * np.log10(0.5)) and abs(full["mean_square_dbfs"][0] + 3.0103) < 1e-4
    assert abs(full["imbalance_db"]) < 1e-9 and abs(full["phase_skew_deg"]) < 1e-9


def test_kernel_has_no_spills():
    path = os.path.join(BUILD, "input_meter.ptxas.log")
    assert os.path.exists(path), f"{path} missing: build the library first (make -C rtlsdr-airband_b200)"
    log = open(path).read()
    entries = re.findall(r"Compiling entry function '(\w+)'", log)
    assert len(entries) == 1 and "abg_input_meter_kernel" in entries[0], entries
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert spills and all(int(a) == 0 and int(b) == 0 for a, b in spills), spills
    regs = [int(r) for r in re.findall(r"Used (\d+) registers", log)]
    assert regs and max(regs) * 256 * 3 <= 65536, regs  # three 256-thread CTAs per SM
