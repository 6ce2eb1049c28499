"""History replay on the CPU: the C ABI and its ctypes mirror, transmission_replay's window arithmetic against the
definition in airband_b200.h, the gather kernel's build, and the squelch settling time the default lead-in rests on,
measured with the CPU oracle."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import oracle_py as op
from airband_b200 import config as cm
from airband_b200 import lib
from test_gpu_activity import quantize

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "rtlsdr-airband_b200", "build")
AGC = cm.AGC_EXTRA


# ---- ABI ----------------------------------------------------------------------------------------------------------------------
def test_header_symbols_and_argtypes():
    hdr = open(os.path.join(ROOT, "include", "airband_b200.h")).read()
    for s in ("abg_history_replay", "abg_debug_replay_time"):
        assert s in lib.SYMBOLS and re.search(r"ABG_API int %s\(" % s, hdr), s
    L = lib.load()
    assert L.abg_history_replay.argtypes == [C.c_void_p, C.c_int, C.POINTER(lib.CReplayJob)]
    assert L.abg_debug_replay_time.argtypes == [C.c_void_p, C.POINTER(C.c_float)]


def test_replay_job_layout_matches_the_header(tmp_path):
    fields = [f for f, _ in lib.CReplayJob._fields_]
    prog = "#include <stdio.h>\n#include <stddef.h>\n#include \"airband_b200.h\"\nint main(void) {\n"
    prog += "".join(f'    printf("%zu\\n", offsetof(abg_replay_job, {f}));\n' for f in fields)
    prog += '    printf("%zu\\n", sizeof(abg_replay_job));\n    return 0;\n}\n'
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text(prog)
    subprocess.run(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [getattr(lib.CReplayJob, f).offset for f in fields] + [C.sizeof(lib.CReplayJob)]


# ---- the gather kernel ------------------------------------------------------------------------------------------------------
def test_gather_kernel_builds_for_sm90a_without_spills_or_stack():
    path = os.path.join(BUILD, "replay.ptxas.log")
    assert os.path.exists(path), f"{path} missing: build the library first (make -C rtlsdr-airband_b200)"
    log = open(path).read()
    assert "sm_90a" in log and "abg_replay_gather_kernel" in log
    assert re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log) == [("0", "0")]
    assert re.findall(r"(\d+) bytes stack frame", log) == ["0"]


# ---- transmission_replay ------------------------------------------------------------------------------------------------------
def _cfg():
    ch = cm.make_channel(120_100_000, 120_000_000, 2048000, 2048, 8000)
    return cm.Config(fft_size=2048, wave_rate=8000, devices=[cm.Device(sample_rate=2048000, sfmt=cm.SFMT_U8, centerfreq=120_000_000,
                                                                       channels=[ch])])


def reads(cfg, job):
    """The samples [S, end) the definition's fresh engine reads for a job."""
    B, hop, N = cfg.wave_batch, cfg.hop(0), cfg.fft_size
    S = job["first_batch"] * B * hop
    return S, S + (AGC + job["n_batches"] * B) * hop + N - hop


def test_transmission_replay_window():
    cfg = _cfg()
    B, hop, N = cfg.wave_batch, cfg.hop(0), cfg.fft_size
    assert (B, hop) == (1000, 256)
    tx = dict(freq_hz=120_033_000.0, first_frame=AGC + 20 * B + 300, last_frame=AGC + 23 * B + 10)
    big = (0, 10 ** 12)
    # lead-in: the latest batch whose first frame is at least lead_s of frames before the first frame
    job = lib.transmission_replay(tx, cfg, 0, big, lead_s=0.5)
    assert job["first_batch"] == 16 and job["n_batches"] == 8  # batches 16 .. 23
    assert tx["first_frame"] - (AGC + 16 * B) >= 0.5 * 8000 > tx["first_frame"] - (AGC + 17 * B)
    assert AGC + 23 * B <= tx["last_frame"] < AGC + 24 * B
    ch = job["channels"][0]
    assert ch.bin == cm.calc_bin(120_033_000, 120_000_000, 2048000, 2048) and ch.modulation == cm.MOD_AM and ch.dm_dphi == 0
    nfm = lib.transmission_replay(tx, cfg, 0, big, lead_s=0.0, modulation=cm.MOD_NFM)["channels"][0]
    assert nfm.modulation == cm.MOD_NFM and nfm.dm_dphi == cm.calc_dm_dphi(120_033_000, 120_000_000, 2048000, 8000)
    assert lib.transmission_replay(tx, cfg, 0, big, lead_s=0.0)["first_batch"] == 20
    # the default lead-in is the measured settling time
    d = lib.transmission_replay(tx, cfg, 0, big)
    assert d["first_batch"] == 20 - lib.REPLAY_SETTLE_BATCHES
    # clipped to the history's start: the first batch whose samples it holds
    first = 18 * B * hop - 1
    job = lib.transmission_replay(tx, cfg, 0, (first, 10 ** 12), lead_s=0.5)
    assert job["first_batch"] == 18 and reads(cfg, job)[0] >= first and job["first_batch"] + job["n_batches"] == 24
    # clipped at its end: the last frame's tail, fft_size - hop samples into the next batch, must be in the history
    s_end, e_end = reads(cfg, dict(first_batch=16, n_batches=8))
    job = lib.transmission_replay(tx, cfg, 0, (0, e_end), lead_s=0.5)
    assert job["n_batches"] == 8 and reads(cfg, job)[1] == e_end
    job = lib.transmission_replay(tx, cfg, 0, (0, e_end - 1), lead_s=0.5)
    assert job["n_batches"] == 7 and reads(cfg, job)[1] <= e_end - 1
    assert reads(cfg, dict(first_batch=16, n_batches=8))[1] - (AGC + 24 * B) * hop == N - hop


def test_transmission_replay_raises_when_nothing_fits():
    cfg = _cfg()
    B, hop = cfg.wave_batch, cfg.hop(0)
    tx = dict(freq_hz=120_000_000.0, first_frame=AGC + 20 * B + 300, last_frame=AGC + 23 * B + 10)
    with pytest.raises(ValueError, match="nothing"):
        lib.transmission_replay(tx, cfg, 0, (24 * B * hop + 1, 10 ** 12))  # history starts after it
    with pytest.raises(ValueError, match="nothing"):
        lib.transmission_replay(tx, cfg, 0, (0, (AGC + 16 * B) * hop), lead_s=0.5)  # ends before its first batch
    with pytest.raises(ValueError, match="nothing"):
        lib.transmission_replay(tx, cfg, 0, (0, 0))  # empty
    with pytest.raises(ValueError):
        lib.transmission_replay(tx, cfg, 0, (0, 10 ** 12), lead_s=-1.0)


# ---- the lead-in ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [1, 7])
def test_default_lead_in_covers_the_squelch_settling_time(seed):
    """A fresh AM channel on the test signals' noise (U8, 2.048 Msps, fft 2048, complex noise of 0.01 full scale per
    component), run by the CPU oracle: its noise level starts from the floor of 5.0 and is within 10 % of its steady value
    (the median of batches 24 .. 31) from batch REPLAY_SETTLE_BATCHES - 1 on, i.e. after REPLAY_SETTLE_BATCHES batches."""
    SR, W, n, cf = 2048000, 8000, 2048, 120_000_000
    ch = cm.make_channel(cf + 77 * (SR // n), cf, SR, n, W)
    cfg = cm.Config(fft_size=n, wave_rate=W, devices=[cm.Device(sample_rate=SR, sfmt=cm.SFMT_U8, centerfreq=cf, channels=[ch])])
    B, hop, nb = cfg.wave_batch, cfg.hop(0), 32
    rng = np.random.default_rng(seed)
    m = (AGC + nb * B) * hop + n
    raw = quantize(rng.normal(0, 0.01, m) + 1j * rng.normal(0, 0.01, m), cm.SFMT_U8, 0.0)
    o = op.Oracle(cfg)
    o.push(0, raw)
    lv = []
    while o.run(1) > 0:
        o.fetch(0)
        lv.append(o.stats(0, 0).noise_level)
    o.close()
    lv = np.asarray(lv)
    assert lv.size == nb
    steady = np.median(lv[24:])
    settled = np.abs(lv / steady - 1.0) <= 0.1
    first = next(i for i in range(nb) if settled[i:].all())
    assert lv[0] > 3 * steady  # it does start far above the noise
    assert first + 1 <= lib.REPLAY_SETTLE_BATCHES
    assert lib.REPLAY_SETTLE_BATCHES * B / W == 0.75
