"""The tensor-core K1 (rtlsdr-airband_b200/csrc/k1_tc.cu) as the compiler built it and as its stage ring runs.

CPU: the `-Xptxas -v` logs the Makefile writes next to the objects show every k1_tc_kernel instantiation issuing its
wgmma without injected warpgroup waits (ptxas C7519 serialises consecutive MMAs), without spills, and with a register
count that leaves room for four of K2's one-warp CTAs on the same SM (the K1/K2 overlap the engine relies on).
GPU: devices with alternating channel plans (two coefficient tables) and frame counts that are no multiple of the
128-frame tile, checked against the CPU oracle.  Runs of 4 batches are ~33 tiles per device, so every launch has 260 to
1060 tiles for 132 persistent CTAs: each CTA's stage ring wraps many times across tile, device and table changes, with
one pair per stage (fft 2048), six short pairs per stage (fft 512) and pairs cut into several stages (fft 8192)."""
import os
import re

import pytest

from airband_b200 import config as cm
from airband_b200 import lib
from airband_b200 import workloads as wl

BUILD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rtlsdr-airband_b200", "build")


def _ptxas(name):
    path = os.path.join(BUILD, f"{name}.ptxas.log")
    assert os.path.exists(path), f"{path} missing: build the library first (make -C rtlsdr-airband_b200)"
    with open(path) as f:
        return f.read()


def _per_kernel(log, pattern):
    """{mangled kernel name: (registers, spill bytes)} for the entry functions matching `pattern`."""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"(?:Compiling entry function|Function properties for) '(\w+)'", line)
        if m:
            cur = m.group(1) if re.search(pattern, m.group(1)) else None
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            regs, _ = out.get(cur, (None, 0))
            out[cur] = (regs, int(m.group(1)) + int(m.group(2)))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            _, spill = out.get(cur, (None, 0))
            out[cur] = (int(m.group(1)), spill)
    return out


def test_no_injected_warpgroup_waits():
    log = _ptxas("k1_tc")
    for code in ("C7519", "C7520"):  # arrive injected / MMAs serialised by an arrive in a divergent path
        assert code not in log, [ln for ln in log.splitlines() if code in ln][:3]


def test_no_spills_and_room_for_k2():
    k1 = _per_kernel(_ptxas("k1_tc"), r"k1_tc_kernel")
    assert len(k1) == 64, sorted(k1)  # ND 3/4 x 8 output widths x U8/S8 x one / several column pairs per stage
    for name, (regs, spill) in k1.items():
        assert regs is not None and spill == 0, (name, regs, spill)
    k2 = _per_kernel(_ptxas("k2_demod"), r"k2_demod_kernelILi1ELb0E")
    assert len(k2) == 1, sorted(k2)
    k2_regs = next(iter(k2.values()))[0]
    # the 8-channel instantiations (every cfg2 / cfg5 device): 384 K1 threads + four one-warp K2 CTAs in one register file
    for name, (regs, _) in k1.items():
        if re.search(r"k1_tc_kernelILi4ELi16ELb[01]ELb[01]E", name):
            assert regs * 384 + 4 * 32 * k2_regs <= 65536, (name, regs, k2_regs)


def _mixed(fft_size, n_devices, n_channels):
    """Even devices: n_channels on a 25 kHz raster; odd devices: n_channels - 3 on a 40 kHz raster (another table)."""
    sr, w, cf = 2560000, 8000, 120000000
    devs = []
    for d in range(n_devices):
        offs = wl._raster(n_channels, 25000) if d % 2 == 0 else wl._raster(n_channels - 3, 40000)
        chans = [cm.make_channel(cf + o, cf, sr, fft_size, w, squelch_dbfs=-30.0) for o in offs]
        devs.append(cm.Device(sample_rate=sr, sfmt=cm.SFMT_U8, centerfreq=cf, channels=chans))
    return cm.Config(fft_size=fft_size, wave_rate=w, devices=devs)


@pytest.mark.gpu
@pytest.mark.parametrize("fft_size,n_devices,n_channels", [(2048, 32, 8), (512, 32, 8), (8192, 8, 32)])
def test_ring_across_tiles_devices_and_tables(fft_size, n_devices, n_channels):
    import oracle_py as op
    from test_gpu_parity import compare

    cfg = _mixed(fft_size, n_devices, n_channels)
    plan = lib.tc_table(fft_size, cm.SFMT_U8, 640, [1] * n_channels)[0]
    assert plan["eligible"] and plan["smem_bytes"] <= 200 * 1024
    if fft_size == 8192:
        assert plan["KBS"] < -(-plan["K"] // 640)  # a column pair's k-steps are cut into several stages
    raws = [wl.synth_iq(cfg, d, wl.samples_for_batches(cfg, d, 5 - d % 2), key_on_s=0.2, key_off_s=0.1) for d in range(n_devices)]
    ores, oorc = op.run_oracle(cfg, raws)
    gres, geng = lib.demodulate_all(cfg, raws, max_batches_per_run=4, fft_mode=3)
    for d in range(n_devices):
        assert geng.fft_path(d) == 3
    compare(cfg, raws, gres, geng, ores, oorc)
    geng.close()
