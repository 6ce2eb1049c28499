"""GPU parity tests of the tensor-core K1 (fft_mode 3, rtlsdr-airband_b200/csrc/k1_tc.cu): the configured bins' DFT as an
integer GEMM on wgmma with the raw bytes as the A operand.  Same gate as every other path (BASELINE.md §3): audio
within 1e-4 of the CPU oracle, identical squelch decisions and counters; plus the properties that do not need the oracle
at BASELINE sizes (twin devices bit-identical, agreement with the FP32 kernels, batching invariance)."""
import numpy as np
import pytest

import oracle_py as op
from airband_b200 import config as cm
from airband_b200 import lib
from airband_b200 import workloads as wl
from cases import CASES
from test_gpu_parity import TOL, compare, gate

pytestmark = pytest.mark.gpu


def _run_tc(cfg, raws, **kw):
    gres, geng = lib.demodulate_all(cfg, raws, fft_mode=3, **kw)
    for d in range(len(cfg.devices)):
        assert geng.fft_path(d) == 3, f"device {d} did not take the tensor-core path"
    return gres, geng


@pytest.mark.parametrize("name", ["am_u8", "s8_two_devices"])
def test_small_cases_match_oracle(name):
    cfg, raws = CASES[name]()
    ores, oorc = op.run_oracle(cfg, raws)
    gres, geng = _run_tc(cfg, raws)
    compare(cfg, raws, gres, geng, ores, oorc)
    geng.close()


def test_other_formats_fall_back_to_the_fp32_kernels():
    cfg, raws = CASES["nfm_s16"]()
    ores, oorc = op.run_oracle(cfg, raws)
    gres, geng = lib.demodulate_all(cfg, raws, fft_mode=3)
    assert geng.fft_path(0) == 2
    compare(cfg, raws, gres, geng, ores, oorc)
    geng.close()


def _small_tc(cfg, nb, **kw):
    raws = [wl.synth_iq(cfg, d, wl.samples_for_batches(cfg, d, nb), key_on_s=0.2, key_off_s=0.1, **kw) for d in range(len(cfg.devices))]
    ores, oorc = op.run_oracle(cfg, raws)
    gres, geng = _run_tc(cfg, raws)
    compare(cfg, raws, gres, geng, ores, oorc)
    geng.close()


def test_cfg1_shape():
    _small_tc(wl.cfg1(two_channels=True), 5)


def test_cfg2_shape_scaled_down():
    _small_tc(wl.cfg2(n_devices=3, n_channels=8), 3)


def test_cfg4_shape():
    _small_tc(wl.cfg4(), 2)


def test_cfg5_shape_scaled_down():
    _small_tc(wl.cfg5(n_devices=5, n_channels=8), 2)


@pytest.mark.parametrize("n", [256, 1024, 4096, 8192])
def test_other_fft_sizes(n):
    _small_tc(wl.cfg2(n_devices=1, n_channels=4, fft_size=n), 2)


@pytest.mark.parametrize("nch", [1, 3, 5, 12, 32])
def test_channel_counts(nch):
    """1..32 channels per device: padded output groups, scalar and vector stores, the 256-column MMA."""
    _small_tc(wl.cfg2(n_devices=2, n_channels=nch, fft_size=1024), 2)


def test_more_than_32_channels_uses_the_fp32_kernel():
    cfg = wl.cfg2(n_devices=1, n_channels=49, fft_size=1024)
    e = lib.Engine(cfg, fft_mode=3)
    assert e.fft_path(0) == 2
    e.close()


@pytest.mark.parametrize("digits", [3, 4])
@pytest.mark.parametrize("n,sfmt", [(512, cm.SFMT_S8), (2048, cm.SFMT_U8), (4096, cm.SFMT_U8)])
def test_bins_agree_with_the_full_spectrum_kernel(n, sfmt, digits, monkeypatch):
    monkeypatch.setenv("ABG_K1_TC_DIGITS", str(digits))
    sr = 2560000
    chans = [cm.make_channel(o, 0, sr, n, 8000, squelch_dbfs=-30.0, rawfile=True) for o in (-600000, -25000, 12500, 333000, 910000)]
    cfg = cm.Config(fft_size=n, wave_rate=8000, devices=[cm.Device(sample_rate=sr, sfmt=sfmt, centerfreq=0, channels=chans)])
    raws = [wl.synth_iq(cfg, 0, wl.samples_for_batches(cfg, 0, 2), key_off_s=0.0, amplitude=0.1)]
    (fw, fi, fa) = lib.demodulate_all(cfg, raws, fft_mode=1)[0][0]
    gres, geng = _run_tc(cfg, raws)
    (tw, ti, ta) = gres[0]
    assert np.array_equal(fa, ta) and np.any(fa == ord('*'))
    scale = np.abs(fi).max()
    assert scale > 1.0 and np.abs(fi - ti).max() / scale < 3e-6
    assert gate(fw, tw) <= 1e-5
    geng.close()


def test_streaming_pushes_of_odd_sizes():
    cfg, raws = CASES["am_u8"](n_batches=4)
    ores, oorc = op.run_oracle(cfg, raws)
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=3, fft_mode=3)
    assert e.fft_path(0) == 3
    rng = np.random.default_rng(3)
    pos, outs = 0, []
    r = raws[0]
    while pos < r.size or e.batches_available(0) > 0:
        if pos < r.size:
            step = 2 * int(rng.integers(1, 90000))
            e.push(0, r[pos:pos + step])
            pos += step
        e.run(-1)
        while True:
            got = e.fetch(0)
            if got is None:
                break
            outs.append(got)
    gw = np.concatenate([x[0] for x in outs], 1)
    assert gw.shape == ores[0][0].shape
    assert gate(gw, ores[0][0]) <= TOL
    assert np.array_equal(np.stack([x[2] for x in outs]), ores[0][2])
    e.close()


def test_uneven_devices_and_batches_per_run():
    cfg, _ = CASES["s8_two_devices"]()
    raws = [wl.synth_iq(cfg, i, wl.samples_for_batches(cfg, i, nb), key_on_s=0.1, key_off_s=0.05) for i, nb in enumerate((2, 5))]
    ores, oorc = op.run_oracle(cfg, raws)
    for nbmax in (1, 4):
        gres, geng = _run_tc(cfg, raws, max_batches_per_run=nbmax)
        compare(cfg, raws, gres, geng, ores, oorc)
        geng.close()


def test_set_bin_rebuilds_the_coefficient_table():
    cfg, _ = CASES["am_u8"]()
    raw = wl.synth_iq(cfg, 0, wl.samples_for_batches(cfg, 0, 6), key_on_s=0.11, key_off_s=0.07, amplitude=0.2)
    b0, b1 = cfg.devices[0].channels[0].bin, cfg.devices[0].channels[1].bin
    o = op.Oracle(cfg)
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=5, fft_mode=3)
    assert e.fft_path(0) == 3
    pos = 0
    for k, new_bin in enumerate((None, b1, b0)):
        need = wl.samples_for_batches(cfg, 0, 2 * (k + 1)) * 2
        if new_bin is not None:
            o.set_bin(0, 0, new_bin)
            e.set_bin(0, 0, new_bin)
        o.push(0, raw[pos:need]); e.push(0, raw[pos:need])
        pos = need
        assert o.run(2) == 2 and e.run(2) == 2
        ow, _, oa = o.fetch_all(0)
        outs = [e.fetch(0) for _ in range(2)]
        gw = np.concatenate([x[0] for x in outs], 1)
        assert np.array_equal(np.stack([x[2] for x in outs]), oa), k
        assert gate(gw, ow) <= TOL, (k, gate(gw, ow))
    e.close(); o.close()


@pytest.mark.parametrize("fill", [127, 0, 255], ids=["midscale", "rail_low", "rail_high"])
def test_constant_input(fill):
    cfg, raws = CASES["am_u8"]()
    raws = [np.full_like(r, fill) for r in raws]
    ores, oorc = op.run_oracle(cfg, raws)
    gres, geng = _run_tc(cfg, raws)
    assert np.isfinite(gres[0][0]).all()
    compare(cfg, raws, gres, geng, ores, oorc)
    geng.close()


def test_full_size_cfg2_properties_and_sampled_oracle_parity():
    """BASELINE.json configs[1] at FULL size through the tensor-core K1: twins bit-identical wherever their tiles ran,
    agreement with the output-pruned FP32 kernel inside the audio gate with identical decisions, 4-batch runs == 1-batch
    runs bit for bit, and the oracle on one device per distinct stream."""
    import bench
    cfg, _ = bench.make_workload("cfg2")
    nb = 4
    raws = bench.synth_streams(cfg, nb, n_unique=4)
    D = len(cfg.devices)
    res, eng = _run_tc(cfg, raws, max_batches_per_run=nb)
    opened = 0
    for d in range(D):
        w, _, a = res[d]
        assert w.shape == (8, nb * cfg.wave_batch)
        w0, _, a0 = res[d % 4]
        assert np.array_equal(w.view(np.uint32), w0.view(np.uint32)) and np.array_equal(a, a0), f"device {d} differs from its twin {d % 4}"
        opened += int((a != ord(' ')).sum())
    assert opened > 0
    res_p, eng_p = lib.demodulate_all(cfg, raws, max_batches_per_run=nb, fft_mode=2)
    res_one, eng_one = _run_tc(cfg, raws, max_batches_per_run=1)
    for d in range(D):
        assert np.array_equal(res[d][2], res_p[d][2])
        assert gate(res[d][0], res_p[d][0]) <= TOL
        assert np.array_equal(res[d][0].view(np.uint32), res_one[d][0].view(np.uint32)) and np.array_equal(res[d][2], res_one[d][2])
    sub = cm.Config(fft_size=cfg.fft_size, wave_rate=cfg.wave_rate, devices=cfg.devices[:4])
    ores, oorc = op.run_oracle(sub, raws[:4])
    for d in range(4):
        ow, _, oa = ores[d]
        assert np.array_equal(res[d][2], oa)
        assert gate(res[d][0], ow) <= TOL
        for c in range(8):
            gs, os_ = eng.stats(d, c), oorc.stats(d, c)
            assert gs.open_count == os_.open_count and gs.active_counter == os_.active_counter
    for e in (eng, eng_p, eng_one):
        e.close()
