"""The four batch monitors together on the GPU (-m gpu): band spectrum, carrier meter, input level meter and sub-band
outputs share one host-side launch path in the engine.  For every on/off subset of them, on a streamed run with
compaction and on resident runs: each monitor that is on adds exactly one upload and one launch per run, the kernel
times and queues of the others stay empty, every monitor reads the same bits as when it is on alone, and the audio,
I/Q, squelch flags and squelch statistics are the bits of the run with every monitor off."""
import itertools

import numpy as np
import pytest

from airband_b200 import config as cm
from airband_b200 import lib
from cases import CASES

pytestmark = pytest.mark.gpu
STAT_FIELDS = [f for f, _ in cm.CSquelchStats._fields_]
MONITORS = ("spectrum", "carrier", "input_meter", "subband")
SUBSETS = [frozenset(s) for n in range(len(MONITORS) + 1) for s in itertools.combinations(MONITORS, n)]
SB_OUTPUTS = {0: (1000.0, 16, 255), 3: (-20000.0, 7, 64)}  # k: (offset_hz, decimation, L)


def switch_on(e, cfg, monitors):
    sr = cfg.devices[0].sample_rate
    if "spectrum" in monitors:
        e.spectrum_configure(0, 3)
    if "carrier" in monitors:
        e.carrier_configure(0, True)
    if "input_meter" in monitors:
        e.input_meter_configure(0, True)
    if "subband" in monitors:
        for k, (off, dec, L) in SB_OUTPUTS.items():
            e.subband_configure(0, k, off, dec, lib.subband_lowpass(L, 0.4 * sr / dec, sr, 60.0))


def kernel_times(e):
    return {"spectrum": e.spectrum_time(), "carrier": e.carrier_time(), "input_meter": e.input_meter_time(),
            "subband": e.subband_time()}


def fetch_monitors(e):
    """Every queued monitor reading of device 0, as bits."""
    got = {m: [] for m in MONITORS}
    while (s := e.fetch_spectrum(0)) is not None:
        got["spectrum"].append((s[0].view(np.uint32).copy(), s[1], s[2]))
    while (c := e.fetch_carrier(0)) is not None:
        got["carrier"].append((c[0].view(np.uint64).copy(), c[1].view(np.uint32).copy(), c[2]))
    while (r := e.fetch_input_levels(0)) is not None:
        got["input_meter"].append((r["batch_seq"], r["n_samples"], r["hist"].copy(), r["peak"].view(np.uint32).copy(),
                                   r["sum"].view(np.uint64).copy(), r["sum_sq"].view(np.uint64).copy(),
                                   np.float64(r["sum_iq"]).view(np.uint64)))
    for k in range(lib.SUBBAND_MAX):
        while (x := e.fetch_subband(0, k)) is not None:
            got["subband"].append((k, x[0].view(np.uint64).copy(), x[1], x[2]))
    return got


def drive(cfg, raw, monitors):
    """Stream `raw` in thirds of a batch through a buffer of 3 batches (so it compacts), then resident runs."""
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=3)
    switch_on(e, cfg, monitors)
    res = dict(audio=[], runs=[], launches=[], readings={m: [] for m in MONITORS}, times=[])
    step = 2 * (cfg.wave_batch * cfg.hop(0) // 3 + 1)
    pos = 0
    while pos < raw.size or e.batches_available(0):
        if pos < raw.size:
            e.push(0, raw[pos:pos + step])
            pos += step
        l0 = e.launch_count()
        n = e.run(-1)
        if n == 0:
            assert e.launch_count() == l0
            continue
        e.sync()
        res["runs"].append(n)
        res["launches"].append(e.launch_count() - l0)
        res["times"].append(kernel_times(e))
        while (g := e.fetch(0)) is not None:
            res["audio"].append((g[0].view(np.uint32).copy(), g[1].view(np.uint64).copy(), g[2].copy()))
        for m, got in fetch_monitors(e).items():
            res["readings"][m] += got
    res["stats"] = [tuple(getattr(e.stats(0, c), f) for f in STAT_FIELDS) for c in range(len(cfg.devices[0].channels))]
    e.resident_load(0, raw[:e.resident_bytes_needed(0)])
    res["resident_launches"] = []
    for _ in range(3):
        l0 = e.launch_count()
        assert e.run_resident(2) == 2
        e.sync()
        res["resident_launches"].append(e.launch_count() - l0)
        res["resident_times"] = kernel_times(e)
    res["resident_queued"] = {m: len(got) for m, got in fetch_monitors(e).items()}
    res["resident_audio"] = e.fetch(0)
    e.close()
    return res


@pytest.fixture(scope="module")
def runs():
    cfg, raws = CASES["am_u8"](n_batches=6)
    assert raws[0].size > 2 * 3 * cfg.wave_batch * cfg.hop(0)  # more than the buffer holds: compaction happens
    return {s: drive(cfg, raws[0], s) for s in SUBSETS}


@pytest.mark.parametrize("subset", SUBSETS, ids=lambda s: "+".join(m for m in MONITORS if m in s) or "none")
def test_every_subset_of_monitors(runs, subset):
    off, got = runs[frozenset()], runs[subset]
    # the same runs; each monitor on adds one upload and one launch to each of them, streamed or resident
    assert got["runs"] == off["runs"] and len(off["runs"]) > 2
    assert got["launches"] == [n + 2 * len(subset) for n in off["launches"]]
    assert got["resident_launches"] == [n + 2 * len(subset) for n in off["resident_launches"]]
    # kernel times and readings only from the monitors that are on
    for times in got["times"] + [got["resident_times"]]:
        assert {m for m, ms in times.items() if ms > 0.0} == set(subset), times
        assert all(ms == 0.0 for m, ms in times.items() if m not in subset)
    for m in MONITORS:
        assert bool(got["readings"][m]) == (m in subset), m
        if m in subset:  # bitwise what it reads alone
            alone = runs[frozenset([m])]["readings"][m]
            assert len(got["readings"][m]) == len(alone)
            for a, b in zip(got["readings"][m], alone):
                assert all(np.array_equal(x, y) for x, y in zip(a, b)), m
    if "subband" in subset:
        assert {k for k, *_ in got["readings"]["subband"]} == set(SB_OUTPUTS)
    # resident runs queue nothing
    assert all(n == 0 for n in got["resident_queued"].values()) and got["resident_audio"] is None
    # the rest of the engine's output is bitwise that of the run with every monitor off
    assert len(got["audio"]) == len(off["audio"]) == sum(off["runs"])
    for a, b in zip(got["audio"], off["audio"]):
        assert all(np.array_equal(x, y) for x, y in zip(a, b))
    assert got["stats"] == off["stats"]
