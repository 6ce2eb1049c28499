"""The seven batch monitors together on the GPU (-m gpu): band spectrum, carrier meter, input level meter, sub-band
outputs, tone meter, activity detector and I/Q history share one host-side path in the engine.  For every on/off subset
of them, on a streamed run with compaction and on resident runs: each monitor that is on adds exactly one upload and one
launch per run, the kernel times and readings of the others stay empty, every monitor reads the same bits as when it is
on alone, and the audio, I/Q, squelch flags and squelch statistics are the bits of the run with every monitor off.  And
a failed allocation of a monitor leaves the engine as it was."""
import itertools

import numpy as np
import pytest

from airband_b200 import config as cm
from airband_b200 import lib
from cases import CASES

pytestmark = pytest.mark.gpu
STAT_FIELDS = [f for f, _ in cm.CSquelchStats._fields_]
SB_OUTPUTS = {0: (1000.0, 16, 255), 3: (-20000.0, 7, 64)}  # k: (offset_hz, decimation, L)
ACT_THR = 40.0  # on the band spectrum's scale: am_u8's carriers reach it, its noise does not
HISTORY_BATCHES = 3


def subband_on(e, cfg):
    sr = cfg.devices[0].sample_rate
    for k, (off, dec, L) in SB_OUTPUTS.items():
        e.subband_configure(0, k, off, dec, lib.subband_lowpass(L, 0.4 * sr / dec, sr, 60.0))


def drain(fetch):
    """Every reading fetch() returns before None."""
    got = []
    while (x := fetch()) is not None:
        got.append(x)
    return got


def subband_readings(e):
    return [(k, x[0].view(np.uint64).copy(), x[1], x[2]) for k in range(lib.SUBBAND_MAX) for x in drain(lambda: e.fetch_subband(0, k))]


def activity_key(r):
    """A truncated reading stores an unspecified subset of its pieces (airband_b200.h): only its count is compared."""
    whole = r["n_total"] <= len(r["pieces"])
    return (r["batch_seq"], r["n_total"], np.array(r["settings"]), r["pieces"].view(np.uint8).copy() if whole else np.zeros(0, np.uint8))


def history_readings(e):
    """The range the history holds and its bytes, or nothing while it is empty."""
    first, end = e.history_range(0)
    return [(first, end, e.history_raw(0, first, end - first).copy())] if end > first else []


# per monitor: switch it on for device 0, every queued reading of device 0 as bits, its kernel time in the latest run
MONITORS = {
    "spectrum": (lambda e, cfg: e.spectrum_configure(0, 3),
                 lambda e: [(s[0].view(np.uint32).copy(), s[1], s[2]) for s in drain(lambda: e.fetch_spectrum(0))],
                 lambda e: e.spectrum_time()),
    "carrier": (lambda e, cfg: e.carrier_configure(0, True),
                lambda e: [(c[0].view(np.uint64).copy(), c[1].view(np.uint32).copy(), c[2]) for c in drain(lambda: e.fetch_carrier(0))],
                lambda e: e.carrier_time()),
    "input_meter": (lambda e, cfg: e.input_meter_configure(0, True),
                    lambda e: [(r["batch_seq"], r["n_samples"], r["hist"].copy(), r["peak"].view(np.uint32).copy(),
                                r["sum"].view(np.uint64).copy(), r["sum_sq"].view(np.uint64).copy(),
                                np.float64(r["sum_iq"]).view(np.uint64)) for r in drain(lambda: e.fetch_input_levels(0))],
                    lambda e: e.input_meter_time()),
    "subband": (subband_on, subband_readings, lambda e: e.subband_time()),
    "tone_meter": (lambda e, cfg: e.tone_meter_configure(0, True),
                   lambda e: [(x[0].view(np.uint64).copy(), x[1].view(np.uint32).copy(), x[2].copy(), x[3])
                              for x in drain(lambda: e.fetch_tone_meter(0))],
                   lambda e: e.tone_meter_time()),
    "activity": (lambda e, cfg: e.activity_configure(0, lib.default_stride(cfg, 0), 1, 2, np.full(cfg.fft_size, ACT_THR, np.float32)),
                 lambda e: [activity_key(r) for r in drain(lambda: e.fetch_activity(0))],
                 lambda e: e.activity_time()),
    "history": (lambda e, cfg: e.history_configure(0, HISTORY_BATCHES), history_readings, lambda e: e.history_time()[0]),
}
SUBSETS = [frozenset(s) for n in range(len(MONITORS) + 1) for s in itertools.combinations(MONITORS, n)]


def readings(e):
    return {m: fetch(e) for m, (_, fetch, _) in MONITORS.items()}


def kernel_times(e):
    return {m: time(e) for m, (_, _, time) in MONITORS.items()}


def drive(cfg, raw, monitors):
    """Stream `raw` in thirds of a batch through a buffer of 3 batches (so it compacts), then resident runs."""
    e = lib.Engine(cfg, max_batches_per_run=2, input_capacity_batches=3)
    for m in monitors:
        MONITORS[m][0](e, cfg)
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
        res["audio"] += [(g[0].view(np.uint32).copy(), g[1].view(np.uint64).copy(), g[2].copy()) for g in drain(lambda: e.fetch(0))]
        for m, got in readings(e).items():
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
    res["resident_queued"] = {m: len(got) for m, got in readings(e).items()}
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
    if "activity" in subset:  # some batch found pieces and stored them all
        assert any(n_total > 0 and len(pieces) > 0 for _, n_total, _, pieces in got["readings"]["activity"])
    # resident runs queue nothing, and leave the history empty
    assert all(n == 0 for n in got["resident_queued"].values()) and got["resident_audio"] is None
    # the rest of the engine's output is bitwise that of the run with every monitor off
    assert len(got["audio"]) == len(off["audio"]) == sum(off["runs"])
    for a, b in zip(got["audio"], off["audio"]):
        assert all(np.array_equal(x, y) for x, y in zip(a, b))
    assert got["stats"] == off["stats"]


def test_failed_allocation_leaves_the_engine_intact():
    """A history ring of 2^31 - 1 batches (275 TB here) exceeds any device's memory: cudaMalloc refuses it at once.  The
    call reports ABG_ENOMEM; the runs after it, and every monitor switched on after it, work as if it had not been made."""
    cfg, raws = CASES["am_u8"](n_batches=6)
    half = raws[0].size // 2

    def stream(e, part):
        e.push(0, part)
        assert e.run(-1) > 0
        e.sync()
        audio = [(g[0].view(np.uint32).copy(), g[1].view(np.uint64).copy(), g[2].copy()) for g in drain(lambda: e.fetch(0))]
        return audio, [tuple(getattr(e.stats(0, c), f) for f in STAT_FIELDS) for c in range(len(cfg.devices[0].channels))]

    ref = lib.Engine(cfg)
    want = stream(ref, raws[0][:half])
    ref.close()
    e = lib.Engine(cfg)
    with pytest.raises(lib.AbgError) as ex:
        e.history_configure(0, 2 ** 31 - 1)
    assert ex.value.code == -3
    assert e.history_range(0) == (0, 0)
    got = stream(e, raws[0][:half])
    assert len(got[0]) == len(want[0]) > 0
    for a, b in zip(got[0], want[0]):
        assert all(np.array_equal(x, y) for x, y in zip(a, b))
    assert got[1] == want[1]
    assert all(not r for r in readings(e).values()) and kernel_times(e)["history"] == 0.0
    for on, _, _ in MONITORS.values():
        on(e, cfg)
    stream(e, raws[0][half:])
    assert all(r for r in readings(e).values())
    assert all(ms > 0.0 for ms in kernel_times(e).values())
    e.close()
