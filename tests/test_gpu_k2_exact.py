"""K2 (rtlsdr-airband_b200/csrc/k2_demod.cu) against the CPU oracle, bit for bit (-m gpu).

K2 uses only correctly rounded IEEE single-precision operations in the reference's order, and its lane-parallel tiles and
speculative blocks claim to produce the very bits of the per-sample path; so given identical inputs its audio, I/Q output,
squelch decisions and every squelch statistic must equal the oracle's exactly.  The one exception is NaN, which matches any
NaN (the GPU's default NaN payload differs from x86's).  Two sources of identical inputs:
  * scenario sets (tests/k2_scenarios.py) injected into both through abg_debug_inject_wavein / abo_debug_inject_wavein,
    1, 2, 3 and 4 batches per call, with the engine's own channels-per-warp choice and with ABG_K2_LPW 2, 8 and 32;
  * real bytes: K1's rows of every GPU run (abg_debug_k1_outputs) injected into the oracle, for the shared parity cases and
    scaled-down cfg2 / cfg3 in every fft_mode.
The coverage test runs the scenario sets once more against the K2 event-counter build (make stats) in a child process and
requires every counted steady-state path to have been taken."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import k2_scenarios as ks
import oracle_py as op
from airband_b200 import config as cm
from airband_b200 import lib
from airband_b200 import workloads as wl
from cases import CASES

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATS_LIB = os.path.join(ROOT, "rtlsdr-airband_b200", "build", "stats", "libairband_b200.so")
STAT_FIELDS = [f for f, _ in cm.CSquelchStats._fields_]


def same_bits(a, b):
    """Equal float32 bit patterns, any NaN matching any NaN."""
    a = np.ascontiguousarray(a, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    if a.shape != b.shape:
        return False
    return bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


def first_difference(a, b):
    a = np.ascontiguousarray(a, np.float32).ravel()
    b = np.ascontiguousarray(b, np.float32).ravel()
    bad = np.flatnonzero((a.view(np.uint32) != b.view(np.uint32)) & ~(np.isnan(a) & np.isnan(b)))
    return (int(bad[0]), float(a[bad[0]]), float(b[bad[0]]), int(bad.size)) if bad.size else None


def stats_tuple(s):
    out = []
    for f in STAT_FIELDS:
        v = getattr(s, f)
        out.append(("nan" if v != v else int(np.float32(v).view(np.uint32))) if isinstance(v, float) else int(v))
    return tuple(out)


def run_side(sset, side):
    """Feed a scenario set to an Engine or an Oracle; returns per device the list of batches (waveout, iq_out, axc) and the
    statistics of every channel after every injection call."""
    cfg = sset["cfg"]
    B = cfg.wave_batch
    out = []
    for d in range(len(cfg.devices)):
        wave, iq = sset["wave"][d], sset["iq"][d]
        nb = wave.shape[1] // B
        batches, stats, pos = [], [], 0
        for k, m in enumerate(ks.calls(nb)):
            if sset["scan"] and sset["scan"][0] == d:
                _, chan, entries = sset["scan"]
                if k == 0:
                    side.scan_configure(d, chan, entries)
                side.scan_select(d, chan, [0, 1, 2, 1, 0, 2, 2, 0][k % 8])
            sl = slice(pos * B, (pos + m) * B)
            assert side.inject_wavein(d, wave[:, sl], iq[:, sl]) == m
            pos += m
            for _ in range(m):
                got = side.fetch(d)
                assert got is not None
                batches.append((got[0].copy(), got[1].copy(), got[2].copy()))
            stats.append([stats_tuple(side.stats(d, c)) for c in range(wave.shape[0])])
        out.append((batches, stats))
    return out


def compare(sset, gpu, ora, what):
    for d, ((gb, gs), (ob, os_)) in enumerate(zip(gpu, ora)):
        assert len(gb) == len(ob)
        for b, (g, o) in enumerate(zip(gb, ob)):
            for c in range(g[0].shape[0]):
                assert same_bits(g[0][c], o[0][c]), f"{what}: audio dev {d} chan {c} batch {b}: first difference {first_difference(g[0][c], o[0][c])}"
                assert same_bits(g[1][c].view(np.float32), o[1][c].view(np.float32)), \
                    f"{what}: iq_out dev {d} chan {c} batch {b}: {first_difference(g[1][c].view(np.float32), o[1][c].view(np.float32))}"
            assert np.array_equal(g[2], o[2]), f"{what}: axcindicate dev {d} batch {b}: {g[2]} vs {o[2]}"
        for k, (g, o) in enumerate(zip(gs, os_)):
            for c in range(len(g)):
                assert g[c] == o[c], f"{what}: stats dev {d} chan {c} after call {k}: " + \
                    str({f: (x, y) for f, x, y in zip(STAT_FIELDS, g[c], o[c]) if x != y})


_SETS = None
_ORACLE = {}


def scenario_sets():
    global _SETS
    if _SETS is None:
        _SETS = ks.scenario_sets()
    return _SETS


def oracle_result(sset):
    if sset["name"] not in _ORACLE:
        o = op.Oracle(sset["cfg"])
        _ORACLE[sset["name"]] = run_side(sset, o)
        o.close()
    return _ORACLE[sset["name"]]


def gpu_result(sset, lpw, monkeypatch):
    if lpw is None:
        monkeypatch.delenv("ABG_K2_LPW", raising=False)
    else:
        monkeypatch.setenv("ABG_K2_LPW", str(lpw))
    e = lib.Engine(sset["cfg"], max_batches_per_run=4)
    try:
        return run_side(sset, e)
    finally:
        e.close()


def test_scenarios_open_close_and_clip():
    """The scenario sets reach the open squelch (checked on the oracle): in every set most channels open at some point, so the
    comparisons below are not of silence."""
    for sset in scenario_sets():
        res = oracle_result(sset)
        batches, stats = res[0]
        axc = np.stack([b[2] for b in batches])
        opened = (axc != ord(" ")).any(axis=0)
        assert opened.mean() > 0.8, (sset["name"], opened)


@pytest.mark.parametrize("lpw", [None, 2, 8, 32], ids=["lpw_auto", "lpw2", "lpw8", "lpw32"])
@pytest.mark.parametrize("which", ["am", "nfm0", "nfm1"])
def test_k2_equals_oracle_bit_for_bit(which, lpw, monkeypatch):
    sset = next(s for s in scenario_sets() if s["name"] == which)
    compare(sset, gpu_result(sset, lpw, monkeypatch), oracle_result(sset), f"{which} lpw={lpw}")


# ---- real bytes: K1's output of every GPU run is the oracle's input ----------------------------------------------------
def _prefixed(cfg, raws):
    """Each stream behind 100 hops + fft_size samples of silence.  The first run's AGC_EXTRA look-back rows are K1 frames
    that abg_debug_k1_outputs does not return; the oracle's first injection starts from the reference's initial look-back
    instead (wavein 20.0, iq_in 0).  For S8 / S16 / F32 silence K1 stores X = 0 exactly, which is the oracle's I/Q look-back;
    the wavein look-back is read only by the AM AGC, which cannot run within the first AGC_EXTRA samples (the squelch opens
    197 samples after it first sees a signal at the earliest).  U8 silence (code 128) is 1/255 off zero: the U8 cases have
    plain AM channels and one rawfile channel that starts keyed off, so none reads that I/Q look-back."""
    out = []
    for d, r in enumerate(raws):
        dev = cfg.devices[d]
        n = 100 * cfg.hop(d) + cfg.fft_size
        z = np.full(2 * n, 128 if dev.sfmt == cm.SFMT_U8 else 0, r.dtype)
        out.append(np.concatenate([z, r]))
    return out


def _real_cases():
    out = {k: v for k, v in CASES.items()}
    out["cfg2_small"] = lambda: (lambda c: (c, [wl.synth_iq(c, d, wl.samples_for_batches(c, d, 3), key_on_s=0.2, key_off_s=0.1)
                                                for d in range(len(c.devices))]))(wl.cfg2(n_devices=2, n_channels=8))
    out["cfg3_small"] = lambda: (lambda c: (c, [wl.synth_iq(c, d, wl.samples_for_batches(c, d, 6), key_on_s=0.25, key_off_s=0.1)
                                                for d in range(len(c.devices))]))(wl.cfg3(n_devices=1, n_channels=8, parity=True))
    return out


REAL = _real_cases()


@pytest.mark.parametrize("fft_mode", [0, 1, 2, 3], ids=["auto", "full_fft", "pruned_fft", "tensor_core"])
@pytest.mark.parametrize("name", list(REAL))
def test_oracle_on_k1_rows_equals_gpu_bit_for_bit(name, fft_mode):
    cfg, raws = REAL[name]()
    raws = _prefixed(cfg, raws)
    B = cfg.wave_batch
    e = lib.Engine(cfg, max_batches_per_run=4, fft_mode=fft_mode)
    o = op.Oracle(cfg)
    g0 = np.cumsum([0] + [len(dv.channels) for dv in cfg.devices])
    pos = [0] * len(raws)
    n_batches = 0
    try:
        while True:
            progressed = False
            for d, r in enumerate(raws):
                if pos[d] < r.size:
                    hop_items = cfg.hop(d) * 2
                    n = 4 * B * hop_items + (100 * hop_items + 2 * cfg.fft_size if pos[d] == 0 else 0)
                    e.push(d, r[pos[d]:pos[d] + n])
                    pos[d] += n
                    progressed = True
            ran = e.run(-1)
            if ran:
                win, iqin = e.k1_outputs()
                for d in range(len(raws)):
                    got = []
                    while True:
                        x = e.fetch(d)
                        if x is None:
                            break
                        got.append(x)
                    if not got:
                        continue
                    cols = slice(g0[d], g0[d + 1])
                    m = len(got)
                    assert o.inject_wavein(d, win[:m * B, cols].T, iqin[:m * B, cols].T) == m
                    for b, g in enumerate(got):
                        w = o.fetch(d)
                        for c in range(g[0].shape[0]):
                            assert same_bits(g[0][c], w[0][c]), f"{name} mode {fft_mode}: audio dev {d} chan {c} batch {n_batches + b}: {first_difference(g[0][c], w[0][c])}"
                            assert same_bits(g[1][c].view(np.float32), w[1][c].view(np.float32)), f"{name}: iq_out dev {d} chan {c}"
                        assert np.array_equal(g[2], w[2]), f"{name} mode {fft_mode}: axcindicate dev {d} batch {n_batches + b}"
                n_batches += 1
            if ran == 0 and not progressed:
                break
        assert n_batches > 0
        for d in range(len(raws)):
            for c in range(len(cfg.devices[d].channels)):
                assert stats_tuple(e.stats(d, c)) == stats_tuple(o.stats(d, c)), (name, d, c)
    finally:
        e.close()
        o.close()


# ---- coverage: the counters of the stats build --------------------------------------------------------------------------
# counter index -> what must have happened at least once (names: tools/k2_stats.py)
REQUIRED = {
    2: "NFM tile attempts OPEN", 3: "NFM tile attempts CLOSING", 4: "NFM tile attempts OPENING", 5: "NFM tile attempts CLOSED",
    6: "NFM tile attempts ABORT", 7: "NFM tile samples OPEN", 8: "NFM tile samples CLOSING", 9: "NFM tile samples OPENING",
    10: "NFM tile samples CLOSED", 11: "NFM tile samples ABORT", 22: "NFM tile attempts held-CLOSED", 23: "NFM tile samples held-CLOSED",
    17: "tiles of 8", 18: "tiles of 16",
    # 14 ("post estimator not live": OPEN / CLOSING with the low-pass on and using_post_ clear) is not required: nothing
    # reaches OPEN but the OPENING delay's end (k2_demod.cu:1825, delay >= 197), using_post_ is cleared only on entering
    # OPENING or CLOSED (:1844 and the CLOSED branch below it) and set again during OPENING once delay >= buffer_size = 102
    # (:1957), so with the low-pass on it is always set in OPEN and CLOSING.
    12: "no room for a tile", 13: "CTCSS window ends in tile", 15: "OPENING at buffer_size boundary",
    16: "CLOSED recent_open pending", 20: "state ends within 8", 21: "noise-floor update within 8",
    24: "refused: low_signal_abort", 25: "refused: lp division range", 26: "refused: sqrt range", 27: "refused: has_signal false",
    28: "refused: CLOSED sees signal", 29: "refused: post < tail", 30: "refused: discriminator division range", 31: "refused: held-CLOSED ends",
    32: "general in CLOSED", 33: "general in OPENING", 34: "general in CLOSING", 35: "general in ABORT", 36: "general in OPEN",
    40: "general: transition sample",
    41: "AM tile attempts OPEN", 42: "AM tile samples OPEN", 43: "AM tile refused OPEN", 44: "AM tile attempts quiet",
    45: "AM tile samples quiet", 46: "AM tile refused quiet", 47: "AM OPEN tile fully capped", 48: "AM OPEN tile never capped",
    57: "AM quiet tile never capped", 49: "AM open_run attempts", 50: "AM open_run refused", 51: "AM quiet_run attempts",
    52: "AM quiet_run refused", 53: "AM open sample: exact division", 54: "NFM block attempts OPEN/CLOSING", 55: "NFM block attempts OPENING",
    56: "NFM block attempts CLOSED", 58: "NFM block samples", 59: "NFM block refused",
}


def _child():
    """Child process (ABG_LIB_PATH = the stats build): run every scenario set with each channels-per-warp setting, check it
    against the oracle, print the summed counters as one JSON line."""
    L = lib.load()
    buf = (C.c_ulonglong * 64)()
    assert L.abg_debug_k2_stats(buf) == 0, "not a stats build"
    total = np.zeros(64, np.uint64)

    class MP:
        def setenv(self, k, v):
            os.environ[k] = v

        def delenv(self, k, raising=False):
            os.environ.pop(k, None)
    for lpw in (None, 2, 8):
        for sset in scenario_sets():
            compare(sset, gpu_result(sset, lpw, MP()), oracle_result(sset), f"stats build {sset['name']} lpw={lpw}")
            assert L.abg_debug_k2_stats(buf) == 0
            total += np.array(list(buf), np.uint64)
    print("K2STATS " + json.dumps([int(x) for x in total]))


def test_stats_build_takes_every_counted_path():
    assert os.path.exists(STATS_LIB), "stats build missing: make -C rtlsdr-airband_b200 stats"
    env = dict(os.environ, ABG_LIB_PATH=STATS_LIB)
    code = "import sys; sys.path[:0] = %r; import test_gpu_k2_exact as t; t._child()" % ([os.path.dirname(os.path.abspath(__file__))] + sys.path,)
    p = subprocess.Popen([sys.executable, "-c", code], env=env, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        out, _ = p.communicate(timeout=600)
    finally:
        if p.poll() is None:
            p.kill()
            p.communicate()
    assert p.returncode == 0, out[-4000:]
    line = [x for x in out.splitlines() if x.startswith("K2STATS ")][-1]
    cnt = json.loads(line[len("K2STATS "):])
    print("\n".join(f"[{i:2d}] {REQUIRED.get(i, '')}: {cnt[i]}" for i in range(64) if cnt[i] or i in REQUIRED))
    missing = {i: n for i, n in REQUIRED.items() if cnt[i] == 0}
    assert not missing, f"paths never taken: {missing}"
