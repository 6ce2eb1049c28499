"""Transmission profiles on the CPU: the C ABI and the C layouts of abg_profile_job and abg_profile, the block plan
abg_history_profile launches (every read inside what its chunk captured, every output and pair exactly once, the budgets
and launch limits), profile_job's window against a brute-force reading of the range rule, the profile kernel's ptxas log,
and the decision rule of profile_summary on a float64 numpy model of the same statistics over synthetic baseband."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from airband_b200 import config as cm
from airband_b200 import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AGC = cm.AGC_EXTRA
PB = lib.PROFILE_BLOCK
NEW = ("abg_history_profile", "abg_debug_history_profile_time", "abg_debug_profile_plan")


# ---- ABI ----------------------------------------------------------------------------------------------------------------------
def test_header_symbols_and_argtypes():
    hdr = open(os.path.join(ROOT, "include", "airband_b200.h")).read()
    for s in NEW:
        assert s in lib.SYMBOLS and re.search(r"ABG_API int %s\(" % s, hdr), s
    assert re.search(r"#define ABG_PROFILE_BLOCK %d\b" % PB, hdr)
    L = lib.load()
    vp, i = C.c_void_p, C.c_int
    assert L.abg_history_profile.argtypes == [vp, i, C.POINTER(lib.CProfileJob)]
    assert L.abg_debug_history_profile_time.argtypes == [vp, C.POINTER(C.c_float)]
    assert L.abg_debug_profile_plan.argtypes == [i, vp, vp, vp, vp, vp, vp, i, C.POINTER(C.c_int32), vp, i, C.POINTER(C.c_int32)]
    for s in NEW:
        assert getattr(L, s).restype == C.c_int


@pytest.mark.parametrize("ctype,cname", [(lib.CProfileJob, "abg_profile_job"), (lib.CProfile, "abg_profile")])
def test_struct_layout_matches_the_header(tmp_path, ctype, cname):
    fields = [f for f, _ in ctype._fields_]
    prog = "#include <stdio.h>\n#include <stddef.h>\n#include \"airband_b200.h\"\nint main(void) {\n"
    prog += "".join(f'    printf("%zu\\n", offsetof({cname}, {f}));\n' for f in fields)
    prog += f'    printf("%zu\\n", sizeof({cname}));\n    return 0;\n}}\n'
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text(prog)
    subprocess.run(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [getattr(ctype, f).offset for f in fields] + [C.sizeof(ctype)]


def test_profile_kernel_has_no_spills_and_no_stack():
    log = open(os.path.join(ROOT, "rtlsdr-airband_b200", "build", "profile.ptxas.log")).read()
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert any("abg_profile_kernel" in p[0] for p in props)
    for name, stack, st, ld in props:
        assert (int(stack), int(st), int(ld)) == (0, 0, 0), name


# ---- the block plan -------------------------------------------------------------------------------------------------------------
def check_plan(first_m, n_out, n_coeffs, n_tones):
    """Every invariant of the plan for one job set; returns the chunk count."""
    lim, P, Bk = lib.profile_plan(first_m, n_out, n_coeffs, n_tones)
    first_m, n_out = np.asarray(first_m, np.int64), np.asarray(n_out, np.int64)
    assert P.shape[0] >= 1 and Bk.shape[0] >= 1
    # chunks in order, pieces and blocks in job order
    assert np.all(np.diff(P[:, 0]) >= 0) and np.all(np.diff(Bk[:, 0]) >= 0) and P[0, 0] == 0 and Bk[0, 0] == 0
    assert np.all(np.diff(Bk[:, 1]) >= 0)
    # every block reads y[off, off + n + succ): inside what its own piece captured, in its own chunk
    ch, job, pc, off, m, n, succ = (Bk[:, k] for k in range(7))
    own = P[pc]
    assert np.array_equal(own[:, 0], ch) and np.array_equal(own[:, 1], job)
    assert np.all((n >= 1) & (n <= PB)) and np.all((succ == 0) | (succ == 1))
    assert np.all(own[:, 4] <= off) and np.all(off + n + succ <= own[:, 4] + own[:, 3])
    assert np.array_equal(off - own[:, 4], m - own[:, 2])  # the scratch slot of output m is the one its capture wrote
    # blocks tile each job's outputs [m0, m0 + n) and pairs [m0, m0 + n - 1) exactly once, anchored at m0
    jb = np.searchsorted(Bk[:, 1], np.arange(first_m.size + 1))  # each job's blocks, in order
    jp = np.searchsorted(P[:, 1], np.arange(first_m.size + 1))
    assert np.all(np.diff(jb) == -(-n_out // PB)) and np.all(np.diff(jp) >= 1)
    k = np.arange(Bk.shape[0]) - np.repeat(jb[:-1], np.diff(jb))  # block index within its job
    last = np.zeros(Bk.shape[0], bool)
    last[jb[1:] - 1] = True
    assert np.array_equal(Bk[:, 4], first_m[Bk[:, 1]] + PB * k)
    assert np.all(Bk[~last, 5] == PB) and np.all(Bk[~last, 6] == 1) and np.all(Bk[last, 6] == 0)
    assert np.array_equal(np.add.reduceat(Bk[:, 5], jb[:-1]), n_out)  # outputs
    assert np.array_equal(np.add.reduceat(Bk[:, 5] - 1 + Bk[:, 6], jb[:-1]), n_out - 1)  # pairs
    assert np.array_equal(P[jp[:-1], 2], first_m) and np.array_equal(P[jp[1:] - 1, 2] + P[jp[1:] - 1, 3], first_m + n_out)
    seam = np.ones(P.shape[0], bool)
    seam[jp[:-1]] = False  # a job's later pieces start on the previous piece's successor output
    assert np.array_equal(P[seam, 2], P[np.flatnonzero(seam) - 1, 2] + P[np.flatnonzero(seam) - 1, 3] - 1)
    # budgets and launch limits per chunk; scratch and coefficient ranges of a chunk's pieces do not overlap
    for ch in np.unique(Bk[:, 0]):
        pc, bc = P[P[:, 0] == ch], Bk[Bk[:, 0] == ch]
        assert bc.shape[0] <= lim["blocks"] <= 65535
        assert (pc[:, 4] + pc[:, 3]).max() <= lim["scratch"]
        o = np.argsort(pc[:, 4])
        assert np.all(pc[o][1:, 4] >= pc[o][:-1, 4] + pc[o][:-1, 3])
        L = np.asarray(n_coeffs, np.int64)[pc[:, 1]]
        assert np.all(np.diff(pc[:, 5]) == L[:-1]) and pc[0, 5] == 0 and (pc[:, 5] + L).max() <= lim["coeffs"]
        K = np.asarray(n_tones, np.int64)[bc[:, 1]]
        size = 8 + 4 * K
        assert np.array_equal(bc[:, 7], np.concatenate([[0], np.cumsum(size)[:-1]])) and (bc[:, 7] + size).max() <= lim["result"]
    assert lim["scratch"] == 8 << 20 and lim["blocks"] == 65535
    return int(Bk[-1, 0]) + 1


def test_plan_of_random_job_sets():
    rng = np.random.default_rng(7)
    chunks = []
    for it in range(40):
        nj = int(rng.integers(1, 30))
        n = np.where(rng.random(nj) < 0.3, 2, rng.integers(2, 3 * PB + 7, nj))
        n[rng.random(nj) < 0.1] = PB
        n[rng.random(nj) < 0.1] = PB + 1
        first = rng.integers(0, 1 << 40, nj).astype(np.uint64)
        first[0] = (1 << 32) - 5  # across the 32-bit phase wrap
        L = np.where(rng.random(nj) < 0.5, 1, rng.choice([4096, 255, 563], nj))
        K = rng.integers(1, 65, nj)
        chunks.append(check_plan(first, n, L, K))
    assert max(chunks) == 1


def test_plan_of_jobs_larger_than_a_chunk():
    # 10 s at D = 1 of a 2.56 Msps device, and a job that fills a chunk exactly to one output short of its end
    n = [25_600_000, (8 << 20) - 1, 8 << 20, 5, (8 << 20) + 1]
    assert check_plan([3, 1 << 33, 77, 0, 12345], n, [4096, 1, 255, 1, 4096], [51, 64, 1, 51, 51]) >= 4


def test_plan_of_many_tiny_jobs():
    nj = 65535
    rng = np.random.default_rng(3)
    assert check_plan(rng.integers(0, 1 << 50, nj).astype(np.uint64), np.full(nj, 2), np.full(nj, 4096), np.full(nj, 51)) >= 2
    assert check_plan(np.arange(nj, dtype=np.uint64), rng.integers(2, 40, nj), np.full(nj, 1), np.full(nj, 64)) >= 2


def test_plan_refuses_what_the_call_refuses():
    for args in (([0], [1], [1], [51]), ([0], [5], [0], [51]), ([0], [5], [4097], [51]), ([0], [5], [1], [0]), ([0], [5], [1], [65])):
        with pytest.raises(lib.AbgError):
            lib.profile_plan(*args)


# ---- profile_job --------------------------------------------------------------------------------------------------------------
CFGS = [(2048000, 512), (2048000, 8192), (2560000, 512), (2560000, 2048), (2560000, 8192), (2506504, 2048)]


@pytest.mark.parametrize("sr,n", CFGS, ids=["%d_%d" % c for c in CFGS])
def test_profile_filter_rule(sr, n):
    cfg = cm.Config(fft_size=n, wave_rate=8008 if sr == 2506504 else 8000,
                    devices=[cm.Device(sample_rate=sr, sfmt=cm.SFMT_U8, centerfreq=120_000_000)])
    D, cutoff, L = lib.profile_filter(cfg, 0)
    bin_hz = sr // n
    assert cutoff >= 5000 + 3000 + bin_hz  # 5 kHz deviation, 3 kHz audio and one bin of uncertainty
    fs_out = sr / D
    assert 1 <= D <= cfg.wave_batch * cfg.hop(0)
    assert L % 2 == 1 and L <= lib.SUBBAND_MAX_COEFFS
    assert (60 - 7.95) / (14.36 * (L - 1)) * sr <= cutoff  # the 60 dB stopband starts by twice the cutoff
    # the output noise is white: the filter's autocorrelation at lag D
    h = lib.subband_lowpass(L, cutoff, sr).astype(np.float64)
    assert abs(np.dot(h[D:], h[:-D]) / np.dot(h, h)) < 0.005
    # the largest instantaneous frequency, one bin off plus 5 kHz of deviation, stays below fs_out / 2
    assert bin_hz + 5000 < fs_out / 2 and max(lib.STANDARD_TONES) < fs_out / 2


def test_profile_job_window_matches_the_range_rule():
    cfg = cm.Config(fft_size=2048, wave_rate=8000, devices=[cm.Device(sample_rate=2048000, sfmt=cm.SFMT_U8, centerfreq=120_000_000)])
    hop, N = cfg.hop(0), cfg.fft_size
    rng = np.random.default_rng(11)
    cases = 0
    for _ in range(300):
        f0 = int(rng.integers(AGC, AGC + 3000))
        tx = dict(freq_hz=120_000_000 + float(rng.uniform(-9e5, 9e5)), first_frame=f0, last_frame=f0 + int(rng.integers(0, 2000)))
        first = int(rng.integers(0, (AGC + 4000) * hop))
        end = first + int(rng.integers(0, 6000 * hop))
        D = int(rng.choice([1, 7, 62, 1000]))
        L = int(rng.choice([1, 63, 301]))
        lo, hi = f0 * hop, tx["last_frame"] * hop + N
        # brute force: the outputs m with m*D in [lo, hi) and every tap in [first, end)
        ms = [m for m in range(lo // D - 1, hi // D + 2) if lo <= m * D < hi and m * D - (L - 1) >= first and m * D < end]
        if len(ms) < 2:
            with pytest.raises(ValueError):
                lib.profile_job(tx, cfg, 0, (first, end), decim=D, n_coeffs=L)
            continue
        j = lib.profile_job(tx, cfg, 0, (first, end), decim=D, n_coeffs=L)
        assert (j["first_m"], j["n_out"]) == (ms[0], len(ms)) and ms == list(range(ms[0], ms[-1] + 1))
        assert j["decim"] == D and j["coeffs"].size == L and j["dev"] == 0 and j["tones"] is None
        assert j["offset_hz"] == tx["freq_hz"] - 120_000_000
        cases += 1
    assert cases > 100


# ---- the decision rule on a float64 model ---------------------------------------------------------------------------------------
def model_sums(y, m0, fs_out, tones=lib.STANDARD_TONES):
    """The profile's sums of the definition in float64 from the outputs y[m0 ...], with the exact phase."""
    y = np.asarray(y).astype(np.complex128)
    p = np.abs(y) ** 2
    a = np.sqrt(p)
    z = y[1:] * np.conj(y[:-1])
    phi = np.concatenate([np.angle(z), [0.0]])
    m = (m0 + np.arange(y.size)) % (1 << 32)
    d = np.array([int(np.floor(float(np.float32(f)) / fs_out * 4294967296.0 + 0.5)) % (1 << 32) for f in tones], np.int64)
    ph = (d[:, None] * m[None, :]) % (1 << 32)
    E = np.exp(-2j * np.pi * ph / 4294967296.0)
    return dict(n=y.size, p1=p.sum(), p2=(p * p).sum(), a1=a.sum(), z=z.sum(), f1=phi.sum(), f2=(phi * phi).sum(),
                tone_fm=E @ phi, tone_am=E @ a)


def synth(kind, x, voice, ctcss, off, fs, n, cnr_db, h, rng):
    """Baseband at fs: kind "am" (depth x), "nfm" (peak deviation x Hz), "carrier" or "noise", modulated by the voice tones
    and a CTCSS tone of 10-15 % of the modulation; plus complex noise shaped by h, carrier over noise cnr_db in its
    passband (the noise's whole power, since h is the passband)."""
    t = np.arange(n) / fs
    parts = []
    if ctcss:
        parts.append((ctcss, rng.uniform(0.10, 0.15)))
    w = rng.uniform(0.5, 1.0, len(voice))
    parts += list(zip(voice, w / w.sum() * (1 - sum(s for _, s in parts))))
    msig = sum(s * np.sin(2 * np.pi * f * t + rng.uniform(0, 2 * np.pi)) for f, s in parts)
    if kind == "am":
        y = (1 + x * msig) * np.exp(2j * np.pi * off * t)
    elif kind == "nfm":
        y = np.exp(1j * (2 * np.pi * off * t + 2 * np.pi * np.cumsum(x * msig) / fs))
    elif kind == "carrier":
        y = np.exp(2j * np.pi * off * t)
    else:
        y = np.zeros(n, np.complex128)
    wn = (rng.normal(size=n + h.size - 1) + 1j * rng.normal(size=n + h.size - 1)) / np.sqrt(2)
    nz = np.convolve(wn, h, "valid")
    nz *= np.sqrt(10 ** (-cnr_db / 10) / np.mean(np.abs(nz) ** 2))
    return (y + nz).astype(np.complex64)


# The model is profile_filter's default job of a 2.048 Msps device at fft 512 (a bin of 4 kHz, the widest uncertainty):
# its output rate, and white noise, which is what the filter's D leaves; the passband is the whole output band.
MODEL_CFG = cm.Config(fft_size=512, wave_rate=8000, devices=[cm.Device(sample_rate=2048000, sfmt=cm.SFMT_F32, fullscale=1.0, centerfreq=0)])
D_MODEL, CUTOFF, L_MODEL = lib.profile_filter(MODEL_CFG, 0)
FS = 2048000 / D_MODEL
SIGNALS = [("am", x) for x in (0.3, 0.6, 0.9)] + [("nfm", x) for x in (1500.0, 2500.0, 5000.0)] + [("carrier", 0.0), ("noise", 0.0)]
CTCSS = (None, 67.0, 69.3, 127.3, 254.1)


def _classify(kind, x, voice, ctcss, off, cnr, rng, seconds=1.0):
    n = int(seconds * FS)
    m0 = int(rng.integers(0, 1 << 34))
    y = synth(kind, x, voice, ctcss, off, FS, n, cnr, np.ones(1), rng)
    job = dict(dev=0, offset_hz=0.0, decim=D_MODEL, coeffs=lib.subband_lowpass(L_MODEL, CUTOFF, 2048000), first_m=m0, n_out=n, tones=None)
    return lib.profile_summary(model_sums(y, m0, FS), job, MODEL_CFG, 0)


def _grid(cnr, seeds):
    rng = np.random.default_rng(cnr * 1000 + seeds)
    bin_hz = 4000  # a whole bin of carrier uncertainty, edges included (fft 512 at 2.048 Msps)
    for seed in range(seeds):
        for kind, x in SIGNALS:
            for ctcss in (CTCSS if kind in ("am", "nfm") else (None,)):
                voice = [1000.0] if seed % 2 == 0 else list(rng.uniform(300, 3000, int(rng.integers(3, 6))))
                off = float(rng.choice([-bin_hz / 2, bin_hz / 2, rng.uniform(-bin_hz / 2, bin_hz / 2)]))
                yield kind, x, voice, ctcss, off, _classify(kind, x, voice, ctcss, off, cnr, rng)


def test_decision_rule_at_20_db():
    n = 0
    for kind, x, voice, ctcss, off, s in _grid(20, 4):
        want = {"am": cm.MOD_AM, "carrier": cm.MOD_AM, "nfm": cm.MOD_NFM, "noise": None}[kind]
        assert s["modulation"] == want, (kind, x, voice, ctcss, off, s)
        if kind != "noise":
            assert s["ctcss_hz"] == ctcss, (kind, x, voice, ctcss, off, s)
            # AM: the noise's pull on arg(z), about rho sigma^2 / C * sin(offset) rad, is removed with an estimate of
            # sigma^2 that a deep envelope spoils; where the SNR estimate fails it is not removed
            tol = 20.0 if kind == "nfm" else 2.0
            assert abs(s["freq_hz"] - off) <= tol, (kind, x, voice, ctcss, off, s)
            assert s["channel_kw"] == dict(modulation=want, ctcss_hz=ctcss or 0.0)
        n += 1
    assert n > 100


def test_decision_rule_at_10_db_is_never_wrong():
    decided = 0
    for kind, x, voice, ctcss, off, s in _grid(10, 3):
        want = {"am": cm.MOD_AM, "carrier": cm.MOD_AM, "nfm": cm.MOD_NFM, "noise": None}[kind]
        assert s["modulation"] in (None, want), (kind, x, voice, ctcss, off, s)
        assert s["ctcss_hz"] in (None, ctcss), (kind, x, voice, ctcss, off, s)
        decided += s["modulation"] is not None
    # at 10 dB the SNR estimate is below PROFILE_MIN_SNR_DB: only AM whose envelope is beyond doubt is decided
    assert decided >= 5


def test_short_windows_name_no_tone():
    rng = np.random.default_rng(5)
    s = _classify("nfm", 2500.0, [1000.0], 127.3, 0.0, 20, rng, seconds=0.3)
    assert s["modulation"] == cm.MOD_NFM and s["ctcss_hz"] is None and s["channel_kw"]["ctcss_hz"] == 0.0
