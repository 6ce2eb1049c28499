"""ORACLE — TEST INFRASTRUCTURE ONLY.

ctypes binding of the CPU oracle (oracle/airband_oracle.h).  May be imported only by tests/, by
__graft_entry__.smoke() and by bench.py's cpu_baseline / `--impl reference` legs — never by the product
package.  Variants (see oracle/Makefile):
    "restated"       oracle/libairband_oracle.so        strict IEEE build: THE parity checker
    "restated_fast"  oracle/libairband_oracle_fast.so   reference's optimisation flags: CPU baseline ("port")
    "ref"            oracle/_ref/libairband_ref.so       reference's own leaf classes, strict
    "ref_fast"       oracle/_ref/libairband_ref_fast.so  reference's own leaf classes + its flags ("reference")
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys
from typing import List, Optional, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_PKG = os.path.join(os.path.dirname(_HERE), "rtlsdr-airband_b200", "py")
if _PKG not in sys.path:
    sys.path.insert(0, _PKG)
from airband_b200.config import CConfig, CSquelchStats, Config  # noqa: E402

_PATHS = {
    "restated": os.path.join(_HERE, "libairband_oracle.so"),
    "restated_fast": os.path.join(_HERE, "libairband_oracle_fast.so"),
    "ref": os.path.join(_HERE, "_ref", "libairband_ref.so"),
    "ref_fast": os.path.join(_HERE, "_ref", "libairband_ref_fast.so"),
}
_LIBS = {}
FP = C.POINTER(C.c_float)


def build(quiet: bool = True) -> None:
    """Run oracle/Makefile (restated always; _ref only where /root/reference exists)."""
    subprocess.run(["make", "-C", _HERE, "-j4"], check=True, stdout=subprocess.DEVNULL if quiet else None)


def available(variant: str) -> bool:
    return os.path.exists(_PATHS[variant])


def lib(variant: str = "restated"):
    if variant in _LIBS:
        return _LIBS[variant]
    path = _PATHS[variant]
    if not os.path.exists(path):
        if variant.startswith("restated"):
            build()
        if not os.path.exists(path):
            raise FileNotFoundError(f"oracle variant {variant!r} not built: {path}")
    L = C.CDLL(path, mode=getattr(os, "RTLD_LOCAL", 0))
    vp, f, i, u32, u64, i32 = C.c_void_p, C.c_float, C.c_int, C.c_uint32, C.c_uint64, C.c_int32
    sig = {
        "abo_create": (vp, [C.POINTER(CConfig)]),
        "abo_destroy": (None, [vp]),
        "abo_wave_batch": (i, [vp]),
        "abo_push": (i, [vp, i, vp, C.c_size_t]),
        "abo_run": (C.c_long, [vp, i, i]),
        "abo_set_discard": (None, [vp, i]),
        "abo_set_pin": (None, [vp, vp, i]),
        "abo_batches_ready": (i, [vp, i]),
        "abo_fetch_batch": (i, [vp, i, vp, vp, vp]),
        "abo_get_stats": (i, [vp, i, i, C.POINTER(CSquelchStats)]),
        "abo_set_bin": (i, [vp, i, i, i]),
        "abo_scan_configure": (i, [vp, i, i, i, vp]),
        "abo_scan_select": (i, [vp, i, i, i]),
        "abo_get_window": (i, [vp, vp]),
        "abo_debug_frame": (i, [vp, i, vp, vp, vp]),
        "abo_debug_inject_wavein": (i, [vp, i, i, vp, vp]),
        "abo_calc_bin": (i32, [i32, i32, i32, i32]),
        "abo_calc_dm_dphi": (u32, [i32, i32, i32, i32]),
        "abo_dbfs_to_level": (f, [f, i32]),
        "abo_level_to_dbfs": (f, [f, i32]),
        "abo_default_alpha": (f, [i32]),
        "abo_sincosf_lut": (None, [u32, FP, FP]),
        "abo_fast_atan2": (f, [f, f]),
        "abo_polar_disc_fast": (f, [f, f, f, f]),
        "abo_fm_quadri_demod": (f, [f, f, f, f]),
        "abo_fft": (None, [i, vp, vp]),
        "abo_fft_seconds": (C.c_double, [i, i]),
        "abo_sq_new": (vp, []),
        "abo_sq_free": (None, [vp]),
        "abo_sq_set_level": (None, [vp, f]),
        "abo_sq_set_snr": (None, [vp, f]),
        "abo_sq_set_ctcss": (None, [vp, f, f]),
        "abo_sq_raw": (None, [vp, f]),
        "abo_sq_filtered": (None, [vp, f]),
        "abo_sq_audio": (None, [vp, f]),
        "abo_sq_is_open": (i, [vp]),
        "abo_sq_should_filter": (i, [vp]),
        "abo_sq_should_process_audio": (i, [vp]),
        "abo_sq_first_open": (i, [vp]),
        "abo_sq_last_open": (i, [vp]),
        "abo_sq_outside_filter": (i, [vp]),
        "abo_sq_noise_level": (f, [vp]),
        "abo_sq_signal_level": (f, [vp]),
        "abo_sq_squelch_level": (f, [vp]),
        "abo_sq_open_count": (u64, [vp]),
        "abo_sq_flappy_count": (u64, [vp]),
        "abo_sq_ctcss_count": (u64, [vp]),
        "abo_sq_no_ctcss_count": (u64, [vp]),
        "abo_sq_trace": (None, [vp, i, vp, vp, vp, vp, vp]),
        "abo_ctcss_new": (vp, [f, f, i]),
        "abo_ctcss_free": (None, [vp]),
        "abo_ctcss_sample": (None, [vp, f]),
        "abo_ctcss_enabled": (i, [vp]),
        "abo_ctcss_enough": (i, [vp]),
        "abo_ctcss_has_tone": (i, [vp]),
        "abo_ctcss_reset": (None, [vp]),
        "abo_ctcss_found": (u64, [vp]),
        "abo_ctcss_not_found": (u64, [vp]),
        "abo_notch_run": (None, [f, f, f, i, vp]),
        "abo_lowpass_run": (None, [f, f, i, vp]),
        "abo_variant": (C.c_char_p, []),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    _LIBS[variant] = L
    return L


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class Oracle:
    """One oracle instance = one rtl_airband process worth of devices[]."""

    def __init__(self, cfg: Config, variant: str = "restated"):
        self.L = lib(variant)
        self.cfg = cfg
        ccfg, self._keep = cfg.to_c()
        self.h = self.L.abo_create(C.byref(ccfg))
        if not self.h:
            raise ValueError("abo_create rejected the configuration")
        self.B = self.L.abo_wave_batch(self.h)

    def close(self):
        if self.h:
            self.L.abo_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def push(self, dev: int, raw: np.ndarray) -> None:
        raw = np.ascontiguousarray(raw)
        assert self.L.abo_push(self.h, dev, _ptr(raw), raw.nbytes) == 0

    def run(self, max_batches: int = -1, n_threads: int = 1) -> int:
        return int(self.L.abo_run(self.h, max_batches, n_threads))

    def set_pin(self, cpus) -> None:
        """Pin abo_run's worker thread t to cpus[t % len(cpus)] (timing runs)."""
        arr = np.ascontiguousarray(cpus, np.int32)
        self.L.abo_set_pin(self.h, _ptr(arr), int(arr.size))

    def set_discard(self, flag: bool) -> None:
        self.L.abo_set_discard(self.h, 1 if flag else 0)

    def fetch(self, dev: int) -> Optional[Tuple[np.ndarray, np.ndarray, np.ndarray]]:
        """Oldest finished batch of a device: (waveout[C,B], iq_out[C,B] complex64, axc[C] uint8) or None."""
        Cn = len(self.cfg.devices[dev].channels)
        wo = np.empty((Cn, self.B), np.float32)
        iq = np.empty((Cn, 2 * self.B), np.float32)
        ax = np.empty(Cn, np.uint8)
        if not self.L.abo_fetch_batch(self.h, dev, _ptr(wo), _ptr(iq), _ptr(ax)):
            return None
        return wo, iq.view(np.complex64), ax

    def fetch_all(self, dev: int):
        """All queued batches concatenated along time: (waveout[C, nb*B], iq_out[C, nb*B], axc[nb, C])."""
        wos, iqs, axs = [], [], []
        while True:
            r = self.fetch(dev)
            if r is None:
                break
            wos.append(r[0]); iqs.append(r[1]); axs.append(r[2])
        if not wos:
            Cn = len(self.cfg.devices[dev].channels)
            return np.zeros((Cn, 0), np.float32), np.zeros((Cn, 0), np.complex64), np.zeros((0, Cn), np.uint8)
        return np.concatenate(wos, 1), np.concatenate(iqs, 1), np.stack(axs, 0)

    def stats(self, dev: int, chan: int) -> CSquelchStats:
        s = CSquelchStats()
        assert self.L.abo_get_stats(self.h, dev, chan, C.byref(s)) == 0
        return s

    def set_bin(self, dev: int, chan: int, bin_: int) -> None:
        assert self.L.abo_set_bin(self.h, dev, chan, bin_) == 0

    def scan_configure(self, dev: int, chan: int, freqs) -> None:
        """Install a scan-mode frequency list (list of config.Channel); entry 0 becomes current."""
        from airband_b200.config import channels_to_c
        arr = channels_to_c(freqs)
        assert self.L.abo_scan_configure(self.h, dev, chan, len(freqs), C.cast(arr, C.c_void_p)) == 0

    def scan_select(self, dev: int, chan: int, freq_idx: int) -> None:
        assert self.L.abo_scan_select(self.h, dev, chan, freq_idx) == 0

    def inject_wavein(self, dev: int, wavein: np.ndarray, iq: Optional[np.ndarray] = None) -> int:
        """Stage tap: wavein[C, n_batches * B] straight into the channel loop (FFT skipped), with iq[C, n_batches * B]
        (complex64) as the X[bin] values of the same frames for channels that need raw I/Q."""
        w = np.ascontiguousarray(wavein, np.float32)
        assert w.ndim == 2 and w.shape[1] % self.B == 0
        q = None if iq is None else np.ascontiguousarray(iq, np.complex64)
        assert q is None or q.shape == w.shape
        return int(self.L.abo_debug_inject_wavein(self.h, dev, w.shape[1] // self.B, _ptr(w), _ptr(q)))

    def window(self) -> np.ndarray:
        w = np.empty(self.cfg.fft_size, np.float32)
        self.L.abo_get_window(self.h, _ptr(w))
        return w

    def debug_frame(self, dev: int, raw_frame: np.ndarray):
        n = self.cfg.fft_size
        fin = np.empty(2 * n, np.float32)
        fout = np.empty(2 * n, np.float32)
        raw_frame = np.ascontiguousarray(raw_frame)
        self.L.abo_debug_frame(self.h, dev, _ptr(raw_frame), _ptr(fin), _ptr(fout))
        return fin.view(np.complex64), fout.view(np.complex64)


class SquelchHarness:
    """Per-sample driver of one Squelch object (ports of reference src/test_squelch.cpp use this)."""

    def __init__(self, variant: str = "restated"):
        self.L = lib(variant)
        self.s = self.L.abo_sq_new()

    def __del__(self):
        try:
            self.L.abo_sq_free(self.s)
        except Exception:
            pass

    def set_level(self, v): self.L.abo_sq_set_level(self.s, v)
    def set_snr(self, v): self.L.abo_sq_set_snr(self.s, v)
    def set_ctcss(self, f, sr): self.L.abo_sq_set_ctcss(self.s, f, sr)
    def raw(self, v): self.L.abo_sq_raw(self.s, v)
    def filtered(self, v): self.L.abo_sq_filtered(self.s, v)
    def audio(self, v): self.L.abo_sq_audio(self.s, v)
    def is_open(self): return bool(self.L.abo_sq_is_open(self.s))
    def should_filter(self): return bool(self.L.abo_sq_should_filter(self.s))
    def should_process_audio(self): return bool(self.L.abo_sq_should_process_audio(self.s))
    def first_open(self): return bool(self.L.abo_sq_first_open(self.s))
    def last_open(self): return bool(self.L.abo_sq_last_open(self.s))
    def noise_level(self): return float(self.L.abo_sq_noise_level(self.s))
    def signal_level(self): return float(self.L.abo_sq_signal_level(self.s))
    def squelch_level(self): return float(self.L.abo_sq_squelch_level(self.s))
    def open_count(self): return int(self.L.abo_sq_open_count(self.s))
    def flappy_count(self): return int(self.L.abo_sq_flappy_count(self.s))
    def ctcss_count(self): return int(self.L.abo_sq_ctcss_count(self.s))
    def no_ctcss_count(self): return int(self.L.abo_sq_no_ctcss_count(self.s))

    def trace(self, raw: np.ndarray, filtered: Optional[np.ndarray] = None, audio: Optional[np.ndarray] = None):
        raw = np.ascontiguousarray(raw, np.float32)
        n = raw.size
        filtered = None if filtered is None else np.ascontiguousarray(filtered, np.float32)
        audio = None if audio is None else np.ascontiguousarray(audio, np.float32)
        levels = np.empty((n, 4), np.float32)
        flags = np.empty(n, np.int32)
        self.L.abo_sq_trace(self.s, n, _ptr(raw), _ptr(filtered), _ptr(audio), _ptr(levels), _ptr(flags))
        return levels, flags


class CtcssHarness:
    def __init__(self, freq: float, sample_rate: float, window: int, variant: str = "restated"):
        self.L = lib(variant)
        self.c = self.L.abo_ctcss_new(freq, sample_rate, window)

    def __del__(self):
        try:
            self.L.abo_ctcss_free(self.c)
        except Exception:
            pass

    def sample(self, v): self.L.abo_ctcss_sample(self.c, v)
    def enabled(self): return bool(self.L.abo_ctcss_enabled(self.c))
    def enough(self): return bool(self.L.abo_ctcss_enough(self.c))
    def has_tone(self): return bool(self.L.abo_ctcss_has_tone(self.c))


def fft(x: np.ndarray, variant: str = "restated") -> np.ndarray:
    x = np.ascontiguousarray(x, np.complex64)
    out = np.empty_like(x)
    lib(variant).abo_fft(x.size, _ptr(x), _ptr(out))
    return out


def notch_run(freq, sr, q, x, variant="restated"):
    y = np.ascontiguousarray(x, np.float32).copy()
    lib(variant).abo_notch_run(freq, sr, q, y.size, _ptr(y))
    return y


def lowpass_run(freq, sr, x, variant="restated"):
    y = np.ascontiguousarray(x, np.complex64).copy()
    lib(variant).abo_lowpass_run(freq, sr, y.size, _ptr(y))
    return y


def run_oracle(cfg: Config, raws: List[np.ndarray], variant: str = "restated", n_threads: int = 1):
    """Push one raw stream per device, run to exhaustion, return per-device (waveout, iq_out, axc) and the instance."""
    o = Oracle(cfg, variant)
    for d, r in enumerate(raws):
        o.push(d, r)
    o.run(-1, n_threads)
    return [o.fetch_all(d) for d in range(len(raws))], o
