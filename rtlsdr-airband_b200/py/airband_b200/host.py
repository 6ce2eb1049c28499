"""ctypes driver of the C++ host adapter test harness (rtlsdr-airband_b200/host): input rings + demodulate_b200() +
an output-thread stand-in, i.e. the reference's thread structure around the GPU engine."""
from __future__ import annotations

import ctypes as C
import os
from typing import List

import numpy as np

from .config import CConfig, Config
from .lib import LIB_DIR

HOST_LIB = os.path.join(LIB_DIR, "libairband_host.so")
HOST_SYMBOLS = ["demodulate_b200", "b200_refresh_stats", "abh_create", "abh_run", "abh_batches", "abh_waveout", "abh_iq_out", "abh_axc",
                "abh_overflows", "abh_overruns", "abh_active_counter", "abh_last_error", "abh_destroy", "abh_set_freqlist", "abh_run_pattern", "pattern_input_new", "abh_pattern_selftest",
                "abh_set_mixers", "abh_add_rawfile", "abh_mixer_batches", "abh_mixer_left", "abh_mixer_right", "abh_mixer_axc", "abh_mixer_overruns", "abh_mixer_is_gpu",
                "abh_failed_calls", "b200_mixer_is_gpu", "b200_write_rawfile"]
_L = None


def load():
    global _L
    if _L is None:
        if not os.path.exists(HOST_LIB):
            raise FileNotFoundError(f"{HOST_LIB} not found: run `make -C {LIB_DIR}`")
        L = C.CDLL(HOST_LIB)
        vp, i = C.c_void_p, C.c_int
        L.abh_create.restype, L.abh_create.argtypes = vp, [C.POINTER(CConfig), i]
        L.abh_run.restype, L.abh_run.argtypes = i, [vp, C.POINTER(vp), C.POINTER(C.c_size_t), i]
        L.abh_batches.restype, L.abh_batches.argtypes = i, [vp, i]
        for f in ("abh_waveout", "abh_iq_out", "abh_axc"):
            getattr(L, f).restype, getattr(L, f).argtypes = vp, [vp, i]
        L.abh_overflows.restype, L.abh_overflows.argtypes = C.c_size_t, [vp, i]
        L.abh_overruns.restype, L.abh_overruns.argtypes = C.c_size_t, [vp, i]
        L.abh_active_counter.restype, L.abh_active_counter.argtypes = C.c_size_t, [vp, i, i]
        L.abh_last_error.restype, L.abh_last_error.argtypes = C.c_char_p, []
        L.abh_destroy.restype, L.abh_destroy.argtypes = None, [vp]
        L.abh_run_pattern.restype, L.abh_run_pattern.argtypes = i, [vp, C.POINTER(vp), C.POINTER(C.c_size_t), C.c_long, C.c_double, i]
        L.abh_pattern_selftest.restype = C.c_long
        L.abh_pattern_selftest.argtypes = [i, i, C.c_size_t, vp, C.c_size_t, C.c_long, C.c_double, i, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
        L.abh_set_freqlist.restype, L.abh_set_freqlist.argtypes = i, [vp, i, i, i, vp, i]
        L.abh_set_mixers.restype, L.abh_set_mixers.argtypes = i, [vp, i, C.POINTER(C.c_int32), vp]
        L.abh_add_rawfile.restype, L.abh_add_rawfile.argtypes = i, [vp, i, i, C.c_char_p]
        L.abh_mixer_batches.restype, L.abh_mixer_batches.argtypes = i, [vp, i]
        for f in ("abh_mixer_left", "abh_mixer_right", "abh_mixer_axc"):
            getattr(L, f).restype, getattr(L, f).argtypes = vp, [vp, i]
        L.abh_mixer_overruns.restype, L.abh_mixer_overruns.argtypes = C.c_size_t, [vp, i]
        L.abh_mixer_is_gpu.restype, L.abh_mixer_is_gpu.argtypes = i, [vp, i]
        L.abh_failed_calls.restype, L.abh_failed_calls.argtypes = i, [vp, i]
        _L = L
    return _L


def run_host_pipeline(cfg: Config, raws: List[np.ndarray], max_batches_per_run: int = 2, timeout_s: int = 120, freqlists=None,
                      pattern=None, mixers=None, rawfiles=None, mixer_out=None):
    """Feed `raws` through input rings into demodulate_b200() and collect what the output thread would see.
    `freqlists` = [(dev, chan, [Channel, ...], freq_idx)] installs scan-mode frequency lists before the thread starts.
    `pattern` = (repeat, speedup): `raws` are blocks replayed by the "pattern" input plugin instead of being fed once.
    `mixers` = [[(dev, chan, ampfactor, balance), ...], ...] creates mixer_t objects + the O_MIXER outputs of their input
    channels; what the output-thread stand-in takes out of mixer_t.channel (CH_READY -> CH_DIRTY) lands in `mixer_out`
    (a list that receives one dict per mixer: left[nb, B], right[nb, B], axc[nb], overruns, is_gpu).
    `rawfiles` = [(dev, chan, path)]: O_RAWFILE stand-in, one .cf32 per entry.
    Returns per device (waveout[C, nb*B], iq_out[C, nb*B] complex64, axc[nb, C], info dict)."""
    L = load()
    ccfg, keep = cfg.to_c()
    h = L.abh_create(C.byref(ccfg), max_batches_per_run)
    for (dev, chan, freqs, idx) in (freqlists or []):
        from .config import channels_to_c
        arr = channels_to_c(freqs)
        keep.append(arr)
        assert L.abh_set_freqlist(h, dev, chan, len(freqs), C.cast(arr, C.c_void_p), idx) == 0
    if mixers:
        from .lib import CMixerInput
        offs, flat = [0], []
        for m in mixers:
            flat.extend(m)
            offs.append(len(flat))
        arr = (CMixerInput * max(1, len(flat)))()
        for k, (d, c, a, b) in enumerate(flat):
            arr[k] = CMixerInput(d, c, a, b)
        co = (C.c_int32 * len(offs))(*offs)
        assert L.abh_set_mixers(h, len(mixers), co, C.cast(arr, C.c_void_p)) == 0
    for (dev, chan, path) in (rawfiles or []):
        assert L.abh_add_rawfile(h, dev, chan, str(path).encode()) == 0
    raws = [np.ascontiguousarray(r) for r in raws]
    ptrs = (C.c_void_p * len(raws))(*[r.ctypes.data for r in raws])
    sizes = (C.c_size_t * len(raws))(*[r.nbytes for r in raws])
    if pattern is not None:
        rc = L.abh_run_pattern(h, ptrs, sizes, int(pattern[0]), float(pattern[1]), timeout_s)
    else:
        rc = L.abh_run(h, ptrs, sizes, timeout_s)
    if rc != 0:
        msg = L.abh_last_error().decode()
        L.abh_destroy(h)
        raise RuntimeError(f"host pipeline failed rc={rc}: {msg}")
    B = cfg.wave_batch
    out = []
    for d in range(len(raws)):
        Cn = len(cfg.devices[d].channels)
        nb = L.abh_batches(h, d)
        wo = np.ctypeslib.as_array(C.cast(L.abh_waveout(h, d), C.POINTER(C.c_float)), shape=(nb, Cn, B)).copy() if nb else np.zeros((0, Cn, B), np.float32)
        iq = np.ctypeslib.as_array(C.cast(L.abh_iq_out(h, d), C.POINTER(C.c_float)), shape=(nb, Cn, 2 * B)).copy() if nb else np.zeros((0, Cn, 2 * B), np.float32)
        ax = np.ctypeslib.as_array(C.cast(L.abh_axc(h, d), C.POINTER(C.c_uint8)), shape=(nb, Cn)).copy() if nb else np.zeros((0, Cn), np.uint8)
        info = {"overflows": int(L.abh_overflows(h, d)), "overruns": int(L.abh_overruns(h, d)),
                "active": [int(L.abh_active_counter(h, d, c)) for c in range(Cn)], "disable_device_outputs_calls": int(L.abh_failed_calls(h, d))}
        out.append((wo.transpose(1, 0, 2).reshape(Cn, nb * B), iq.transpose(1, 0, 2).reshape(Cn, nb * 2 * B).view(np.complex64), ax, info))
    if mixers and mixer_out is not None:
        for m in range(len(mixers)):
            nb = L.abh_mixer_batches(h, m)
            grab = lambda fn, typ, shape: (np.ctypeslib.as_array(C.cast(fn(h, m), C.POINTER(typ)), shape=shape).copy() if nb else np.zeros(shape, np.float32))
            mixer_out.append({"left": grab(L.abh_mixer_left, C.c_float, (nb, B)), "right": grab(L.abh_mixer_right, C.c_float, (nb, B)),
                              "axc": grab(L.abh_mixer_axc, C.c_uint8, (nb,)), "overruns": int(L.abh_mixer_overruns(h, m)),
                              "is_gpu": bool(L.abh_mixer_is_gpu(h, m))})
    L.abh_destroy(h)
    return out


def pattern_selftest(block: np.ndarray, sfmt: int, sample_rate: int, fft_size: int, repeat: int, speedup: float, consumer_delay_us: int = 0):
    """CPU-only: the "pattern" input plugin into a ring drained by a checking consumer.  Returns (mismatches, bytes consumed, overflows)."""
    L = load()
    block = np.ascontiguousarray(block)
    consumed, overflows = C.c_size_t(0), C.c_size_t(0)
    bad = L.abh_pattern_selftest(sfmt, sample_rate, fft_size, block.ctypes.data, block.nbytes, repeat, float(speedup), consumer_delay_us,
                                 C.byref(consumed), C.byref(overflows))
    return int(bad), int(consumed.value), int(overflows.value)
