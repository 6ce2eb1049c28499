"""ctypes binding of the product: rtlsdr-airband_b200/libairband_b200.so (C ABI in include/airband_b200.h).

There is no fallback of any kind here: if the shared library is missing, or no sm_90 (H100) device is present,
construction raises.  (The CPU oracle under oracle/ is test infrastructure and is never imported from here.)
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence, Tuple

import numpy as np

from .config import CConfig, CSquelchStats, Config

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_DIR = os.path.abspath(os.path.join(_HERE, "..", ".."))
LIB_PATH = os.environ.get("ABG_LIB_PATH") or os.path.join(LIB_DIR, "libairband_b200.so")  # override: A/B-testing builds

# every symbol include/airband_b200.h declares (tests check the library exports all of them)
SYMBOLS = [
    "abg_last_error", "abg_version", "abg_create", "abg_destroy", "abg_wave_batch", "abg_hop", "abg_push",
    "abg_batches_available", "abg_run", "abg_sync", "abg_join", "abg_batches_ready", "abg_fetch_batch", "abg_fetch_batches", "abg_get_stats", "abg_set_bin",
    "abg_resident_load", "abg_run_resident", "abg_set_stream", "abg_launch_count", "abg_mixers_configure",
    "abg_fetch_mixer_batch", "abg_mixer_device_buffers", "abg_debug_frame", "abg_last_run_times", "abg_debug_timeline", "abg_scan_configure", "abg_scan_select", "abg_host_register", "abg_host_unregister", "abg_ingest_sync", "abg_fft_path", "abg_debug_tc_table", "abg_debug_inject_wavein", "abg_debug_k1tc_trace", "abg_debug_k2_stats",
    "abg_debug_run_outputs", "abg_debug_k1_outputs", "abg_spectrum_configure", "abg_fetch_spectrum", "abg_debug_spectrum_time",
    "abg_carrier_configure", "abg_fetch_carrier", "abg_debug_carrier_time",
    "abg_input_meter_configure", "abg_fetch_input_levels", "abg_debug_input_meter_time",
]


class COptions(C.Structure):
    _fields_ = [
        ("cuda_device", C.c_int32),
        ("max_batches_per_run", C.c_int32),
        ("input_capacity_batches", C.c_int32),
        ("fft_mode", C.c_int32),
        ("reserved", C.c_int32 * 4),
    ]


class CMixerInput(C.Structure):
    _fields_ = [("dev", C.c_int32), ("chan", C.c_int32), ("ampfactor", C.c_float), ("balance", C.c_float)]


class CInputLevels(C.Structure):
    """abg_input_levels: one input level meter reading (definition in airband_b200.h)."""
    _fields_ = [
        ("batch_seq", C.c_uint64),
        ("n_samples", C.c_uint64),
        ("sum", C.c_double * 2),
        ("sum_sq", C.c_double * 2),
        ("sum_iq", C.c_double),
        ("peak", C.c_float * 2),
        ("hist", (C.c_uint32 * 256) * 2),
    ]


class AbgError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"airband_b200 error {code}: {msg}")
        self.code = code


_LIB = None


def load():
    """dlopen the engine library (raises FileNotFoundError with build instructions if it has not been built)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise FileNotFoundError(f"{LIB_PATH} not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
                                f"(or `make -C {LIB_DIR}`) first. There is no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    L.abg_last_error.restype, L.abg_last_error.argtypes = C.c_char_p, []
    L.abg_version.restype, L.abg_version.argtypes = C.c_char_p, []
    L.abg_create.restype, L.abg_create.argtypes = i, [C.POINTER(CConfig), C.POINTER(COptions), C.POINTER(vp)]
    L.abg_destroy.restype, L.abg_destroy.argtypes = None, [vp]
    L.abg_wave_batch.restype, L.abg_wave_batch.argtypes = i, [vp]
    L.abg_hop.restype, L.abg_hop.argtypes = i, [vp, i]
    L.abg_push.restype, L.abg_push.argtypes = i, [vp, i, vp, C.c_size_t]
    L.abg_batches_available.restype, L.abg_batches_available.argtypes = i, [vp, i]
    L.abg_run.restype, L.abg_run.argtypes = i, [vp, i]
    L.abg_sync.restype, L.abg_sync.argtypes = i, [vp]
    L.abg_join.restype, L.abg_join.argtypes = i, [vp]
    L.abg_batches_ready.restype, L.abg_batches_ready.argtypes = i, [vp, i]
    L.abg_fetch_batch.restype, L.abg_fetch_batch.argtypes = i, [vp, i, vp, vp, vp]
    L.abg_fetch_batches.restype, L.abg_fetch_batches.argtypes = i, [vp, i, i, vp, vp, vp]
    L.abg_get_stats.restype, L.abg_get_stats.argtypes = i, [vp, i, i, C.POINTER(CSquelchStats)]
    L.abg_set_bin.restype, L.abg_set_bin.argtypes = i, [vp, i, i, i]
    L.abg_resident_load.restype, L.abg_resident_load.argtypes = i, [vp, i, vp, C.c_size_t]
    L.abg_run_resident.restype, L.abg_run_resident.argtypes = i, [vp, i]
    L.abg_set_stream.restype, L.abg_set_stream.argtypes = i, [vp, vp]
    L.abg_launch_count.restype, L.abg_launch_count.argtypes = C.c_uint64, [vp]
    L.abg_mixers_configure.restype, L.abg_mixers_configure.argtypes = i, [vp, i, C.POINTER(C.c_int32), C.POINTER(CMixerInput)]
    L.abg_fetch_mixer_batch.restype, L.abg_fetch_mixer_batch.argtypes = i, [vp, i, vp, vp, C.POINTER(C.c_int)]
    L.abg_mixer_device_buffers.restype, L.abg_mixer_device_buffers.argtypes = i, [vp, C.POINTER(vp), C.POINTER(vp)]
    L.abg_debug_frame.restype, L.abg_debug_frame.argtypes = i, [vp, i, vp, vp]
    L.abg_debug_run_outputs.restype, L.abg_debug_run_outputs.argtypes = i, [vp, vp, vp, vp]
    L.abg_debug_k1_outputs.restype, L.abg_debug_k1_outputs.argtypes = i, [vp, vp, vp, vp]
    L.abg_last_run_times.restype, L.abg_last_run_times.argtypes = i, [vp, C.POINTER(C.c_float)]
    L.abg_host_register.restype, L.abg_host_register.argtypes = i, [vp, C.c_size_t]
    L.abg_host_unregister.restype, L.abg_host_unregister.argtypes = i, [vp]
    L.abg_ingest_sync.restype, L.abg_ingest_sync.argtypes = i, [vp]
    L.abg_scan_configure.restype, L.abg_scan_configure.argtypes = i, [vp, i, i, i, vp]
    L.abg_scan_select.restype, L.abg_scan_select.argtypes = i, [vp, i, i, i]
    L.abg_debug_timeline.restype, L.abg_debug_timeline.argtypes = i, [vp, i, C.POINTER(C.c_float)]
    L.abg_fft_path.restype, L.abg_fft_path.argtypes = i, [vp, i]
    L.abg_debug_inject_wavein.restype, L.abg_debug_inject_wavein.argtypes = i, [vp, i, i, vp, vp]
    L.abg_debug_k1tc_trace.restype, L.abg_debug_k1tc_trace.argtypes = i, [vp]
    L.abg_debug_k2_stats.restype, L.abg_debug_k2_stats.argtypes = i, [vp]
    L.abg_spectrum_configure.restype, L.abg_spectrum_configure.argtypes = i, [vp, i, i]
    L.abg_fetch_spectrum.restype = i
    L.abg_fetch_spectrum.argtypes = [vp, i, vp, C.POINTER(C.c_uint64), C.POINTER(C.c_int32)]
    L.abg_debug_spectrum_time.restype, L.abg_debug_spectrum_time.argtypes = i, [vp, C.POINTER(C.c_float)]
    L.abg_carrier_configure.restype, L.abg_carrier_configure.argtypes = i, [vp, i, i]
    L.abg_fetch_carrier.restype, L.abg_fetch_carrier.argtypes = i, [vp, i, vp, vp, C.POINTER(C.c_uint64)]
    L.abg_debug_carrier_time.restype, L.abg_debug_carrier_time.argtypes = i, [vp, C.POINTER(C.c_float)]
    L.abg_input_meter_configure.restype, L.abg_input_meter_configure.argtypes = i, [vp, i, i]
    L.abg_fetch_input_levels.restype, L.abg_fetch_input_levels.argtypes = i, [vp, i, C.POINTER(CInputLevels)]
    L.abg_debug_input_meter_time.restype, L.abg_debug_input_meter_time.argtypes = i, [vp, C.POINTER(C.c_float)]
    L.abg_debug_tc_table.restype = i
    L.abg_debug_tc_table.argtypes = [i, i, i, f, i, vp, i, vp, vp, C.c_size_t, vp, C.POINTER(C.c_double)]
    _LIB = L
    return L


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class Engine:
    """One engine = one GPU's contiguous range of devices[] (a demod_params_t{device_start, device_end})."""

    def __init__(self, cfg: Config, *, cuda_device: int = -1, max_batches_per_run: int = 4, input_capacity_batches: int = 0,
                 fft_mode: int = 0):
        self.L = load()
        self.cfg = cfg
        ccfg, self._keep = cfg.to_c()
        opt = COptions(cuda_device, max_batches_per_run, input_capacity_batches, fft_mode)
        h = C.c_void_p()
        self.h = None
        self._chk(self.L.abg_create(C.byref(ccfg), C.byref(opt), C.byref(h)))
        self.h = h
        self.B = self.L.abg_wave_batch(self.h)
        self.nbmax = max_batches_per_run

    def _chk(self, rc: int) -> int:
        if rc < 0:
            raise AbgError(rc, (self.L.abg_last_error() or b"").decode())
        return rc

    def close(self):
        if self.h:
            self.L.abg_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- streaming path -------------------------------------------------------------------------------------------
    def push(self, dev: int, raw: np.ndarray) -> None:
        raw = np.ascontiguousarray(raw)
        self._chk(self.L.abg_push(self.h, dev, _ptr(raw), raw.nbytes))

    def push_ptr(self, dev: int, ptr: int, nbytes: int) -> None:
        self._chk(self.L.abg_push(self.h, dev, C.c_void_p(ptr), nbytes))

    def batches_available(self, dev: int) -> int:
        return self._chk(self.L.abg_batches_available(self.h, dev))

    def run(self, max_batches: int = -1) -> int:
        return self._chk(self.L.abg_run(self.h, max_batches))

    def sync(self) -> None:
        self._chk(self.L.abg_sync(self.h))

    def join(self) -> None:
        self._chk(self.L.abg_join(self.h))

    def batches_ready(self, dev: int) -> int:
        return self._chk(self.L.abg_batches_ready(self.h, dev))

    def fetch(self, dev: int, want_iq: bool = True) -> Optional[Tuple[np.ndarray, np.ndarray, np.ndarray]]:
        Cn = len(self.cfg.devices[dev].channels)
        wo = np.empty((Cn, self.B), np.float32)
        iq = np.empty((Cn, 2 * self.B), np.float32) if want_iq else None
        ax = np.empty(Cn, np.uint8)
        if not self._chk(self.L.abg_fetch_batch(self.h, dev, _ptr(wo), _ptr(iq), _ptr(ax))):
            return None
        return wo, (iq.view(np.complex64) if iq is not None else None), ax

    def fetch_into(self, dev: int, wo: np.ndarray, ax: np.ndarray) -> bool:
        return bool(self._chk(self.L.abg_fetch_batch(self.h, dev, _ptr(wo), None, _ptr(ax))))

    def fetch_many_into(self, dev: int, max_batches: int, wo: np.ndarray, ax: np.ndarray) -> int:
        """Pop up to max_batches batches of a device into wo[n, C, B] / ax[n, C]; returns how many."""
        return self._chk(self.L.abg_fetch_batches(self.h, dev, max_batches, _ptr(wo), None, _ptr(ax)))

    def fetch_all(self, dev: int):
        wos, iqs, axs = [], [], []
        while True:
            r = self.fetch(dev)
            if r is None:
                break
            wos.append(r[0]); iqs.append(r[1]); axs.append(r[2])
        Cn = len(self.cfg.devices[dev].channels)
        if not wos:
            return np.zeros((Cn, 0), np.float32), np.zeros((Cn, 0), np.complex64), np.zeros((0, Cn), np.uint8)
        return np.concatenate(wos, 1), np.concatenate(iqs, 1), np.stack(axs, 0)

    def stats(self, dev: int, chan: int) -> CSquelchStats:
        s = CSquelchStats()
        self._chk(self.L.abg_get_stats(self.h, dev, chan, C.byref(s)))
        return s

    def fft_path(self, dev: int) -> int:
        """1 full-spectrum FFT, 2 output-pruned FFT, 3 tensor-core DFT (which K1 the device's frames go through)."""
        return self._chk(self.L.abg_fft_path(self.h, dev))

    def set_bin(self, dev: int, chan: int, bin_: int) -> None:
        self._chk(self.L.abg_set_bin(self.h, dev, chan, bin_))

    # ---- resident (benchmark) path -------------------------------------------------------------------------------
    def resident_load(self, dev: int, raw: np.ndarray) -> None:
        raw = np.ascontiguousarray(raw)
        self._chk(self.L.abg_resident_load(self.h, dev, _ptr(raw), raw.nbytes))

    def resident_bytes_needed(self, dev: int) -> int:
        d = self.cfg.devices[dev]
        hop_b = self.cfg.hop(dev) * 2 * d.bytes_per_sample
        return (self.nbmax * self.B + 100 - 1) * hop_b + self.cfg.fft_size * 2 * d.bytes_per_sample

    def run_resident(self, n_batches: int) -> int:
        return self._chk(self.L.abg_run_resident(self.h, n_batches))

    def run_outputs(self):
        """(wout[G, P], axc[max_batches_per_run, G]) of the most recent run, resident runs included (abg_debug_run_outputs)."""
        dims = np.zeros(4, np.int32)
        self._chk(self.L.abg_debug_run_outputs(self.h, _ptr(dims), None, None))
        G, Gp, P, nb = (int(x) for x in dims)
        wout = np.empty((Gp, P), np.float32)
        axc = np.empty((nb, Gp), np.uint8)
        self._chk(self.L.abg_debug_run_outputs(self.h, _ptr(dims), _ptr(wout), _ptr(axc)))
        return wout[:G], axc[:, :G]

    def k1_outputs(self):
        """(win[rows, G] float32, iqin[rows, G] complex64) as K1 of the most recent run stored them, rows = max_batches_per_run *
        WAVE_BATCH starting at the run's first batch (abg_debug_k1_outputs); a device's rows beyond its batches of that run are
        stale."""
        dims = np.zeros(4, np.int32)
        self._chk(self.L.abg_debug_k1_outputs(self.h, _ptr(dims), None, None))
        G, Gp, rows, _ = (int(x) for x in dims)
        win = np.empty((rows, Gp), np.float32)
        iqin = np.empty((rows, 2 * Gp), np.float32)
        self._chk(self.L.abg_debug_k1_outputs(self.h, _ptr(dims), _ptr(win), _ptr(iqin)))
        return win[:, :G], iqin.view(np.complex64)[:, :G]

    def set_stream(self, cuda_stream_ptr: int) -> None:
        self._chk(self.L.abg_set_stream(self.h, C.c_void_p(cuda_stream_ptr)))

    def last_run_times(self):
        """(k1_ms, k2_ms, tail_ms, total_ms) of the most recent run, from CUDA events on the engine's stream."""
        a = (C.c_float * 4)()
        self._chk(self.L.abg_last_run_times(self.h, a))
        return tuple(float(x) for x in a)

    def timeline(self, n_runs: int = 8) -> np.ndarray:
        """[n_runs, 5] ms: K1 start, K1 end, K2 start, K2 end, end of run, relative to the oldest run's K1 start."""
        a = (C.c_float * (5 * n_runs))()
        self._chk(self.L.abg_debug_timeline(self.h, n_runs, a))
        return np.array(a, dtype=np.float32).reshape(n_runs, 5)

    def scan_configure(self, dev: int, chan: int, freqs) -> None:
        """Install a scan-mode frequency list (list of config.Channel); entry 0 becomes current."""
        from .config import channels_to_c
        arr = channels_to_c(freqs)
        self._chk(self.L.abg_scan_configure(self.h, dev, chan, len(freqs), C.cast(arr, C.c_void_p)))

    def scan_select(self, dev: int, chan: int, freq_idx: int) -> None:
        self._chk(self.L.abg_scan_select(self.h, dev, chan, freq_idx))

    def launch_count(self) -> int:
        return int(self.L.abg_launch_count(self.h))

    # ---- band spectrum monitor -----------------------------------------------------------------------------------
    def spectrum_configure(self, dev: int, stride: int) -> None:
        """Batch-averaged power spectrum of a device every `stride`-th frame of each batch (0 = off, the default); applies
        to batches enqueued by later runs.  `default_stride(cfg, dev)` selects non-overlapping frames."""
        self._chk(self.L.abg_spectrum_configure(self.h, dev, stride))

    def fetch_spectrum(self, dev: int) -> Optional[Tuple[np.ndarray, int, int]]:
        """Oldest unfetched spectrum of a device: (power[fft_size] float32, batch_seq, n_frames), or None.  Lossy: at most
        max_batches_per_run + 2 are kept per device."""
        p = np.empty(self.cfg.fft_size, np.float32)
        seq, nf = C.c_uint64(0), C.c_int32(0)
        if not self._chk(self.L.abg_fetch_spectrum(self.h, dev, _ptr(p), C.byref(seq), C.byref(nf))):
            return None
        return p, int(seq.value), int(nf.value)

    def spectrum_time(self) -> float:
        """ms of the spectrum kernel in the most recent run (CUDA events on the K1 stream); 0 if it computed none."""
        ms = C.c_float(0.0)
        self._chk(self.L.abg_debug_spectrum_time(self.h, C.byref(ms)))
        return float(ms.value)

    # ---- carrier frequency meter ---------------------------------------------------------------------------------
    def carrier_configure(self, dev: int, on: bool) -> None:
        """Lag-one correlation and energy of every channel's bin per batch (off by default); applies to batches enqueued
        by later runs.  `carrier_offset_hz` turns a reading into the carrier's frequency error."""
        self._chk(self.L.abg_carrier_configure(self.h, dev, int(on)))

    def fetch_carrier(self, dev: int) -> Optional[Tuple[np.ndarray, np.ndarray, int]]:
        """Oldest unfetched meter reading of a device: (lag1 complex64[C], energy float32[C], batch_seq), or None.  Lossy:
        at most max_batches_per_run + 2 are kept per device."""
        Cn = len(self.cfg.devices[dev].channels) if 0 <= dev < len(self.cfg.devices) else 0  # (a bad index: the C call reports it)
        lag1 = np.empty(2 * Cn, np.float32)
        energy = np.empty(Cn, np.float32)
        seq = C.c_uint64(0)
        if not self._chk(self.L.abg_fetch_carrier(self.h, dev, _ptr(lag1), _ptr(energy), C.byref(seq))):
            return None
        return lag1.view(np.complex64), energy, int(seq.value)

    def carrier_time(self) -> float:
        """ms of the carrier meter kernel in the most recent run (CUDA events on the K1 stream); 0 if it metered nothing."""
        ms = C.c_float(0.0)
        self._chk(self.L.abg_debug_carrier_time(self.h, C.byref(ms)))
        return float(ms.value)

    # ---- input level meter ---------------------------------------------------------------------------------------
    def input_meter_configure(self, dev: int, on: bool) -> None:
        """Histogram, peak and moments of a device's I and Q input levels per batch (off by default); applies to batches
        enqueued by later runs.  `input_levels` turns a reading into DC offset, dBFS, clipping and I/Q balance."""
        self._chk(self.L.abg_input_meter_configure(self.h, dev, int(on)))

    def fetch_input_levels(self, dev: int) -> Optional[dict]:
        """Oldest unfetched reading of a device, or None: a dict of batch_seq, n_samples (int), sum, sum_sq (float64[2]),
        sum_iq (float), peak (float32[2]) and hist (uint32[2, 256]).  Lossy: at most max_batches_per_run + 2 are kept per
        device."""
        r = CInputLevels()
        if not self._chk(self.L.abg_fetch_input_levels(self.h, dev, C.byref(r))):
            return None
        return dict(batch_seq=int(r.batch_seq), n_samples=int(r.n_samples), sum=np.array(r.sum, np.float64),
                    sum_sq=np.array(r.sum_sq, np.float64), sum_iq=float(r.sum_iq), peak=np.array(r.peak, np.float32),
                    hist=np.ctypeslib.as_array(r.hist).astype(np.uint32).reshape(2, 256))

    def input_meter_time(self) -> float:
        """ms of the input meter kernel in the most recent run (CUDA events on the K1 stream); 0 if it metered nothing."""
        ms = C.c_float(0.0)
        self._chk(self.L.abg_debug_input_meter_time(self.h, C.byref(ms)))
        return float(ms.value)

    # ---- mixers ---------------------------------------------------------------------------------------------------
    def configure_mixers(self, mixers: Sequence[Sequence[Tuple[int, int, float, float]]]) -> None:
        """mixers[m] = [(dev, chan, ampfactor, balance), ...]"""
        offs = [0]
        flat = []
        for m in mixers:
            flat.extend(m)
            offs.append(len(flat))
        arr = (CMixerInput * max(1, len(flat)))()
        for k, (d, c, a, b) in enumerate(flat):
            arr[k] = CMixerInput(d, c, a, b)
        co = (C.c_int32 * len(offs))(*offs)
        self._chk(self.L.abg_mixers_configure(self.h, len(mixers), co, arr))

    def fetch_mixer(self, mixer: int):
        left = np.empty(self.B, np.float32)
        right = np.empty(self.B, np.float32)
        sig = C.c_int(0)
        if not self._chk(self.L.abg_fetch_mixer_batch(self.h, mixer, _ptr(left), _ptr(right), C.byref(sig))):
            return None
        return left, right, bool(sig.value)

    def mixer_device_buffers(self) -> Tuple[int, int]:
        a, b = C.c_void_p(), C.c_void_p()
        self._chk(self.L.abg_mixer_device_buffers(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def inject_wavein(self, dev: int, wavein: np.ndarray, iq: Optional[np.ndarray] = None) -> int:
        """Stage tap: wavein[C, n_batches * B] straight into the demodulation state machine (K1 skipped), with iq[C,
        n_batches * B] (complex64) as the X[bin] values of the same frames for channels that need raw I/Q."""
        w = np.ascontiguousarray(wavein, np.float32)
        assert w.ndim == 2 and w.shape[1] % self.B == 0
        q = None if iq is None else np.ascontiguousarray(iq, np.complex64)
        assert q is None or q.shape == w.shape
        return self._chk(self.L.abg_debug_inject_wavein(self.h, dev, w.shape[1] // self.B, _ptr(w), _ptr(q)))

    # ---- stage tap ------------------------------------------------------------------------------------------------
    def debug_frame(self, dev: int, raw_frame: np.ndarray) -> np.ndarray:
        out = np.empty(2 * self.cfg.fft_size, np.float32)
        raw_frame = np.ascontiguousarray(raw_frame)
        self._chk(self.L.abg_debug_frame(self.h, dev, _ptr(raw_frame), _ptr(out)))
        return out.view(np.complex64)


def default_stride(cfg: Config, dev: int) -> int:
    """ceil(fft_size / hop): the spectrum stride that selects non-overlapping frames of a device."""
    return -(-cfg.fft_size // cfg.hop(dev))


def spectrum_dbfs(power: np.ndarray, fft_size: int) -> np.ndarray:
    """level_to_dBFS(sqrtf(P)) per bin (reference src/util.cpp:169-180), the scale of abg_squelch_stats' *_dbfs fields:
    min(0, 20*log10f(level / fft_size) + 7.54 + 10*log10f(fft_size / 2) - 2.38), in float32.  A zero bin gives -inf."""
    f32 = np.float32
    level = np.sqrt(np.asarray(power, np.float32))
    offset = f32(f32(7.54) + f32(10.0) * np.log10(f32(fft_size // 2))) - f32(2.38)
    with np.errstate(divide="ignore"):
        db = f32(20.0) * np.log10(level / f32(fft_size)) + offset
    return np.minimum(f32(0.0), db.astype(np.float32))


def carrier_offset_hz(lag1, channel_offset_hz, sample_rate: float, hop: int) -> np.ndarray:
    """Carrier frequency error in Hz relative to the configured channel from a carrier meter reading (definition in
    airband_b200.h): wrap(arg(R) / (2 pi) - channel_offset_hz * hop / sample_rate) * sample_rate / hop, wrapped to
    [-0.5, 0.5) frames, i.e. unambiguous within +-sample_rate / (2 hop).  channel_offset_hz = freq - centerfreq of the
    channel (or of the scan entry the batch used); hop = abg_hop() / Config.hop(dev).  Arrays broadcast."""
    cyc = np.angle(np.asarray(lag1, np.complex128)) / (2.0 * np.pi) - np.asarray(channel_offset_hz, np.float64) * hop / sample_rate
    return (cyc - np.floor(cyc + 0.5)) * sample_rate / hop


def input_levels(reading: dict) -> dict:
    """What an operator reads off an input level meter reading (Engine.fetch_input_levels; definition in airband_b200.h),
    per component k = 0 (I), 1 (Q) where an array:
      dc_offset           mean v_k, in full scale
      mean_square_dbfs    10 log10(mean v_k^2); a full-scale sine reads -3.01 dBFS, and the DC offset counts
      full_scale_fraction (hist[k][0] + hist[k][255]) / n: the components at the ends of the range (8-bit: clipped codes)
      codes_in_use        non-empty bins (8-bit: distinct ADC codes)
      imbalance_db        10 log10(var_I / var_Q)
      phase_skew_deg      asin(cov_IQ / sqrt(var_I var_Q)) in degrees; I = cos, Q = sin(. + phi) reads phi
    Variances and the covariance are about the means."""
    n = float(reading["n_samples"])
    s = np.asarray(reading["sum"], np.float64)
    ss = np.asarray(reading["sum_sq"], np.float64)
    h = np.asarray(reading["hist"]).reshape(2, 256)
    mean = s / n
    ms = ss / n
    var = ms - mean * mean
    cov = float(reading["sum_iq"]) / n - mean[0] * mean[1]
    with np.errstate(divide="ignore", invalid="ignore"):
        ms_db = 10.0 * np.log10(ms)
        imb = float(10.0 * np.log10(var[0] / var[1]))
        skew = float(np.degrees(np.arcsin(np.clip(cov / np.sqrt(var[0] * var[1]), -1.0, 1.0))))
    return dict(dc_offset=mean, mean_square_dbfs=ms_db, full_scale_fraction=(h[:, 0] + h[:, 255]).astype(np.float64) / n,
                codes_in_use=np.count_nonzero(h, axis=1), imbalance_db=imb, phase_skew_deg=skew)


TC_PLAN_FIELDS = ("eligible", "K", "HC", "S", "NC", "ND", "C2p", "KBS", "NSTB", "acc_regs", "smem_bytes", "halo", "consumer_warpgroups", "pps")


def tc_plan(fft_size: int, sfmt: int, hop_bytes: int, n_channels: int, digits: int = 4) -> dict:
    """Host-only: the tensor-core K1's geometry for a launch group whose largest device has n_channels channels
    (abg_debug_tc_table with no table); plan["eligible"] == 0 when the group would use the FP32 kernels."""
    plan = np.zeros(len(TC_PLAN_FIELDS), np.int32)
    load().abg_debug_tc_table(fft_size, sfmt, hop_bytes, 1.0, n_channels, None, digits, _ptr(plan), None, 0, None, None)
    return dict(zip(TC_PLAN_FIELDS, (int(x) for x in plan)))


def tc_table(fft_size: int, sfmt: int, hop_bytes: int, bins: Sequence[int], digits: int = 4, fullscale: float = 1.0):
    """Host-only view of the tensor-core K1's plan and coefficient table (abg_debug_tc_table).  Returns (plan dict,
    tab int8[K/32, 2, NC, 16], sq int64[C2p], cscale) or (plan, None, None, None) when the shape is not eligible."""
    L = load()
    b = np.asarray(bins, np.int32)
    pd = tc_plan(fft_size, sfmt, hop_bytes, len(b), digits)
    if not pd["eligible"]:
        return pd, None, None, None
    plan = np.zeros(len(TC_PLAN_FIELDS), np.int32)
    tab = np.zeros(pd["K"] * pd["NC"], np.int8)
    sq = np.zeros(pd["C2p"], np.int64)
    cs = C.c_double(0.0)
    rc = L.abg_debug_tc_table(fft_size, sfmt, hop_bytes, fullscale, len(b), _ptr(b), digits, _ptr(plan), _ptr(tab), tab.nbytes, _ptr(sq), C.byref(cs))
    if rc < 0:
        raise AbgError(rc, (L.abg_last_error() or b"").decode())
    return pd, tab.reshape(pd["K"] // 32, 2, pd["NC"], 16), sq, cs.value


def demodulate_all(cfg: Config, raws: List[np.ndarray], *, max_batches_per_run: int = 4, chunk_batches: int = 0, **kw):
    """Push one raw stream per device and run to exhaustion (the file-input use of the path).  Returns per-device
    (waveout[C, n], iq_out[C, n], axc[nb, C]) and the engine."""
    e = Engine(cfg, max_batches_per_run=max_batches_per_run, **kw)
    pos = [0] * len(raws)
    outs = [([], [], []) for _ in raws]
    step_b = chunk_batches or max_batches_per_run
    while True:
        progressed = False
        for d, r in enumerate(raws):
            if pos[d] < r.size:
                hop_items = cfg.hop(d) * 2  # array items per hop (I and Q)
                n = step_b * e.B * hop_items + (100 * hop_items + 2 * cfg.fft_size if pos[d] == 0 else 0)
                e.push(d, r[pos[d]:pos[d] + n])
                pos[d] += n
                progressed = True
        n = e.run(-1)
        for d in range(len(raws)):
            while True:
                got = e.fetch(d)
                if got is None:
                    break
                for k in range(3):
                    outs[d][k].append(got[k])
        if n == 0 and not progressed:
            break
    res = []
    for d in range(len(raws)):
        Cn = len(cfg.devices[d].channels)
        if outs[d][0]:
            res.append((np.concatenate(outs[d][0], 1), np.concatenate(outs[d][1], 1), np.stack(outs[d][2], 0)))
        else:
            res.append((np.zeros((Cn, 0), np.float32), np.zeros((Cn, 0), np.complex64), np.zeros((0, Cn), np.uint8)))
    return res, e
