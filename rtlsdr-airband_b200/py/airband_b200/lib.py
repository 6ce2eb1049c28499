"""ctypes binding of the product: rtlsdr-airband_b200/libairband_b200.so (C ABI in include/airband_b200.h).

There is no fallback of any kind here: if the shared library is missing, or no sm_90 (H100) device is present,
construction raises.  (The CPU oracle under oracle/ is test infrastructure and is never imported from here.)
"""
from __future__ import annotations

import ctypes as C
import functools
import os
from typing import List, Optional, Sequence, Tuple

import numpy as np

from .config import AGC_EXTRA, CChannelCfg, CConfig, CSquelchStats, Config, channels_to_c, make_channel

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_DIR = os.path.abspath(os.path.join(_HERE, "..", ".."))
LIB_PATH = os.environ.get("ABG_LIB_PATH") or os.path.join(LIB_DIR, "libairband_b200.so")  # override: A/B-testing builds

# every symbol include/airband_b200.h declares (tests check the library exports all of them)
SYMBOLS = [
    "abg_last_error", "abg_version", "abg_create", "abg_destroy", "abg_wave_batch", "abg_hop", "abg_push",
    "abg_batches_available", "abg_run", "abg_sync", "abg_join", "abg_batches_ready", "abg_fetch_batch", "abg_fetch_batches", "abg_get_stats", "abg_set_bin",
    "abg_resident_load", "abg_run_resident", "abg_set_stream", "abg_launch_count", "abg_mixers_configure",
    "abg_fetch_mixer_batch", "abg_mixer_device_buffers", "abg_debug_frame", "abg_last_run_times", "abg_debug_timeline", "abg_scan_configure", "abg_scan_select", "abg_host_register", "abg_host_unregister", "abg_ingest_sync", "abg_fft_path", "abg_debug_tc_table", "abg_debug_inject_wavein", "abg_debug_k1tc_trace", "abg_debug_k2_stats",
    "abg_debug_run_outputs", "abg_debug_k1_outputs", "abg_debug_k1_spectra", "abg_spectrum_configure", "abg_fetch_spectrum", "abg_debug_spectrum_time",
    "abg_carrier_configure", "abg_fetch_carrier", "abg_debug_carrier_time",
    "abg_input_meter_configure", "abg_fetch_input_levels", "abg_debug_input_meter_time",
    "abg_subband_configure", "abg_fetch_subband", "abg_debug_subband_time",
    "abg_tone_meter_configure", "abg_tone_meter_set_tones", "abg_fetch_tone_meter", "abg_debug_tone_meter_time",
    "abg_activity_configure", "abg_fetch_activity", "abg_debug_activity_time",
    "abg_history_configure", "abg_history_range", "abg_history_raw", "abg_history_subband", "abg_debug_history_time",
    "abg_history_replay", "abg_debug_replay_time",
    "abg_follow_open", "abg_follow_close", "abg_follow_run", "abg_follow_fetch", "abg_follow_info", "abg_follow_stats",
    "abg_debug_follow_time",
    "abg_history_spectrogram", "abg_history_activity", "abg_debug_history_analysis_time",
    "abg_history_profile", "abg_debug_history_profile_time", "abg_debug_profile_plan",
]

SUBBAND_MAX = 8            # ABG_SUBBAND_MAX: sub-band outputs per device
SUBBAND_MAX_COEFFS = 4096  # ABG_SUBBAND_MAX_COEFFS
TONE_MAX = 64              # ABG_TONE_MAX: tones in the tone meter's list
ACTIVITY_MAX_RECORDS = 4096  # ABG_ACTIVITY_MAX_RECORDS: pieces one activity reading stores
PROFILE_BLOCK = 1024       # ABG_PROFILE_BLOCK: outputs per block of a transmission profile
BURST_OPEN_START, BURST_OPEN_END = 1, 2  # ABG_BURST_OPEN_START / ABG_BURST_OPEN_END
# the tone meter's default list: the reference's standard CTCSS tones (CTCSS::standard_tones, src/ctcss.cpp:87-89)
STANDARD_TONES = (67.0, 69.3, 71.9, 74.4, 77.0, 79.7, 82.5, 85.4, 88.5, 91.5, 94.8, 97.4, 100.0, 103.5, 107.2, 110.9, 114.8,
                  118.8, 123.0, 127.3, 131.8, 136.5, 141.3, 146.2, 150.0, 151.4, 156.7, 159.8, 162.2, 165.5, 167.9, 171.3,
                  173.8, 177.3, 179.9, 183.5, 186.2, 189.9, 192.8, 196.6, 199.5, 203.5, 206.5, 210.7, 218.1, 225.7, 229.1,
                  233.6, 241.8, 250.3, 254.1)


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


class CBurst(C.Structure):
    """abg_burst: one piece (or, after merge_bursts, one burst) of the band activity detector (definition in airband_b200.h)."""
    _fields_ = [
        ("bin", C.c_int32),
        ("flags", C.c_int32),
        ("first_frame", C.c_uint64),
        ("last_frame", C.c_uint64),
        ("n_active", C.c_int32),
        ("peak", C.c_float),
        ("sum", C.c_float),
        ("reserved", C.c_int32),
    ]


class CReplayJob(C.Structure):
    """abg_replay_job: one history replay job (definition in airband_b200.h)."""
    _fields_ = [
        ("dev", C.c_int32),
        ("n_batches", C.c_int32),
        ("first_batch", C.c_uint64),
        ("n_channels", C.c_int32),
        ("channels", C.POINTER(CChannelCfg)),
        ("waveout", C.c_void_p),
        ("iq_out", C.c_void_p),
        ("axcindicate", C.c_void_p),
        ("stats", C.POINTER(CSquelchStats)),
    ]


class CFollowStatus(C.Structure):
    """abg_follow_status: what abg_follow_info reports of a live follow session (definition in airband_b200.h)."""
    _fields_ = [
        ("dev", C.c_int32),
        ("n_channels", C.c_int32),
        ("next_batch", C.c_uint64),
        ("queued", C.c_int32),
        ("lost", C.c_int32),
    ]


class CSpectrogramJob(C.Structure):
    """abg_spectrogram_job: one history spectrogram job (definition in airband_b200.h)."""
    _fields_ = [
        ("dev", C.c_int32),
        ("n_rows", C.c_int32),
        ("first_frame", C.c_uint64),
        ("frames_per_row", C.c_int32),
        ("stride", C.c_int32),
        ("power", C.c_void_p),
    ]


class CActivityJob(C.Structure):
    """abg_activity_job: one history activity job (definition in airband_b200.h); n_bursts and n_truncated are written
    back."""
    _fields_ = [
        ("dev", C.c_int32),
        ("n_batches", C.c_int32),
        ("first_batch", C.c_uint64),
        ("stride", C.c_int32),
        ("hang", C.c_int32),
        ("min_span", C.c_int32),
        ("cap", C.c_int32),
        ("thr", C.c_void_p),
        ("out", C.c_void_p),
        ("n_bursts", C.c_int32),
        ("n_truncated", C.c_int32),
    ]


class CProfile(C.Structure):
    """abg_profile: the sums of one transmission profile (definition in airband_b200.h)."""
    _fields_ = [
        ("n", C.c_int64),
        ("n_tones", C.c_int32),
        ("reserved", C.c_int32),
        ("p1", C.c_double),
        ("p2", C.c_double),
        ("a1", C.c_double),
        ("z", C.c_double * 2),
        ("f1", C.c_double),
        ("f2", C.c_double),
        ("tone_fm", (C.c_double * 2) * TONE_MAX),
        ("tone_am", (C.c_double * 2) * TONE_MAX),
    ]


class CProfileJob(C.Structure):
    """abg_profile_job: one transmission profile job (definition in airband_b200.h)."""
    _fields_ = [
        ("dev", C.c_int32),
        ("decim", C.c_int32),
        ("offset_hz", C.c_double),
        ("n_coeffs", C.c_int32),
        ("n_tones", C.c_int32),
        ("coeffs", C.c_void_p),
        ("first_m", C.c_uint64),
        ("n_out", C.c_int64),
        ("tones", C.c_void_p),
        ("out", C.POINTER(CProfile)),
    ]


# numpy mirror of abg_burst: fetch_activity returns arrays of it, merge_bursts takes and returns them
BURST_DTYPE = np.dtype({"names": [f for f, _ in CBurst._fields_],
                        "formats": ["<i4", "<i4", "<u8", "<u8", "<i4", "<f4", "<f4", "<i4"],
                        "offsets": [getattr(CBurst, f).offset for f, _ in CBurst._fields_], "itemsize": C.sizeof(CBurst)})


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
    L.abg_debug_k1_spectra.restype, L.abg_debug_k1_spectra.argtypes = i, [vp, i, vp, vp]
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
    L.abg_subband_configure.restype, L.abg_subband_configure.argtypes = i, [vp, i, i, C.c_double, i, i, vp]
    L.abg_fetch_subband.restype = i
    L.abg_fetch_subband.argtypes = [vp, i, i, vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_int32)]
    L.abg_debug_subband_time.restype, L.abg_debug_subband_time.argtypes = i, [vp, C.POINTER(C.c_float)]
    L.abg_tone_meter_configure.restype, L.abg_tone_meter_configure.argtypes = i, [vp, i, i]
    L.abg_tone_meter_set_tones.restype, L.abg_tone_meter_set_tones.argtypes = i, [vp, i, vp]
    L.abg_fetch_tone_meter.restype = i
    L.abg_fetch_tone_meter.argtypes = [vp, i, vp, vp, vp, C.POINTER(C.c_uint64), C.POINTER(C.c_int32)]
    L.abg_debug_tone_meter_time.restype, L.abg_debug_tone_meter_time.argtypes = i, [vp, C.POINTER(C.c_float)]
    L.abg_activity_configure.restype, L.abg_activity_configure.argtypes = i, [vp, i, i, i, i, vp]
    L.abg_fetch_activity.restype = i
    L.abg_fetch_activity.argtypes = [vp, i, vp, i, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_uint64), vp]
    L.abg_debug_activity_time.restype, L.abg_debug_activity_time.argtypes = i, [vp, C.POINTER(C.c_float)]
    L.abg_history_configure.restype, L.abg_history_configure.argtypes = i, [vp, i, i]
    L.abg_history_range.restype = i
    L.abg_history_range.argtypes = [vp, i, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    L.abg_history_raw.restype, L.abg_history_raw.argtypes = i, [vp, i, C.c_uint64, C.c_int64, vp]
    L.abg_history_subband.restype = i
    L.abg_history_subband.argtypes = [vp, i, C.c_double, i, i, vp, C.c_uint64, C.c_int64, vp]
    L.abg_debug_history_time.restype, L.abg_debug_history_time.argtypes = i, [vp, C.POINTER(C.c_float)]
    L.abg_history_replay.restype, L.abg_history_replay.argtypes = i, [vp, i, C.POINTER(CReplayJob)]
    L.abg_debug_replay_time.restype, L.abg_debug_replay_time.argtypes = i, [vp, C.POINTER(C.c_float)]
    L.abg_follow_open.restype = i
    L.abg_follow_open.argtypes = [vp, i, C.c_uint64, i, C.POINTER(CChannelCfg), i, C.POINTER(C.c_int32)]
    L.abg_follow_close.restype, L.abg_follow_close.argtypes = i, [vp, C.c_int32]
    L.abg_follow_run.restype, L.abg_follow_run.argtypes = i, [vp, i]
    L.abg_follow_fetch.restype = i
    L.abg_follow_fetch.argtypes = [vp, C.c_int32, i, vp, vp, vp, C.POINTER(C.c_uint64)]
    L.abg_follow_info.restype, L.abg_follow_info.argtypes = i, [vp, C.c_int32, C.POINTER(CFollowStatus)]
    L.abg_follow_stats.restype, L.abg_follow_stats.argtypes = i, [vp, C.c_int32, i, C.POINTER(CSquelchStats)]
    L.abg_debug_follow_time.restype, L.abg_debug_follow_time.argtypes = i, [vp, C.POINTER(C.c_float)]
    L.abg_history_spectrogram.restype, L.abg_history_spectrogram.argtypes = i, [vp, i, C.POINTER(CSpectrogramJob)]
    L.abg_history_activity.restype, L.abg_history_activity.argtypes = i, [vp, i, C.POINTER(CActivityJob)]
    L.abg_debug_history_analysis_time.restype, L.abg_debug_history_analysis_time.argtypes = i, [vp, C.POINTER(C.c_float)]
    L.abg_history_profile.restype, L.abg_history_profile.argtypes = i, [vp, i, C.POINTER(CProfileJob)]
    L.abg_debug_history_profile_time.restype, L.abg_debug_history_profile_time.argtypes = i, [vp, C.POINTER(C.c_float)]
    L.abg_debug_profile_plan.restype = i
    L.abg_debug_profile_plan.argtypes = [i, vp, vp, vp, vp, vp, vp, i, C.POINTER(C.c_int32), vp, i, C.POINTER(C.c_int32)]
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
        self._sb_decim = {}  # (dev, k) -> smallest decimation configured: sizes fetch_subband's buffer

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

    def k1_spectra(self, dev: int) -> np.ndarray:
        """complex64 [batches, fft_size]: the full spectrum of each batch-final frame that K1 of the device's most recent launch
        kept for AFC, natural bin order (abg_debug_k1_spectra; devices with an AFC channel only)."""
        n = np.zeros(1, np.int32)
        self._chk(self.L.abg_debug_k1_spectra(self.h, dev, _ptr(n), None))
        out = np.empty((int(n[0]), 2 * self.cfg.fft_size), np.float32)
        self._chk(self.L.abg_debug_k1_spectra(self.h, dev, _ptr(n), _ptr(out) if out.size else None))
        return out.view(np.complex64)

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

    def _kernel_time(self, debug_time) -> float:
        """ms between a monitor kernel's CUDA events in the most recent run, from its abg_debug_*_time."""
        ms = C.c_float(0.0)
        self._chk(debug_time(self.h, C.byref(ms)))
        return float(ms.value)

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
        return self._kernel_time(self.L.abg_debug_spectrum_time)

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
        return self._kernel_time(self.L.abg_debug_carrier_time)

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
        return self._kernel_time(self.L.abg_debug_input_meter_time)

    # ---- sub-band I/Q outputs ------------------------------------------------------------------------------------
    def subband_configure(self, dev: int, k: int, offset_hz: float, decim: int, coeffs=None) -> None:
        """Output k (0 .. SUBBAND_MAX-1) of a device: the band around offset_hz (from the centre frequency) mixed to 0 Hz,
        filtered by the real FIR `coeffs` and decimated by `decim`, as cf32 (definition in airband_b200.h; `subband_lowpass`
        designs a filter).  decim = 0 switches it off.  Applies to batches enqueued by later runs; a new configuration
        restarts the output."""
        if decim == 0:
            self._chk(self.L.abg_subband_configure(self.h, dev, k, 0.0, 0, 0, None))
            return
        h = None if coeffs is None else np.ascontiguousarray(coeffs, dtype=np.float32)
        self._chk(self.L.abg_subband_configure(self.h, dev, k, float(offset_hz), int(decim), 0 if h is None else h.size, _ptr(h)))
        self._sb_decim[(dev, k)] = min(int(decim), self._sb_decim.get((dev, k), int(decim)))

    def fetch_subband(self, dev: int, k: int) -> Optional[Tuple[np.ndarray, int, int]]:
        """Oldest unfetched batch of output k: (complex64[n], batch_seq, first_index), first_index = m of its first
        output; or None.  Lossy: at most max_batches_per_run + 2 are kept per output."""
        n_in = self.B * self.cfg.hop(dev)
        d = self._sb_decim.get((dev, k), 1)
        buf = np.empty(2 * (-(-n_in // d)), np.float32)
        seq, first, n = C.c_uint64(0), C.c_uint64(0), C.c_int32(0)
        if not self._chk(self.L.abg_fetch_subband(self.h, dev, k, _ptr(buf), C.byref(seq), C.byref(first), C.byref(n))):
            return None
        return buf[:2 * n.value].view(np.complex64).copy(), int(seq.value), int(first.value)

    def subband_time(self) -> float:
        """ms of the sub-band kernel in the most recent run (CUDA events on the K1 stream); 0 if it computed nothing."""
        return self._kernel_time(self.L.abg_debug_subband_time)

    # ---- CTCSS tone meter -----------------------------------------------------------------------------------------
    def tone_meter_configure(self, dev: int, on: bool) -> None:
        """DFT of every channel's audio at each tone of the engine's list, its energy and its non-zero samples, per batch
        (off by default); applies to batches enqueued by later runs, injected ones included.  `ctcss_identify` names the
        tone."""
        self._chk(self.L.abg_tone_meter_configure(self.h, dev, int(on)))

    def tone_meter_set_tones(self, freqs=None) -> None:
        """The engine's tone list (at most TONE_MAX tones, each in (0, wave_rate / 2) Hz) for batches of later runs; None or
        an empty list restores STANDARD_TONES."""
        f = None if freqs is None or len(freqs) == 0 else np.ascontiguousarray(freqs, dtype=np.float32)
        self._chk(self.L.abg_tone_meter_set_tones(self.h, 0 if f is None else f.size, _ptr(f)))

    def fetch_tone_meter(self, dev: int) -> Optional[Tuple[np.ndarray, np.ndarray, np.ndarray, int]]:
        """Oldest unfetched reading of a device: (S complex64[C, K], E float32[C], active int32[C], batch_seq), or None.
        K is the tone count the reading was computed with.  Lossy: at most max_batches_per_run + 2 are kept per device."""
        Cn = len(self.cfg.devices[dev].channels) if 0 <= dev < len(self.cfg.devices) else 0  # (a bad index: the C call reports it)
        tones = np.empty(2 * TONE_MAX * Cn, np.float32)
        energy = np.empty(Cn, np.float32)
        active = np.empty(Cn, np.int32)
        seq, k = C.c_uint64(0), C.c_int32(0)
        if not self._chk(self.L.abg_fetch_tone_meter(self.h, dev, _ptr(tones), _ptr(energy), _ptr(active), C.byref(seq), C.byref(k))):
            return None
        K = int(k.value)
        return tones[:2 * K * Cn].view(np.complex64).reshape(Cn, K).copy(), energy, active, int(seq.value)

    def tone_meter_time(self) -> float:
        """ms of the tone meter kernel in the most recent run (CUDA events on the K2 stream); 0 if it metered nothing."""
        return self._kernel_time(self.L.abg_debug_tone_meter_time)

    # ---- band activity detector -----------------------------------------------------------------------------------
    def activity_configure(self, dev: int, stride: int, hang: int = 0, min_span: int = 1, thr=None) -> None:
        """Every burst above thr[fft_size] (on the band spectrum's scale) in a device's band, per batch, at every
        `stride`-th frame; `hang` and `min_span` in selected frames (definition in airband_b200.h).  stride = 0 switches it
        off.  Applies to batches enqueued by later runs.  `activity_threshold` builds thr from fetched spectra."""
        t = None if thr is None else np.ascontiguousarray(thr, dtype=np.float32)
        self._chk(self.L.abg_activity_configure(self.h, dev, int(stride), int(hang), int(min_span), _ptr(t)))

    def fetch_activity(self, dev: int) -> Optional[dict]:
        """Oldest unfetched reading of a device, or None: a dict of pieces (BURST_DTYPE array sorted by (bin, first_frame)),
        n_total (pieces found; more than len(pieces) means truncated), batch_seq, settings = (stride, hang, min_span) and
        wave_batch (frames per batch, which merge_bursts needs).
        Lossy: at most max_batches_per_run + 2 are kept per device."""
        buf = np.empty(ACTIVITY_MAX_RECORDS, BURST_DTYPE)
        ns, nt, seq = C.c_int32(0), C.c_int32(0), C.c_uint64(0)
        st = np.zeros(3, np.int32)
        if not self._chk(self.L.abg_fetch_activity(self.h, dev, _ptr(buf), buf.size, C.byref(ns), C.byref(nt), C.byref(seq), _ptr(st))):
            return None
        return dict(pieces=buf[:ns.value].copy(), n_total=int(nt.value), batch_seq=int(seq.value),
                    settings=tuple(int(x) for x in st), wave_batch=self.B)

    def activity_time(self) -> float:
        """ms of the activity detector kernel in the most recent run (CUDA events on the K1 stream); 0 if it ran none."""
        return self._kernel_time(self.L.abg_debug_activity_time)

    # ---- I/Q history ----------------------------------------------------------------------------------------------
    def history_configure(self, dev: int, n_batches: int) -> None:
        """Keep a device's most recent n_batches * wave_batch * hop raw samples in HBM (definition in airband_b200.h), from
        the batches of later runs on; 0 switches it off and frees it.  A change of capacity empties it."""
        self._chk(self.L.abg_history_configure(self.h, dev, int(n_batches)))

    def history_range(self, dev: int) -> Tuple[int, int]:
        """(first, end): the absolute samples [first, end) the history holds once every run enqueued so far has finished."""
        first, end = C.c_uint64(0), C.c_uint64(0)
        self._chk(self.L.abg_history_range(self.h, dev, C.byref(first), C.byref(end)))
        return int(first.value), int(end.value)

    def history_raw(self, dev: int, first: int, n: int) -> np.ndarray:
        """Samples [first, first + n) exactly as pushed: the ring dtype (uint8, int8, int16 or float32), I and Q
        interleaved, 2 * n items."""
        dt = {1: np.uint8, 2: np.int8, 3: np.int16, 4: np.float32}[self.cfg.devices[dev].sfmt] if 0 <= dev < len(self.cfg.devices) else np.uint8
        out = np.empty(2 * max(int(n), 0), dt)
        self._chk(self.L.abg_history_raw(self.h, dev, int(first), int(n), _ptr(out)))
        return out

    def history_subband(self, dev: int, offset_hz: float, decim: int, coeffs, first_m: int, n_out: int) -> np.ndarray:
        """y[m] of the sub-band definition for m in [first_m, first_m + n_out), computed from the history: complex64[n_out],
        bitwise what a live output of the same settings computes once all its taps follow its start."""
        h = np.ascontiguousarray(coeffs, dtype=np.float32)
        out = np.empty(2 * max(int(n_out), 0), np.float32)
        self._chk(self.L.abg_history_subband(self.h, dev, float(offset_hz), int(decim), h.size, _ptr(h), int(first_m), int(n_out),
                                             _ptr(out)))
        return out.view(np.complex64)

    def history_time(self) -> Tuple[float, float]:
        """(append ms of the most recent run, kernel ms of the most recent history_subband), from CUDA events on the K1
        stream; 0 where there was none."""
        ms = (C.c_float * 2)()
        self._chk(self.L.abg_debug_history_time(self.h, ms))
        return float(ms[0]), float(ms[1])

    def history_replay(self, jobs, want_iq: bool = True) -> List[dict]:
        """Demodulate stretches of the history as fresh channels listening there would have (definition in
        airband_b200.h), all jobs in one call.  jobs: dicts with dev, first_batch, n_batches and channels (a list of
        config.Channel), e.g. from transmission_replay.  Returns per job a dict with waveout float32[n_batches, C, B],
        iq complex64[n_batches, C, B] (None unless want_iq), axc uint8[n_batches, C] and stats (a CSquelchStats per
        channel after the last batch)."""
        arr = (CReplayJob * max(len(jobs), 1))()
        keep, out = [], []
        for k, j in enumerate(jobs):
            chans = channels_to_c(j["channels"])
            nb, Cn = int(j["n_batches"]), len(j["channels"])
            r = dict(waveout=np.zeros((max(nb, 0), Cn, self.B), np.float32),
                     iq=np.zeros((max(nb, 0), Cn, 2 * self.B), np.float32) if want_iq else None,
                     axc=np.zeros((max(nb, 0), Cn), np.uint8), stats=(CSquelchStats * max(Cn, 1))())
            keep.append(chans)
            arr[k] = CReplayJob(int(j["dev"]), nb, int(j["first_batch"]), Cn, C.cast(chans, C.POINTER(CChannelCfg)),
                                _ptr(r["waveout"]), _ptr(r["iq"]), _ptr(r["axc"]), C.cast(r["stats"], C.POINTER(CSquelchStats)))
            out.append(r)
        self._chk(self.L.abg_history_replay(self.h, len(jobs), arr))
        for r in out:
            r["iq"] = r["iq"].view(np.complex64) if r["iq"] is not None else None
            r["stats"] = list(r["stats"])[:r["waveout"].shape[1]]
        return out

    def replay_time(self) -> Tuple[float, float]:
        """(gather ms, replay engine run ms) of the most recent history_replay, from CUDA events; 0 before the first."""
        ms = (C.c_float * 2)()
        self._chk(self.L.abg_debug_replay_time(self.h, ms))
        return float(ms[0]), float(ms[1])

    # ---- live follow ----------------------------------------------------------------------------------------------
    def follow_open(self, dev: int, first_batch: int, channels, queue_batches: int = 16) -> int:
        """Open a live follow session (definition in airband_b200.h): a history replay of device dev from first_batch on,
        with no end, that follow_run keeps advancing as the history grows.  channels: a list of config.Channel, e.g.
        from transmission_follow (follow_open(**job)).  Returns the session id."""
        chans = channels_to_c(channels)
        sid = C.c_int32(-1)
        self._chk(self.L.abg_follow_open(self.h, int(dev), int(first_batch), len(channels), C.cast(chans, C.POINTER(CChannelCfg)),
                                         int(queue_batches), C.byref(sid)))
        return int(sid.value)

    def follow_close(self, session: int) -> None:
        self._chk(self.L.abg_follow_close(self.h, int(session)))

    def follow_run(self, max_batches: int = -1) -> int:
        """Advance every open session by up to max_batches batches (< 0: as far as the history and queue room allow);
        returns the session-batches enqueued.  Does not wait for the live engine."""
        return self._chk(self.L.abg_follow_run(self.h, int(max_batches)))

    def follow_info(self, session: int) -> dict:
        """dev, n_channels, next_batch (the next batch follow_run enqueues), queued (unfetched batches) and lost."""
        st = CFollowStatus()
        self._chk(self.L.abg_follow_info(self.h, int(session), C.byref(st)))
        return dict(dev=st.dev, n_channels=st.n_channels, next_batch=int(st.next_batch), queued=st.queued, lost=bool(st.lost))

    def follow_fetch(self, session: int, max_batches: Optional[int] = None, want_iq: bool = True) -> dict:
        """Pop up to max_batches (default: every queued one) of a session's oldest batches, waiting for them: a dict with
        first_batch (batch number of the first, None if none was popped), waveout float32[n, C, B], iq complex64[n, C, B]
        (None unless want_iq) and axc uint8[n, C].  Raises AbgError (ABG_ERANGE) once a lost session has nothing left."""
        info = self.follow_info(session)
        n, Cn = info["queued"] if max_batches is None else int(max_batches), info["n_channels"]
        wo = np.zeros((max(n, 0), Cn, self.B), np.float32)
        iq = np.zeros((max(n, 0), Cn, 2 * self.B), np.float32) if want_iq else None
        ax = np.zeros((max(n, 0), Cn), np.uint8)
        first = C.c_uint64(0)
        got = self._chk(self.L.abg_follow_fetch(self.h, int(session), n, _ptr(wo), _ptr(iq), _ptr(ax), C.byref(first)))
        return dict(first_batch=int(first.value) if got else None, waveout=wo[:got],
                    iq=iq[:got].view(np.complex64) if want_iq else None, axc=ax[:got])

    def follow_stats(self, session: int, chan: int) -> CSquelchStats:
        """Squelch statistics of a session's channel after its batch next_batch - 1 (waits for it)."""
        st = CSquelchStats()
        self._chk(self.L.abg_follow_stats(self.h, int(session), int(chan), C.byref(st)))
        return st

    def follow_time(self) -> Tuple[float, float]:
        """(gather ms, follow-engine run ms) of the most recent follow_run, from CUDA events; 0 if it enqueued nothing."""
        ms = (C.c_float * 2)()
        self._chk(self.L.abg_debug_follow_time(self.h, ms))
        return float(ms[0]), float(ms[1])

    # ---- history analysis -----------------------------------------------------------------------------------------
    def history_spectrogram(self, jobs) -> List[np.ndarray]:
        """Band spectra of windows of the history, all jobs in one call (definition in airband_b200.h).  jobs: dicts with
        dev, first_frame, n_rows, stride and frames_per_row (default wave_batch); with frames_per_row = wave_batch and
        first_frame = AGC_EXTRA + b * wave_batch, row r is bitwise the live spectrum of batch b + r.  Returns per job
        float32[n_rows, fft_size].  history_window gives a window the history holds."""
        arr = (CSpectrogramJob * max(len(jobs), 1))()
        out = []
        for k, j in enumerate(jobs):
            p = np.zeros((max(int(j["n_rows"]), 0), self.cfg.fft_size), np.float32)
            arr[k] = CSpectrogramJob(int(j["dev"]), int(j["n_rows"]), int(j["first_frame"]), int(j.get("frames_per_row", self.B)),
                                     int(j["stride"]), _ptr(p))
            out.append(p)
        self._chk(self.L.abg_history_spectrogram(self.h, len(jobs), arr))
        return out

    def history_activity(self, jobs) -> List[dict]:
        """The activity detector over windows of the history, all jobs in one call (definition in airband_b200.h).  jobs:
        dicts with dev, first_batch, n_batches, stride, thr[fft_size], hang (default 0) and min_span (default 1).
        Returns per job a dict of bursts (BURST_DTYPE, sorted by (bin, first_frame): merge_bursts of the live readings,
        with OPEN_START / OPEN_END on the bursts at the window's edges, kept whatever their span) and n_truncated (batches
        whose pieces did not all fit a reading; their bursts are unspecified)."""
        def call(caps):
            arr = (CActivityJob * max(len(jobs), 1))()
            keep = []
            for k, j in enumerate(jobs):
                t = np.ascontiguousarray(j["thr"], dtype=np.float32)
                b = np.zeros(caps[k], BURST_DTYPE)
                keep.append((t, b))
                arr[k] = CActivityJob(int(j["dev"]), int(j["n_batches"]), int(j["first_batch"]), int(j["stride"]), int(j.get("hang", 0)),
                                      int(j.get("min_span", 1)), caps[k], _ptr(t), _ptr(b) if caps[k] else None, 0, 0)
            self._chk(self.L.abg_history_activity(self.h, len(jobs), arr))
            return arr, keep

        caps = [4096] * len(jobs)
        arr, keep = call(caps)
        if any(arr[k].n_bursts > caps[k] for k in range(len(jobs))):  # the results do not depend on the call: repeat with room
            arr, keep = call([max(caps[k], arr[k].n_bursts) for k in range(len(jobs))])
        return [dict(bursts=keep[k][1][:arr[k].n_bursts].copy(), n_truncated=int(arr[k].n_truncated)) for k in range(len(jobs))]

    def history_analysis_time(self) -> Tuple[float, float, float]:
        """(gather ms, spectrum kernel ms, detector kernel ms) of the most recent history_spectrogram or history_activity,
        summed over its chunks, from CUDA events; 0 where it had none."""
        ms = (C.c_float * 3)()
        self._chk(self.L.abg_debug_history_analysis_time(self.h, ms))
        return float(ms[0]), float(ms[1]), float(ms[2])

    # ---- transmission profiles ------------------------------------------------------------------------------------
    def history_profile(self, jobs) -> List[dict]:
        """The profile sums of windows of the history, all jobs in one call (definition in airband_b200.h).  jobs: dicts
        with dev, offset_hz, decim, coeffs, first_m, n_out and tones (None: the 51 standard tones), e.g. from profile_job.
        Returns per job a dict: n, p1, p2, a1, z (complex), f1, f2, tone_fm and tone_am (complex128[K])."""
        arr = (CProfileJob * max(len(jobs), 1))()
        outs = (CProfile * max(len(jobs), 1))()
        keep = []
        for k, j in enumerate(jobs):
            h = np.ascontiguousarray(j["coeffs"], dtype=np.float32)
            t = j.get("tones")
            t = np.ascontiguousarray(t, dtype=np.float32) if t is not None and len(t) else None
            keep.append((h, t))
            arr[k] = CProfileJob(int(j["dev"]), int(j["decim"]), float(j["offset_hz"]), h.size, 0 if t is None else t.size, _ptr(h),
                                 int(j["first_m"]), int(j["n_out"]), _ptr(t), C.pointer(outs[k]))
        self._chk(self.L.abg_history_profile(self.h, len(jobs), arr))
        res = []
        for k in range(len(jobs)):
            o, K = outs[k], outs[k].n_tones
            fm, am = np.ctypeslib.as_array(o.tone_fm)[:K], np.ctypeslib.as_array(o.tone_am)[:K]
            res.append(dict(n=int(o.n), p1=o.p1, p2=o.p2, a1=o.a1, z=complex(o.z[0], o.z[1]), f1=o.f1, f2=o.f2,
                            tone_fm=fm[:, 0] + 1j * fm[:, 1], tone_am=am[:, 0] + 1j * am[:, 1]))
        return res

    def history_profile_time(self) -> Tuple[float, float]:
        """(capture ms, profile kernel ms) of the most recent history_profile, summed over its chunks, from CUDA events;
        0 before the first."""
        ms = (C.c_float * 2)()
        self._chk(self.L.abg_debug_history_profile_time(self.h, ms))
        return float(ms[0]), float(ms[1])

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


def subband_frequency(offset_hz: float, sample_rate: float) -> float:
    """The frequency a sub-band output actually sits at, relative to the centre frequency: delta * sample_rate / 2^32
    with delta = llround(offset_hz / sample_rate * 2^32) mod 2^32, folded into [-sample_rate/2, sample_rate/2)."""
    x = float(offset_hz) / float(sample_rate) * 4294967296.0
    r = int(np.floor(abs(x) + 0.5)) * (1 if x >= 0 else -1)  # llround: halves away from zero
    delta = r % (1 << 32)
    if delta >= 1 << 31:
        delta -= 1 << 32
    return delta * float(sample_rate) / 4294967296.0


def tone_meter_frequency(f: float, wave_rate: float) -> float:
    """The frequency the tone meter measures for a listed tone f: delta * wave_rate / 2^32 with
    delta = llround(f / wave_rate * 2^32) (f in (0, wave_rate / 2))."""
    x = float(np.float32(f)) / float(wave_rate) * 4294967296.0
    return int(np.floor(x + 0.5)) * float(wave_rate) / 4294967296.0


def tone_powers(readings) -> np.ndarray:
    """Power share of each tone over consecutive tone meter readings of one device (Engine.fetch_tone_meter tuples, oldest
    first): with S, E and n = active summed over the readings, 2 |S|^2 / (n E), float64[C, K].  Adding S gives the DFT of
    the whole window, since the meter's phase is that of the absolute audio index.  n counts the samples with audio, so a
    squelch that was closed for part of the window does not dilute the share; a channel without audio reads 0.  A pure
    tone reads about 1.  Raises ValueError on a gap in batch_seq or a change of the tone count."""
    readings = list(readings)
    if not readings:
        raise ValueError("tone_powers: no readings")
    S = np.zeros(readings[0][0].shape, np.complex128)
    E = np.zeros(readings[0][1].shape, np.float64)
    n = np.zeros(readings[0][2].shape, np.float64)
    for i, (s, e, a, seq) in enumerate(readings):
        if s.shape != S.shape:
            raise ValueError(f"tone_powers: reading {i} has {s.shape[-1]} tones, the first has {S.shape[-1]}")
        if i and seq != readings[i - 1][3] + 1:
            raise ValueError(f"tone_powers: gap in batch_seq: {readings[i - 1][3]} then {seq}")
        S += s
        E += e
        n += a
    den = n * E
    with np.errstate(divide="ignore", invalid="ignore"):
        share = np.where(den[:, None] > 0, 2.0 * np.abs(S) ** 2 / den[:, None], 0.0)
    return share


def ctcss_identify(readings, min_share: float = 0.005, tones: Optional[Sequence[float]] = None):
    """The CTCSS tone of each channel from consecutive tone meter readings (see tone_powers; 4 batches, 0.5 s, tell every
    standard tone apart): per channel (tone_hz, share) of the strongest tone, or None when its share is below min_share.
    tones: the list the readings were computed with (default STANDARD_TONES)."""
    share = tone_powers(readings)
    tones = STANDARD_TONES if tones is None else tuple(tones)
    if len(tones) != share.shape[1]:
        raise ValueError(f"ctcss_identify: {len(tones)} tones given, the readings have {share.shape[1]}")
    out = []
    for row in share:
        k = int(np.argmax(row))
        out.append((float(tones[k]), float(row[k])) if row[k] >= min_share else None)
    return out


def subband_lowpass(n_coeffs: int, cutoff_hz: float, sample_rate: float, atten_db: float = 60.0) -> np.ndarray:
    """Kaiser-windowed sinc low-pass for a sub-band output: float32[n_coeffs], the ideal sinc's edge at cutoff_hz, unit
    gain at DC.  Kaiser's beta for a stopband atten_db below the passband; the stopband starts about
    (atten_db - 7.95) / (14.36 * (n_coeffs - 1)) * sample_rate above the cutoff."""
    if n_coeffs < 1 or n_coeffs > SUBBAND_MAX_COEFFS:
        raise ValueError(f"n_coeffs must be in [1, {SUBBAND_MAX_COEFFS}]")
    if not 0 < cutoff_hz <= sample_rate / 2:
        raise ValueError("cutoff_hz must be in (0, sample_rate/2]")
    a = float(atten_db)
    beta = 0.1102 * (a - 8.7) if a > 50 else (0.5842 * (a - 21) ** 0.4 + 0.07886 * (a - 21) if a >= 21 else 0.0)
    t = np.arange(n_coeffs, dtype=np.float64) - (n_coeffs - 1) / 2.0
    fc = 2.0 * cutoff_hz / sample_rate
    h = fc * np.sinc(fc * t) * np.kaiser(n_coeffs, beta)
    return (h / h.sum()).astype(np.float32)


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


def activity_threshold(power, margin_db: float, half_width: int) -> np.ndarray:
    """Per-bin thresholds for Engine.activity_configure from band spectra (Engine.fetch_spectrum powers, one [fft_size] or
    several [n, fft_size], averaged): the running median of the power over +-half_width bins, times 10^(margin_db / 10),
    float32.  The median runs in frequency order and its window is cut at the band edges rather than wrapped, so it follows
    the passband roll-off of the SDR's filter there; the carriers it is meant to catch sit margin_db above their
    neighbourhood's median, as long as a carrier is narrower than half the window.  Bins whose median is zero get the
    smallest positive float32 times the margin, so every threshold is > 0."""
    p = np.asarray(power, np.float64)
    if p.ndim == 2:
        p = p.mean(axis=0)
    if p.ndim != 1 or half_width < 0:
        raise ValueError("activity_threshold: power must be [fft_size] or [n, fft_size], half_width >= 0")
    n = p.size
    f = np.fft.fftshift(p)  # frequency order: the band edges at both ends
    w = 2 * half_width + 1
    padded = np.concatenate([np.full(half_width, np.nan), f, np.full(half_width, np.nan)])
    med = np.nanmedian(np.lib.stride_tricks.sliding_window_view(padded, w), axis=1)
    med = np.maximum(np.fft.ifftshift(med), float(np.finfo(np.float32).tiny))
    thr = (med * 10.0 ** (margin_db / 10.0)).astype(np.float32)
    assert thr.size == n
    return np.maximum(thr, np.finfo(np.float32).tiny)


def merge_bursts(readings) -> np.ndarray:
    """Stitch the pieces of consecutive activity readings of one device (Engine.fetch_activity dicts, oldest first) into
    bursts (definition in airband_b200.h): a piece with OPEN_END joins the same bin's OPEN_START piece of the next reading
    when their gap is <= hang + 1 selected frames, then bursts shorter than min_span are dropped.  Pieces still open at the
    last reading end there.  Returns a BURST_DTYPE array sorted by (bin, first_frame), flags 0; a joined burst's sum is the
    float32 sum of its pieces' sums.  Raises ValueError on a gap in batch_seq, a change of settings or a truncated
    reading."""
    readings = list(readings)
    out = []
    if not readings:
        return np.zeros(0, BURST_DTYPE)
    s, h, m = readings[0]["settings"]
    B = readings[0]["wave_batch"]
    n_sel = -(-B // s)

    def q_of(frame, seq):  # absolute selected index q = seq * n + i of frame f = AGC_EXTRA + seq * B + i * s
        return seq * n_sel + (int(frame) - AGC_EXTRA - seq * B) // s

    open_ = {}  # bin -> [record, q_first, q_last] of the burst that may still grow
    for idx, r in enumerate(readings):
        if tuple(r["settings"]) != (s, h, m):
            raise ValueError(f"merge_bursts: reading {idx} has settings {tuple(r['settings'])}, the first {(s, h, m)}")
        if idx and r["batch_seq"] != readings[idx - 1]["batch_seq"] + 1:
            raise ValueError(f"merge_bursts: gap in batch_seq: {readings[idx - 1]['batch_seq']} then {r['batch_seq']}")
        if r["n_total"] > len(r["pieces"]):
            raise ValueError(f"merge_bursts: reading {idx} (batch_seq {r['batch_seq']}) is truncated: {len(r['pieces'])} of {r['n_total']} pieces")
        seq = r["batch_seq"]
        nxt = {}
        for p in np.sort(r["pieces"], order=["bin", "first_frame"]):
            k = int(p["bin"])
            qf, ql = q_of(p["first_frame"], seq), q_of(p["last_frame"], seq)
            cur = None
            if p["flags"] & BURST_OPEN_START and k in open_ and qf - open_[k][2] <= h + 1:
                cur = open_.pop(k)
                rec = cur[0]
                rec["last_frame"] = p["last_frame"]
                rec["n_active"] += p["n_active"]
                rec["peak"] = max(rec["peak"], p["peak"])
                rec["sum"] = np.float32(np.float32(rec["sum"]) + np.float32(p["sum"]))
                cur[2] = ql
            else:
                rec = p.copy()
                rec["flags"] = 0
                cur = [rec, qf, ql]
            if p["flags"] & BURST_OPEN_END:
                nxt[k] = cur
            elif cur[2] - cur[1] + 1 >= m:
                out.append(cur[0])
        for cur in open_.values():  # not continued in this reading
            if cur[2] - cur[1] + 1 >= m:
                out.append(cur[0])
        open_ = nxt
    for cur in open_.values():
        if cur[2] - cur[1] + 1 >= m:
            out.append(cur[0])
    res = np.array(out, BURST_DTYPE) if out else np.zeros(0, BURST_DTYPE)
    return np.sort(res, order=["bin", "first_frame"])


def group_transmissions(bursts, cfg: Config, dev: int, max_bin_gap: int = 1, centerfreq: Optional[float] = None) -> List[dict]:
    """Group the bursts of one device (merge_bursts output) into transmissions: bursts whose bins are at most max_bin_gap
    apart in frequency and whose frame spans overlap join, transitively, so a carrier's main lobe and its sidebands become
    one transmission.  Bins are taken in frequency order, bin k at offset k (k < fft_size / 2) or k - fft_size bins from
    the centre, the inverse of config.calc_bin's wrap; one bin is sample_rate // fft_size Hz as in calc_bin.  Per
    transmission, oldest first: freq_hz = centerfreq + the bursts' power-weighted (by sum) mean offset in bins times the bin
    width; bins = (lowest, highest) signed offset; first_frame, last_frame; start_s / end_s = those frames' first samples
    (frame * hop / sample_rate, the device's stream time); peak; energy = the sum of the bursts' sums; n_bursts; and
    monitored = a configured channel's bin lies in [lowest, highest].  centerfreq defaults to the Device's."""
    b = np.asarray(bursts, BURST_DTYPE)
    d = cfg.devices[dev]
    centerfreq = d.centerfreq if centerfreq is None else centerfreq
    N = cfg.fft_size
    bin_hz = d.sample_rate // N
    hop = cfg.hop(dev)
    sb = np.where(b["bin"] < N // 2, b["bin"], b["bin"] - N).astype(np.int64)
    parent = list(range(b.size))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    order = np.argsort(sb, kind="stable")
    for ii, x in enumerate(order):  # neighbours in frequency: only bursts up to max_bin_gap bins higher
        for y in order[ii + 1:]:
            if sb[y] - sb[x] > max_bin_gap:
                break
            if b["first_frame"][x] <= b["last_frame"][y] and b["first_frame"][y] <= b["last_frame"][x]:
                parent[find(x)] = find(y)
    groups = {}
    for x in range(b.size):
        groups.setdefault(find(x), []).append(x)
    chan_bins = [c.bin if c.bin < N // 2 else c.bin - N for c in d.channels]
    out = []
    for members in groups.values():
        m = np.asarray(members)
        w = b["sum"][m].astype(np.float64)
        lo, hi = int(sb[m].min()), int(sb[m].max())
        first, last = int(b["first_frame"][m].min()), int(b["last_frame"][m].max())
        out.append(dict(freq_hz=float(centerfreq) + float(np.sum(w * sb[m]) / np.sum(w)) * bin_hz, bins=(lo, hi),
                        first_frame=first, last_frame=last, start_s=first * hop / d.sample_rate, end_s=last * hop / d.sample_rate,
                        peak=float(b["peak"][m].max()), energy=float(w.sum()), n_bursts=int(m.size),
                        monitored=any(lo <= c <= hi for c in chan_bins)))
    out.sort(key=lambda t: (t["first_frame"], t["freq_hz"]))
    return out


def transmission_capture(tx: dict, cfg: Config, dev: int, history_range: Tuple[int, int], decim: int, n_coeffs: int,
                         pad_s: float = 0.0) -> Tuple[float, int, int]:
    """The Engine.history_subband window of one transmission (a group_transmissions dict of device dev): returns
    (offset_hz, first_m, n_out).  offset_hz is tx["freq_hz"] from the device's centre frequency.  The window covers the
    transmission's samples [first_frame * hop, last_frame * hop + fft_size), widened by pad_s seconds on each side, as the
    outputs m with m * decim inside it, clipped so that every tap lies in history_range = (first, end):
    m * decim - (n_coeffs - 1) >= first and m * decim < end.  Raises ValueError if no output is left."""
    d = cfg.devices[dev]
    hop, D, L = cfg.hop(dev), int(decim), int(n_coeffs)
    if D < 1 or L < 1:
        raise ValueError("transmission_capture: decim and n_coeffs must be >= 1")
    pad = int(round(pad_s * d.sample_rate))
    lo = max(int(tx["first_frame"]) * hop - pad, 0)
    hi = int(tx["last_frame"]) * hop + cfg.fft_size + pad  # exclusive
    first, end = history_range
    m_lo = max(-(-lo // D), -(-(first + L - 1) // D))
    m_hi = min(-(-hi // D), -(-end // D))  # exclusive: m * D < hi and m * D < end
    if m_hi <= m_lo:
        raise ValueError(f"transmission_capture: nothing of the transmission (samples [{lo}, {hi})) is left in the history "
                         f"[{first}, {end}) with {L} taps at decimation {D}")
    return float(tx["freq_hz"]) - float(d.centerfreq), m_lo, m_hi - m_lo


# A fresh AM channel's auto squelch starts from a noise floor of 5.0.  On the test signals' noise (U8 at 2.048 Msps, fft
# 2048, complex noise of 0.01 full scale per component) the CPU oracle's noise level is within 10 % of its steady value
# from the 6th batch on (tests/test_history_replay_cpu.py measures it): 6 batches of lead-in.
REPLAY_SETTLE_BATCHES = 6


def _lead_in_batch(tx: dict, cfg: Config, dev: int, history_range: Tuple[int, int], lead_s: Optional[float], fn: str):
    """(first batch, lead_s) of a replay or follow session for one transmission: the latest batch whose first frame lies
    at least lead_s seconds of frames (default REPLAY_SETTLE_BATCHES batches) before the transmission's first frame, or
    the first batch whose samples the history holds if that is later."""
    B, hop = cfg.wave_batch, cfg.hop(dev)
    if lead_s is None:
        lead_s = REPLAY_SETTLE_BATCHES * B / cfg.wave_rate
    if lead_s < 0:
        raise ValueError(f"{fn}: lead_s must be >= 0")
    lead = int(np.ceil(lead_s * cfg.devices[dev].sample_rate / hop))  # frames
    b_lead = (int(tx["first_frame"]) - AGC_EXTRA - lead) // B
    b_first = -(-int(history_range[0]) // (B * hop))
    return max(b_lead, b_first, 0), lead_s


def transmission_replay(tx: dict, cfg: Config, dev: int, history_range: Tuple[int, int], lead_s: Optional[float] = None,
                        **channel_kw) -> dict:
    """An Engine.history_replay job that listens to one transmission (a group_transmissions dict of device dev): a channel
    from config.make_channel at tx["freq_hz"] (its bin, and dm_dphi for NFM; channel_kw goes to make_channel, e.g.
    modulation, bandwidth, ctcss_hz).  first_batch is the latest batch whose first frame lies at least lead_s seconds of
    frames before the transmission's first frame, or the first batch whose samples the history holds if that is later;
    n_batches runs to the batch of its last frame, or as far as the history reaches: every sample read,
    [first_batch * B * hop, (AGC_EXTRA + (first_batch + n_batches) * B) * hop + fft_size - hop), lies in history_range.
    lead_s defaults to REPLAY_SETTLE_BATCHES batches (0.75 s at wave_rate 8000): the time a fresh channel's squelch takes
    to find the noise floor, so that the transmission opens it as a configured channel's would.  Raises ValueError if
    nothing of the transmission fits."""
    d = cfg.devices[dev]
    B, hop, N = cfg.wave_batch, cfg.hop(dev), cfg.fft_size
    b0, lead_s = _lead_in_batch(tx, cfg, dev, history_range, lead_s, "transmission_replay")
    first, end = history_range
    b_last = (int(tx["last_frame"]) - AGC_EXTRA) // B
    b_end = ((int(end) - N + hop) // hop - AGC_EXTRA) // B  # batches b < b_end have every sample in the history
    n = min(b_last + 1, b_end) - b0
    if end <= first or n < 1:
        raise ValueError(f"transmission_replay: nothing of the transmission (frames [{tx['first_frame']}, {tx['last_frame']}]) fits "
                         f"the history [{first}, {end}) with {lead_s} s of lead-in")
    ch = make_channel(int(round(tx["freq_hz"])), d.centerfreq, d.sample_rate, N, cfg.wave_rate, **channel_kw)
    return dict(dev=dev, first_batch=b0, n_batches=n, channels=[ch])


def transmission_follow(tx: dict, cfg: Config, dev: int, history_range: Tuple[int, int], lead_s: Optional[float] = None,
                        **channel_kw) -> dict:
    """An Engine.follow_open session that listens to one transmission (a group_transmissions dict of device dev) from its
    lead-in on and keeps listening as the history grows: dev, first_batch and channels as transmission_replay gives
    them (same channel, same start rule), with no end.  first_batch may lie past the history's end when the
    transmission was reported ahead of it; the session then waits for its samples."""
    d = cfg.devices[dev]
    b0, _ = _lead_in_batch(tx, cfg, dev, history_range, lead_s, "transmission_follow")
    ch = make_channel(int(round(tx["freq_hz"])), d.centerfreq, d.sample_rate, cfg.fft_size, cfg.wave_rate, **channel_kw)
    return dict(dev=dev, first_batch=b0, channels=[ch])


def history_window(cfg: Config, dev: int, history_range: Tuple[int, int], stride: int = 1, frames_per_row: Optional[int] = None,
                   seconds: Optional[float] = None) -> Tuple[int, int]:
    """The longest window of device dev that the history (history_range = (first, end), Engine.history_range) fully holds
    for history analysis at this stride, with the engine's rule: every sample of every selected frame lies in [first, end).
    frames_per_row None: the detector's window, whole batches, returned as (first_batch, n_batches).  frames_per_row F: a
    spectrogram's window of F-frame rows on the grid of rows that start at frame AGC_EXTRA + k * F (with F = wave_batch, the
    batches), returned as (first_frame, n_rows).  seconds: only the newest units that cover at least that long.  Raises
    ValueError if not one unit fits."""
    B, hop, N = cfg.wave_batch, cfg.hop(dev), cfg.fft_size
    step = B if frames_per_row is None else int(frames_per_row)
    if stride < 1 or step < 1 or stride > step:
        raise ValueError(f"history_window: stride {stride} must be in [1, {step}]")
    n_sel = -(-step // stride)
    first, end = (int(x) for x in history_range)
    # unit k reads the samples [(AGC_EXTRA + k*step) * hop, (AGC_EXTRA + k*step + (n_sel - 1) * stride) * hop + N)
    k_lo = max(0, -(-(-(-first // hop) - AGC_EXTRA) // step))
    k_hi = ((end - N) // hop - (n_sel - 1) * stride - AGC_EXTRA) // step  # inclusive
    n = k_hi - k_lo + 1
    if seconds is not None:
        n = min(n, max(1, int(np.ceil(seconds * cfg.devices[dev].sample_rate / (step * hop)))))
        k_lo = k_hi - n + 1
    if end <= first or n < 1:
        raise ValueError(f"history_window: no {'batch' if frames_per_row is None else 'row'} of {step} frames at stride {stride} "
                         f"fits the history [{first}, {end})")
    return (k_lo, n) if frames_per_row is None else (AGC_EXTRA + k_lo * step, n)


def history_transmissions(e: Engine, cfg: Config, dev: int, margin_db: float, half_width: int, stride: int, hang: int = 0,
                          min_span: int = 1, seconds: Optional[float] = None, max_bin_gap: int = 1) -> List[dict]:
    """What transmitted on device dev during the window its history holds (the newest `seconds` of it, if given), with
    nothing configured in advance but the history: a spectrogram of the window's batches at `stride` (Engine.
    history_spectrogram, F = wave_batch), thresholds from it (activity_threshold(margin_db, half_width)), the detector
    over the same batches (Engine.history_activity with stride, hang and min_span), and the bursts grouped
    (group_transmissions).  Returns group_transmissions' list, which transmission_replay and transmission_follow take."""
    b0, nb = history_window(cfg, dev, e.history_range(dev), stride=stride, seconds=seconds)
    B = cfg.wave_batch
    spec = e.history_spectrogram([dict(dev=dev, first_frame=AGC_EXTRA + b0 * B, n_rows=nb, frames_per_row=B, stride=stride)])[0]
    thr = activity_threshold(spec, margin_db, half_width)
    act = e.history_activity([dict(dev=dev, first_batch=b0, n_batches=nb, stride=stride, hang=hang, min_span=min_span, thr=thr)])[0]
    return group_transmissions(act["bursts"], cfg, dev, max_bin_gap=max_bin_gap)


# ---- transmission profiles ----------------------------------------------------------------------------------------------
def profile_plan(first_m, n_out, n_coeffs, n_tones):
    """Host-only: the chunk and block plan abg_history_profile launches for jobs of these shapes (abg_debug_profile_plan).
    Returns (limits dict, pieces int64[P, 6], blocks int64[Q, 8]); the columns are named in airband_b200.h."""
    L = load()
    fm = np.ascontiguousarray(first_m, np.uint64)
    n = np.ascontiguousarray(n_out, np.int64)
    lc = np.ascontiguousarray(n_coeffs, np.int32)
    k = np.ascontiguousarray(n_tones, np.int32)
    lim = np.zeros(4, np.int64)
    npc, nbk = C.c_int32(0), C.c_int32(0)
    args = lambda p, cp, b, cb: (fm.size, _ptr(fm), _ptr(n), _ptr(lc), _ptr(k), _ptr(lim), _ptr(p), cp, C.byref(npc), _ptr(b), cb, C.byref(nbk))  # noqa: E731
    rc = L.abg_debug_profile_plan(*args(None, 0, None, 0))
    if rc < 0:
        raise AbgError(rc, (L.abg_last_error() or b"").decode())
    pieces, blocks = np.zeros((npc.value, 6), np.int64), np.zeros((nbk.value, 8), np.int64)
    L.abg_debug_profile_plan(*args(pieces, pieces.shape[0], blocks, blocks.shape[0]))
    return dict(scratch=int(lim[0]), blocks=int(lim[1]), result=int(lim[2]), coeffs=int(lim[3])), pieces, blocks


# The default down-converter of a profile job.  Its passband has to hold an NFM signal of 5 kHz deviation with 3 kHz audio
# (Carson: 8 kHz each side) wherever the transmission's frequency puts it: group_transmissions' frequency is good to about
# one bin, sample_rate // fft_size.  So the cutoff is 8 kHz + one bin, and the Kaiser filter's 60 dB stopband starts at
# twice the cutoff: L = ceil((60 - 7.95) / (14.36 cutoff) * sample_rate) + 1, odd.  The decimation makes the output noise
# white: D is the integer in [0.8, 1.2] * sample_rate / (2 cutoff) where the filter's autocorrelation at lag D (the output
# noise's lag-1 correlation rho) is smallest.  That keeps the noise's own real lag-1 term rho sigma^2 out of z, which
# otherwise pulls arg(z) towards the down-converter's frequency (12 Hz at a 2 kHz offset and 20 dB with rho = 0.6), and
# needs no estimate of sigma^2, which a deep AM envelope spoils.  It lands at fs_out ~ 1.77 cutoff; the largest
# instantaneous frequency, one bin + 5 kHz, stays below fs_out / 2.  At 2.048 and 2.56 Msps and fft 512 to 8192 that is
# cutoff 8.25 - 13 kHz, fs_out 14.6 - 23 kHz, L 621 - 1119 and |rho| < 0.004.
PROFILE_SWING_HZ = 8000.0


def profile_filter(cfg: Config, dev: int) -> Tuple[int, float, int]:
    """(decim, cutoff_hz, n_coeffs) of the default profile down-converter of device dev (the rule above)."""
    return _profile_filter(int(cfg.devices[dev].sample_rate), int(cfg.fft_size))[:3]


@functools.lru_cache(maxsize=64)
def _profile_filter(sr: int, fft_size: int):
    """(D, cutoff, L, h) of the rule above; the search over D costs about a millisecond, so it is done once per shape."""
    cutoff = PROFILE_SWING_HZ + sr // fft_size
    L = min((int(np.ceil((60.0 - 7.95) / (14.36 * cutoff) * sr)) + 1) | 1, SUBBAND_MAX_COEFFS - 1)
    h = subband_lowpass(L, cutoff, sr).astype(np.float64)
    e = float(np.dot(h, h))
    d0 = sr / (2.0 * cutoff)
    cand = range(max(1, int(0.8 * d0)), max(1, int(1.2 * d0)) + 1)
    D = min(cand, key=lambda D: abs(float(np.dot(h[D:], h[:-D])) / e) if D < L else 0.0)
    return int(D), float(cutoff), L, h.astype(np.float32)


def profile_job(tx: dict, cfg: Config, dev: int, history_range: Tuple[int, int], decim: Optional[int] = None,
                cutoff_hz: Optional[float] = None, n_coeffs: Optional[int] = None, tones: Optional[Sequence[float]] = None) -> dict:
    """An Engine.history_profile job for one transmission (a group_transmissions dict of device dev): the down-converter
    at tx["freq_hz"] (defaults from profile_filter, coefficients from subband_lowpass) over the transmission's samples
    [first_frame * hop, last_frame * hop + fft_size), as the outputs m with m * decim inside them, clipped so that every
    tap lies in history_range (transmission_capture's window).  tones None: the 51 standard tones.  Raises ValueError
    if fewer than 2 outputs are left."""
    D0, c0, L0 = profile_filter(cfg, dev)
    D = D0 if decim is None else int(decim)
    cutoff = c0 if cutoff_hz is None else float(cutoff_hz)
    L = L0 if n_coeffs is None else int(n_coeffs)
    off, m0, n = transmission_capture(tx, cfg, dev, history_range, D, L)
    if n < 2:
        raise ValueError(f"profile_job: {n} output of the transmission fits the history (at least 2)")
    if (D, cutoff, L) == (D0, c0, L0):
        h = _profile_filter(int(cfg.devices[dev].sample_rate), int(cfg.fft_size))[3].copy()
    else:
        h = subband_lowpass(L, min(cutoff, cfg.devices[dev].sample_rate / 2), cfg.devices[dev].sample_rate)
    return dict(dev=dev, offset_hz=off, decim=D, coeffs=h, first_m=m0, n_out=n, tones=list(tones) if tones is not None and len(tones) else None)


# The decision rule (DESIGN §4, "Transmission profiles", gives its calibration).  With the output noise's lag-1
# correlation rho (the filter's autocorrelation at lag D over its energy), u = var(a) / mean(a)^2 and w = var(phi):
# circular noise adds sigma^2 / 2C to u and (1 - rho) sigma^2 / C to w, so an AM envelope shows as d = u - w / (2 (1 - rho))
# > 0 and FM as d < 0, the noise cancelling.  Below about 15 dB the phase noise is no longer Gaussian (clicks) and d loses
# its sign, so the rule decides only when the SNR estimate, the larger of the two hypotheses' own estimates (from the
# envelope's kurtosis for a constant envelope, from w for a constant phase), is at least PROFILE_MIN_SNR_DB.
PROFILE_MIN_SNR_DB = 15.0
PROFILE_AM_MIN_D = -0.006       # d above it: AM (a bare carrier reads d ~ 0)
PROFILE_AM_SURE_D = 0.04        # d above it: AM at any SNR (nothing else reads above -0.006 at 10 dB)
PROFILE_NOISE_KAPPA = 0.9       # envelope spread of noise alone: 1
PROFILE_CTCSS_MIN_SHARE = 0.005  # ctcss_identify's share rule
PROFILE_CTCSS_MIN_S = 0.4        # the reference's CTCSS window


def _tone_basis(m0: int, count: int, tones, fs_out: float) -> np.ndarray:
    """sum_{m0 <= m < m0 + count} exp(-2 pi i (delta_k m mod 2^32) / 2^32) per tone, in double (a geometric series)."""
    d = np.array([int(np.floor(float(np.float32(f)) / fs_out * 4294967296.0 + 0.5)) % (1 << 32) for f in tones], np.float64)
    w = -2.0 * np.pi * d / 4294967296.0
    out = np.empty(len(d), np.complex128)
    for k, wk in enumerate(w):
        r = np.exp(1j * wk)
        out[k] = count if abs(1 - r) < 1e-15 else np.exp(1j * ((int(d[k]) * (m0 % (1 << 32))) % (1 << 32)) * -2.0 * np.pi / 4294967296.0) * (1 - r ** count) / (1 - r)
    return out


def profile_summary(reading: dict, job: dict, cfg: Config, dev: int) -> dict:
    """What a profile reading (Engine.history_profile) says of its transmission: freq_hz (absolute: centre +
    subband_frequency(offset) + the measured offset, from arg(z) for AM and from f1 / (n - 1) for NFM), modulation
    (config.MOD_AM, MOD_NFM or None when undecided; a bare carrier counts as AM), am_depth, fm_deviation_hz (peak, for a
    sinusoidal modulation), snr_db, ctcss_hz and ctcss_share (the strongest tone of the decided modulation's tone sums by
    tone_powers' share, after removing the mean's own leakage; None below PROFILE_CTCSS_MIN_SHARE or for windows under
    PROFILE_CTCSS_MIN_S), and channel_kw = dict(modulation=..., ctcss_hz=...) for transmission_replay (ctcss_hz 0.0 for
    no tone, as make_channel takes it; an undecided profile's modulation is None, which make_channel refuses)."""
    from .config import MOD_AM, MOD_NFM
    d = cfg.devices[dev]
    D = int(job["decim"])
    fs_out = d.sample_rate / D
    h = np.asarray(job["coeffs"], np.float64)
    rho = float(np.dot(h[D:], h[:-D]) / np.dot(h, h)) if D < h.size else 0.0
    n = int(reading["n"])
    npair = n - 1
    mean_a = reading["a1"] / n
    u = max(reading["p1"] / n - mean_a ** 2, 0.0) / mean_a ** 2 if mean_a > 0 else 1.0
    mean_phi = reading["f1"] / npair
    w = max(reading["f2"] / npair - mean_phi ** 2, 0.0)
    kappa = n * reading["p2"] / reading["p1"] ** 2 - 1.0 if reading["p1"] > 0 else 1.0
    s_fm = ((1 - kappa) + np.sqrt(1 - kappa)) / kappa if 0 < kappa < 1 else (np.inf if kappa <= 0 else 0.0)
    s_am = (1 - rho) / w if w > 0 else np.inf
    snr = max(s_fm, s_am)
    snr_db = float(10 * np.log10(snr)) if snr > 0 else -np.inf
    dstat = u - w / (2 * (1 - rho))
    mod = None
    if snr_db >= PROFILE_MIN_SNR_DB:
        mod = MOD_AM if dstat > PROFILE_AM_MIN_D else MOD_NFM
    elif dstat > PROFILE_AM_SURE_D and kappa < PROFILE_NOISE_KAPPA:  # deep AM: its troughs spoil both SNR estimates
        mod = MOD_AM
    if mod == MOD_NFM:
        off = mean_phi * fs_out / (2 * np.pi)
    else:  # the noise's own lag-1 correlation, rho sigma^2 per pair, is real and pulls arg(z) towards 0; profile_filter's
        # D makes rho ~ 0, and for other filters sigma^2 = P / (1 + s) removes it to first order
        sigma2 = reading["p1"] / n / (1.0 + s_am) if np.isfinite(s_am) and snr_db >= PROFILE_MIN_SNR_DB else 0.0
        off = float(np.angle(reading["z"] - rho * sigma2 * npair)) * fs_out / (2 * np.pi)
    freq = float(d.centerfreq) + subband_frequency(job["offset_hz"], d.sample_rate) + off
    tones = job.get("tones")
    tones = tuple(tones) if tones is not None and len(tones) else STANDARD_TONES  # [] or None: the standard tones, as the call takes them
    ctcss = share = None
    if mod is not None and n / fs_out >= PROFILE_CTCSS_MIN_S:
        if mod == MOD_NFM:
            S = reading["tone_fm"] - mean_phi * _tone_basis(job["first_m"], npair, tones, fs_out)
            cnt, E = npair, npair * w
        else:
            S = reading["tone_am"] - mean_a * _tone_basis(job["first_m"], n, tones, fs_out)
            cnt, E = n, n * u * mean_a ** 2
        sh = 2.0 * np.abs(S) ** 2 / (cnt * E) if E > 0 else np.zeros(len(tones))
        k = int(np.argmax(sh))
        if sh[k] >= PROFILE_CTCSS_MIN_SHARE:
            ctcss, share = float(tones[k]), float(sh[k])
    return dict(freq_hz=freq, modulation=mod, snr_db=snr_db,
                am_depth=float(np.sqrt(2 * max(dstat, 0.0))) if mod == MOD_AM else None,
                fm_deviation_hz=float(np.sqrt(2 * max(w - 2 * (1 - rho) * u, 0.0)) * fs_out / (2 * np.pi)) if mod == MOD_NFM else None,
                ctcss_hz=ctcss, ctcss_share=share, channel_kw=dict(modulation=mod, ctcss_hz=ctcss or 0.0))


def history_profiles(e: Engine, cfg: Config, dev: int, txs, **job_kw) -> List[dict]:
    """profile_summary of every transmission of device dev (group_transmissions dicts, e.g. from history_transmissions),
    measured in one Engine.history_profile call; job_kw goes to profile_job.  Each summary also holds its job.  The
    result plugs into transmission_replay: transmission_replay(dict(tx, freq_hz=s["freq_hz"]), cfg, dev, hist,
    **s["channel_kw"])."""
    hist = e.history_range(dev)
    jobs = [profile_job(tx, cfg, dev, hist, **job_kw) for tx in txs]
    if not jobs:
        return []
    readings = e.history_profile(jobs)
    return [dict(profile_summary(r, j, cfg, dev), job=j) for r, j in zip(readings, jobs)]
