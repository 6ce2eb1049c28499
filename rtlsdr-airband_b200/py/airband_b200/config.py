"""Configuration records for the GPU demodulation path and their C layout.

The C structs are declared in include/airband_b200.h (abg_channel_cfg / abg_device_cfg / abg_config); they
carry exactly what the reference's demodulate() reads from device_t / channel_t / freq_t / input_t
(reference src/rtl_airband.h:223-286, src/input-common.h:39-57) after config.cpp has resolved the config file.

The helper formulas below restate the reference's config-time arithmetic so that tests and benchmarks can
build configurations from frequencies the way a .conf file would:
  calc_bin       reference src/config.cpp:666-667 (note the integer division sample_rate / fft_size)
  calc_dm_dphi   reference src/config.cpp:679-712
  dbfs_to_level  reference src/util.cpp:169-176
  default_alpha  reference src/rtl_airband.cpp:87
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, field
from typing import List

import numpy as np

SFMT_U8, SFMT_S8, SFMT_S16, SFMT_F32 = 1, 2, 3, 4  # sample_format_t, reference src/input-common.h:31
MOD_AM, MOD_NFM = 0, 1  # enum modulations, reference src/rtl_airband.h:193-199
FM_FAST_ATAN2, FM_QUADRI_DEMOD = 0, 1  # reference src/rtl_airband.cpp:88
AGC_EXTRA = 100  # reference src/rtl_airband.h:74

BYTES_PER_SAMPLE = {SFMT_U8: 1, SFMT_S8: 1, SFMT_S16: 2, SFMT_F32: 4}
NP_DTYPE = {SFMT_U8: np.uint8, SFMT_S8: np.int8, SFMT_S16: np.int16, SFMT_F32: np.float32}
# input_t.fullscale defaults: file/rtlsdr U8 (reference src/input-file.cpp:172), soapysdr S16/F32 (input-soapysdr.cpp:56-64)
DEFAULT_FULLSCALE = {SFMT_U8: 126.5, SFMT_S8: 127.5, SFMT_S16: 32766.5, SFMT_F32: 1.0}


class CChannelCfg(C.Structure):
    _fields_ = [
        ("bin", C.c_int32),
        ("modulation", C.c_int32),
        ("needs_raw_iq", C.c_int32),
        ("has_iq_outputs", C.c_int32),
        ("dm_dphi", C.c_uint32),
        ("alpha", C.c_float),
        ("ampfactor", C.c_float),
        ("squelch_level", C.c_float),
        ("squelch_snr_db", C.c_float),
        ("lowpass_hz", C.c_float),
        ("notch_hz", C.c_float),
        ("notch_q", C.c_float),
        ("ctcss_hz", C.c_float),
        ("afc", C.c_int32),
    ]


class CDeviceCfg(C.Structure):
    _fields_ = [
        ("sfmt", C.c_int32),
        ("fullscale", C.c_float),
        ("sample_rate", C.c_int32),
        ("n_channels", C.c_int32),
        ("channels", C.POINTER(CChannelCfg)),
    ]


class CConfig(C.Structure):
    _fields_ = [
        ("fft_size", C.c_int32),
        ("wave_rate", C.c_int32),
        ("fm_demod", C.c_int32),
        ("n_devices", C.c_int32),
        ("devices", C.POINTER(CDeviceCfg)),
    ]


class CSquelchStats(C.Structure):
    _fields_ = [
        ("noise_level", C.c_float),
        ("signal_level", C.c_float),
        ("squelch_level", C.c_float),
        ("open_count", C.c_uint64),
        ("flappy_count", C.c_uint64),
        ("ctcss_count", C.c_uint64),
        ("no_ctcss_count", C.c_uint64),
        ("agcavgfast", C.c_float),
        ("dm_phi", C.c_uint32),
        ("bin", C.c_int32),
        ("active_counter", C.c_uint64),
        # level_to_dBFS() of the three levels, util.cpp:169-180
        ("noise_level_dbfs", C.c_float),
        ("signal_level_dbfs", C.c_float),
        ("squelch_level_dbfs", C.c_float),
    ]


def calc_bin(freq: int, centerfreq: int, sample_rate: int, fft_size: int) -> int:
    return int(math.ceil((freq + sample_rate - centerfreq) / float(sample_rate // fft_size) - 1.0)) % fft_size


def calc_dm_dphi(freq: int, centerfreq: int, sample_rate: int, wave_rate: int) -> int:
    dm = float(freq - centerfreq)
    decim = sample_rate / wave_rate
    rounded = math.floor(decim + 0.5) if decim >= 0 else -math.floor(-decim + 0.5)  # C round(): half away from zero
    corr = wave_rate / 2.0
    corr *= decim - rounded
    corr *= float(freq - centerfreq) / (sample_rate / 2.0)
    dm -= corr
    dm /= float(wave_rate)
    dm -= math.trunc(dm)
    dm *= 256.0 * 65536.0
    return int(dm) & 0xFFFFFFFF  # (uint32_t)(int)dm_dphi


def dbfs_to_level(dbfs: float, fft_size: int) -> float:
    f32 = np.float32
    offset = f32(f32(7.54) + f32(10.0) * np.log10(f32(fft_size // 2), dtype=f32) - f32(2.38))
    return float(f32(math.pow(10.0, float(f32(f32(dbfs) - offset) / f32(20.0))) * fft_size))


def default_alpha(wave_rate: int) -> float:
    return float(np.float32(math.exp(-1.0 / (wave_rate * 2e-4))))


def hop_samples(sample_rate: int, wave_rate: int) -> int:
    """Complex samples per output audio sample: round(sample_rate / WAVE_RATE), reference src/rtl_airband.cpp:394."""
    x = sample_rate / wave_rate
    return int(math.floor(x + 0.5))


@dataclass
class Channel:
    bin: int
    modulation: int = MOD_AM
    needs_raw_iq: int = 0
    has_iq_outputs: int = 0
    dm_dphi: int = 0
    alpha: float = 0.0
    ampfactor: float = 1.0
    squelch_level: float = 0.0  # > 0: manual level (set_squelch_level_threshold)
    squelch_snr_db: float = -1.0  # >= 0: set_squelch_snr_threshold
    lowpass_hz: float = 0.0  # bandwidth / 2
    notch_hz: float = 0.0
    notch_q: float = 10.0  # reference src/config.cpp:517
    ctcss_hz: float = 0.0
    afc: int = 0
    # informational (not sent to C): tuned frequency offset from centre in Hz, used by the synthetic generator
    offset_hz: float = 0.0
    synth_ctcss_hz: float = -1.0  # generator only: sub-tone actually transmitted (< 0: same as ctcss_hz)


@dataclass
class Device:
    sample_rate: int = 2560000
    sfmt: int = SFMT_U8
    fullscale: float = 0.0  # 0 -> DEFAULT_FULLSCALE[sfmt]
    centerfreq: int = 0
    channels: List[Channel] = field(default_factory=list)

    def __post_init__(self):
        if not self.fullscale:
            self.fullscale = DEFAULT_FULLSCALE[self.sfmt]

    @property
    def bytes_per_sample(self) -> int:
        return BYTES_PER_SAMPLE[self.sfmt]


def channels_to_c(channels):
    """ctypes array of abg_channel_cfg / abo_channel_cfg for a list of Channel (also used for scan-mode frequency lists)."""
    chans = (CChannelCfg * len(channels))()
    for j, c in enumerate(channels):
        cc = chans[j]
        cc.bin, cc.modulation, cc.needs_raw_iq, cc.has_iq_outputs = c.bin, c.modulation, c.needs_raw_iq, c.has_iq_outputs
        cc.dm_dphi, cc.alpha, cc.ampfactor = c.dm_dphi & 0xFFFFFFFF, c.alpha, c.ampfactor
        cc.squelch_level, cc.squelch_snr_db = c.squelch_level, c.squelch_snr_db
        cc.lowpass_hz, cc.notch_hz, cc.notch_q, cc.ctcss_hz, cc.afc = c.lowpass_hz, c.notch_hz, c.notch_q, c.ctcss_hz, c.afc
    return chans


@dataclass
class Config:
    fft_size: int = 512
    wave_rate: int = 8000
    fm_demod: int = FM_FAST_ATAN2
    devices: List[Device] = field(default_factory=list)

    @property
    def wave_batch(self) -> int:
        return self.wave_rate // 8  # WAVE_BATCH, reference src/rtl_airband.h:73

    def hop(self, dev: int) -> int:
        return hop_samples(self.devices[dev].sample_rate, self.wave_rate)

    def to_c(self):
        """Returns (CConfig, keepalive) — keepalive owns the nested arrays."""
        keep = []
        devs = (CDeviceCfg * len(self.devices))()
        for i, d in enumerate(self.devices):
            chans = channels_to_c(d.channels)
            keep.append(chans)
            devs[i].sfmt, devs[i].fullscale, devs[i].sample_rate = d.sfmt, d.fullscale, d.sample_rate
            devs[i].n_channels = len(d.channels)
            devs[i].channels = C.cast(chans, C.POINTER(CChannelCfg))
        keep.append(devs)
        cfg = CConfig(self.fft_size, self.wave_rate, self.fm_demod, len(self.devices), C.cast(devs, C.POINTER(CDeviceCfg)))
        return cfg, keep


def make_channel(freq: int, centerfreq: int, sample_rate: int, fft_size: int, wave_rate: int, *, modulation=MOD_AM,
                 bandwidth: int = 0, rawfile: bool = False, squelch_dbfs: float = 0.0, squelch_snr_db: float = -1.0,
                 ampfactor: float = 1.0, notch_hz: float = 0.0, notch_q: float = 10.0, ctcss_hz: float = 0.0, afc: int = 0,
                 tau_us: int | None = None) -> Channel:
    """Resolve one channels[] entry the way parse_channels() does (reference src/config.cpp:306-726)."""
    needs_raw_iq = 1 if (modulation == MOD_NFM or bandwidth > 0 or rawfile) else 0
    if tau_us is None:
        alpha = default_alpha(wave_rate)
    else:  # reference src/config.cpp:636-638
        alpha = 0.0 if tau_us == 0 else float(np.float32(math.exp(-1.0 / (wave_rate * 1e-6 * tau_us))))
    return Channel(
        bin=calc_bin(freq, centerfreq, sample_rate, fft_size),
        modulation=modulation,
        needs_raw_iq=needs_raw_iq,
        has_iq_outputs=1 if rawfile else 0,
        dm_dphi=calc_dm_dphi(freq, centerfreq, sample_rate, wave_rate) if needs_raw_iq else 0,
        alpha=alpha,
        ampfactor=ampfactor,
        squelch_level=dbfs_to_level(squelch_dbfs, fft_size) if squelch_dbfs < 0 else 0.0,
        squelch_snr_db=squelch_snr_db,
        lowpass_hz=bandwidth / 2.0 if bandwidth > 0 else 0.0,
        notch_hz=notch_hz,
        notch_q=notch_q,
        ctcss_hz=ctcss_hz,
        afc=afc,
        offset_hz=float(freq - centerfreq),
    )
