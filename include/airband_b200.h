/*
 * airband_b200.h — C ABI of the H100 (sm_90a) multichannel demodulation engine.
 *
 * Drop-in boundary for ONE path of RTLSDR-Airband: the body of demodulate()
 * (reference src/rtl_airband.cpp:286-672) — sample conversion + Blackman-Harris window + sliding FFT + per-channel
 * bin extraction + AM / NFM demodulation with squelch, CTCSS, low-pass and notch.  Everything around it
 * (config.cpp, input-*.cpp ring producers, output.cpp / mixer.cpp consumers) stays reference code and talks to this
 * library through plain pointers and sizes.  INTEGRATION.md shows the WITH_B200 branch a maintainer adds next to
 * the existing WITH_BCM_VC branch (reference src/rtl_airband.cpp:293-314,404-412,457-481), whose C API
 * gpu_fft_prepare / gpu_fft_execute / gpu_fft_release (reference src/hello_fft/gpu_fft.h:66-74) is the precedent
 * for this one.
 *
 * Conventions: every function returns 0 on success and a negative ABG_E* code on failure (the VideoCore engine
 * uses -1/-2/-3 the same way, reference src/rtl_airband.cpp:296-310); abg_last_error() gives the text the caller
 * passes to log(LOG_CRIT, ...) before error().  All buffers are caller-owned host memory unless named dev_*.
 * No CPU fallback exists: without a CUDA device abg_create() fails with ABG_ENODEV.
 */
#ifndef AIRBAND_B200_H
#define AIRBAND_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ABG_API __attribute__((visibility("default")))

/* sample_format_t, reference src/input-common.h:31 (same numeric values) */
enum { ABG_SFMT_U8 = 1, ABG_SFMT_S8 = 2, ABG_SFMT_S16 = 3, ABG_SFMT_F32 = 4 };
/* enum modulations, reference src/rtl_airband.h:193-199 */
enum { ABG_MOD_AM = 0, ABG_MOD_NFM = 1 };
/* enum fm_demod_algo, reference src/rtl_airband.cpp:88 (-Q command line switch, :728-730) */
enum { ABG_FM_FAST_ATAN2 = 0, ABG_FM_QUADRI_DEMOD = 1 };
/* enum status (channel_t.axcindicate), reference src/rtl_airband.h:101 */
enum { ABG_NO_SIGNAL = ' ', ABG_SIGNAL = '*', ABG_AFC_UP = '<', ABG_AFC_DOWN = '>' };

enum {
    ABG_OK = 0,
    ABG_ENODEV = -1,   /* no CUDA device / driver (cf. "Unable to enable V3D", rtl_airband.cpp:299) */
    ABG_EINVAL = -2,   /* unsupported configuration (cf. "log2_N=%d not supported", rtl_airband.cpp:303) */
    ABG_ENOMEM = -3,   /* device or host allocation failed (cf. "Out of memory", rtl_airband.cpp:307) */
    ABG_ECUDA = -4,    /* a CUDA call or kernel failed; abg_last_error() has cudaGetErrorString() */
    ABG_ERANGE = -5,   /* device / channel index out of range */
    ABG_EOVERFLOW = -6 /* abg_push: device-side input buffer full (cf. input_t.overflow_count, input-helpers.cpp:56-60) */
};

/* What demodulate() reads from channel_t + freq_t for one channel (reference src/rtl_airband.h:223-263), after
 * parse_channels() has resolved the config file (reference src/config.cpp:306-726). */
typedef struct abg_channel_cfg {
    int32_t bin;            /* dev->bins[i] == dev->base_bins[i], reference src/config.cpp:666-667 */
    int32_t modulation;     /* freq_t.modulation */
    int32_t needs_raw_iq;   /* channel_t.needs_raw_iq */
    int32_t has_iq_outputs; /* channel_t.has_iq_outputs */
    uint32_t dm_dphi;       /* channel_t.dm_dphi, reference src/config.cpp:679-712 */
    float alpha;            /* channel_t.alpha (NFM de-emphasis, reference src/rtl_airband.cpp:87, config.cpp:636-638) */
    float ampfactor;        /* freq_t.ampfactor */
    float squelch_level;    /* > 0: Squelch::set_squelch_level_threshold(level) (config.cpp:437-472) */
    float squelch_snr_db;   /* >= 0: Squelch::set_squelch_snr_threshold(db) afterwards (config.cpp:473-515) */
    float lowpass_hz;       /* > 0: LowpassFilter(lowpass_hz, WAVE_RATE); config passes bandwidth/2 (config.cpp:604,615) */
    float notch_hz;         /* > 0: NotchFilter(notch_hz, WAVE_RATE, notch_q) (config.cpp:541,557) */
    float notch_q;
    float ctcss_hz;         /* > 0: Squelch::set_ctcss_freq(ctcss_hz, WAVE_RATE) (config.cpp:575,584) */
    int32_t afc;            /* channel_t.afc, 0 = off */
} abg_channel_cfg;

/* What demodulate() reads from device_t + input_t (reference src/rtl_airband.h:266-286, src/input-common.h:39-57). */
typedef struct abg_device_cfg {
    int32_t sfmt;        /* input_t.sfmt */
    float fullscale;     /* input_t.fullscale (used by the S16 / F32 branches only, rtl_airband.cpp:403,421) */
    int32_t sample_rate; /* input_t.sample_rate */
    int32_t n_channels;  /* device_t.channel_count */
    const abg_channel_cfg* channels;
} abg_device_cfg;

/* Process-wide settings: globals fft_size and fm_demod (reference src/rtl_airband.cpp:83-90) and the compile-time
 * WAVE_RATE (8000, or 16000 in an -DNFM=ON build, reference src/rtl_airband.h:65-71) as a run-time value. */
typedef struct abg_config {
    int32_t fft_size;
    int32_t wave_rate;
    int32_t fm_demod;
    int32_t n_devices; /* devices[device_start .. device_end) of one demod thread (demod_params_t, rtl_airband.h:310-320) */
    const abg_device_cfg* devices;
} abg_config;

/* Squelch getters the stats file / TUI read (reference src/squelch.h:89-96, src/output.cpp:606-766) plus the
 * channel scalars tests compare. */
typedef struct abg_squelch_stats {
    float noise_level, signal_level, squelch_level;
    uint64_t open_count, flappy_count, ctcss_count, no_ctcss_count;
    float agcavgfast;        /* freq_t.agcavgfast */
    uint32_t dm_phi;         /* channel_t.dm_phi */
    int32_t bin;             /* current dev->bins[i] */
    uint64_t active_counter; /* freq_t.active_counter, reference src/rtl_airband.cpp:645-647 */
    /* the three levels as the stats file and the TUI print them: level_to_dBFS(), reference src/util.cpp:169-180
     * (output.cpp:624-700 channel_dbfs_*_level gauges, rtl_airband.cpp:632-643) */
    float noise_level_dbfs, signal_level_dbfs, squelch_level_dbfs;
} abg_squelch_stats;

/* Engine tuning (0 = default everywhere). */
typedef struct abg_options {
    int32_t cuda_device;        /* ordinal; -1 = current device */
    int32_t max_batches_per_run;/* capacity of one abg_run() per device, in WAVE_BATCH units (default 4) */
    int32_t input_capacity_batches; /* device-side raw sample buffer per device, in batches of input (default max_batches_per_run + 2) */
    int32_t fft_mode;           /* 0 auto, 1 full spectrum every frame, 2 output-pruned last pass (only the configured bins, FP32 pipes),
                                   3 the configured bins' DFT as an integer GEMM on the tensor cores (U8/S8 input whose hop is a
                                   multiple of 16 samples; other devices use 2) */
    int32_t reserved[4];
} abg_options;

typedef struct abg_engine abg_engine;

ABG_API const char* abg_last_error(void);
ABG_API const char* abg_version(void);

/* init_demod() + the engine set-up at the top of demodulate() (reference src/rtl_airband.cpp:253-266,292-351). */
ABG_API int abg_create(const abg_config* cfg, const abg_options* opt, abg_engine** out);
/* gpu_fft_release() analogue (reference src/rtl_airband.cpp:361-364). */
ABG_API void abg_destroy(abg_engine* e);

/* WAVE_BATCH (= wave_rate / 8) and the hop in complex samples for a device (rtl_airband.cpp:394). */
ABG_API int abg_wave_batch(const abg_engine* e);
ABG_API int abg_hop(const abg_engine* e, int dev);

/* Consumer side of the input ring (reference src/rtl_airband.cpp:370-375,402-455,669): hand over `nbytes` of raw
 * ring-format bytes for one device, in order.  The adapter copies [bufs, bufs + n) out of input_t.buffer and advances
 * bufs by what it pushed.  Copies host->device asynchronously on the engine's ingest stream. */
ABG_API int abg_push(abg_engine* e, int dev, const void* iq, size_t nbytes);
/* Batches a device could complete right now under the reference's fill rule
 * `available >= bps + fft_size*bytes_per_sample*2` (rtl_airband.cpp:394-400). */
ABG_API int abg_batches_available(const abg_engine* e, int dev);

/* One pass of the hot path: every device with enough buffered input advances by up to max_batches batches
 * (0 < max_batches <= options.max_batches_per_run; < 0 means the maximum).  Asynchronous; returns the number of
 * device-batches enqueued.  Finished batches are queued per device in order. */
ABG_API int abg_run(abg_engine* e, int max_batches);
/* Wait for everything enqueued so far. */
ABG_API int abg_sync(abg_engine* e);
/* Make the engine's main stream (see abg_set_stream) wait for all demodulation work enqueued so far, without blocking
 * the host: a caller-side event recorded on that stream afterwards covers K1, K2 and the result copies.  (K2 runs on
 * an internal second stream so that it overlaps the next run's K1.) */
ABG_API int abg_join(abg_engine* e);

/* Number of finished, unfetched batches of a device (the reference's dev->waveavail flag, one level deeper). */
ABG_API int abg_batches_ready(abg_engine* e, int dev);
/* What output_thread()/process_outputs() consume for the oldest finished batch of a device
 * (reference src/output.cpp:456-559,903-923): waveout[C][WAVE_BATCH] (= channel_t.waveout[0..WAVE_BATCH) before the
 * AGC_EXTRA tail copy at output.cpp:920, which the engine performs itself), iq_out[C][2*WAVE_BATCH] (may be NULL),
 * axcindicate[C].  Returns 1 if a batch was popped, 0 if none is ready, < 0 on error.  Synchronises as needed. */
ABG_API int abg_fetch_batch(abg_engine* e, int dev, float* waveout, float* iq_out, char* axcindicate);
/* Same for up to max_batches finished batches of one device in one call: waveout[n][C][WAVE_BATCH], iq_out[n][C][2*WAVE_BATCH]
 * (may be NULL), axcindicate[n][C].  Returns the number of batches popped. */
ABG_API int abg_fetch_batches(abg_engine* e, int dev, int max_batches, float* waveout, float* iq_out, char* axcindicate);

ABG_API int abg_get_stats(abg_engine* e, int dev, int chan, abg_squelch_stats* out);
/* Retune a channel's bin between batches: scan mode (controller_thread, reference src/rtl_airband.cpp:101-139) or an
 * external AFC.  Sets both bins[] and base_bins[]. */
ABG_API int abg_set_bin(abg_engine* e, int dev, int chan, int bin);

/* Which K1 implementation a device's frames go through: 1 full-spectrum FFT, 2 output-pruned FFT, 3 tensor-core DFT. */
ABG_API int abg_fft_path(const abg_engine* e, int dev);

/* ---- benchmark / multi-GPU helpers (not part of the reference surface) -------------------------------------- */
/* Upload a raw stream that stays resident in HBM and is replayed by abg_run_resident(): the timed region of the
 * throughput benchmark then starts with inputs already on the device. `nbytes` must cover max_batches_per_run batches. */
ABG_API int abg_resident_load(abg_engine* e, int dev, const void* iq, size_t nbytes);
/* Process n_batches batches of every device from its resident stream (channel state carries over between calls). */
ABG_API int abg_run_resident(abg_engine* e, int n_batches);
/* Use an existing CUDA stream (cudaStream_t as void*) as the engine's main stream, e.g. torch's current stream, so
 * that caller-side CUDA events bracket the engine's work. */
ABG_API int abg_set_stream(abg_engine* e, void* cuda_stream);
/* Kernel launches issued by this engine since creation (bench.py reports it as gpu_launches). */
ABG_API uint64_t abg_launch_count(const abg_engine* e);

/* Device time of the most recent run, from CUDA events recorded on the engine's stream around its kernels:
 * ms4[0] = K1 (convert+window+FFT+bins, all groups), ms4[1] = K2 (demodulation), ms4[2] = mixers + result copies + tail
 * copy, ms4[3] = whole run.  Waits for that run to finish. */
/* Optional: page-lock a host buffer that abg_push will be fed from (in the reference: input_t.buffer, the ring filled by
   the SDR threads, src/input-helpers.cpp:27-36; buf_size + 2*bytes_per_sample*fft_size bytes) so the host->device copies
   are asynchronous DMA.  Unregister before freeing the buffer. */
ABG_API int abg_host_register(void* ptr, size_t nbytes);
ABG_API int abg_host_unregister(void* ptr);
/* Returns once every abg_push so far has been read out of the caller's memory (with page-locked memory the copies are
   asynchronous): call it before letting a producer overwrite ring space that was pushed from.  Does not wait for kernels. */
ABG_API int abg_ingest_sync(abg_engine* e);

/* Scan mode.  Reference: an R_SCAN device has one channel with freqlist[freq_count] (src/rtl_airband.h:250-252); every
   freq_t owns its Squelch, NotchFilter, LowpassFilter, agcavgfast, ampfactor, modulation and active_counter
   (src/rtl_airband.h:223-233).  controller_thread switches channels[0].freq_idx and retunes the input
   (src/rtl_airband.cpp:101-139); demodulate() picks fparms = freqlist + freq_idx at the start of every batch (:498).
   abg_scan_configure installs the list for a channel: freqs[i] supplies the freq_t part of entry i (modulation,
   ampfactor, squelch_*, lowpass_hz, notch_*, ctcss_hz; the channel_t part - bin, dm_dphi, alpha, afc, needs_raw_iq,
   has_iq_outputs - stays what abg_create was given).  Every entry starts from a fresh freq_t; entry 0 becomes current.
   abg_scan_select makes entry freq_idx current for all batches demodulated by later abg_run calls; the state of the
   entry it replaces is kept on the device and resumes when that entry is selected again. */
ABG_API int abg_scan_configure(abg_engine* e, int dev, int chan, int n_freqs, const abg_channel_cfg* freqs);
ABG_API int abg_scan_select(abg_engine* e, int dev, int chan, int freq_idx);

ABG_API int abg_last_run_times(abg_engine* e, float* ms4);
/* Measurement aid: 5 timestamps (K1 start, K1 end, K2 start, K2 end, end of run; ms since the oldest run's K1 start) for
   each of the last n_runs (1..8) runs into ms[5*n_runs]; shows how consecutive runs overlap on the device. */
ABG_API int abg_debug_timeline(abg_engine* e, int n_runs, float* ms);

/* Band spectrum monitor (not part of the reference surface: the reference opens each SDR exclusively, so there is no
 * other way to see the band while it runs).  For a device with the monitor on at stride s >= 1, batch b of that device
 * covers the B = WAVE_BATCH frames whose |X[bin]| fill wavein[AGC_EXTRA + j], j in [0, B); counted from the device's first
 * frame that is frame f = AGC_EXTRA + b*B + j.  The frames with j % s == 0 are selected, n = ceil(B / s), and
 *     P[k] = (1/n) * sum over the selected f of |X_f[k]|^2,   k = 0 .. fft_size-1, natural bin order,
 * where X_f is what fftwf_execute writes at reference src/rtl_airband.cpp:460: the unnormalised forward DFT of the
 * converted, windowed frame, with the same LUTs, full-scale and Blackman-Harris window as the audio path.  The selection is
 * relative to the batch, so spectra do not depend on how batches are grouped into runs, and the sums are bitwise
 * reproducible.  sqrtf(P[k]) is on the scale of the squelch levels: level_to_dBFS(sqrtf(P[k])) (reference
 * src/util.cpp:169-180) is comparable with abg_squelch_stats.noise_level_dbfs / signal_level_dbfs.  A stride of
 * ceil(fft_size / hop) selects non-overlapping frames.
 * Computed on the GPU by one extra kernel per run, after K1 on the K1 stream (it delays the next run's K1, not K2).
 * With every device off (the default) nothing is launched, allocated or copied.  Resident runs (abg_run_resident) compute
 * spectra but queue none; batches fed through abg_debug_inject_wavein have no frames and produce no spectrum.
 *
 * abg_spectrum_configure: frame_stride 0 = off, >= 1 = on, for batches enqueued by later abg_run / abg_run_resident calls.
 * ABG_ERANGE for a bad device, ABG_EINVAL for a negative stride.  Waits for the engine's K1 stream. */
ABG_API int abg_spectrum_configure(abg_engine* e, int dev, int frame_stride);
/* Pop the oldest unfetched spectrum of a device: power[fft_size] (may be NULL), batch_seq = the device's batch number
 * among the batches abg_run demodulated since abg_create (0 = the first), n_frames = n.  Returns 1 if one was popped, 0
 * if none is ready, < 0 on error; waits for the run that computed it.  Lossy by design: a device keeps at most
 * max_batches_per_run + 2 spectra and a newer one overwrites the oldest (gaps show in batch_seq); the monitor never holds
 * a result slot or makes abg_run report ABG_EOVERFLOW.  Spectra already queued stay fetchable after the monitor is
 * switched off or its stride changed. */
ABG_API int abg_fetch_spectrum(abg_engine* e, int dev, float* power, uint64_t* batch_seq, int32_t* n_frames);
/* Measurement aid: device time of the spectrum kernel of the most recent run, from CUDA events around it on the K1 stream
 * (0 if that run computed no spectrum).  Waits for it. */
ABG_API int abg_debug_spectrum_time(abg_engine* e, float* ms);

/* Carrier frequency meter (not part of the reference surface: it shows how far each transmitter sits from its configured
 * frequency while the engine holds the SDRs, to well below one FFT bin).  For a device with the meter on, batch b covers
 * the same B = WAVE_BATCH frames as the band spectrum, f_j = AGC_EXTRA + b*B + j, j in [0, B).  With X_f the value of the
 * channel's bin in frame f (channel_t.iq_in, reference src/rtl_airband.cpp:483-489; the bin the batch used, so AFC moves
 * it between batches), for every channel c
 *     R[c] = sum_{j=0}^{B-2} X_{f_{j+1}} * conj(X_{f_j})    (complex, float32)
 *     E[c] = sum_{j=0}^{B-1} |X_{f_j}|^2                     (float32)
 * Only pairs inside the batch count, so the results do not depend on how batches are grouped into runs, and the sums are
 * bitwise reproducible (fixed reduction order).
 * Consecutive frames start hop = abg_hop() samples apart, so a tone at baseband frequency f gives X_{f+1} = X_f *
 * exp(2*pi*i * f * hop / sample_rate) for any bin of its main lobe: arg(R) / (2*pi) is f * hop / sample_rate modulo 1.
 * An AM envelope leaves the phase alone, and a symmetric FM tone of peak deviation D shrinks |R| by
 * J0(2*pi*D*hop/sample_rate) and keeps its direction while that is positive (D below about 3 kHz at 8000 frames/s), as
 * long as the window weighs the upper and lower sidebands alike.  Once the carrier is off its bin's centre they are
 * weighed unequally and the reading is biased towards the stronger one: with the 7-term Blackman-Harris window, a 60 % AM
 * tone at 1 kHz 3.5 kHz from the centre reads about 4 Hz off in a 10 kHz bin and 0.3 Hz off in a 39 kHz bin, NFM with
 * D = 2.5 kHz about 180 Hz and 15 Hz off; a steady carrier reads exactly.  The carrier's error relative
 * to the configured frequency, unambiguous within +-sample_rate / (2*hop) (about +-WAVE_RATE/2), is
 *     offset_hz = wrap(arg(R) / (2*pi) - channel_offset_hz * hop / sample_rate) * sample_rate / hop,  wrap to [-0.5, 0.5)
 * with channel_offset_hz = freq - centerfreq of the configured channel (or of the scan entry the batch used); use hop, not
 * WAVE_RATE, when sample_rate / WAVE_RATE is not an integer (as calc_dm_dphi does, reference src/config.cpp:679-712).
 * |R| / E lies in [0, 1] (Cauchy-Schwarz): about 1 for a carrier with a steady envelope, 0.955 for a 60 % AM tone at
 * 1 kHz.  It is NOT a noise gate: consecutive frames overlap, so white noise alone gives |R| / E ~ rho_w(hop) =
 * sum w[n] w[n+hop] / sum w[n]^2 of the Blackman-Harris window, with its phase at the bin centre: 0 when fft_size <= hop,
 * 0.59 at fft_size 2048 / hop 320, 0.92 at 4096 / 256, 0.98 at 8192 / 256.  Read the offset on batches whose
 * axcindicate shows a signal: the squelch is the gate.
 * Computed on the GPU by one extra kernel per run on the K1 stream, after K1 (and after the band spectrum when that is
 * on); K2 does not wait for it.  With every device off (the default) nothing is launched, allocated or copied.
 * Resident runs (abg_run_resident) compute the sums but queue none; batches fed through abg_debug_inject_wavein have no
 * frames and produce none.
 *
 * abg_carrier_configure: on = 1 / 0 switches the meter on / off for batches enqueued by later abg_run / abg_run_resident
 * calls.  ABG_ERANGE for a bad device, ABG_EINVAL for any other value of on.  Waits for the engine's K1 stream. */
ABG_API int abg_carrier_configure(abg_engine* e, int dev, int on);
/* Pop the oldest unfetched meter reading of a device: lag1[n_channels][2] = R (re, im), energy[n_channels] = E (either may
 * be NULL), batch_seq numbered as for abg_fetch_spectrum.  Returns 1 if one was popped, 0 if none is ready, < 0 on error;
 * waits for the run that computed it.  The queue is lossy exactly like the spectrum's: max_batches_per_run + 2 readings
 * per device, the oldest overwritten first; the meter never holds a result slot or causes ABG_EOVERFLOW, and readings
 * already queued stay fetchable after the meter is switched off. */
ABG_API int abg_fetch_carrier(abg_engine* e, int dev, float* lag1, float* energy, uint64_t* batch_seq);
/* Measurement aid: device time of the meter kernel of the most recent run, from CUDA events around it on the K1 stream
 * (0 if that run metered nothing).  Waits for it. */
ABG_API int abg_debug_carrier_time(abg_engine* e, float* ms);

/* Input level meter (not part of the reference surface: it shows how a device's gain sits in its ADC's range while the
 * engine holds the SDR, which rtl_test or an SDR program's IQ histogram would otherwise need the dongle for).  For a device
 * with the meter on, batch b (numbered as for the band spectrum) covers the n = WAVE_BATCH * hop complex samples
 * s in [s0, s0 + n), s0 = (AGC_EXTRA + b*WAVE_BATCH) * hop, hop = abg_hop(): the first hop samples of each of the batch's
 * frames.  Consecutive batches tile the stream after its first AGC_EXTRA * hop samples; no sample counts twice, and a
 * reading depends on its batch only, never on how batches are grouped into runs or on push sizes.
 * For each component k (0 = I, 1 = Q) of each sample the level v is the reference's conversion before the window
 * (src/rtl_airband.cpp:316-324,402-455), in float32, rounded to nearest, no contraction:
 *     U8: (c - 127.5f) / 127.5f     S8: c / 128.0f     S16: (1.0f / fullscale) * (float)x     F32: (1.0f / fullscale) * x
 * and per batch
 *     hist[k][i] = number of components with clamp(floor((v + 1.0f) * 128.0f), 0, 255) == i      (float32)
 *     peak[k]    = max |v|                                                                            (float32)
 *     sum[k] = sum v,   sum_sq[k] = sum v^2,   sum_iq = sum v_I * v_Q                                 (double)
 * For U8 and S8 every ADC code has a bin of its own (U8: bin = code, S8: bin = code + 128), so hist is the code histogram
 * and hist[k][0] + hist[k][255] counts the components at the ends of the ADC's range (U8 codes 0 and 255, S8 -128 and
 * 127).  S16 and F32 bins are 1/128 of full scale wide: only the 8-bit formats give a per-code histogram; the end bins
 * hold the outer 1/128 of the range and every level beyond full scale, and peak shows how far beyond it went.
 * The sums of the integer formats are exact integer sums of the codes, converted once: they are the sums of the exact
 * levels (2c - 255) / 255 (U8), c / 128 (S8) and x * (double)(1.0f / fullscale) (S16), before the float32 rounding of v.
 * F32 sums add the float32 v in double, in a fixed order.  Every field is bitwise reproducible.
 * Computed on the GPU by one extra kernel per run on the K1 stream, after K1 (and after the band spectrum and the carrier
 * meter when those are on); it re-reads the device's raw bytes, K2 does not wait for it.  With every device off (the
 * default) nothing is launched, allocated or copied.  Resident runs (abg_run_resident) compute readings but queue none;
 * batches fed through abg_debug_inject_wavein have no samples and produce none. */
typedef struct abg_input_levels {
    uint64_t batch_seq;   /* as for abg_fetch_spectrum */
    uint64_t n_samples;   /* complex samples, WAVE_BATCH * hop */
    double sum[2];        /* [I, Q] */
    double sum_sq[2];
    double sum_iq;
    float peak[2];
    uint32_t hist[2][256];
} abg_input_levels;
/* abg_input_meter_configure: on = 1 / 0 switches the meter on / off for batches enqueued by later abg_run /
 * abg_run_resident calls.  ABG_ERANGE for a bad device, ABG_EINVAL for any other value of on.  Waits for the engine's K1
 * stream. */
ABG_API int abg_input_meter_configure(abg_engine* e, int dev, int on);
/* Pop the oldest unfetched reading of a device into *out.  Returns 1 if one was popped, 0 if none is ready, < 0 on error;
 * waits for the run that computed it.  The queue is lossy exactly like the spectrum's: max_batches_per_run + 2 readings per
 * device, the oldest overwritten first; the meter never holds a result slot or causes ABG_EOVERFLOW, and readings already
 * queued stay fetchable after the meter is switched off. */
ABG_API int abg_fetch_input_levels(abg_engine* e, int dev, abg_input_levels* out);
/* Measurement aid: device time of the meter kernel of the most recent run, from CUDA events around it on the K1 stream
 * (0 if that run metered nothing).  Waits for it. */
ABG_API int abg_debug_input_meter_time(abg_engine* e, float* ms);

/* Mixer path (reference src/mixer.cpp:82-83,114-140,189-214): mixer m's output for a batch is, per sample,
 * sum over its inputs (in input order) of waveout * (ampfactor * ampl) [left] and * (ampfactor * ampr) [right], taken
 * over the inputs whose channel had axcindicate != NO_SIGNAL in that batch (mixer_put_samples' has_signal), where
 * ampl = fminf(1, 1 - balance), ampr = fminf(1, 1 + balance).  The reference paces this with wall-clock intervals
 * (mixer.cpp:142-156); here it is deterministic: batch b of a run mixes every input whose device produced batch b in
 * that run.  The sums are computed on the device right after demodulation. */
typedef struct abg_mixer_input {
    int32_t dev, chan;
    float ampfactor; /* mixinput_t.ampfactor */
    float balance;   /* -1..1 (mixer.cpp:82-83) */
} abg_mixer_input;
/* Define all mixers at once: mixer m owns inputs[input_offsets[m] .. input_offsets[m+1]). */
ABG_API int abg_mixers_configure(abg_engine* e, int n_mixers, const int32_t* input_offsets, const abg_mixer_input* inputs);
/* Pop the oldest finished batch of one mixer: left[WAVE_BATCH], right[WAVE_BATCH] (may be NULL), has_signal
 * (channel->axcindicate of the mixer channel: 1 = SIGNAL).  Returns 1 if popped, 0 if none. */
ABG_API int abg_fetch_mixer_batch(abg_engine* e, int mixer, float* left, float* right, int* has_signal);
/* Device pointers to the partial sums of the LATEST run, for a cross-GPU reduction when a mixer's inputs are sharded
 * over several engines: sums float[max_batches_per_run][n_mixers][2][WAVE_BATCH], flags int32[max_batches_per_run][n_mixers]. */
ABG_API int abg_mixer_device_buffers(abg_engine* e, float** dev_sums, int32_t** dev_flags);

/* ---- stage taps for tests ---------------------------------------------------------------------------------- */
/* Run conversion + window + FFT on one frame of `dev`'s format and return the full spectrum in natural bin order
 * (fftout[2*fft_size]); exercises the same kernel code as abg_run. */
ABG_API int abg_debug_frame(abg_engine* e, int dev, const void* iq_frame, float* fftout);
/* The most recent run's results as the device holds them (resident runs export nothing): wout float[Gp][P] channel-major
 * audio ([0, AGC_EXTRA) is already the next run's look-back), axc[max_batches_per_run][Gp]; dims[4] = {G, Gp, P, nb}. */
ABG_API int abg_debug_run_outputs(abg_engine* e, int32_t* dims, float* wout, unsigned char* axc);
/* What K1 of the most recent run stored (resident runs included), before any demodulation: rows [AGC_EXTRA, AGC_EXTRA + rows)
 * of its time-major output buffers, win float[rows][Gp] = |X[bin]| (channel_t.wavein) and iqin float[rows][Gp][2] = X[bin]
 * (channel_t.iq_in); dims[4] = {G, Gp, rows, nb} with rows = max_batches_per_run * WAVE_BATCH.  Row j of a device that ran n
 * batches is its frame AGC_EXTRA + (batches before the run) * WAVE_BATCH + j for j < n * WAVE_BATCH and stale beyond.  K2 never
 * writes these rows, so closed-squelch stretches are visible here.  Waits for the run; either pointer may be NULL. */
ABG_API int abg_debug_k1_outputs(abg_engine* e, int32_t* dims, float* win, float* iqin);
/* Feed |X[bin]| values straight into the demodulation state machine of one device (K1 skipped): wavein[C][n_batches *
 * WAVE_BATCH] becomes channel_t.wavein[AGC_EXTRA ...], and iq_in[C][n_batches * WAVE_BATCH][2] (may be NULL) the X[bin]
 * values of the same frames (channel_t.iq_in, where K1 would have stored them); results are fetched as usual.  For the
 * ports of the reference's own Squelch / CTCSS unit tests (reference src/test_squelch.cpp:51-281, src/test_ctcss.cpp:122-155)
 * and the exact comparisons of the demodulation kernel with the CPU oracle.  The device must not be fed with abg_push; its
 * channels must not use AFC, and with iq_in == NULL must not need raw I/Q.  Returns the number of batches enqueued. */
ABG_API int abg_debug_inject_wavein(abg_engine* e, int dev, int n_batches, const float* wavein, const float* iq_in);
/* Measurement aid: per-role clock64 stamps of the tensor-core K1 (environment variable ABG_K1_TC_TRACE set at launch time);
 * out[256 CTAs][4 roles: producer, epilogue, loader, MMA][16 tiles][4 events]. */
ABG_API int abg_debug_k1tc_trace(long long* out);
/* Measurement aid: 64 event counters of the K2 tile paths (copied and cleared); only the `make stats` build counts. */
ABG_API int abg_debug_k2_stats(unsigned long long* out);
/* Host-only: plan and coefficient table of the tensor-core K1 (fft_mode 3) for one device, as abg_create builds them
 * (window * twiddle quantised to `digits` signed 8-bit digits, in the shared-memory image the MMA reads).
 * plan[14] = {eligible, K, HC, S, NC, ND, C2p, KBS, NSTB, acc_regs, smem_bytes, halo, consumer_warpgroups, pps} (KBS = k-steps
 * per column pair and shared-memory stage at most, NSTB = stages in the ring, pps = column pairs per stage at most);
 * tab == NULL queries the plan only. */
ABG_API int abg_debug_tc_table(int fft_size, int sfmt, int hop_bytes, float fullscale, int n_channels, const int32_t* bins, int digits,
                               int32_t* plan, signed char* tab, size_t tab_cap, long long* sq, double* cscale);

#ifdef __cplusplus
}
#endif
#endif /* AIRBAND_B200_H */
