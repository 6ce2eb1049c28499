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

/* Sub-band I/Q outputs (not part of the reference surface: a channel's iq_out is one FFT bin at WAVE_RATE and zero while
 * its squelch is closed, so a decoder of a wider or ungated signal, or a recorder of a whole sub-band, would otherwise
 * need a dongle of its own).  Each device has up to ABG_SUBBAND_MAX outputs; output k of device dev is a digital
 * down-converter: mixer, FIR low-pass and decimator, computed on the GPU from the raw samples the engine already holds.
 * With offset_hz, decimation D (1 <= D <= WAVE_BATCH * hop) and real coefficients h[0..L) (1 <= L <= ABG_SUBBAND_MAX_COEFFS):
 *     v[s]  = complex level of absolute sample s (counted from the device's first pushed sample), the input meter's
 *             float32 conversion: U8 (c - 127.5f) / 127.5f, S8 c / 128.0f, S16 / F32 (1.0f / fullscale) * x
 *     delta = llround(offset_hz / sample_rate * 2^32) mod 2^32; the output's true frequency is delta * sample_rate / 2^32
 *             folded into [-sample_rate/2, sample_rate/2)
 *     y[m]  = sum_{j=0}^{L-1} h[j] * v[mD - j] * exp(-2 pi i ((delta * (mD - j)) mod 2^32) / 2^32)
 * The phase is exact integer arithmetic on the absolute sample index: the oscillator neither drifts nor depends on how
 * batches are grouped.  Batch b (numbered as for the band spectrum) covers the input meter's samples s in [s0, s0 + n),
 * s0 = (AGC_EXTRA + b*WAVE_BATCH) * hop, n = WAVE_BATCH * hop, and carries the outputs m with s0 <= mD < s0 + n:
 * m = ceil(s0 / D) .. ceil((s0 + n) / D) - 1, floor(n / D) or ceil(n / D) of them.  An output's input starts at s0 of the
 * first batch it covers after it was switched on or reconfigured; earlier samples count as zero, so its first L - 1
 * outputs carry the filter's start-up transient.  A scan-mode retune moves the centre frequency and the output with it.
 * Each y[m] is summed in a fixed order that depends on (m, L) only: outputs are bitwise reproducible for every
 * max_batches_per_run, push pattern and fft_mode.  Against float64 each output is within a few L * 2^-24 * sum|h| * max|v|.
 * Computed by one extra kernel per run on the K1 stream, after K1 and the other monitors; K2 does not wait for it.  While
 * any output of a device is on, abg_push's compaction keeps (L_max - 1) samples before the next unconsumed one (L_max:
 * the longest filter switched on), so the input buffer holds up to that many samples less of new input than
 * input_capacity_batches says.  With every output off (the default) nothing is launched, allocated or copied and
 * compaction is unchanged.  Resident runs (abg_run_resident) compute outputs over the resident buffer (samples before it
 * count as zero) but queue none; batches fed through abg_debug_inject_wavein have no samples and produce none. */
#define ABG_SUBBAND_MAX 8
#define ABG_SUBBAND_MAX_COEFFS 4096
/* abg_subband_configure: decim = 0 switches output k off; otherwise it is (re)configured and restarts, for batches
 * enqueued by later abg_run / abg_run_resident calls.  ABG_ERANGE for a bad dev or k; ABG_EINVAL for |offset_hz| >
 * sample_rate / 2 (or not finite), decim outside [0, WAVE_BATCH * hop], n_coeffs outside [1, ABG_SUBBAND_MAX_COEFFS],
 * null coeffs or a coefficient that is not finite.  Waits for the engine's K1 stream. */
ABG_API int abg_subband_configure(abg_engine* e, int dev, int k, double offset_hz, int decim, int n_coeffs, const float* coeffs);
/* Pop the oldest unfetched batch of output k: iq[2 * n_samples] interleaved cf32 (room for 2 * ceil(n / D) floats; may be
 * NULL), batch_seq as for abg_fetch_spectrum, first_index = m of its first output (gaps show in both), n_samples.
 * Returns 1 if one was popped, 0 if none is ready, < 0 on error; waits for the run that computed it.  Lossy like the
 * spectrum's queue: max_batches_per_run + 2 batches per output, the oldest overwritten first; never holds a result slot or
 * causes ABG_EOVERFLOW, and batches already queued stay fetchable after the output is switched off or reconfigured. */
ABG_API int abg_fetch_subband(abg_engine* e, int dev, int k, float* iq, uint64_t* batch_seq, uint64_t* first_index, int32_t* n_samples);
/* Measurement aid: device time of the sub-band kernel of the most recent run, from CUDA events around it on the K1 stream
 * (0 if that run computed no output).  Waits for it. */
ABG_API int abg_debug_subband_time(abg_engine* e, float* ms);

/* CTCSS tone meter (not part of the reference surface: the CTCSS gate only works if the operator knows which tone each
 * transmitter sends, and an SDR program's CTCSS decoder or a scanner would need the dongle to find out).  Per channel and
 * batch it measures how much of each sub-audible tone of a list is in the audio the channel produced.
 * B = WAVE_BATCH.  A device's audio batch number a counts the batches it queued for abg_fetch_batch since abg_create,
 * pushed and injected alike (for a pushed device it is the batch_seq of the other monitors).  y[c][aB + j] = waveout[c][j]
 * of that batch, exactly as abg_fetch_batch returns it: the audio after the squelch gate, notch, ampfactor and clamp
 * (reference src/rtl_airband.cpp:584-611).  The tone list f_k, k < K <= ABG_TONE_MAX, applies to the whole engine; by
 * default it is the reference's 51 standard tones (CTCSS::standard_tones, src/ctcss.cpp:87-89).
 *     delta_k   = llround(f_k / wave_rate * 2^32) mod 2^32; the tone measured is delta_k * wave_rate / 2^32
 *     S[c][k]   = sum_{j<B} y[c][aB+j] * exp(-2 pi i ((delta_k * (aB+j)) mod 2^32) / 2^32)     complex float32
 *     E[c]      = sum_{j<B} y[c][aB+j]^2                                                        float32
 *     active[c] = number of j with y[c][aB+j] != 0                                              int32
 * The phase is exact integer arithmetic on the absolute audio index, so the S of consecutive batches add up to the DFT of
 * the longer window: the reference needs 0.4 s to tell every standard tone apart (src/squelch.cpp:111-115), and 4 batches
 * (0.5 s) added on the host give that.  A tone of amplitude A at f_k gives |S| ~ A n / 2 over n samples, and its share of
 * the audio power is 2 |S|^2 / (n E).  Every sum is taken in a fixed order that depends on (B, K) only, so readings are
 * bitwise reproducible whenever the audio is.  Against the sums in float64 with the exact phase, each component of S is
 * within (B + 8) * 2^-23 * sum_j |y_j| and E within (B + 1) * 2^-24 * E; active is exact.
 * Caveats: the meter sees the audio after the gate, so it reads zeros while the squelch is closed; a channel with ctcss
 * set only opens on its own tone (to find an unknown tone, run the channel without ctcss); a notch set at the tone
 * removes it.
 * Computed on the GPU by one extra kernel per run on the K2 stream (stream B), after K2 and the mixers and before the
 * end-of-run export: while the meter is on its time is part of abg_last_run_times ms4[2] and ms4[3].  With every device
 * off (the default) nothing is launched, allocated or copied.  Resident runs (abg_run_resident) compute readings but queue
 * none; batches fed through abg_debug_inject_wavein produce readings like pushed ones. */
#define ABG_TONE_MAX 64
/* abg_tone_meter_configure: on = 1 / 0 switches the meter on / off for the device's batches enqueued by later abg_run /
 * abg_run_resident / abg_debug_inject_wavein calls.  ABG_ERANGE for a bad device, ABG_EINVAL for any other value of on.
 * Waits for the engine's K2 stream. */
ABG_API int abg_tone_meter_configure(abg_engine* e, int dev, int on);
/* Set the engine's tone list for batches of later runs: freqs[n_tones] in Hz, each finite and in (0, wave_rate / 2);
 * freqs == NULL or n_tones == 0 restores the 51 standard tones.  ABG_EINVAL for n_tones outside [0, ABG_TONE_MAX] or a bad
 * frequency (the list is then unchanged).  Waits for the engine's K2 stream. */
ABG_API int abg_tone_meter_set_tones(abg_engine* e, int n_tones, const float* freqs);
/* Pop the oldest unfetched reading of a device: tones[n_channels][K][2] = S (re, im), energy[n_channels] = E,
 * active[n_channels] (any may be NULL; tones needs room for K = the tone count it was computed with, at most
 * ABG_TONE_MAX), batch_seq = a, n_tones = K.  Returns 1 if one was popped, 0 if none is ready, < 0 on error; waits for the
 * run that computed it.  The queue is lossy exactly like the spectrum's: max_batches_per_run + 2 readings per device, the
 * oldest overwritten first; the meter never holds a result slot or causes ABG_EOVERFLOW, and readings already queued stay
 * fetchable, with the K they were computed with, after the meter is switched off or the tone list changed. */
ABG_API int abg_fetch_tone_meter(abg_engine* e, int dev, float* tones, float* energy, int32_t* active, uint64_t* batch_seq,
                                 int32_t* n_tones);
/* Measurement aid: device time of the tone meter kernel of the most recent run, from CUDA events around it on the K2
 * stream (0 if that run metered nothing).  Waits for it. */
ABG_API int abg_debug_tone_meter_time(abg_engine* e, float* ms);

/* Band activity detector (not part of the reference surface: it answers what is transmitting in the band that no channel
 * listens to, and when, while the engine holds the SDR; the band spectrum averages a whole batch, so a short burst sinks
 * into its average).  It reports every burst above a per-bin threshold at the resolution of single frames.
 * A device with the detector on has a frame stride s >= 1, a hang 0 <= h < n, a minimum span m >= 1 (h and m in selected
 * frames) and a threshold thr[k] > 0 for each bin k < fft_size, on the scale of the band spectrum's P[k] (|X|^2).
 *   Frames: batch b (numbered as for the band spectrum) covers f = AGC_EXTRA + b*B + j, j in [0, B), B = WAVE_BATCH.  The
 *     frames with j % s == 0 are selected, numbered i = j / s in [0, n), n = ceil(B / s); the absolute selected index is
 *     q = b*n + i.
 *   Power: p_f[k] = fmaf(re, re, im*im) of X_f[k], the same unnormalised DFT of the converted, windowed frame as the band
 *     spectrum's, in the same float32 expression.  Frame f is active in bin k iff p_f[k] > thr[k].
 *   Burst (independent of batches): a maximal set of active selected frames of one bin in which consecutive members are
 *     at most h + 1 apart in q; it is reported iff q_last - q_first + 1 >= m.  Fields: bin, first_frame and last_frame (f
 *     of its first and last member), n_active (members), peak = max p, sum = sum of p over its members.
 *   Pieces: per batch the detector emits the same grouping restricted to the batch's selected frames, with the flags
 *     ABG_BURST_OPEN_START iff its first i <= h and ABG_BURST_OPEN_END iff its last i >= n - 1 - h.  A piece with neither
 *     flag and a span < m can never grow and is dropped; every other piece is emitted.  sum is added in frame order in
 *     float32, so pieces are bitwise reproducible (for every max_batches_per_run, push pattern, fft_mode and set of other
 *     monitors).
 *   Merging: a piece with OPEN_END in batch b and one with OPEN_START in batch b + 1, in the same bin, join iff their gap
 *     in q is <= h + 1; the m filter is applied after joining.  Merging the pieces of consecutive batches this way gives
 *     exactly the bursts of the definition above: because h < n, a gap that spans a whole batch is longer than h + 1, so
 *     no join reaches past the next batch.
 * Capacity: a reading stores at most ABG_ACTIVITY_MAX_RECORDS pieces and counts all of them (n_total, after the drop
 * above).  When n_total exceeds the capacity the reading is truncated and which pieces are stored is unspecified;
 * otherwise abg_fetch_activity returns them all, sorted by (bin, first_frame) on the host.
 * Computed on the GPU by one extra kernel per run on the K1 stream, after K1 and the other monitors of that stream (the
 * sub-band outputs last); it re-reads the device's raw bytes, K2 does not wait for it.  With every device off (the default)
 * nothing is launched, allocated or copied.  Resident runs (abg_run_resident) compute pieces but queue none; batches fed
 * through abg_debug_inject_wavein have no frames and produce none. */
#define ABG_ACTIVITY_MAX_RECORDS 4096
enum { ABG_BURST_OPEN_START = 1, ABG_BURST_OPEN_END = 2 };
typedef struct abg_burst {
    int32_t bin;              /* natural bin order, 0 .. fft_size-1 */
    int32_t flags;            /* ABG_BURST_OPEN_START | ABG_BURST_OPEN_END */
    uint64_t first_frame;     /* absolute frame number f of the first active frame */
    uint64_t last_frame;      /* ... of the last */
    int32_t n_active;         /* active selected frames */
    float peak;               /* max p */
    float sum;                /* sum of p, in frame order, float32 */
    int32_t reserved;         /* 0; keeps the size at 40 bytes */
} abg_burst;
/* abg_activity_configure: stride = 0 switches the detector off; otherwise it is (re)configured with hang, min_span and
 * thr[fft_size], for batches enqueued by later abg_run / abg_run_resident calls.  ABG_ERANGE for a bad device; ABG_EINVAL
 * for a negative argument, and when stride > 0 for a null thr, a threshold that is not finite or is <= 0, stride >
 * WAVE_BATCH, hang >= ceil(WAVE_BATCH / stride) or min_span < 1.  Waits for the engine's K1 stream. */
ABG_API int abg_activity_configure(abg_engine* e, int dev, int stride, int hang, int min_span, const float* thr);
/* Pop the oldest unfetched reading of a device: the first min(n_stored, cap) of its stored pieces, sorted by (bin,
 * first_frame), into out[cap] (may be NULL with cap = 0); n_stored = pieces the reading stored (min(n_total,
 * ABG_ACTIVITY_MAX_RECORDS)); n_total = pieces it found (n_total > n_stored: truncated); batch_seq as for
 * abg_fetch_spectrum; settings3 = {stride, hang, min_span} it was computed with, so that a caller can refuse to stitch
 * across a change.  Any output pointer may be NULL.  Returns 1 if one was popped, 0 if none is ready, < 0 on error
 * (ABG_EINVAL for cap < 0); waits for the run that computed it.  The queue is lossy exactly like the spectrum's:
 * max_batches_per_run + 2 readings per device, the oldest overwritten first; the detector never holds a result slot or
 * causes ABG_EOVERFLOW, and readings already queued stay fetchable after it is switched off or reconfigured. */
ABG_API int abg_fetch_activity(abg_engine* e, int dev, abg_burst* out, int cap, int32_t* n_stored, int32_t* n_total,
                               uint64_t* batch_seq, int32_t* settings3);
/* Measurement aid: device time of the detector kernel of the most recent run, from CUDA events around it on the K1 stream
 * (0 if that run detected nothing).  Waits for it. */
ABG_API int abg_debug_activity_time(abg_engine* e, float* ms);

/* I/Q history (not part of the reference surface: the activity detector reports a burst only after its batch has been
 * demodulated, and a sub-band output starts at the first batch after it is configured, so without it nothing the detector
 * finds could be captured; an SDR recorder would need a dongle of its own).  A device with the history on keeps its most
 * recent raw samples in HBM, in ring format (never expanded to float), and any sub-band can be cut out of them later.
 * Names as for the sub-band outputs: v[s] is the float32 level of absolute sample s (counted from the device's first pushed
 * sample), and batch b covers the samples [s0, s0 + n), s0 = (AGC_EXTRA + b*WAVE_BATCH) * hop, n = WAVE_BATCH * hop.
 *   What it holds: a device with the history on appends the samples [s0, s0 + n) of every batch that later abg_run calls
 *     demodulate.  Those ranges tile the stream, so the history is always one contiguous range [first, end) of absolute
 *     samples, at most the capacity long; the oldest samples are overwritten first.
 *   Capture: abg_history_subband computes y[m] of the sub-band definition (same delta, same g[j] built on the host by the
 *     same function, same summation order) from the stored samples.  For any m whose live sub-band output with the same
 *     offset_hz, decimation and coefficients had all L taps after its start, the captured y[m] is bitwise equal to the live
 *     one.  Every tap has to lie in the history: there is no zero fill.
 * Computed on the GPU: one extra kernel per run appends the run's bytes, on the K1 stream after K1 and every other monitor of
 * that stream (it re-reads the device's raw bytes, K2 does not wait for it); captures are enqueued on the same stream, so
 * every append they read is ahead of them and every later one that would overwrite their samples queues behind them.  With
 * every device off (the default) nothing is allocated, uploaded, launched or recorded.  Resident runs (abg_run_resident)
 * append from the replay buffer, so that their cost can be measured, but leave the history empty: a capture never mixes
 * replayed and streamed samples.  Batches fed through abg_debug_inject_wavein append nothing.  A scan-mode retune moves the
 * centre frequency under the recorded samples: a capture across a retune mixes both tunings.
 *
 * abg_history_configure: n_batches = 0 switches the history off and frees it; n_batches > 0 gives a capacity of
 * n_batches * WAVE_BATCH * hop samples (abg_hop) for batches enqueued by later abg_run calls.  A change of capacity empties
 * the history; a call that changes nothing returns at once.  ABG_ERANGE for a bad device, ABG_EINVAL for a negative count,
 * ABG_ENOMEM if the allocation fails (the history is then off).  Waits for the engine's K1 stream. */
ABG_API int abg_history_configure(abg_engine* e, int dev, int n_batches);
/* The range [*first, *end) of absolute samples the history holds once every run enqueued so far has finished (first == end:
 * empty).  Does not wait. */
ABG_API int abg_history_range(abg_engine* e, int dev, uint64_t* first, uint64_t* end);
/* Copy the ring-format bytes of samples [first, first + n) into out[n * bytes per complex sample]: byte for byte what was
 * pushed.  ABG_ERANGE if any of them lies outside the range, ABG_EINVAL for n < 0 or a null out.  Waits for the runs that
 * appended them. */
ABG_API int abg_history_raw(abg_engine* e, int dev, uint64_t first, int64_t n, void* out);
/* Down-convert y[m], m in [first_m, first_m + n_out), from the history into iq[2 * n_out] (interleaved cf32, caller memory).
 * ABG_EINVAL for arguments abg_subband_configure refuses with decim >= 1 (decim outside [1, WAVE_BATCH * hop], the offset,
 * the coefficients), n_out < 1 or a null iq; ABG_ERANGE unless first_m * decim - (n_coeffs - 1) >= first and
 * (first_m + n_out - 1) * decim < end.  Any n_out that fits is accepted (large requests are split internally).  Waits for
 * the capture to finish. */
ABG_API int abg_history_subband(abg_engine* e, int dev, double offset_hz, int decim, int n_coeffs, const float* coeffs,
                                uint64_t first_m, int64_t n_out, float* iq);
/* Measurement aid: ms2[0] = device time of the append kernel of the most recent run (0 if that run appended nothing; waits
 * for it), ms2[1] = device time of the kernels of the most recent abg_history_subband (0 before the first), both from CUDA
 * events on the K1 stream. */
ABG_API int abg_debug_history_time(abg_engine* e, float* ms2);

/* History replay (not part of the reference surface: it demodulates any frequency of a device's I/Q history to audio, as a
 * channel configured there in advance would have, so that every transmission the activity detector finds can be heard).
 * Job j replays device dev from batch first_batch (numbered as for the band spectrum) for n_batches batches through the
 * engine's own K1 and K2.  Its outputs are bitwise what this fresh engine produces:
 *   config   abg_create with this engine's fft_size, wave_rate and fm_demod, one device with dev's sfmt, fullscale and
 *            sample_rate, and channels[n_channels] of the job;
 *   options  this engine's cuda_device and fft_mode, everything else default;
 *   input    dev's stream from sample S = first_batch * WAVE_BATCH * hop on (what abg_history_raw(e, dev, S, ...) returns),
 *            run until it has produced n_batches batches.
 * Frame AGC_EXTRA + b*WAVE_BATCH + i of that engine is frame AGC_EXTRA + (first_batch + b)*WAVE_BATCH + i of dev, so
 * replayed batch b is dev's batch first_batch + b, demodulated from a fresh channel state.  The results do not depend on
 * how many jobs share a call or their order, on max_batches_per_run, or on the push pattern the history was filled with.
 * Every sample that engine reads must lie in the history: [S, S + (AGC_EXTRA + n_batches*WAVE_BATCH)*hop + fft_size - hop)
 * inside abg_history_range (its last frame reaches fft_size - hop samples into the batch after the last one).  Several
 * jobs may replay the same device.  Scan mode does not apply to replayed channels.
 * Computed on the GPU: the engine keeps a private replay engine on the same CUDA device with one device per job, so all
 * of a call's jobs share each K1 and K2 launch.  A gather kernel on the K1 stream moves the window's bytes from the history
 * ring into that engine's input buffers (behind every append it reads, ahead of every later one that would overwrite
 * them), in chunks of max_batches_per_run batches.  Nothing is allocated before the first replay; the replay engine is
 * kept for later calls, grows only when a call needs more devices of a shape than it holds, and is freed when the last
 * history is switched off.  Live runs, outputs and monitors are unaffected.
 * The call waits for its results. */
typedef struct abg_replay_job {
    int32_t dev;                      /* device whose history is replayed */
    int32_t n_batches;                /* >= 1 */
    uint64_t first_batch;             /* dev's batch number of the first replayed batch */
    int32_t n_channels;               /* >= 1 */
    const abg_channel_cfg* channels;  /* as abg_create takes them */
    float* waveout;                   /* [n_batches][n_channels][WAVE_BATCH], caller memory */
    float* iq_out;                    /* [n_batches][n_channels][2*WAVE_BATCH] or NULL */
    char* axcindicate;                /* [n_batches][n_channels] */
    abg_squelch_stats* stats;         /* [n_channels] after the last batch, or NULL */
} abg_replay_job;
/* ABG_ERANGE for a bad dev or a window with a sample outside the history (the message gives the range needed), also when
 * the history is off; ABG_EINVAL for n_jobs outside [1, 65535], a null jobs, a channel list abg_create refuses, n_batches < 1 and null
 * waveout or axcindicate. */
ABG_API int abg_history_replay(abg_engine* e, int n_jobs, const abg_replay_job* jobs);
/* Measurement aid: device time of the most recent abg_history_replay: ms2[0] = its gathers, ms2[1] = its replay engine's
 * runs (K1 start to end of run, summed over the chunks); 0 before the first. */
ABG_API int abg_debug_replay_time(abg_engine* e, float* ms2);

/* Live follow (not part of the reference surface: many transmissions the activity detector reports are still going when
 * they are found, and a replay job stops at the history's end).  A follow session is the streaming form of a replay job:
 * it is opened with a job's dev, first_batch and channels but no n_batches, and every abg_follow_run advances it over what
 * the history has gained since, with its channel state carried over.
 *   Output: batch b >= first_batch of a session (waveout, iq_out, axcindicate) is bitwise batch b - first_batch of
 *     abg_history_replay on the job {dev, first_batch, n_batches >= b - first_batch + 1, channels}, and abg_follow_stats
 *     after batch b is that job's stats.  It does not depend on how abg_follow_run calls split the batches, on
 *     max_batches_per_run or the push pattern, on other sessions opening, closing, advancing or falling behind, or on
 *     abg_history_replay calls in between.
 *   Availability: batch b can be demodulated once the history holds every sample the replay reads for it, i.e. end >=
 *     (AGC_EXTRA + (b+1)*WAVE_BATCH)*hop + fft_size - hop, while history batch L ends at (AGC_EXTRA + (L+1)*WAVE_BATCH)*hop.
 *     Where WAVE_BATCH*hop >= fft_size - hop a session therefore trails the live engine by one batch at most (125 ms at
 *     wave_rate 8000): after abg_follow_run its next_batch is the live engine's last batch L (L + 1 when fft_size <= hop).
 *     abg_create also accepts configurations without it (fft_size 8192 with hop <= 8 at WAVE_BATCH 1000, for one); there
 *     a session trails by ceil((fft_size - hop) / (WAVE_BATCH*hop)) batches.
 *   Lost: once the history overwrites the session's next sample not yet read, the session is lost: its queued batches
 *     stay fetchable, then abg_follow_fetch returns ABG_ERANGE.  A session falls behind when its queue is full or when
 *     abg_follow_run is not called often enough.
 *   Queue: a session holds at most queue_batches unfetched batches (enqueued or finished).  abg_follow_run advances it
 *     only into free room, so an unfetched session stops; it does not stall other sessions or hold result slots they need.
 * Computed on the GPU: private follow engines on the same CUDA device, built like the replay engine and kept apart from
 * it, each a pool of devices built for one session shape; sessions in one engine share every K1 and K2 launch.  An engine
 * is never rebuilt: a closed session's device goes back to the pool and is reset for the next session of its shape.  Per
 * chunk of max_batches_per_run batches (one with AFC), abg_follow_run enqueues one gather kernel on the K1 stream (behind
 * every append it reads, ahead of every later one that would overwrite them) and one run per follow engine with work; it
 * decides availability and loss on the host from the enqueued history range and never waits for the live engine's work.
 * Finished batches move from the follow engines' result slots into the sessions' queues at a later abg_follow_run or at
 * the fetch that needs them.  Nothing is allocated before the first open; the follow engines are freed when the last
 * history is switched off (abg_history_configure refuses any change to a device with open sessions) and by abg_destroy.
 * The live engine's channels, outputs and runs are unaffected.  Scan mode does not apply to followed channels. */
typedef struct abg_follow_status {
    int32_t dev;          /* device whose history the session follows */
    int32_t n_channels;
    uint64_t next_batch;  /* the next batch abg_follow_run enqueues */
    int32_t queued;       /* batches enqueued and not fetched yet: [next_batch - queued, next_batch) */
    int32_t lost;         /* 1 once the history overwrote a sample the session still needed */
} abg_follow_status;
/* Open a session on dev from batch first_batch; *session receives its id (ids are never reused within an engine's
 * lifetime).  first_batch may lie beyond the live edge: the session then waits until its samples arrive.  ABG_EINVAL for
 * a channel list abg_create refuses, queue_batches < 1 and null arguments; ABG_ERANGE for a bad dev, a device whose
 * history is off, and a start sample first_batch * WAVE_BATCH * hop below abg_history_range's first (the message gives
 * the range).  Checks everything before any engine state is touched; may wait for the follow engines. */
ABG_API int abg_follow_open(abg_engine* e, int dev, uint64_t first_batch, int n_channels, const abg_channel_cfg* channels,
                            int queue_batches, int32_t* session);
/* Close a session: its unfetched batches are dropped.  ABG_ERANGE for an unknown or closed id. */
ABG_API int abg_follow_close(abg_engine* e, int32_t session);
/* Advance every open session by up to max_batches batches (< 0: as far as the history and its queue room allow, over as
 * many chunks as needed); returns the session-batches enqueued.  Does not wait for the live engine's work; a call that
 * enqueues more than three chunks for one follow engine waits for that engine's run three chunks back. */
ABG_API int abg_follow_run(abg_engine* e, int max_batches);
/* Pop up to max_batches of a session's oldest batches into waveout[n][n_channels][WAVE_BATCH], iq_out[n][n_channels]
 * [2*WAVE_BATCH] (may be NULL) and axcindicate[n][n_channels]; *first_batch (may be NULL) = the batch number of the first
 * popped.  Returns the number popped, 0 if none is queued; waits for the runs that compute them.  ABG_ERANGE for an
 * unknown id and for a lost session with nothing left queued; ABG_EINVAL for max_batches < 0 and null outputs. */
ABG_API int abg_follow_fetch(abg_engine* e, int32_t session, int max_batches, float* waveout, float* iq_out, char* axcindicate,
                             uint64_t* first_batch);
/* A session's device, channel count, next batch, queued batches and lost flag.  Does not wait. */
ABG_API int abg_follow_info(abg_engine* e, int32_t session, abg_follow_status* out);
/* Squelch statistics of channel chan of a session after its batch next_batch - 1, as abg_get_stats gives them; waits for
 * it.  ABG_ERANGE for an unknown id or a bad channel index, ABG_EINVAL for a null out. */
ABG_API int abg_follow_stats(abg_engine* e, int32_t session, int chan, abg_squelch_stats* out);
/* Measurement aid: device time of the most recent abg_follow_run: ms2[0] = its gathers, ms2[1] = its follow-engine runs
 * (from the end of the chunk's gather to the end of the run, summed); 0 if it enqueued nothing.  Waits for them. */
ABG_API int abg_debug_follow_time(abg_engine* e, float* ms2);

/* History analysis (not part of the reference surface: the band spectrum and the activity detector only see the batches
 * after they are switched on, with the settings they had then, so "what was on the band 20 s ago" has no answer unless
 * they were on and set right).  Both can be run over any window of a device's I/Q history, with any settings, after the
 * fact.  Names as for the history: frame f reads the samples [f*hop, f*hop + fft_size), and batch b covers the frames
 * AGC_EXTRA + b*B + j, j in [0, B), B = WAVE_BATCH.
 *   Spectrogram: a job names dev, first_frame, n_rows >= 1, frames_per_row F >= 1 and a stride 1 <= s <= F.  Row r covers
 *     the frames first_frame + r*F + j, j in [0, F); those with j % s == 0 are selected, n = ceil(F / s) of them, and the row
 *     is the band spectrum's P[k] = (1/n) * sum |X_f[k]|^2 over them: the same conversion, window, FFT and float32
 *     expression, summed in the same order (chunks of 32 selected frames, each in frame order, then the chunk sums in chunk
 *     order).  So with F = B and first_frame = AGC_EXTRA + b*B, row r is bitwise the live spectrum of batch b + r at stride s;
 *     any other F (or a first_frame off the batch grid) is the same arithmetic on other frames.
 *   Activity: a job names dev, first_batch, n_batches >= 1 and the detector's stride, hang, min_span and thr[fft_size],
 *     checked as abg_activity_configure checks them.  Its result is the merged bursts over the window: the pieces the live
 *     detector emits for those batches with those settings, joined as merging joins them, except at the window's edges.  A
 *     burst whose first piece had OPEN_START in the window's first batch carries ABG_BURST_OPEN_START, one whose last piece
 *     had OPEN_END in the last batch carries ABG_BURST_OPEN_END, and such edge bursts are kept even with a span below
 *     min_span, since they may continue outside the window; every other burst has flags 0.  Bursts are sorted by (bin,
 *     first_frame), a joined burst's sum is the float32 sum of its pieces' sums in batch order, and every field is bitwise
 *     reproducible.  A batch with more than ABG_ACTIVITY_MAX_RECORDS pieces is counted in n_truncated; the bursts of such a
 *     batch are unspecified, as in a truncated live reading.
 *   Window: every sample of every selected frame must lie in abg_history_range (ABG_ERANGE otherwise, the message gives the
 *     range needed).  A batch's last frames reach fft_size - hop samples into the next batch, so the newest history batch
 *     can be analysed once its successor has been appended, the same lag as live follow.
 * Results do not depend on how jobs are grouped into calls or ordered, on max_batches_per_run or the push pattern, on
 * whether the live spectrum or detector is on, or on other calls in between.  Several jobs may name the same device.  A
 * scan-mode retune inside a window mixes both tunings, as for a capture.
 * Computed on the GPU by the band spectrum's and the detector's own kernels: per chunk, one gather launch on the K1 stream
 * copies every job's window from its history ring into a private scratch buffer (behind every append it reads, ahead of
 * every later one that would overwrite them), then one spectrum or detector launch covers every job.  Partial sums,
 * counters, thresholds, scratch and results are the calls' own: the live monitors are untouched and live runs launch
 * nothing new.  Nothing is allocated before the first call; everything is freed when the last history is switched off and
 * by abg_destroy.  The calls wait for their results.  ABG_EINVAL for n_jobs outside [1, 65535] or a null jobs. */
typedef struct abg_spectrogram_job {
    int32_t dev;
    int32_t n_rows;          /* >= 1 */
    uint64_t first_frame;    /* absolute frame number of row 0's first frame */
    int32_t frames_per_row;  /* F >= 1 */
    int32_t stride;          /* 1 <= stride <= F */
    float* power;            /* [n_rows][fft_size], caller memory */
} abg_spectrogram_job;
/* ABG_ERANGE for a bad dev or a window outside the history (also when the history is off); ABG_EINVAL for n_rows < 1, F < 1,
 * a stride outside [1, F] and a null power. */
ABG_API int abg_history_spectrogram(abg_engine* e, int n_jobs, const abg_spectrogram_job* jobs);
typedef struct abg_activity_job {
    int32_t dev;
    int32_t n_batches;       /* >= 1 */
    uint64_t first_batch;
    int32_t stride, hang, min_span;
    int32_t cap;             /* room in out, >= 0 */
    const float* thr;        /* [fft_size] */
    abg_burst* out;          /* [cap], caller memory; may be NULL with cap = 0 */
    int32_t n_bursts;        /* written: bursts found; the first min(n_bursts, cap) of them are stored */
    int32_t n_truncated;     /* written: batches with more than ABG_ACTIVITY_MAX_RECORDS pieces */
} abg_activity_job;
/* ABG_ERANGE for a bad dev or a window outside the history (also when the history is off); ABG_EINVAL for what
 * abg_activity_configure refuses with stride > 0, for stride 0, n_batches < 1, cap < 0 and a null out with cap > 0. */
ABG_API int abg_history_activity(abg_engine* e, int n_jobs, abg_activity_job* jobs);
/* Measurement aid: device time of the most recent abg_history_spectrogram or abg_history_activity, summed over its chunks:
 * ms3[0] = its gathers, ms3[1] = its spectrum kernels, ms3[2] = its detector kernels; 0 where it had none. */
ABG_API int abg_debug_history_analysis_time(abg_engine* e, float* ms3);

/* Transmission profiles (not part of the reference surface: replaying or following a transmission the activity detector
 * found needs its modulation and CTCSS tone, and a frequency better than the detector's bin; the carrier and tone meters
 * only read configured channels, and the tone meter reads gated audio).  A profile is measured on the raw baseband,
 * before any demodulation.
 * A job names dev, a down-converter (offset_hz, decimation D, coefficients h[0..L)), checked as abg_history_subband checks
 * them, an output window m in [m0, m0 + n), n >= 2, and a tone list f_k, k < K <= ABG_TONE_MAX, each finite and in
 * (0, fs_out / 2) with fs_out = sample_rate / D (tones == NULL or n_tones == 0: the 51 standard tones).  y[m] is bitwise what
 * abg_history_subband(dev, offset_hz, D, L, h, m0, n) returns; then, in float32:
 *     p[m]   = fmaf(y.re, y.re, y.im * y.im)          a[m] = sqrtf(p[m])
 *     z[m]   = y[m+1] * conj(y[m]):  z.re = fmaf(y1.re, y0.re, y1.im * y0.im),  z.im = fmaf(y1.im, y0.re, -(y1.re * y0.im))
 *     phi[m] = atan2f(z.im, z.re)                     for m < m0 + n - 1 (the n - 1 pairs)
 *     delta_k = llround(f_k / fs_out * 2^32) mod 2^32 (the tone meter's integer phase, on the absolute output index m);
 *     c + i s = the float32 cospi / sinpi (sincospif) of (float)(int32_t)(delta_k * m mod 2^32) * 2^-31
 *     tone_fm[k] += (fmaf(phi, c, .), fmaf(-phi, s, .))    tone_am[k] += (fmaf(a, c, .), fmaf(-a, s, .))
 * and the reading holds n, p1 = sum p, p2 = sum p^2 (fmaf(p, p, .)), a1 = sum a, z = sum z, f1 = sum phi, f2 = sum phi^2
 * (fmaf(phi, phi, .)), tone_fm[k] = sum phi[m] exp(-2 pi i ((delta_k m) mod 2^32) / 2^32), tone_am[k] the same sum of a[m]
 * (a phi of an output without a successor counts as 0), and n_tones = K.  Meaning: arg(z) * fs_out / 2 pi is the carrier's
 * offset from the down-converter's true frequency (lib.subband_frequency); f2 about the mean f1 / (n - 1) gives the FM
 * deviation; n * p2 / p1^2 - 1 the envelope's spread; the tone sums carry a CTCSS tone in NFM (tone_fm) and AM (tone_am).
 * Order: the outputs are cut into blocks of ABG_PROFILE_BLOCK outputs (and their pairs) anchored at m0.  Within a block,
 * thread t of 256 adds the terms of outputs t, t + 256, t + 512, t + 768 in that order and a fixed xor-shuffle tree and the
 * 8 warps in order add those; a tone sum is added by lane l over l, l + 32, ... in order, then by the xor tree.  The host
 * adds the block sums in double, in block order.  A reading is therefore bitwise reproducible for any grouping of jobs
 * into calls, job order, chunking, max_batches_per_run, push pattern and set of live monitors.
 * Bound: against float64 sums of the same float32 terms with the exact phase, each of p1, p2, a1, z, f1, f2 is within
 * 16 * 2^-24 * sum |term| (15 float32 roundings per term at most, then the double sum), and each component of a tone sum
 * within 40 * 2^-24 * sum |x| (x = phi or a: 37 roundings at most, the phase's rounding to float, pi * 2^-25, and
 * sincospif's 1 ulp).
 * Window: every tap of every output must lie in abg_history_range, by abg_history_subband's rule: ABG_ERANGE when it does
 * not (the message gives the needed range), when the history is off, and for a bad dev; ABG_EINVAL for n_jobs outside
 * [1, 65535], a null jobs or out, n < 2 and a bad tone list.  The call waits for its results.
 * Computed on the GPU: per chunk, one launch of the history capture per job piece writes y into the profile's own scratch
 * (one extra output at a seam, so that the pair across it is formed from captured values), then one launch of the profile
 * kernel covers every block of every job of the chunk, one CTA per block; the block sums go to a results buffer the host
 * reads after the chunk.  Chunks hold at most 8 M outputs of scratch and 65535 blocks.  Everything runs on the K1 stream,
 * behind every append it reads.  Nothing is allocated before the first call; everything is freed when the last history is
 * switched off and by abg_destroy.  Live runs launch nothing new. */
#define ABG_PROFILE_BLOCK 1024
typedef struct abg_profile {
    int64_t n;                          /* outputs */
    int32_t n_tones;                    /* K */
    int32_t reserved;                   /* 0 */
    double p1, p2, a1;
    double z[2];
    double f1, f2;
    double tone_fm[ABG_TONE_MAX][2];    /* [K][re, im] */
    double tone_am[ABG_TONE_MAX][2];
} abg_profile;
typedef struct abg_profile_job {
    int32_t dev;
    int32_t decim;                      /* D, 1 .. WAVE_BATCH * hop */
    double offset_hz;
    int32_t n_coeffs;                   /* L, 1 .. ABG_SUBBAND_MAX_COEFFS */
    int32_t n_tones;                    /* K, 0 .. ABG_TONE_MAX (0: the 51 standard tones) */
    const float* coeffs;                /* h[L] */
    uint64_t first_m;                   /* m0 */
    int64_t n_out;                      /* n >= 2 */
    const float* tones;                 /* f_k [K] in Hz, or NULL */
    abg_profile* out;                   /* written */
} abg_profile_job;
ABG_API int abg_history_profile(abg_engine* e, int n_jobs, abg_profile_job* jobs);
/* Measurement aid: device time of the most recent abg_history_profile, summed over its chunks: ms2[0] = its capture
 * kernels, ms2[1] = its profile kernels; 0 before the first. */
ABG_API int abg_debug_history_profile_time(abg_engine* e, float* ms2);
/* Host-only: the chunk and block plan abg_history_profile launches for jobs of these shapes (first_m, n_out, n_coeffs and
 * n_tones as in abg_profile_job, n_tones already resolved, 1 .. ABG_TONE_MAX), without an engine.  limits[4] = {scratch
 * outputs, blocks, result floats, coefficients} per chunk.  pieces[cap_pieces][6] = {chunk, job, first output captured,
 * outputs captured, scratch offset, coefficient offset}: one capture launch each, in launch order.  blocks[cap_blocks][8] =
 * {chunk, job, piece, scratch offset, first output, outputs, successor (0 / 1), result offset}: one CTA each.  *n_pieces
 * and *n_blocks are always written; rows past a cap are not.  ABG_EINVAL for what abg_history_profile refuses of these
 * fields. */
ABG_API int abg_debug_profile_plan(int n_jobs, const uint64_t* first_m, const int64_t* n_out, const int32_t* n_coeffs,
                                   const int32_t* n_tones, int64_t* limits, int64_t* pieces, int cap_pieces, int32_t* n_pieces,
                                   int64_t* blocks, int cap_blocks, int32_t* n_blocks);

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
/* The full spectra K1 of the device's most recent launch kept for AFC (K2's AFC block reads them, and only reads them):
 * out float[n_rows][fft_size][2], natural bin order.  Row b is the spectrum of the last frame of the run's batch b, the
 * frame whose iqin row is (b + 1) * WAVE_BATCH - 1 in abg_debug_k1_outputs; its value at a channel's bin is that row's
 * iqin bit for bit.  *n_rows = batches of that launch (0 if the device had none).  ABG_EINVAL for a device without an AFC
 * channel or before any run.  Waits for the run; out may be NULL to query n_rows. */
ABG_API int abg_debug_k1_spectra(abg_engine* e, int dev, int32_t* n_rows, float* out);
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
