/* ORACLE — TEST INFRASTRUCTURE ONLY.
 *
 * C ABI of the CPU oracle: a restatement of the reference's demodulate() hot path
 * (reference src/rtl_airband.cpp:286-672) as a pure function of (configuration, raw I/Q bytes).
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load this.
 * The product (rtlsdr-airband_b200/) never links or calls it.
 *
 * Two shared objects export this same ABI:
 *   oracle/libairband_oracle.so      — everything restated (oracle/leaf_dsp.cpp), builds anywhere
 *   oracle/_ref/libairband_ref.so    — same loop, but Squelch/CTCSS/NotchFilter/LowpassFilter are the
 *                                      reference's own squelch.cpp/ctcss.cpp/filters.cpp compiled in place
 *                                      from /root/reference/src (see oracle/Makefile)
 * Struct layouts are identical to include/airband_b200.h on purpose so one Python description serves both.
 */
#ifndef AIRBAND_ORACLE_H
#define AIRBAND_ORACLE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* sample_format_t values, reference src/input-common.h:31 */
enum { ABO_SFMT_U8 = 1, ABO_SFMT_S8 = 2, ABO_SFMT_S16 = 3, ABO_SFMT_F32 = 4 };
/* enum modulations, reference src/rtl_airband.h:193-199 */
enum { ABO_MOD_AM = 0, ABO_MOD_NFM = 1 };
/* enum fm_demod_algo, reference src/rtl_airband.cpp:88 */
enum { ABO_FM_FAST_ATAN2 = 0, ABO_FM_QUADRI_DEMOD = 1 };

typedef struct abo_channel_cfg {
    int32_t bin;            /* dev->bins[i], reference src/config.cpp:666-667 */
    int32_t modulation;     /* freq_t.modulation */
    int32_t needs_raw_iq;   /* channel_t.needs_raw_iq (NFM, bandwidth, or rawfile output) */
    int32_t has_iq_outputs; /* channel_t.has_iq_outputs */
    uint32_t dm_dphi;       /* channel_t.dm_dphi, reference src/config.cpp:679-712 */
    float alpha;            /* channel_t.alpha (NFM de-emphasis) */
    float ampfactor;        /* freq_t.ampfactor */
    float squelch_level;    /* > 0: set_squelch_level_threshold(level) is called (config.cpp:437-472) */
    float squelch_snr_db;   /* >= 0: set_squelch_snr_threshold(db) is called afterwards (config.cpp:473-515) */
    float lowpass_hz;       /* > 0: lowpass_filter = LowpassFilter(lowpass_hz, wave_rate); = bandwidth/2 */
    float notch_hz;         /* > 0: notch_filter = NotchFilter(notch_hz, wave_rate, notch_q) */
    float notch_q;
    float ctcss_hz;         /* > 0: squelch.set_ctcss_freq(ctcss_hz, wave_rate) */
    int32_t afc;            /* channel_t.afc */
} abo_channel_cfg;

typedef struct abo_device_cfg {
    int32_t sfmt;          /* input_t.sfmt */
    float fullscale;       /* input_t.fullscale (S16/F32 only) */
    int32_t sample_rate;   /* input_t.sample_rate */
    int32_t n_channels;    /* device_t.channel_count */
    const abo_channel_cfg* channels;
} abo_device_cfg;

typedef struct abo_config {
    int32_t fft_size;   /* global fft_size, 256..8192 */
    int32_t wave_rate;  /* WAVE_RATE: 8000, or 16000 for an NFM build (reference src/rtl_airband.h:65-71) */
    int32_t fm_demod;   /* global fm_demod */
    int32_t n_devices;
    const abo_device_cfg* devices;
} abo_config;

typedef struct abo_squelch_stats {
    float noise_level, signal_level, squelch_level; /* Squelch getters, reference src/squelch.h:89-91 */
    uint64_t open_count, flappy_count, ctcss_count, no_ctcss_count;
    float agcavgfast; /* freq_t.agcavgfast */
    uint32_t dm_phi;  /* channel_t.dm_phi */
    int32_t bin;      /* current dev->bins[i] (AFC may have moved it) */
    uint64_t active_counter;
    float noise_level_dbfs, signal_level_dbfs, squelch_level_dbfs; /* level_to_dBFS(), reference src/util.cpp:169-180 */
} abo_squelch_stats;

void* abo_create(const abo_config* cfg);
void abo_destroy(void* h);
int abo_wave_batch(void* h); /* WAVE_BATCH = wave_rate / 8 */
/* append raw ring-format bytes for one device */
int abo_push(void* h, int dev, const void* iq, size_t nbytes);
/* run every device until it lacks input or has produced max_batches more batches (max_batches < 0: no cap);
 * n_threads > 1 splits the device range across threads like multiple_demod_threads.  Returns batches produced. */
long abo_run(void* h, int max_batches, int n_threads);
void abo_set_discard(void* h, int discard); /* 1: do not queue outputs (timing runs) */
void abo_set_pin(void* h, const int* cpus, int n); /* timing runs: worker thread t of abo_run is pinned to cpus[t % n] */
int abo_batches_ready(void* h, int dev);
/* pop the oldest finished batch of a device: waveout[C*B], iq_out[C*2*B] (may be NULL), axc[C]; 1 if popped */
int abo_fetch_batch(void* h, int dev, float* waveout, float* iq_out, char* axc);
int abo_get_stats(void* h, int dev, int chan, abo_squelch_stats* out);
int abo_set_bin(void* h, int dev, int chan, int bin);
/* scan mode (rtl_airband.h:250-252, rtl_airband.cpp:101-139,498): install a frequency list for a channel (entry 0
 * current, all entries fresh); select the entry the next batch uses */
int abo_scan_configure(void* h, int dev, int chan, int n_freqs, const abo_channel_cfg* freqs);
int abo_scan_select(void* h, int dev, int chan, int freq_idx);
/* the stage boundaries, for tests: window[N]; one frame converted+windowed (2N floats) and its spectrum (2N) */
int abo_get_window(void* h, float* window);
int abo_debug_frame(void* h, int dev, const void* iq_frame, float* fftin, float* fftout);
/* |X[bin]| values straight into the per-sample channel loop (K1 / FFT skipped): wavein[C][n_batches * WAVE_BATCH], and the
 * X[bin] values of the same frames iq_in[C][n_batches * WAVE_BATCH][2] (may be NULL: then no channel may need raw I/Q) */
int abo_debug_inject_wavein(void* h, int dev, int n_batches, const float* wavein, const float* iq_in);

/* ---- host-side config formulas (reference src/config.cpp, src/util.cpp) ------------------------------- */
int32_t abo_calc_bin(int32_t freq, int32_t centerfreq, int32_t sample_rate, int32_t fft_size); /* config.cpp:666-667 */
uint32_t abo_calc_dm_dphi(int32_t freq, int32_t centerfreq, int32_t sample_rate, int32_t wave_rate); /* :679-712 */
float abo_dbfs_to_level(float dbfs, int32_t fft_size); /* util.cpp:169-176 */
float abo_level_to_dbfs(float level, int32_t fft_size); /* util.cpp:178-180 */
float abo_default_alpha(int32_t wave_rate);            /* rtl_airband.cpp:87 */
void abo_sincosf_lut(uint32_t phi, float* s, float* c); /* util.cpp:103-127 */
float abo_fast_atan2(float y, float x);                 /* rtl_airband.cpp:147-166 */
float abo_polar_disc_fast(float ar, float aj, float br, float bj);
float abo_fm_quadri_demod(float ar, float aj, float br, float bj);
void abo_fft(int n, const float* in, float* out);
double abo_fft_seconds(int n, int reps); /* seconds per n-point transform, persistent plan (CPU baseline self-description) */

/* ---- per-sample leaf harness (ports of reference src/test_squelch.cpp / test_ctcss.cpp use these) ------ */
void* abo_sq_new(void);
void abo_sq_free(void* s);
void abo_sq_set_level(void* s, float level);
void abo_sq_set_snr(void* s, float db);
void abo_sq_set_ctcss(void* s, float freq, float sample_rate);
void abo_sq_raw(void* s, float v);
void abo_sq_filtered(void* s, float v);
void abo_sq_audio(void* s, float v);
int abo_sq_is_open(void* s);
int abo_sq_should_filter(void* s);
int abo_sq_should_process_audio(void* s);
int abo_sq_first_open(void* s);
int abo_sq_last_open(void* s);
int abo_sq_outside_filter(void* s);
float abo_sq_noise_level(void* s);
float abo_sq_signal_level(void* s);
float abo_sq_squelch_level(void* s);
uint64_t abo_sq_open_count(void* s);
uint64_t abo_sq_flappy_count(void* s);
uint64_t abo_sq_ctcss_count(void* s);
uint64_t abo_sq_no_ctcss_count(void* s);
/* drive n samples exactly like the demod loop does (raw -> [filtered] -> [audio]) and record a trace:
 * levels[4*i..] = noise, signal, squelch level, 0 ; flags[i] bit0 open,1 filter,2 audio,3 first,4 last,5 outside */
void abo_sq_trace(void* s, int n, const float* raw, const float* filtered, const float* audio, float* levels, int32_t* flags);

void* abo_ctcss_new(float freq, float sample_rate, int window);
void abo_ctcss_free(void* c);
void abo_ctcss_sample(void* c, float v);
int abo_ctcss_enabled(void* c);
int abo_ctcss_enough(void* c);
int abo_ctcss_has_tone(void* c);
void abo_ctcss_reset(void* c);
uint64_t abo_ctcss_found(void* c);
uint64_t abo_ctcss_not_found(void* c);

void abo_notch_run(float freq, float sample_rate, float q, int n, float* inout);
void abo_lowpass_run(float freq, float sample_rate, int n, float* inout_iq);

const char* abo_variant(void); /* "restated" or "reference-leaf" */

#ifdef __cplusplus
}
#endif
#endif
