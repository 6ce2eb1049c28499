// Internal layouts shared by the host engine and the two sm_90a kernels.
//
// Data layout in HBM (per engine = one GPU's share of devices[]):
//   raw[d]            ring-format bytes of device d, linear, frames overlap in place (never expanded to float in HBM)
//   win[P][Gp]        |X[bin]| per (frame position, channel)  — channel_t.wavein, time-major so that the K2 warp
//   iqin[P][Gp]       X[bin]                                     (32 channels) reads one 128/256-byte line per sample
//   wout[Gp][P]       channel_t.waveout, channel-major (what the output thread consumes, contiguous per channel)
//   iqout[Gp][nb*B]   channel_t.iq_out
//   state[Gp]         per-channel scalars (Squelch, filters, AGC, NFM) — ChanState
//   sqbuf[102][Gp]    Squelch::buffer_ delay line
//   tone_*[2][NT][Gp] Goertzel banks of the fast / slow CTCSS detectors
// P = AGC_EXTRA + max_batches_per_run * WAVE_BATCH positions; position j of a run is exactly index j of the
// reference's wavein[]/waveout[] arrays when max_batches_per_run == 1.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/airband_b200.h"

#include <mutex>

// Kernel function attributes (dynamic shared-memory opt-in, carveout) are per CUDA device: several engines may live on
// different GPUs of one process and several demod threads may launch concurrently.  One slot per device ordinal keeps the
// largest size configured so far for a kernel instantiation; `apply` runs (under the lock) only when it has to grow.
struct AbgPerDeviceSize {
    std::mutex m;
    size_t v[64] = {};
    template <class F>
    cudaError_t ensure(size_t want, F&& apply) {
        int dev = 0;
        cudaGetDevice(&dev);
        dev &= 63;
        std::lock_guard<std::mutex> lock(m);
        if (want > v[dev]) {
            cudaError_t e = apply();
            if (e != cudaSuccess) return e;
            v[dev] = want;
        }
        return cudaSuccess;
    }
};

#define ABG_AGC_EXTRA 100     // reference src/rtl_airband.h:74
#define ABG_SQ_BUF 102        // Squelch::buffer_size_, reference src/squelch.cpp:67
#define ABG_MAX_TONES 52      // wanted tone + 51 standard tones, reference src/ctcss.cpp:89-111

// Squelch::State, reference src/squelch.h:104-110
enum { SQ_CLOSED = 0, SQ_OPENING = 1, SQ_CLOSING = 2, SQ_LOW_SIGNAL_ABORT = 3, SQ_OPEN = 4 };

// Per-channel constants, resolved on the host at abg_create() (reference config.cpp / filters.cpp / squelch.cpp ctor maths).
struct ChanParams {
    int32_t dev;            // owning device index (engine-local)
    int32_t modulation;     // ABG_MOD_*
    int32_t needs_raw_iq, has_iq_outputs;
    uint32_t dm_dphi;
    float alpha, ampfactor;
    int32_t afc;
    // NotchFilter (filters.cpp:30-47)
    int32_t notch_on;
    float nd0, nd1, nd2;
    // LowpassFilter (filters.cpp:67-96)
    int32_t lp_on;
    float lp_gain, lp_yc0, lp_yc1;
    // CTCSS (ctcss.cpp:92-111, squelch.cpp:110-116)
    int32_t ctcss_on;
    int32_t n_tones[2];     // detectors in the fast / slow bank (bank entry 0 is the wanted tone)
    int32_t window[2];      // window sizes: wave_rate*0.05, wave_rate*0.4
};

// Per-channel mutable state: Squelch (squelch.h:117-158), filters' delay elements, freq_t / channel_t scalars.
struct ChanState {
    // --- Squelch ---
    float noise_floor;
    int32_t manual;
    float manual_level, normal_ratio, flappy_ratio, avg_cap;
    float pre_full, pre_capped, post_full, post_capped;
    float level_cache;
    int32_t using_post;
    int32_t next_state, cur_state, delay;
    uint32_t sample_count_mod16;     // only sample_count_ % 16 is ever observed (squelch.cpp:213)
    int32_t low_signal_count;
    uint32_t recent_open_count, closed_sample_count;
    int32_t head;                    // buffer_head_; buffer_tail_ == (head + 1) % 102 always (squelch.cpp:69,457-458)
    unsigned long long open_count, flappy_count;
    // --- CTCSS fast [0] / slow [1] (ctcss.h:78-95) ---
    int32_t ct_enough[2], ct_count[2], ct_has_tone[2];
    unsigned long long ct_found[2], ct_not_found[2];
    // --- NotchFilter x[1],x[2],y[1],y[2] (filters.cpp:49-64) ---
    float nx1, nx2, ny1, ny2;
    // --- LowpassFilter xv[1],xv[2],yv[1],yv[2] (filters.cpp:146-163) ---
    float lx1r, lx1i, lx2r, lx2i, ly1r, ly1i, ly2r, ly2i;
    // --- freq_t / channel_t ---
    float agcavgfast;
    uint32_t dm_phi;
    float pr, pj, prev_waveout;
    unsigned long long active_counter;
    int32_t axc_prev;                // axcindicate of the previous batch (AFC edge detect, rtl_airband.cpp:222)
};

// Per-device, per-launch arguments of K1 (uploaded before every run).
struct K1Dev {
    const unsigned char* raw;  // base of the device's raw byte buffer (16-byte aligned)
    unsigned long long start_byte;  // byte offset of this launch's first frame
    int32_t n_frames;          // frames this launch computes for the device
    int32_t pos0;              // position (row of win/iqin) of the first frame
    int32_t g0, n_channels;    // channel index range [g0, g0 + n_channels)
    int32_t hop_bytes;         // bytes between consecutive frames (bps in the reference, rtl_airband.cpp:394)
    int32_t sfmt;
    float2* spec;              // when non-null: full spectrum of the last frame of every batch goes here (AFC)
    int32_t spec_first_pos;    // position of the first batch-final frame; then every WAVE_BATCH positions
    int32_t wave_batch;
};

// Per-device, per-launch arguments of K2.
struct K2Dev {
    int32_t n_batches;         // batches this launch demodulates for the device (0 = skip)
    int32_t fft_size;
    const float2* spec;        // spectra of batch-final frames [n_batches][fft_size] (AFC) or null
};

// ---- kernel launchers (defined in k1_fft.cu / k2_demod.cu) -------------------------------------------------------
struct K1Launch {
    int fft_size;
    int n_devices;             // grid.y
    int max_frames;            // max n_frames over devices
    int frames_per_tile;
    int tile_bytes_cap;        // dynamic smem reserved for the raw tile
    const K1Dev* devs;         // device memory
    const int32_t* bins;       // [Gp] current bin per channel
    const float* window_scaled;// [N] window * (1/fullscale-type factor) per sample format -> see engine
    const float2* tw1;         // inter-pass twiddles, layout [k1][n2]
    const float2* tw2;         // second inter-pass table for 3-pass sizes (N = 8192) or null
    float* win;                // [P][Gp]
    float2* iqin;              // [P][Gp]
    int Gp;
    int sfmt;                  // all devices of one launch share a format (the engine groups launches by format)
};
cudaError_t abg_launch_k1(const K1Launch& L, cudaStream_t s);
int abg_k1_tile_frames(int fft_size, int sfmt, int hop_bytes, int* tile_bytes_cap);
// output-pruned variant (k1_pruned.cu): only the configured bins are evaluated in the last pass
cudaError_t abg_launch_k1_pruned(const K1Launch& L, const float2* twn, int max_channels, cudaStream_t s);
int abg_k1p_tile_frames(int fft_size, int sfmt, int hop_bytes, int max_channels, int* tile_bytes_cap);

// tensor-core variant (k1_tc.cu): the bins' DFT as an integer GEMM on wgmma (8-bit formats, hop_bytes % 32 == 0)
struct K1TcPlan {  // a ring stage = pps column pairs of a tile (or part of one pair's k-steps); KBS: k-steps per pair and stage at most; NSTB: stages
    int eligible;
    int K, HC, S, NC, ND, C2p, KBS, NSTB, acc_regs, smem_bytes, halo, consumer_warpgroups;
    int pps;
    size_t table_bytes;
};
struct K1TcTables {
    const int32_t* tab_of_dev;  // [n_devices of the group] coefficient table of each device
    const signed char* btab;    // [n_tables][K * NC]
    const long long* sq;        // [n_tables][C2p]
    int* counter;               // tile queue head, zero at launch
    int32_t* status;            // != 0 after a pipeline stall inside the kernel (bounded waits, never hangs)
    double cscale;
};
int abg_k1tc_plan(int fft_size, int sfmt, int hop_bytes, int max_channels, int digits, K1TcPlan* p);
void abg_k1tc_build_table(const K1TcPlan& p, int fft_size, int sfmt, const float* wsc, const int32_t* bins, int n_channels, signed char* tab,
                          long long* sq, double* cscale);
cudaError_t abg_launch_k1_tc(const K1Launch& L, const K1TcPlan& p, const K1TcTables& T, int sm_count, cudaStream_t s);
int abg_k1tc_trace_dump(long long* out);  // measurement aid (ABG_K1_TC_TRACE): 256*4*16*4 clock64 stamps

// band spectrum monitor (spectrum.cu): see abg_spectrum_configure in include/airband_b200.h
#define ABG_SPEC_FPC 32  // selected frames per chunk (work item) of one batch
struct SpecCfg {  // per monitored device; written by abg_spectrum_configure
    const float* wsc;       // the device's K1 window table (window * 1/full-scale)
    float* partial;         // [max_batches_per_run][n_chunks][N] chunk sums
    int32_t* counter;       // [max_batches_per_run] chunks finished per batch; zero between launches
    float* ring;            // device view of the page-locked result ring [ring_cap][N]
    int32_t hop_bytes, sfmt, stride, n_sel, n_chunks, ring_cap;
};
struct SpecRun {  // per monitored device; uploaded with every run
    const unsigned char* raw;
    unsigned long long first_byte;  // first byte of frame j = 0 of the run's first batch
    int32_t n_batches;              // batches of this run (0 = none)
    int32_t ring_pos0;              // ring entry of the run's first batch; < 0: resident run, the ring is left alone
};
struct SpecArgs {
    const SpecCfg* cfg;  // [monitored devices]
    const SpecRun* run;
    const float2* tw1;
    const float2* tw2;
    int wave_batch;
};
cudaError_t abg_launch_spectrum(int fft_size, const SpecArgs& a, int n_devices, int max_items, cudaStream_t s);

// carrier frequency meter (carrier.cu): see abg_carrier_configure in include/airband_b200.h
struct CarCfg {  // per metered device; written by abg_carrier_configure
    float* ring;         // device view of the page-locked result ring [ring_cap][3 * n_channels]: lag1 re/im pairs, then energies
    int32_t g0, n_channels, ring_cap;
};
struct CarRun {  // per metered device; uploaded with every run
    int32_t n_batches;  // batches of this run (0 = none)
    int32_t ring_pos0;  // ring entry of the run's first batch; < 0: resident run, the ring is left alone
};
struct CarArgs {
    const CarCfg* cfg;  // [metered devices]
    const CarRun* run;
    const float2* iqin;  // [P][Gp] the run's K1 output
    int Gp, wave_batch;
};
cudaError_t abg_launch_carrier(const CarArgs& a, int n_devices, int max_items, cudaStream_t s);
int abg_carrier_items(int n_channels);  // work items per batch of a device

// input level meter (input_meter.cu): see abg_input_meter_configure in include/airband_b200.h
struct InmCfg {  // per metered device; written by abg_input_meter_configure
    unsigned char* ring;   // device view of the page-locked result ring [ring_cap] of abg_input_levels
    uint32_t* hist;        // [max_batches_per_run][2][256] histogram of each batch of the run; zero between launches
    int32_t* counter;      // [max_batches_per_run] chunks finished per batch; zero between launches
    long long* partial;    // [max_batches_per_run][n_chunks][ABG_INM_PARTIAL] chunk sums (int64, or double for F32)
    int32_t sfmt, hop_bytes, n_chunks, ring_cap;
    float scale;           // 1.0f / fullscale (S16, F32)
};
#define ABG_INM_PARTIAL 6  // per chunk: sum[2], sum_sq[2], sum_iq, then peak[2] as two float bit patterns
struct InmRun {  // per metered device; uploaded with every run
    const unsigned char* raw;
    unsigned long long first_byte;  // first byte of the run's first batch
    int32_t n_batches;              // batches of this run (0 = none)
    int32_t ring_pos0;              // ring entry of the run's first batch; < 0: resident run, the ring is left alone
};
struct InmArgs {
    const InmCfg* cfg;  // [metered devices]
    const InmRun* run;
    int wave_batch;
};
cudaError_t abg_launch_input_meter(const InmArgs& a, int n_devices, int max_items, cudaStream_t s);
int abg_input_meter_chunks(int batch_bytes);  // work items per batch of a device

// sub-band I/Q outputs (subband.cu): see abg_subband_configure in include/airband_b200.h
struct SbOut {  // one switched-on output
    const float2* coef;      // [n_coeffs] h[j] * exp(+2 pi i delta j / 2^32), built in double, stored as float32
    unsigned char* ring;     // device view of the page-locked result ring [ring_cap][entry_bytes]
    uint32_t delta;          // phase step per sample, 2^-32 turns
    int32_t decim, n_coeffs, ring_cap, entry_bytes;
};
struct SbCfg {  // per device with an output on; written by abg_subband_configure
    SbOut out[ABG_SUBBAND_MAX];
    int32_t n_out, sfmt, bpc, batch_samples, n_chunks;
    int32_t hist;            // L_max - 1: history samples staged before each chunk
    float scale;             // 1.0f / fullscale (S16, F32)
};
struct SbRun {  // per device with an output on; uploaded with every run
    const unsigned char* raw;
    long long base;          // absolute sample index of raw[0]; samples below it read as zero
    long long s0;            // absolute sample index of the run's first batch
    int32_t n_batches;       // batches of this run (0 = none)
    int32_t ring_pos0[ABG_SUBBAND_MAX];  // ring entry of the run's first batch per output; < 0: resident run, no output
    int32_t lead[ABG_SUBBAND_MAX];       // s0 - (first input sample of the output), at most 2^30: earlier samples are zero
};
struct SbArgs {
    const SbCfg* cfg;  // [devices with an output on]
    const SbRun* run;
};
cudaError_t abg_launch_subband(const SbArgs& a, int n_devices, int max_items, int max_hist, cudaStream_t s);
int abg_subband_chunks(int batch_samples);  // work items per batch of a device

// CTCSS tone meter (tone_meter.cu): see abg_tone_meter_configure in include/airband_b200.h
#define ABG_TM_COLS 64  // tone-table columns per tile: 32 tones, cos and -sin interleaved
struct TmCfg {  // per metered device; written by abg_tone_meter_configure
    float* ring;       // device view of the page-locked result ring [ring_cap][n_channels * (2 * ABG_TONE_MAX + 2)] floats
    int32_t g0, n_channels;
    int32_t first;     // index of the device's channel 0 in the metered channel list
    int32_t ring_cap;
};
struct TmRun {  // per metered device; uploaded with every run
    unsigned long long seq0;  // audio batch number of the run's first batch
    int32_t n_batches;        // batches of this run (0 = none)
    int32_t ring_pos0;        // ring entry of the run's first batch; < 0: resident run, the ring is left alone
};
struct TmArgs {
    const TmCfg* cfg;         // [metered devices]
    const TmRun* run;
    const int32_t* chan_dev;  // [n_chan] metered channel -> index into cfg / run
    const float* table;       // [wave_batch][n_cols]: cos, -sin of (delta_k * j mod 2^32) 2 pi / 2^32, zero columns past 2K
    const float* wout;        // [Gp][P] the run's audio, batch b of channel g at g * P + b * wave_batch
    int P, wave_batch, K, n_cols, n_chan;
    uint32_t delta[ABG_TONE_MAX];
};
cudaError_t abg_launch_tone_meter(const TmArgs& a, int max_batches, cudaStream_t s);

// band activity detector (activity.cu): see abg_activity_configure in include/airband_b200.h
#define ABG_ACT_HEAD_BYTES 16  // ring entry head: int32 {n_total, stride, hang, min_span}, then abg_burst[ABG_ACTIVITY_MAX_RECORDS]
struct ActCfg {  // per device with the detector on; written by abg_activity_configure
    const float* wsc;        // the device's K1 window table (window * 1/full-scale)
    const float* thr;        // [N] per-bin thresholds
    unsigned char* ring;     // device view of the page-locked result ring [ring_cap][entry_bytes]
    int32_t hop_bytes, sfmt, stride, n_sel, hang, min_span, ring_cap, entry_bytes;
};
struct ActRun {  // per device with the detector on; uploaded with every run
    const unsigned char* raw;
    unsigned long long first_byte;   // first byte of frame j = 0 of the run's first batch
    unsigned long long first_frame;  // absolute frame number of that frame: AGC_EXTRA + batch_seq * wave_batch
    int32_t n_batches;               // batches of this run (0 = none)
    int32_t ring_pos0;               // ring entry of the run's first batch; < 0: resident run, the ring is left alone
};
struct ActArgs {
    const ActCfg* cfg;  // [devices with the detector on]
    const ActRun* run;
    const float2* tw1;
    const float2* tw2;
    int wave_batch;
};
cudaError_t abg_launch_activity(int fft_size, const ActArgs& a, int n_devices, int max_batches, cudaStream_t s);

// I/Q history (history.cu): see abg_history_configure in include/airband_b200.h
struct HiCfg {  // per device with the history on; written by abg_history_configure
    unsigned char* ring;             // device [ring_bytes]: stream byte b at b mod ring_bytes
    unsigned long long ring_bytes;   // a multiple of 16
};
struct HiRun {  // per device with the history on; uploaded with every run
    const unsigned char* src;        // first byte this run appends (its address agrees with dst modulo 16)
    unsigned long long dst;          // ring byte of src[0], < ring_bytes
    unsigned long long n_bytes;      // bytes this run appends, at most ring_bytes (0 = none)
};
struct HiArgs {
    const HiCfg* cfg;  // [devices with the history on]
    const HiRun* run;
};
cudaError_t abg_launch_history_append(const HiArgs& a, int n_devices, int blocks_per_device, cudaStream_t s);
int abg_history_blocks(unsigned long long max_bytes, int n_devices, int sm_count);  // append CTAs per device
struct HiCapture {  // one capture launch: outputs [m0, m0 + n_out) of one device's history
    const unsigned char* ring;
    unsigned long long ring_bytes;
    const float2* coef;      // [n_coeffs] g[j], as the sub-band outputs build them
    float2* out;             // device [n_out]
    long long m0;
    int32_t n_out, decim, n_coeffs, sfmt;
    uint32_t delta;
    float scale;             // 1.0f / fullscale (S16, F32)
    int32_t per_item, stage; // set by the launcher
};
cudaError_t abg_launch_history_capture(HiCapture c, cudaStream_t s);

// transmission profiles (profile.cu): see abg_history_profile in include/airband_b200.h
#define ABG_PROFILE_SUMS 8  // p1, p2, a1, z.re, z.im, f1, f2, 0; then tone_fm[K][2], tone_am[K][2]
struct ProfBlock {  // one CTA: every device read it makes is bounded by its own fields
    unsigned long long off;  // scratch index of y[m]
    unsigned long long res;  // result index (floats) of its ABG_PROFILE_SUMS + 4 K sums
    long long m;             // absolute output index of its first output
    int32_t n;               // outputs, 1 .. ABG_PROFILE_BLOCK
    int32_t succ;            // 1: y[m + n] is captured at off + n, so the pair of its last output is formed
    int32_t tones;           // index of its delta_0 in the delta table
    int32_t K;               // tones, 1 .. ABG_TONE_MAX
};
struct ProfArgs {
    const float2* y;         // the chunk's captured outputs
    const ProfBlock* blocks;   // [n_blocks]
    const uint32_t* delta;   // the chunk's tone phases
    float* res;              // block sums
};
cudaError_t abg_launch_profile(const ProfArgs& a, int n_blocks, cudaStream_t s);

// history replay (replay.cu): see abg_history_replay in include/airband_b200.h
struct RpGather {  // one job's bytes of one chunk
    const unsigned char* ring;       // the parent device's history ring: stream byte b at b mod ring_bytes
    unsigned long long ring_bytes;   // a multiple of 16
    unsigned long long src;          // stream byte of dst[0]
    unsigned char* dst;              // raw[cur] + fill of the job's device in the replay engine, any alignment
    unsigned long long n_bytes;      // 0 = none
};
cudaError_t abg_launch_replay_gather(const RpGather* jobs, int n_jobs, int blocks_per_job, cudaStream_t s);

struct K2Launch {
    int G, Gp, P, wave_batch, fm_demod, iq_stride;  // iq_stride = nbmax * B
    int lanes_per_warp;       // channels handled by one warp of K2: 1, 2, 4, 8, 16 or 32
    int nfm_blocks;           // some channel (or scan-list entry) is NFM: run the kernel build with the NFM steady-state blocks
    const ChanParams* params;
    ChanState* state;
    const K2Dev* devs;
    int32_t* bins;
    const int32_t* base_bins;
    float* win;               // [P][Gp] buffer K1 filled for THIS run
    float2* iqin;
    float* win_next;          // buffer the next run's K1 fills: receives the AGC_EXTRA look-back rows
    float2* iqin_next;
    float* wout;
    float2* iqout;            // may be null when no channel has I/Q outputs
    float* sqbuf;             // [102][Gp]
    const float* tone_coeff;  // [2][NT][Gp]
    float* tone_q1;           // [2][NT][Gp]
    float* tone_q2;
    float* tone_mag;
    unsigned char* axc;       // [nbmax][Gp]
    const float* sincos_lut;  // [2][257] sin then cos (util.cpp:103-111)
};
cudaError_t abg_launch_k2(const K2Launch& L, cudaStream_t s);
int abg_k2_stats_dump(unsigned long long* out);  // event counters of the ABG_K2_STATS build (k2_demod.cu)

// mixer sums (reference src/mixer.cpp:133-140,189-214), defined in k2_demod.cu (compiled without FMA contraction)
struct MixInput {
    int32_t g;          // global channel index of the input
    int32_t dev;
    float mult_l, mult_r;  // ampfactor * ampl, ampfactor * ampr
};
struct MixLaunch {
    int n_mixers, n_batches, wave_batch, P, Gp;
    const int32_t* offsets;   // [n_mixers + 1]
    const MixInput* inputs;
    const K2Dev* devs;
    const float* wout;        // [Gp][P]
    const unsigned char* axc; // [nbmax][Gp]
    float* sums;              // [nbmax][n_mixers][2][B]
    int32_t* flags;           // [nbmax][n_mixers]
    float* host_sums;         // same layout in the pinned result slot, or null
    int32_t* host_flags;
};
cudaError_t abg_launch_mix(const MixLaunch& L, cudaStream_t s);
// host-visible (pinned, mapped) result slot the end-of-run kernel writes; all null = no export (resident benchmark runs)
struct K2Export {
    float* host_wout;          // [G][stride]
    float2* host_iqout;        // [G][stride] or null
    unsigned char* host_axc;   // [nbmax][Gp]
    size_t stride;             // nbmax * WAVE_BATCH
};
cudaError_t abg_launch_k2_tail(const K2Launch& L, const K2Export& X, cudaStream_t s);
