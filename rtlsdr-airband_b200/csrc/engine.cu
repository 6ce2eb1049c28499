// Host side of the demodulation engine: configuration -> device tables and per-channel state, raw-sample
// ingest, run scheduling (K1 then K2 per run), result queueing, and the C ABI declared in include/airband_b200.h.
//
// Config-time arithmetic restated here (host, double/float exactly as the reference does it):
//   window                      reference src/rtl_airband.cpp:335-351
//   sincos LUT                  reference src/util.cpp:103-111
//   Squelch constructor/setters reference src/squelch.cpp:36-116
//   Goertzel coefficients, bank reference src/ctcss.cpp:31-42,62-73,92-111
//   NotchFilter coefficients    reference src/filters.cpp:30-47
//   LowpassFilter design        reference src/filters.cpp:67-144
//   initial channel state       reference src/config.cpp:265-281,313-331
// There is no CPU execution path: every entry point needs a CUDA device.
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <complex>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/airband_b200.h"
#include "abg_internal.h"

namespace {

// Small host->device parameter uploads go through a KERNEL (payload passed by value), not cudaMemcpyAsync: a copy would
// queue on the host->device copy engine behind whatever bulk ingest copies (abg_push of the NEXT run) are already
// enqueued, and the run that needs these few hundred bytes would wait for megabytes of unrelated input.  A launch is
// ordered only by its own stream.
struct UploadBlob {
    uint4 q[240];  // 3840 bytes: stays below the 4 KB kernel-parameter limit together with the other arguments
};
__global__ void upload_kernel(const UploadBlob b, uint4* dst, int n16) {
    const int i = threadIdx.x;
    if (i < n16) dst[i] = b.q[i];
}
// dst: 16-byte aligned device buffer with room for nbytes rounded up to 16; returns the number of launches (or -1)
int upload_small(void* dst, const void* src, size_t nbytes, cudaStream_t s) {
    int launches = 0;
    for (size_t off = 0; off < nbytes; off += sizeof(UploadBlob)) {
        const size_t chunk = std::min(sizeof(UploadBlob), nbytes - off);
        UploadBlob b;
        memcpy(b.q, static_cast<const char*>(src) + off, chunk);
        if (chunk % 16) memset(reinterpret_cast<char*>(b.q) + chunk, 0, 16 - chunk % 16);
        const int n16 = (int)((chunk + 15) / 16);
        upload_kernel<<<1, 256, 0, s>>>(b, reinterpret_cast<uint4*>(static_cast<char*>(dst) + off), n16);
        if (cudaGetLastError() != cudaSuccess) return -1;
        ++launches;
    }
    return launches;
}

thread_local std::string g_err;
int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}
#define CU(call)                                                                                              \
    do {                                                                                                      \
        cudaError_t _e = (call);                                                                              \
        if (_e != cudaSuccess) return fail(ABG_ECUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

const float kStandardTones[51] = {67.0,  69.3,  71.9,  74.4,  77.0,  79.7,  82.5,  85.4,  88.5,  91.5,  94.8,  97.4,  100.0,
                                  103.5, 107.2, 110.9, 114.8, 118.8, 123.0, 127.3, 131.8, 136.5, 141.3, 146.2, 150.0, 151.4,
                                  156.7, 159.8, 162.2, 165.5, 167.9, 171.3, 173.8, 177.3, 179.9, 183.5, 186.2, 189.9, 192.8,
                                  196.6, 199.5, 203.5, 206.5, 210.7, 218.1, 225.7, 229.1, 233.6, 241.8, 250.3, 254.1};  // ctcss.cpp:87-89

// Goertzel coefficient of one detector, ctcss.cpp:31-42 (same operand types: int*float/float, +0.5 in double, float omega)
float goertzel_coeff(float tone_freq, float sample_rate, int window_size) {
    int k = (0.5 + window_size * tone_freq / sample_rate);
    float omega = (2.0 * M_PI * k) / window_size;
    float coeff = 2.0 * cos(omega);
    return coeff;
}
// bank for one CTCSS object: wanted tone first, then standard tones not within 5 Hz, dropping coefficient collisions
std::vector<float> tone_bank(float ctcss_freq, float sample_rate, int window_size) {
    std::vector<float> coeffs;
    auto try_add = [&](float f) {
        float c = goertzel_coeff(f, sample_rate, window_size);
        for (float e : coeffs)
            if (e == c) return;
        coeffs.push_back(c);
    };
    try_add(ctcss_freq);
    for (float tone : kStandardTones) {
        if (std::abs(ctcss_freq - tone) < 5) continue;
        try_add(tone);
    }
    return coeffs;
}

// LowpassFilter::LowpassFilter, filters.cpp:67-96 (+ blt/expand/multin/eval :98-144)
typedef std::complex<double> cd;
cd lp_blt(cd pz) { return (2.0 + pz) / (2.0 - pz); }
void lp_multin(cd w, int npz, cd coeffs[]) {
    cd nw = -w;
    for (int i = npz; i >= 1; i--) coeffs[i] = (nw * coeffs[i]) + coeffs[i - 1];
    coeffs[0] = nw * coeffs[0];
}
bool lp_expand(cd pz[], int npz, cd coeffs[]) {
    coeffs[0] = 1.0;
    for (int i = 0; i < npz; i++) coeffs[i + 1] = 0.0;
    for (int i = 0; i < npz; i++) lp_multin(pz[i], npz, coeffs);
    for (int i = 0; i < npz + 1; i++)
        if (fabs(coeffs[i].imag()) > 1e-10) return false;
    return true;
}
cd lp_eval(cd coeffs[], int npz, cd z) {
    cd sum(0.0);
    for (int i = npz; i >= 0; i--) sum = (sum * z) + coeffs[i];
    return sum;
}
bool lowpass_design(float freq, float sample_freq, float* gain, float* yc0, float* yc1) {
    double raw_alpha = (double)freq / sample_freq;
    double warped_alpha = tan(M_PI * raw_alpha) / M_PI;
    cd zeros[2] = {-1.0, -1.0};
    cd poles[2];
    poles[0] = lp_blt(M_PI * 2 * warped_alpha * cd(-1.10160133059e+00, 6.36009824757e-01));
    poles[1] = lp_blt(M_PI * 2 * warped_alpha * conj(cd(-1.10160133059e+00, 6.36009824757e-01)));
    cd top[3], bot[3];
    if (!lp_expand(zeros, 2, top) || !lp_expand(poles, 2, bot)) return false;
    cd g = lp_eval(top, 2, 1.0) / lp_eval(bot, 2, 1.0);
    *gain = hypot(g.imag(), g.real());
    *yc0 = -(bot[0].real() / bot[2].real());
    *yc1 = -(bot[1].real() / bot[2].real());
    return true;
}

struct Plan {
    int r1, r2, r3;
};
bool plan_for(int n, Plan* p) {  // must match Plan<LOGN> in k1_fft.cu
    switch (n) {
        case 256: *p = {16, 16, 0}; return true;
        case 512: *p = {32, 16, 0}; return true;
        case 1024: *p = {32, 32, 0}; return true;
        case 2048: *p = {64, 32, 0}; return true;
        case 4096: *p = {64, 64, 0}; return true;
        case 8192: *p = {32, 16, 16}; return true;
    }
    return false;
}

// Device memory.  A failed allocation leaves the buffer empty and clears the runtime's last error (an allocation error is
// not sticky), so that the next launch check does not report it.
template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    cudaError_t alloc(size_t count) {
        const cudaError_t er = cudaMalloc((void**)&p, std::max<size_t>(count, 1) * sizeof(T));
        if (er == cudaSuccess) {
            n = count;
        } else {
            cudaGetLastError();
            p = nullptr;
        }
        return er;
    }
    void free() {
        if (p) cudaFree(p);
        p = nullptr;
        n = 0;
    }
};

// Result queue of one device's batch monitor (band spectrum, carrier meter, input level meter, sub-band output, tone
// meter, activity detector).  The monitor's kernel writes the result of every batch straight into a page-locked, mapped ring of `cap` =
// max_batches_per_run + 2 entries; the host keeps the unfetched entries, oldest first.  Lossy by design: queueing a run
// drops the oldest unfetched entries beyond the ring's size (gaps show in their batch_seq), so a monitor never holds a
// result slot or causes ABG_EOVERFLOW.
struct MonitorQueue {
    struct Entry {
        int pos;      // ring entry
        int32_t aux;  // monitor-specific: frames averaged (spectrum), decimation (sub-band output), tones (tone meter), 0 otherwise
        uint64_t seq, run;
    };
    unsigned char* ring = nullptr;  // [cap][entry_bytes]; allocated when the monitor is first switched on, kept until abg_destroy
    size_t entry_bytes = 0;
    int cap = 0, next = 0;
    std::deque<Entry> ready;

    // Room for entries of entry_bytes_ for an engine of max_batches_per_run.  A larger entry than the ring has moves the
    // ring, entry by entry, so that what is queued survives (an entry size grows for sub-band outputs only); so do
    // entries queued before the monitor was switched off and on again.  false: out of page-locked memory, the old ring
    // is kept and the runtime's last error is cleared.
    bool reserve(int max_batches_per_run, size_t entry_bytes_) {
        if (ring && entry_bytes_ <= entry_bytes) return true;
        const int cap_ = max_batches_per_run + 2;
        unsigned char* grown = nullptr;
        if (cudaHostAlloc((void**)&grown, (size_t)cap_ * entry_bytes_, cudaHostAllocMapped) != cudaSuccess) {
            cudaGetLastError();
            return false;
        }
        if (ring) {
            for (int i = 0; i < cap; i++) memcpy(grown + (size_t)i * entry_bytes_, ring + (size_t)i * entry_bytes, entry_bytes);
            cudaFreeHost(ring);
        }
        ring = grown;
        cap = cap_;
        entry_bytes = entry_bytes_;
        return true;
    }
    void release() {
        if (ring) cudaFreeHost(ring);
        ring = nullptr;
    }
    // Queue the n batches of run `run` whose first is batch number seq0; returns the ring entry of the first.
    int queue(int n, uint64_t seq0, uint64_t run, int32_t aux) {
        const int pos0 = next;
        for (int b = 0; b < n; b++) ready.push_back({(next + b) % cap, aux, seq0 + (uint64_t)b, run});
        while ((int)ready.size() > cap) ready.pop_front();
        next = (next + n) % cap;
        return pos0;
    }
};

constexpr int TL_RUNS = 8;  // runs whose timing events are kept

// Host side of one batch monitor: its state per engine device, and its launch, one kernel per run that covers every
// device the monitor is on for.  The sequence around it is shared (monitor_dev, monitor_configure, monitor_publish,
// monitor_launch, monitor_time, monitor_fetch); DESIGN.md §4, "Engine plumbing", states its contract.  Dev is the
// monitor's own per-device state: on() tells whether the launch covers the device, release() frees what it holds.
template <typename Cfg, typename Run, typename Dev>
struct MonitorLaunch {
    const char* name;        // in error messages
    bool reads_raw;          // reads raw[] after K1: records ev_raw, which abg_push's compaction waits for
    bool after_k2;           // runs on stream B after K2 (it reads the audio), not on stream A after K1
    std::vector<Dev> dev;    // [engine devices]; nothing is allocated for a device until it is first switched on
    std::vector<int> devs;   // covered devices in launch order (grid.y of the kernel)
    DevBuf<Cfg> cfg;         // [devs.size()], written when a configure call changes the list
    DevBuf<Run> run;         // room for every device, uploaded with every run
    std::vector<Run> h_run;  // [devs.size()]
    cudaEvent_t tl[TL_RUNS][2] = {};  // kernel start / end of the last TL_RUNS runs
    bool ran[TL_RUNS] = {};

    MonitorLaunch(const char* name_, bool reads_raw_, bool after_k2_ = false) : name(name_), reads_raw(reads_raw_), after_k2(after_k2_) {}
    void release() {
        for (auto& d : dev) d.release();
        cfg.free();
        run.free();
        for (auto& row : tl)
            for (auto& ev : row)
                if (ev) cudaEventDestroy(ev);
    }
};

// band spectrum (abg_spectrum_configure)
struct SpecDev {
    int stride = 0, n_sel = 0, chunks = 0;
    DevBuf<unsigned char> work;  // chunk sums float[nbmax][chunks][N], then the batch counters int32[nbmax]
    MonitorQueue q;              // finished spectra float[N] per entry
    bool on() const { return stride > 0; }
    MonitorQueue& queue(int) { return q; }
    void release() { work.free(); q.release(); }
};
// carrier frequency meter (abg_carrier_configure)
struct CarDev {
    bool enabled = false;
    MonitorQueue q;  // lag1 float[C][2], then energy float[C] per entry
    bool on() const { return enabled; }
    MonitorQueue& queue(int) { return q; }
    void release() { q.release(); }
};
// input level meter (abg_input_meter_configure)
struct InmDev {
    bool enabled = false;
    int chunks = 0;
    DevBuf<unsigned char> work;  // histograms uint32[nbmax][2][256], counters int32[nbmax], chunk sums int64[nbmax][chunks][ABG_INM_PARTIAL]; kept once allocated
    MonitorQueue q;              // abg_input_levels per entry
    bool on() const { return enabled; }
    MonitorQueue& queue(int) { return q; }
    void release() { work.free(); q.release(); }
};
// sub-band I/Q outputs (abg_subband_configure)
struct SbDev {
    struct Output {
        bool on = false;
        bool restart = false;        // the next streamed run starts the output's input at its first batch
        int decim = 0, n_coeffs = 0;
        uint32_t delta = 0;
        long long start = 0;         // absolute sample index of the output's first input sample
        DevBuf<float2> coef;         // h[j] * exp(+2 pi i delta j / 2^32); kept once allocated
        MonitorQueue q;              // cf32 [ceil(n / decim)] per entry, Entry.aux = decim
    } out[ABG_SUBBAND_MAX];
    int hist = 0;                    // L_max - 1 over the outputs switched on: samples abg_push's compaction keeps before `consumed`
    bool on() const { return std::any_of(std::begin(out), std::end(out), [](const Output& o) { return o.on; }); }
    MonitorQueue& queue(int k) { return out[k].q; }
    void release() {
        for (auto& o : out) {
            o.coef.free();
            o.q.release();
        }
    }
};
struct SubbandLaunch : MonitorLaunch<SbCfg, SbRun, SbDev> {
    using MonitorLaunch::MonitorLaunch;
    int max_hist = 0;  // largest SbDev::hist of devs
};
// CTCSS tone meter (abg_tone_meter_configure)
struct TmDev {
    bool enabled = false;
    MonitorQueue q;  // S float[C][K][2], E float[C], active int32[C] per entry (room for ABG_TONE_MAX), Entry.aux = K
    bool on() const { return enabled; }
    MonitorQueue& queue(int) { return q; }
    void release() { q.release(); }
};
struct ToneMeterLaunch : MonitorLaunch<TmCfg, TmRun, TmDev> {
    using MonitorLaunch::MonitorLaunch;
    // the engine-wide tone list and, once the meter is first switched on, its [B][cols] table
    std::vector<float> freqs{std::begin(kStandardTones), std::end(kStandardTones)};
    std::vector<uint32_t> delta;
    DevBuf<float> table;
    int cols = 0;
    DevBuf<int32_t> chan_dev;  // metered channel -> index into devs
    int n_chan = 0;
    void release() {
        MonitorLaunch::release();
        table.free();
        chan_dev.free();
    }
};
// band activity detector (abg_activity_configure)
struct ActDev {
    int stride = 0, hang = 0, min_span = 0, n_sel = 0;
    DevBuf<float> thr;  // [N] thresholds; kept once allocated
    MonitorQueue q;     // head int32[4] {n_total, stride, hang, min_span}, then abg_burst[ABG_ACTIVITY_MAX_RECORDS]
    bool on() const { return stride > 0; }
    MonitorQueue& queue(int) { return q; }
    void release() { thr.free(); q.release(); }
};
// I/Q history (abg_history_configure); its ring is freed when it is switched off
struct HiDev {
    int batches = 0;                       // capacity in batches, 0 = off
    DevBuf<unsigned char> ring;            // stream byte b at b mod ring.n; ring.n = cap * bpc rounded up to a multiple of 16
    unsigned long long cap = 0;            // capacity in samples
    unsigned long long first = 0, end = 0;  // samples [first, end) the ring holds once every enqueued run has finished
    bool on() const { return ring.p != nullptr; }
    void release() { ring.free(); }
};
struct HistoryLaunch : MonitorLaunch<HiCfg, HiRun, HiDev> {
    using MonitorLaunch::MonitorLaunch;
    // captures: coefficient and output scratch (allocated by the first capture) and the last capture's kernel time
    DevBuf<float2> coef, out;
    cudaEvent_t ev[2] = {nullptr, nullptr};
    float capture_ms = 0.0f;
    void release() {
        MonitorLaunch::release();
        coef.free();
        out.free();
        for (auto& x : ev)
            if (x) cudaEventDestroy(x);
    }
};

struct Device {
    int sfmt = 0, bpc = 0, sample_rate = 0, hop = 0, hop_bytes = 0;
    float fullscale = 0;
    int g0 = 0, C = 0, group = 0;
    bool primed = false, has_afc = false;
    // raw sample stream (ping-pong linear buffers)
    unsigned char* raw[2] = {nullptr, nullptr};
    int cur = 0;
    size_t cap = 0, fill = 0, consumed = 0;
    int runs_since_compaction = 1;  // K1 launches that read raw[cur] since the last compaction
    // resident replay stream
    unsigned char* res = nullptr;
    size_t res_bytes = 0;
    bool res_primed = false;
    float2* spec = nullptr;  // [nbmax][N] when has_afc
    std::deque<std::pair<int, int>> ready;  // (slot, batch-in-run)
    uint64_t batch_seq = 0;  // batches of the pushed stream enqueued since abg_create
    uint64_t audio_seq = 0;  // batches queued for abg_fetch_batch since abg_create, pushed and injected
    size_t dropped = 0;      // stream bytes compaction has dropped: raw[cur][0] is byte `dropped` of the stream
};

// ---- scan mode: per-frequency freq_t sets (rtl_airband.h:223-233,250-252) ------------------------------------------------
// A scan channel keeps one FreqSet per freqlist[] entry in device memory.  The live slot (params/state/sqbuf/tone banks
// of channel g, what K2 reads) holds the current entry; abg_scan_select() swaps entries with one small kernel on the
// K2 stream, i.e. between the batches of two runs, which is when demodulate() re-reads freq_idx (rtl_airband.cpp:498).
struct FreqSet {
    ChanParams p;  // freq-level fields only: modulation, ampfactor, notch, low-pass, CTCSS
    ChanState s;   // freq-level fields only: Squelch, CTCSS counters, filter delay elements, agcavgfast, active_counter
    float sqbuf[ABG_SQ_BUF];
    float tone_coeff[2][ABG_MAX_TONES], tone_q1[2][ABG_MAX_TONES], tone_q2[2][ABG_MAX_TONES], tone_mag[2][ABG_MAX_TONES];
};
struct ScanView {
    ChanParams* params;
    ChanState* state;
    float *sqbuf, *tone_coeff, *tone_q1, *tone_q2, *tone_mag;
    int Gp;
};
__device__ void freq_fields_copy(ChanParams& dp, ChanState& ds, const ChanParams& sp, const ChanState& ss) {
    // channel_t members stay with the channel: dev, needs_raw_iq, has_iq_outputs, dm_dphi, alpha, afc / dm_phi, pr, pj,
    // prev_waveout, axc_prev
    dp.modulation = sp.modulation; dp.ampfactor = sp.ampfactor;
    dp.notch_on = sp.notch_on; dp.nd0 = sp.nd0; dp.nd1 = sp.nd1; dp.nd2 = sp.nd2;
    dp.lp_on = sp.lp_on; dp.lp_gain = sp.lp_gain; dp.lp_yc0 = sp.lp_yc0; dp.lp_yc1 = sp.lp_yc1;
    dp.ctcss_on = sp.ctcss_on;
    for (int w = 0; w < 2; w++) { dp.n_tones[w] = sp.n_tones[w]; dp.window[w] = sp.window[w]; }
    const uint32_t dm_phi = ds.dm_phi;
    const float pr = ds.pr, pj = ds.pj, prev_waveout = ds.prev_waveout;
    const int32_t axc_prev = ds.axc_prev;
    ds = ss;
    ds.dm_phi = dm_phi; ds.pr = pr; ds.pj = pj; ds.prev_waveout = prev_waveout; ds.axc_prev = axc_prev;
}
__global__ void scan_swap_kernel(const ScanView v, int g, FreqSet* save_to, const FreqSet* load_from) {
    const int t = threadIdx.x, Gp = v.Gp;
    if (t == 0) {
        save_to->p = v.params[g];
        save_to->s = v.state[g];
        ChanParams p = v.params[g];
        ChanState s = v.state[g];
        freq_fields_copy(p, s, load_from->p, load_from->s);
        v.params[g] = p;
        v.state[g] = s;
    }
    for (int i = t; i < ABG_SQ_BUF; i += blockDim.x) {
        save_to->sqbuf[i] = v.sqbuf[(size_t)i * Gp + g];
        v.sqbuf[(size_t)i * Gp + g] = load_from->sqbuf[i];
    }
    for (int i = t; i < 2 * ABG_MAX_TONES; i += blockDim.x) {
        const int w = i / ABG_MAX_TONES, k = i % ABG_MAX_TONES;
        const size_t o = (size_t)i * Gp + g;
        save_to->tone_coeff[w][k] = v.tone_coeff[o]; v.tone_coeff[o] = load_from->tone_coeff[w][k];
        save_to->tone_q1[w][k] = v.tone_q1[o];       v.tone_q1[o] = load_from->tone_q1[w][k];
        save_to->tone_q2[w][k] = v.tone_q2[o];       v.tone_q2[o] = load_from->tone_q2[w][k];
        save_to->tone_mag[w][k] = v.tone_mag[o];     v.tone_mag[o] = load_from->tone_mag[w][k];
    }
}

struct Group {
    int sfmt, hop_bytes;
    float fullscale;
    std::vector<int> devs;
    int frames_per_tile = 0, tile_bytes_cap = 0;      // full-spectrum kernel (k1_fft.cu)
    int p_frames_per_tile = 0, p_tile_bytes_cap = 0;  // output-pruned kernel (k1_pruned.cu)
    int max_channels = 0;
    bool pruned = false;                               // which kernel this group runs
    DevBuf<float> wsc;
    std::vector<float> h_wsc;
    K1Dev* d_k1 = nullptr;  // device array [devs.size() + 1]: the extra (all-zero) entry is the tensor-core kernel's tile counter
    std::vector<K1Dev> h_k1;  // host copy, uploaded by value with every run (upload_small)
    // tensor-core K1 (k1_tc.cu)
    bool use_tc = false;
    K1TcPlan tc{};
    DevBuf<signed char> tc_btab;
    DevBuf<long long> tc_sq;
    DevBuf<int32_t> tc_tab_of_dev;
    double tc_cscale = 0.0;
    int tc_tables = 0;  // tables the buffers have room for
};

struct Slot {
    float* wout = nullptr;    // pinned [G][nbmax*B]
    float* iqout = nullptr;   // pinned [G][nbmax*B][2] or null
    unsigned char* axc = nullptr;  // pinned [nbmax][Gp]
    float* mix = nullptr;     // pinned [nbmax][n_mixers][2][B]
    int32_t* mixflag = nullptr;  // pinned [nbmax][n_mixers]
    int mix_pending = 0;
    cudaEvent_t done = nullptr;
    int pending = 0;          // unfetched device-batches referencing this slot
};

}  // namespace

struct abg_engine {
    int N = 0, W = 0, B = 0, fm_demod = 0, nbmax = 4, P = 0, G = 0, Gp = 0, fft_mode = 0;
    int cuda_dev = 0, sm_count = 132, tc_digits = 4;
    bool tc_auto = true;               // fft_mode 0 picks the tensor-core K1 for eligible groups (ABG_K1_TC_AUTO=0: FP32 kernels only)
    int32_t* tc_status = nullptr;      // pinned + mapped: the tensor-core K1 reports a stalled pipeline here (never hangs)
    int32_t* tc_status_dev = nullptr;
    bool any_iq_out = false;
    std::vector<Device> dev;
    std::vector<Group> groups;
    std::vector<ChanParams> h_params;
    bool any_nfm = false;  // some channel or scan-list entry demodulates NFM
    struct ScanChan {
        int g = 0, n_freqs = 0, cur = 0;
        FreqSet* stash = nullptr;  // device array [n_freqs]; entry `cur` is stale while it is live
    };
    std::vector<ScanChan> scan;
    // device memory
    DevBuf<ChanParams> params;
    DevBuf<ChanState> state;
    DevBuf<int32_t> bins, base_bins;
    DevBuf<float> win[2], wout, sqbuf, tone_coeff, tone_q1, tone_q2, tone_mag, lut;  // win/iqin are double-buffered: K1 of run i+1
    DevBuf<float2> iqin[2], iqout, tw1, tw2, twn;                                           // fills one while K2 of run i reads the other
    DevBuf<unsigned char> axc;
    K2Dev* d_k2 = nullptr;
    std::vector<K2Dev> h_k2;  // host copy, uploaded by value with every run (upload_small)
    std::vector<Slot> slots;
    int next_slot = 0;
    cudaStream_t stream = nullptr;   // stream A: ingest copies + K1
    bool own_stream = false;
    cudaStream_t stream_b = nullptr; // stream B: K2, mixers, result copies, tail copy
    cudaStream_t stream_c = nullptr; // stream C: ingest (abg_push host->device copies, buffer compaction)
    cudaEvent_t ev_ingest = nullptr; // last ingest operation
    bool ingest_dirty = false;
    cudaEvent_t ev_k1[2] = {nullptr, nullptr}, ev_k2[2] = {nullptr, nullptr};
    uint64_t run_index = 0;
    bool any_afc = false;
    int k2_lpw = 32;
    uint64_t launches = 0;
    // timing events of the last TL_RUNS runs: [0] K1 start, [1] K1 end (stream A); [2] K2 start, [3] K2 end, [4] end of run (stream B)
    cudaEvent_t tl[TL_RUNS][5] = {};
    bool tev_valid = false;
    std::vector<int32_t> h_bins;
    // batch monitors: the first four, the activity detector and the I/Q history's append are launched in this order on
    // stream A after K1, the tone meter on stream B after K2
    MonitorLaunch<SpecCfg, SpecRun, SpecDev> spectrum{"spectrum", true};
    MonitorLaunch<CarCfg, CarRun, CarDev> carrier{"carrier meter", false};
    MonitorLaunch<InmCfg, InmRun, InmDev> input_meter{"input meter", true};
    SubbandLaunch subband{"sub-band", true};
    ToneMeterLaunch tone_meter{"tone meter", false, true};
    MonitorLaunch<ActCfg, ActRun, ActDev> activity{"activity detector", true};
    HistoryLaunch history{"I/Q history", true};  // the append, last on stream A
    template <typename F>
    void each_monitor(F&& f) {
        f(spectrum); f(carrier); f(input_meter); f(subband); f(tone_meter); f(activity); f(history);
    }
    // after the last monitor that read raw[] in the latest run of each parity that launched one; created when the first
    // such monitor is switched on
    cudaEvent_t ev_raw[2] = {nullptr, nullptr};
    // mixers (reference src/mixer.cpp)
    int n_mixers = 0;
    DevBuf<int32_t> mix_offsets;
    DevBuf<MixInput> mix_inputs;
    DevBuf<float> mix_sums;     // [nbmax][n_mixers][2][B]
    DevBuf<int32_t> mix_flags;  // [nbmax][n_mixers]
    std::deque<std::pair<int, int>> mix_ready;  // (slot, batch-in-run), same for every mixer
    std::vector<int> mix_fetched;               // per mixer: entries of mix_ready already popped by that mixer
    // history replay (abg_history_replay): the replay engine, one device per job, and the gather's records; created by the
    // first replay, kept while its shape fits, freed when the last history is switched off
    bool replay_engine = false;       // this engine is one: K1 groups split by the path a one-device engine would take
    struct ReplayDevice {  // one device of the replay engine: the shape it was built for and its latest channel list
        int32_t sfmt = 0, sample_rate = 0;
        float fullscale = 0.0f;
        bool afc = false, iq = false;  // some channel has AFC / I/Q outputs
        std::vector<abg_channel_cfg> chans;
        bool same_shape(const ReplayDevice& o) const {
            return sfmt == o.sfmt && sample_rate == o.sample_rate && memcmp(&fullscale, &o.fullscale, sizeof(float)) == 0 &&
                   afc == o.afc && iq == o.iq && chans.size() == o.chans.size();
        }
    };
    abg_engine* replay = nullptr;
    std::vector<ReplayDevice> replay_pool;  // [replay->dev.size()]
    DevBuf<RpGather> replay_gather;
    cudaEvent_t replay_ev[2] = {nullptr, nullptr};  // gather start, gather end (the replay's K1 waits on it)
    float replay_ms[2] = {0.0f, 0.0f};
    // live follow (abg_follow_open ...): follow engines, each a pool of devices built for one session shape, and the open
    // sessions; created by the first open, kept while a history is on, never rebuilt
    struct FollowBatch {
        std::vector<float> wout, iq;  // [C][B], [C][2B]
        std::vector<char> axc;        // [C]
    };
    struct FollowSession {
        int dev = 0, eng = 0, slot = 0;        // parent device; follow engine and its device
        int C = 0, queue_batches = 0;
        uint64_t first_batch = 0, next_batch = 0;  // next_batch: the next batch to enqueue
        unsigned long long pushed = 0, valid = 0;  // bytes of the window in the follow device's buffer / gathered from the history
        bool lost = false;
        std::deque<FollowBatch> q;  // finished batches moved out of the follow engine's result slots, oldest first
    };
    struct FollowEngine {
        abg_engine* r = nullptr;
        std::vector<ReplayDevice> pool;  // [r->dev.size()]
        std::vector<int32_t> owner;      // session id per device, -1 = free
        cudaEvent_t ev_compact = nullptr;  // after the compactions of a chunk on r's ingest stream
    };
    std::vector<FollowEngine> follow;
    std::map<int32_t, FollowSession> sessions;
    int32_t next_session = 0;
    DevBuf<RpGather> follow_gather;
    std::vector<cudaEvent_t> follow_tev;  // (start, end) pairs: the latest abg_follow_run's gathers and runs
    std::vector<int> follow_kind;         // per pair: 0 = gather, 1 = follow-engine run
    int follow_pairs = 0;
    // history analysis (abg_history_spectrogram, abg_history_activity): the calls' own buffers, never the live monitors';
    // created by the first call, freed when the last history is switched off
    struct Analysis {
        DevBuf<unsigned char> scratch;   // one chunk's gathered window bytes
        DevBuf<unsigned char> work;      // one chunk's spectrum chunk sums, then int32 counters per row (zero between launches)
        DevBuf<unsigned char> table;     // one chunk's gather records, kernel tables and thresholds
        unsigned char* h_table = nullptr;  // page-locked staging of `table`
        size_t h_table_bytes = 0;
        unsigned char* result = nullptr;   // page-locked, mapped: one chunk's spectrogram rows or detector entries
        size_t result_bytes = 0;
        cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};  // gather start, gather end, kernel end
        float ms[3] = {0.0f, 0.0f, 0.0f};  // the latest call: gathers, spectrum kernels, detector kernels
    } analysis;
    // transmission profiles (abg_history_profile): the call's own buffers; created by the first call, freed when the last
    // history is switched off
    struct Profile {
        DevBuf<float2> scratch;            // one chunk's captured outputs
        DevBuf<unsigned char> table;       // one chunk's coefficients, tone phases and block table
        DevBuf<float> res;                 // one chunk's block sums
        unsigned char* h_table = nullptr;  // page-locked staging of `table`
        float* h_res = nullptr;            // page-locked copy of `res`
        cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};  // captures start, captures end, profile kernel end
        float ms[2] = {0.0f, 0.0f};        // the latest call: captures, profile kernels
    } profile;

    K2Launch k2_launch(int cur) const {
        K2Launch L{};
        L.G = G; L.Gp = Gp; L.P = P; L.wave_batch = B; L.fm_demod = fm_demod; L.iq_stride = nbmax * B;
        L.lanes_per_warp = k2_lpw;
        L.nfm_blocks = any_nfm ? 1 : 0;
        L.params = params.p; L.state = state.p; L.devs = d_k2; L.bins = bins.p; L.base_bins = base_bins.p;
        L.win = win[cur].p; L.iqin = iqin[cur].p; L.win_next = win[cur ^ 1].p; L.iqin_next = iqin[cur ^ 1].p; L.wout = wout.p; L.iqout = any_iq_out ? iqout.p : nullptr;
        L.sqbuf = sqbuf.p; L.tone_coeff = tone_coeff.p; L.tone_q1 = tone_q1.p; L.tone_q2 = tone_q2.p; L.tone_mag = tone_mag.p;
        L.axc = axc.p; L.sincos_lut = lut.p;
        return L;
    }
};

namespace {

// The stream a monitor's kernel runs on: B after K2 for a monitor of the audio, A after K1 for the others.
template <typename Cfg, typename Run, typename Dev>
cudaStream_t monitor_stream(const abg_engine* e, const MonitorLaunch<Cfg, Run, Dev>& m) {
    return m.after_k2 ? e->stream_b : e->stream;
}

// Device `dev`'s state in monitor m; null, after an ABG_ERANGE failure naming the entry point fn, for a device the engine
// does not have.
template <typename Cfg, typename Run, typename Dev>
Dev* monitor_dev(abg_engine* e, MonitorLaunch<Cfg, Run, Dev>& m, int dev, const char* fn) {
    if (dev >= 0 && dev < (int)m.dev.size()) return &m.dev[dev];
    fail(ABG_ERANGE, "%s: device %d out of range", fn, dev);
    return nullptr;
}

// Start of a configure call that changes something, after its own checks: wait until no enqueued kernel of the monitor
// can still read its tables and buffers, then, if the call switches a device on, create the monitor's timing events
// and, if it reads raw[], ev_raw (each once).
template <typename Cfg, typename Run, typename Dev>
int monitor_configure(abg_engine* e, MonitorLaunch<Cfg, Run, Dev>& m, bool on) {
    cudaSetDevice(e->cuda_dev);
    CU(cudaStreamSynchronize(monitor_stream(e, m)));
    if (!on) return ABG_OK;
    if (!m.tl[0][0])
        for (auto& row : m.tl)
            for (auto& ev : row) CU(cudaEventCreate(&ev));
    if (m.reads_raw && !e->ev_raw[0])
        for (int k = 0; k < 2; k++) CU(cudaEventCreateWithFlags(&e->ev_raw[k], cudaEventDisableTiming));
    return ABG_OK;
}

// End of a configure call: rebuild the launch's device list and static table from the per-device state, in device
// order.  `fill(device, state, cfg)` writes the table entry of each device the monitor is on for and returns ABG_OK or
// an error.  With no device left nothing is allocated.
template <typename Cfg, typename Run, typename Dev, typename Fill>
int monitor_publish(abg_engine* e, MonitorLaunch<Cfg, Run, Dev>& m, Fill&& fill) {
    std::vector<int> devs;
    std::vector<Cfg> cfgs;
    for (int i = 0; i < (int)m.dev.size(); i++) {
        if (!m.dev[i].on()) continue;
        Cfg c{};
        const int rc = fill(e->dev[i], m.dev[i], c);
        if (rc != ABG_OK) return rc;
        devs.push_back(i);
        cfgs.push_back(c);
    }
    m.devs = devs;
    m.cfg.free();
    m.h_run.assign(devs.size(), Run{});
    if (cfgs.empty()) return ABG_OK;
    if (m.cfg.alloc(cfgs.size())) return fail(ABG_ENOMEM, "Out of device memory for the %s tables", m.name);
    CU(cudaMemcpy(m.cfg.p, cfgs.data(), sizeof(Cfg) * cfgs.size(), cudaMemcpyHostToDevice));
    // upload_small writes whole 16-byte words: room for every device plus up to 15 bytes of rounding
    if (!m.run.p && m.run.alloc(e->dev.size() + (15 + sizeof(Run) - 1) / sizeof(Run)))
        return fail(ABG_ENOMEM, "Out of device memory for the %s tables", m.name);
    return ABG_OK;
}

// Per-run records of a monitor: `each(run record, monitor state, device, n)` for every device it covers, n the device's
// batches in this run.
template <typename Cfg, typename Run, typename Dev, typename Each>
void monitor_runs(abg_engine* e, MonitorLaunch<Cfg, Run, Dev>& m, const std::vector<int>& nb, Each&& each) {
    for (size_t k = 0; k < m.devs.size(); k++) {
        const int i = m.devs[k];
        each(m.h_run[k], m.dev[i], e->dev[i], nb[i]);
    }
}

// One run of a monitor on its stream, after its h_run records are filled: their upload, then
// `kernel(n_devices, max_items, stream)` between the timing events, then ev_raw if it reads raw[].  Nothing when max_items
// is 0.
template <typename Cfg, typename Run, typename Dev, typename Kernel>
int monitor_launch(abg_engine* e, MonitorLaunch<Cfg, Run, Dev>& m, int max_items, Kernel&& kernel) {
    if (max_items <= 0) return ABG_OK;
    const cudaStream_t st = monitor_stream(e, m);
    const int t = (int)(e->run_index % TL_RUNS);
    const int nl = upload_small(m.run.p, m.h_run.data(), sizeof(Run) * m.devs.size(), st);
    if (nl < 0) return fail(ABG_ECUDA, "%s parameter upload failed: %s", m.name, cudaGetErrorString(cudaGetLastError()));
    e->launches += (uint64_t)nl;
    CU(cudaEventRecord(m.tl[t][0], st));
    const cudaError_t er = kernel((int)m.devs.size(), max_items, st);
    if (er != cudaSuccess) return fail(ABG_ECUDA, "%s launch failed: %s", m.name, cudaGetErrorString(er));
    e->launches++;
    CU(cudaEventRecord(m.tl[t][1], st));
    if (m.reads_raw) CU(cudaEventRecord(e->ev_raw[e->run_index & 1], st));
    m.ran[t] = true;
    return ABG_OK;
}

// ms of the monitor's kernel in the most recent run; 0 if that run did not launch it.  `fn` names the entry point.
template <typename Cfg, typename Run, typename Dev>
int monitor_time(abg_engine* e, const MonitorLaunch<Cfg, Run, Dev>& m, float* ms, const char* fn) {
    if (!ms) return fail(ABG_EINVAL, "%s: null argument", fn);
    *ms = 0.0f;
    if (e->run_index == 0 || !m.ran[(e->run_index - 1) % TL_RUNS]) return ABG_OK;
    cudaSetDevice(e->cuda_dev);
    const cudaEvent_t* ts = m.tl[(e->run_index - 1) % TL_RUNS];
    CU(cudaEventSynchronize(ts[1]));
    CU(cudaEventElapsedTime(ms, ts[0], ts[1]));
    return ABG_OK;
}

// Start of a fetch: pop the oldest entry of device dev's queue k once m's kernel of the entry's run has finished.  Returns
// 1 and the entry's ring bytes in *data, 0 if the queue is empty, < 0 on error (ABG_ERANGE for a device the engine does not
// have, naming the entry point fn).
template <typename Cfg, typename Run, typename Dev>
int monitor_fetch(abg_engine* e, MonitorLaunch<Cfg, Run, Dev>& m, int dev, int k, const char* fn, const unsigned char** data,
                  MonitorQueue::Entry* got) {
    Dev* d = monitor_dev(e, m, dev, fn);
    if (!d) return ABG_ERANGE;
    MonitorQueue& q = d->queue(k);
    if (q.ready.empty()) return 0;
    *got = q.ready.front();
    cudaSetDevice(e->cuda_dev);
    CU(cudaEventSynchronize(m.tl[got->run % TL_RUNS][1]));  // (a later record of it is a later run: also fine)
    *data = q.ring + (size_t)got->pos * q.entry_bytes;
    q.ready.pop_front();  // the bytes stay put until a later run is enqueued
    return 1;
}

void engine_free(abg_engine* e);

// The replay engine and the gather's records and events (abg_history_replay).
void replay_free(abg_engine* e) {
    if (e->replay) engine_free(e->replay);
    e->replay = nullptr;
    e->replay_pool.clear();
    e->replay_gather.free();
    for (auto& ev : e->replay_ev) {
        if (ev) cudaEventDestroy(ev);
        ev = nullptr;
    }
}

// The follow engines, every session and the follow gather's records and events (abg_follow_open ...).
void follow_free(abg_engine* e) {
    for (auto& f : e->follow) {
        engine_free(f.r);
        if (f.ev_compact) cudaEventDestroy(f.ev_compact);
    }
    e->follow.clear();
    e->sessions.clear();
    e->follow_gather.free();
    for (auto ev : e->follow_tev) cudaEventDestroy(ev);
    e->follow_tev.clear();
    e->follow_kind.clear();
    e->follow_pairs = 0;
}

// The history analysis buffers and events (abg_history_spectrogram, abg_history_activity).
void analysis_free(abg_engine* e) {
    auto& a = e->analysis;
    a.scratch.free();
    a.work.free();
    a.table.free();
    if (a.h_table) cudaFreeHost(a.h_table);
    if (a.result) cudaFreeHost(a.result);
    a.h_table = a.result = nullptr;
    a.h_table_bytes = a.result_bytes = 0;
    for (auto& ev : a.ev) {
        if (ev) cudaEventDestroy(ev);
        ev = nullptr;
    }
}

// The transmission profile buffers and events (abg_history_profile).
void profile_free(abg_engine* e) {
    auto& p = e->profile;
    p.scratch.free();
    p.table.free();
    p.res.free();
    if (p.h_table) cudaFreeHost(p.h_table);
    if (p.h_res) cudaFreeHost(p.h_res);
    p.h_table = nullptr;
    p.h_res = nullptr;
    for (auto& ev : p.ev) {
        if (ev) cudaEventDestroy(ev);
        ev = nullptr;
    }
}

void engine_free(abg_engine* e) {
    if (!e) return;
    cudaSetDevice(e->cuda_dev);
    if (e->stream) cudaStreamSynchronize(e->stream);
    if (e->stream_b) cudaStreamSynchronize(e->stream_b);
    replay_free(e);
    follow_free(e);
    analysis_free(e);
    profile_free(e);
    for (auto& d : e->dev) {
        for (int i = 0; i < 2; i++)
            if (d.raw[i]) cudaFree(d.raw[i]);
        if (d.res) cudaFree(d.res);
        if (d.spec) cudaFree(d.spec);
    }
    e->each_monitor([](auto& m) { m.release(); });
    for (auto& g : e->groups) {
        g.wsc.free();
        g.tc_btab.free(); g.tc_sq.free(); g.tc_tab_of_dev.free();
        if (g.d_k1) cudaFree(g.d_k1);
    }
    if (e->tc_status) cudaFreeHost(e->tc_status);
    e->params.free(); e->state.free(); e->bins.free(); e->base_bins.free(); e->win[0].free(); e->win[1].free(); e->wout.free(); e->sqbuf.free();
    e->tone_coeff.free(); e->tone_q1.free(); e->tone_q2.free(); e->tone_mag.free(); e->lut.free(); e->iqin[0].free(); e->iqin[1].free(); e->iqout.free();
    e->tw1.free(); e->tw2.free(); e->twn.free(); e->axc.free(); e->mix_sums.free(); e->mix_flags.free(); e->mix_offsets.free(); e->mix_inputs.free();
    if (e->d_k2) cudaFree(e->d_k2);
    for (auto& sc : e->scan)
        if (sc.stash) cudaFree(sc.stash);
    for (auto& s : e->slots) {
        if (s.wout) cudaFreeHost(s.wout);
        if (s.iqout) cudaFreeHost(s.iqout);
        if (s.axc) cudaFreeHost(s.axc);
        if (s.mix) cudaFreeHost(s.mix);
        if (s.mixflag) cudaFreeHost(s.mixflag);
        if (s.done) cudaEventDestroy(s.done);
    }
    for (auto& row : e->tl)
        for (auto& ev : row)
            if (ev) cudaEventDestroy(ev);
    for (int k = 0; k < 2; k++) {
        if (e->ev_k1[k]) cudaEventDestroy(e->ev_k1[k]);
        if (e->ev_k2[k]) cudaEventDestroy(e->ev_k2[k]);
        if (e->ev_raw[k]) cudaEventDestroy(e->ev_raw[k]);
    }
    if (e->stream_b) cudaStreamDestroy(e->stream_b);
    if (e->stream_c) {
        cudaStreamSynchronize(e->stream_c);
        cudaStreamDestroy(e->stream_c);
    }
    if (e->ev_ingest) cudaEventDestroy(e->ev_ingest);
    if (e->own_stream && e->stream) cudaStreamDestroy(e->stream);
    delete e;
}

int frames_available(const abg_engine* e, const Device& d, size_t fill, size_t consumed) {
    // reference src/rtl_airband.cpp:394-400: a frame is taken only while available >= bps + fft_size*bytes_per_sample*2
    const size_t avail = fill - consumed;
    const size_t need = (size_t)d.hop_bytes + (size_t)e->N * d.bpc;
    if (avail < need) return 0;
    return (int)((avail - need) / d.hop_bytes) + 1;
}

// The freq_t part of one channel as parse_channels() sets it up (config.cpp:437-619): Squelch, NotchFilter,
// LowpassFilter, CTCSS banks, ampfactor, modulation, agcavgfast.  Used for channels[] at abg_create() and for every
// entry of a scan-mode frequency list (abg_scan_configure).  Channel-level fields of p / s are left alone.
int build_freq(int W, const abg_channel_cfg& cc, ChanParams& p, ChanState& s, std::vector<float> banks[2], const char* what) {
    if (cc.modulation != ABG_MOD_AM && cc.modulation != ABG_MOD_NFM) return fail(ABG_EINVAL, "%s: unknown modulation", what);
    p.modulation = cc.modulation;
    p.ampfactor = cc.ampfactor;
    p.notch_on = p.lp_on = p.ctcss_on = 0;
    p.n_tones[0] = p.n_tones[1] = 0;
    banks[0].clear();
    banks[1].clear();
    // ---- Squelch::Squelch(), squelch.cpp:36-82 ----
    s.noise_floor = 5.0f;
    s.manual = 0;
    s.normal_ratio = pow(10.0, 9.54f / 20.0);
    s.flappy_ratio = s.normal_ratio * 0.9f;
    s.avg_cap = 1.5f * s.normal_ratio * s.noise_floor;
    s.manual_level = -1.0;
    s.pre_full = s.pre_capped = s.post_full = s.post_capped = 0.001f;
    s.level_cache = 0.0f;
    s.using_post = 0;
    s.next_state = s.cur_state = SQ_CLOSED;
    s.delay = 0;
    s.sample_count_mod16 = 15u;  // sample_count_ = (size_t)-1: the first sample makes it 0 (squelch.cpp:58,204)
    s.head = 0;
    // ---- config.cpp:437-515: level first, then SNR ----
    if (cc.squelch_level > 0) {  // set_squelch_level_threshold, squelch.cpp:84-96
        s.manual = 1;
        s.manual_level = cc.squelch_level;
        s.avg_cap = 1.5f * s.manual_level;
    }
    if (cc.squelch_snr_db >= 0) {  // set_squelch_snr_threshold, squelch.cpp:98-108
        s.manual = 0;
        s.normal_ratio = pow(10.0, cc.squelch_snr_db / 20.0);
        s.flappy_ratio = s.normal_ratio * 0.9f;
        s.avg_cap = 1.5f * s.normal_ratio * s.noise_floor;
    }
    // ---- NotchFilter, filters.cpp:30-47 ----
    if (cc.notch_hz > 0) {
        float sample_freq = W, q = cc.notch_q;
        float wo = 2 * M_PI * (cc.notch_hz / sample_freq);
        float en = 1 / (1 + tan(wo / (q * 2)));
        float pn = cos(wo);
        p.notch_on = 1;
        p.nd0 = en;
        p.nd1 = 2 * en * pn;
        p.nd2 = (2 * en - 1);
    }
    // ---- LowpassFilter, filters.cpp:67-96 ----
    if (cc.lowpass_hz > 0) {
        if (!lowpass_design(cc.lowpass_hz, (float)W, &p.lp_gain, &p.lp_yc0, &p.lp_yc1))
            return fail(ABG_EINVAL, "%s: lowpass design failed (poles not conjugate)", what);
        p.lp_on = 1;
    }
    // ---- CTCSS, squelch.cpp:110-116 ----
    if (cc.ctcss_hz > 0) {
        const float sr = W;
        p.ctcss_on = 1;
        p.window[0] = sr * 0.05;
        p.window[1] = sr * 0.4;
        for (int w = 0; w < 2; w++) {
            std::vector<float> bank = tone_bank(cc.ctcss_hz, sr, p.window[w]);
            if ((int)bank.size() > ABG_MAX_TONES) return fail(ABG_EINVAL, "CTCSS bank too large");
            p.n_tones[w] = (int)bank.size();
            banks[w] = bank;
        }
    }
    s.agcavgfast = 0.5f;  // mk_freqlist / parse_channels, config.cpp:265-281
    return ABG_OK;
}

// 7-term Blackman-Harris window: float literals held in double, evaluated in double, stored float (rtl_airband.cpp:335-351)
std::vector<float> make_window(int N) {
    std::vector<float> window(N);
    const double a0 = 0.27105140069342f, a1 = 0.43329793923448f, a2 = 0.21812299954311f, a3 = 0.06592544638803f;
    const double a4 = 0.01081174209837f, a5 = 0.00077658482522f, a6 = 0.00001388721735f;
    const size_t fft_size = N;
    for (size_t i = 0; i < fft_size; i++) {
        double x = a0 - (a1 * cos((2.0 * M_PI * i) / (fft_size - 1))) + (a2 * cos((4.0 * M_PI * i) / (fft_size - 1))) - (a3 * cos((6.0 * M_PI * i) / (fft_size - 1))) +
                   (a4 * cos((8.0 * M_PI * i) / (fft_size - 1))) - (a5 * cos((10.0 * M_PI * i) / (fft_size - 1))) + (a6 * cos((12.0 * M_PI * i) / (fft_size - 1)));
        window[i] = (float)x;
    }
    return window;
}
float sample_scale(int sfmt, float fullscale) {
    // U8 levels are (i-127.5)/127.5, S8 i/128 (rtl_airband.cpp:319-324); S16/F32 scale = 1/fullscale (:403,421)
    return sfmt == ABG_SFMT_U8 ? 1.0f / 127.5f : sfmt == ABG_SFMT_S8 ? 1.0f / 128.0f : 1.0f / fullscale;
}

// (Re)build the tensor-core K1's coefficient tables of one launch group from the host copy of bins[]: one table per
// distinct list of bins (synthetic many-device configs share one), tab_of_dev[] maps the group's devices to tables.
int rebuild_tc_tables(abg_engine* e, Group& g) {
    std::vector<std::vector<int32_t>> keys;
    std::vector<int32_t> tab_of_dev(g.devs.size());
    for (size_t k = 0; k < g.devs.size(); k++) {
        const Device& d = e->dev[g.devs[k]];
        std::vector<int32_t> key(e->h_bins.begin() + d.g0, e->h_bins.begin() + d.g0 + d.C);
        size_t t = 0;
        while (t < keys.size() && keys[t] != key) t++;
        if (t == keys.size()) keys.push_back(key);
        tab_of_dev[k] = (int32_t)t;
    }
    const size_t nt = keys.size();
    std::vector<signed char> tab(nt * g.tc.table_bytes);
    std::vector<long long> sq(nt * g.tc.C2p);
    for (size_t t = 0; t < nt; t++)
        abg_k1tc_build_table(g.tc, e->N, g.sfmt, g.h_wsc.data(), keys[t].data(), (int)keys[t].size(), tab.data() + t * g.tc.table_bytes,
                             sq.data() + t * g.tc.C2p, &g.tc_cscale);
    if ((int)nt > g.tc_tables) {  // grow only: a smaller set of tables uses the front of the buffers
        g.tc_btab.free(); g.tc_sq.free();
        if (g.tc_btab.alloc(tab.size()) || g.tc_sq.alloc(sq.size())) return fail(ABG_ENOMEM, "Out of device memory for the tensor-core coefficient tables");
        g.tc_tables = (int)nt;
    }
    if (!g.tc_tab_of_dev.p && g.tc_tab_of_dev.alloc(tab_of_dev.size())) return fail(ABG_ENOMEM, "Out of device memory for the tensor-core coefficient tables");
    CU(cudaMemcpy(g.tc_btab.p, tab.data(), tab.size(), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(g.tc_sq.p, sq.data(), sizeof(long long) * sq.size(), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(g.tc_tab_of_dev.p, tab_of_dev.data(), sizeof(int32_t) * tab_of_dev.size(), cudaMemcpyHostToDevice));
    return ABG_OK;
}

// The channels of cfg as parse_channels() resolves them (config.cpp:265-281,306-726): parameters, initial state, bins and
// CTCSS banks of every channel into hp, hs, hb and h_coeff ([Gp] and [2][ABG_MAX_TONES][Gp]), and the engine flags that
// follow from them.  The engine's devices are laid out already.  abg_create and every history replay start from it.
// Which K1 a launch group of this format and hop takes, from its largest channel count and whether a device has AFC (a
// group with AFC needs whole spectra): *use_tc with fft_mode 3, or 0 with tc_auto, when a tensor-core plan exists (into
// *tc); *pruned unless fft_mode is 1 when the output-pruned kernel fits (its tile into *p_frames, *p_cap).  build() decides
// every group with it, and a replay engine groups its devices by what it decides for each device alone.
void k1_choice(const abg_engine* e, int sfmt, int hop_bytes, int max_channels, bool afc, bool* pruned, bool* use_tc, K1TcPlan* tc,
               int* p_frames, int* p_cap) {
    *p_frames = abg_k1p_tile_frames(e->N, sfmt, hop_bytes, max_channels, p_cap);
    *pruned = (e->fft_mode != 1) && !afc && *p_frames >= 1;
    const bool want_tc = e->fft_mode == 3 || (e->fft_mode == 0 && e->tc_auto);
    *use_tc = want_tc && !afc && abg_k1tc_plan(e->N, sfmt, hop_bytes, max_channels, e->tc_digits, tc) == 1;
}

int resolve_channels(abg_engine* e, const abg_config* cfg, std::vector<ChanParams>& hp, std::vector<ChanState>& hs,
                     std::vector<int32_t>& hb, std::vector<float>& h_coeff) {
    const int N = e->N, G = e->G, Gp = e->Gp;
    hp.assign(Gp, ChanParams{});
    hs.assign(Gp, ChanState{});
    hb.assign(Gp, 0);
    h_coeff.assign((size_t)2 * ABG_MAX_TONES * Gp, 0.0f);
    memset(hp.data(), 0, sizeof(ChanParams) * Gp);
    memset(hs.data(), 0, sizeof(ChanState) * Gp);
    e->any_iq_out = e->any_nfm = false;
    for (int i = 0; i < cfg->n_devices; i++) {
        const abg_device_cfg& dc = cfg->devices[i];
        Device& d = e->dev[i];
        d.has_afc = false;
        for (int c = 0; c < dc.n_channels; c++) {
            const abg_channel_cfg& cc = dc.channels[c];
            const int g = d.g0 + c;
            if (cc.bin < 0 || cc.bin >= N) return fail(ABG_EINVAL, "devices[%d].channels[%d]: bin %d outside 0..%d", i, c, cc.bin, N - 1);
            ChanParams& p = hp[g];
            ChanState& s = hs[g];
            hb[g] = cc.bin;
            p.dev = i;
            p.needs_raw_iq = cc.needs_raw_iq ? 1 : 0;
            p.has_iq_outputs = cc.has_iq_outputs ? 1 : 0;
            if (p.has_iq_outputs) e->any_iq_out = true;
            p.dm_dphi = cc.dm_dphi;
            p.alpha = cc.alpha;
            p.afc = cc.afc & 0xff;
            if (p.afc) d.has_afc = true;
            {
                char what[64];
                snprintf(what, sizeof(what), "devices[%d].channels[%d]", i, c);
                std::vector<float> banks[2];
                const int rc = build_freq(e->W, cc, p, s, banks, what);
                if (rc != ABG_OK) return rc;
                for (int w = 0; w < 2; w++)
                    for (size_t t = 0; t < banks[w].size(); t++) h_coeff[((size_t)w * ABG_MAX_TONES + t) * Gp + g] = banks[w][t];
            }
            // ---- mk_freqlist / parse_channels initial values, config.cpp:265-281,313-331 ----
            s.dm_phi = 0;
            s.pr = s.pj = 0.0f;
            s.prev_waveout = 0.5f;
            s.axc_prev = ABG_NO_SIGNAL;
        }
    }
    e->h_params = hp;
    for (int g = 0; g < G; g++)
        if (hp[g].modulation == ABG_MOD_NFM) e->any_nfm = true;
    e->h_bins = hb;
    return ABG_OK;
}

// Upload what resolve_channels built and reset every buffer K2 carries from batch to batch, the AGC look-back rows
// primed: the channel state abg_create leaves behind.
int upload_channels(abg_engine* e, const std::vector<ChanParams>& hp, const std::vector<ChanState>& hs, const std::vector<int32_t>& hb,
                    const std::vector<float>& h_coeff) {
    const int Gp = e->Gp, B = e->B;
    const size_t PG = (size_t)e->P * Gp;
    CU(cudaMemcpy(e->params.p, hp.data(), sizeof(ChanParams) * Gp, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(e->state.p, hs.data(), sizeof(ChanState) * Gp, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(e->bins.p, hb.data(), sizeof(int32_t) * Gp, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(e->base_bins.p, hb.data(), sizeof(int32_t) * Gp, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(e->tone_coeff.p, h_coeff.data(), sizeof(float) * h_coeff.size(), cudaMemcpyHostToDevice));
    CU(cudaMemset(e->tone_q1.p, 0, sizeof(float) * h_coeff.size()));
    CU(cudaMemset(e->tone_q2.p, 0, sizeof(float) * h_coeff.size()));
    CU(cudaMemset(e->tone_mag.p, 0, sizeof(float) * h_coeff.size()));
    CU(cudaMemset(e->sqbuf.p, 0, sizeof(float) * ABG_SQ_BUF * Gp));  // calloc, squelch.cpp:70
    CU(cudaMemset(e->iqin[0].p, 0, sizeof(float2) * PG));
    CU(cudaMemset(e->iqin[1].p, 0, sizeof(float2) * PG));
    if (e->any_iq_out) CU(cudaMemset(e->iqout.p, 0, sizeof(float2) * (size_t)Gp * e->nbmax * B));
    {
        // config.cpp:313-316: wavein[0..AGC_EXTRA) = 20, waveout[0..AGC_EXTRA) = 0.5.  (wavein's priming values are
        // overwritten by the first AGC_EXTRA frames because waveend starts at 0, config.cpp:805; kept for fidelity.)
        std::vector<float> hw(PG, 0.0f), ho(PG, 0.0f);
        for (int k = 0; k < ABG_AGC_EXTRA; k++)
            for (int g = 0; g < Gp; g++) hw[(size_t)k * Gp + g] = 20.0f;
        for (int g = 0; g < Gp; g++)
            for (int k = 0; k < ABG_AGC_EXTRA; k++) ho[(size_t)g * e->P + k] = 0.5f;
        CU(cudaMemcpy(e->win[0].p, hw.data(), sizeof(float) * PG, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(e->win[1].p, hw.data(), sizeof(float) * PG, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(e->wout.p, ho.data(), sizeof(float) * PG, cudaMemcpyHostToDevice));
    }
    return ABG_OK;
}

int build(abg_engine* e, const abg_config* cfg, const abg_options* opt) {
    Plan plan;
    if (!plan_for(cfg->fft_size, &plan)) return fail(ABG_EINVAL, "fft_size=%d not supported. Try a power of two between 256 and 8192.", cfg->fft_size);
    if (cfg->wave_rate < 8 || cfg->wave_rate % 8) return fail(ABG_EINVAL, "wave_rate=%d must be a positive multiple of 8", cfg->wave_rate);
    if (cfg->n_devices < 1 || !cfg->devices) return fail(ABG_EINVAL, "no devices configured");
    e->N = cfg->fft_size;
    e->W = cfg->wave_rate;
    e->B = cfg->wave_rate / 8;  // WAVE_BATCH, rtl_airband.h:73
    if (e->B < ABG_AGC_EXTRA) return fail(ABG_EINVAL, "wave_rate too small: WAVE_BATCH must be >= AGC_EXTRA");
    e->fm_demod = cfg->fm_demod;
    e->nbmax = (opt && opt->max_batches_per_run > 0) ? opt->max_batches_per_run : 4;
    e->fft_mode = opt ? opt->fft_mode : 0;
    if (const char* ev = getenv("ABG_K1_TC_DIGITS")) e->tc_digits = atoi(ev) == 3 ? 3 : 4;
    if (const char* ev = getenv("ABG_K1_TC_AUTO")) e->tc_auto = atoi(ev) != 0;
    const int in_cap_batches = (opt && opt->input_capacity_batches > 0) ? opt->input_capacity_batches : e->nbmax + 2;
    e->P = ABG_AGC_EXTRA + e->nbmax * e->B;
    const int N = e->N, B = e->B;

    // ---- devices, channel index space ------------------------------------------------------------------------
    e->dev.resize(cfg->n_devices);
    e->each_monitor([&](auto& m) { m.dev.resize(cfg->n_devices); });
    int G = 0;
    for (int i = 0; i < cfg->n_devices; i++) {
        const abg_device_cfg& dc = cfg->devices[i];
        Device& d = e->dev[i];
        d.sfmt = dc.sfmt;
        switch (dc.sfmt) {
            case ABG_SFMT_U8: case ABG_SFMT_S8: d.bpc = 2; break;
            case ABG_SFMT_S16: d.bpc = 4; break;
            case ABG_SFMT_F32: d.bpc = 8; break;
            default: return fail(ABG_EINVAL, "devices[%d]: unknown sample format %d", i, dc.sfmt);
        }
        if (dc.n_channels < 1 || !dc.channels) return fail(ABG_EINVAL, "devices[%d]: no channels configured", i);
        if (dc.sample_rate <= cfg->wave_rate) return fail(ABG_EINVAL, "devices[%d]: sample_rate must be greater than %d", i, cfg->wave_rate);
        if ((dc.sfmt == ABG_SFMT_S16 || dc.sfmt == ABG_SFMT_F32) && !(dc.fullscale > 0)) return fail(ABG_EINVAL, "devices[%d]: fullscale must be > 0", i);
        d.sample_rate = dc.sample_rate;
        d.fullscale = dc.fullscale;
        d.hop = (int)round((double)dc.sample_rate / (double)cfg->wave_rate);  // rtl_airband.cpp:394
        d.hop_bytes = d.hop * d.bpc;
        d.g0 = G;
        d.C = dc.n_channels;
        G += dc.n_channels;
    }
    e->G = G;
    e->Gp = (G + 31) & ~31;
    const int Gp = e->Gp;

    std::vector<ChanParams> hp;
    std::vector<ChanState> hs;
    std::vector<int32_t> hb;
    std::vector<float> h_coeff;
    int rc = resolve_channels(e, cfg, hp, hs, hb, h_coeff);  // per-channel parameters and initial state
    if (rc != ABG_OK) return rc;

    // ---- tables -----------------------------------------------------------------------------------------------------
    const std::vector<float> window = make_window(N);
    std::vector<float> h_lut(2 * 257);
    for (uint32_t i = 0; i < 256; i++) sincosf(2.0F * M_PI * (float)i / 256.0f, &h_lut[i], &h_lut[257 + i]);  // util.cpp:105-110
    h_lut[256] = h_lut[0];
    h_lut[257 + 256] = h_lut[257];
    const int M1 = N / plan.r1;
    std::vector<float2> h_tw1((size_t)N);
    for (int k1 = 0; k1 < plan.r1; k1++)
        for (int n2 = 0; n2 < M1; n2++) {
            double ang = -2.0 * M_PI * (double)(((long)k1 * n2) % N) / (double)N;
            h_tw1[(size_t)k1 * M1 + n2] = make_float2((float)cos(ang), (float)sin(ang));
        }
    std::vector<float2> h_tw2;
    if (plan.r3) {
        const int M2 = plan.r3;
        h_tw2.resize((size_t)plan.r2 * M2);
        for (int k = 0; k < plan.r2; k++)
            for (int n3 = 0; n3 < M2; n3++) {
                double ang = -2.0 * M_PI * (double)(k * n3) / (double)M1;
                h_tw2[(size_t)k * M2 + n3] = make_float2((float)cos(ang), (float)sin(ang));
            }
    }

    std::vector<float2> h_twn((size_t)N);
    for (int m = 0; m < N; m++) {
        double ang = -2.0 * M_PI * (double)m / (double)N;
        h_twn[m] = make_float2((float)cos(ang), (float)sin(ang));
    }

    // ---- groups (one K1 launch per sample format / full-scale / hop) ------------------------------------------------------
    // A replay engine also keeps devices apart whose one-device engines would take different K1 paths (below): the paths
    // do not round alike, and a replayed job must be bitwise what such an engine computes.
    auto alone_path = [&](const Device& d) {
        if (!e->replay_engine) return 0;
        bool pruned = false, use_tc = false;
        K1TcPlan tc{};
        int frames = 0, cap = 0;
        k1_choice(e, d.sfmt, d.hop_bytes, d.C, d.has_afc, &pruned, &use_tc, &tc, &frames, &cap);
        return use_tc ? 3 : pruned ? 2 : 1;
    };
    std::vector<int> group_path;
    for (int i = 0; i < (int)e->dev.size(); i++) {
        Device& d = e->dev[i];
        int gi = -1;
        for (int k = 0; k < (int)e->groups.size(); k++)
            if (e->groups[k].sfmt == d.sfmt && e->groups[k].hop_bytes == d.hop_bytes &&
                (d.sfmt == ABG_SFMT_U8 || d.sfmt == ABG_SFMT_S8 || e->groups[k].fullscale == d.fullscale) && group_path[k] == alone_path(d))
                gi = k;
        if (gi < 0) {
            Group g;
            g.sfmt = d.sfmt;
            g.hop_bytes = d.hop_bytes;
            g.fullscale = d.fullscale;
            e->groups.push_back(g);
            group_path.push_back(alone_path(d));
            gi = (int)e->groups.size() - 1;
        }
        d.group = gi;
        e->groups[gi].devs.push_back(i);
    }

    // ---- CUDA resources ----------------------------------------------------------------------------------------------------
    {
        const char* pe = getenv("ABG_K2_PRIO");  // measurement knob: -1 = K1's stream above K2's
        int lo = 0, hi = 0;
        CU(cudaDeviceGetStreamPriorityRange(&lo, &hi));
        CU(cudaStreamCreateWithPriority(&e->stream, cudaStreamNonBlocking, (pe && atoi(pe) < 0) ? hi : lo));
    }
    e->own_stream = true;
    CU(cudaHostAlloc((void**)&e->tc_status, 64, cudaHostAllocMapped));
    memset(e->tc_status, 0, 64);
    CU(cudaHostGetDevicePointer((void**)&e->tc_status_dev, e->tc_status, 0));
    {
        // K2's few long-running warps must get their SM slots ahead of the next run's K1 blocks
        int lo = 0, hi = 0;
        CU(cudaDeviceGetStreamPriorityRange(&lo, &hi));
        const char* pe = getenv("ABG_K2_PRIO");  // measurement knob: 0 = K2's stream at the default priority
        CU(cudaStreamCreateWithPriority(&e->stream_b, cudaStreamNonBlocking, (pe && atoi(pe) <= 0) ? lo : hi));
    }
    for (int k = 0; k < 2; k++) {
        CU(cudaEventCreateWithFlags(&e->ev_k1[k], cudaEventDisableTiming));
        CU(cudaEventCreateWithFlags(&e->ev_k2[k], cudaEventDisableTiming));
    }
    for (auto& row : e->tl)
        for (auto& ev : row) CU(cudaEventCreate(&ev));
    CU(cudaStreamCreateWithFlags(&e->stream_c, cudaStreamNonBlocking));
    CU(cudaEventCreateWithFlags(&e->ev_ingest, cudaEventDisableTiming));
    for (auto& d : e->dev)
        if (d.has_afc) e->any_afc = true;
    {
        // K2 is a sequential recurrence per channel.  One channel per warp (lane-parallel tiles, no divergence between
        // channels in different squelch states) as long as that is at most 8 warps per SM sub-partition; beyond that as
        // few channels per warp as keeps the warp count near two per sub-partition.
        const int subparts = 4 * e->sm_count;
        int lpw = 1;
        if (e->G > 8 * subparts)
            while (lpw < 32 && (e->G + lpw - 1) / lpw > 2 * subparts) lpw <<= 1;
        const char* env = getenv("ABG_K2_LPW");
        if (env && atoi(env) > 0) {
            lpw = 1;
            while (lpw < 32 && lpw < atoi(env)) lpw <<= 1;
        }
        e->k2_lpw = lpw;
    }
    for (auto& g : e->groups) {
        g.frames_per_tile = abg_k1_tile_frames(N, g.sfmt, g.hop_bytes, &g.tile_bytes_cap);
        if (g.frames_per_tile < 1) return fail(ABG_EINVAL, "fft_size=%d with this sample format does not fit shared memory", N);
        bool group_afc = false;
        for (int di : g.devs) {
            g.max_channels = std::max(g.max_channels, e->dev[di].C);
            if (e->dev[di].has_afc) group_afc = true;
        }
        // fft_mode: 0 auto; 1 = full spectrum every frame; 2 = output-pruned last pass on the FP32 pipes; 3 = the bins' DFT as an
        // integer GEMM on the tensor cores (8-bit formats; other groups fall back to 2).  Groups with AFC need whole spectra.
        k1_choice(e, g.sfmt, g.hop_bytes, g.max_channels, group_afc, &g.pruned, &g.use_tc, &g.tc, &g.p_frames_per_tile, &g.p_tile_bytes_cap);
        const float scale = sample_scale(g.sfmt, g.fullscale);  // window * 1/full-scale
        std::vector<float> wsc(N);
        for (int i = 0; i < N; i++) wsc[i] = window[i] * scale;
        g.h_wsc = wsc;
        CU(g.wsc.alloc(N));
        CU(cudaMemcpy(g.wsc.p, wsc.data(), N * sizeof(float), cudaMemcpyHostToDevice));
        CU(cudaMalloc((void**)&g.d_k1, sizeof(K1Dev) * (g.devs.size() + 1)));
        g.h_k1.assign(g.devs.size() + 1, K1Dev{});
        if (g.use_tc) {
            const int rc = rebuild_tc_tables(e, g);
            if (rc != ABG_OK) return rc;
        }
    }
    for (auto& d : e->dev) {
        // room for in_cap_batches batches + the AGC_EXTRA priming frames + one window, + slack for 16-byte TMA rounding
        d.cap = ((size_t)(in_cap_batches * B + ABG_AGC_EXTRA) * d.hop_bytes + (size_t)N * d.bpc + (size_t)d.hop_bytes + 255) & ~(size_t)255;
        for (int k = 0; k < 2; k++) {
            cudaError_t er = cudaMalloc((void**)&d.raw[k], d.cap + 256);
            if (er != cudaSuccess) return fail(ABG_ENOMEM, "Out of device memory for input buffers (%s)", cudaGetErrorString(er));
            CU(cudaMemsetAsync(d.raw[k], 0, d.cap + 256, e->stream));
        }
        if (d.has_afc) CU(cudaMalloc((void**)&d.spec, sizeof(float2) * (size_t)e->nbmax * N));
    }
    const size_t PG = (size_t)e->P * Gp;
    if (e->params.alloc(Gp) || e->state.alloc(Gp) || e->bins.alloc(Gp) || e->base_bins.alloc(Gp) || e->win[0].alloc(PG) || e->win[1].alloc(PG) || e->iqin[0].alloc(PG) || e->iqin[1].alloc(PG) ||
        e->wout.alloc(PG) || e->sqbuf.alloc((size_t)ABG_SQ_BUF * Gp) || e->tone_coeff.alloc(h_coeff.size()) || e->tone_q1.alloc(h_coeff.size()) ||
        e->tone_q2.alloc(h_coeff.size()) || e->tone_mag.alloc(h_coeff.size()) || e->lut.alloc(h_lut.size()) || e->tw1.alloc(h_tw1.size()) ||
        e->tw2.alloc(std::max<size_t>(h_tw2.size(), 1)) || e->twn.alloc(h_twn.size()) || e->axc.alloc((size_t)e->nbmax * Gp) ||
        (e->any_iq_out && e->iqout.alloc((size_t)Gp * e->nbmax * B)))
        return fail(ABG_ENOMEM, "Out of device memory. Try fewer devices per GPU or a smaller max_batches_per_run.");
    CU(cudaMemcpy(e->lut.p, h_lut.data(), sizeof(float) * h_lut.size(), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(e->tw1.p, h_tw1.data(), sizeof(float2) * h_tw1.size(), cudaMemcpyHostToDevice));
    if (!h_tw2.empty()) CU(cudaMemcpy(e->tw2.p, h_tw2.data(), sizeof(float2) * h_tw2.size(), cudaMemcpyHostToDevice));
    CU(cudaMemcpy(e->twn.p, h_twn.data(), sizeof(float2) * h_twn.size(), cudaMemcpyHostToDevice));
    rc = upload_channels(e, hp, hs, hb, h_coeff);
    if (rc != ABG_OK) return rc;
    CU(cudaMalloc((void**)&e->d_k2, sizeof(K2Dev) * e->dev.size() + 16));
    e->h_k2.assign(e->dev.size(), K2Dev{});
    e->slots.resize(3);
    for (auto& s : e->slots) {
        CU(cudaMallocHost((void**)&s.wout, sizeof(float) * (size_t)std::max(G, 1) * e->nbmax * B));
        if (e->any_iq_out) CU(cudaMallocHost((void**)&s.iqout, sizeof(float2) * (size_t)std::max(G, 1) * e->nbmax * B));
        CU(cudaMallocHost((void**)&s.axc, (size_t)e->nbmax * Gp));
        CU(cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming));
    }
    CU(cudaStreamSynchronize(e->stream));
    return ABG_OK;
}

// Byte of frame j = 0 of the run's first batch in the buffer K1 reads this run (the resident buffer is a stream of its
// own): the first AGC_EXTRA frames of a stream only prime the AGC look-back.
unsigned long long run_first_byte(const Device& d, bool resident) {
    const unsigned long long look_back = (unsigned long long)ABG_AGC_EXTRA * d.hop_bytes;
    return resident ? look_back : (unsigned long long)d.consumed + (d.primed ? 0ull : look_back);
}

// enqueue K1 (+K2) for the per-device batch counts in nb[]; `resident` selects the replay buffers.
int enqueue_run(abg_engine* e, const std::vector<int>& nb, bool resident, bool queue_outputs, int* n_enqueued, bool skip_k1 = false) {
    const int B = e->B, N = e->N;
    int total = 0, nbrun = 0;
    for (int v : nb) {
        total += v;
        nbrun = std::max(nbrun, v);
    }
    *n_enqueued = total;
    if (total == 0) return ABG_OK;
    int slot = -1;
    if (queue_outputs) {
        slot = e->next_slot;
        if (e->slots[slot].pending > 0 || e->slots[slot].mix_pending > 0)
            return fail(ABG_EOVERFLOW, "output overrun: %d finished device batches and %d mixer batches of an earlier run not fetched yet (every configured mixer has to be drained with abg_fetch_mixer_batch)",
                        e->slots[slot].pending, e->slots[slot].mix_pending);
        e->next_slot = (e->next_slot + 1) % (int)e->slots.size();
    }
    cudaStream_t sa = e->stream, sb = e->stream_b;
    const uint64_t ri = e->run_index;
    const int cur = (int)(ri & 1);
    // K1 of this run overwrites win/iqin[cur], last read by K2 of run ri-2; with AFC it also needs the bins K2 of
    // run ri-1 chose.  (ev_k2[x] is re-recorded by every run of that parity; the wait binds to the latest record.)
    if (ri >= 2) CU(cudaStreamWaitEvent(sa, e->ev_k2[cur], 0));
    if (ri >= 1 && e->any_afc) CU(cudaStreamWaitEvent(sa, e->ev_k2[cur ^ 1], 0));
    if (!resident && e->ingest_dirty) {  // K1 reads what abg_push copied on the ingest stream
        CU(cudaEventRecord(e->ev_ingest, e->stream_c));
        CU(cudaStreamWaitEvent(sa, e->ev_ingest, 0));
        e->ingest_dirty = false;
    }
    cudaEvent_t* tl = e->tl[ri % TL_RUNS];
    CU(cudaEventRecord(tl[0], sa));
    // ---- K1 per group (stream A) ----
    for (auto& g : e->groups) {
        if (skip_k1) break;  // abg_debug_inject_wavein: the magnitudes were written into win[cur] directly
        int max_frames = 0;
        for (size_t k = 0; k < g.devs.size(); k++) {
            const int di = g.devs[k];
            Device& d = e->dev[di];
            K1Dev& a = g.h_k1[k];
            const bool primed = resident ? d.res_primed : d.primed;
            a.raw = resident ? d.res : d.raw[d.cur];
            a.n_frames = nb[di] > 0 ? nb[di] * B + (primed ? 0 : ABG_AGC_EXTRA) : 0;
            a.pos0 = primed ? ABG_AGC_EXTRA : 0;
            a.start_byte = resident ? (primed ? (unsigned long long)ABG_AGC_EXTRA * d.hop_bytes : 0ull) : (unsigned long long)d.consumed;
            a.g0 = d.g0;
            a.n_channels = d.C;
            a.hop_bytes = d.hop_bytes;
            a.sfmt = d.sfmt;
            a.spec = d.has_afc ? d.spec : nullptr;
            a.spec_first_pos = ABG_AGC_EXTRA + B - 1;  // the frame that completes batch 0 of the run (waveend hits B+100)
            a.wave_batch = B;
            max_frames = std::max(max_frames, a.n_frames);
        }
        if (max_frames == 0) continue;
        {
            // (the trailing all-zero entry resets the tensor-core kernel's tile counter)
            const int nl = upload_small(g.d_k1, g.h_k1.data(), sizeof(K1Dev) * (g.devs.size() + (g.use_tc ? 1 : 0)), sa);
            if (nl < 0) return fail(ABG_ECUDA, "K1 parameter upload failed: %s", cudaGetErrorString(cudaGetLastError()));
            e->launches += (uint64_t)nl;
        }
        K1Launch L{};
        L.fft_size = N; L.n_devices = (int)g.devs.size(); L.max_frames = max_frames;
        L.frames_per_tile = g.pruned ? g.p_frames_per_tile : g.frames_per_tile;
        L.tile_bytes_cap = g.pruned ? g.p_tile_bytes_cap : g.tile_bytes_cap;
        L.devs = g.d_k1; L.bins = e->bins.p; L.window_scaled = g.wsc.p; L.tw1 = e->tw1.p;
        L.tw2 = e->tw2.p; L.win = e->win[cur].p; L.iqin = e->iqin[cur].p; L.Gp = e->Gp; L.sfmt = g.sfmt;
        cudaError_t er1;
        if (g.use_tc) {
            K1TcTables T{};
            T.tab_of_dev = g.tc_tab_of_dev.p; T.btab = g.tc_btab.p; T.sq = g.tc_sq.p;
            T.counter = reinterpret_cast<int*>(g.d_k1 + g.devs.size());
            T.status = e->tc_status_dev; T.cscale = g.tc_cscale;
            er1 = abg_launch_k1_tc(L, g.tc, T, e->sm_count, sa);
        } else {
            er1 = g.pruned ? abg_launch_k1_pruned(L, e->twn.p, g.max_channels, sa) : abg_launch_k1(L, sa);
        }
        if (er1 != cudaSuccess) return fail(ABG_ECUDA, "K1 launch failed: %s", cudaGetErrorString(er1));
        e->launches += g.use_tc ? 1 : g.pruned ? (uint64_t)((g.max_channels + 31) / 32) : 1;
    }
    CU(cudaEventRecord(tl[1], sa));
    CU(cudaEventRecord(e->ev_k1[cur], sa));
    // ---- batch monitors (stream A after K1 in this order: the spectrum, the carrier meter, the input meter, the sub-band
    // outputs, the activity detector; K2 does not wait for them past ev_k1).  Injected batches have no frames and launch
    // none. ----
    const int t = (int)(ri % TL_RUNS);
    e->each_monitor([t](auto& m) { m.ran[t] = false; });
    // n_batches and ring_pos0 of a monitor with one queue per device: resident runs queue nothing
    auto queue_run = [&](auto& r, MonitorQueue& q, int n, uint64_t seq0, int32_t aux) {
        r.n_batches = n;
        r.ring_pos0 = queue_outputs && n > 0 ? q.queue(n, seq0, ri, aux) : -1;
    };
    if (!skip_k1) {
        int max_items = 0;
        monitor_runs(e, e->spectrum, nb, [&](SpecRun& r, SpecDev& s, Device& d, int n) {
            r.raw = resident ? d.res : d.raw[d.cur];
            r.first_byte = run_first_byte(d, resident);
            queue_run(r, s.q, n, d.batch_seq, s.n_sel);
            max_items = std::max(max_items, n * s.chunks);
        });
        int rc = monitor_launch(e, e->spectrum, max_items, [&](int n_devices, int items, cudaStream_t s) {
            SpecArgs A{};
            A.cfg = e->spectrum.cfg.p; A.run = e->spectrum.run.p; A.tw1 = e->tw1.p; A.tw2 = e->tw2.p; A.wave_batch = B;
            return abg_launch_spectrum(N, A, n_devices, items, s);
        });
        if (rc != ABG_OK) return rc;
        // the carrier meter reads iqin[cur], which the next K1 to write it, two runs later, queues behind on this stream
        max_items = 0;
        monitor_runs(e, e->carrier, nb, [&](CarRun& r, CarDev& s, Device& d, int n) {
            queue_run(r, s.q, n, d.batch_seq, 0);
            max_items = std::max(max_items, n * abg_carrier_items(d.C));
        });
        rc = monitor_launch(e, e->carrier, max_items, [&](int n_devices, int items, cudaStream_t s) {
            CarArgs A{};
            A.cfg = e->carrier.cfg.p; A.run = e->carrier.run.p; A.iqin = e->iqin[cur].p; A.Gp = e->Gp; A.wave_batch = B;
            return abg_launch_carrier(A, n_devices, items, s);
        });
        if (rc != ABG_OK) return rc;
        max_items = 0;
        monitor_runs(e, e->input_meter, nb, [&](InmRun& r, InmDev& s, Device& d, int n) {
            r.raw = resident ? d.res : d.raw[d.cur];
            r.first_byte = run_first_byte(d, resident);
            queue_run(r, s.q, n, d.batch_seq, 0);
            max_items = std::max(max_items, n * s.chunks);
        });
        rc = monitor_launch(e, e->input_meter, max_items, [&](int n_devices, int items, cudaStream_t s) {
            InmArgs A{};
            A.cfg = e->input_meter.cfg.p; A.run = e->input_meter.run.p; A.wave_batch = B;
            return abg_launch_input_meter(A, n_devices, items, s);
        });
        if (rc != ABG_OK) return rc;
        max_items = 0;
        monitor_runs(e, e->subband, nb, [&](SbRun& r, SbDev& s, Device& d, int n) {
            r.raw = resident ? d.res : d.raw[d.cur];
            r.base = resident ? 0 : (long long)(d.dropped / d.bpc);
            r.s0 = r.base + (long long)(run_first_byte(d, resident) / d.bpc);
            r.n_batches = n;
            int o = 0;
            for (auto& so : s.out) {
                if (!so.on) continue;
                if (!resident && n > 0 && so.restart) {
                    so.start = r.s0;
                    so.restart = false;
                }
                r.lead[o] = (int32_t)std::min<long long>(r.s0 - (resident ? 0 : so.start), 1ll << 30);
                r.ring_pos0[o] = queue_outputs && n > 0 ? so.q.queue(n, d.batch_seq, ri, so.decim) : -1;
                o++;
            }
            max_items = std::max(max_items, n * abg_subband_chunks(B * d.hop));
        });
        rc = monitor_launch(e, e->subband, max_items, [&](int n_devices, int items, cudaStream_t s) {
            SbArgs A{};
            A.cfg = e->subband.cfg.p; A.run = e->subband.run.p;
            return abg_launch_subband(A, n_devices, items, e->subband.max_hist, s);
        });
        if (rc != ABG_OK) return rc;
        max_items = 0;
        monitor_runs(e, e->activity, nb, [&](ActRun& r, ActDev& s, Device& d, int n) {
            r.raw = resident ? d.res : d.raw[d.cur];
            r.first_byte = run_first_byte(d, resident);
            r.first_frame = (unsigned long long)ABG_AGC_EXTRA + d.batch_seq * (unsigned long long)B;
            queue_run(r, s.q, n, d.batch_seq, 0);
            max_items = std::max(max_items, n);
        });
        rc = monitor_launch(e, e->activity, max_items, [&](int n_devices, int items, cudaStream_t s) {
            ActArgs A{};
            A.cfg = e->activity.cfg.p; A.run = e->activity.run.p; A.tw1 = e->tw1.p; A.tw2 = e->tw2.p; A.wave_batch = B;
            return abg_launch_activity(N, A, n_devices, items, s);
        });
        if (rc != ABG_OK) return rc;
        // the I/Q history's append: the run's samples [s0, s0 + n) of every device with the history on, at most the last
        // ring-full of them.  Resident runs append from the replay buffer at its own offsets and leave the history empty.
        unsigned long long max_bytes = 0;
        monitor_runs(e, e->history, nb, [&](HiRun& r, HiDev& h, Device& d, int n) {
            const unsigned long long first_byte = run_first_byte(d, resident);
            const unsigned long long stream_byte = (resident ? 0ull : (unsigned long long)d.dropped) + first_byte;
            const unsigned long long bytes = (unsigned long long)n * B * d.hop_bytes, R = h.ring.n;
            const unsigned long long skip = bytes > R ? bytes - R : 0;
            r.src = (resident ? d.res : d.raw[d.cur]) + first_byte + skip;
            r.dst = (stream_byte + skip) % R;
            r.n_bytes = bytes - skip;
            max_bytes = std::max(max_bytes, r.n_bytes);
            if (n == 0) return;
            if (resident) {
                h.first = h.end = 0;
                return;
            }
            const unsigned long long s0 = stream_byte / d.bpc;
            if (h.first == h.end || s0 != h.end) h.first = s0;
            h.end = s0 + (unsigned long long)n * B * d.hop;
            if (h.end - h.first > h.cap) h.first = h.end - h.cap;
        });
        max_items = max_bytes > 0 ? abg_history_blocks(max_bytes, (int)e->history.devs.size(), e->sm_count) : 0;
        rc = monitor_launch(e, e->history, max_items, [&](int n_devices, int items, cudaStream_t s) {
            HiArgs A{};
            A.cfg = e->history.cfg.p; A.run = e->history.run.p;
            return abg_launch_history_append(A, n_devices, items, s);
        });
        if (rc != ABG_OK) return rc;
    }
    // ---- K2 (stream B, after this run's K1; overlaps the next run's K1) ----
    CU(cudaStreamWaitEvent(sb, e->ev_k1[cur], 0));
    for (size_t i = 0; i < e->dev.size(); i++) {
        e->h_k2[i].n_batches = nb[i];
        e->h_k2[i].fft_size = N;
        e->h_k2[i].spec = e->dev[i].has_afc ? e->dev[i].spec : nullptr;
    }
    {
        const int nl = upload_small(e->d_k2, e->h_k2.data(), sizeof(K2Dev) * e->dev.size(), sb);
        if (nl < 0) return fail(ABG_ECUDA, "K2 parameter upload failed: %s", cudaGetErrorString(cudaGetLastError()));
        e->launches += (uint64_t)nl;
    }
    CU(cudaEventRecord(tl[2], sb));
    K2Launch L2 = e->k2_launch(cur);
    cudaError_t er = abg_launch_k2(L2, sb);
    if (er != cudaSuccess) return fail(ABG_ECUDA, "K2 launch failed: %s", cudaGetErrorString(er));
    e->launches++;
    CU(cudaEventRecord(tl[3], sb));
    // ---- mixers: sums over the just-finished batches, before the tail copy (output.cpp:533-535 -> mixer.cpp) ----
    if (e->n_mixers > 0) {
        MixLaunch M{};
        M.n_mixers = e->n_mixers; M.n_batches = nbrun; M.wave_batch = B; M.P = e->P; M.Gp = e->Gp; M.offsets = e->mix_offsets.p;
        M.inputs = e->mix_inputs.p; M.devs = e->d_k2; M.wout = e->wout.p; M.axc = e->axc.p; M.sums = e->mix_sums.p; M.flags = e->mix_flags.p;
        if (queue_outputs) {
            M.host_sums = e->slots[slot].mix;
            M.host_flags = e->slots[slot].mixflag;
        }
        er = abg_launch_mix(M, sb);
        if (er != cudaSuccess) return fail(ABG_ECUDA, "mixer launch failed: %s", cudaGetErrorString(er));
        e->launches++;
    }
    // ---- tone meter (stream B after K2 and the mixers, pushed and injected batches alike): it reads wout[0, nb*B) before
    // the tail copy below overwrites [0, AGC_EXTRA), and the next run's K2 queues behind it on this stream ----
    {
        ToneMeterLaunch& m = e->tone_meter;
        const int K = (int)m.freqs.size();
        int max_items = 0;
        monitor_runs(e, m, nb, [&](TmRun& r, TmDev& s, Device& d, int n) {
            r.seq0 = d.audio_seq;
            queue_run(r, s.q, n, d.audio_seq, K);
            max_items = std::max(max_items, n);
        });
        const int rc = monitor_launch(e, m, max_items, [&](int, int items, cudaStream_t s) {
            TmArgs A{};
            A.cfg = m.cfg.p; A.run = m.run.p; A.chan_dev = m.chan_dev.p; A.table = m.table.p;
            A.wout = e->wout.p; A.P = e->P; A.wave_batch = B; A.K = K; A.n_cols = m.cols; A.n_chan = m.n_chan;
            for (int k = 0; k < K; k++) A.delta[k] = m.delta[k];
            return abg_launch_tone_meter(A, items, s);
        });
        if (rc != ABG_OK) return rc;
    }
    // ---- results: the end-of-run kernel writes them straight into the pinned slot, then does the consumer's tail copy ----
    K2Export X{};
    if (queue_outputs) {
        Slot& s = e->slots[slot];
        X.host_wout = s.wout;
        X.host_iqout = e->any_iq_out ? reinterpret_cast<float2*>(s.iqout) : nullptr;
        X.host_axc = s.axc;
        X.stride = (size_t)e->nbmax * B;
    }
    er = abg_launch_k2_tail(L2, X, sb);
    if (er != cudaSuccess) return fail(ABG_ECUDA, "export/tail-copy launch failed: %s", cudaGetErrorString(er));
    e->launches++;
    if (queue_outputs) {
        Slot& s = e->slots[slot];
        CU(cudaEventRecord(s.done, sb));
        for (size_t i = 0; i < e->dev.size(); i++)
            for (int b = 0; b < nb[i]; b++) {
                e->dev[i].ready.emplace_back(slot, b);
                s.pending++;
            }
        if (e->n_mixers > 0)
            for (int b = 0; b < nbrun; b++) {
                e->mix_ready.emplace_back(slot, b);
                s.mix_pending += e->n_mixers;
            }
    }
    CU(cudaEventRecord(tl[4], sb));
    CU(cudaEventRecord(e->ev_k2[cur], sb));
    e->tev_valid = true;
    e->run_index++;
    // ---- bookkeeping ----
    for (size_t i = 0; i < e->dev.size(); i++) {
        if (nb[i] <= 0) continue;
        Device& d = e->dev[i];
        if (!resident) d.audio_seq += (uint64_t)nb[i];
        if (skip_k1) {
            // nothing was consumed from the raw stream
        } else if (resident) {
            d.res_primed = true;
        } else {
            const int frames = nb[i] * B + (d.primed ? 0 : ABG_AGC_EXTRA);
            d.consumed += (size_t)frames * d.hop_bytes;
            d.primed = true;
            d.batch_seq += (uint64_t)nb[i];
            d.runs_since_compaction++;
        }
    }
    return ABG_OK;
}

// Room for nbytes more input of device dev at raw[cur] + fill, compacting the buffer first when they do not fit: what
// abg_push does before its copy, and the history replay before its gather.
int ingest_room(abg_engine* e, int dev, size_t nbytes, const char* fn) {
    Device& d = e->dev[dev];
    if (d.fill + nbytes > d.cap) {
        // compact: move the unconsumed tail to the front of the other buffer.  Ingest runs on its own stream so that
        // host->device copies overlap K1; the other buffer may still be read by the most recent K1, so wait for it.
        // keep the copy 16-byte aligned on both sides; with a sub-band output on, keep its filter's history too
        const size_t hist = (size_t)e->subband.dev[dev].hist * d.bpc;
        const size_t keep_from = (d.consumed > hist ? d.consumed - hist : 0) & ~(size_t)15;
        const size_t rem = d.fill - keep_from;
        if (rem + nbytes > d.cap) {
            return fail(ABG_EOVERFLOW, "%s: device %d input buffer overflow (%zu buffered + %zu new > %zu)", fn, dev, d.fill - d.consumed, nbytes, d.cap);
        }
        // the destination buffer was last read by a K1 launched before the previous compaction: with at least one run since
        // then that is run_index-2 or older, so the copy overlaps the K1 that is reading the current buffer right now
        // (the band spectrum, the input meter, the sub-band outputs, the activity detector and the I/Q history's append read
        // the same bytes right after that K1: ev_raw follows the last of them)
        if (d.runs_since_compaction >= 1) {
            if (e->run_index >= 2) {
                CU(cudaStreamWaitEvent(e->stream_c, e->ev_k1[(e->run_index - 2) & 1], 0));
                if (e->ev_raw[0]) CU(cudaStreamWaitEvent(e->stream_c, e->ev_raw[(e->run_index - 2) & 1], 0));
            }
        } else if (e->run_index >= 1) {
            CU(cudaStreamWaitEvent(e->stream_c, e->ev_k1[(e->run_index - 1) & 1], 0));
            if (e->ev_raw[0]) CU(cudaStreamWaitEvent(e->stream_c, e->ev_raw[(e->run_index - 1) & 1], 0));
        }
        d.runs_since_compaction = 0;
        CU(cudaMemcpyAsync(d.raw[d.cur ^ 1], d.raw[d.cur] + keep_from, rem, cudaMemcpyDeviceToDevice, e->stream_c));
        d.cur ^= 1;
        d.fill = rem;
        d.consumed -= keep_from;
        d.dropped += keep_from;
    }
    return ABG_OK;
}

// abg_create; a replay engine (abg_history_replay) splits its K1 groups by the path each device alone would take.
int create_engine(const abg_config* cfg, const abg_options* opt, bool replay_engine, abg_engine** out) {
    if (!cfg || !out) return fail(ABG_EINVAL, "abg_create: null argument");
    *out = nullptr;
    int ndev = 0;
    cudaError_t er = cudaGetDeviceCount(&ndev);
    if (er != cudaSuccess || ndev < 1)
        return fail(ABG_ENODEV, "Unable to find a CUDA device (%s). This engine has no CPU fallback.", er == cudaSuccess ? "device count is 0" : cudaGetErrorString(er));
    abg_engine* e = new abg_engine();
    e->replay_engine = replay_engine;
    if (opt && opt->cuda_device >= 0) {
        e->cuda_dev = opt->cuda_device;
        if (cudaSetDevice(e->cuda_dev) != cudaSuccess) {
            delete e;
            return fail(ABG_ENODEV, "cudaSetDevice(%d) failed", opt->cuda_device);
        }
    } else {
        cudaGetDevice(&e->cuda_dev);
    }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, e->cuda_dev) != cudaSuccess || prop.major != 9 || prop.minor != 0) {
        const int major = prop.major, minor = prop.minor;
        delete e;
        return fail(ABG_ENODEV, "CUDA device has compute capability %d.%d; this library contains sm_90a code only", major, minor);
    }
    e->sm_count = prop.multiProcessorCount;
    int rc = build(e, cfg, opt);
    if (rc != ABG_OK) {
        std::string keep = g_err;
        engine_free(e);
        g_err = keep;
        return rc;
    }
    *out = e;
    return ABG_OK;
}

}  // namespace

// =========================================================================================================================
// C ABI
// =========================================================================================================================
extern "C" {

const char* abg_last_error(void) { return g_err.c_str(); }
const char* abg_version(void) { return "airband-b200 0.1 (sm_90a)"; }

int abg_create(const abg_config* cfg, const abg_options* opt, abg_engine** out) { return create_engine(cfg, opt, false, out); }

void abg_destroy(abg_engine* e) { engine_free(e); }
int abg_wave_batch(const abg_engine* e) { return e->B; }
int abg_hop(const abg_engine* e, int dev) { return (dev < 0 || dev >= (int)e->dev.size()) ? ABG_ERANGE : e->dev[dev].hop; }

int abg_push(abg_engine* e, int dev, const void* iq, size_t nbytes) {
    if (dev < 0 || dev >= (int)e->dev.size()) return fail(ABG_ERANGE, "abg_push: device %d out of range", dev);
    Device& d = e->dev[dev];
    if (nbytes == 0) return ABG_OK;
    if (nbytes % d.bpc) return fail(ABG_EINVAL, "abg_push: %zu bytes is not a whole number of complex samples", nbytes);
    cudaSetDevice(e->cuda_dev);
    const int rc = ingest_room(e, dev, nbytes, "abg_push");
    if (rc != ABG_OK) return rc;
    CU(cudaMemcpyAsync(d.raw[d.cur] + d.fill, iq, nbytes, cudaMemcpyHostToDevice, e->stream_c));
    e->ingest_dirty = true;
    d.fill += nbytes;
    return ABG_OK;
}

int abg_batches_available(const abg_engine* e, int dev) {
    if (dev < 0 || dev >= (int)e->dev.size()) return ABG_ERANGE;
    const Device& d = e->dev[dev];
    const int frames = frames_available(e, d, d.fill, d.consumed) - (d.primed ? 0 : ABG_AGC_EXTRA);
    return frames <= 0 ? 0 : frames / e->B;
}

int abg_run(abg_engine* e, int max_batches) {
    cudaSetDevice(e->cuda_dev);
    if (max_batches < 0 || max_batches > e->nbmax) max_batches = e->nbmax;
    // AFC moves bins[] between batches (rtl_airband.cpp:629): with any AFC channel the run advances one batch at a
    // time so that K1 of batch k+1 sees the bins K2 chose at the end of batch k.
    // (only the AFC devices: the others still advance by up to max_batches in the same run)
    std::vector<int> nb(e->dev.size());
    for (size_t i = 0; i < e->dev.size(); i++) nb[i] = std::min(e->dev[i].has_afc ? 1 : max_batches, abg_batches_available(e, (int)i));
    int n = 0;
    int rc = enqueue_run(e, nb, false, true, &n);
    return rc != ABG_OK ? rc : n;
}

int abg_sync(abg_engine* e) {
    cudaSetDevice(e->cuda_dev);
    CU(cudaStreamSynchronize(e->stream_c));
    CU(cudaStreamSynchronize(e->stream));
    CU(cudaStreamSynchronize(e->stream_b));
    if (e->tc_status && e->tc_status[0]) return fail(ABG_ECUDA, "tensor-core K1 pipeline stalled (wait code %d); results of that run are invalid", e->tc_status[0]);
    return ABG_OK;
}

int abg_join(abg_engine* e) {
    cudaSetDevice(e->cuda_dev);
    if (e->run_index > 0) CU(cudaStreamWaitEvent(e->stream, e->ev_k2[(e->run_index - 1) & 1], 0));
    return ABG_OK;
}

int abg_batches_ready(abg_engine* e, int dev) {
    if (dev < 0 || dev >= (int)e->dev.size()) return ABG_ERANGE;
    return (int)e->dev[dev].ready.size();
}

int abg_fetch_batch(abg_engine* e, int dev, float* waveout, float* iq_out, char* axcindicate) {
    if (dev < 0 || dev >= (int)e->dev.size()) return fail(ABG_ERANGE, "abg_fetch_batch: device %d out of range", dev);
    Device& d = e->dev[dev];
    if (d.ready.empty()) return 0;
    const std::pair<int, int> r = d.ready.front();
    Slot& s = e->slots[r.first];
    cudaSetDevice(e->cuda_dev);
    CU(cudaEventSynchronize(s.done));
    if (e->tc_status && e->tc_status[0]) return fail(ABG_ECUDA, "tensor-core K1 pipeline stalled (wait code %d); results of that run are invalid", e->tc_status[0]);
    const int B = e->B;
    const size_t stride = (size_t)e->nbmax * B;
    for (int c = 0; c < d.C; c++) {
        const size_t g = (size_t)d.g0 + c;
        if (waveout) memcpy(waveout + (size_t)c * B, s.wout + g * stride + (size_t)r.second * B, sizeof(float) * B);
        if (iq_out) {
            if (s.iqout)
                memcpy(iq_out + (size_t)c * 2 * B, s.iqout + 2 * (g * stride + (size_t)r.second * B), sizeof(float) * 2 * B);
            else
                memset(iq_out + (size_t)c * 2 * B, 0, sizeof(float) * 2 * B);
        }
        if (axcindicate) axcindicate[c] = (char)s.axc[(size_t)r.second * e->Gp + g];
    }
    d.ready.pop_front();
    s.pending--;
    return 1;
}

int abg_fetch_batches(abg_engine* e, int dev, int max_batches, float* waveout, float* iq_out, char* axcindicate) {
    if (dev < 0 || dev >= (int)e->dev.size()) return fail(ABG_ERANGE, "abg_fetch_batches: device %d out of range", dev);
    const Device& d = e->dev[dev];
    const size_t C = (size_t)d.C, B = (size_t)e->B;
    int n = 0;
    while (n < max_batches) {
        int rc = abg_fetch_batch(e, dev, waveout ? waveout + (size_t)n * C * B : nullptr, iq_out ? iq_out + (size_t)n * C * 2 * B : nullptr,
                                 axcindicate ? axcindicate + (size_t)n * C : nullptr);
        if (rc < 0) return rc;
        if (rc == 0) break;
        n++;
    }
    return n;
}

int abg_get_stats(abg_engine* e, int dev, int chan, abg_squelch_stats* out) {
    if (dev < 0 || dev >= (int)e->dev.size()) return fail(ABG_ERANGE, "abg_get_stats: device %d out of range", dev);
    Device& d = e->dev[dev];
    if (chan < 0 || chan >= d.C || !out) return fail(ABG_ERANGE, "abg_get_stats: channel %d out of range", chan);
    cudaSetDevice(e->cuda_dev);
    CU(cudaStreamSynchronize(e->stream));
    CU(cudaStreamSynchronize(e->stream_b));
    ChanState s;
    int32_t bin;
    CU(cudaMemcpy(&s, e->state.p + d.g0 + chan, sizeof(s), cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&bin, e->bins.p + d.g0 + chan, sizeof(bin), cudaMemcpyDeviceToHost));
    out->noise_level = s.noise_floor;
    out->signal_level = s.pre_full;
    // Squelch::squelch_level(), squelch.cpp:164-177 (read-only evaluation)
    if (s.manual)
        out->squelch_level = s.manual_level;
    else if (s.level_cache != 0.0f)
        out->squelch_level = s.level_cache;
    else
        out->squelch_level = ((s.recent_open_count >= 3u && s.flappy_ratio < s.normal_ratio) ? s.flappy_ratio : s.normal_ratio) * s.noise_floor;
    out->open_count = s.open_count;
    out->flappy_count = s.flappy_count;
    out->ctcss_count = s.ct_found[1];
    out->no_ctcss_count = s.ct_not_found[1];
    out->agcavgfast = s.agcavgfast;
    out->dm_phi = s.dm_phi;
    out->bin = bin;
    out->active_counter = s.active_counter;
    // level_to_dBFS(), util.cpp:169-180: min(0, 20*log10f(level / fft_size) + 7.54f + 10*log10f(fft_size / 2) - 2.38f)
    const size_t fft_size = (size_t)e->N;
    const float offset = 7.54f + 10.0f * log10f(fft_size / 2) - 2.38f;
    auto to_dbfs = [&](float level) { return std::min(0.0f, 20.0f * log10f(level / fft_size) + offset); };
    out->noise_level_dbfs = to_dbfs(out->noise_level);
    out->signal_level_dbfs = to_dbfs(out->signal_level);
    out->squelch_level_dbfs = to_dbfs(out->squelch_level);
    return ABG_OK;
}

int abg_set_bin(abg_engine* e, int dev, int chan, int bin) {
    if (dev < 0 || dev >= (int)e->dev.size()) return fail(ABG_ERANGE, "abg_set_bin: device %d out of range", dev);
    Device& d = e->dev[dev];
    if (chan < 0 || chan >= d.C) return fail(ABG_ERANGE, "abg_set_bin: channel %d out of range", chan);
    if (bin < 0 || bin >= e->N) return fail(ABG_EINVAL, "abg_set_bin: bin %d outside 0..%d", bin, e->N - 1);
    cudaSetDevice(e->cuda_dev);
    CU(cudaStreamSynchronize(e->stream_b));
    int32_t v = bin;
    CU(cudaMemcpyAsync(e->bins.p + d.g0 + chan, &v, sizeof(v), cudaMemcpyHostToDevice, e->stream));
    CU(cudaMemcpyAsync(e->base_bins.p + d.g0 + chan, &v, sizeof(v), cudaMemcpyHostToDevice, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    e->h_bins[d.g0 + chan] = bin;
    Group& g = e->groups[d.group];
    if (g.use_tc) return rebuild_tc_tables(e, g);  // the coefficient table carries the bin
    return ABG_OK;
}

int abg_fft_path(const abg_engine* e, int dev) {
    if (dev < 0 || dev >= (int)e->dev.size()) return ABG_ERANGE;
    const Group& g = e->groups[e->dev[dev].group];
    return g.use_tc ? 3 : (g.pruned ? 2 : 1);
}

// ---- band spectrum monitor (definition in airband_b200.h) -------------------------------------------------------------
int abg_spectrum_configure(abg_engine* e, int dev, int frame_stride) {
    SpecDev* d = monitor_dev(e, e->spectrum, dev, __func__);
    if (!d) return ABG_ERANGE;
    if (frame_stride < 0) return fail(ABG_EINVAL, "abg_spectrum_configure: frame_stride %d is negative", frame_stride);
    if (frame_stride == d->stride) return ABG_OK;
    int rc = monitor_configure(e, e->spectrum, frame_stride > 0);  // an enqueued spectrum kernel may still use the work buffer
    if (rc != ABG_OK) return rc;
    const int N = e->N, B = e->B, nbmax = e->nbmax;
    d->work.free();
    d->stride = d->n_sel = d->chunks = 0;
    if (frame_stride > 0) {
        if (!d->q.reserve(nbmax, sizeof(float) * N)) return fail(ABG_ENOMEM, "Out of page-locked host memory for the spectrum ring");
        const int n_sel = (B + frame_stride - 1) / frame_stride;
        const int chunks = (n_sel + ABG_SPEC_FPC - 1) / ABG_SPEC_FPC;
        const size_t sums = sizeof(float) * (size_t)nbmax * chunks * N;
        if (d->work.alloc(sums + sizeof(int32_t) * nbmax)) return fail(ABG_ENOMEM, "Out of device memory for the spectrum of device %d", dev);
        CU(cudaMemset(d->work.p + sums, 0, sizeof(int32_t) * nbmax));
        d->stride = frame_stride;
        d->n_sel = n_sel;
        d->chunks = chunks;
    }
    return monitor_publish(e, e->spectrum, [&](const Device& x, const SpecDev& s, SpecCfg& c) -> int {
        c.wsc = e->groups[x.group].wsc.p;
        c.partial = reinterpret_cast<float*>(s.work.p);
        c.counter = reinterpret_cast<int32_t*>(s.work.p + sizeof(float) * (size_t)nbmax * s.chunks * N);
        CU(cudaHostGetDevicePointer((void**)&c.ring, s.q.ring, 0));
        c.hop_bytes = x.hop_bytes; c.sfmt = x.sfmt; c.stride = s.stride; c.n_sel = s.n_sel; c.n_chunks = s.chunks;
        c.ring_cap = s.q.cap;
        return ABG_OK;
    });
}

int abg_fetch_spectrum(abg_engine* e, int dev, float* power, uint64_t* batch_seq, int32_t* n_frames) {
    const unsigned char* src = nullptr;
    MonitorQueue::Entry r{};
    const int rc = monitor_fetch(e, e->spectrum, dev, 0, __func__, &src, &r);
    if (rc <= 0) return rc;
    if (power) memcpy(power, src, sizeof(float) * e->N);
    if (batch_seq) *batch_seq = r.seq;
    if (n_frames) *n_frames = r.aux;
    return 1;
}

int abg_debug_spectrum_time(abg_engine* e, float* ms) { return monitor_time(e, e->spectrum, ms, __func__); }

// ---- carrier frequency meter (definition in airband_b200.h) -----------------------------------------------------------
int abg_carrier_configure(abg_engine* e, int dev, int on) {
    CarDev* d = monitor_dev(e, e->carrier, dev, __func__);
    if (!d) return ABG_ERANGE;
    if (on != 0 && on != 1) return fail(ABG_EINVAL, "abg_carrier_configure: on = %d is neither 0 nor 1", on);
    if ((on == 1) == d->enabled) return ABG_OK;
    const int rc = monitor_configure(e, e->carrier, on == 1);
    if (rc != ABG_OK) return rc;
    if (on && !d->q.reserve(e->nbmax, sizeof(float) * 3 * (size_t)std::max(e->dev[dev].C, 1)))
        return fail(ABG_ENOMEM, "Out of page-locked host memory for the carrier meter ring");
    d->enabled = on == 1;
    return monitor_publish(e, e->carrier, [](const Device& x, const CarDev& s, CarCfg& c) -> int {
        CU(cudaHostGetDevicePointer((void**)&c.ring, s.q.ring, 0));
        c.g0 = x.g0; c.n_channels = x.C; c.ring_cap = s.q.cap;
        return ABG_OK;
    });
}

int abg_fetch_carrier(abg_engine* e, int dev, float* lag1, float* energy, uint64_t* batch_seq) {
    const unsigned char* src = nullptr;
    MonitorQueue::Entry r{};
    const int rc = monitor_fetch(e, e->carrier, dev, 0, __func__, &src, &r);
    if (rc <= 0) return rc;
    const int C = e->dev[dev].C;
    if (lag1) memcpy(lag1, src, sizeof(float) * 2 * C);
    if (energy) memcpy(energy, src + sizeof(float) * 2 * C, sizeof(float) * C);
    if (batch_seq) *batch_seq = r.seq;
    return 1;
}

int abg_debug_carrier_time(abg_engine* e, float* ms) { return monitor_time(e, e->carrier, ms, __func__); }

// ---- input level meter (definition in airband_b200.h) -----------------------------------------------------------------
int abg_input_meter_configure(abg_engine* e, int dev, int on) {
    InmDev* d = monitor_dev(e, e->input_meter, dev, __func__);
    if (!d) return ABG_ERANGE;
    if (on != 0 && on != 1) return fail(ABG_EINVAL, "abg_input_meter_configure: on = %d is neither 0 nor 1", on);
    if ((on == 1) == d->enabled) return ABG_OK;
    int rc = monitor_configure(e, e->input_meter, on == 1);
    if (rc != ABG_OK) return rc;
    const int nbmax = e->nbmax;
    const size_t hist_bytes = sizeof(uint32_t) * 512 * (size_t)nbmax, counter_bytes = sizeof(int32_t) * (size_t)nbmax;
    const size_t part_off = (hist_bytes + counter_bytes + 15) & ~(size_t)15;
    if (on) {
        if (!d->q.reserve(nbmax, sizeof(abg_input_levels))) return fail(ABG_ENOMEM, "Out of page-locked host memory for the input meter ring");
        const int chunks = abg_input_meter_chunks(e->B * e->dev[dev].hop_bytes);
        if (!d->work.p) {
            // histograms and counters start at zero; every launch leaves them at zero again
            if (d->work.alloc(part_off + sizeof(long long) * ABG_INM_PARTIAL * (size_t)nbmax * chunks))
                return fail(ABG_ENOMEM, "Out of device memory for the input meter of device %d", dev);
            CU(cudaMemset(d->work.p, 0, part_off));
        }
        d->chunks = chunks;
    }
    d->enabled = on == 1;
    return monitor_publish(e, e->input_meter, [&](const Device& x, const InmDev& s, InmCfg& c) -> int {
        CU(cudaHostGetDevicePointer((void**)&c.ring, s.q.ring, 0));
        c.hist = reinterpret_cast<uint32_t*>(s.work.p);
        c.counter = reinterpret_cast<int32_t*>(s.work.p + hist_bytes);
        c.partial = reinterpret_cast<long long*>(s.work.p + part_off);
        c.sfmt = x.sfmt; c.hop_bytes = x.hop_bytes; c.n_chunks = s.chunks; c.ring_cap = s.q.cap;
        c.scale = 1.0f / x.fullscale;
        return ABG_OK;
    });
}

int abg_fetch_input_levels(abg_engine* e, int dev, abg_input_levels* out) {
    const unsigned char* src = nullptr;
    MonitorQueue::Entry r{};
    const int rc = monitor_fetch(e, e->input_meter, dev, 0, __func__, &src, &r);
    if (rc <= 0) return rc;
    if (out) {
        memcpy(out, src, sizeof(abg_input_levels));
        out->batch_seq = r.seq;
    }
    return 1;
}

int abg_debug_input_meter_time(abg_engine* e, float* ms) { return monitor_time(e, e->input_meter, ms, __func__); }

// ---- sub-band I/Q outputs (definition in airband_b200.h) ---------------------------------------------------------------
// The arguments of a down-converter that is on (decim >= 1), as abg_subband_configure and abg_history_subband accept them.
static int subband_check(const char* fn, const Device& d, int batch_samples, double offset_hz, int decim, int n_coeffs, const float* coeffs) {
    if (decim < 1 || decim > batch_samples) return fail(ABG_EINVAL, "%s: decimation %d outside [1, %d]", fn, decim, batch_samples);
    if (!std::isfinite(offset_hz) || fabs(offset_hz) > d.sample_rate / 2.0)
        return fail(ABG_EINVAL, "%s: offset %g Hz outside +-sample_rate/2", fn, offset_hz);
    if (n_coeffs < 1 || n_coeffs > ABG_SUBBAND_MAX_COEFFS)
        return fail(ABG_EINVAL, "%s: %d coefficients outside [1, %d]", fn, n_coeffs, ABG_SUBBAND_MAX_COEFFS);
    if (!coeffs) return fail(ABG_EINVAL, "%s: null coefficients", fn);
    for (int j = 0; j < n_coeffs; j++)
        if (!std::isfinite(coeffs[j])) return fail(ABG_EINVAL, "%s: coefficient %d is not finite", fn, j);
    return ABG_OK;
}

// delta = llround(offset / fs * 2^32) mod 2^32; g[j] = h[j] exp(+2 pi i delta j / 2^32) in double, then float32
static uint32_t subband_coefficients(double offset_hz, int sample_rate, int n_coeffs, const float* coeffs, std::vector<float2>& g) {
    const uint32_t delta = (uint32_t)(unsigned long long)llround(offset_hz / sample_rate * 4294967296.0);
    g.resize(n_coeffs);
    for (int j = 0; j < n_coeffs; j++) {
        const double turns = (double)(int32_t)(delta * (uint32_t)j) * 0x1p-32;  // exact, in [-1/2, 1/2)
        const double a = 2.0 * M_PI * turns;
        g[j] = make_float2((float)(coeffs[j] * cos(a)), (float)(coeffs[j] * sin(a)));
    }
    return delta;
}

int abg_subband_configure(abg_engine* e, int dev, int k, double offset_hz, int decim, int n_coeffs, const float* coeffs) {
    SbDev* s = monitor_dev(e, e->subband, dev, __func__);
    if (!s) return ABG_ERANGE;
    if (k < 0 || k >= ABG_SUBBAND_MAX) return fail(ABG_ERANGE, "abg_subband_configure: output %d out of range [0, %d)", k, ABG_SUBBAND_MAX);
    const Device& d = e->dev[dev];
    const int n = e->B * d.hop;  // samples per batch
    if (decim < 0 || decim > n) return fail(ABG_EINVAL, "abg_subband_configure: decimation %d outside [0, %d]", decim, n);
    if (decim > 0) {
        const int rc = subband_check("abg_subband_configure", d, n, offset_hz, decim, n_coeffs, coeffs);
        if (rc != ABG_OK) return rc;
    }
    SbDev::Output& so = s->out[k];
    if (decim == 0 && !so.on) return ABG_OK;
    const int rc = monitor_configure(e, e->subband, decim > 0);  // an enqueued kernel may still read the coefficients or the ring
    if (rc != ABG_OK) return rc;
    if (decim > 0) {
        std::vector<float2> g;
        const uint32_t delta = subband_coefficients(offset_hz, d.sample_rate, n_coeffs, coeffs, g);
        if (so.coef.n < (size_t)n_coeffs) {
            so.coef.free();
            if (so.coef.alloc(n_coeffs)) return fail(ABG_ENOMEM, "Out of device memory for the sub-band coefficients of device %d", dev);
        }
        CU(cudaMemcpy(so.coef.p, g.data(), sizeof(float2) * n_coeffs, cudaMemcpyHostToDevice));
        if (!so.q.reserve(e->nbmax, sizeof(float2) * (size_t)((n + decim - 1) / decim)))
            return fail(ABG_ENOMEM, "Out of page-locked host memory for the sub-band ring");
        so.decim = decim;
        so.n_coeffs = n_coeffs;
        so.delta = delta;
        so.restart = true;
    }
    so.on = decim > 0;
    s->hist = 0;
    for (const auto& x : s->out)
        if (x.on) s->hist = std::max(s->hist, x.n_coeffs - 1);
    e->subband.max_hist = 0;
    return monitor_publish(e, e->subband, [&](const Device& x, const SbDev& y, SbCfg& c) -> int {
        for (const auto& o : y.out) {
            if (!o.on) continue;
            SbOut& w = c.out[c.n_out++];
            w.coef = o.coef.p;
            CU(cudaHostGetDevicePointer((void**)&w.ring, o.q.ring, 0));
            w.delta = o.delta; w.decim = o.decim; w.n_coeffs = o.n_coeffs;
            w.ring_cap = o.q.cap; w.entry_bytes = (int32_t)o.q.entry_bytes;
        }
        c.sfmt = x.sfmt; c.bpc = x.bpc; c.batch_samples = e->B * x.hop; c.n_chunks = abg_subband_chunks(c.batch_samples);
        c.hist = y.hist;
        c.scale = 1.0f / x.fullscale;
        e->subband.max_hist = std::max(e->subband.max_hist, y.hist);
        return ABG_OK;
    });
}

int abg_fetch_subband(abg_engine* e, int dev, int k, float* iq, uint64_t* batch_seq, uint64_t* first_index, int32_t* n_samples) {
    if (k < 0 || k >= ABG_SUBBAND_MAX) return fail(ABG_ERANGE, "abg_fetch_subband: output %d out of range [0, %d)", k, ABG_SUBBAND_MAX);
    const unsigned char* src = nullptr;
    MonitorQueue::Entry r{};
    const int rc = monitor_fetch(e, e->subband, dev, k, __func__, &src, &r);
    if (rc <= 0) return rc;
    const Device& d = e->dev[dev];
    // the batch's outputs: s0 <= mD < s0 + n with D the decimation the batch was computed with
    const unsigned long long n = (unsigned long long)e->B * d.hop, D = (unsigned long long)r.aux;
    const unsigned long long s0 = ((unsigned long long)ABG_AGC_EXTRA + r.seq * e->B) * d.hop;
    const unsigned long long m0 = (s0 + D - 1) / D, m1 = (s0 + n + D - 1) / D;
    if (iq) memcpy(iq, src, sizeof(float2) * (m1 - m0));
    if (batch_seq) *batch_seq = r.seq;
    if (first_index) *first_index = m0;
    if (n_samples) *n_samples = (int32_t)(m1 - m0);
    return 1;
}

int abg_debug_subband_time(abg_engine* e, float* ms) { return monitor_time(e, e->subband, ms, __func__); }

// ---- CTCSS tone meter (definition in airband_b200.h) -------------------------------------------------------------------
// The tone table of the current list: T[j][2k] = cos, T[j][2k+1] = -sin of 2 pi (delta_k j mod 2^32) / 2^32, built in double
// and rounded once to float32; columns 2K .. cols are zero.  The caller has waited for stream B.
static int tone_meter_table(abg_engine* e) {
    ToneMeterLaunch& m = e->tone_meter;
    const int K = (int)m.freqs.size(), B = e->B;
    const int cols = (2 * K + ABG_TM_COLS - 1) / ABG_TM_COLS * ABG_TM_COLS;
    m.delta.resize(K);
    for (int k = 0; k < K; k++)
        m.delta[k] = (uint32_t)(unsigned long long)llround((double)m.freqs[k] / e->W * 4294967296.0);
    std::vector<float> t((size_t)B * cols, 0.0f);
    for (int j = 0; j < B; j++)
        for (int k = 0; k < K; k++) {
            const double turns = (double)(int32_t)(m.delta[k] * (uint32_t)j) * 0x1p-32;  // exact, in [-1/2, 1/2)
            t[(size_t)j * cols + 2 * k] = (float)cos(2.0 * M_PI * turns);
            t[(size_t)j * cols + 2 * k + 1] = (float)-sin(2.0 * M_PI * turns);
        }
    if (cols != m.cols) {
        m.table.free();
        m.cols = 0;
        if (m.table.alloc(t.size())) return fail(ABG_ENOMEM, "Out of device memory for the tone meter table");
        m.cols = cols;
    }
    CU(cudaMemcpy(m.table.p, t.data(), sizeof(float) * t.size(), cudaMemcpyHostToDevice));
    return ABG_OK;
}

int abg_tone_meter_configure(abg_engine* e, int dev, int on) {
    ToneMeterLaunch& m = e->tone_meter;
    TmDev* d = monitor_dev(e, m, dev, __func__);
    if (!d) return ABG_ERANGE;
    if (on != 0 && on != 1) return fail(ABG_EINVAL, "abg_tone_meter_configure: on = %d is neither 0 nor 1", on);
    if ((on == 1) == d->enabled) return ABG_OK;
    int rc = monitor_configure(e, m, on == 1);
    if (rc != ABG_OK) return rc;
    if (on) {
        if (!d->q.reserve(e->nbmax, sizeof(float) * (2 * ABG_TONE_MAX + 2) * (size_t)std::max(e->dev[dev].C, 1)))
            return fail(ABG_ENOMEM, "Out of page-locked host memory for the tone meter ring");
        if (!m.table.p && (rc = tone_meter_table(e)) != ABG_OK) return rc;
    }
    d->enabled = on == 1;
    std::vector<int32_t> chan_dev;  // the channel map
    int32_t k = 0;
    rc = monitor_publish(e, m, [&](const Device& x, const TmDev& s, TmCfg& c) -> int {
        CU(cudaHostGetDevicePointer((void**)&c.ring, s.q.ring, 0));
        c.g0 = x.g0; c.n_channels = x.C; c.first = (int32_t)chan_dev.size(); c.ring_cap = s.q.cap;
        chan_dev.insert(chan_dev.end(), x.C, k++);
        return ABG_OK;
    });
    if (rc != ABG_OK) return rc;
    m.chan_dev.free();
    m.n_chan = 0;
    if (chan_dev.empty()) return ABG_OK;
    if (m.chan_dev.alloc(chan_dev.size())) return fail(ABG_ENOMEM, "Out of device memory for the tone meter tables");
    CU(cudaMemcpy(m.chan_dev.p, chan_dev.data(), sizeof(int32_t) * chan_dev.size(), cudaMemcpyHostToDevice));
    m.n_chan = (int)chan_dev.size();
    return ABG_OK;
}

int abg_tone_meter_set_tones(abg_engine* e, int n_tones, const float* freqs) {
    if (n_tones < 0 || n_tones > ABG_TONE_MAX)
        return fail(ABG_EINVAL, "abg_tone_meter_set_tones: %d tones outside [0, %d]", n_tones, ABG_TONE_MAX);
    std::vector<float> list(std::begin(kStandardTones), std::end(kStandardTones));
    if (freqs && n_tones > 0) {
        list.assign(freqs, freqs + n_tones);
        for (int k = 0; k < n_tones; k++)
            if (!std::isfinite(freqs[k]) || !(freqs[k] > 0.0f) || !((double)freqs[k] < e->W / 2.0))
                return fail(ABG_EINVAL, "abg_tone_meter_set_tones: tone %d (%g Hz) outside (0, %d) Hz", k, (double)freqs[k], e->W / 2);
    }
    cudaSetDevice(e->cuda_dev);
    CU(cudaStreamSynchronize(monitor_stream(e, e->tone_meter)));  // an enqueued meter kernel may still read the table
    e->tone_meter.freqs = list;
    return e->tone_meter.table.p ? tone_meter_table(e) : ABG_OK;
}

int abg_fetch_tone_meter(abg_engine* e, int dev, float* tones, float* energy, int32_t* active, uint64_t* batch_seq, int32_t* n_tones) {
    const unsigned char* src = nullptr;
    MonitorQueue::Entry r{};
    const int rc = monitor_fetch(e, e->tone_meter, dev, 0, __func__, &src, &r);
    if (rc <= 0) return rc;
    const size_t C = (size_t)e->dev[dev].C, K = (size_t)r.aux;
    if (tones) memcpy(tones, src, sizeof(float) * 2 * K * C);
    if (energy) memcpy(energy, src + sizeof(float) * 2 * K * C, sizeof(float) * C);
    if (active) memcpy(active, src + sizeof(float) * (2 * K + 1) * C, sizeof(int32_t) * C);
    if (batch_seq) *batch_seq = r.seq;
    if (n_tones) *n_tones = r.aux;
    return 1;
}

int abg_debug_tone_meter_time(abg_engine* e, float* ms) { return monitor_time(e, e->tone_meter, ms, __func__); }

// ---- band activity detector (definition in airband_b200.h) ----------------------------------------------------------
// The detector settings abg_activity_configure accepts, for abg_activity_configure and abg_history_activity (fn names the
// caller in errors): stride 0 passes here and means off.
static int activity_check(const abg_engine* e, const char* fn, int stride, int hang, int min_span, const float* thr) {
    if (stride < 0 || hang < 0 || min_span < 0)
        return fail(ABG_EINVAL, "%s: negative argument (stride %d, hang %d, min_span %d)", fn, stride, hang, min_span);
    const int N = e->N, B = e->B;
    if (stride > 0) {
        if (stride > B) return fail(ABG_EINVAL, "%s: stride %d exceeds the batch of %d frames", fn, stride, B);
        const int n_sel = (B + stride - 1) / stride;
        if (hang >= n_sel) return fail(ABG_EINVAL, "%s: hang %d is not below the %d selected frames of a batch", fn, hang, n_sel);
        if (min_span < 1) return fail(ABG_EINVAL, "%s: min_span %d is below 1", fn, min_span);
        if (!thr) return fail(ABG_EINVAL, "%s: null thresholds", fn);
        for (int k = 0; k < N; k++)
            if (!std::isfinite(thr[k]) || !(thr[k] > 0.0f))
                return fail(ABG_EINVAL, "%s: threshold of bin %d (%g) is not finite and positive", fn, k, (double)thr[k]);
    }
    return ABG_OK;
}

int abg_activity_configure(abg_engine* e, int dev, int stride, int hang, int min_span, const float* thr) {
    ActDev* d = monitor_dev(e, e->activity, dev, __func__);
    if (!d) return ABG_ERANGE;
    const int rc_check = activity_check(e, __func__, stride, hang, min_span, thr);
    if (rc_check != ABG_OK) return rc_check;
    const int N = e->N, B = e->B;
    if (stride == 0 && d->stride == 0) return ABG_OK;
    const int rc = monitor_configure(e, e->activity, stride > 0);  // an enqueued detector kernel may still read the thresholds
    if (rc != ABG_OK) return rc;
    if (stride > 0) {
        if (!d->q.reserve(e->nbmax, ABG_ACT_HEAD_BYTES + sizeof(abg_burst) * (size_t)ABG_ACTIVITY_MAX_RECORDS))
            return fail(ABG_ENOMEM, "Out of page-locked host memory for the activity ring");
        if (!d->thr.p && d->thr.alloc(N)) return fail(ABG_ENOMEM, "Out of device memory for the activity thresholds of device %d", dev);
        CU(cudaMemcpy(d->thr.p, thr, sizeof(float) * N, cudaMemcpyHostToDevice));
        d->n_sel = (B + stride - 1) / stride;
    }
    d->stride = stride;
    d->hang = stride > 0 ? hang : 0;
    d->min_span = stride > 0 ? min_span : 0;
    return monitor_publish(e, e->activity, [&](const Device& x, const ActDev& s, ActCfg& c) -> int {
        c.wsc = e->groups[x.group].wsc.p;
        c.thr = s.thr.p;
        CU(cudaHostGetDevicePointer((void**)&c.ring, s.q.ring, 0));
        c.hop_bytes = x.hop_bytes; c.sfmt = x.sfmt; c.stride = s.stride; c.n_sel = s.n_sel;
        c.hang = s.hang; c.min_span = s.min_span;
        c.ring_cap = s.q.cap; c.entry_bytes = (int32_t)s.q.entry_bytes;
        return ABG_OK;
    });
}

static_assert(sizeof(abg_burst) == 40, "abg_burst has a fixed 40-byte layout");

int abg_fetch_activity(abg_engine* e, int dev, abg_burst* out, int cap, int32_t* n_stored, int32_t* n_total, uint64_t* batch_seq,
                       int32_t* settings3) {
    if (cap < 0) return fail(ABG_EINVAL, "abg_fetch_activity: cap %d is negative", cap);
    const unsigned char* src = nullptr;
    MonitorQueue::Entry r{};
    const int rc = monitor_fetch(e, e->activity, dev, 0, __func__, &src, &r);
    if (rc <= 0) return rc;
    int32_t head[4];
    memcpy(head, src, sizeof(head));
    const int stored = std::min(head[0], (int32_t)ABG_ACTIVITY_MAX_RECORDS);
    if (out && cap > 0) {
        std::vector<abg_burst> v(stored);
        memcpy(v.data(), src + ABG_ACT_HEAD_BYTES, sizeof(abg_burst) * (size_t)stored);
        std::sort(v.begin(), v.end(), [](const abg_burst& a, const abg_burst& b) {
            return a.bin != b.bin ? a.bin < b.bin : a.first_frame < b.first_frame;
        });
        memcpy(out, v.data(), sizeof(abg_burst) * (size_t)std::min(stored, cap));
    }
    if (n_stored) *n_stored = stored;
    if (n_total) *n_total = head[0];
    if (batch_seq) *batch_seq = r.seq;
    if (settings3) memcpy(settings3, head + 1, sizeof(int32_t) * 3);
    return 1;
}

int abg_debug_activity_time(abg_engine* e, float* ms) { return monitor_time(e, e->activity, ms, __func__); }

// ---- I/Q history (definition in airband_b200.h) ---------------------------------------------------------------------
constexpr long long kHistoryCaptureChunk = 1 << 20;  // outputs per capture launch: the output scratch is 8 MB

int abg_history_configure(abg_engine* e, int dev, int n_batches) {
    HiDev* h = monitor_dev(e, e->history, dev, __func__);
    if (!h) return ABG_ERANGE;
    if (n_batches < 0) return fail(ABG_EINVAL, "abg_history_configure: n_batches %d is negative", n_batches);
    if (n_batches == h->batches) return ABG_OK;
    // a change of capacity empties the history under the device's follow sessions
    for (const auto& s : e->sessions)
        if (s.second.dev == dev)
            return fail(ABG_EINVAL, "abg_history_configure: device %d has open follow sessions (session %d)", dev, (int)s.first);
    int rc = monitor_configure(e, e->history, n_batches > 0);  // an enqueued append or capture may still use the ring
    if (rc != ABG_OK) return rc;
    const Device& d = e->dev[dev];
    h->ring.free();
    h->batches = 0;
    h->cap = h->first = h->end = 0;
    if (n_batches > 0) {
        const unsigned long long cap = (unsigned long long)n_batches * e->B * d.hop;
        const unsigned long long R = (cap * d.bpc + 15) & ~15ull;
        if (h->ring.alloc(R)) {
            rc = fail(ABG_ENOMEM, "Out of device memory for the I/Q history of device %d (%llu bytes)", dev, R);
        } else {
            h->batches = n_batches;
            h->cap = cap;
        }
    }
    const int rp = monitor_publish(e, e->history, [](const Device&, const HiDev& s, HiCfg& c) -> int {
        c.ring = s.ring.p;
        c.ring_bytes = s.ring.n;
        return ABG_OK;
    });
    if (e->history.devs.empty()) {  // nothing left to replay, follow or analyse (no session is open: see above)
        replay_free(e);
        follow_free(e);
        analysis_free(e);
        profile_free(e);
    }
    return rc != ABG_OK ? rc : rp;
}

int abg_history_range(abg_engine* e, int dev, uint64_t* first, uint64_t* end) {
    const HiDev* h = monitor_dev(e, e->history, dev, __func__);
    if (!h) return ABG_ERANGE;
    if (!first || !end) return fail(ABG_EINVAL, "abg_history_range: null argument");
    *first = h->first;
    *end = h->end;
    return ABG_OK;
}

// [first, first + n) inside the device's history (n >= 1)
static bool history_holds(const HiDev& h, unsigned __int128 first, unsigned __int128 n) {
    return h.first < h.end && first >= h.first && first + n <= h.end;
}

int abg_history_raw(abg_engine* e, int dev, uint64_t first, int64_t n, void* out) {
    const HiDev* h = monitor_dev(e, e->history, dev, __func__);
    if (!h) return ABG_ERANGE;
    if (n < 0 || (n > 0 && !out)) return fail(ABG_EINVAL, "abg_history_raw: %lld samples into %p", (long long)n, out);
    if (n == 0) return ABG_OK;
    if (!history_holds(*h, first, (unsigned long long)n))
        return fail(ABG_ERANGE, "abg_history_raw: samples [%llu, +%lld) outside the history [%llu, %llu)", (unsigned long long)first,
                    (long long)n, (unsigned long long)h->first, (unsigned long long)h->end);
    cudaSetDevice(e->cuda_dev);
    // on the K1 stream, behind the appends that wrote them; n <= capacity, so at most one wrap
    const int bpc = e->dev[dev].bpc;
    const unsigned long long R = h->ring.n, b0 = (unsigned long long)first * bpc % R, len = (unsigned long long)n * bpc;
    const unsigned long long len0 = std::min(len, R - b0);
    CU(cudaMemcpyAsync(out, h->ring.p + b0, len0, cudaMemcpyDeviceToHost, e->stream));
    if (len0 < len) CU(cudaMemcpyAsync(static_cast<char*>(out) + len0, h->ring.p, len - len0, cudaMemcpyDeviceToHost, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    return ABG_OK;
}

int abg_history_subband(abg_engine* e, int dev, double offset_hz, int decim, int n_coeffs, const float* coeffs, uint64_t first_m,
                        int64_t n_out, float* iq) {
    HistoryLaunch& m = e->history;
    const HiDev* h = monitor_dev(e, m, dev, __func__);
    if (!h) return ABG_ERANGE;
    const Device& d = e->dev[dev];
    int rc = subband_check("abg_history_subband", d, e->B * d.hop, offset_hz, decim, n_coeffs, coeffs);
    if (rc != ABG_OK) return rc;
    if (n_out < 1 || !iq) return fail(ABG_EINVAL, "abg_history_subband: %lld outputs into %p", (long long)n_out, (void*)iq);
    // every tap in the history: first_m D - (L - 1) >= first and (first_m + n_out - 1) D < end
    const unsigned __int128 D = (unsigned)decim, lo = (unsigned __int128)first_m * D, hi = ((unsigned __int128)first_m + n_out - 1) * D;
    if (h->first == h->end || lo < (unsigned __int128)h->first + (n_coeffs - 1) || hi >= h->end)
        return fail(ABG_ERANGE, "abg_history_subband: outputs [%llu, +%lld) at decimation %d with %d coefficients read samples outside the history [%llu, %llu)",
                    (unsigned long long)first_m, (long long)n_out, decim, n_coeffs, (unsigned long long)h->first, (unsigned long long)h->end);
    std::vector<float2> g;
    const uint32_t delta = subband_coefficients(offset_hz, d.sample_rate, n_coeffs, coeffs, g);
    cudaSetDevice(e->cuda_dev);
    if (!m.out.p) {
        if (m.coef.alloc(ABG_SUBBAND_MAX_COEFFS) || m.out.alloc(kHistoryCaptureChunk)) {
            m.coef.free();
            return fail(ABG_ENOMEM, "Out of device memory for the I/Q history capture");
        }
        for (auto& ev : m.ev) CU(cudaEventCreate(&ev));
    }
    // on the K1 stream: behind every append it reads, and ahead of every later one that would overwrite its samples
    CU(cudaMemcpyAsync(m.coef.p, g.data(), sizeof(float2) * n_coeffs, cudaMemcpyHostToDevice, e->stream));
    HiCapture c{};
    c.ring = h->ring.p; c.ring_bytes = h->ring.n; c.coef = m.coef.p; c.out = m.out.p;
    c.decim = decim; c.n_coeffs = n_coeffs; c.sfmt = d.sfmt; c.delta = delta; c.scale = 1.0f / d.fullscale;
    float total_ms = 0.0f;
    for (long long done = 0; done < n_out;) {
        const long long cnt = std::min<long long>(kHistoryCaptureChunk, n_out - done);
        c.m0 = (long long)(first_m + (uint64_t)done);
        c.n_out = (int32_t)cnt;
        CU(cudaEventRecord(m.ev[0], e->stream));
        const cudaError_t er = abg_launch_history_capture(c, e->stream);
        if (er != cudaSuccess) return fail(ABG_ECUDA, "I/Q history capture launch failed: %s", cudaGetErrorString(er));
        e->launches++;
        CU(cudaEventRecord(m.ev[1], e->stream));
        CU(cudaMemcpyAsync(iq + 2 * done, m.out.p, sizeof(float2) * cnt, cudaMemcpyDeviceToHost, e->stream));
        CU(cudaStreamSynchronize(e->stream));
        float ms = 0.0f;
        CU(cudaEventElapsedTime(&ms, m.ev[0], m.ev[1]));
        total_ms += ms;
        done += cnt;
    }
    m.capture_ms = total_ms;
    return ABG_OK;
}

int abg_debug_history_time(abg_engine* e, float* ms2) {
    if (!ms2) return fail(ABG_EINVAL, "abg_debug_history_time: null argument");
    const int rc = monitor_time(e, e->history, ms2, __func__);
    if (rc != ABG_OK) return rc;
    ms2[1] = e->history.capture_ms;
    return ABG_OK;
}

// ---- history replay (definition in airband_b200.h) ---------------------------------------------------------------------
// The replay engine is a pool of devices, each built for one shape of job (format, full scale, sample rate, channel count,
// AFC, I/Q outputs: what sizes its buffers and picks its K1 path).  A call takes, for every job, an unused pool device of
// its shape; the others get no input and advance no further.  The pool only grows: it is rebuilt, with every device it
// had plus one for each job that found none, only when a call needs more devices of a shape than it holds, because
// freeing device memory waits for the whole GPU.  Otherwise the channels of every pool device are re-resolved (an idle
// device keeps the last channel list it ran) and the state reset to what abg_create leaves.
static int replay_reset(abg_engine* r, const abg_config* c) {
    CU(cudaStreamSynchronize(r->stream_c));
    CU(cudaStreamSynchronize(r->stream));
    CU(cudaStreamSynchronize(r->stream_b));
    std::vector<ChanParams> hp;
    std::vector<ChanState> hs;
    std::vector<int32_t> hb;
    std::vector<float> h_coeff;
    int rc = resolve_channels(r, c, hp, hs, hb, h_coeff);
    if (rc != ABG_OK) return rc;
    if ((rc = upload_channels(r, hp, hs, hb, h_coeff)) != ABG_OK) return rc;
    for (auto& g : r->groups)
        if (g.use_tc && (rc = rebuild_tc_tables(r, g)) != ABG_OK) return rc;
    for (auto& d : r->dev) {
        d.primed = false;
        d.cur = 0;
        d.fill = d.consumed = d.dropped = 0;
        d.runs_since_compaction = 1;
        d.ready.clear();
        d.batch_seq = d.audio_seq = 0;
    }
    for (auto& s : r->slots) s.pending = 0;
    // upload_channels writes on the legacy stream, which the engine's non-blocking streams are not ordered after
    CU(cudaStreamSynchronize(0));
    return ABG_OK;
}

// The pool-device shape of a channel list for device d, after checking what abg_create refuses in it (`who` names the
// list in errors): replay jobs and follow sessions check their lists with it before any engine state is touched.
static int channel_shape(const abg_engine* e, const Device& d, int n_channels, const abg_channel_cfg* channels, const char* who,
                         abg_engine::ReplayDevice* w) {
    const int N = e->N;
    bool afc = false, iq = false;
    for (int c = 0; c < n_channels; c++) {
        const abg_channel_cfg& cc = channels[c];
        char what[96];
        snprintf(what, sizeof(what), "%s.channels[%d]", who, c);
        if (cc.bin < 0 || cc.bin >= N) return fail(ABG_EINVAL, "%s: bin %d outside 0..%d", what, cc.bin, N - 1);
        ChanParams p{};
        ChanState st{};
        std::vector<float> banks[2];
        const int rc = build_freq(e->W, cc, p, st, banks, what);
        if (rc != ABG_OK) return rc;
        afc |= (cc.afc & 0xff) != 0;
        iq |= cc.has_iq_outputs != 0;
    }
    w->sfmt = d.sfmt;
    w->fullscale = d.fullscale;
    w->sample_rate = d.sample_rate;
    w->afc = afc;
    w->iq = iq;
    w->chans.assign(channels, channels + n_channels);
    return ABG_OK;
}

int abg_history_replay(abg_engine* e, int n_jobs, const abg_replay_job* jobs) {
    if (n_jobs < 1 || n_jobs > 65535 || !jobs) return fail(ABG_EINVAL, "abg_history_replay: %d jobs at %p (1 to 65535)", n_jobs, (const void*)jobs);
    const int B = e->B, N = e->N;
    std::vector<abg_engine::ReplayDevice> want(n_jobs);
    for (int j = 0; j < n_jobs; j++) {
        const abg_replay_job& J = jobs[j];
        const HiDev* h = monitor_dev(e, e->history, J.dev, __func__);
        if (!h) return ABG_ERANGE;
        if (J.n_batches < 1 || J.n_channels < 1 || !J.channels || !J.waveout || !J.axcindicate)
            return fail(ABG_EINVAL, "abg_history_replay: job %d: %d batches of %d channels (%p) into waveout %p, axcindicate %p", j, J.n_batches,
                        J.n_channels, (const void*)J.channels, (void*)J.waveout, (void*)J.axcindicate);
        const Device& d = e->dev[J.dev];
        // the samples the replay reads: from S to the end of its last frame, fft_size - hop into the batch after the last
        const unsigned __int128 S = (unsigned __int128)J.first_batch * B * d.hop;
        const unsigned __int128 end = S + (unsigned __int128)(ABG_AGC_EXTRA + (unsigned long long)J.n_batches * B) * d.hop + N - d.hop;
        if (h->first == h->end || S < h->first || end > h->end)
            return fail(ABG_ERANGE, "abg_history_replay: job %d reads samples [%llu, %llu) of device %d, outside its history [%llu, %llu)", j,
                        (unsigned long long)S, (unsigned long long)end, J.dev, (unsigned long long)h->first, (unsigned long long)h->end);
        char who[48];
        snprintf(who, sizeof(who), "abg_history_replay: jobs[%d]", j);
        const int rc = channel_shape(e, d, J.n_channels, J.channels, who, &want[j]);
        if (rc != ABG_OK) return rc;
    }
    // every job to an unused pool device of its shape; the pool grows by the jobs that find none
    std::vector<abg_engine::ReplayDevice> pool = e->replay_pool;
    std::vector<int> slot(n_jobs, -1);
    std::vector<bool> used(pool.size(), false);
    bool grow = !e->replay;
    for (int j = 0; j < n_jobs; j++) {
        for (size_t p = 0; p < pool.size() && slot[j] < 0; p++)
            if (!used[p] && pool[p].same_shape(want[j])) {
                slot[j] = (int)p;
                used[p] = true;
            }
        if (slot[j] < 0) {
            slot[j] = (int)pool.size();
            pool.push_back(want[j]);
            used.push_back(true);
            grow = true;
        }
        pool[slot[j]].chans = want[j].chans;
    }
    std::vector<abg_device_cfg> devs(pool.size());
    for (size_t p = 0; p < pool.size(); p++)
        devs[p] = abg_device_cfg{pool[p].sfmt, pool[p].fullscale, pool[p].sample_rate, (int32_t)pool[p].chans.size(), pool[p].chans.data()};
    const abg_config rc_cfg{N, e->W, e->fm_demod, (int32_t)pool.size(), devs.data()};
    cudaSetDevice(e->cuda_dev);
    int rc;
    if (!grow) {
        rc = replay_reset(e->replay, &rc_cfg);
    } else {
        if (e->replay) engine_free(e->replay);
        e->replay = nullptr;
        e->replay_pool.clear();
        abg_options o{};
        o.cuda_device = e->cuda_dev;
        o.max_batches_per_run = e->nbmax;
        o.fft_mode = e->fft_mode;
        rc = create_engine(&rc_cfg, &o, true, &e->replay);
        if (rc == ABG_OK && !e->replay_ev[0])
            for (auto& ev : e->replay_ev) CU(cudaEventCreate(&ev));
    }
    if (rc != ABG_OK) return rc;
    e->replay_pool = pool;
    cudaSetDevice(e->cuda_dev);
    // upload_small writes whole 16-byte words: one record of room for the rounding
    if (e->replay_gather.n < (size_t)n_jobs + 1) {
        e->replay_gather.free();
        if (e->replay_gather.alloc((size_t)n_jobs + 1)) return fail(ABG_ENOMEM, "Out of device memory for the history replay");
    }
    abg_engine* r = e->replay;
    std::vector<int> done(n_jobs, 0);                       // batches fetched
    std::vector<unsigned long long> pushed(n_jobs, 0);      // bytes gathered
    std::vector<RpGather> g(n_jobs);
    float ms_gather = 0.0f, ms_run = 0.0f;
    for (;;) {
        // the chunk: up to max_batches_per_run more batches of every job (AFC devices advance one batch per run)
        std::vector<int> nb(n_jobs, 0);
        unsigned long long max_bytes = 0;
        int total = 0;
        for (int j = 0; j < n_jobs; j++) {
            const abg_replay_job& J = jobs[j];
            const Device& d = e->dev[J.dev];
            const HiDev& h = e->history.dev[J.dev];
            Device& rd = r->dev[slot[j]];
            nb[j] = std::min(rd.has_afc ? 1 : r->nbmax, J.n_batches - done[j]);
            g[j] = RpGather{h.ring.p, h.ring.n, J.first_batch * B * d.hop * d.bpc + pushed[j], nullptr, 0};
            if (nb[j] == 0) continue;
            // the bytes the fill rule needs for done + nb batches (rtl_airband.cpp:394-400)
            const unsigned long long want_bytes = ((ABG_AGC_EXTRA + (unsigned long long)(done[j] + nb[j]) * B) * d.hop + N) * d.bpc;
            const unsigned long long n = want_bytes - pushed[j];
            if ((rc = ingest_room(r, slot[j], n, "abg_history_replay")) != ABG_OK) return rc;
            g[j].dst = rd.raw[rd.cur] + rd.fill;
            g[j].n_bytes = n;
            rd.fill += n;
            pushed[j] = want_bytes;
            max_bytes = std::max(max_bytes, n);
            total += nb[j];
        }
        if (total == 0) break;
        // the gather on the K1 stream: behind every append it reads, ahead of every later one that would overwrite them
        const int nl = upload_small(e->replay_gather.p, g.data(), sizeof(RpGather) * n_jobs, e->stream);
        if (nl < 0) return fail(ABG_ECUDA, "history replay parameter upload failed: %s", cudaGetErrorString(cudaGetLastError()));
        e->launches += (uint64_t)nl;
        CU(cudaEventRecord(e->replay_ev[0], e->stream));
        const cudaError_t er = abg_launch_replay_gather(e->replay_gather.p, n_jobs, abg_history_blocks(max_bytes, n_jobs, e->sm_count), e->stream);
        if (er != cudaSuccess) return fail(ABG_ECUDA, "history replay gather launch failed: %s", cudaGetErrorString(er));
        e->launches++;
        CU(cudaEventRecord(e->replay_ev[1], e->stream));
        CU(cudaStreamWaitEvent(r->stream, e->replay_ev[1], 0));
        r->ingest_dirty = true;  // and behind any compaction on the replay engine's ingest stream
        const int ran = abg_run(r, -1);
        if (ran < 0) return ran;
        if (ran != total) return fail(ABG_ECUDA, "abg_history_replay: the replay engine ran %d of %d batches", ran, total);
        for (int j = 0; j < n_jobs; j++) {
            const abg_replay_job& J = jobs[j];
            const size_t C = (size_t)J.n_channels, o = (size_t)done[j];
            const int got = abg_fetch_batches(r, slot[j], nb[j], J.waveout + o * C * B, J.iq_out ? J.iq_out + o * C * 2 * B : nullptr,
                                              J.axcindicate + o * C);
            if (got < 0) return got;
            done[j] += got;
        }
        float ms = 0.0f, ms4[4];
        CU(cudaEventElapsedTime(&ms, e->replay_ev[0], e->replay_ev[1]));
        if ((rc = abg_last_run_times(r, ms4)) != ABG_OK) return rc;
        ms_gather += ms;
        ms_run += ms4[3];
    }
    for (int j = 0; j < n_jobs; j++)
        for (int c = 0; jobs[j].stats && c < jobs[j].n_channels; c++)
            if ((rc = abg_get_stats(r, slot[j], c, jobs[j].stats + c)) != ABG_OK) return rc;
    e->replay_ms[0] = ms_gather;
    e->replay_ms[1] = ms_run;
    return ABG_OK;
}

int abg_debug_replay_time(abg_engine* e, float* ms2) {
    if (!ms2) return fail(ABG_EINVAL, "abg_debug_replay_time: null argument");
    ms2[0] = e->replay_ms[0];
    ms2[1] = e->replay_ms[1];
    return ABG_OK;
}

// ---- live follow (definition in airband_b200.h) -------------------------------------------------------------------------
// A session is a replay job without an end, on a device of its own in a follow engine: a private engine built like the
// replay engine (K1 groups split by the path a one-device engine takes), kept apart from it because replay_reset resets
// every device of its pool.  A follow engine is never rebuilt, since that would have to carry every open session's channel
// state across layouts.  A closed session's device goes back to the pool, and the next session of its shape resets only
// that device (follow_reset); a session that finds no free device of its shape gets a new engine with as many devices of
// that shape as exist already, so the number of engines grows logarithmically.
static abg_engine::FollowSession* follow_session(abg_engine* e, int32_t id, const char* fn) {
    const auto it = e->sessions.find(id);
    if (it != e->sessions.end()) return &it->second;
    fail(ABG_ERANGE, "%s: no open follow session %d", fn, (int)id);
    return nullptr;
}

// Device p of follow engine f back to the state a fresh engine with the channel list f.pool[p].chans leaves it in, its
// neighbours untouched: parameters, state, bins and CTCSS banks of its channels, their tone-bank and Squelch delay-line
// columns, their look-back rows in both run parities, its group's tensor-core tables and its ingest bookkeeping.
static int follow_reset(abg_engine::FollowEngine& f, int p) {
    abg_engine* r = f.r;
    CU(cudaStreamSynchronize(r->stream_c));
    CU(cudaStreamSynchronize(r->stream));
    CU(cudaStreamSynchronize(r->stream_b));
    std::vector<abg_device_cfg> devs(f.pool.size());
    for (size_t k = 0; k < f.pool.size(); k++)
        devs[k] = abg_device_cfg{f.pool[k].sfmt, f.pool[k].fullscale, f.pool[k].sample_rate, (int32_t)f.pool[k].chans.size(), f.pool[k].chans.data()};
    const abg_config cfg{r->N, r->W, r->fm_demod, (int32_t)devs.size(), devs.data()};
    std::vector<ChanParams> hp;
    std::vector<ChanState> hs;
    std::vector<int32_t> hb;
    std::vector<float> hc;
    int rc = resolve_channels(r, &cfg, hp, hs, hb, hc);  // the other devices resolve to the lists they were opened with
    if (rc != ABG_OK) return rc;
    Device& d = r->dev[p];
    const int g0 = d.g0, C = d.C, Gp = r->Gp, P = r->P;
    const size_t row = sizeof(float) * Gp, cols = sizeof(float) * C;
    CU(cudaMemcpy(r->params.p + g0, hp.data() + g0, sizeof(ChanParams) * C, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(r->state.p + g0, hs.data() + g0, sizeof(ChanState) * C, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(r->bins.p + g0, hb.data() + g0, sizeof(int32_t) * C, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(r->base_bins.p + g0, hb.data() + g0, sizeof(int32_t) * C, cudaMemcpyHostToDevice));
    CU(cudaMemcpy2D(r->tone_coeff.p + g0, row, hc.data() + g0, row, cols, 2 * ABG_MAX_TONES, cudaMemcpyHostToDevice));
    for (DevBuf<float>* t : {&r->tone_q1, &r->tone_q2, &r->tone_mag}) CU(cudaMemset2D(t->p + g0, row, 0, cols, 2 * ABG_MAX_TONES));
    CU(cudaMemset2D(r->sqbuf.p + g0, row, 0, cols, ABG_SQ_BUF));
    // the AGC look-back rows as upload_channels primes them: win [P][Gp] time-major, wout [Gp][P] channel-major
    std::vector<float> hw((size_t)P * C, 0.0f), ho((size_t)C * P, 0.0f);
    for (int k = 0; k < ABG_AGC_EXTRA; k++)
        for (int c = 0; c < C; c++) {
            hw[(size_t)k * C + c] = 20.0f;
            ho[(size_t)c * P + k] = 0.5f;
        }
    for (int k = 0; k < 2; k++) {
        CU(cudaMemcpy2D(r->win[k].p + g0, row, hw.data(), cols, cols, P, cudaMemcpyHostToDevice));
        CU(cudaMemset2D(r->iqin[k].p + g0, sizeof(float2) * Gp, 0, sizeof(float2) * C, P));
    }
    CU(cudaMemcpy(r->wout.p + (size_t)g0 * P, ho.data(), sizeof(float) * ho.size(), cudaMemcpyHostToDevice));
    if (r->any_iq_out) CU(cudaMemset(r->iqout.p + (size_t)g0 * r->nbmax * r->B, 0, sizeof(float2) * (size_t)C * r->nbmax * r->B));
    Group& g = r->groups[d.group];
    if (g.use_tc && (rc = rebuild_tc_tables(r, g)) != ABG_OK) return rc;  // the coefficient tables carry the bins
    d.primed = false;
    d.cur = 0;
    d.fill = d.consumed = d.dropped = 0;
    d.runs_since_compaction = 1;
    d.ready.clear();
    d.batch_seq = d.audio_seq = 0;
    // the writes above use the legacy stream, which the engine's non-blocking streams are not ordered after
    CU(cudaStreamSynchronize(0));
    return ABG_OK;
}

int abg_follow_open(abg_engine* e, int dev, uint64_t first_batch, int n_channels, const abg_channel_cfg* channels, int queue_batches,
                    int32_t* session) {
    const HiDev* h = monitor_dev(e, e->history, dev, __func__);
    if (!h) return ABG_ERANGE;
    if (n_channels < 1 || !channels || queue_batches < 1 || !session)
        return fail(ABG_EINVAL, "abg_follow_open: %d channels (%p), a queue of %d batches, session %p", n_channels, (const void*)channels,
                    queue_batches, (void*)session);
    if (!h->on()) return fail(ABG_ERANGE, "abg_follow_open: device %d has no history", dev);
    const Device& d = e->dev[dev];
    const unsigned __int128 S = (unsigned __int128)first_batch * e->B * d.hop;
    if (S < h->first || S >= ((unsigned __int128)1 << 63))
        return fail(ABG_ERANGE, "abg_follow_open: a session from batch %llu reads samples from %llu on; device %d's history holds [%llu, %llu)",
                    (unsigned long long)first_batch, (unsigned long long)S, dev, (unsigned long long)h->first, (unsigned long long)h->end);
    abg_engine::ReplayDevice want;
    int rc = channel_shape(e, d, n_channels, channels, "abg_follow_open", &want);
    if (rc != ABG_OK) return rc;
    cudaSetDevice(e->cuda_dev);
    // a free device of the session's shape, or a new follow engine with as many devices of it as exist already
    int fi = -1, p = -1, have = 0;
    for (int k = 0; k < (int)e->follow.size(); k++)
        for (int q = 0; q < (int)e->follow[k].pool.size(); q++) {
            if (!e->follow[k].pool[q].same_shape(want)) continue;
            have++;
            if (fi < 0 && e->follow[k].owner[q] < 0) {
                fi = k;
                p = q;
            }
        }
    if (fi >= 0) {
        abg_engine::FollowEngine& f = e->follow[fi];
        f.pool[p].chans = want.chans;
        if ((rc = follow_reset(f, p)) != ABG_OK) return rc;
    } else {
        const int n = std::max(have, 1);
        abg_engine::FollowEngine f;
        f.pool.assign(n, want);
        f.owner.assign(n, -1);
        std::vector<abg_device_cfg> devs(n, abg_device_cfg{want.sfmt, want.fullscale, want.sample_rate, n_channels, channels});
        const abg_config cfg{e->N, e->W, e->fm_demod, n, devs.data()};
        abg_options o{};
        o.cuda_device = e->cuda_dev;
        o.max_batches_per_run = e->nbmax;
        o.fft_mode = e->fft_mode;
        if ((rc = create_engine(&cfg, &o, true, &f.r)) != ABG_OK) return rc;
        cudaSetDevice(e->cuda_dev);
        if (cudaEventCreateWithFlags(&f.ev_compact, cudaEventDisableTiming) != cudaSuccess) {
            engine_free(f.r);
            return fail(ABG_ECUDA, "abg_follow_open: event creation failed");
        }
        e->follow.push_back(f);
        fi = (int)e->follow.size() - 1;
        p = 0;
    }
    const int32_t id = e->next_session++;
    e->follow[fi].owner[p] = id;
    abg_engine::FollowSession& s = e->sessions[id];
    s.dev = dev;
    s.eng = fi;
    s.slot = p;
    s.C = n_channels;
    s.queue_batches = queue_batches;
    s.first_batch = s.next_batch = first_batch;
    *session = id;
    return ABG_OK;
}

int abg_follow_close(abg_engine* e, int32_t session) {
    abg_engine::FollowSession* s = follow_session(e, session, __func__);
    if (!s) return ABG_ERANGE;
    abg_engine::FollowEngine& f = e->follow[s->eng];
    Device& d = f.r->dev[s->slot];
    for (const auto& x : d.ready) f.r->slots[x.first].pending--;  // its unfetched batches give their result slots back
    d.ready.clear();
    f.owner[s->slot] = -1;
    e->sessions.erase(session);
    return ABG_OK;
}

// Move session s's finished batches out of its follow engine's result slots into its queue, oldest first, until the queue
// holds `until` batches; with only_slot >= 0 only those in that slot.  Waits for the runs that computed them.
static int follow_drain(abg_engine* e, abg_engine::FollowSession& s, int only_slot, size_t until) {
    abg_engine* r = e->follow[s.eng].r;
    Device& d = r->dev[s.slot];
    const size_t B = r->B, C = s.C;
    while (!d.ready.empty() && s.q.size() < until && (only_slot < 0 || d.ready.front().first == only_slot)) {
        abg_engine::FollowBatch b;
        b.wout.resize(C * B);
        b.iq.resize(C * 2 * B);
        b.axc.resize(C);
        const int rc = abg_fetch_batch(r, s.slot, b.wout.data(), b.iq.data(), b.axc.data());
        if (rc < 0) return rc;
        s.q.push_back(std::move(b));
    }
    return ABG_OK;
}

// A (start, end) pair of timing events for the current abg_follow_run: kind 0 = a gather, 1 = a follow-engine run.
static int follow_pair(abg_engine* e, int kind, int* idx) {
    if (e->follow_tev.size() < 2 * (size_t)(e->follow_pairs + 1)) {
        cudaEvent_t ev[2];
        CU(cudaEventCreate(&ev[0]));
        if (cudaEventCreate(&ev[1]) != cudaSuccess) {
            cudaEventDestroy(ev[0]);
            return fail(ABG_ECUDA, "abg_follow_run: event creation failed");
        }
        e->follow_tev.insert(e->follow_tev.end(), ev, ev + 2);
        e->follow_kind.push_back(0);
    }
    e->follow_kind[e->follow_pairs] = kind;
    *idx = 2 * e->follow_pairs++;
    return ABG_OK;
}

int abg_follow_run(abg_engine* e, int max_batches) {
    cudaSetDevice(e->cuda_dev);
    e->follow_pairs = 0;
    if (max_batches == 0 || e->sessions.empty()) return 0;
    const long long budget = max_batches < 0 ? LLONG_MAX : max_batches;
    const int B = e->B, N = e->N;
    std::map<int32_t, long long> advanced;  // batches this call enqueued per session
    int total = 0, rc;
    for (;;) {
        // the chunk: every session's next batches, as far as the history, its queue room, max_batches_per_run (one batch
        // with AFC) and this call's max_batches allow, decided on the host from the enqueued history range
        std::vector<std::vector<int>> nb(e->follow.size());
        for (size_t k = 0; k < e->follow.size(); k++) nb[k].assign(e->follow[k].r->dev.size(), 0);
        std::vector<bool> compacted(e->follow.size(), false);
        std::vector<RpGather> g;
        unsigned long long max_bytes = 0;
        int chunk = 0;
        for (auto& it : e->sessions) {
            abg_engine::FollowSession& s = it.second;
            if (s.lost) continue;
            const Device& d = e->dev[s.dev];
            const HiDev& h = e->history.dev[s.dev];
            if (h.first == h.end) continue;
            const unsigned long long S = s.first_batch * B * d.hop;
            if (h.first > S + s.valid / d.bpc) {  // the history overwrote the next sample the session has not gathered
                s.lost = true;
                continue;
            }
            // batch b is available once (AGC_EXTRA + (b+1)*B)*hop + fft_size - hop <= end: for b < b_end
            const unsigned long long fl = h.end + d.hop >= (unsigned long long)N ? (h.end + d.hop - N) / d.hop : 0;
            const unsigned long long b_end = fl >= (unsigned long long)ABG_AGC_EXTRA ? (fl - ABG_AGC_EXTRA) / B : 0;
            abg_engine::FollowEngine& f = e->follow[s.eng];
            Device& rd = f.r->dev[s.slot];
            const long long room = (long long)s.queue_batches - (long long)(s.q.size() + rd.ready.size());
            const long long n = std::min({b_end > s.next_batch ? (long long)(b_end - s.next_batch) : 0ll, room,
                                          (long long)(rd.has_afc ? 1 : f.r->nbmax), budget - advanced[it.first]});
            if (n <= 0) continue;
            // the bytes the fill rule needs for every batch so far (rtl_airband.cpp:394-400).  Its last hop samples may lie
            // past the history's end; they are never read by these batches, and the next chunk gathers them again.
            const unsigned long long done = s.next_batch - s.first_batch;
            const unsigned long long want = ((ABG_AGC_EXTRA + (done + n) * B) * d.hop + N) * d.bpc;
            const unsigned long long valid = std::min(want, (h.end - S) * d.bpc);
            const size_t dropped = rd.dropped;
            if ((rc = ingest_room(f.r, s.slot, want - s.pushed, "abg_follow_run")) != ABG_OK) return rc;
            if (rd.dropped != dropped) compacted[s.eng] = true;
            g.push_back(RpGather{h.ring.p, h.ring.n, S * d.bpc + s.valid, rd.raw[rd.cur] + rd.fill - (s.pushed - s.valid), want - s.valid});
            max_bytes = std::max(max_bytes, want - s.valid);
            rd.fill += want - s.pushed;
            s.pushed = want;
            s.valid = valid;
            s.next_batch += n;
            advanced[it.first] += n;
            nb[s.eng][s.slot] = (int)n;
            chunk += (int)n;
        }
        if (chunk == 0) break;
        // the gather on the parent's K1 stream: behind every append it reads, ahead of every later one that would overwrite
        // them.  Behind the chunk's compactions too: each waited for the follow engine's K1 that last read the buffer the
        // gather now writes, and moved the bytes the previous chunk left past the history's end, which the gather replaces.
        for (size_t k = 0; k < e->follow.size(); k++)
            if (compacted[k]) {
                CU(cudaEventRecord(e->follow[k].ev_compact, e->follow[k].r->stream_c));
                CU(cudaStreamWaitEvent(e->stream, e->follow[k].ev_compact, 0));
            }
        // upload_small writes whole 16-byte words: one record of room for the rounding
        if (e->follow_gather.n < g.size() + 1) {
            e->follow_gather.free();
            if (e->follow_gather.alloc(2 * g.size() + 1)) return fail(ABG_ENOMEM, "Out of device memory for the live follow");
        }
        const int nl = upload_small(e->follow_gather.p, g.data(), sizeof(RpGather) * g.size(), e->stream);
        if (nl < 0) return fail(ABG_ECUDA, "live follow parameter upload failed: %s", cudaGetErrorString(cudaGetLastError()));
        e->launches += (uint64_t)nl;
        int ig;
        if ((rc = follow_pair(e, 0, &ig)) != ABG_OK) return rc;
        CU(cudaEventRecord(e->follow_tev[ig], e->stream));
        const cudaError_t er = abg_launch_replay_gather(e->follow_gather.p, (int)g.size(), abg_history_blocks(max_bytes, (int)g.size(), e->sm_count), e->stream);
        if (er != cudaSuccess) return fail(ABG_ECUDA, "live follow gather launch failed: %s", cudaGetErrorString(er));
        e->launches++;
        const cudaEvent_t gathered = e->follow_tev[ig + 1];
        CU(cudaEventRecord(gathered, e->stream));
        // one run per follow engine with work; its ingest stream, and so its K1 and later compactions, wait for the gather
        for (size_t k = 0; k < e->follow.size(); k++) {
            if (std::all_of(nb[k].begin(), nb[k].end(), [](int v) { return v == 0; })) continue;
            abg_engine::FollowEngine& f = e->follow[k];
            abg_engine* r = f.r;
            CU(cudaStreamWaitEvent(r->stream_c, gathered, 0));
            r->ingest_dirty = true;
            // the result slot this run exports into: move what it still holds into the sessions' queues
            const int sl = r->next_slot;
            for (size_t q = 0; q < f.owner.size() && r->slots[sl].pending > 0; q++)
                if (f.owner[q] >= 0 && (rc = follow_drain(e, e->sessions[f.owner[q]], sl, SIZE_MAX)) != ABG_OK) return rc;
            int it;
            if ((rc = follow_pair(e, 1, &it)) != ABG_OK) return rc;
            CU(cudaStreamWaitEvent(r->stream, gathered, 0));
            CU(cudaEventRecord(e->follow_tev[it], r->stream));
            int ran = 0;
            if ((rc = enqueue_run(r, nb[k], false, true, &ran)) != ABG_OK) return rc;
            CU(cudaEventRecord(e->follow_tev[it + 1], r->stream_b));
        }
        total += chunk;
    }
    return total;
}

int abg_follow_fetch(abg_engine* e, int32_t session, int max_batches, float* waveout, float* iq_out, char* axcindicate,
                     uint64_t* first_batch) {
    abg_engine::FollowSession* s = follow_session(e, session, __func__);
    if (!s) return ABG_ERANGE;
    if (max_batches < 0 || (max_batches > 0 && (!waveout || !axcindicate)))
        return fail(ABG_EINVAL, "abg_follow_fetch: %d batches into waveout %p, axcindicate %p", max_batches, (void*)waveout, (void*)axcindicate);
    const Device& rd = e->follow[s->eng].r->dev[s->slot];
    const uint64_t first = s->next_batch - (uint64_t)(s->q.size() + rd.ready.size());  // the oldest unfetched batch
    cudaSetDevice(e->cuda_dev);
    const int rc = follow_drain(e, *s, -1, (size_t)max_batches);
    if (rc != ABG_OK) return rc;
    if (s->q.empty() && s->lost)
        return fail(ABG_ERANGE, "abg_follow_fetch: session %d is lost: device %d's history overwrote batch %llu before it was read", (int)session,
                    s->dev, (unsigned long long)s->next_batch);
    const int n = (int)std::min<size_t>((size_t)max_batches, s->q.size());
    const size_t C = s->C, B = e->B;
    for (int k = 0; k < n; k++) {
        const abg_engine::FollowBatch& b = s->q.front();
        memcpy(waveout + k * C * B, b.wout.data(), sizeof(float) * C * B);
        if (iq_out) memcpy(iq_out + k * C * 2 * B, b.iq.data(), sizeof(float) * C * 2 * B);
        memcpy(axcindicate + k * C, b.axc.data(), C);
        s->q.pop_front();
    }
    if (first_batch) *first_batch = first;
    return n;
}

int abg_follow_info(abg_engine* e, int32_t session, abg_follow_status* out) {
    const abg_engine::FollowSession* s = follow_session(e, session, __func__);
    if (!s) return ABG_ERANGE;
    if (!out) return fail(ABG_EINVAL, "abg_follow_info: null argument");
    out->dev = s->dev;
    out->n_channels = s->C;
    out->next_batch = s->next_batch;
    out->queued = (int32_t)(s->q.size() + e->follow[s->eng].r->dev[s->slot].ready.size());
    out->lost = s->lost ? 1 : 0;
    return ABG_OK;
}

int abg_follow_stats(abg_engine* e, int32_t session, int chan, abg_squelch_stats* out) {
    const abg_engine::FollowSession* s = follow_session(e, session, __func__);
    if (!s) return ABG_ERANGE;
    if (chan < 0 || chan >= s->C) return fail(ABG_ERANGE, "abg_follow_stats: channel %d out of range", chan);
    if (!out) return fail(ABG_EINVAL, "abg_follow_stats: null argument");
    return abg_get_stats(e->follow[s->eng].r, s->slot, chan, out);
}

int abg_debug_follow_time(abg_engine* e, float* ms2) {
    if (!ms2) return fail(ABG_EINVAL, "abg_debug_follow_time: null argument");
    ms2[0] = ms2[1] = 0.0f;
    cudaSetDevice(e->cuda_dev);
    for (int k = 0; k < e->follow_pairs; k++) {
        float ms = 0.0f;
        CU(cudaEventSynchronize(e->follow_tev[2 * k + 1]));
        CU(cudaEventElapsedTime(&ms, e->follow_tev[2 * k], e->follow_tev[2 * k + 1]));
        ms2[e->follow_kind[k]] += ms;
    }
    return ABG_OK;
}

// ---- history analysis (definition in airband_b200.h) ---------------------------------------------------------------------
// A job is a run of units of one device, spectrogram rows or detector batches: unit u starts at frame base + u*step and
// selects n_sel frames `stride` apart.  A call is cut into chunks of whole units within fixed budgets.  Per chunk, the
// replay gather copies each job's share of the window from its history ring into the scratch buffer, at the stream byte's
// offset modulo 16 (the alignment the live raw buffer gives it), and one launch of the live monitor's kernel reads it there.
constexpr size_t kAnalysisScratch = 64ull << 20;  // gathered bytes per chunk: a 10 s window of one cfg2 device is 51 MB
constexpr size_t kAnalysisWork = 64ull << 20;     // spectrum chunk sums per chunk
constexpr size_t kAnalysisResult = 32ull << 20;   // page-locked results per chunk: rows of fft_size floats, detector entries of 160 KB
constexpr int kAnalysisMaxUnits = 65535;          // rows of a spectrum launch (its grid.y), pieces of a detector launch

struct AnJob {
    int dev;
    unsigned __int128 base;    // frames
    unsigned long long step;   // frames
    int n_units, n_sel, stride;
    size_t unit_result, unit_work;  // bytes per unit
};
struct AnPiece {  // units [u0, u0 + n) of job `job`: stream bytes [src, src + bytes) at scratch offset off
    int job, u0, n;
    unsigned long long src, off, bytes;
};

static size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

// The samples units [u0, u0 + n) of job J read: [*first, *end).  128 bits, so that a window far past the history is
// refused rather than wrapped.
static void analysis_span(const abg_engine* e, const AnJob& J, long long u0, long long n, unsigned __int128* first, unsigned __int128* end) {
    const unsigned hop = (unsigned)e->dev[J.dev].hop;
    const unsigned __int128 f0 = J.base + (unsigned __int128)u0 * J.step;
    *first = f0 * hop;
    *end = (f0 + (unsigned __int128)(n - 1) * J.step + (unsigned __int128)(J.n_sel - 1) * J.stride) * hop + (unsigned)e->N;
}

static int analysis_window(abg_engine* e, const char* fn, int j, const AnJob& J) {
    const HiDev& h = e->history.dev[J.dev];
    unsigned __int128 lo, hi;
    analysis_span(e, J, 0, J.n_units, &lo, &hi);
    if (h.first == h.end || lo < h.first || hi > h.end)
        return fail(ABG_ERANGE, "%s: job %d reads samples [%llu, %llu) of device %d, outside its history [%llu, %llu)", fn, j,
                    (unsigned long long)lo, (unsigned long long)hi, J.dev, (unsigned long long)h.first, (unsigned long long)h.end);
    return ABG_OK;
}

// Buffers for chunks of the jobs' units (they only grow, each to its budget or to the largest single unit), the events,
// and the times reset.
static int analysis_prepare(abg_engine* e, const std::vector<AnJob>& jobs, size_t* scratch_cap, size_t* work_cap, size_t* result_cap) {
    auto& a = e->analysis;
    size_t sc = kAnalysisScratch, wk = kAnalysisWork, rs = kAnalysisResult;
    for (const AnJob& J : jobs) {
        unsigned __int128 lo, hi;
        analysis_span(e, J, 0, 1, &lo, &hi);
        sc = std::max(sc, (size_t)(hi - lo) * e->dev[J.dev].bpc + 32);
        wk = std::max(wk, J.unit_work);
        rs = std::max(rs, J.unit_result);
    }
    cudaSetDevice(e->cuda_dev);
    if (!a.ev[0])
        for (auto& ev : a.ev) CU(cudaEventCreate(&ev));
    if (a.scratch.n < sc) {
        a.scratch.free();
        if (a.scratch.alloc(sc)) return fail(ABG_ENOMEM, "Out of device memory for the history analysis scratch (%zu bytes)", sc);
    }
    const size_t counters = sizeof(int32_t) * kAnalysisMaxUnits;
    if (a.work.n < wk + counters) {
        a.work.free();
        if (a.work.alloc(wk + counters)) return fail(ABG_ENOMEM, "Out of device memory for the history analysis sums (%zu bytes)", wk);
        CU(cudaMemsetAsync(a.work.p + wk, 0, counters, e->stream));
    }
    if (a.result_bytes < rs) {
        if (a.result) cudaFreeHost(a.result);
        a.result = nullptr;
        a.result_bytes = 0;
        if (cudaHostAlloc((void**)&a.result, rs, cudaHostAllocMapped) != cudaSuccess) {
            cudaGetLastError();
            a.result = nullptr;
            return fail(ABG_ENOMEM, "Out of page-locked host memory for the history analysis results (%zu bytes)", rs);
        }
        a.result_bytes = rs;
    }
    *scratch_cap = a.scratch.n;
    *work_cap = a.work.n - counters;
    *result_cap = a.result_bytes;
    a.ms[0] = a.ms[1] = a.ms[2] = 0.0f;
    return ABG_OK;
}

// Cut the jobs' units into chunks, in job and unit order, and call run(pieces) for each: a chunk's gathered bytes, results
// and spectrum sums stay within the buffers, its units and pieces within kAnalysisMaxUnits.
static int analysis_chunks(abg_engine* e, const std::vector<AnJob>& jobs, const std::function<int(const std::vector<AnPiece>&)>& run) {
    size_t scratch_cap, work_cap, result_cap;
    int rc = analysis_prepare(e, jobs, &scratch_cap, &work_cap, &result_cap);
    if (rc != ABG_OK) return rc;
    std::vector<AnPiece> ps;
    size_t used_res = 0, used_work = 0;
    int units = 0;
    for (int j = 0; j < (int)jobs.size(); j++) {
        const AnJob& J = jobs[j];
        const int bpc = e->dev[J.dev].bpc;
        for (int u = 0; u < J.n_units; u++) {
            for (;;) {
                const bool extend = !ps.empty() && ps.back().job == j;
                AnPiece p = extend ? ps.back() : AnPiece{j, u, 0, 0, 0, 0};
                unsigned __int128 lo, hi;
                analysis_span(e, J, p.u0, p.n + 1, &lo, &hi);
                p.n++;
                p.src = (unsigned long long)lo * bpc;
                p.bytes = (unsigned long long)(hi - lo) * bpc;
                if (!extend) p.off = align16(ps.empty() ? 0 : ps.back().off + ps.back().bytes) + p.src % 16;
                const bool fits = p.off + p.bytes <= scratch_cap && used_res + J.unit_result <= result_cap &&
                                  used_work + J.unit_work <= work_cap && units < kAnalysisMaxUnits;
                if (fits || ps.empty()) {  // (a unit alone always fits: the buffers were sized for it)
                    if (extend)
                        ps.back() = p;
                    else
                        ps.push_back(p);
                    used_res += J.unit_result;
                    used_work += J.unit_work;
                    units++;
                    break;
                }
                if ((rc = run(ps)) != ABG_OK) return rc;
                ps.clear();
                used_res = used_work = 0;
                units = 0;
            }
        }
    }
    return ps.empty() ? ABG_OK : run(ps);
}

// One chunk on the K1 stream: the upload of its records, the gather of every piece into the scratch (behind every append
// it reads, ahead of every later one that would overwrite its bytes), then kernel(device tables, stream).  fill(host
// tables) writes `tables` bytes of kernel records first.  Waits for the chunk and adds the gather's device time to ms[0],
// the kernel's to ms[which].
static int analysis_launch(abg_engine* e, const std::vector<AnJob>& jobs, const std::vector<AnPiece>& ps, size_t tables, int which,
                           const std::function<void(unsigned char*)>& fill,
                           const std::function<cudaError_t(unsigned char*, cudaStream_t)>& kernel) {
    auto& a = e->analysis;
    const size_t gb = align16(sizeof(RpGather) * ps.size()), need = gb + tables;
    if (a.table.n < need) {
        a.table.free();
        if (a.table.alloc(2 * need)) return fail(ABG_ENOMEM, "Out of device memory for the history analysis tables");
    }
    if (a.h_table_bytes < need) {
        if (a.h_table) cudaFreeHost(a.h_table);
        a.h_table_bytes = 0;
        if (cudaHostAlloc((void**)&a.h_table, 2 * need, cudaHostAllocDefault) != cudaSuccess) {
            cudaGetLastError();
            a.h_table = nullptr;
            return fail(ABG_ENOMEM, "Out of page-locked host memory for the history analysis tables");
        }
        a.h_table_bytes = 2 * need;
    }
    RpGather* g = reinterpret_cast<RpGather*>(a.h_table);
    unsigned long long max_bytes = 0;
    for (size_t i = 0; i < ps.size(); i++) {
        const HiDev& h = e->history.dev[jobs[ps[i].job].dev];
        g[i] = RpGather{h.ring.p, h.ring.n, ps[i].src, a.scratch.p + ps[i].off, ps[i].bytes};
        max_bytes = std::max(max_bytes, ps[i].bytes);
    }
    fill(a.h_table + gb);
    const cudaStream_t s = e->stream;
    CU(cudaMemcpyAsync(a.table.p, a.h_table, need, cudaMemcpyHostToDevice, s));
    CU(cudaEventRecord(a.ev[0], s));
    cudaError_t er = abg_launch_replay_gather(reinterpret_cast<const RpGather*>(a.table.p), (int)ps.size(),
                                              abg_history_blocks(max_bytes, (int)ps.size(), e->sm_count), s);
    if (er != cudaSuccess) return fail(ABG_ECUDA, "history analysis gather launch failed: %s", cudaGetErrorString(er));
    e->launches++;
    CU(cudaEventRecord(a.ev[1], s));
    er = kernel(a.table.p + gb, s);
    if (er != cudaSuccess) return fail(ABG_ECUDA, "history analysis %s launch failed: %s", which == 1 ? "spectrum" : "detector", cudaGetErrorString(er));
    e->launches++;
    CU(cudaEventRecord(a.ev[2], s));
    CU(cudaStreamSynchronize(s));
    float ms = 0.0f;
    CU(cudaEventElapsedTime(&ms, a.ev[0], a.ev[1]));
    a.ms[0] += ms;
    CU(cudaEventElapsedTime(&ms, a.ev[1], a.ev[2]));
    a.ms[which] += ms;
    return ABG_OK;
}

int abg_history_spectrogram(abg_engine* e, int n_jobs, const abg_spectrogram_job* jobs) {
    if (n_jobs < 1 || n_jobs > 65535 || !jobs)
        return fail(ABG_EINVAL, "abg_history_spectrogram: %d jobs at %p (1 to 65535)", n_jobs, (const void*)jobs);
    const int N = e->N;
    std::vector<AnJob> an(n_jobs);
    for (int j = 0; j < n_jobs; j++) {
        const abg_spectrogram_job& J = jobs[j];
        if (!monitor_dev(e, e->history, J.dev, __func__)) return ABG_ERANGE;
        const int F = J.frames_per_row, s = J.stride;
        if (J.n_rows < 1 || F < 1 || s < 1 || s > F || !J.power)
            return fail(ABG_EINVAL, "abg_history_spectrogram: job %d: %d rows of %d frames at stride %d into %p", j, J.n_rows, F, s, (void*)J.power);
        const int n_sel = (F + s - 1) / s, chunks = (n_sel + ABG_SPEC_FPC - 1) / ABG_SPEC_FPC;
        an[j] = AnJob{J.dev, J.first_frame, (unsigned long long)F, J.n_rows, n_sel, s, sizeof(float) * N,
                      chunks > 1 ? sizeof(float) * (size_t)chunks * N : 0};
        const int rc = analysis_window(e, __func__, j, an[j]);
        if (rc != ABG_OK) return rc;
    }
    auto& a = e->analysis;
    return analysis_chunks(e, an, [&](const std::vector<AnPiece>& ps) -> int {
        int rows = 0;
        for (const AnPiece& p : ps) rows += p.n;
        const size_t cfg_bytes = align16(sizeof(SpecCfg) * rows);
        float* ring = nullptr;
        CU(cudaHostGetDevicePointer((void**)&ring, a.result, 0));
        int max_items = 0;
        const int rc = analysis_launch(
            e, an, ps, cfg_bytes + sizeof(SpecRun) * rows, 1,
            [&](unsigned char* h) {
                SpecCfg* hc = reinterpret_cast<SpecCfg*>(h);
                SpecRun* hr = reinterpret_cast<SpecRun*>(h + cfg_bytes);
                int32_t* counters = reinterpret_cast<int32_t*>(a.work.p + a.work.n) - kAnalysisMaxUnits;
                size_t work = 0;
                int r = 0;
                // every row is a device of its own with one batch, so the kernel's batch step is never taken
                for (const AnPiece& p : ps) {
                    const AnJob& J = an[p.job];
                    const Device& d = e->dev[J.dev];
                    for (int u = 0; u < p.n; u++, r++) {
                        SpecCfg& c = hc[r];
                        c.wsc = e->groups[d.group].wsc.p;
                        c.partial = reinterpret_cast<float*>(a.work.p + work);
                        c.counter = counters + r;
                        c.ring = ring + (size_t)r * N;
                        c.hop_bytes = d.hop_bytes; c.sfmt = d.sfmt; c.stride = J.stride; c.n_sel = J.n_sel;
                        c.n_chunks = (J.n_sel + ABG_SPEC_FPC - 1) / ABG_SPEC_FPC;
                        c.ring_cap = 1;
                        work += J.unit_work;
                        hr[r] = SpecRun{a.scratch.p, p.off + (unsigned long long)u * J.step * d.hop_bytes, 1, 0};
                        max_items = std::max(max_items, c.n_chunks);
                    }
                }
            },
            [&](unsigned char* dv, cudaStream_t s) {
                SpecArgs A{};
                A.cfg = reinterpret_cast<const SpecCfg*>(dv); A.run = reinterpret_cast<const SpecRun*>(dv + cfg_bytes);
                A.tw1 = e->tw1.p; A.tw2 = e->tw2.p; A.wave_batch = 0;
                return abg_launch_spectrum(N, A, rows, max_items, s);
            });
        if (rc != ABG_OK) return rc;
        const float* res = reinterpret_cast<const float*>(a.result);
        for (const AnPiece& p : ps) {
            memcpy(jobs[p.job].power + (size_t)p.u0 * N, res, sizeof(float) * (size_t)p.n * N);
            res += (size_t)p.n * N;
        }
        return ABG_OK;
    });
}

// A job's detector pieces joined batch by batch with merge_bursts' rule (lib.py), plus the window's edge flags.  Within a
// batch, only a bin's first piece can carry OPEN_START and only its last OPEN_END, so the pieces are taken in the order
// the kernel stored them; the bursts are sorted once at the end.
struct BurstMerge {
    struct Open {
        abg_burst rec;
        long long q0, q1;  // selected index of its first and last member, counted from the window's start
        bool live;
    };
    std::vector<Open> open, next;      // [fft_size]: per bin the burst that may continue in the next batch
    std::vector<int32_t> open_bins, next_bins;
    std::vector<abg_burst> out;
    int truncated = 0;
    void keep(const Open& o, int min_span) {
        if (o.rec.flags != 0 || o.q1 - o.q0 + 1 >= min_span) out.push_back(o.rec);
    }
    // batch bi (of n_batches) of the window, its detector entry at `entry`
    void batch(const abg_activity_job& J, int N, int B, int n_sel, int bi, const unsigned char* entry) {
        if (open.empty()) open.assign(N, Open{}), next.assign(N, Open{});
        int32_t head[4];
        memcpy(head, entry, sizeof(head));
        const int stored = std::min(head[0], (int32_t)ABG_ACTIVITY_MAX_RECORDS);
        if (head[0] > ABG_ACTIVITY_MAX_RECORDS) truncated++;
        const unsigned long long f0 = ABG_AGC_EXTRA + (J.first_batch + (unsigned long long)bi) * B;
        auto q = [&](uint64_t f) { return (long long)bi * n_sel + (long long)((f - f0) / (unsigned)J.stride); };
        for (int i = 0; i < stored; i++) {
            abg_burst p;
            memcpy(&p, entry + ABG_ACT_HEAD_BYTES + sizeof(abg_burst) * (size_t)i, sizeof(p));
            Open cur;
            Open& prev = open[p.bin];
            if ((p.flags & ABG_BURST_OPEN_START) && prev.live && q(p.first_frame) - prev.q1 <= J.hang + 1) {
                cur = prev;
                prev.live = false;
                cur.rec.last_frame = p.last_frame;
                cur.rec.n_active += p.n_active;
                cur.rec.peak = std::max(cur.rec.peak, p.peak);
                cur.rec.sum = cur.rec.sum + p.sum;
                cur.q1 = q(p.last_frame);
            } else {
                cur.rec = p;
                cur.rec.flags = bi == 0 && (p.flags & ABG_BURST_OPEN_START) ? ABG_BURST_OPEN_START : 0;
                cur.q0 = q(p.first_frame);
                cur.q1 = q(p.last_frame);
            }
            cur.live = true;
            if (p.flags & ABG_BURST_OPEN_END) {
                next[p.bin] = cur;
                next_bins.push_back(p.bin);
            } else {
                keep(cur, J.min_span);
            }
        }
        for (const int32_t k : open_bins)  // not continued in this batch
            if (open[k].live) {
                keep(open[k], J.min_span);
                open[k].live = false;
            }
        open.swap(next);
        open_bins.swap(next_bins);
        next_bins.clear();
        if (bi + 1 < J.n_batches) return;
        for (const int32_t k : open_bins) {
            open[k].rec.flags |= ABG_BURST_OPEN_END;
            out.push_back(open[k].rec);
            open[k].live = false;
        }
        open_bins.clear();
    }
};

int abg_history_activity(abg_engine* e, int n_jobs, abg_activity_job* jobs) {
    if (n_jobs < 1 || n_jobs > 65535 || !jobs)
        return fail(ABG_EINVAL, "abg_history_activity: %d jobs at %p (1 to 65535)", n_jobs, (const void*)jobs);
    const int N = e->N, B = e->B;
    const size_t entry = ABG_ACT_HEAD_BYTES + sizeof(abg_burst) * (size_t)ABG_ACTIVITY_MAX_RECORDS;
    std::vector<AnJob> an(n_jobs);
    for (int j = 0; j < n_jobs; j++) {
        const abg_activity_job& J = jobs[j];
        if (!monitor_dev(e, e->history, J.dev, __func__)) return ABG_ERANGE;
        char who[48];
        snprintf(who, sizeof(who), "abg_history_activity: jobs[%d]", j);
        int rc = activity_check(e, who, J.stride, J.hang, J.min_span, J.thr);
        if (rc != ABG_OK) return rc;
        if (J.stride == 0 || J.n_batches < 1 || J.cap < 0 || (J.cap > 0 && !J.out))
            return fail(ABG_EINVAL, "%s: stride %d, %d batches, %d bursts into %p", who, J.stride, J.n_batches, J.cap, (void*)J.out);
        an[j] = AnJob{J.dev, ABG_AGC_EXTRA + (unsigned __int128)J.first_batch * B, (unsigned long long)B, J.n_batches,
                      (B + J.stride - 1) / J.stride, J.stride, entry, 0};
        if ((rc = analysis_window(e, __func__, j, an[j])) != ABG_OK) return rc;
    }
    auto& a = e->analysis;
    std::vector<BurstMerge> merge(n_jobs);
    const int rc = analysis_chunks(e, an, [&](const std::vector<AnPiece>& ps) -> int {
        const int np = (int)ps.size();
        const size_t cfg_bytes = align16(sizeof(ActCfg) * np), run_bytes = align16(sizeof(ActRun) * np), thr_bytes = sizeof(float) * N;
        unsigned char* ring = nullptr;
        CU(cudaHostGetDevicePointer((void**)&ring, a.result, 0));
        int max_batches = 0;
        int rc2 = analysis_launch(
            e, an, ps, cfg_bytes + run_bytes + thr_bytes * np, 2,
            [&](unsigned char* h) {
                ActCfg* hc = reinterpret_cast<ActCfg*>(h);
                ActRun* hr = reinterpret_cast<ActRun*>(h + cfg_bytes);
                size_t ent = 0;
                for (int i = 0; i < np; i++) {
                    const AnPiece& p = ps[i];
                    const abg_activity_job& J = jobs[p.job];
                    const Device& d = e->dev[J.dev];
                    memcpy(h + cfg_bytes + run_bytes + thr_bytes * i, J.thr, thr_bytes);
                    ActCfg& c = hc[i];
                    c.wsc = e->groups[d.group].wsc.p;
                    c.thr = reinterpret_cast<const float*>(a.table.p + align16(sizeof(RpGather) * ps.size()) + cfg_bytes + run_bytes + thr_bytes * i);
                    c.ring = ring + ent * entry;
                    c.hop_bytes = d.hop_bytes; c.sfmt = d.sfmt; c.stride = J.stride; c.n_sel = an[p.job].n_sel;
                    c.hang = J.hang; c.min_span = J.min_span; c.ring_cap = p.n; c.entry_bytes = (int32_t)entry;
                    hr[i] = ActRun{a.scratch.p, p.off, (unsigned long long)ABG_AGC_EXTRA + (J.first_batch + (unsigned long long)p.u0) * B, p.n, 0};
                    ent += p.n;
                    max_batches = std::max(max_batches, p.n);
                }
            },
            [&](unsigned char* dv, cudaStream_t s) {
                ActArgs A{};
                A.cfg = reinterpret_cast<const ActCfg*>(dv); A.run = reinterpret_cast<const ActRun*>(dv + cfg_bytes);
                A.tw1 = e->tw1.p; A.tw2 = e->tw2.p; A.wave_batch = B;
                return abg_launch_activity(N, A, np, max_batches, s);
            });
        if (rc2 != ABG_OK) return rc2;
        const unsigned char* res = a.result;
        for (const AnPiece& p : ps)
            for (int b = 0; b < p.n; b++, res += entry) merge[p.job].batch(jobs[p.job], N, B, an[p.job].n_sel, p.u0 + b, res);
        return ABG_OK;
    });
    if (rc != ABG_OK) return rc;
    for (int j = 0; j < n_jobs; j++) {
        std::vector<abg_burst>& v = merge[j].out;
        std::sort(v.begin(), v.end(), [](const abg_burst& x, const abg_burst& y) {
            return x.bin != y.bin ? x.bin < y.bin : x.first_frame < y.first_frame;
        });
        if (jobs[j].cap > 0) memcpy(jobs[j].out, v.data(), sizeof(abg_burst) * std::min(v.size(), (size_t)jobs[j].cap));
        jobs[j].n_bursts = (int32_t)v.size();
        jobs[j].n_truncated = merge[j].truncated;
    }
    return ABG_OK;
}

int abg_debug_history_analysis_time(abg_engine* e, float* ms3) {
    if (!ms3) return fail(ABG_EINVAL, "abg_debug_history_analysis_time: null argument");
    memcpy(ms3, e->analysis.ms, sizeof(e->analysis.ms));
    return ABG_OK;
}

// ---- transmission profiles (definition in airband_b200.h) ----------------------------------------------------------------
// A job's outputs are cut into blocks of ABG_PROFILE_BLOCK anchored at its m0; a call is cut into chunks of whole blocks,
// in job and block order, within fixed budgets.  A chunk holds one piece per job it touches: the piece's consecutive
// blocks, captured by one launch of the history capture into the scratch, plus the output after its last block when the
// job goes on (the successor of the pair across the seam).  The plan is a pure host function, so that every index the
// kernel reads can be checked without a GPU (abg_debug_profile_plan).
constexpr long long kProfileScratch = 8ll << 20;  // captured outputs per chunk: 64 MB of float2, the analysis figure
constexpr int kProfileBlocks = 65535;             // CTAs of a profile launch
constexpr long long kProfileResult = 8ll << 20;   // block sums per chunk (floats): 32 MB
constexpr long long kProfileCoeffs = 2ll << 20;   // capture coefficients per chunk (float2): 16 MB

static_assert(sizeof(abg_profile) == 2120 && sizeof(abg_profile_job) == 64, "the profile structs have a fixed layout");

struct ProfShape {  // what the plan needs of a job
    unsigned long long m0;
    long long n;
    int L, K;
};
struct ProfPiece {  // one capture: outputs [m, m + count) of job `job` at scratch index off
    int chunk, job;
    unsigned long long m;
    long long count;
    unsigned long long off, coef, tones;  // scratch index; index of its g[0] and its delta_0 in the chunk's tables
};
struct ProfPlanned {
    int chunk, job, piece;
    ProfBlock b;
};

static void profile_plan(const std::vector<ProfShape>& jobs, std::vector<ProfPiece>& pieces, std::vector<ProfPlanned>& blocks) {
    constexpr long long PB = ABG_PROFILE_BLOCK;
    int chunk = 0, nb = 0;
    long long scratch = 0, res = 0, coef = 0, tones = 0;
    for (int j = 0; j < (int)jobs.size(); j++) {
        const ProfShape& J = jobs[j];
        const long long nblk = (J.n + PB - 1) / PB, rb = ABG_PROFILE_SUMS + 4ll * J.K;
        for (long long k = 0; k < nblk; k++) {
            const unsigned long long m = J.m0 + (unsigned long long)(k * PB);
            const long long cnt = std::min(PB, J.n - k * PB);
            const int succ = k + 1 < nblk ? 1 : 0;
            for (;;) {
                const bool extend = !pieces.empty() && pieces.back().chunk == chunk && pieces.back().job == j;
                // extending: the previous block of the piece had a successor, which is this block's first output
                const long long s_need = extend ? (long long)pieces.back().off + pieces.back().count - 1 + cnt + succ : scratch + cnt + succ;
                const long long c_need = coef + (extend ? 0 : J.L), t_need = tones + (extend ? 0 : J.K);
                const bool fits = s_need <= kProfileScratch && nb < kProfileBlocks && res + rb <= kProfileResult && c_need <= kProfileCoeffs;
                if (!fits && nb > 0) {  // (a block alone always fits)
                    chunk++;
                    nb = 0;
                    scratch = res = coef = tones = 0;
                    continue;
                }
                if (extend) {
                    pieces.back().count += cnt + succ - 1;
                } else {
                    pieces.push_back(ProfPiece{chunk, j, m, cnt + succ, (unsigned long long)scratch, (unsigned long long)coef, (unsigned long long)tones});
                    coef = c_need;
                    tones = t_need;
                }
                const ProfPiece& p = pieces.back();
                scratch = s_need;
                blocks.push_back(ProfPlanned{chunk, j, (int)pieces.size() - 1,
                                           ProfBlock{p.off + (m - p.m), (unsigned long long)res, (long long)m, (int32_t)cnt, succ, (int32_t)p.tones, J.K}});
                res += rb;
                nb++;
                break;
            }
        }
    }
}

// The shape fields of a job as abg_history_profile checks them.
static int profile_shape_check(const char* who, long long n, int L, int K) {
    if (n < 2) return fail(ABG_EINVAL, "%s: %lld outputs (at least 2)", who, n);
    if (L < 1 || L > ABG_SUBBAND_MAX_COEFFS) return fail(ABG_EINVAL, "%s: %d coefficients outside [1, %d]", who, L, ABG_SUBBAND_MAX_COEFFS);
    if (K < 1 || K > ABG_TONE_MAX) return fail(ABG_EINVAL, "%s: %d tones outside [1, %d]", who, K, ABG_TONE_MAX);
    return ABG_OK;
}

int abg_debug_profile_plan(int n_jobs, const uint64_t* first_m, const int64_t* n_out, const int32_t* n_coeffs, const int32_t* n_tones,
                           int64_t* limits, int64_t* pieces, int cap_pieces, int32_t* n_pieces, int64_t* blocks, int cap_blocks,
                           int32_t* n_blocks) {
    if (n_jobs < 1 || n_jobs > 65535 || !first_m || !n_out || !n_coeffs || !n_tones || !n_pieces || !n_blocks)
        return fail(ABG_EINVAL, "abg_debug_profile_plan: %d jobs (1 to 65535) or a null argument", n_jobs);
    std::vector<ProfShape> shapes(n_jobs);
    for (int j = 0; j < n_jobs; j++) {
        char who[48];
        snprintf(who, sizeof(who), "abg_debug_profile_plan: jobs[%d]", j);
        const int rc = profile_shape_check(who, n_out[j], n_coeffs[j], n_tones[j]);
        if (rc != ABG_OK) return rc;
        shapes[j] = ProfShape{first_m[j], n_out[j], n_coeffs[j], n_tones[j]};
    }
    std::vector<ProfPiece> ps;
    std::vector<ProfPlanned> bs;
    profile_plan(shapes, ps, bs);
    if (limits) {
        const int64_t lim[4] = {kProfileScratch, kProfileBlocks, kProfileResult, kProfileCoeffs};
        memcpy(limits, lim, sizeof(lim));
    }
    *n_pieces = (int32_t)ps.size();
    *n_blocks = (int32_t)bs.size();
    for (int i = 0; pieces && i < (int)ps.size() && i < cap_pieces; i++) {
        const ProfPiece& p = ps[i];
        const int64_t row[6] = {p.chunk, p.job, (int64_t)p.m, p.count, (int64_t)p.off, (int64_t)p.coef};
        memcpy(pieces + 6 * (size_t)i, row, sizeof(row));
    }
    for (int i = 0; blocks && i < (int)bs.size() && i < cap_blocks; i++) {
        const ProfPlanned& q = bs[i];
        const int64_t row[8] = {q.chunk, q.job, q.piece, (int64_t)q.b.off, q.b.m, q.b.n, q.b.succ, (int64_t)q.b.res};
        memcpy(blocks + 8 * (size_t)i, row, sizeof(row));
    }
    return ABG_OK;
}

// One chunk: pieces [p0, p1) and blocks [b0, b1) of the plan.  On the K1 stream: the upload of its tables, one capture
// per piece into the scratch (behind every append it reads, ahead of every later one that would overwrite its samples),
// the profile kernel, and the copy of the block sums; waits for them.
static int profile_chunk(abg_engine* e, const abg_profile_job* jobs, const std::vector<uint32_t>& tdelta, const std::vector<ProfPiece>& ps,
                         size_t p0, size_t p1, const std::vector<ProfPlanned>& bs, size_t b0, size_t b1) {
    auto& P = e->profile;
    const ProfPiece& last = ps[p1 - 1];
    const size_t n_coef = last.coef + jobs[last.job].n_coeffs, n_delta = last.tones + tdelta[(size_t)last.job * (ABG_TONE_MAX + 1)];
    const size_t coef_bytes = align16(sizeof(float2) * n_coef), delta_bytes = align16(sizeof(uint32_t) * n_delta);
    const size_t need = coef_bytes + delta_bytes + sizeof(ProfBlock) * (b1 - b0);
    if (P.table.n < need) {
        P.table.free();
        if (P.table.alloc(2 * need)) return fail(ABG_ENOMEM, "Out of device memory for the transmission profile tables");
        if (P.h_table) cudaFreeHost(P.h_table);
        if (cudaHostAlloc((void**)&P.h_table, 2 * need, cudaHostAllocDefault) != cudaSuccess) {
            cudaGetLastError();
            P.h_table = nullptr;
            P.table.free();
            return fail(ABG_ENOMEM, "Out of page-locked host memory for the transmission profile tables");
        }
    }
    float2* hc = reinterpret_cast<float2*>(P.h_table);
    uint32_t* hd = reinterpret_cast<uint32_t*>(P.h_table + coef_bytes);
    ProfBlock* hb = reinterpret_cast<ProfBlock*>(P.h_table + coef_bytes + delta_bytes);
    std::vector<float2> g;
    std::vector<uint32_t> sb_delta(p1 - p0);
    for (size_t i = p0; i < p1; i++) {
        const abg_profile_job& J = jobs[ps[i].job];
        sb_delta[i - p0] = subband_coefficients(J.offset_hz, e->dev[J.dev].sample_rate, J.n_coeffs, J.coeffs, g);
        memcpy(hc + ps[i].coef, g.data(), sizeof(float2) * J.n_coeffs);
        const uint32_t* td = &tdelta[(size_t)ps[i].job * (ABG_TONE_MAX + 1)];
        memcpy(hd + ps[i].tones, td + 1, sizeof(uint32_t) * td[0]);
    }
    unsigned long long res_floats = 0;
    for (size_t i = b0; i < b1; i++) {
        hb[i - b0] = bs[i].b;
        res_floats = std::max(res_floats, bs[i].b.res + ABG_PROFILE_SUMS + 4ull * bs[i].b.K);
    }
    const cudaStream_t s = e->stream;
    CU(cudaMemcpyAsync(P.table.p, P.h_table, need, cudaMemcpyHostToDevice, s));
    CU(cudaEventRecord(P.ev[0], s));
    for (size_t i = p0; i < p1; i++) {
        const ProfPiece& p = ps[i];
        const abg_profile_job& J = jobs[p.job];
        const Device& d = e->dev[J.dev];
        const HiDev& h = e->history.dev[J.dev];
        HiCapture c{};
        c.ring = h.ring.p; c.ring_bytes = h.ring.n; c.coef = reinterpret_cast<const float2*>(P.table.p) + p.coef;
        c.out = P.scratch.p + p.off; c.m0 = (long long)p.m; c.n_out = (int32_t)p.count;
        c.decim = J.decim; c.n_coeffs = J.n_coeffs; c.sfmt = d.sfmt; c.delta = sb_delta[i - p0]; c.scale = 1.0f / d.fullscale;
        const cudaError_t er = abg_launch_history_capture(c, s);
        if (er != cudaSuccess) return fail(ABG_ECUDA, "transmission profile capture launch failed: %s", cudaGetErrorString(er));
        e->launches++;
    }
    CU(cudaEventRecord(P.ev[1], s));
    ProfArgs A{};
    A.y = P.scratch.p; A.blocks = reinterpret_cast<const ProfBlock*>(P.table.p + coef_bytes + delta_bytes);
    A.delta = reinterpret_cast<const uint32_t*>(P.table.p + coef_bytes); A.res = P.res.p;
    const cudaError_t er = abg_launch_profile(A, (int)(b1 - b0), s);
    if (er != cudaSuccess) return fail(ABG_ECUDA, "transmission profile launch failed: %s", cudaGetErrorString(er));
    e->launches++;
    CU(cudaEventRecord(P.ev[2], s));
    CU(cudaMemcpyAsync(P.h_res, P.res.p, sizeof(float) * res_floats, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    float ms = 0.0f;
    CU(cudaEventElapsedTime(&ms, P.ev[0], P.ev[1]));
    P.ms[0] += ms;
    CU(cudaEventElapsedTime(&ms, P.ev[1], P.ev[2]));
    P.ms[1] += ms;
    return ABG_OK;
}

int abg_history_profile(abg_engine* e, int n_jobs, abg_profile_job* jobs) {
    if (n_jobs < 1 || n_jobs > 65535 || !jobs)
        return fail(ABG_EINVAL, "abg_history_profile: %d jobs at %p (1 to 65535)", n_jobs, (const void*)jobs);
    std::vector<ProfShape> shapes(n_jobs);
    std::vector<uint32_t> tdelta((size_t)n_jobs * (ABG_TONE_MAX + 1));  // per job: K, then delta_k
    for (int j = 0; j < n_jobs; j++) {
        const abg_profile_job& J = jobs[j];
        char who[48];
        snprintf(who, sizeof(who), "abg_history_profile: jobs[%d]", j);
        const HiDev* h = monitor_dev(e, e->history, J.dev, who);
        if (!h) return ABG_ERANGE;
        const Device& d = e->dev[J.dev];
        int rc = subband_check(who, d, e->B * d.hop, J.offset_hz, J.decim, J.n_coeffs, J.coeffs);
        if (rc != ABG_OK) return rc;
        if (J.n_tones < 0 || J.n_tones > ABG_TONE_MAX)
            return fail(ABG_EINVAL, "%s: %d tones outside [0, %d]", who, J.n_tones, ABG_TONE_MAX);
        const bool custom = J.tones && J.n_tones > 0;
        const int K = custom ? J.n_tones : 51;
        if ((rc = profile_shape_check(who, J.n_out, J.n_coeffs, K)) != ABG_OK) return rc;
        if (!J.out) return fail(ABG_EINVAL, "%s: null out", who);
        const double fs_out = (double)d.sample_rate / J.decim;
        uint32_t* td = &tdelta[(size_t)j * (ABG_TONE_MAX + 1)];
        td[0] = (uint32_t)K;
        for (int k = 0; k < K; k++) {
            const float f = custom ? J.tones[k] : kStandardTones[k];
            if (!std::isfinite(f) || !(f > 0.0f) || !((double)f < fs_out / 2.0))
                return fail(ABG_EINVAL, "%s: tone %d (%g Hz) outside (0, %g) Hz", who, k, (double)f, fs_out / 2.0);
            td[1 + k] = (uint32_t)(unsigned long long)llround((double)f / fs_out * 4294967296.0);
        }
        // every tap in the history, abg_history_subband's rule: first_m D - (L - 1) >= first and (first_m + n - 1) D < end
        const unsigned __int128 D = (unsigned)J.decim, lo = (unsigned __int128)J.first_m * D,
                                hi = ((unsigned __int128)J.first_m + (unsigned long long)J.n_out - 1) * D;
        if (h->first == h->end || lo < (unsigned __int128)h->first + (J.n_coeffs - 1) || hi >= h->end) {
            const unsigned long long need_lo = (unsigned long long)(lo - std::min<unsigned __int128>(lo, J.n_coeffs - 1));
            return fail(ABG_ERANGE, "%s: outputs [%llu, +%lld) at decimation %d with %d coefficients read samples [%llu, %llu], outside the history [%llu, %llu) of device %d",
                        who, (unsigned long long)J.first_m, (long long)J.n_out, J.decim, J.n_coeffs, need_lo, (unsigned long long)hi,
                        (unsigned long long)h->first, (unsigned long long)h->end, J.dev);
        }
        shapes[j] = ProfShape{J.first_m, J.n_out, J.n_coeffs, K};
    }
    std::vector<ProfPiece> ps;
    std::vector<ProfPlanned> bs;
    profile_plan(shapes, ps, bs);

    auto& P = e->profile;
    cudaSetDevice(e->cuda_dev);
    if (!P.ev[0]) {
        if (P.scratch.alloc(kProfileScratch) || P.res.alloc(kProfileResult)) {
            P.scratch.free();
            P.res.free();
            return fail(ABG_ENOMEM, "Out of device memory for the transmission profile scratch");
        }
        if (cudaHostAlloc((void**)&P.h_res, sizeof(float) * kProfileResult, cudaHostAllocDefault) != cudaSuccess) {
            cudaGetLastError();
            P.h_res = nullptr;
            P.scratch.free();
            P.res.free();
            return fail(ABG_ENOMEM, "Out of page-locked host memory for the transmission profile results");
        }
        for (auto& ev : P.ev) CU(cudaEventCreate(&ev));
    }
    P.ms[0] = P.ms[1] = 0.0f;
    // per job: the sums in double, added block by block in block order
    std::vector<abg_profile> acc(n_jobs);
    memset(acc.data(), 0, sizeof(abg_profile) * n_jobs);
    for (size_t p0 = 0, b0 = 0; p0 < ps.size();) {
        size_t p1 = p0, b1 = b0;
        while (p1 < ps.size() && ps[p1].chunk == ps[p0].chunk) p1++;
        while (b1 < bs.size() && bs[b1].chunk == ps[p0].chunk) b1++;
        const int rc = profile_chunk(e, jobs, tdelta, ps, p0, p1, bs, b0, b1);
        if (rc != ABG_OK) return rc;
        for (size_t i = b0; i < b1; i++) {
            const ProfBlock& b = bs[i].b;
            const float* r = P.h_res + b.res;
            abg_profile& o = acc[bs[i].job];
            o.p1 += r[0]; o.p2 += r[1]; o.a1 += r[2]; o.z[0] += r[3]; o.z[1] += r[4]; o.f1 += r[5]; o.f2 += r[6];
            for (int k = 0; k < b.K; k++) {
                o.tone_fm[k][0] += r[ABG_PROFILE_SUMS + 2 * k];
                o.tone_fm[k][1] += r[ABG_PROFILE_SUMS + 2 * k + 1];
                o.tone_am[k][0] += r[ABG_PROFILE_SUMS + 2 * b.K + 2 * k];
                o.tone_am[k][1] += r[ABG_PROFILE_SUMS + 2 * b.K + 2 * k + 1];
            }
        }
        p0 = p1;
        b0 = b1;
    }
    for (int j = 0; j < n_jobs; j++) {
        acc[j].n = jobs[j].n_out;
        acc[j].n_tones = shapes[j].K;
        memcpy(jobs[j].out, &acc[j], sizeof(abg_profile));
    }
    return ABG_OK;
}

int abg_debug_history_profile_time(abg_engine* e, float* ms2) {
    if (!ms2) return fail(ABG_EINVAL, "abg_debug_history_profile_time: null argument");
    memcpy(ms2, e->profile.ms, sizeof(e->profile.ms));
    return ABG_OK;
}

// ---- scan mode -------------------------------------------------------------------------------------------------------
static ScanView scan_view(abg_engine* e) {
    ScanView v;
    v.params = e->params.p; v.state = e->state.p; v.sqbuf = e->sqbuf.p; v.tone_coeff = e->tone_coeff.p;
    v.tone_q1 = e->tone_q1.p; v.tone_q2 = e->tone_q2.p; v.tone_mag = e->tone_mag.p; v.Gp = e->Gp;
    return v;
}

int abg_scan_configure(abg_engine* e, int dev, int chan, int n_freqs, const abg_channel_cfg* freqs) {
    if (dev < 0 || dev >= (int)e->dev.size()) return fail(ABG_ERANGE, "abg_scan_configure: device %d out of range", dev);
    Device& d = e->dev[dev];
    if (chan < 0 || chan >= d.C) return fail(ABG_ERANGE, "abg_scan_configure: channel %d out of range", chan);
    if (n_freqs < 1 || !freqs) return fail(ABG_EINVAL, "abg_scan_configure: empty frequency list");
    const int g = d.g0 + chan;
    cudaSetDevice(e->cuda_dev);
    CU(cudaStreamSynchronize(e->stream));
    CU(cudaStreamSynchronize(e->stream_b));
    std::vector<FreqSet> sets((size_t)n_freqs);
    for (int i = 0; i < n_freqs; i++) {
        FreqSet& f = sets[i];
        memset(&f, 0, sizeof(f));
        char what[64];
        snprintf(what, sizeof(what), "abg_scan_configure: freqs[%d]", i);
        std::vector<float> banks[2];
        const int rc = build_freq(e->W, freqs[i], f.p, f.s, banks, what);
        if (rc != ABG_OK) return rc;
        if (f.p.modulation == ABG_MOD_NFM) e->any_nfm = true;
        for (int w = 0; w < 2; w++)
            for (size_t t = 0; t < banks[w].size(); t++) f.tone_coeff[w][t] = banks[w][t];
    }
    abg_engine::ScanChan* sc = nullptr;
    for (auto& x : e->scan)
        if (x.g == g) sc = &x;
    if (!sc) {
        e->scan.emplace_back();
        sc = &e->scan.back();
        sc->g = g;
    }
    if (sc->stash) cudaFree(sc->stash);
    sc->stash = nullptr;
    // one extra entry: scratch that receives the state being replaced below
    if (cudaMalloc((void**)&sc->stash, sizeof(FreqSet) * (size_t)(n_freqs + 1)) != cudaSuccess) return fail(ABG_ENOMEM, "Out of device memory for the scan frequency list");
    CU(cudaMemcpy(sc->stash, sets.data(), sizeof(FreqSet) * (size_t)n_freqs, cudaMemcpyHostToDevice));
    sc->n_freqs = n_freqs;
    sc->cur = 0;
    scan_swap_kernel<<<1, 128, 0, e->stream_b>>>(scan_view(e), g, sc->stash + n_freqs, sc->stash + 0);  // entry 0 goes live, fresh
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(e->stream_b));
    return ABG_OK;
}

int abg_scan_select(abg_engine* e, int dev, int chan, int freq_idx) {
    if (dev < 0 || dev >= (int)e->dev.size()) return fail(ABG_ERANGE, "abg_scan_select: device %d out of range", dev);
    Device& d = e->dev[dev];
    if (chan < 0 || chan >= d.C) return fail(ABG_ERANGE, "abg_scan_select: channel %d out of range", chan);
    const int g = d.g0 + chan;
    abg_engine::ScanChan* sc = nullptr;
    for (auto& x : e->scan)
        if (x.g == g) sc = &x;
    if (!sc) return fail(ABG_EINVAL, "abg_scan_select: devices[%d].channels[%d] has no frequency list (abg_scan_configure)", dev, chan);
    if (freq_idx < 0 || freq_idx >= sc->n_freqs) return fail(ABG_ERANGE, "abg_scan_select: frequency index %d outside 0..%d", freq_idx, sc->n_freqs - 1);
    if (freq_idx == sc->cur) return ABG_OK;
    cudaSetDevice(e->cuda_dev);
    // stream B: after every K2 already enqueued, before the next one = between two batches (rtl_airband.cpp:498)
    scan_swap_kernel<<<1, 128, 0, e->stream_b>>>(scan_view(e), g, sc->stash + sc->cur, sc->stash + freq_idx);
    CU(cudaGetLastError());
    e->launches++;
    sc->cur = freq_idx;
    return ABG_OK;
}

// Pin (page-lock) a host buffer the caller keeps pushing from - in the reference that is input_t.buffer, the ring the
// SDR driver threads fill (input-helpers.cpp:27-36) - so that abg_push's host->device copies are real asynchronous DMA
// instead of being staged through the driver's bounce buffer.  Optional: abg_push works with pageable memory too.
int abg_host_register(void* ptr, size_t nbytes) {
    if (!ptr || nbytes == 0) return fail(ABG_EINVAL, "abg_host_register: empty range");
    cudaError_t er = cudaHostRegister(ptr, nbytes, cudaHostRegisterPortable);
    if (er == cudaErrorHostMemoryAlreadyRegistered) {
        cudaGetLastError();
        return ABG_OK;
    }
    if (er != cudaSuccess) {
        cudaGetLastError();
        return fail(ABG_ECUDA, "abg_host_register: %s", cudaGetErrorString(er));
    }
    return ABG_OK;
}

// Returns once every abg_push so far has been read out of the caller's buffers (needed before reusing page-locked
// memory that was pushed from: with abg_host_register the copies are asynchronous).  Does not wait for kernels.
int abg_ingest_sync(abg_engine* e) {
    cudaSetDevice(e->cuda_dev);
    CU(cudaStreamSynchronize(e->stream_c));
    return ABG_OK;
}

int abg_host_unregister(void* ptr) {
    if (!ptr) return ABG_OK;
    cudaError_t er = cudaHostUnregister(ptr);
    if (er != cudaSuccess) {
        cudaGetLastError();
        return fail(ABG_ECUDA, "abg_host_unregister: %s", cudaGetErrorString(er));
    }
    return ABG_OK;
}

int abg_resident_load(abg_engine* e, int dev, const void* iq, size_t nbytes) {
    if (dev < 0 || dev >= (int)e->dev.size()) return fail(ABG_ERANGE, "abg_resident_load: device %d out of range", dev);
    Device& d = e->dev[dev];
    const size_t need = (size_t)(e->nbmax * e->B + ABG_AGC_EXTRA - 1) * d.hop_bytes + (size_t)e->N * d.bpc;
    if (nbytes < need) return fail(ABG_EINVAL, "abg_resident_load: need at least %zu bytes for %d batches, got %zu", need, e->nbmax, nbytes);
    // The input meter reads the first hop samples of every frame of a batch, up to (AGC_EXTRA + nbmax*B) * hop_bytes:
    // past `need` when hop > fft_size.  The tail it reads there is zeros (resident runs queue no readings).
    const size_t meter_end = (size_t)(e->nbmax * e->B + ABG_AGC_EXTRA) * d.hop_bytes;
    const size_t alloc = std::max(need, meter_end) + 256;
    cudaSetDevice(e->cuda_dev);
    if (d.res) cudaFree(d.res);
    d.res = nullptr;
    if (cudaMalloc((void**)&d.res, alloc) != cudaSuccess) return fail(ABG_ENOMEM, "Out of device memory for the resident stream");
    d.res_bytes = need;
    CU(cudaMemsetAsync(d.res + need, 0, alloc - need, e->stream));
    CU(cudaMemcpyAsync(d.res, iq, need, cudaMemcpyHostToDevice, e->stream));
    CU(cudaStreamSynchronize(e->stream));
    return ABG_OK;
}

int abg_run_resident(abg_engine* e, int n_batches) {
    cudaSetDevice(e->cuda_dev);
    if (n_batches < 1 || n_batches > e->nbmax) return fail(ABG_EINVAL, "abg_run_resident: n_batches must be 1..%d", e->nbmax);
    std::vector<int> nb(e->dev.size(), n_batches);
    for (auto& d : e->dev)
        if (!d.res) return fail(ABG_EINVAL, "abg_run_resident: abg_resident_load() was not called for every device");
    int n = 0;
    int rc = enqueue_run(e, nb, true, false, &n);
    return rc != ABG_OK ? rc : n;
}

int abg_set_stream(abg_engine* e, void* cuda_stream) {
    cudaSetDevice(e->cuda_dev);
    CU(cudaStreamSynchronize(e->stream));
    CU(cudaStreamSynchronize(e->stream_b));
    if (e->own_stream) cudaStreamDestroy(e->stream);
    e->stream = (cudaStream_t)cuda_stream;
    e->own_stream = false;
    return ABG_OK;
}

uint64_t abg_launch_count(const abg_engine* e) { return e->launches; }

int abg_last_run_times(abg_engine* e, float* ms4) {
    if (!e->tev_valid) return fail(ABG_EINVAL, "abg_last_run_times: no run yet");
    cudaSetDevice(e->cuda_dev);
    cudaEvent_t* tl = e->tl[(e->run_index - 1) % TL_RUNS];
    CU(cudaEventSynchronize(tl[4]));
    CU(cudaEventElapsedTime(&ms4[0], tl[0], tl[1]));  // K1 on stream A
    CU(cudaEventElapsedTime(&ms4[1], tl[2], tl[3]));  // K2 on stream B
    CU(cudaEventElapsedTime(&ms4[2], tl[3], tl[4]));  // mixers + result export + tail copy
    CU(cudaEventElapsedTime(&ms4[3], tl[0], tl[4]));  // first K1 launch to end of run
    return ABG_OK;
}

// Timeline of the last n_runs (<= 8) runs: 5 timestamps per run (K1 start, K1 end, K2 start, K2 end, end of run) in ms
// relative to the oldest run's K1 start.  Measurement aid: shows how runs overlap inside the stream pipeline.
int abg_debug_timeline(abg_engine* e, int n_runs, float* ms) {
    if (!ms || n_runs < 1 || n_runs > TL_RUNS || (uint64_t)n_runs > e->run_index)
        return fail(ABG_EINVAL, "abg_debug_timeline: bad arguments");
    cudaSetDevice(e->cuda_dev);
    cudaEvent_t* last = e->tl[(e->run_index - 1) % TL_RUNS];
    CU(cudaEventSynchronize(last[4]));
    cudaEvent_t origin = e->tl[(e->run_index - n_runs) % TL_RUNS][0];
    for (int r = 0; r < n_runs; r++) {
        cudaEvent_t* tl = e->tl[(e->run_index - n_runs + r) % TL_RUNS];
        for (int k = 0; k < 5; k++) CU(cudaEventElapsedTime(&ms[r * 5 + k], origin, tl[k]));
    }
    return ABG_OK;
}

int abg_mixers_configure(abg_engine* e, int n_mixers, const int32_t* input_offsets, const abg_mixer_input* inputs) {
    if (n_mixers < 0 || (n_mixers > 0 && (!input_offsets || !inputs))) return fail(ABG_EINVAL, "abg_mixers_configure: bad arguments");
    cudaSetDevice(e->cuda_dev);
    CU(cudaStreamSynchronize(e->stream));
    CU(cudaStreamSynchronize(e->stream_b));
    if (!e->mix_ready.empty()) return fail(ABG_EINVAL, "abg_mixers_configure: unfetched mixer batches pending");
    const int total = n_mixers ? input_offsets[n_mixers] : 0;
    std::vector<MixInput> mi(total);
    for (int i = 0; i < total; i++) {
        const abg_mixer_input& in = inputs[i];
        if (in.dev < 0 || in.dev >= (int)e->dev.size()) return fail(ABG_ERANGE, "mixer input %d: device %d out of range", i, in.dev);
        if (in.chan < 0 || in.chan >= e->dev[in.dev].C) return fail(ABG_ERANGE, "mixer input %d: channel %d out of range", i, in.chan);
        mi[i].g = e->dev[in.dev].g0 + in.chan;
        mi[i].dev = in.dev;
        const float ampl = fminf(1.0f, 1.0f - in.balance), ampr = fminf(1.0f, 1.0f + in.balance);  // mixer.cpp:82-83
        mi[i].mult_l = in.ampfactor * ampl;  // mixer.cpp:203,206
        mi[i].mult_r = in.ampfactor * ampr;
    }
    e->mix_offsets.free(); e->mix_inputs.free(); e->mix_sums.free(); e->mix_flags.free();
    for (auto& s : e->slots) {
        if (s.mix) cudaFreeHost(s.mix);
        if (s.mixflag) cudaFreeHost(s.mixflag);
        s.mix = nullptr; s.mixflag = nullptr;
    }
    e->n_mixers = n_mixers;
    e->mix_fetched.assign(n_mixers, 0);
    if (n_mixers == 0) return ABG_OK;
    const size_t nsum = (size_t)e->nbmax * n_mixers * 2 * e->B;
    if (e->mix_offsets.alloc(n_mixers + 1) || e->mix_inputs.alloc(total) || e->mix_sums.alloc(nsum) || e->mix_flags.alloc((size_t)e->nbmax * n_mixers))
        return fail(ABG_ENOMEM, "Out of device memory for mixers");
    CU(cudaMemcpy(e->mix_offsets.p, input_offsets, sizeof(int32_t) * (n_mixers + 1), cudaMemcpyHostToDevice));
    if (total) CU(cudaMemcpy(e->mix_inputs.p, mi.data(), sizeof(MixInput) * total, cudaMemcpyHostToDevice));
    CU(cudaMemset(e->mix_sums.p, 0, sizeof(float) * nsum));
    CU(cudaMemset(e->mix_flags.p, 0, sizeof(int32_t) * (size_t)e->nbmax * n_mixers));
    for (auto& s : e->slots) {
        CU(cudaMallocHost((void**)&s.mix, sizeof(float) * nsum));
        CU(cudaMallocHost((void**)&s.mixflag, sizeof(int32_t) * (size_t)e->nbmax * n_mixers));
    }
    return ABG_OK;
}

int abg_fetch_mixer_batch(abg_engine* e, int mixer, float* left, float* right, int* has_signal) {
    if (mixer < 0 || mixer >= e->n_mixers) return fail(ABG_ERANGE, "abg_fetch_mixer_batch: mixer %d out of range", mixer);
    const int idx = e->mix_fetched[mixer];
    if (idx >= (int)e->mix_ready.size()) return 0;
    const std::pair<int, int> r = e->mix_ready[idx];
    Slot& s = e->slots[r.first];
    cudaSetDevice(e->cuda_dev);
    CU(cudaEventSynchronize(s.done));
    const int B = e->B;
    const float* base = s.mix + (((size_t)r.second * e->n_mixers + mixer) * 2) * B;
    if (left) memcpy(left, base, sizeof(float) * B);
    if (right) memcpy(right, base + B, sizeof(float) * B);
    if (has_signal) *has_signal = s.mixflag[(size_t)r.second * e->n_mixers + mixer];
    e->mix_fetched[mixer]++;
    s.mix_pending--;
    // drop queue entries every mixer has consumed
    int mn = e->mix_fetched[0];
    for (int v : e->mix_fetched) mn = std::min(mn, v);
    while (mn > 0) {
        e->mix_ready.pop_front();
        for (int& v : e->mix_fetched) v--;
        mn--;
    }
    return 1;
}

int abg_mixer_device_buffers(abg_engine* e, float** dev_sums, int32_t** dev_flags) {
    if (e->n_mixers <= 0) return fail(ABG_EINVAL, "abg_mixer_device_buffers: no mixers configured");
    if (dev_sums) *dev_sums = e->mix_sums.p;
    if (dev_flags) *dev_flags = e->mix_flags.p;
    return ABG_OK;
}

// Host-only (no device needed): the tensor-core K1's plan and coefficient table for one device, exactly as abg_create
// builds them.  plan[14] = {eligible, K, HC, S, NC, ND, C2p, KBS, NSTB, acc_regs, smem_bytes, halo, consumer_warpgroups, pps}.  tab may be
// null to query the plan; otherwise tab_cap >= K*NC bytes and sq has C2p entries.
int abg_debug_tc_table(int fft_size, int sfmt, int hop_bytes, float fullscale, int n_channels, const int32_t* bins, int digits, int32_t* plan,
                       signed char* tab, size_t tab_cap, long long* sq, double* cscale) {
    K1TcPlan p;
    abg_k1tc_plan(fft_size, sfmt, hop_bytes, n_channels, digits, &p);
    const int32_t v[14] = {p.eligible, p.K, p.HC, p.S, p.NC, p.ND, p.C2p, p.KBS, p.NSTB, p.acc_regs, p.smem_bytes, p.halo, p.consumer_warpgroups, p.pps};
    if (plan) memcpy(plan, v, sizeof(v));
    if (!p.eligible) return fail(ABG_EINVAL, "abg_debug_tc_table: configuration not eligible for the tensor-core K1");
    if (!tab) return ABG_OK;
    if (tab_cap < p.table_bytes || !sq || !cscale || !bins) return fail(ABG_EINVAL, "abg_debug_tc_table: buffers too small");
    std::vector<float> wsc = make_window(fft_size);
    const float scale = sample_scale(sfmt, fullscale);
    for (auto& w : wsc) w = w * scale;
    abg_k1tc_build_table(p, fft_size, sfmt, wsc.data(), bins, n_channels, tab, sq, cscale);
    return ABG_OK;
}

// Stage tap for the upstream squelch / CTCSS behavioural tests (reference src/test_squelch.cpp, src/test_ctcss.cpp) and for
// the exact K2-against-oracle tests: feed |X[bin]| values (and, optionally, X[bin] itself) straight into the demodulation
// state machine.  wavein[C][n_batches * WAVE_BATCH] becomes channel_t.wavein[AGC_EXTRA ...] of the device's channels (the AGC
// look-back keeps its initial 20.0, config.cpp:313-316, on the first call and the previous tail afterwards); iq_in[C][n_batches
// * WAVE_BATCH][2], if given, goes to the iqin rows K1 would have filled for the same frames.  K1 is skipped, K2 runs n_batches
// batches, results are fetched as usual.  A device driven this way must not be fed with abg_push; without iq_in its channels
// must not need raw I/Q, and AFC channels are refused either way (AFC reads the spectrum of the batch's last frame).
int abg_debug_inject_wavein(abg_engine* e, int dev, int n_batches, const float* wavein, const float* iq_in) {
    if (dev < 0 || dev >= (int)e->dev.size()) return fail(ABG_ERANGE, "abg_debug_inject_wavein: device %d out of range", dev);
    if (n_batches < 1 || n_batches > e->nbmax || !wavein) return fail(ABG_EINVAL, "abg_debug_inject_wavein: n_batches must be 1..%d", e->nbmax);
    Device& d = e->dev[dev];
    for (int c = 0; c < d.C; c++) {
        if (e->h_params[d.g0 + c].afc) return fail(ABG_EINVAL, "abg_debug_inject_wavein: channel %d uses AFC", c);
        if (e->h_params[d.g0 + c].needs_raw_iq && !iq_in) return fail(ABG_EINVAL, "abg_debug_inject_wavein: channel %d needs raw I/Q (iq_in)", c);
    }
    cudaSetDevice(e->cuda_dev);
    CU(cudaStreamSynchronize(e->stream_c));
    CU(cudaStreamSynchronize(e->stream));
    CU(cudaStreamSynchronize(e->stream_b));
    const int B = e->B, cur = (int)(e->run_index & 1);
    const size_t rows = (size_t)n_batches * B;
    std::vector<float> tm(rows * d.C);  // time-major like win[][]
    for (int c = 0; c < d.C; c++)
        for (size_t r = 0; r < rows; r++) tm[r * d.C + c] = wavein[(size_t)c * rows + r];
    CU(cudaMemcpy2D(e->win[cur].p + (size_t)ABG_AGC_EXTRA * e->Gp + d.g0, sizeof(float) * e->Gp, tm.data(), sizeof(float) * d.C, sizeof(float) * d.C, rows,
                    cudaMemcpyHostToDevice));
    if (iq_in) {
        std::vector<float2> tq(rows * d.C);
        for (int c = 0; c < d.C; c++)
            for (size_t r = 0; r < rows; r++) tq[r * d.C + c] = make_float2(iq_in[2 * ((size_t)c * rows + r)], iq_in[2 * ((size_t)c * rows + r) + 1]);
        CU(cudaMemcpy2D(e->iqin[cur].p + (size_t)ABG_AGC_EXTRA * e->Gp + d.g0, sizeof(float2) * e->Gp, tq.data(), sizeof(float2) * d.C, sizeof(float2) * d.C,
                        rows, cudaMemcpyHostToDevice));
    }
    std::vector<int> nb(e->dev.size(), 0);
    nb[dev] = n_batches;
    int n = 0;
    int rc = enqueue_run(e, nb, false, true, &n, true);
    return rc != ABG_OK ? rc : n;
}

// measurement aid: clock64 stamps of the tensor-core K1's roles for the first 16 tiles of every CTA (set ABG_K1_TC_TRACE before
// abg_create); out[256][4 roles][16 tiles][4 events]
int abg_debug_k2_stats(unsigned long long* out) { return abg_k2_stats_dump(out) == 0 ? ABG_OK : fail(ABG_EINVAL, "no counters: not an ABG_K2_STATS build (make stats)"); }
int abg_debug_k1tc_trace(long long* out) { return abg_k1tc_trace_dump(out) == 0 ? ABG_OK : fail(ABG_EINVAL, "no trace: ABG_K1_TC_TRACE was not set"); }

// see airband_b200.h: the most recent run's wout[Gp][P] and axc[max_batches_per_run][Gp] as the device holds them
int abg_debug_run_outputs(abg_engine* e, int32_t* dims, float* wout, unsigned char* axc) {
    if (dims) {
        dims[0] = e->G; dims[1] = e->Gp; dims[2] = e->P; dims[3] = e->nbmax;
    }
    if (!wout && !axc) return ABG_OK;
    cudaSetDevice(e->cuda_dev);
    CU(cudaDeviceSynchronize());
    if (wout) CU(cudaMemcpy(wout, e->wout.p, sizeof(float) * (size_t)e->Gp * e->P, cudaMemcpyDeviceToHost));
    if (axc) CU(cudaMemcpy(axc, e->axc.p, (size_t)e->nbmax * e->Gp, cudaMemcpyDeviceToHost));
    return ABG_OK;
}

// see airband_b200.h: rows [AGC_EXTRA, AGC_EXTRA + nbmax*B) of the win / iqin buffer the most recent run's K1 filled.  K2 of
// that run only reads it; what K2 writes are the look-back rows [0, AGC_EXTRA) of the other buffer (k2_launch: win_next).
int abg_debug_k1_outputs(abg_engine* e, int32_t* dims, float* win, float* iqin) {
    const int rows = e->nbmax * e->B;
    if (dims) {
        dims[0] = e->G; dims[1] = e->Gp; dims[2] = rows; dims[3] = e->nbmax;
    }
    if (!win && !iqin) return ABG_OK;
    if (e->run_index == 0) return fail(ABG_EINVAL, "abg_debug_k1_outputs: nothing has run yet");
    int rc = abg_sync(e);
    if (rc != ABG_OK) return rc;
    const int cur = (int)((e->run_index - 1) & 1);
    const size_t first = (size_t)ABG_AGC_EXTRA * e->Gp, n = (size_t)rows * e->Gp;
    if (win) CU(cudaMemcpy(win, e->win[cur].p + first, sizeof(float) * n, cudaMemcpyDeviceToHost));
    if (iqin) CU(cudaMemcpy(iqin, e->iqin[cur].p + first, sizeof(float2) * n, cudaMemcpyDeviceToHost));
    return ABG_OK;
}

// see airband_b200.h: the Device::spec rows the device's most recent K1 launch wrote.  Its K1Dev record stays on the host
// after the upload; row b is the frame at spec_first_pos + b * B, so the launch wrote the rows whose frame it computed.
int abg_debug_k1_spectra(abg_engine* e, int dev, int32_t* n_rows, float* out) {
    if (dev < 0 || dev >= (int)e->dev.size()) return fail(ABG_ERANGE, "abg_debug_k1_spectra: device %d out of range", dev);
    const Device& d = e->dev[dev];
    if (!d.has_afc) return fail(ABG_EINVAL, "abg_debug_k1_spectra: device %d has no AFC channel, so K1 keeps no spectrum", dev);
    if (e->run_index == 0) return fail(ABG_EINVAL, "abg_debug_k1_spectra: nothing has run yet");
    const Group& g = e->groups[d.group];
    const size_t k = std::find(g.devs.begin(), g.devs.end(), dev) - g.devs.begin();
    const K1Dev& a = g.h_k1[k];
    const int rows = a.n_frames > 0 ? (a.pos0 + a.n_frames - a.spec_first_pos + a.wave_batch - 1) / a.wave_batch : 0;
    if (n_rows) *n_rows = rows;
    if (!out || rows == 0) return ABG_OK;
    int rc = abg_sync(e);
    if (rc != ABG_OK) return rc;
    CU(cudaMemcpy(out, d.spec, sizeof(float2) * (size_t)rows * e->N, cudaMemcpyDeviceToHost));
    return ABG_OK;
}

int abg_debug_frame(abg_engine* e, int dev, const void* iq_frame, float* fftout) {
    if (dev < 0 || dev >= (int)e->dev.size()) return fail(ABG_ERANGE, "abg_debug_frame: device %d out of range", dev);
    cudaSetDevice(e->cuda_dev);
    Device& d = e->dev[dev];
    Group& g = e->groups[d.group];
    const int N = e->N;
    unsigned char* raw = nullptr;
    float2* spec = nullptr;
    K1Dev* dk = nullptr;
    const size_t bytes = (size_t)N * d.bpc;
    CU(cudaMalloc((void**)&raw, bytes + 256));
    CU(cudaMalloc((void**)&spec, sizeof(float2) * N));
    CU(cudaMalloc((void**)&dk, sizeof(K1Dev)));
    CU(cudaMemset(raw, 0, bytes + 256));
    CU(cudaMemcpy(raw, iq_frame, bytes, cudaMemcpyHostToDevice));
    K1Dev a{};
    a.raw = raw; a.start_byte = 0; a.n_frames = 1; a.pos0 = 0; a.g0 = d.g0; a.n_channels = 0; a.hop_bytes = d.hop_bytes; a.sfmt = d.sfmt;
    a.spec = spec; a.spec_first_pos = 0; a.wave_batch = e->B;
    CU(cudaMemcpy(dk, &a, sizeof(a), cudaMemcpyHostToDevice));
    K1Launch L{};
    L.fft_size = N; L.n_devices = 1; L.max_frames = 1; L.frames_per_tile = g.frames_per_tile; L.tile_bytes_cap = g.tile_bytes_cap; L.devs = dk;
    L.bins = e->bins.p; L.window_scaled = g.wsc.p; L.tw1 = e->tw1.p; L.tw2 = e->tw2.p; L.win = e->win[0].p; L.iqin = e->iqin[0].p; L.Gp = e->Gp; L.sfmt = g.sfmt;
    CU(cudaStreamSynchronize(e->stream));
    CU(cudaStreamSynchronize(e->stream_b));
    cudaError_t er = abg_launch_k1(L, e->stream);
    if (er != cudaSuccess) return fail(ABG_ECUDA, "K1 launch failed: %s", cudaGetErrorString(er));
    e->launches++;
    CU(cudaStreamSynchronize(e->stream));
    CU(cudaMemcpy(fftout, spec, sizeof(float2) * N, cudaMemcpyDeviceToHost));
    cudaFree(raw); cudaFree(spec); cudaFree(dk);
    return ABG_OK;
}

}  // extern "C"
