// ORACLE — TEST INFRASTRUCTURE ONLY.  Never linked, imported or executed by the product path.
//
// CPU restatement of the reference hot path demodulate() (reference src/rtl_airband.cpp:286-672) as a
// deterministic, single-writer function of (configuration, raw I/Q bytes):
//   * ring fill rule and hop                       rtl_airband.cpp:394-400, 669
//   * sample LUTs + 7-term Blackman-Harris window  rtl_airband.cpp:316-351
//   * convert + window                             rtl_airband.cpp:402-455 (non-VC branches)
//   * forward FFT                                  rtl_airband.cpp:460  (fftwf stand-in: oracle/fft32.cpp)
//   * bin extraction                               rtl_airband.cpp:483-489
//   * batch trigger, per-sample channel loop       rtl_airband.cpp:492-620
//   * history shift, AFC                           rtl_airband.cpp:621-629, 180-251
//   * output-thread tail copy, run synchronously   output.cpp:917-922
//   * initial channel/freq state                   config.cpp:265-281, 313-331
//   * sincos LUT, dBFS conversions                 util.cpp:103-127, 169-180
//   * bin / dm_dphi formulas                       config.cpp:666-667, 679-712
// Built twice (oracle/Makefile): with the restated leaf classes (leaf_dsp.cpp) and, as oracle/_ref, with the
// reference's own squelch.cpp / ctcss.cpp / filters.cpp compiled in place from /root/reference/src.
//
// PARITY PIN STATUS: the reference holds no golden vectors for this path (SURVEY.md §8c).  The leaf classes
// are pinned against the reference's own objects (oracle/_ref) and the upstream behavioural tests; the FFT
// call is pinned against numpy/scipy complex128 only ("parity unpinned" against fftw3f itself, which is not
// installable here); the loop body is a literal restatement.
#include "airband_oracle.h"

#include <math.h>
#include <stdint.h>
#include <string.h>
#include <time.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <deque>
#include <memory>
#include <pthread.h>
#include <sched.h>
#include <thread>
#include <vector>

#include "fft32.h"

#ifdef ABO_REF_LEAF
// reference classes, compiled in place from /root/reference/src (never copied into this repo)
#include "filters.h"
#include "squelch.h"
#define ABO_VARIANT "reference-leaf"
#else
#include "leaf_dsp.h"
using abo::CTCSS;
using abo::LowpassFilter;
using abo::NotchFilter;
using abo::Squelch;
#define ABO_VARIANT "restated"
#endif

namespace {

const int AGC_EXTRA = 100;  // rtl_airband.h:74
enum { NO_SIGNAL = ' ', SIGNAL = '*', AFC_UP = '<', AFC_DOWN = '>' };  // rtl_airband.h:101

// ---- util.cpp:103-127 -----------------------------------------------------------------------------------------
struct SinCosLut {
    float s[257], c[257];
    SinCosLut() {
        for (uint32_t i = 0; i < 256; i++) sincosf(2.0F * M_PI * (float)i / 256.0f, s + i, c + i);
        s[256] = s[0];
        c[256] = c[0];
    }
    void get(uint32_t phi, float* sine, float* cosine) const {
        uint32_t idx = phi >> 16;
        float fract = (float)(phi & 0xffff) / 65536.0f;
        float v1 = s[idx], v2 = s[idx + 1];
        *sine = v1 + (v2 - v1) * fract;
        v1 = c[idx];
        v2 = c[idx + 1];
        *cosine = v1 + (v2 - v1) * fract;
    }
};
const SinCosLut g_lut;

// ---- rtl_airband.cpp:141-176 ------------------------------------------------------------------------------------
inline void multiply(float ar, float aj, float br, float bj, float* cr, float* cj) {
    *cr = ar * br - aj * bj;
    *cj = aj * br + ar * bj;
}
float fast_atan2(float y, float x) {
    float yabs, angle;
    float pi4 = M_PI_4, pi34 = 3 * M_PI_4;
    if (x == 0.0f && y == 0.0f) return 0;
    yabs = y;
    if (yabs < 0.0f) yabs = -yabs;
    if (x >= 0.0f)
        angle = pi4 - pi4 * (x - yabs) / (x + yabs);
    else
        angle = pi34 - pi4 * (x + yabs) / (yabs - x);
    if (y < 0.0f) return -angle;
    return angle;
}
float polar_disc_fast(float ar, float aj, float br, float bj) {
    float cr, cj;
    multiply(ar, aj, br, -bj, &cr, &cj);
    return (float)(fast_atan2(cj, cr) * M_1_PI);
}
float fm_quadri_demod(float ar, float aj, float br, float bj) { return (float)((br * aj - ar * bj) / (ar * ar + aj * aj + 1.0f) * M_1_PI); }

// freq_t, rtl_airband.h:223-233
struct Freq {
    float agcavgfast = 0.5f, ampfactor = 1.0f;
    int modulation = ABO_MOD_AM;
    uint64_t active_counter = 0;
    Squelch squelch;
    NotchFilter notch_filter;
    LowpassFilter lowpass_filter;
};

struct Channel {
    // channel_t, rtl_airband.h:234-263 (only what the hot path touches)
    std::vector<float> wavein, waveout, iq_in, iq_out;
    float pr = 0, pj = 0, prev_waveout = 0.5f, alpha = 0;
    uint32_t dm_dphi = 0, dm_phi = 0;
    int axcindicate = NO_SIGNAL;
    int afc = 0;
    int needs_raw_iq = 0, has_iq_outputs = 0;
    // scan mode: freqlist / freq_idx, rtl_airband.h:250-252 (one entry unless abo_scan_configure() installs a list)
    std::vector<std::unique_ptr<Freq>> freqlist;
    int freq_idx = 0;
};

struct Batch {
    std::vector<float> waveout;  // C*B
    std::vector<float> iq_out;   // C*2B
    std::vector<char> axc;       // C
};

struct Device {
    int sfmt, bytes_per_sample, sample_rate;
    float fullscale;
    std::vector<unsigned char> in;  // raw bytes not yet consumed start at `bufs`
    size_t bufs = 0;
    std::vector<size_t> bins, base_bins;
    std::vector<std::unique_ptr<Channel>> ch;
    int waveend = 0;
    uint64_t batches_done = 0;
    std::deque<Batch> ready;
};

struct Oracle {
    int fft_size, wave_rate, wave_batch, wave_len, fm_demod;
    bool discard = false;
    std::vector<int> pin_cpus;  // worker thread t runs on pin_cpus[t % size] (timing runs; empty = scheduler's choice)
    std::vector<float> window;
    float levels_u8[256], levels_s8[256];
    std::vector<std::unique_ptr<Device>> devp;
    Device& D(int i) { return *devp[i]; }
    int ndev() const { return (int)devp.size(); }
};

// ---- AFC, rtl_airband.cpp:180-251 ----------------------------------------------------------------------------------
struct Afc {
    const int prev_axc;
    size_t fft_size;
    Afc(const Channel& c, size_t n) : prev_axc(c.axcindicate), fft_size(n) {}
    static float square(const float* f, size_t i) { return f[2 * i] * f[2 * i] + f[2 * i + 1] * f[2 * i + 1]; }
    template <int STEP>
    size_t check(const float* f, const size_t base, const float base_value, unsigned char afc) {
        float threshold = 0;
        size_t bin;
        for (bin = base;; bin += STEP) {
            if (STEP < 0) {
                if (bin < (size_t)-STEP) break;
            } else if ((size_t)(bin + STEP) >= fft_size)
                break;
            const float value = square(f, (size_t)(bin + STEP));
            if (value <= base_value) break;
            if (base == (size_t)bin) {
                threshold = (value - base_value) / (float)afc;
            } else {
                if ((value - base_value) < threshold) break;
                threshold += threshold / 10.0;
            }
        }
        return bin;
    }
    void finalize(Device& d, int index, const float* f) {
        Channel& c = *d.ch[index];
        if (c.afc == 0) return;
        const int axc = c.axcindicate;
        if (axc != NO_SIGNAL && prev_axc == NO_SIGNAL) {
            const size_t base = d.base_bins[index];
            const float base_value = square(f, base);
            size_t bin = check<-1>(f, base, base_value, (unsigned char)c.afc);
            if (bin == base) bin = check<1>(f, base, base_value, (unsigned char)c.afc);
            if (d.bins[index] != bin) {
                d.bins[index] = bin;
                if (bin > base)
                    c.axcindicate = AFC_UP;
                else if (bin < base)
                    c.axcindicate = AFC_DOWN;
            }
        } else if (axc == NO_SIGNAL && prev_axc != NO_SIGNAL)
            d.bins[index] = d.base_bins[index];
    }
};

struct Worker {  // the per-thread part of demod_params_t (fftin/fftout/plan), rtl_airband.h:310-320
    abo::Fft32 fft;
    std::vector<float> fftin, fftout;
    explicit Worker(size_t n) : fft(n), fftin(2 * n), fftout(2 * n) {}
};

// convert + window for one frame, rtl_airband.cpp:402-455
void convert_frame(const Oracle& o, const Device& d, const unsigned char* p, float* fftin) {
    const size_t N = o.fft_size;
    const float* window = o.window.data();
    if (d.sfmt == ABO_SFMT_S16) {
        float const scale = 1.0f / d.fullscale;
        const short* b = (const short*)p;
        for (size_t i = 0; i < N; i++, b += 2) {
            fftin[2 * i] = scale * (float)b[0] * window[i];
            fftin[2 * i + 1] = scale * (float)b[1] * window[i];
        }
    } else if (d.sfmt == ABO_SFMT_F32) {
        float const scale = 1.0f / d.fullscale;
        const float* b = (const float*)p;
        for (size_t i = 0; i < N; i++, b += 2) {
            fftin[2 * i] = scale * b[0] * window[i];
            fftin[2 * i + 1] = scale * b[1] * window[i];
        }
    } else {
        const float* lv = (d.sfmt == ABO_SFMT_U8 ? o.levels_u8 : o.levels_s8);
        for (size_t i = 0; i < N; i++, p += 2) {
            fftin[2 * i] = lv[p[0]] * window[i];
            fftin[2 * i + 1] = lv[p[1]] * window[i];
        }
    }
}

// one freq_t as parse_channels() sets it up (config.cpp:437-619: level first, SNR (if given) afterwards)
std::unique_ptr<Freq> make_freq(const abo_channel_cfg& cc, int wave_rate) {
    std::unique_ptr<Freq> fp(new Freq());
    Freq& f = *fp;
    f.ampfactor = cc.ampfactor;
    f.modulation = cc.modulation;
    if (cc.squelch_level > 0) f.squelch.set_squelch_level_threshold(cc.squelch_level);
    if (cc.squelch_snr_db >= 0) f.squelch.set_squelch_snr_threshold(cc.squelch_snr_db);
    if (cc.notch_hz > 0) f.notch_filter = NotchFilter(cc.notch_hz, wave_rate, cc.notch_q);
    if (cc.ctcss_hz > 0) f.squelch.set_ctcss_freq(cc.ctcss_hz, wave_rate);
    if (cc.lowpass_hz > 0) f.lowpass_filter = LowpassFilter(cc.lowpass_hz, wave_rate);
    return fp;
}

// the per-sample channel loop of one batch, rtl_airband.cpp:495-648
void demod_batch(Oracle& o, Device& d, const float* last_fftout) {
    const int B = o.wave_batch;
    for (size_t i = 0; i < d.ch.size(); i++) {
        Channel& c = *d.ch[i];
        Freq& f = *c.freqlist[c.freq_idx];  // fparms = channel->freqlist + channel->freq_idx, rtl_airband.cpp:498
        Afc afc(c, o.fft_size);
        c.axcindicate = NO_SIGNAL;
        for (int j = AGC_EXTRA; j < B + AGC_EXTRA; j++) {
            float& real = c.iq_in[2 * (j - AGC_EXTRA)];
            float& imag = c.iq_in[2 * (j - AGC_EXTRA) + 1];

            f.squelch.process_raw_sample(c.wavein[j]);

            if (f.squelch.should_filter_sample() && c.needs_raw_iq) {
                float swf, cwf, re_tmp, im_tmp;
                g_lut.get(c.dm_phi, &swf, &cwf);
                multiply(real, imag, cwf, -swf, &re_tmp, &im_tmp);
                c.dm_phi += c.dm_dphi;
                c.dm_phi &= 0xffffff;
                f.lowpass_filter.apply(re_tmp, im_tmp);
                real = re_tmp;
                imag = im_tmp;
                c.wavein[j] = sqrt(real * real + imag * imag);
                if (f.lowpass_filter.enabled()) f.squelch.process_filtered_sample(c.wavein[j]);
            }

            if (f.modulation == ABO_MOD_AM) {
                if (f.squelch.first_open_sample()) {
                    for (int k = j - AGC_EXTRA; k < j; k++) {
                        if (c.wavein[k] >= f.squelch.squelch_level()) f.agcavgfast = f.agcavgfast * 0.9f + c.wavein[k] * 0.1f;
                    }
                } else if (f.squelch.last_open_sample()) {
                    for (int k = j - AGC_EXTRA + 1; k < j; k++) c.waveout[k] = c.waveout[k - 1] * 0.94f;
                }
            }

            float& waveout = c.waveout[j];

            if (f.squelch.should_process_audio()) {
                if (f.modulation == ABO_MOD_AM) {
                    if (c.wavein[j] > f.squelch.squelch_level()) f.agcavgfast = f.agcavgfast * 0.995f + c.wavein[j] * 0.005f;
                    waveout = (c.wavein[j - AGC_EXTRA] - f.agcavgfast) / (f.agcavgfast * 1.5f);
                    if (std::abs(waveout) > 0.8f) {
                        waveout *= 0.85f;
                        f.agcavgfast *= 1.15f;
                    }
                } else if (f.modulation == ABO_MOD_NFM) {
                    if (o.fm_demod == ABO_FM_FAST_ATAN2)
                        waveout = polar_disc_fast(real, imag, c.pr, c.pj);
                    else if (o.fm_demod == ABO_FM_QUADRI_DEMOD)
                        waveout = fm_quadri_demod(real, imag, c.pr, c.pj);
                    c.pr = real;
                    c.pj = imag;
                    f.agcavgfast = f.agcavgfast * 0.995f + waveout * 0.005f;
                    waveout -= f.agcavgfast;
                    waveout = waveout * (1.0f - c.alpha) + c.prev_waveout * c.alpha;
                    c.prev_waveout = waveout;
                }
                f.squelch.process_audio_sample(waveout);
            }

            if (f.squelch.is_open()) {
                f.notch_filter.apply(waveout);
                waveout *= f.ampfactor;
                if (std::isnan(waveout)) {
                    waveout = 0.0;
                } else if (waveout > 1.0) {
                    waveout = 1.0;
                } else if (waveout < -1.0) {
                    waveout = -1.0;
                }
                c.axcindicate = SIGNAL;
                if (c.has_iq_outputs) {
                    c.iq_out[2 * (j - AGC_EXTRA)] = real;
                    c.iq_out[2 * (j - AGC_EXTRA) + 1] = imag;
                }
            } else {
                waveout = 0;
                if (c.has_iq_outputs) {
                    c.iq_out[2 * (j - AGC_EXTRA)] = 0;
                    c.iq_out[2 * (j - AGC_EXTRA) + 1] = 0;
                }
            }
        }
        memmove(c.wavein.data(), c.wavein.data() + B, (d.waveend - B) * sizeof(float));
        if (c.needs_raw_iq) memmove(c.iq_in.data(), c.iq_in.data() + 2 * B, (d.waveend - B) * sizeof(float) * 2);

        afc.finalize(d, (int)i, last_fftout);

        if (c.axcindicate != NO_SIGNAL) f.active_counter++;
    }

    // output thread, run synchronously: consume waveout[0..B) / iq_out[0..2B), then the tail copy (output.cpp:917-922)
    if (!o.discard) {
        Batch b;
        const size_t C = d.ch.size();
        b.waveout.resize(C * B);
        b.iq_out.resize(C * 2 * B);
        b.axc.resize(C);
        for (size_t i = 0; i < C; i++) {
            Channel& c = *d.ch[i];
            memcpy(&b.waveout[i * B], c.waveout.data(), B * sizeof(float));
            memcpy(&b.iq_out[i * 2 * B], c.iq_out.data(), 2 * B * sizeof(float));
            b.axc[i] = (char)c.axcindicate;
        }
        d.ready.push_back(std::move(b));
    }
    for (auto& cp : d.ch) memcpy(cp->waveout.data(), cp->waveout.data() + B, AGC_EXTRA * 4);
    d.waveend -= B;
    d.batches_done++;
}

// one device: consume frames while the ring rule allows it (rtl_airband.cpp:394-400) and the batch cap is not hit
long run_device(Oracle& o, Device& d, Worker& w, int max_batches) {
    const size_t N = o.fft_size;
    const size_t bps = 2 * d.bytes_per_sample * (size_t)round((double)d.sample_rate / (double)o.wave_rate);
    const size_t need = bps + N * d.bytes_per_sample * 2;
    long produced = 0;
    while (max_batches < 0 || produced < max_batches) {
        size_t available = d.in.size() - d.bufs;
        if (available < need) break;
        convert_frame(o, d, d.in.data() + d.bufs, w.fftin.data());
        w.fft.forward(w.fftin.data(), w.fftout.data());
        const float* fo = w.fftout.data();
        for (size_t j = 0; j < d.ch.size(); j++) {
            Channel& c = *d.ch[j];
            const size_t b = d.bins[j];
            c.wavein[d.waveend] = sqrtf(fo[2 * b] * fo[2 * b] + fo[2 * b + 1] * fo[2 * b + 1]);
            if (c.needs_raw_iq) {
                c.iq_in[2 * d.waveend] = fo[2 * b];
                c.iq_in[2 * d.waveend + 1] = fo[2 * b + 1];
            }
        }
        d.waveend += 1;
        if (d.waveend >= o.wave_batch + AGC_EXTRA) {
            demod_batch(o, d, fo);
            produced++;
        }
        d.bufs += bps;
    }
    // drop consumed bytes now and then so long runs do not grow without bound
    if (d.bufs > (1u << 22)) {
        d.in.erase(d.in.begin(), d.in.begin() + d.bufs);
        d.bufs = 0;
    }
    return produced;
}

}  // namespace

// =================================================================================================================
// C ABI
// =================================================================================================================
#pragma GCC visibility push(default)
extern "C" {

const char* abo_variant(void) { return ABO_VARIANT; }

void* abo_create(const abo_config* cfg) {
    if (!cfg || cfg->fft_size < 256 || cfg->fft_size > 8192 || (cfg->fft_size & (cfg->fft_size - 1))) return nullptr;
    if (cfg->wave_rate <= 0 || cfg->wave_rate % 8) return nullptr;
    Oracle* o = new Oracle();
    o->fft_size = cfg->fft_size;
    o->wave_rate = cfg->wave_rate;
    o->wave_batch = cfg->wave_rate / 8;               // rtl_airband.h:73
    o->wave_len = 2 * o->wave_batch + AGC_EXTRA;      // rtl_airband.h:75
    o->fm_demod = cfg->fm_demod;
    // rtl_airband.cpp:319-324
    for (int i = 0; i < 256; i++) o->levels_u8[i] = (i - 127.5f) / 127.5f;
    for (int16_t i = -127; i < 128; i++) o->levels_s8[(uint8_t)i] = i / 128.0f;
    o->levels_s8[128] = -128 / 128.0f;  // (uint8_t)-128 is never written by the reference loop (stack garbage there); we extend i/128
    // rtl_airband.cpp:335-351 — float literals stored in double, evaluated in double, rounded to float
    const double a0 = 0.27105140069342f, a1 = 0.43329793923448f, a2 = 0.21812299954311f, a3 = 0.06592544638803f;
    const double a4 = 0.01081174209837f, a5 = 0.00077658482522f, a6 = 0.00001388721735f;
    const size_t fft_size = o->fft_size;
    o->window.resize(fft_size);
    for (size_t i = 0; i < fft_size; i++) {
        double x = a0 - (a1 * cos((2.0 * M_PI * i) / (fft_size - 1))) + (a2 * cos((4.0 * M_PI * i) / (fft_size - 1))) - (a3 * cos((6.0 * M_PI * i) / (fft_size - 1))) +
                   (a4 * cos((8.0 * M_PI * i) / (fft_size - 1))) - (a5 * cos((10.0 * M_PI * i) / (fft_size - 1))) + (a6 * cos((12.0 * M_PI * i) / (fft_size - 1)));
        o->window[i] = (float)x;
    }
    for (int di = 0; di < cfg->n_devices; di++) o->devp.emplace_back(new Device());
    for (int di = 0; di < cfg->n_devices; di++) {
        const abo_device_cfg& dc = cfg->devices[di];
        Device& d = o->D(di);
        d.sfmt = dc.sfmt;
        d.fullscale = dc.fullscale;
        d.sample_rate = dc.sample_rate;
        switch (dc.sfmt) {
            case ABO_SFMT_U8:
            case ABO_SFMT_S8: d.bytes_per_sample = 1; break;
            case ABO_SFMT_S16: d.bytes_per_sample = 2; break;
            case ABO_SFMT_F32: d.bytes_per_sample = 4; break;
            default: delete o; return nullptr;
        }
        for (int ci = 0; ci < dc.n_channels; ci++) {
            const abo_channel_cfg& cc = dc.channels[ci];
            std::unique_ptr<Channel> cp(new Channel());
            Channel& c = *cp;
            c.wavein.assign(o->wave_len, 0.0f);
            c.waveout.assign(o->wave_len, 0.0f);
            c.iq_in.assign(2 * o->wave_len, 0.0f);
            c.iq_out.assign(2 * o->wave_len, 0.0f);
            for (int k = 0; k < AGC_EXTRA; k++) {  // config.cpp:313-316
                c.wavein[k] = 20;
                c.waveout[k] = 0.5;
            }
            c.alpha = cc.alpha;
            c.dm_dphi = cc.dm_dphi;
            c.afc = cc.afc;
            c.needs_raw_iq = cc.needs_raw_iq;
            c.has_iq_outputs = cc.has_iq_outputs;
            c.freqlist.push_back(make_freq(cc, o->wave_rate));
            d.bins.push_back((size_t)cc.bin);
            d.base_bins.push_back((size_t)cc.bin);
            d.ch.push_back(std::move(cp));
        }
    }
    return o;
}

void abo_destroy(void* h) { delete (Oracle*)h; }
int abo_wave_batch(void* h) { return ((Oracle*)h)->wave_batch; }

int abo_push(void* h, int dev, const void* iq, size_t nbytes) {
    Oracle* o = (Oracle*)h;
    if (dev < 0 || dev >= o->ndev()) return -1;
    Device& d = o->D(dev);
    const unsigned char* p = (const unsigned char*)iq;
    d.in.insert(d.in.end(), p, p + nbytes);
    return 0;
}

long abo_run(void* h, int max_batches, int n_threads) {
    Oracle* o = (Oracle*)h;
    const int D = o->ndev();
    if (n_threads <= 1 || D <= 1) {
        Worker w(o->fft_size);
        long total = 0;
        for (auto& dp : o->devp) total += run_device(*o, *dp, w, max_batches);
        return total;
    }
    n_threads = std::min(n_threads, D);
    std::vector<long> part(n_threads, 0);
    std::vector<std::thread> th;
    for (int t = 0; t < n_threads; t++) {
        th.emplace_back([&, t]() {
            if (!o->pin_cpus.empty()) {
                cpu_set_t set;
                CPU_ZERO(&set);
                CPU_SET(o->pin_cpus[t % o->pin_cpus.size()], &set);
                pthread_setaffinity_np(pthread_self(), sizeof(set), &set);
            }
            Worker w(o->fft_size);
            // contiguous device ranges like init_demod(device_start, device_end), rtl_airband.cpp:1070-1086
            int lo = (int)((long)D * t / n_threads), hi = (int)((long)D * (t + 1) / n_threads);
            for (int i = lo; i < hi; i++) part[t] += run_device(*o, o->D(i), w, max_batches);
        });
    }
    for (auto& t : th) t.join();
    long total = 0;
    for (long p : part) total += p;
    return total;
}

// stage tap (mirrors abg_debug_inject_wavein): wavein[C][n_batches * B] becomes channel_t.wavein[AGC_EXTRA ...] and iq_in
// [C][n_batches * B][2] channel_t.iq_in[2 * AGC_EXTRA ...] (where run_device() stores frame waveend), batch by batch
int abo_debug_inject_wavein(void* h, int dev, int n_batches, const float* wavein, const float* iq_in) {
    Oracle* o = (Oracle*)h;
    if (dev < 0 || dev >= o->ndev() || n_batches < 1 || !wavein) return -1;
    Device& d = o->D(dev);
    const int B = o->wave_batch;
    for (auto& cp : d.ch)
        if ((cp->needs_raw_iq && !iq_in) || cp->afc) return -1;
    if (d.waveend != 0 && d.waveend != AGC_EXTRA) return -1;  // mixing injection with real frames is not supported
    for (int b = 0; b < n_batches; b++) {
        for (size_t c = 0; c < d.ch.size(); c++) {
            memcpy(d.ch[c]->wavein.data() + AGC_EXTRA, wavein + (c * (size_t)n_batches + b) * B, sizeof(float) * B);
            if (iq_in && d.ch[c]->needs_raw_iq)
                memcpy(d.ch[c]->iq_in.data() + 2 * AGC_EXTRA, iq_in + 2 * ((c * (size_t)n_batches + b) * B), sizeof(float) * 2 * B);
        }
        d.waveend = B + AGC_EXTRA;
        demod_batch(*o, d, nullptr);
    }
    return n_batches;
}

void abo_set_discard(void* h, int discard) { ((Oracle*)h)->discard = discard != 0; }
void abo_set_pin(void* h, const int* cpus, int n) {
    Oracle* o = (Oracle*)h;
    o->pin_cpus.assign(cpus, cpus + (n > 0 ? n : 0));
}
int abo_batches_ready(void* h, int dev) { return (int)((Oracle*)h)->D(dev).ready.size(); }

int abo_fetch_batch(void* h, int dev, float* waveout, float* iq_out, char* axc) {
    Oracle* o = (Oracle*)h;
    Device& d = o->D(dev);
    if (d.ready.empty()) return 0;
    Batch& b = d.ready.front();
    if (waveout) memcpy(waveout, b.waveout.data(), b.waveout.size() * sizeof(float));
    if (iq_out) memcpy(iq_out, b.iq_out.data(), b.iq_out.size() * sizeof(float));
    if (axc) memcpy(axc, b.axc.data(), b.axc.size());
    d.ready.pop_front();
    return 1;
}

int abo_get_stats(void* h, int dev, int chan, abo_squelch_stats* out) {
    Oracle* o = (Oracle*)h;
    if (dev < 0 || dev >= o->ndev()) return -1;
    Device& d = o->D(dev);
    if (chan < 0 || chan >= (int)d.ch.size()) return -1;
    Channel& c = *d.ch[chan];
    Freq& f = *c.freqlist[c.freq_idx];
    out->noise_level = f.squelch.noise_level();
    out->signal_level = f.squelch.signal_level();
    out->squelch_level = f.squelch.squelch_level();
    out->open_count = f.squelch.open_count();
    out->flappy_count = f.squelch.flappy_count();
    out->ctcss_count = f.squelch.ctcss_count();
    out->no_ctcss_count = f.squelch.no_ctcss_count();
    out->agcavgfast = f.agcavgfast;
    out->dm_phi = c.dm_phi;
    out->bin = (int32_t)d.bins[chan];
    out->active_counter = f.active_counter;
    out->noise_level_dbfs = abo_level_to_dbfs(out->noise_level, o->fft_size);
    out->signal_level_dbfs = abo_level_to_dbfs(out->signal_level, o->fft_size);
    out->squelch_level_dbfs = abo_level_to_dbfs(out->squelch_level, o->fft_size);
    return 0;
}

// scan mode: install a frequency list for one channel (entry 0 becomes current, every entry starts from a fresh freq_t)
int abo_scan_configure(void* h, int dev, int chan, int n_freqs, const abo_channel_cfg* freqs) {
    Oracle* o = (Oracle*)h;
    if (dev < 0 || dev >= o->ndev() || n_freqs < 1 || !freqs) return -1;
    Device& d = o->D(dev);
    if (chan < 0 || chan >= (int)d.ch.size()) return -1;
    Channel& c = *d.ch[chan];
    c.freqlist.clear();
    for (int i = 0; i < n_freqs; i++) c.freqlist.push_back(make_freq(freqs[i], o->wave_rate));
    c.freq_idx = 0;
    return 0;
}

// what controller_thread does to channels[0].freq_idx (rtl_airband.cpp:117-119); takes effect with the next batch (:498)
int abo_scan_select(void* h, int dev, int chan, int freq_idx) {
    Oracle* o = (Oracle*)h;
    if (dev < 0 || dev >= o->ndev()) return -1;
    Device& d = o->D(dev);
    if (chan < 0 || chan >= (int)d.ch.size()) return -1;
    Channel& c = *d.ch[chan];
    if (freq_idx < 0 || freq_idx >= (int)c.freqlist.size()) return -1;
    c.freq_idx = freq_idx;
    return 0;
}

int abo_set_bin(void* h, int dev, int chan, int bin) {
    Oracle* o = (Oracle*)h;
    Device& d = o->D(dev);
    d.bins[chan] = d.base_bins[chan] = (size_t)bin;
    return 0;
}

int abo_get_window(void* h, float* window) {
    Oracle* o = (Oracle*)h;
    memcpy(window, o->window.data(), o->window.size() * sizeof(float));
    return 0;
}

int abo_debug_frame(void* h, int dev, const void* iq_frame, float* fftin, float* fftout) {
    Oracle* o = (Oracle*)h;
    Worker w(o->fft_size);
    convert_frame(*o, o->D(dev), (const unsigned char*)iq_frame, w.fftin.data());
    w.fft.forward(w.fftin.data(), w.fftout.data());
    if (fftin) memcpy(fftin, w.fftin.data(), w.fftin.size() * sizeof(float));
    if (fftout) memcpy(fftout, w.fftout.data(), w.fftout.size() * sizeof(float));
    return 0;
}

// ---- config formulas --------------------------------------------------------------------------------------------
int32_t abo_calc_bin(int32_t freq, int32_t centerfreq, int32_t sample_rate, int32_t fft_size) {
    // config.cpp:666-667 — note the INTEGER division sample_rate / fft_size
    size_t fs = (size_t)fft_size;
    return (int32_t)((size_t)ceil((freq + sample_rate - centerfreq) / (double)(sample_rate / fs) - 1.0) % fs);
}

uint32_t abo_calc_dm_dphi(int32_t freq, int32_t centerfreq, int32_t sample_rate, int32_t wave_rate) {
    // config.cpp:679-712
    double dm_dphi = (double)(freq - centerfreq);
    double decimation_factor = ((double)sample_rate / (double)wave_rate);
    double dm_dphi_correction = (double)wave_rate / 2.0;
    dm_dphi_correction *= (decimation_factor - round(decimation_factor));
    dm_dphi_correction *= (double)(freq - centerfreq) / ((double)sample_rate / 2.0);
    dm_dphi -= dm_dphi_correction;
    dm_dphi /= (double)wave_rate;
    dm_dphi -= trunc(dm_dphi);
    dm_dphi *= 256.0 * 65536.0;
    return (uint32_t)((int)dm_dphi);
}

static float dbfs_offset(int32_t fft_size) { return 7.54f + 10.0f * log10f((size_t)fft_size / 2) - 2.38f; }  // util.cpp:169-172
float abo_dbfs_to_level(float dbfs, int32_t fft_size) { return pow(10.0, (dbfs - dbfs_offset(fft_size)) / 20.0f) * (size_t)fft_size; }
float abo_level_to_dbfs(float level, int32_t fft_size) { return std::min(0.0f, 20.0f * log10f(level / (size_t)fft_size) + dbfs_offset(fft_size)); }
float abo_default_alpha(int32_t wave_rate) { return exp(-1.0f / (wave_rate * 2e-4)); }  // rtl_airband.cpp:87
void abo_sincosf_lut(uint32_t phi, float* s, float* c) { g_lut.get(phi, s, c); }
float abo_fast_atan2(float y, float x) { return fast_atan2(y, x); }
float abo_polar_disc_fast(float ar, float aj, float br, float bj) { return polar_disc_fast(ar, aj, br, bj); }
float abo_fm_quadri_demod(float ar, float aj, float br, float bj) { return fm_quadri_demod(ar, aj, br, bj); }
// seconds per transform of the oracle's FFT stand-in with a persistent plan (what the demod loop pays per frame); lets the
// CPU baseline say how far its FFT is from FFTW-class throughput on the box it ran on
double abo_fft_seconds(int n, int reps) {
    abo::Fft32 f(n);
    std::vector<float> a(2 * (size_t)n), b(2 * (size_t)n);
    for (size_t i = 0; i < a.size(); i++) a[i] = (float)((i * 7919u) % 1000u) / 1000.0f - 0.5f;
    for (int i = 0; i < 16; i++) f.forward(a.data(), b.data());
    timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    for (int i = 0; i < reps; i++) f.forward(a.data(), b.data());
    clock_gettime(CLOCK_MONOTONIC, &t1);
    volatile float sink = b[1];
    (void)sink;
    return ((t1.tv_sec - t0.tv_sec) + 1e-9 * (t1.tv_nsec - t0.tv_nsec)) / (reps > 0 ? reps : 1);
}
void abo_fft(int n, const float* in, float* out) {
    abo::Fft32 f(n);
    f.forward(in, out);
}

// ---- leaf harness -------------------------------------------------------------------------------------------------
void* abo_sq_new(void) { return new Squelch(); }
void abo_sq_free(void* s) { delete (Squelch*)s; }
void abo_sq_set_level(void* s, float level) { ((Squelch*)s)->set_squelch_level_threshold(level); }
void abo_sq_set_snr(void* s, float db) { ((Squelch*)s)->set_squelch_snr_threshold(db); }
void abo_sq_set_ctcss(void* s, float freq, float sample_rate) { ((Squelch*)s)->set_ctcss_freq(freq, sample_rate); }
void abo_sq_raw(void* s, float v) { ((Squelch*)s)->process_raw_sample(v); }
void abo_sq_filtered(void* s, float v) { ((Squelch*)s)->process_filtered_sample(v); }
void abo_sq_audio(void* s, float v) { ((Squelch*)s)->process_audio_sample(v); }
int abo_sq_is_open(void* s) { return ((Squelch*)s)->is_open(); }
int abo_sq_should_filter(void* s) { return ((Squelch*)s)->should_filter_sample(); }
int abo_sq_should_process_audio(void* s) { return ((Squelch*)s)->should_process_audio(); }
int abo_sq_first_open(void* s) { return ((Squelch*)s)->first_open_sample(); }
int abo_sq_last_open(void* s) { return ((Squelch*)s)->last_open_sample(); }
int abo_sq_outside_filter(void* s) { return ((Squelch*)s)->signal_outside_filter(); }
float abo_sq_noise_level(void* s) { return ((Squelch*)s)->noise_level(); }
float abo_sq_signal_level(void* s) { return ((Squelch*)s)->signal_level(); }
float abo_sq_squelch_level(void* s) { return ((Squelch*)s)->squelch_level(); }
uint64_t abo_sq_open_count(void* s) { return ((Squelch*)s)->open_count(); }
uint64_t abo_sq_flappy_count(void* s) { return ((Squelch*)s)->flappy_count(); }
uint64_t abo_sq_ctcss_count(void* s) { return ((Squelch*)s)->ctcss_count(); }
uint64_t abo_sq_no_ctcss_count(void* s) { return ((Squelch*)s)->no_ctcss_count(); }

void abo_sq_trace(void* sp, int n, const float* raw, const float* filtered, const float* audio, float* levels, int32_t* flags) {
    Squelch& s = *(Squelch*)sp;
    for (int i = 0; i < n; i++) {
        s.process_raw_sample(raw[i]);
        bool filt = s.should_filter_sample();
        if (filtered && filt) s.process_filtered_sample(filtered[i]);
        bool first = s.first_open_sample(), last = s.last_open_sample();
        bool aud = s.should_process_audio();
        if (audio && aud) s.process_audio_sample(audio[i]);
        bool open = s.is_open();
        levels[4 * i + 0] = s.noise_level();
        levels[4 * i + 1] = s.signal_level();
        levels[4 * i + 2] = s.squelch_level();
        levels[4 * i + 3] = 0;
        flags[i] = (open ? 1 : 0) | (filt ? 2 : 0) | (aud ? 4 : 0) | (first ? 8 : 0) | (last ? 16 : 0) | (s.signal_outside_filter() ? 32 : 0);
    }
}

void* abo_ctcss_new(float freq, float sample_rate, int window) {
    if (freq <= 0) return new CTCSS();
    return new CTCSS(freq, sample_rate, window);
}
void abo_ctcss_free(void* c) { delete (CTCSS*)c; }
void abo_ctcss_sample(void* c, float v) { ((CTCSS*)c)->process_audio_sample(v); }
int abo_ctcss_enabled(void* c) { return ((CTCSS*)c)->is_enabled(); }
int abo_ctcss_enough(void* c) { return ((CTCSS*)c)->enough_samples(); }
int abo_ctcss_has_tone(void* c) { return ((CTCSS*)c)->has_tone(); }
void abo_ctcss_reset(void* c) { ((CTCSS*)c)->reset(); }
uint64_t abo_ctcss_found(void* c) { return ((CTCSS*)c)->found_count(); }
uint64_t abo_ctcss_not_found(void* c) { return ((CTCSS*)c)->not_found_count(); }

void abo_notch_run(float freq, float sample_rate, float q, int n, float* inout) {
    NotchFilter f(freq, sample_rate, q);
    for (int i = 0; i < n; i++) f.apply(inout[i]);
}
void abo_lowpass_run(float freq, float sample_rate, int n, float* inout_iq) {
    LowpassFilter f(freq, sample_rate);
    for (int i = 0; i < n; i++) f.apply(inout_iq[2 * i], inout_iq[2 * i + 1]);
}

}  // extern "C"
#pragma GCC visibility pop
