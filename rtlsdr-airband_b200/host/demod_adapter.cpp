// demodulate_b200(): the reference's demod thread function re-expressed over the C ABI of the GPU engine.
// Same contract as demodulate() (reference src/rtl_airband.cpp:286-672): it owns devices[device_start..device_end),
// consumes each input ring under the reference's locking discipline (:370-375, bufs advanced without the lock, :669),
// follows the input state machine (:377-391, including disable_device_outputs() for a dead receiver), delivers finished
// batches into channel_t.waveout / iq_out / axcindicate, bumps active_counter (:645-647), raises waveavail or counts an
// overrun (:649-654), and signals the output thread (:662).  Mixers whose inputs all live on this thread's devices are
// summed on the GPU and handed to the output thread through mixer_t.channel with the reference's CH_DIRTY -> CH_WORKING ->
// CH_READY handshake (mixer.cpp:157-261 producer side, output.cpp:888-896 consumer side).  Fatal engine errors are
// reported like the VideoCore branch does (:296-310): message + exit.
//
// One source, two bindings (b200_adapter.h): the reference's own structs (ABG_WITH_REFERENCE_HEADERS, inside the reference
// tree) or the mirror of the same fields used by this repository's tests.
#include "b200_adapter.h"

#include <errno.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <deque>
#include <vector>

b200_globals g_b200;

#ifndef ABG_WITH_REFERENCE_HEADERS
void Signal::wait_ms(int ms) {
    timespec ts;
    clock_gettime(CLOCK_REALTIME, &ts);
    ts.tv_nsec += (long)(ms % 1000) * 1000000L;
    ts.tv_sec += ms / 1000 + ts.tv_nsec / 1000000000L;
    ts.tv_nsec %= 1000000000L;
    pthread_mutex_lock(&mutex_);
    pthread_cond_timedwait(&cond_, &mutex_, &ts);
    pthread_mutex_unlock(&mutex_);
}
#endif

static void fatal(const char* what) {
    snprintf(g_b200.last_error, sizeof(g_b200.last_error), "%s: %s", what, abg_last_error());
#ifdef ABG_WITH_REFERENCE_HEADERS
    log(LOG_CRIT, "%s\n", g_b200.last_error);
    error();
#else
    fprintf(stderr, "%s\n", g_b200.last_error);
    bd::exit_flag() = 1;  // error() = _Exit(1) in the reference tree; the test harness wants to survive
#endif
}

// channel_t / freq_t -> abg_channel_cfg
static void fill_channel_cfg(const device_t* dev, int c, const freq_t* f, abg_channel_cfg* out) {
    const channel_t* ch = dev->channels + c;
    abg_channel_cfg& o = *out;
    memset(&o, 0, sizeof(o));
    o.bin = (int32_t)dev->bins[c];
    o.modulation = bd::is_nfm(f) ? ABG_MOD_NFM : ABG_MOD_AM;
    o.needs_raw_iq = ch->needs_raw_iq;
    o.has_iq_outputs = ch->has_iq_outputs;
    o.dm_dphi = ch->dm_dphi;
    o.alpha = bd::channel_alpha(ch);
    o.ampfactor = f->ampfactor;
    o.squelch_level = f->b200_cfg.squelch_level;
    o.squelch_snr_db = f->b200_cfg.squelch_snr_db;
    o.lowpass_hz = f->b200_cfg.lowpass_hz;
    o.notch_hz = f->b200_cfg.notch_hz;
    o.notch_q = f->b200_cfg.notch_q;
    o.ctcss_hz = f->b200_cfg.ctcss_hz;
    o.afc = ch->afc;
}

// ---- mixers summed on the GPU -------------------------------------------------------------------------------------------
namespace {
struct GpuMixer {
    mixer_t* mixer;  // the reference's object; its channel receives the sums
};
std::vector<GpuMixer> g_gpu_mixers;  // engine mixer index -> mixer (one demod thread owns a mixer entirely, or it stays on the CPU path)
std::vector<int> g_mixer_devs;        // engine device indices that feed a GPU-summed mixer
}  // namespace

// process_outputs() asks this before mixer_put_samples (output.cpp:533-535): inputs of a GPU-summed mixer are not put again
extern "C" ABG_API int b200_mixer_is_gpu(const mixer_t* m) {
    for (const GpuMixer& g : g_gpu_mixers)
        if (g.mixer == m) return 1;
    return 0;
}

// Mixers all of whose inputs are channels of devices[d0, d1): (dev, chan, ampfactor, balance) per input in input order.
static int configure_gpu_mixers(abg_engine* eng, device_t* devices, int d0, int d1) {
    g_gpu_mixers.clear();
    mixer_t* mixers = bd::mixer_array();
    const int nm = bd::mixer_n();
    if (!mixers || nm <= 0) return ABG_OK;
    std::vector<std::vector<abg_mixer_input>> found(nm);
    std::vector<std::vector<int>> slot(nm);
    for (int i = d0; i < d1; i++) {
        device_t* dev = devices + i;
        for (int c = 0; c < dev->channel_count; c++) {
            channel_t* ch = dev->channels + c;
            for (int k = 0; k < ch->output_count; k++) {
                if (ch->outputs[k].type != O_MIXER || !ch->outputs[k].enabled) continue;
                mixer_data* md = (mixer_data*)ch->outputs[k].data;
                const int m = (int)(md->mixer - mixers);
                if (m < 0 || m >= nm) continue;
                const mixinput_t& in = md->mixer->inputs[md->input];
                abg_mixer_input mi;
                mi.dev = i - d0;
                mi.chan = c;
                mi.ampfactor = in.ampfactor;
                // ampl = fminf(1, 1 - balance), ampr = fminf(1, 1 + balance) (mixer.cpp:82-83), inverted
                mi.balance = in.ampl < 1.0f ? 1.0f - in.ampl : (in.ampr < 1.0f ? in.ampr - 1.0f : 0.0f);
                found[m].push_back(mi);
                slot[m].push_back(md->input);
            }
        }
    }
    std::vector<int32_t> offs(1, 0);
    std::vector<abg_mixer_input> flat;
    for (int m = 0; m < nm; m++) {
        if (!mixers[m].enabled || (int)found[m].size() != mixers[m].input_count || found[m].empty()) continue;  // some input lives elsewhere
        std::vector<int> order(found[m].size());
        for (size_t k = 0; k < order.size(); k++) order[k] = (int)k;
        std::sort(order.begin(), order.end(), [&](int a, int b) { return slot[m][a] < slot[m][b]; });  // mix in input order (mixer.cpp:189)
        for (int k : order) flat.push_back(found[m][k]);
        offs.push_back((int32_t)flat.size());
        g_gpu_mixers.push_back(GpuMixer{mixers + m});
    }
    g_mixer_devs.clear();
    for (const abg_mixer_input& mi : flat)
        if (std::find(g_mixer_devs.begin(), g_mixer_devs.end(), mi.dev) == g_mixer_devs.end()) g_mixer_devs.push_back(mi.dev);
    if (g_gpu_mixers.empty()) return ABG_OK;
    return abg_mixers_configure(eng, (int)g_gpu_mixers.size(), offs.data(), flat.data());
}

// Producer side of the mixer hand-off (what mixer_thread does once all inputs are in, mixer.cpp:186-252).
static bool deliver_mixers(abg_engine* eng, Signal* sig, int B, std::vector<float>& left, std::vector<float>& right) {
    bool any = false;
    left.resize(B);
    right.resize(B);
    for (size_t em = 0; em < g_gpu_mixers.size(); em++) {
        mixer_t* mixer = g_gpu_mixers[em].mixer;
        channel_t* channel = &mixer->channel;
        for (;;) {
            if (g_b200.wait_for_consumer && channel->state == CH_READY) break;  // offline pacing: the output thread has not taken the last one yet
            int has_signal = 0;
            int rc = abg_fetch_mixer_batch(eng, (int)em, left.data(), right.data(), &has_signal);
            if (rc <= 0) break;
            if (channel->state == CH_READY) mixer->output_overrun_count++;  // previous output not yet handled (mixer.cpp:163-170)
            channel->state = CH_WORKING;
            memcpy(channel->waveout, left.data(), sizeof(float) * B);
            if (channel->mode == MM_STEREO) memcpy(channel->waveout_r, right.data(), sizeof(float) * B);
            channel->axcindicate = has_signal ? SIGNAL : NO_SIGNAL;
            channel->state = CH_READY;
            sig->send();
            any = true;
            if (g_b200.wait_for_consumer) break;
        }
    }
    return any;
}

extern "C" void* demodulate_b200(void* params) {
    demod_params_t* dp = (demod_params_t*)params;
    const int d0 = dp->device_start, d1 = dp->device_end, nd = d1 - d0;
    device_t* devices = bd::devs();
    const int B = bd::wave_rate() / 8;  // WAVE_BATCH

    // ---- engine set-up: init_demod() + top of demodulate() (:253-266,292-351) ----
    std::vector<abg_device_cfg> dcfg(nd);
    std::vector<std::vector<abg_channel_cfg>> ccfg(nd);
    for (int i = 0; i < nd; i++) {
        device_t* dev = devices + d0 + i;
        ccfg[i].resize(dev->channel_count);
        for (int c = 0; c < dev->channel_count; c++) {
            channel_t* ch = dev->channels + c;
            fill_channel_cfg(dev, c, ch->freqlist + ch->freq_idx, &ccfg[i][c]);
        }
        dcfg[i].sfmt = (int32_t)dev->input->sfmt;
        dcfg[i].fullscale = dev->input->fullscale;
        dcfg[i].sample_rate = dev->input->sample_rate;
        dcfg[i].n_channels = dev->channel_count;
        dcfg[i].channels = ccfg[i].data();
    }
    abg_config cfg;
    cfg.fft_size = (int32_t)bd::fft();
    cfg.wave_rate = bd::wave_rate();
    cfg.fm_demod = bd::fm_demod_algo();
    cfg.n_devices = nd;
    cfg.devices = dcfg.data();
    abg_options opt;
    memset(&opt, 0, sizeof(opt));
    opt.cuda_device = -1;
    opt.max_batches_per_run = g_b200.max_batches_per_run > 0 ? g_b200.max_batches_per_run : 2;
    opt.input_capacity_batches = opt.max_batches_per_run + 2;
    abg_engine* eng = nullptr;
    if (abg_create(&cfg, &opt, &eng) != ABG_OK) {
        fatal("Unable to start the GPU demodulation engine");
        return NULL;
    }
    // ---- ingest bridge: pin the input rings in place so that abg_push is asynchronous DMA straight out of the ring the
    // SDR threads fill (ring + wrap tail, input-helpers.cpp:27-36).  Best effort: pageable rings still work. ----
    std::vector<unsigned char*> pinned_rings;
    for (int i = 0; i < nd; i++) {
        input_t* in = devices[d0 + i].input;
        const size_t ring_bytes = in->buf_size + 2 * (size_t)in->bytes_per_sample * bd::fft();
        if (abg_host_register(in->buffer, ring_bytes) == ABG_OK) pinned_rings.push_back(in->buffer);
    }
    struct Unpin {
        std::vector<unsigned char*>& v;
        ~Unpin() {
            for (unsigned char* p : v) abg_host_unregister(p);
        }
    } unpin{pinned_rings};
    // ---- scan mode: channels with a frequency list (rtl_airband.h:250-252) hand the whole list to the engine; the entry
    // in use follows channel_t.freq_idx, which controller_thread changes (rtl_airband.cpp:117-119) ----
    std::vector<std::vector<int>> scan_idx(nd);  // freq_idx the engine currently uses, -1 = not a scan channel
    for (int i = 0; i < nd; i++) {
        device_t* dev = devices + d0 + i;
        scan_idx[i].assign(dev->channel_count, -1);
        for (int c = 0; c < dev->channel_count; c++) {
            channel_t* ch = dev->channels + c;
            if (ch->freq_count < 2) continue;
            std::vector<abg_channel_cfg> list(ch->freq_count);
            for (int k = 0; k < ch->freq_count; k++) fill_channel_cfg(dev, c, ch->freqlist + k, &list[k]);
            if (abg_scan_configure(eng, i, c, ch->freq_count, list.data()) != ABG_OK) {
                fatal("abg_scan_configure failed");
                abg_destroy(eng);
                return NULL;
            }
            scan_idx[i][c] = 0;
        }
    }
    if (configure_gpu_mixers(eng, devices, d0, d1) != ABG_OK) {
        fatal("abg_mixers_configure failed");
        abg_destroy(eng);
        return NULL;
    }
    // which freqlist[] entry each enqueued batch was demodulated with (the engine is pipelined: by delivery time
    // controller_thread may have moved freq_idx on, and active_counter belongs to the entry that produced the audio, :645)
    struct Enq {
        int n;
        std::vector<int> idx;
    };
    std::vector<std::deque<Enq>> enq(nd);
    g_b200.engine_ready = 1;
    std::vector<float> wo, iq, mleft, mright;
    std::vector<char> axc;
    bool idle = false;  // the previous pass neither pushed, demodulated nor delivered anything
    auto lockstep_wait_since = std::chrono::steady_clock::now();
    while (true) {
        if (bd::exit_flag()) {
            abg_destroy(eng);
            g_gpu_mixers.clear();
            return NULL;
        }
        if (bd::running() == 0 && idle) {  // :377-381 — but only once everything buffered has been delivered
#ifdef ABG_WITH_REFERENCE_HEADERS
            log(LOG_ERR, "All receivers failed, exiting\n");
#endif
            bd::exit_flag() = 1;
            continue;
        }
        bool pushed = false;
        std::vector<size_t> new_bufs(nd);
        std::vector<char> ring_has_more(nd, 0);  // bytes of this device still wait in its ring after this pass's push
        for (int i = 0; i < nd; i++) {
            device_t* dev = devices + d0 + i;
            input_t* in = dev->input;
            size_t available;
            pthread_mutex_lock(&in->buffer_lock);  // :370-375
            if (in->bufe >= in->bufs)
                available = in->bufe - in->bufs;
            else
                available = in->buf_size - in->bufs + in->bufe;
            pthread_mutex_unlock(&in->buffer_lock);
            if (in->state != INPUT_RUNNING) {  // :383-391
                if (in->state == INPUT_FAILED) {
                    in->state = INPUT_DISABLED;
                    bd::device_failed(dev);  // disable_device_outputs(dev), :386
                    bd::running()--;
                }
                // whatever is still buffered is demodulated (the reference also drains until `available` runs short)
            }
            const size_t bpc = 2 * (size_t)in->bytes_per_sample;
            const size_t hop_bytes = bpc * (size_t)abg_hop(eng, i);
            // hand over whole hops only (the reference advances bufs hop by hop, :669), at most one batch per visit
            size_t n = std::min(available / hop_bytes, (size_t)B) * hop_bytes;
            if (in->state != INPUT_RUNNING && n == 0 && available >= bpc) n = (available / bpc) * bpc;  // final partial hop at EOF
            size_t local_bufs = in->bufs;
            while (n > 0) {
                const size_t chunk = std::min(n, in->buf_size - local_bufs);  // up to the physical end of the ring
                int rc = abg_push(eng, i, in->buffer + local_bufs, chunk);
                if (rc == ABG_EOVERFLOW) break;  // engine buffer full: demodulate first
                if (rc != ABG_OK) {
                    fatal("abg_push failed");
                    abg_destroy(eng);
                    return NULL;
                }
                // the ring space is released (bufs advanced, not under the lock, like :669) only after the copy has
                // left the ring: with a page-locked ring abg_push is asynchronous
                local_bufs = (local_bufs + chunk) % in->buf_size;
                n -= chunk;
                available -= chunk;
                pushed = true;
            }
            new_bufs[i] = local_bufs;
            ring_has_more[i] = available >= bpc;
        }
        for (int i = 0; i < nd; i++) {  // fparms = freqlist + freq_idx, re-read before every batch (:498)
            device_t* dev = devices + d0 + i;
            for (int c = 0; c < dev->channel_count; c++) {
                const int want = dev->channels[c].freq_idx;
                if (scan_idx[i][c] < 0 || want == scan_idx[i][c]) continue;
                if (abg_scan_select(eng, i, c, want) != ABG_OK) {
                    fatal("abg_scan_select failed");
                    abg_destroy(eng);
                    return NULL;
                }
                scan_idx[i][c] = want;
            }
        }
        std::vector<int> ready_before(nd);
        for (int i = 0; i < nd; i++) ready_before[i] = abg_batches_ready(eng, i);
        // The engine sums batch b of a run over the mixer inputs that have a batch b in that run, so the devices feeding a
        // GPU-summed mixer are demodulated in lock step (the reference's mixer likewise waits for every enabled input,
        // mixer.cpp:186-190, and gives up on a late one only after its interval): a run takes as many batches as every
        // mixer device that still has input holds.  A running device that delivers nothing for a second no longer holds
        // the others up (its input has stalled; the engine then sums without it, like a mixer input that is not ready).
        int run_batches = -1;
        if (!g_gpu_mixers.empty()) {
            int lo = 1 << 30;
            for (int i : g_mixer_devs) {
                const int av = abg_batches_available(eng, i);
                // (a finished input still counts while its ring or the engine holds samples of it)
                if (av > 0 || ring_has_more[i] || devices[d0 + i].input->state == INPUT_RUNNING) lo = std::min(lo, av);
            }
            if (lo != (1 << 30)) run_batches = lo;
            const auto now = std::chrono::steady_clock::now();
            if (run_batches != 0) lockstep_wait_since = now;
            else if (now - lockstep_wait_since > std::chrono::seconds(1)) run_batches = -1;
        }
        int produced = run_batches == 0 ? 0 : abg_run(eng, run_batches);
        if (produced < 0 && produced != ABG_EOVERFLOW) {
            fatal("abg_run failed");
            abg_destroy(eng);
            return NULL;
        }
        for (int i = 0; i < nd; i++) {
            const int n_new = abg_batches_ready(eng, i) - ready_before[i];
            if (n_new > 0) enq[i].push_back(Enq{n_new, scan_idx[i]});
        }
        // (after abg_run, so that waiting for the copies overlaps the kernels that were just enqueued)
        if (pushed) {
            if (abg_ingest_sync(eng) != ABG_OK) {
                fatal("abg_ingest_sync failed");
                abg_destroy(eng);
                return NULL;
            }
            for (int i = 0; i < nd; i++) devices[d0 + i].input->bufs = new_bufs[i];
        }
        // ---- deliver finished batches (:621-662 + output.cpp:903-923 hand-shake) ----
        bool delivered = false;
        for (int i = 0; i < nd; i++) {
            device_t* dev = devices + d0 + i;
            while (abg_batches_ready(eng, i) > 0) {
                if (g_b200.wait_for_consumer && dev->waveavail == 1) break;  // offline pacing: do not overrun the output thread
                const int C = dev->channel_count;
                wo.resize((size_t)C * B);
                iq.resize((size_t)C * 2 * B);
                axc.resize(C);
                int rc = abg_fetch_batch(eng, i, wo.data(), iq.data(), axc.data());
                if (rc < 0) {
                    fatal("abg_fetch_batch failed");
                    abg_destroy(eng);
                    return NULL;
                }
                if (rc == 0) break;
                const std::vector<int>* used = nullptr;
                if (!enq[i].empty()) {
                    used = &enq[i].front().idx;
                }
                for (int c = 0; c < C; c++) {
                    channel_t* ch = dev->channels + c;
                    memcpy(ch->waveout, wo.data() + (size_t)c * B, sizeof(float) * B);
                    if (ch->has_iq_outputs) memcpy(ch->iq_out, iq.data() + (size_t)c * 2 * B, sizeof(float) * 2 * B);
                    ch->axcindicate = (enum status)axc[c];
                    if (ch->axcindicate != NO_SIGNAL) {  // :645-647
                        const int fi = (used && (*used)[c] >= 0) ? (*used)[c] : ch->freq_idx;
                        ch->freqlist[fi].active_counter++;
                    }
                }
                if (!enq[i].empty() && --enq[i].front().n == 0) enq[i].pop_front();
                if (dev->waveavail == 1)
                    dev->output_overrun_count++;  // :649-652
                else
                    dev->waveavail = 1;
                dp->mp3_signal->send();  // :662
                delivered = true;
                if (g_b200.wait_for_consumer) break;
            }
        }
        if (!g_gpu_mixers.empty() && deliver_mixers(eng, dp->mp3_signal, B, mleft, mright)) delivered = true;
        idle = !pushed && !delivered && produced <= 0;
        if (idle) {
            bool waiting = false;  // batches held back only because the output thread has not consumed the previous one
            for (int i = 0; i < nd; i++) waiting = waiting || abg_batches_ready(eng, i) > 0;
            // (deliver_mixers does not look further while the output thread has not taken a mixer's last batch: more may be
            // queued behind it)
            if (g_b200.wait_for_consumer)
                for (const auto& gm : g_gpu_mixers) waiting = waiting || gm.mixer->channel.state == CH_READY;
            if (waiting) idle = false;
            usleep(waiting ? 200 : 10 * 1000);  // SLEEP(10), :398
        }
    }
}

// refresh the Squelch read-outs of one device's channels for the stats file / TUI (output.cpp:598-869, rtl_airband.cpp:632-643)
extern "C" ABG_API int b200_refresh_stats(abg_engine* eng, int dev_local, device_t* dev) {
    for (int c = 0; c < dev->channel_count; c++) {
        abg_squelch_stats s;
        int rc = abg_get_stats(eng, dev_local, c, &s);
        if (rc != ABG_OK) return rc;
        freq_t* f = dev->channels[c].freqlist + dev->channels[c].freq_idx;
        f->b200_stats.noise_level = s.noise_level;
        f->b200_stats.signal_level = s.signal_level;
        f->b200_stats.squelch_level = s.squelch_level;
        f->b200_stats.noise_level_dbfs = s.noise_level_dbfs;
        f->b200_stats.signal_level_dbfs = s.signal_level_dbfs;
        f->b200_stats.squelch_level_dbfs = s.squelch_level_dbfs;
        f->b200_stats.open_count = s.open_count;
        f->b200_stats.flappy_count = s.flappy_count;
        f->b200_stats.ctcss_count = s.ctcss_count;
        f->b200_stats.no_ctcss_count = s.no_ctcss_count;
        f->agcavgfast = s.agcavgfast;
        dev->bins[c] = (size_t)s.bin;
    }
    return ABG_OK;
}

// output.cpp:519-522: buflen = 2 * sizeof(float) * WAVE_BATCH; fwrite(channel->iq_out, 1, buflen, f)
extern "C" ABG_API size_t b200_write_rawfile(FILE* f, const channel_t* channel, int wave_batch) {
    const size_t buflen = 2 * sizeof(float) * (size_t)wave_batch;
    return fwrite(channel->iq_out, 1, buflen, f);
}
