// Band activity detector (abg_activity_configure / abg_fetch_activity): every burst above a per-bin threshold in a device's
// band, at frame resolution.  The power of each selected frame is p_f[k] = |X_f[k]|^2 from the same raw bytes, conversion,
// window and FFT as the band spectrum (k1_fft.cuh), in the same float32 expression.  The definition is in
// include/airband_b200.h.
//
// One launch per run covers every device with the detector on.  Work item = (device, batch of the run): the walk over a
// bin's frames is sequential in frame order, so one CTA owns a whole batch and every bin of it.
//   * the S slots of a CTA each run one frame through fft_frame() and write p to their row of `pw`; then every thread walks
//     its bins (t, t + BLOCK, ...) through the S rows in frame order.  With one frame in flight (S = 1, N = 8192) the rows
//     are skipped: the emit of the last FFT pass visits every bin once per frame, so it walks the bins itself.
//   * the open piece of every bin lives in shared memory, 16 bytes a bin (first|last i packed, count, peak, sum): 128 KB at
//     N = 8192 next to the 68 KB exchange buffer.  A bin's state is touched only on its active frames.
//   * a piece closes when the next active frame is more than h + 1 frames later, or at the batch's end.  Closed pieces
//     that may still matter (an open flag, or a span >= m) take an index from a shared counter and, below the capacity,
//     are written straight into the device's page-locked result ring entry (mapped).  One CTA owns the entry, so the
//     counter needs no reset between launches.  Resident runs count pieces but store none.
// Pieces depend on the batch, its frames and the settings only, never on how batches are grouped into runs; the order in
// which they land in the ring is not specified (the host sorts them).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/airband_b200.h"
#include "abg_internal.h"
#include "k1_common.cuh"
#include "k1_fft.cuh"

namespace {
using namespace k1;

constexpr uint32_t kNone = 0xFFFFFFFFu;  // span of a bin without an open piece

template <int LOGN>
struct ActShape {
    using F = FftShape<LOGN>;
    static constexpr int N = F::N;
    static constexpr int BLOCK = Plan<LOGN>::BLOCK;
    static constexpr bool ROWS = F::S > 1;                 // several frames in flight: power rows, walked after each group
    static constexpr int PWN = F::THREE ? N + N / 32 : N;  // power row (the 3-pass last stage writes bins 32 apart: pad)
    static constexpr size_t ex_bytes = sizeof(float2) * (size_t)F::S * F::EXN;
    static constexpr size_t pw_bytes = ROWS ? sizeof(float) * (size_t)F::S * PWN : 0;
    static constexpr size_t smem = ex_bytes + pw_bytes + 16 * (size_t)N;
    static __device__ __forceinline__ int pw_index(int b) {
        if constexpr (F::THREE)
            return b + (b >> 5);
        else
            return b;
    }
};

struct Walk {
    uint32_t* span;  // [N] first | last << 16 of the open piece, kNone without one
    int32_t* cnt;    // [N] active frames of the open piece
    float* peak;     // [N]
    float* sum;      // [N] added in frame order
    abg_burst* out;  // the entry's records, or nullptr (resident run)
    int* counter;    // shared: pieces kept so far
    unsigned long long frame0;  // absolute frame number of the batch's frame j = 0
    int stride, n, hang, min_span;

    // Close bin k's open piece: keep it if it may join a neighbouring batch's piece or is long enough already.
    __device__ __forceinline__ void close(int k, uint32_t sp) const {
        const int first = (int)(sp & 0xFFFFu), last = (int)(sp >> 16);
        const int flags = (first <= hang ? ABG_BURST_OPEN_START : 0) | (last >= n - 1 - hang ? ABG_BURST_OPEN_END : 0);
        if (flags == 0 && last - first + 1 < min_span) return;
        const int idx = atomicAdd(counter, 1);
        if (!out || idx >= ABG_ACTIVITY_MAX_RECORDS) return;
        abg_burst* r = out + idx;
        r->bin = k;
        r->flags = flags;
        r->first_frame = frame0 + (unsigned long long)first * stride;
        r->last_frame = frame0 + (unsigned long long)last * stride;
        r->n_active = cnt[k];
        r->peak = peak[k];
        r->sum = sum[k];
        r->reserved = 0;
    }
    // Selected frame i of the batch is active in bin k with power p.
    __device__ __forceinline__ void step(int k, int i, float p) const {
        const uint32_t sp = span[k];
        if (sp != kNone && i - (int)(sp >> 16) <= hang + 1) {
            span[k] = (sp & 0xFFFFu) | ((uint32_t)i << 16);
            cnt[k] += 1;
            peak[k] = fmaxf(peak[k], p);
            sum[k] = sum[k] + p;
            return;
        }
        if (sp != kNone) close(k, sp);
        span[k] = (uint32_t)i | ((uint32_t)i << 16);
        cnt[k] = 1;
        peak[k] = p;
        sum[k] = p;
    }
};

template <int LOGN, int SFMT>
__device__ __forceinline__ void activity_item(const ActArgs& a, const ActCfg& cf, const ActRun& rn, int b, unsigned char* smem) {
    using F = FftShape<LOGN>;
    using AS = ActShape<LOGN>;
    constexpr int N = F::N, T = Plan<LOGN>::T, S = F::S, RL = F::RL, BLOCK = AS::BLOCK;
    float2* ex_all = reinterpret_cast<float2*>(smem);
    float* pw = reinterpret_cast<float*>(smem + AS::ex_bytes);
    unsigned char* st = smem + AS::ex_bytes + AS::pw_bytes;
    __shared__ int counter;
    const int tid = threadIdx.x, slot = tid / T, lt = tid % T;
    float2* ex = ex_all + (size_t)slot * F::EXN;
    float* pws = pw + (size_t)slot * AS::PWN;

    const float* __restrict__ thr = cf.thr;
    Walk w;
    w.span = reinterpret_cast<uint32_t*>(st);
    w.cnt = reinterpret_cast<int32_t*>(st + 4 * (size_t)N);
    w.peak = reinterpret_cast<float*>(st + 8 * (size_t)N);
    w.sum = reinterpret_cast<float*>(st + 12 * (size_t)N);
    w.out = rn.ring_pos0 >= 0
                ? reinterpret_cast<abg_burst*>(cf.ring + (size_t)((rn.ring_pos0 + b) % cf.ring_cap) * cf.entry_bytes + ABG_ACT_HEAD_BYTES)
                : nullptr;
    w.counter = &counter;
    w.frame0 = rn.first_frame + (unsigned long long)b * a.wave_batch;
    w.stride = cf.stride; w.n = cf.n_sel; w.hang = cf.hang; w.min_span = cf.min_span;

    for (int k = tid; k < N; k += BLOCK) w.span[k] = kNone;
    if (tid == 0) counter = 0;
    __syncthreads();

    const unsigned long long batch_byte = rn.first_byte + (unsigned long long)b * a.wave_batch * cf.hop_bytes;
    const unsigned long long frame_step = (unsigned long long)cf.stride * cf.hop_bytes;
    const int nsel = cf.n_sel;
    const int iters = (nsel + S - 1) / S;
    for (int it = 0; it < iters; ++it) {
        const int fl = it * S + slot;
        const bool active = fl < nsel;
        const unsigned char* src = rn.raw + (active ? batch_byte + (unsigned long long)fl * frame_step : 0ull);
        if constexpr (AS::ROWS) {
            fft_frame<LOGN, SFMT>(src, active, slot, lt, ex, cf.wsc, a.tw1, a.tw2, [&](const float2(&v)[RL], int q) {
#pragma unroll
                for (int r = 0; r < RL; ++r) {
                    const float2 x = v[brev<RL>(r)];
                    pws[AS::pw_index(F::bin_of(q, r))] = fmaf(x.x, x.x, x.y * x.y);
                }
            });
            __syncthreads();
            const int nact = min(S, nsel - it * S);
#pragma unroll 1
            for (int k = tid; k < N; k += BLOCK) {
                const float t = __ldg(thr + k);
                const int p_i = AS::pw_index(k);
                for (int sl = 0; sl < nact; ++sl) {
                    const float p = pw[(size_t)sl * AS::PWN + p_i];
                    if (p > t) w.step(k, it * S + sl, p);
                }
            }
            __syncthreads();  // pw is rewritten by the next frames
        } else {
            // one frame in flight (fl == it): every bin is visited once, by a fixed thread, between the frame's barriers
            fft_frame<LOGN, SFMT>(src, active, slot, lt, ex, cf.wsc, a.tw1, a.tw2, [&](const float2(&v)[RL], int q) {
#pragma unroll
                for (int r = 0; r < RL; ++r) {
                    const float2 x = v[brev<RL>(r)];
                    const float p = fmaf(x.x, x.x, x.y * x.y);
                    const int k = F::bin_of(q, r);
                    if (p > __ldg(thr + k)) w.step(k, fl, p);
                }
            });
        }
    }
    __syncthreads();
    for (int k = tid; k < N; k += BLOCK) {
        const uint32_t sp = w.span[k];
        if (sp != kNone) w.close(k, sp);
    }
    __syncthreads();
    if (tid == 0 && w.out) {
        int32_t* head = reinterpret_cast<int32_t*>(reinterpret_cast<unsigned char*>(w.out) - ABG_ACT_HEAD_BYTES);
        head[0] = counter;
        head[1] = cf.stride;
        head[2] = cf.hang;
        head[3] = cf.min_span;
    }
}

template <int LOGN>
__global__ void __launch_bounds__(Plan<LOGN>::BLOCK, 1) abg_activity_kernel(const ActArgs a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const ActCfg cf = a.cfg[blockIdx.y];
    const ActRun rn = a.run[blockIdx.y];
    const int b = blockIdx.x;
    if (b >= rn.n_batches) return;
    switch (cf.sfmt) {
        case ABG_SFMT_U8: activity_item<LOGN, ABG_SFMT_U8>(a, cf, rn, b, smem); break;
        case ABG_SFMT_S8: activity_item<LOGN, ABG_SFMT_S8>(a, cf, rn, b, smem); break;
        case ABG_SFMT_S16: activity_item<LOGN, ABG_SFMT_S16>(a, cf, rn, b, smem); break;
        default: activity_item<LOGN, ABG_SFMT_F32>(a, cf, rn, b, smem); break;
    }
}

template <int LOGN>
cudaError_t launch(const ActArgs& a, int n_devices, int max_batches, cudaStream_t s) {
    constexpr size_t smem = ActShape<LOGN>::smem;
    auto kern = abg_activity_kernel<LOGN>;
    static AbgPerDeviceSize configured;
    cudaError_t e = configured.ensure(smem, [&]() { return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); });
    if (e != cudaSuccess) return e;
    kern<<<dim3(max_batches, n_devices, 1), Plan<LOGN>::BLOCK, smem, s>>>(a);
    return cudaGetLastError();
}

}  // namespace

cudaError_t abg_launch_activity(int fft_size, const ActArgs& a, int n_devices, int max_batches, cudaStream_t s) {
    if (n_devices < 1 || max_batches < 1) return cudaSuccess;
    switch (fft_size) {
        case 256: return launch<8>(a, n_devices, max_batches, s);
        case 512: return launch<9>(a, n_devices, max_batches, s);
        case 1024: return launch<10>(a, n_devices, max_batches, s);
        case 2048: return launch<11>(a, n_devices, max_batches, s);
        case 4096: return launch<12>(a, n_devices, max_batches, s);
        case 8192: return launch<13>(a, n_devices, max_batches, s);
    }
    return cudaErrorInvalidValue;
}
