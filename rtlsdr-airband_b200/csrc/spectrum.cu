// Band spectrum monitor (abg_spectrum_configure / abg_fetch_spectrum): the batch-averaged power of every FFT bin of a
// device, P[k] = (1/n) * sum over the selected frames of |X_f[k]|^2, from the same raw bytes, conversion, window and FFT
// as K1's full-spectrum kernel (k1_fft.cuh).  The definition is in include/airband_b200.h.
//
// One launch per run covers every monitored device.  Work item = (device, batch of the run, chunk): a chunk is FPC
// consecutive selected frames of one batch, counted from the batch's first frame, so the items depend on the batch and
// the stride only, never on how batches are grouped into runs.
//   * the S slots of a CTA each run one frame through fft_frame() and write |X|^2 to their row of `pw`; then the whole CTA
//     adds the S rows, in frame order, into per-thread accumulators (thread t owns bins t, t + BLOCK, ...).  A chunk's
//     sum is therefore ((p_0 + p_1) + p_2) + ... over its frames.
//   * a batch with one chunk is finished by its CTA.  Otherwise every CTA stores its chunk sum to partial[batch][chunk][N],
//     and the CTA that arrives last at the batch's counter adds the chunks in chunk order, divides by n and resets the
//     counter.  Sums are bitwise reproducible and independent of max_batches_per_run and of the push pattern.
//   * the finished spectrum goes straight into the device's page-locked result ring (mapped), or, for resident runs, into
//     the first partial row of the batch.
// Raw samples are read from global memory (L2) rather than staged as a tile: at the default stride the selected frames do
// not overlap.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/airband_b200.h"
#include "abg_internal.h"
#include "k1_common.cuh"
#include "k1_fft.cuh"

namespace {
using namespace k1;

template <int LOGN>
struct SpecShape {
    using F = FftShape<LOGN>;
    static constexpr int N = F::N;
    static constexpr int BLOCK = Plan<LOGN>::BLOCK;
    static constexpr int NB = N / BLOCK;                  // accumulated bins per thread
    static constexpr int PWN = F::THREE ? N + N / 32 : N;  // power row (the 3-pass last stage writes bins 32 apart: pad)
    static constexpr size_t smem = sizeof(float2) * (size_t)F::S * F::EXN + sizeof(float) * (size_t)F::S * PWN;
    static __device__ __forceinline__ int pw_index(int b) {
        if constexpr (F::THREE)
            return b + (b >> 5);
        else
            return b;
    }
};

template <int LOGN, int SFMT>
__device__ __forceinline__ void spectrum_item(const SpecArgs& a, const SpecCfg& cf, const SpecRun& rn, int k, int c, unsigned char* smem) {
    using F = FftShape<LOGN>;
    using SS = SpecShape<LOGN>;
    constexpr int N = F::N, T = Plan<LOGN>::T, S = F::S, RL = F::RL, BLOCK = SS::BLOCK, NB = SS::NB;
    float2* ex_all = reinterpret_cast<float2*>(smem);
    float* pw = reinterpret_cast<float*>(ex_all + (size_t)S * F::EXN);
    const int tid = threadIdx.x, slot = tid / T, lt = tid % T;
    float2* ex = ex_all + (size_t)slot * F::EXN;
    float* pws = pw + (size_t)slot * SS::PWN;

    const int i0 = c * ABG_SPEC_FPC;
    const int nsel = min(ABG_SPEC_FPC, cf.n_sel - i0);
    const unsigned long long batch_byte = rn.first_byte + (unsigned long long)k * a.wave_batch * cf.hop_bytes;
    const unsigned long long frame_step = (unsigned long long)cf.stride * cf.hop_bytes;

    float acc[NB];
#pragma unroll
    for (int m = 0; m < NB; ++m) acc[m] = 0.0f;
    const int iters = (nsel + S - 1) / S;
    for (int it = 0; it < iters; ++it) {
        const int fl = it * S + slot;
        const bool active = fl < nsel;
        const unsigned char* src = rn.raw + (active ? batch_byte + (unsigned long long)(i0 + fl) * frame_step : 0ull);
        fft_frame<LOGN, SFMT>(src, active, slot, lt, ex, cf.wsc, a.tw1, a.tw2, [&](const float2(&v)[RL], int q) {
#pragma unroll
            for (int r = 0; r < RL; ++r) {
                const float2 x = v[brev<RL>(r)];
                pws[SS::pw_index(F::bin_of(q, r))] = fmaf(x.x, x.x, x.y * x.y);
            }
        });
        __syncthreads();
        const int nact = min(S, nsel - it * S);
#pragma unroll
        for (int m = 0; m < NB; ++m) {
            const int p = SS::pw_index(tid + m * BLOCK);
            float s = acc[m];
            for (int sl = 0; sl < nact; ++sl) s += pw[(size_t)sl * SS::PWN + p];
            acc[m] = s;
        }
        __syncthreads();  // pw is rewritten by the next frames
    }

    float* batch_part = cf.partial + (size_t)k * cf.n_chunks * N;
    float* out = rn.ring_pos0 >= 0 ? cf.ring + (size_t)((rn.ring_pos0 + k) % cf.ring_cap) * N : batch_part;
    const float n_f = (float)cf.n_sel;
    if (cf.n_chunks == 1) {
#pragma unroll
        for (int m = 0; m < NB; ++m) out[tid + m * BLOCK] = acc[m] / n_f;
        return;
    }
    float* mine = batch_part + (size_t)c * N;
#pragma unroll
    for (int m = 0; m < NB; ++m) mine[tid + m * BLOCK] = acc[m];
    __threadfence();
    __syncthreads();
    __shared__ int last;
    if (tid == 0) last = atomicAdd(cf.counter + k, 1) == cf.n_chunks - 1;
    __syncthreads();
    if (!last) return;
    __threadfence();
#pragma unroll
    for (int m = 0; m < NB; ++m) {
        const int b = tid + m * BLOCK;
        float s = 0.0f;
        for (int cc = 0; cc < cf.n_chunks; ++cc) s += __ldcg(batch_part + (size_t)cc * N + b);
        out[b] = s / n_f;
    }
    if (tid == 0) cf.counter[k] = 0;
}

template <int LOGN>
__global__ void __launch_bounds__(Plan<LOGN>::BLOCK) abg_band_spectrum_kernel(const SpecArgs a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const SpecCfg cf = a.cfg[blockIdx.y];
    const SpecRun rn = a.run[blockIdx.y];
    const int item = blockIdx.x;
    if (item >= rn.n_batches * cf.n_chunks) return;
    const int k = item / cf.n_chunks, c = item % cf.n_chunks;
    switch (cf.sfmt) {
        case ABG_SFMT_U8: spectrum_item<LOGN, ABG_SFMT_U8>(a, cf, rn, k, c, smem); break;
        case ABG_SFMT_S8: spectrum_item<LOGN, ABG_SFMT_S8>(a, cf, rn, k, c, smem); break;
        case ABG_SFMT_S16: spectrum_item<LOGN, ABG_SFMT_S16>(a, cf, rn, k, c, smem); break;
        default: spectrum_item<LOGN, ABG_SFMT_F32>(a, cf, rn, k, c, smem); break;
    }
}

template <int LOGN>
cudaError_t launch(const SpecArgs& a, int n_devices, int max_items, cudaStream_t s) {
    constexpr size_t smem = SpecShape<LOGN>::smem;
    auto kern = abg_band_spectrum_kernel<LOGN>;
    static AbgPerDeviceSize configured;
    cudaError_t e = configured.ensure(smem, [&]() { return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); });
    if (e != cudaSuccess) return e;
    kern<<<dim3(max_items, n_devices, 1), Plan<LOGN>::BLOCK, smem, s>>>(a);
    return cudaGetLastError();
}

}  // namespace

cudaError_t abg_launch_spectrum(int fft_size, const SpecArgs& a, int n_devices, int max_items, cudaStream_t s) {
    if (n_devices < 1 || max_items < 1) return cudaSuccess;
    switch (fft_size) {
        case 256: return launch<8>(a, n_devices, max_items, s);
        case 512: return launch<9>(a, n_devices, max_items, s);
        case 1024: return launch<10>(a, n_devices, max_items, s);
        case 2048: return launch<11>(a, n_devices, max_items, s);
        case 4096: return launch<12>(a, n_devices, max_items, s);
        case 8192: return launch<13>(a, n_devices, max_items, s);
    }
    return cudaErrorInvalidValue;
}
