// K1 — fused sample conversion + Blackman-Harris window + batched FFT + per-channel bin extraction (sm_90a).
//
// Replaces, for every frame of every device, the reference's three hot loops
//   convert+window   reference src/rtl_airband.cpp:402-455
//   fftwf_execute    reference src/rtl_airband.cpp:460   (or gpu_fft_execute on the VideoCore build, :458)
//   bin extraction   reference src/rtl_airband.cpp:483-489
// and writes only |X[bin]| and X[bin] for the configured channels — the N-point spectrum never goes to HBM
// (except the batch-final frame of devices with AFC, reference src/rtl_airband.cpp:180-251,629).
//
// Shape of the computation
//   * one CTA = one tile of consecutive frames of one device.  Frames overlap by N-hop samples, so the CTA stages
//     the tile's raw bytes ((TF-1)*hop + N samples) ONCE in shared memory with a single TMA bulk copy
//     (cp.async.bulk ... mbarrier::complete_tx) and every frame converts from there: HBM sees each input byte
//     about once per tile (+ the N-hop overlap between neighbouring tiles, which hits L2).
//   * an N-point FFT (fft_frame() in k1_fft.cuh, shared with the band-spectrum kernel) is 2 (3 for N=8192) register passes: each thread holds one radix-R1 column in registers
//     (R1 up to 64 complex values), runs a fully unrolled decimation-in-time FFT on it whose twiddles are
//     compile-time immediates, applies the inter-pass twiddle, and exchanges through a padded shared-memory
//     buffer; the last pass leaves bin k1 + R1*k2 in register k2 of thread k1.
//   * radix-2 DIT butterflies are written FMA-first: a' = a + W*b costs 4 FFMA, b' = 2a - a' costs 2 (6 per
//     butterfly instead of 10 flops in 8 instructions).
//   * window and twiddle tables are read through the L1 (they are the only L1 traffic: the sample stream goes
//     global -> shared by TMA).  The window table already contains the 1/full-scale factor of the sample format.
//   * bin extraction: a per-CTA 64-bit "wanted" mask per last-pass butterfly, built from the CURRENT bins[] in
//     global memory (so AFC / scan retunes take effect on the next launch), selects registers with compile-time
//     indices; no dynamic register indexing, no spectrum store.
// Tensor cores are not used: there is no dense contraction on this path (BASELINE.json north_star).
#include <cuda_runtime.h>
#include <stdint.h>

#include <utility>

#include "../../include/airband_b200.h"
#include "abg_internal.h"
#include "k1_common.cuh"
#include "k1_fft.cuh"

namespace {
using namespace k1;

struct K1Args {
    const K1Dev* devs;
    const int32_t* bins;
    const float* wsc;
    const float2* tw1;
    const float2* tw2;
    float* win;
    float2* iqin;
    int Gp;
    int frames_per_tile;
    int tile_bytes_cap;
};

// emit the wanted bins of one last-pass butterfly
template <int R, typename BinOf>
__device__ __forceinline__ void emit_bins(const float2 (&v)[R], unsigned long long mask, int q, const K1Dev& dv, const K1Args& a, int pos,
                                          float2* spec_row, BinOf bin_of) {
    if (spec_row != nullptr) {  // batch-final frame of a device with AFC: keep the whole spectrum, natural bin order
#pragma unroll
        for (int r = 0; r < R; ++r) spec_row[bin_of(q, r)] = v[brev<R>(r)];
    }
    if (mask == 0ull) return;
#pragma unroll
    for (int r = 0; r < R; ++r) {
        if ((mask >> r) & 1ull) {
            const float2 x = v[brev<R>(r)];
            const int b = bin_of(q, r);
            // same association as the reference (no FMA contraction): sqrtf(re*re + im*im), rtl_airband.cpp:484
            const float mag = sqrtf(__fadd_rn(__fmul_rn(x.x, x.x), __fmul_rn(x.y, x.y)));
            for (int c = 0; c < dv.n_channels; ++c) {
                if (a.bins[dv.g0 + c] == b) {
                    const size_t o = (size_t)pos * a.Gp + dv.g0 + c;
                    a.win[o] = mag;
                    a.iqin[o] = x;
                }
            }
        }
    }
}

template <int LOGN, int SFMT>
__global__ void __launch_bounds__(Plan<LOGN>::BLOCK) k1_fft_kernel(const K1Args a) {
    using P = Plan<LOGN>;
    using F = FftShape<LOGN>;
    constexpr int N = F::N;
    constexpr int R1 = P::R1, R2 = P::R2, T = P::T, BLOCK = P::BLOCK;
    constexpr bool THREE = F::THREE;
    constexpr int RL = F::RL, S = F::S, EXN = F::EXN, NQL = F::NQL;
    constexpr int BPC = bytes_per_cplx<SFMT>();
    static_assert(S >= 1, "block too small");

    extern __shared__ __align__(128) unsigned char smem[];
    unsigned long long* mbar = reinterpret_cast<unsigned long long*>(smem);
    unsigned long long* want = reinterpret_cast<unsigned long long*>(smem + 16);
    float2* ex_all = reinterpret_cast<float2*>(smem + 16 + sizeof(unsigned long long) * NQL);
    unsigned char* tile = smem + 16 + sizeof(unsigned long long) * NQL + sizeof(float2) * (size_t)S * EXN;
    // (16 + 8*NQL + 8*S*EXN is a multiple of 16 for every plan, so `tile` is 16-byte aligned as TMA requires)

    const K1Dev dv = a.devs[blockIdx.y];
    const int f0 = blockIdx.x * a.frames_per_tile;
    if (f0 >= dv.n_frames) return;
    const int nf = min(a.frames_per_tile, dv.n_frames - f0);
    const int tid = threadIdx.x;

    // ---- stage the tile's raw bytes with one TMA bulk copy ---------------------------------------------------
    const unsigned long long s_byte = dv.start_byte + (unsigned long long)f0 * dv.hop_bytes;
    const unsigned long long a_byte = s_byte & ~15ull;
    const int pre = (int)(s_byte - a_byte);
    const unsigned int copy_bytes = (unsigned int)((pre + (nf - 1) * dv.hop_bytes + N * BPC + 15) & ~15);
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(mbar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = tid; i < NQL; i += BLOCK) want[i] = 0ull;
    __syncthreads();
    if (tid == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(mbar)), "r"(copy_bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(tile)),
                     "l"(dv.raw + a_byte), "r"(copy_bytes), "r"(smem_u32(mbar))
                     : "memory");
    }
    // ---- meanwhile: which last-pass butterfly / register holds each configured bin ----------------------------
    for (int c = tid; c < dv.n_channels; c += BLOCK) {
        const int b = a.bins[dv.g0 + c] & (N - 1);
        int q, r;
        if constexpr (!THREE) {
            q = b % R1;
            r = b / R1;
        } else {
            const int k1 = b % R1, rest = b / R1;
            q = k1 * R2 + rest % R2;
            r = rest / R2;
        }
        atomicOr(&want[q], 1ull << r);
    }
    __syncthreads();
    {
        uint32_t done = 0;
        while (!done) {
            asm volatile(
                "{\n\t.reg .pred p;\n\t"
                "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
                "selp.u32 %0, 1, 0, p;\n\t}"
                : "=r"(done)
                : "r"(smem_u32(mbar))
                : "memory");
        }
    }

    const int slot = tid / T, lt = tid % T;
    float2* ex = ex_all + (size_t)slot * EXN;

    const int iters = (nf + S - 1) / S;
    for (int it = 0; it < iters; ++it) {
        const int fl = it * S + slot;  // frame within the tile
        const bool active = fl < nf;
        const int fo = pre + fl * dv.hop_bytes;
        const int pos = dv.pos0 + f0 + fl;
        float2* spec_row = nullptr;
        if (active && dv.spec != nullptr && pos >= dv.spec_first_pos && ((pos - dv.spec_first_pos) % dv.wave_batch) == 0)
            spec_row = dv.spec + (size_t)((pos - dv.spec_first_pos) / dv.wave_batch) * N;
        fft_frame<LOGN, SFMT>(tile + fo, active, slot, lt, ex, a.wsc, a.tw1, a.tw2, [&](const float2(&v)[RL], int q) {
            emit_bins<RL>(v, want[q], q, dv, a, pos, spec_row, F::bin_of);
        });
    }
}

template <int LOGN>
constexpr size_t k1_fixed_smem() {
    using P = Plan<LOGN>;
    constexpr int N = 1 << LOGN;
    constexpr int RL = P::R3 ? P::R3 : P::R2;
    constexpr int EXN = N + N / RL;
    constexpr int S = P::BLOCK / P::T;
    return 16 + sizeof(unsigned long long) * (N / RL) + sizeof(float2) * (size_t)S * EXN;
}

size_t k1_fixed_smem_rt(int logn) {
    switch (logn) {
        case 8: return k1_fixed_smem<8>();
        case 9: return k1_fixed_smem<9>();
        case 10: return k1_fixed_smem<10>();
        case 11: return k1_fixed_smem<11>();
        case 12: return k1_fixed_smem<12>();
        case 13: return k1_fixed_smem<13>();
    }
    return 0;
}

template <int LOGN, int SFMT>
cudaError_t launch_one(const K1Launch& L, const K1Args& args, cudaStream_t s) {
    using P = Plan<LOGN>;
    const size_t smem = k1_fixed_smem<LOGN>() + (size_t)L.tile_bytes_cap;
    auto kern = k1_fft_kernel<LOGN, SFMT>;
    static AbgPerDeviceSize configured;  // per instantiation, per CUDA device
    {
        cudaError_t e = configured.ensure(smem, [&]() {
            cudaError_t e2 = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e2 != cudaSuccess) return e2;
            cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            return cudaSuccess;
        });
        if (e != cudaSuccess) return e;
    }
    const int tiles = (L.max_frames + L.frames_per_tile - 1) / L.frames_per_tile;
    dim3 grid(tiles, L.n_devices, 1), block(P::BLOCK, 1, 1);
    kern<<<grid, block, smem, s>>>(args);
    return cudaGetLastError();
}

template <int LOGN>
cudaError_t launch_fmt(const K1Launch& L, const K1Args& args, cudaStream_t s) {
    switch (L.sfmt) {
        case ABG_SFMT_U8: return launch_one<LOGN, ABG_SFMT_U8>(L, args, s);
        case ABG_SFMT_S8: return launch_one<LOGN, ABG_SFMT_S8>(L, args, s);
        case ABG_SFMT_S16: return launch_one<LOGN, ABG_SFMT_S16>(L, args, s);
        case ABG_SFMT_F32: return launch_one<LOGN, ABG_SFMT_F32>(L, args, s);
    }
    return cudaErrorInvalidValue;
}

}  // namespace

// Frames per tile and the raw-tile shared-memory reservation for a (size, format, hop) combination.
// Targets two CTAs per SM: fixed + tile <= ~110 KB, tile >= one frame.
int abg_k1_tile_frames(int fft_size, int sfmt, int hop_bytes, int* tile_bytes_cap) {
    int logn = 0;
    while ((1 << logn) < fft_size) logn++;
    const int bpc = (sfmt == ABG_SFMT_U8 || sfmt == ABG_SFMT_S8) ? 2 : (sfmt == ABG_SFMT_S16 ? 4 : 8);
    const size_t fixed = k1_fixed_smem_rt(logn);
    const size_t frame_bytes = (size_t)fft_size * bpc;
    const size_t per_cta_budget = 112 * 1024;
    size_t budget = per_cta_budget > fixed + frame_bytes + 64 ? per_cta_budget - fixed : frame_bytes + 64;
    if (fixed + budget > 220 * 1024) budget = 220 * 1024 - fixed;
    int tf = 1;
    if (budget > frame_bytes + 64) tf = 1 + (int)((budget - frame_bytes - 64) / (size_t)hop_bytes);
    if (tf > 64) tf = 64;
    if (tf < 1) tf = 1;
    size_t cap = (size_t)(tf - 1) * hop_bytes + frame_bytes + 48;  // + alignment slack (pre <= 15, round-up <= 15)
    cap = (cap + 15) & ~(size_t)15;
    if (fixed + cap > 227 * 1024) return -1;
    *tile_bytes_cap = (int)cap;
    return tf;
}

cudaError_t abg_launch_k1(const K1Launch& L, cudaStream_t s) {
    K1Args args;
    args.devs = L.devs;
    args.bins = L.bins;
    args.wsc = L.window_scaled;
    args.tw1 = L.tw1;
    args.tw2 = L.tw2;
    args.win = L.win;
    args.iqin = L.iqin;
    args.Gp = L.Gp;
    args.frames_per_tile = L.frames_per_tile;
    args.tile_bytes_cap = L.tile_bytes_cap;
    switch (L.fft_size) {
        case 256: return launch_fmt<8>(L, args, s);
        case 512: return launch_fmt<9>(L, args, s);
        case 1024: return launch_fmt<10>(L, args, s);
        case 2048: return launch_fmt<11>(L, args, s);
        case 4096: return launch_fmt<12>(L, args, s);
        case 8192: return launch_fmt<13>(L, args, s);
    }
    return cudaErrorInvalidValue;
}
