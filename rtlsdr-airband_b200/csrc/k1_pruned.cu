// K1 (output-pruned) — fused sample conversion + window + FFT + per-channel bin extraction, computing ONLY the
// configured bins in the last pass (sm_90a).  Same inputs, same outputs as k1_fft.cu; replaces the same reference
// code (reference src/rtl_airband.cpp:402-455 convert+window, :460 fftwf_execute, :483-489 bin extraction).
//
// The reference runs a full N-point FFT per frame and then reads C of the N bins (C = channels of the device,
// 1..49 in the shipped configs).  A decimation-in-time split N = R1 * M1 (R1 = 8 or 16) makes the second half
// of that work sparse:
//     X[b] = sum_{c < M1}  W_N^(c*b) * Y_c[b mod R1],        Y_c = R1-point DFT of the column x[c + M1*n1]
// so this kernel runs the R1-point column FFTs for every column (fully unrolled register FFT, compile-time
// twiddles) and then, per configured bin, one complex dot product over the M1 columns — instead of the remaining
// log2(M1) butterfly stages over all N points.  One warp owns one frame; lane l holds columns
// 2l + 64m + {0,1}; the dot product is a per-lane partial (coefficients factor as W^(2l*b) * W^((64m+p)*b): the second
// factor is warp-uniform and is read as a shared-memory broadcast, the first is applied once per channel) followed by
// one shared-memory transposed reduction for all channels of the frame.  No spectrum ever leaves registers, no
// inter-pass exchange buffer, no block-wide barrier inside the frame loop.  The window multiply is folded into the first
// radix-2 stage, and the channels are visited in FFT-row order (sorted once per CTA) so that the row a channel reads is
// a compile-time register index.
//
// Frames of a tile are staged once by a TMA bulk copy exactly as in k1_fft.cu (frames overlap by N-hop samples).
// Devices with AFC need the whole spectrum of batch-final frames (reference src/rtl_airband.cpp:180-251) and keep
// using the full-spectrum kernel.
#include <algorithm>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include <type_traits>

#include "../../include/airband_b200.h"
#include "abg_internal.h"
#include "k1_common.cuh"

namespace {
using namespace k1;

constexpr int PR_WARPS = 4;          // warps (= frames in flight) per CTA
constexpr int PR_MAXCH = 32;         // channels handled per pass of the kernel
constexpr int PR_PAD = 33;           // padded row length of the partial-sum matrix
constexpr int PR_ROWTAB = 20;        // row-start table (R1 + 1 <= 17 entries), padded to a multiple of 16 bytes


struct PrArgs {
    const K1Dev* devs;
    const int32_t* bins;
    const float* wsc;       // window * 1/full-scale, [N]
    const float2* twn;      // W_N^m, m = 0..N-1
    float* win;
    float2* iqin;
    int Gp;
    int frames_per_tile;
    int ch0;                // first channel of the device handled by this launch
    int nchmax;             // channels per pass the shared-memory layout is sized for (<= PR_MAXCH)
};

// per-lane conversion of one sample to (I, Q) before scaling; U8 uses one PRMT + one FADD per component:
// 0x47000000 | b << 8 is the float 32768 + b (ulp 2^-8), minus 32895.5 gives b - 127.5 exactly.
template <int SFMT>
__device__ __forceinline__ float2 load_sample_pr(const unsigned char* tile, int byte_off) {
    if constexpr (SFMT == ABG_SFMT_U8) {
        const unsigned int u = *reinterpret_cast<const unsigned short*>(tile + byte_off);
        const float i = __uint_as_float(__byte_perm(u, 0x47000000u, 0x7604)) - 32895.5f;  // bytes: [3]=0x47 [2]=0x00 [1]=u.b0 [0]=0x00
        const float q = __uint_as_float(__byte_perm(u, 0x47000000u, 0x7614)) - 32895.5f;  // [1]=u.b1
        return make_float2(i, q);
    } else {
        return load_sample<SFMT>(tile, byte_off);
    }
}

// two adjacent samples (n, n+1); for 8-bit formats one 32-bit shared load when the pair is 4-byte aligned
template <int SFMT, bool AL4>
__device__ __forceinline__ void load_pair_pr(const unsigned char* tile, int byte_off, float2& x0, float2& x1) {
    if constexpr (SFMT == ABG_SFMT_U8 && AL4) {
        const unsigned int u = *reinterpret_cast<const unsigned int*>(tile + byte_off);
        x0.x = __uint_as_float(__byte_perm(u, 0x47000000u, 0x7604)) - 32895.5f;
        x0.y = __uint_as_float(__byte_perm(u, 0x47000000u, 0x7614)) - 32895.5f;
        x1.x = __uint_as_float(__byte_perm(u, 0x47000000u, 0x7624)) - 32895.5f;
        x1.y = __uint_as_float(__byte_perm(u, 0x47000000u, 0x7634)) - 32895.5f;
    } else {
        x0 = load_sample_pr<SFMT>(tile, byte_off);
        x1 = load_sample_pr<SFMT>(tile, byte_off + bytes_per_cplx<SFMT>());
    }
}

// f(std::integral_constant<int, 0>{}), ..., f(std::integral_constant<int, N - 1>{})
template <int... Is, class F>
__device__ __forceinline__ void pr_static_for_impl(std::integer_sequence<int, Is...>, F& f) {
    (f(std::integral_constant<int, Is>{}), ...);
}
template <int N, class F>
__device__ __forceinline__ void pr_static_for(F& f) {
    pr_static_for_impl(std::make_integer_sequence<int, N>{}, f);
}

template <int LOGN, int SFMT, int R1, int PR_GELEM>
__global__ void __launch_bounds__(PR_WARPS * 32) k1_pruned_kernel(const PrArgs a) {
    constexpr int N = 1 << LOGN;
    constexpr int E = N / 32;                  // samples per lane
    static_assert(E >= R1, "column radix larger than the per-lane share");
    constexpr int NCOL = E / R1;               // columns per lane
    constexpr int M1 = N / R1;                 // columns per frame
    constexpr int PAIR = NCOL >= 2 ? 2 : 1;    // adjacent columns owned by one lane
    constexpr int GELEM = PR_GELEM;            // complex values held in registers at once (per lane)
    constexpr int GCOL = (NCOL * R1 > GELEM) ? (GELEM / R1 >= PAIR ? GELEM / R1 : PAIR) : NCOL;  // columns per register group
    constexpr int NGRP = NCOL / GCOL;
    constexpr int BPC = bytes_per_cplx<SFMT>();

    extern __shared__ __align__(128) unsigned char smem[];
    unsigned long long* mbar = reinterpret_cast<unsigned long long*>(smem);
    const int CM = a.nchmax;                                                         // multiple of 4
    int* s_order = reinterpret_cast<int*>(smem + 16);                                // [CM] channels sorted by FFT row (bin mod R1)
    int* s_rowstart = s_order + CM;                                                  // [PR_ROWTAB] first sorted position of every row
    float2* s_U = reinterpret_cast<float2*>(smem + 16 + (CM + PR_ROWTAB) * sizeof(int));  // [CM][NCOL] warp-uniform factors
    float2* s_base = s_U + CM * NCOL;                                                // [CM][32] per-lane factors
    float* s_part = reinterpret_cast<float*>(s_base + CM * 32);                      // [PR_WARPS][2*CM][PR_PAD]
    unsigned char* tile = reinterpret_cast<unsigned char*>(s_part + PR_WARPS * 2 * CM * PR_PAD);
    // CM is a multiple of 4, so every section is a multiple of 16 bytes and `tile` stays 16-byte aligned for TMA

    const K1Dev dv = a.devs[blockIdx.y];
    const int f0 = blockIdx.x * a.frames_per_tile;
    if (f0 >= dv.n_frames) return;
    const int nch = min(CM, dv.n_channels - a.ch0);
    if (nch <= 0) return;
    const int nf = min(a.frames_per_tile, dv.n_frames - f0);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    // ---- stage the tile's raw bytes with one TMA bulk copy ----
    const unsigned long long s_byte = dv.start_byte + (unsigned long long)f0 * dv.hop_bytes;
    const unsigned long long a_byte = s_byte & ~15ull;
    const int pre = (int)(s_byte - a_byte);
    const unsigned int copy_bytes = (unsigned int)((pre + (nf - 1) * dv.hop_bytes + N * BPC + 15) & ~15);
    if (tid == 0) mbar_init(mbar);
    __syncthreads();
    if (tid == 0) tma_tile_load(mbar, tile, dv.raw + a_byte, copy_bytes);

    // ---- meanwhile: per-channel tables for this device ----
    const int gbase = dv.g0 + a.ch0;
    // The channel loop below walks the FFT rows in a fixed (unrolled) order and, inside a row, the channels whose bin
    // falls on it: the row is then a compile-time register index and no per-channel dispatch is needed.  Warp 0 sorts the
    // (<= 32) channels by row with a rank count.
    if (tid < 32) {
        const int myrow = (tid < nch) ? (a.bins[gbase + tid] & (N - 1)) % R1 : R1;  // R1 = "no channel"
        int rank = 0, below = 0;
        for (int o = 0; o < nch; ++o) {
            const int ro = __shfl_sync(0xffffffffu, myrow, o);
            rank += (ro < myrow || (ro == myrow && o < tid)) ? 1 : 0;
            below += (ro < tid) ? 1 : 0;      // channels on rows < tid
        }
        if (tid < nch) s_order[rank] = tid;
        if (tid <= R1) s_rowstart[tid] = below;
    }
    for (int i = tid; i < nch * NCOL; i += PR_WARPS * 32) {
        const int c = i / NCOL, j = i % NCOL;
        const int b = a.bins[gbase + c] & (N - 1);
        const int coff = (PAIR * 32) * (j / PAIR) + (j % PAIR);        // column offset that does not depend on the lane
        s_U[c * NCOL + j] = __ldg(a.twn + ((coff * b) & (N - 1)));
    }
    for (int i = tid; i < nch * 32; i += PR_WARPS * 32) {
        const int c = i >> 5, l = i & 31;
        const int b = a.bins[gbase + c] & (N - 1);
        s_base[c * 32 + l] = __ldg(a.twn + (((PAIR * l) * b) & (N - 1)));
    }
    __syncthreads();
    mbar_wait0(mbar);

    float* part = s_part + warp * (2 * CM * PR_PAD);
    // (partial sums go through shared memory: register-resident accumulators across the groups for devices with few
    // channels need ~100 registers and a much larger unrolled body)
    const float* __restrict__ wsc = a.wsc;
    const int iters = (nf + PR_WARPS - 1) / PR_WARPS;
    for (int it = 0; it < iters; ++it) {
        const int fl = it * PR_WARPS + warp;
        if (fl >= nf) break;  // warp-uniform
        const int fo = pre + fl * dv.hop_bytes;
        const int pos = dv.pos0 + f0 + fl;
#pragma unroll 1
        for (int grp = 0; grp < NGRP; ++grp) {
            // ---- load + convert + window: GCOL columns of R1 samples ----
            float2 v[GCOL][R1];
            // The window multiply is folded into the first radix-2 stage of the column FFT: that stage pairs sample n1 with
            // sample n1 + R1/2 (logical A[2m], A[2m+1] live in v[m'] and v[m' + R1/2]), so with a = xa*wa the butterfly
            // outputs are fma(xb, wb, a) and fma(-xb, wb, a): 3 instructions per real pair instead of 2 FMUL + 2 FADD.
            auto load_group = [&](auto al4_tag) {
                constexpr bool AL4 = decltype(al4_tag)::value;
#pragma unroll
                for (int jj = 0; jj < GCOL; jj += PAIR) {
                    const int j = grp * GCOL + jj;
                    const int c0 = PAIR * lane + (PAIR * 32) * (j / PAIR);     // first column of the pair
#pragma unroll
                    for (int n1 = 0; n1 < R1 / 2; ++n1) {
                        const int na = c0 + M1 * n1, nb = c0 + M1 * (n1 + R1 / 2);
                        if constexpr (PAIR == 2) {
                            const float2 wa = __ldg(reinterpret_cast<const float2*>(wsc + na));
                            const float2 wb = __ldg(reinterpret_cast<const float2*>(wsc + nb));
                            float2 xa0, xa1, xb0, xb1;
                            load_pair_pr<SFMT, AL4>(tile, fo + na * BPC, xa0, xa1);
                            load_pair_pr<SFMT, AL4>(tile, fo + nb * BPC, xb0, xb1);
                            const float a0x = xa0.x * wa.x, a0y = xa0.y * wa.x, a1x = xa1.x * wa.y, a1y = xa1.y * wa.y;
                            v[jj][n1] = make_float2(fmaf(xb0.x, wb.x, a0x), fmaf(xb0.y, wb.x, a0y));
                            v[jj][n1 + R1 / 2] = make_float2(fmaf(-xb0.x, wb.x, a0x), fmaf(-xb0.y, wb.x, a0y));
                            v[jj + 1][n1] = make_float2(fmaf(xb1.x, wb.y, a1x), fmaf(xb1.y, wb.y, a1y));
                            v[jj + 1][n1 + R1 / 2] = make_float2(fmaf(-xb1.x, wb.y, a1x), fmaf(-xb1.y, wb.y, a1y));
                        } else {
                            const float wa = __ldg(wsc + na), wb = __ldg(wsc + nb);
                            const float2 xa = load_sample_pr<SFMT>(tile, fo + na * BPC);
                            const float2 xb = load_sample_pr<SFMT>(tile, fo + nb * BPC);
                            const float ax = xa.x * wa, ay = xa.y * wa;
                            v[jj][n1] = make_float2(fmaf(xb.x, wb, ax), fmaf(xb.y, wb, ay));
                            v[jj][n1 + R1 / 2] = make_float2(fmaf(-xb.x, wb, ax), fmaf(-xb.y, wb, ay));
                        }
                    }
                }
            };
            if (SFMT == ABG_SFMT_U8 && PAIR == 2 && (fo & 3) == 0)  // frame start 4-byte aligned in the tile (always, for even hops)
                load_group(std::true_type{});
            else
                load_group(std::false_type{});
            // ---- remaining stages of the R1-point FFT of every column (result row k in v[col][brev(k)]) ----
#pragma unroll
            for (int jj = 0; jj < GCOL; ++jj) dit_from<R1, 4>(v[jj]);

            // ---- per FFT row, per channel on that row: lane-partial of the dot product over this group's columns ----
            auto row_channels = [&](auto row_tag) {
                constexpr int R = decltype(row_tag)::value;
                const int i1 = s_rowstart[R + 1];
#pragma unroll 1
                for (int i = s_rowstart[R]; i < i1; ++i) {  // warp-uniform bounds
                    const int c = s_order[i];
                    const float2* U = s_U + c * NCOL + grp * GCOL;
                    // the group's warp-uniform factors (16-byte rows: s_U and GCOL*8 are multiples of 16 bytes, so two
                    // columns come with one 128-bit broadcast load)
                    float2 uu[GCOL];
                    if constexpr (GCOL % 2 == 0) {
#pragma unroll
                        for (int jj = 0; jj < GCOL; jj += 2) {
                            const float4 t4 = *reinterpret_cast<const float4*>(U + jj);
                            uu[jj] = make_float2(t4.x, t4.y);
                            uu[jj + 1] = make_float2(t4.z, t4.w);
                        }
                    } else {
#pragma unroll
                        for (int jj = 0; jj < GCOL; ++jj) uu[jj] = U[jj];
                    }
                    float sr = 0.0f, si = 0.0f;
#pragma unroll
                    for (int jj = 0; jj < GCOL; ++jj) {
                        const float2 u = uu[jj];
                        const float2 y = v[jj][brev<R1>(R)];
                        sr = fmaf(y.x, u.x, sr);
                        sr = fmaf(-y.y, u.y, sr);
                        si = fmaf(y.x, u.y, si);
                        si = fmaf(y.y, u.x, si);
                    }
                    // sums of the groups accumulate in shared memory; the per-lane factor W^(PAIR*lane*b) is the same for
                    // every group, so it is applied once, by the last one
                    if (NGRP > 1 && grp > 0) {
                        sr += part[(2 * c) * PR_PAD + lane];
                        si += part[(2 * c + 1) * PR_PAD + lane];
                    }
                    if (grp == NGRP - 1) {
                        const float2 bf = s_base[c * 32 + lane];
                        const float tr = fmaf(sr, bf.x, -si * bf.y), ti = fmaf(sr, bf.y, si * bf.x);
                        sr = tr;
                        si = ti;
                    }
                    part[(2 * c) * PR_PAD + lane] = sr;
                    part[(2 * c + 1) * PR_PAD + lane] = si;
                }
            };
            pr_static_for<R1>(row_channels);
        }
        __syncwarp();

        // ---- reduce over the 32 lanes, all channels of the frame at once (transposed read of the partial matrix):
        //      value index vi = 2*ch + {re,im}; NVP values are handled per pass by 32/NVP lanes each
        const int nv = 2 * nch;
        const int NVP = nv >= 32 ? 32 : (nv > 16 ? 32 : (nv > 8 ? 16 : (nv > 4 ? 8 : (nv > 2 ? 4 : 2))));
        const int SUB = 32 / NVP;            // lanes sharing one value
        const int LPS = 32 / SUB;            // partials each of them adds up (= NVP)
        for (int vi0 = 0; vi0 < nv; vi0 += NVP) {
            const int vi = vi0 + (lane & (NVP - 1));
            const int sub = lane / NVP;
            float sum = 0.0f;
            if (vi < nv) {
                const float* pv = part + vi * PR_PAD + sub * LPS;
#pragma unroll 4
                for (int l = 0; l < LPS; ++l) sum += pv[l];
            }
            for (int o = NVP; o < 32; o <<= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
            const float other = __shfl_xor_sync(0xffffffffu, sum, 1);  // (re, im) of a channel sit in adjacent lanes
            if (vi < nv && !(vi & 1) && lane < NVP) {
                const int c = vi >> 1;
                const float re = sum, imv = other;
                const float mag = sqrtf(__fadd_rn(__fmul_rn(re, re), __fmul_rn(imv, imv)));  // rtl_airband.cpp:484
                const size_t o = (size_t)pos * a.Gp + gbase + c;
                a.win[o] = mag;
                a.iqin[o] = make_float2(re, imv);
            }
        }
        __syncwarp();
    }
}

size_t pr_fixed_smem(int fft_size, int r1, int cm) {
    const int ncol = fft_size / 32 / r1;
    return 16 + (cm + PR_ROWTAB) * sizeof(int) + sizeof(float2) * (size_t)cm * ncol + sizeof(float2) * (size_t)cm * 32 + sizeof(float) * PR_WARPS * 2 * (size_t)cm * PR_PAD;
}
int pr_cm(int max_channels) {  // channels per pass: multiple of 4, at most PR_MAXCH
    int cm = (max_channels + 3) & ~3;
    return cm < 4 ? 4 : (cm > PR_MAXCH ? PR_MAXCH : cm);
}

template <int LOGN, int SFMT, int R1, int GE>
cudaError_t pr_launch_one2(const K1Launch& L, const PrArgs& args, cudaStream_t s) {
    size_t smem = pr_fixed_smem(1 << LOGN, R1, args.nchmax) + (size_t)L.tile_bytes_cap;
    // experiment knob: cap the resident CTAs per SM by padding the shared-memory request (228 KB per SM, 1 KB reserved per CTA)
    static int max_ctas = -1;
    if (max_ctas < 0) {
        const char* e = getenv("ABG_K1_MAX_CTAS_PER_SM");
        max_ctas = e ? atoi(e) : 0;
    }
    if (max_ctas > 0) smem = std::max(smem, (size_t)(228 * 1024 / (max_ctas + 1) + 1024));
    auto kern = k1_pruned_kernel<LOGN, SFMT, R1, GE>;
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
    dim3 grid(tiles, L.n_devices, 1), block(PR_WARPS * 32, 1, 1);
    kern<<<grid, block, smem, s>>>(args);
    return cudaGetLastError();
}

template <int LOGN, int SFMT, int R1>
cudaError_t pr_launch_one(const K1Launch& L, const PrArgs& args, cudaStream_t s) {
    // complex values held in registers per lane at once: 64 (a whole 2048-point frame in one pass over the channels, 167
    // registers, 12 warps/SM) or, with ABG_K1_GELEM=32, 32 (two passes, 96 registers, 20 warps/SM).  Since the channel loop
    // lost its per-channel dispatch the single pass wins (cfg2: K1 0.450 vs 0.480 ms alone, step 0.615 vs 0.655 ms).
    static int ge = 0;
    if (ge == 0) {
        const char* e = getenv("ABG_K1_GELEM");
        ge = (e && atoi(e) == 32) ? 32 : 64;
    }
    if (ge == 32) return pr_launch_one2<LOGN, SFMT, R1, 32>(L, args, s);
    return pr_launch_one2<LOGN, SFMT, R1, 64>(L, args, s);
}

template <int LOGN, int R1>
cudaError_t pr_launch_fmt(const K1Launch& L, const PrArgs& args, cudaStream_t s) {
    switch (L.sfmt) {
        case ABG_SFMT_U8: return pr_launch_one<LOGN, ABG_SFMT_U8, R1>(L, args, s);
        case ABG_SFMT_S8: return pr_launch_one<LOGN, ABG_SFMT_S8, R1>(L, args, s);
        case ABG_SFMT_S16: return pr_launch_one<LOGN, ABG_SFMT_S16, R1>(L, args, s);
        case ABG_SFMT_F32: return pr_launch_one<LOGN, ABG_SFMT_F32, R1>(L, args, s);
    }
    return cudaErrorInvalidValue;
}

int pr_radix(int fft_size, int max_channels) {
    // R1 = 8 keeps the column FFTs cheapest; with many channels the dot products dominate and R1 = 16 halves them
    if (fft_size <= 256) return 8;
    return max_channels > 12 ? 16 : 8;
}

}  // namespace

// Frames per tile / raw-tile bytes for the pruned kernel (targets 3-4 CTAs per SM).
int abg_k1p_tile_frames(int fft_size, int sfmt, int hop_bytes, int max_channels, int* tile_bytes_cap) {
    const int r1 = pr_radix(fft_size, max_channels);
    const int bpc = (sfmt == ABG_SFMT_U8 || sfmt == ABG_SFMT_S8) ? 2 : (sfmt == ABG_SFMT_S16 ? 4 : 8);
    const size_t fixed = pr_fixed_smem(fft_size, r1, pr_cm(max_channels));
    const size_t frame_bytes = (size_t)fft_size * bpc;
    size_t per_cta = 48 * 1024;  // 3 CTAs per SM are register-limited (167 registers/thread); 48 KB tiles measured best on cfg2
    if (const char* e = getenv("ABG_K1_CTA_KB")) per_cta = (size_t)atoi(e) * 1024;
    size_t budget = per_cta > fixed + frame_bytes + 64 ? per_cta - fixed : frame_bytes + 64;
    if (fixed + budget > 220 * 1024) return -1;
    int tf = 1;
    if (budget > frame_bytes + 64) tf = 1 + (int)((budget - frame_bytes - 64) / (size_t)hop_bytes);
    tf = (tf / PR_WARPS) * PR_WARPS;
    if (tf > 64) tf = 64;
    if (tf < PR_WARPS) tf = PR_WARPS;
    size_t cap = (size_t)(tf - 1) * hop_bytes + frame_bytes + 48;
    cap = (cap + 15) & ~(size_t)15;
    if (fixed + cap > 227 * 1024) return -1;
    *tile_bytes_cap = (int)cap;
    return tf;
}

// `twn` = W_N^m table; `max_channels` = largest channel count among the launch's devices.
cudaError_t abg_launch_k1_pruned(const K1Launch& L, const float2* twn, int max_channels, cudaStream_t s) {
    const int r1 = pr_radix(L.fft_size, max_channels);
    cudaError_t err = cudaSuccess;
    for (int ch0 = 0; ch0 < max_channels && err == cudaSuccess; ch0 += PR_MAXCH) {
        PrArgs args;
        args.devs = L.devs; args.bins = L.bins; args.wsc = L.window_scaled; args.twn = twn; args.win = L.win; args.iqin = L.iqin;
        args.Gp = L.Gp; args.frames_per_tile = L.frames_per_tile; args.ch0 = ch0; args.nchmax = pr_cm(max_channels);
#define PR_DISPATCH(LOGN)                                                                                       \
    err = (r1 == 8) ? pr_launch_fmt<LOGN, 8>(L, args, s) : pr_launch_fmt<LOGN, 16>(L, args, s);                \
    break;
        switch (L.fft_size) {
            case 256: err = pr_launch_fmt<8, 8>(L, args, s); break;
            case 512: PR_DISPATCH(9)
            case 1024: PR_DISPATCH(10)
            case 2048: PR_DISPATCH(11)
            case 4096: PR_DISPATCH(12)
            case 8192: PR_DISPATCH(13)
            default: err = cudaErrorInvalidValue;
        }
#undef PR_DISPATCH
    }
    return err;
}
