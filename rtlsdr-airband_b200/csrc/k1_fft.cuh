// The full-spectrum FFT of one frame, shared by K1's full-spectrum kernel (k1_fft.cu) and the band-spectrum kernel
// (spectrum.cu): conversion + window fused into the first pass, then 2 (3 for N = 8192) register passes that exchange
// through a padded shared-memory buffer.  The caller supplies what happens to the last pass's registers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "k1_common.cuh"

namespace k1 {

// ---------------------------------------------------------------------------------------------------------------
// per-size plan: pass radices, threads per frame (T) and threads per CTA (BLOCK); BLOCK / T frames are in flight
// ---------------------------------------------------------------------------------------------------------------
template <int LOGN>
struct Plan;
template <>
struct Plan<8> { static constexpr int R1 = 16, R2 = 16, R3 = 0, T = 16, BLOCK = 128; };
template <>
struct Plan<9> { static constexpr int R1 = 32, R2 = 16, R3 = 0, T = 16, BLOCK = 128; };
template <>
struct Plan<10> { static constexpr int R1 = 32, R2 = 32, R3 = 0, T = 32, BLOCK = 128; };
template <>
struct Plan<11> { static constexpr int R1 = 64, R2 = 32, R3 = 0, T = 32, BLOCK = 128; };
template <>
struct Plan<12> { static constexpr int R1 = 64, R2 = 64, R3 = 0, T = 64, BLOCK = 128; };
template <>
struct Plan<13> { static constexpr int R1 = 32, R2 = 16, R3 = 16, T = 256, BLOCK = 256; };

template <int LOGN>
struct FftShape {
    using P = Plan<LOGN>;
    static constexpr int N = 1 << LOGN;
    static constexpr bool THREE = P::R3 != 0;
    static constexpr int RL = THREE ? P::R3 : P::R2;  // last-pass radix
    static constexpr int M1 = N / P::R1;               // pass-1 butterflies per frame
    static constexpr int S = P::BLOCK / P::T;          // frames in flight per CTA
    static constexpr int PADSH = ilog2(RL);            // exchange padding: one float2 every RL
    static constexpr int EXN = N + (N >> PADSH);       // padded exchange elements per frame
    static constexpr int NQL = N / RL;                 // last-pass butterflies per frame
    // natural-order bin held in register r of last-pass butterfly q
    static __device__ __forceinline__ int bin_of(int q, int r) {
        if constexpr (!THREE)
            return q + P::R1 * r;
        else
            return (q / P::R2) + P::R1 * ((q % P::R2) + P::R2 * r);
    }
};

template <int T>
__device__ __forceinline__ void frame_sync(int slot) {
    if constexpr (T <= 32) {
        __syncwarp();
    } else {
        asm volatile("bar.sync %0, %1;" ::"r"(slot + 1), "r"(T) : "memory");
    }
}

// One frame on the T threads of a slot (lt = thread within the slot).  `src` points at the frame's first raw byte (shared
// or global memory); `ex` is the slot's exchange buffer (EXN float2).  For each last-pass butterfly q of this thread,
// emit(v, q) receives the registers: bin bin_of(q, r) is v[brev<RL>(r)].  Every thread of the slot calls this, active or
// not: it contains the slot's barriers, including the final one after which `ex` may be reused.
template <int LOGN, int SFMT, typename Emit>
__device__ __forceinline__ void fft_frame(const unsigned char* src, bool active, int slot, int lt, float2* ex, const float* __restrict__ wsc,
                                          const float2* __restrict__ tw1, const float2* __restrict__ tw2, Emit&& emit) {
    using P = Plan<LOGN>;
    using F = FftShape<LOGN>;
    constexpr int R1 = P::R1, R2 = P::R2, R3 = P::R3, T = P::T;
    constexpr int M1 = F::M1, PADSH = F::PADSH, NQL = F::NQL;
    constexpr int BPC = bytes_per_cplx<SFMT>();

    // ---------------- pass 1: radix-R1 columns, window fused into the load -----------------------------
    if (active) {
#pragma unroll 1
        for (int n2 = lt; n2 < M1; n2 += T) {
            float2 v[R1];
#pragma unroll
            for (int n1 = 0; n1 < R1; ++n1) {
                const int n = n2 + M1 * n1;
                const float2 x = load_sample<SFMT>(src, n * BPC);
                const float w = __ldg(wsc + n);
                v[n1] = make_float2(x.x * w, x.y * w);
            }
            reg_fft<R1>(v);
            ex[n2 + (n2 >> PADSH)] = v[0];
#pragma unroll
            for (int k1 = 1; k1 < R1; ++k1) {
                const float2 t = __ldg(tw1 + k1 * M1 + n2);
                const float2 y = v[brev<R1>(k1)];
                const int e = k1 * M1 + n2;
                ex[e + (e >> PADSH)] = make_float2(fmaf(-y.y, t.y, y.x * t.x), fmaf(y.y, t.x, y.x * t.y));
            }
        }
    }
    frame_sync<T>(slot);

    if constexpr (!F::THREE) {
        // ------------- pass 2 (last): rows of length R2 = M1; bin k1 + R1*k2 ends up in register k2 -------
        if (active) {
#pragma unroll 1
            for (int q = lt; q < NQL; q += T) {
                float2 v[R2];
#pragma unroll
                for (int j = 0; j < R2; ++j) {
                    const int e = q * M1 + j;
                    v[j] = ex[e + (e >> PADSH)];
                }
                reg_fft<R2>(v);
                emit(v, q);
            }
        }
    } else {
        // ------------- pass 2 of 3: radix R2 inside each length-M1 block, twiddle W_M1^(n3*k2a) ------------
        constexpr int M2 = R3;
        if (active) {
#pragma unroll 1
            for (int q = lt; q < F::N / R2; q += T) {
                const int k1 = q / M2, n3 = q % M2;
                const int base = k1 * M1 + n3;
                float2 v[R2];
#pragma unroll
                for (int j = 0; j < R2; ++j) {
                    const int e = base + M2 * j;
                    v[j] = ex[e + (e >> PADSH)];
                }
                reg_fft<R2>(v);
                ex[base + (base >> PADSH)] = v[0];
#pragma unroll
                for (int k = 1; k < R2; ++k) {
                    const float2 t = __ldg(tw2 + k * M2 + n3);
                    const float2 y = v[brev<R2>(k)];
                    const int e = base + M2 * k;
                    ex[e + (e >> PADSH)] = make_float2(fmaf(-y.y, t.y, y.x * t.x), fmaf(y.y, t.x, y.x * t.y));
                }
            }
        }
        frame_sync<T>(slot);
        // ------------- pass 3 (last) -----------------------------------------------------------------------
        if (active) {
#pragma unroll 1
            for (int q = lt; q < NQL; q += T) {
                float2 v[R3 == 0 ? 1 : R3];
#pragma unroll
                for (int j = 0; j < R3; ++j) {
                    const int e = q * R3 + j;
                    v[j] = ex[e + (e >> PADSH)];
                }
                reg_fft<(R3 == 0 ? 1 : R3)>(v);
                emit(v, q);
            }
        }
    }
    frame_sync<T>(slot);  // the exchange buffer is reused by this slot's next frame
}

}  // namespace k1
