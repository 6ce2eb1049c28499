// The arithmetic that fixes the bits of a sub-band output (definition at abg_subband_configure in include/airband_b200.h),
// shared by the live outputs (subband.cu) and the capture from the I/Q history (history.cu), so that both compute every
// y[m] with the same operations in the same order: level conversion, tap sum, rotation.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/airband_b200.h"

// One complex sample at p (2, 4 or 8 bytes, aligned to its size): the input meter's float32 levels
template <int SFMT>
__device__ __forceinline__ float2 sb_level(const unsigned char* p, float scale, const float* lut8) {
    if constexpr (SFMT == ABG_SFMT_U8) {
        const uchar2 c = *reinterpret_cast<const uchar2*>(p);
        return make_float2(lut8[c.x], lut8[c.y]);
    } else if constexpr (SFMT == ABG_SFMT_S8) {
        const char2 c = *reinterpret_cast<const char2*>(p);
        return make_float2(__fmul_rn((float)c.x, 0.0078125f), __fmul_rn((float)c.y, 0.0078125f));  // c / 128.0f, exact
    } else if constexpr (SFMT == ABG_SFMT_S16) {
        const short2 x = *reinterpret_cast<const short2*>(p);
        return make_float2(__fmul_rn(scale, (float)x.x), __fmul_rn(scale, (float)x.y));
    } else {
        const float2 x = *reinterpret_cast<const float2*>(p);
        return make_float2(__fmul_rn(scale, x.x), __fmul_rn(scale, x.y));
    }
}

// 16 bytes that start with an I component -> 16 / bpc samples at dst (16-byte aligned)
template <int SFMT>
__device__ __forceinline__ void sb_level_vec(uint4 q, float scale, const float* lut8, float2* dst) {
    float4* d4 = reinterpret_cast<float4*>(dst);
    if constexpr (SFMT == ABG_SFMT_U8 || SFMT == ABG_SFMT_S8) {
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {  // two samples per word: I0 Q0 I1 Q1
            float c[4];
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                const uint32_t code = (w[i] >> (8 * b)) & 0xffu;
                c[b] = SFMT == ABG_SFMT_U8 ? lut8[code] : __fmul_rn((float)(signed char)code, 0.0078125f);
            }
            d4[i] = make_float4(c[0], c[1], c[2], c[3]);
        }
    } else if constexpr (SFMT == ABG_SFMT_S16) {
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
        float c[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            c[2 * i] = __fmul_rn(scale, (float)(short)(w[i] & 0xffffu));
            c[2 * i + 1] = __fmul_rn(scale, (float)(short)(w[i] >> 16));
        }
        d4[0] = make_float4(c[0], c[1], c[2], c[3]);
        d4[1] = make_float4(c[4], c[5], c[6], c[7]);
    } else {
        d4[0] = make_float4(__fmul_rn(scale, __uint_as_float(q.x)), __fmul_rn(scale, __uint_as_float(q.y)),
                            __fmul_rn(scale, __uint_as_float(q.z)), __fmul_rn(scale, __uint_as_float(q.w)));
    }
}

// The U8 level table, one entry per thread of a 256-thread block (the caller synchronises before use)
__device__ __forceinline__ void sb_lut8_fill(float* lut8, int tid) { lut8[tid] = __fdiv_rn(__fsub_rn((float)tid, 127.5f), 127.5f); }

// One tap of y[m] = sum_j g[j] v[mD - j]: complex h * v added to (ar, ai) in the fixed order of the four roundings.  A
// warp sums one output: lane l adds the taps j = l, l + 32, ... in order (the loop stays in each caller: the live kernel
// keeps its register allocation only with the loop in its own body), then sb_xor_tree adds the 32 lanes.
__device__ __forceinline__ void sb_tap(float2 h, float2 v, float& ar, float& ai) {
    ar = __fmaf_rn(h.x, v.x, ar);
    ar = __fmaf_rn(-h.y, v.y, ar);
    ai = __fmaf_rn(h.x, v.y, ai);
    ai = __fmaf_rn(h.y, v.x, ai);
}

// The warp's fixed xor-shuffle tree: afterwards every lane holds the sum of all 32 lanes' partial sums
__device__ __forceinline__ void sb_xor_tree(float& ar, float& ai) {
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) {
        ar = __fadd_rn(ar, __shfl_xor_sync(0xffffffffu, ar, s));
        ai = __fadd_rn(ai, __shfl_xor_sync(0xffffffffu, ai, s));
    }
}

// y * exp(-2 pi i p / 2^32) with p = delta * x mod 2^32 (x = mD, the output's newest sample), as a signed turn fraction in
// [-1/2, 1/2): the exact integer phase through a double sincospi
__device__ __forceinline__ float2 sb_rotate(float yr, float yi, uint32_t delta, long long x) {
    const int32_t p = (int32_t)(delta * (uint32_t)(unsigned long long)x);
    double sn, cs;
    sincospi((double)p * 0x1p-31, &sn, &cs);
    const float cf32 = (float)cs, sf32 = (float)sn;
    return make_float2(__fmaf_rn(yr, cf32, __fmul_rn(yi, sf32)), __fmaf_rn(yi, cf32, -__fmul_rn(yr, sf32)));
}
