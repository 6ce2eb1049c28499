// Transmission profiles (abg_history_profile): the statistics of a captured sub-band that tell its modulation, carrier
// offset and CTCSS tone.  The definition is in include/airband_b200.h.
//
// One CTA per entry of a host-built block table.  An entry names the scratch index of its first output, its output count
// n <= ABG_PROFILE_BLOCK and whether the output after its last one was captured (succ); every read of the captured
// outputs stays in [off, off + n + succ), and nothing is derived here from a job's size.
//   * outputs: thread t takes the block's outputs t, t + 256, t + 512, t + 768, computes p, a and (where the successor is
//     in the block or succ is set) z and phi, adds them to its sums in that order and stages phi and a in shared memory;
//     the 7 sums then go through a fixed xor-shuffle tree and the 8 warps' results are added in warp order.
//   * tones: warp w takes the tones w, w + 8, ...; lane l walks the outputs l, l + 32, ... in order, one sincospif of the
//     exact integer phase per output and tone, and adds phi and a times it; then the xor tree.
// Every add is an explicit round-to-nearest intrinsic, so the order written in the header is the order computed.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/airband_b200.h"
#include "abg_internal.h"

namespace {

constexpr int BLOCK = 256;
constexpr int WARPS = BLOCK / 32;
constexpr int PB = ABG_PROFILE_BLOCK;
static_assert(PB % BLOCK == 0, "whole rounds of outputs per thread");
constexpr int NS = 7;  // p1, p2, a1, z.re, z.im, f1, f2

__device__ __forceinline__ float xor_sum(float v) {
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, s));
    return v;
}

__global__ void __launch_bounds__(BLOCK) abg_profile_kernel(const ProfArgs a) {
    __shared__ float s_phi[PB], s_amp[PB];
    __shared__ float s_part[WARPS][NS];
    const ProfBlock b = a.blocks[blockIdx.x];
    const int tid = threadIdx.x, lane = tid % 32, warp = tid / 32;
    const float2* y = a.y + b.off;
    const int n_pairs = b.n - 1 + b.succ;  // pairs (i, i + 1) with i < n_pairs: i + 1 < n + succ
    float acc[NS] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
    for (int r = 0; r < PB / BLOCK; ++r) {
        const int i = tid + r * BLOCK;
        float phi = 0.0f, am = 0.0f;
        if (i < b.n) {
            const float2 u = y[i];
            const float p = __fmaf_rn(u.x, u.x, __fmul_rn(u.y, u.y));
            am = __fsqrt_rn(p);
            acc[0] = __fadd_rn(acc[0], p);
            acc[1] = __fmaf_rn(p, p, acc[1]);
            acc[2] = __fadd_rn(acc[2], am);
            if (i < n_pairs) {
                const float2 v = y[i + 1];
                const float zr = __fmaf_rn(v.x, u.x, __fmul_rn(v.y, u.y));
                const float zi = __fmaf_rn(v.y, u.x, -__fmul_rn(v.x, u.y));
                phi = atan2f(zi, zr);
                acc[3] = __fadd_rn(acc[3], zr);
                acc[4] = __fadd_rn(acc[4], zi);
                acc[5] = __fadd_rn(acc[5], phi);
                acc[6] = __fmaf_rn(phi, phi, acc[6]);
            }
        }
        s_phi[i] = phi;
        s_amp[i] = am;
    }
#pragma unroll
    for (int q = 0; q < NS; ++q) {
        const float v = xor_sum(acc[q]);
        if (lane == 0) s_part[warp][q] = v;
    }
    __syncthreads();
    float* res = a.res + b.res;
    if (tid < NS) {
        float v = s_part[0][tid];
#pragma unroll
        for (int w = 1; w < WARPS; ++w) v = __fadd_rn(v, s_part[w][tid]);
        res[tid] = v;
    } else if (tid == NS) {
        res[NS] = 0.0f;
    }

    const int K = b.K;
    const uint32_t mb = (uint32_t)(unsigned long long)b.m;  // m mod 2^32
    for (int k = warp; k < K; k += WARPS) {
        const uint32_t d = a.delta[b.tones + k];
        float fr = 0.0f, fi = 0.0f, ar = 0.0f, ai = 0.0f;
        for (int i = lane; i < b.n; i += 32) {
            const int32_t ph = (int32_t)(d * (mb + (uint32_t)i));
            float sn, cs;
            sincospif((float)ph * 0x1p-31f, &sn, &cs);
            const float phi = s_phi[i], am = s_amp[i];
            fr = __fmaf_rn(phi, cs, fr);
            fi = __fmaf_rn(-phi, sn, fi);
            ar = __fmaf_rn(am, cs, ar);
            ai = __fmaf_rn(-am, sn, ai);
        }
        fr = xor_sum(fr);
        fi = xor_sum(fi);
        ar = xor_sum(ar);
        ai = xor_sum(ai);
        if (lane == 0) {
            res[ABG_PROFILE_SUMS + 2 * k] = fr;
            res[ABG_PROFILE_SUMS + 2 * k + 1] = fi;
            res[ABG_PROFILE_SUMS + 2 * K + 2 * k] = ar;
            res[ABG_PROFILE_SUMS + 2 * K + 2 * k + 1] = ai;
        }
    }
}

}  // namespace

cudaError_t abg_launch_profile(const ProfArgs& a, int n_blocks, cudaStream_t s) {
    if (n_blocks < 1) return cudaSuccess;
    if (n_blocks > 65535) return cudaErrorInvalidConfiguration;
    abg_profile_kernel<<<n_blocks, BLOCK, 0, s>>>(a);
    return cudaGetLastError();
}
