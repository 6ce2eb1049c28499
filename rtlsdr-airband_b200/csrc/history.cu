// I/Q history (abg_history_configure / abg_history_raw / abg_history_subband): per device a ring of the most recent raw
// bytes in HBM, and a down-converter that cuts a sub-band out of it after the fact.  The definition is in
// include/airband_b200.h.
//
// Ring: R bytes, R a multiple of 16; stream byte b (sample s starts at b = s * bpc) lives at b mod R.  Positions keep
// stream offsets modulo 16, so a 16-byte vector of the stream is a 16-byte vector of the ring and never straddles the wrap.
//   * append: one launch per run for every device with the history on, after the run's other readers of raw[].  Work item
//     = (slice of the device's bytes, device): the run's bytes are a contiguous range of raw[cur] (or of the resident
//     buffer) whose address agrees with its ring position modulo 16, so the copy is 16-byte loads and stores, with the
//     head and tail up to a 16-byte boundary done byte by byte.  The host passes at most the last R bytes of a run, so no
//     ring byte is written twice in a launch.
//   * capture: a digital down-converter over the ring with the sub-band outputs' own arithmetic (subband_dsp.cuh).  Work
//     item = up to `per_item` consecutive outputs m; the CTA stages the samples [m_lo D - (L - 1), m_hi D] they read as
//     float32 levels, then one warp sums 32 outputs in turn and rotates them, one per lane, exactly as subband.cu does.
//     Every tap of every output lies in the history (the host checks it), so there is no zero fill, and each y[m] is
//     bitwise what a live output with all L taps after its start computes.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "../../include/airband_b200.h"
#include "abg_internal.h"
#include "subband_dsp.cuh"

namespace {

constexpr int BLOCK = 256;
constexpr int WARPS = BLOCK / 32;
constexpr int CHUNK = 8192;  // staged input samples per capture item, at most, beyond the filter's L - 1
constexpr int TILE = 256;    // outputs per capture item, at most
constexpr int PAD = 8;       // the staging origin is rounded down to a 16-byte boundary: up to 7 extra samples

__global__ void __launch_bounds__(BLOCK) abg_history_append_kernel(const HiArgs a) {
    const HiCfg cf = a.cfg[blockIdx.y];
    const HiRun rn = a.run[blockIdx.y];
    const unsigned long long n = rn.n_bytes, R = cf.ring_bytes;
    if (n == 0) return;
    const unsigned char* src = rn.src;
    unsigned char* ring = cf.ring;
    // rn.dst < R and every offset i < n <= R: one conditional subtraction wraps
    const unsigned long long head = min(n, (unsigned long long)((16 - ((uintptr_t)src & 15)) & 15));
    const unsigned long long n_vec = (n - head) / 16, tail0 = head + n_vec * 16;
    const int tid = threadIdx.x;
    if (blockIdx.x == 0) {
        if ((unsigned long long)tid < head) {
            const unsigned long long p = rn.dst + tid;
            ring[p >= R ? p - R : p] = src[tid];
        } else if (tid >= 32 && (unsigned long long)(tid - 32) < n - tail0) {
            const unsigned long long i = tail0 + (tid - 32), p = rn.dst + i;
            ring[p >= R ? p - R : p] = src[i];
        }
    }
    const unsigned long long stride = (unsigned long long)gridDim.x * BLOCK;
#pragma unroll 4
    for (unsigned long long v = (unsigned long long)blockIdx.x * BLOCK + tid; v < n_vec; v += stride) {
        const unsigned long long i = head + v * 16, p = rn.dst + i;
        const uint4 q = __ldg(reinterpret_cast<const uint4*>(src + i));
        __stcs(reinterpret_cast<uint4*>(ring + (p >= R ? p - R : p)), q);
    }
}

template <int SFMT>
__device__ void capture_item(const HiCapture& c, unsigned char* smem) {
    constexpr int BPC = SFMT == ABG_SFMT_F32 ? 8 : SFMT == ABG_SFMT_S16 ? 4 : 2;  // bytes per complex sample
    constexpr int SPV = 16 / BPC;                                               // samples per 16-byte vector
    const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
    float2* sv = reinterpret_cast<float2*>(smem);
    float* lut8 = reinterpret_cast<float*>(sv + c.stage);
    if constexpr (SFMT == ABG_SFMT_U8) {
        static_assert(BLOCK == 256, "one thread per U8 code");
        sb_lut8_fill(lut8, tid);
        __syncthreads();
    }
    const float scale = c.scale;
    const long long D = c.decim;
    const int L = c.n_coeffs;
    const long long m_lo = c.m0 + (long long)blockIdx.x * c.per_item;
    const int cnt = (int)min((long long)c.per_item, c.m0 + c.n_out - m_lo);

    // ---- stage samples [a_lo, a_hi) at sv[a - a_org]; every one lies in the history, a_lo >= 0 ----
    const long long a_lo = m_lo * D - (L - 1), a_hi = (m_lo + cnt - 1) * D + 1;
    const long long a_org = a_lo & ~(long long)(SPV - 1);
    long long v_lo = (a_lo + SPV - 1) & ~(long long)(SPV - 1), v_hi = a_hi & ~(long long)(SPV - 1);
    if (v_hi < v_lo) v_lo = v_hi = a_hi;  // no whole vector inside: all head
    const unsigned char* ring = c.ring;
    const unsigned long long R = c.ring_bytes;
    const int n_head = (int)(v_lo - a_lo), n_tail = (int)(a_hi - v_hi), n_vec = (int)((v_hi - v_lo) / SPV);
    if (tid < n_head) {
        const long long a = a_lo + tid;
        sv[a - a_org] = sb_level<SFMT>(ring + (unsigned long long)a * BPC % R, scale, lut8);
    } else if (tid >= 32 && tid - 32 < n_tail) {
        const long long a = v_hi + (tid - 32);
        sv[a - a_org] = sb_level<SFMT>(ring + (unsigned long long)a * BPC % R, scale, lut8);
    }
#pragma unroll 4
    for (int i = tid; i < n_vec; i += BLOCK) {
        const long long a = v_lo + (long long)i * SPV;  // a * BPC % 16 == 0, so its ring position is 16-byte aligned
        sb_level_vec<SFMT>(__ldg(reinterpret_cast<const uint4*>(ring + (unsigned long long)a * BPC % R)), scale, lut8, sv + (a - a_org));
    }
    __syncthreads();

    // ---- the item's outputs: warp w sums outputs 32w .. 32w + 31 one after another; lane q keeps output q's sum ----
    const float2* g = c.coef;
    for (int i0 = warp * 32; i0 < cnt; i0 += WARPS * 32) {
        const int nq = min(32, cnt - i0);
        float yr = 0.0f, yi = 0.0f;
        for (int q = 0; q < nq; ++q) {
            const long long x = (m_lo + i0 + q) * D;  // absolute index of the output's newest sample
            const float2* vx = sv + (x - a_org);
            float ar = 0.0f, ai = 0.0f;
#pragma unroll 4
            for (int j = lane; j < L; j += 32) sb_tap(__ldg(g + j), vx[-j], ar, ai);
            sb_xor_tree(ar, ai);
            if (lane == q) {
                yr = ar;
                yi = ai;
            }
        }
        if (lane < nq) c.out[m_lo - c.m0 + i0 + lane] = sb_rotate(yr, yi, c.delta, (m_lo + i0 + lane) * D);
    }
}

__global__ void __launch_bounds__(BLOCK) abg_history_capture_kernel(const HiCapture c) {
    extern __shared__ __align__(16) unsigned char smem[];
    switch (c.sfmt) {
        case ABG_SFMT_U8: capture_item<ABG_SFMT_U8>(c, smem); break;
        case ABG_SFMT_S8: capture_item<ABG_SFMT_S8>(c, smem); break;
        case ABG_SFMT_S16: capture_item<ABG_SFMT_S16>(c, smem); break;
        default: capture_item<ABG_SFMT_F32>(c, smem); break;
    }
}

}  // namespace

int abg_history_blocks(unsigned long long max_bytes, int n_devices, int sm_count) {
    // one wave of 8 CTAs per SM over all devices, but no CTA without a vector to copy
    const unsigned long long fill = ((unsigned long long)sm_count * 8 + n_devices - 1) / n_devices;
    const unsigned long long need = (max_bytes / 16 + BLOCK - 1) / BLOCK;
    return (int)std::max(1ull, std::min(fill, need));
}

cudaError_t abg_launch_history_append(const HiArgs& a, int n_devices, int blocks_per_device, cudaStream_t s) {
    if (n_devices < 1 || blocks_per_device < 1) return cudaSuccess;
    abg_history_append_kernel<<<dim3(blocks_per_device, n_devices, 1), BLOCK, 0, s>>>(a);
    return cudaGetLastError();
}

int abg_history_per_item(long long decim) { return (int)std::max(1ll, std::min((long long)TILE, CHUNK / decim)); }

cudaError_t abg_launch_history_capture(HiCapture c, cudaStream_t s) {
    if (c.n_out < 1) return cudaSuccess;
    c.per_item = abg_history_per_item(c.decim);
    c.stage = (int)((c.per_item - 1) * (long long)c.decim + c.n_coeffs + PAD);
    c.stage = (c.stage + 1) & ~1;  // the U8 table after the samples stays 16-byte aligned
    const size_t smem = sizeof(float2) * (size_t)c.stage + sizeof(float) * 256;
    if (smem > 48 * 1024) {  // a host-side attribute of the current device, no launch
        const cudaError_t er = cudaFuncSetAttribute(abg_history_capture_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (er != cudaSuccess) return er;
    }
    const int items = (c.n_out + c.per_item - 1) / c.per_item;
    abg_history_capture_kernel<<<items, BLOCK, smem, s>>>(c);
    return cudaGetLastError();
}
