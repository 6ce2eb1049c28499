// Sub-band I/Q outputs (abg_subband_configure / abg_fetch_subband): per device up to ABG_SUBBAND_MAX digital
// down-converters (mixer, FIR low-pass, decimator) over the raw samples.  The definition is in include/airband_b200.h.
//
// One launch per run covers every device with an output on.  Work item = (device, batch of the run, chunk): a chunk is
// CHUNK consecutive input samples counted from the batch's first sample, and carries the outputs m of every output of
// the device with mD inside it, so the items depend on the batch only, never on how batches are grouped into runs.
//   * staging: the CTA converts the chunk plus the device's hist = L_max - 1 samples before it into shared memory once
//     (float32 levels exactly as the input meter's conversion), then computes every output of the device from it: the
//     raw bytes are read once per device, not once per output.  Samples below the buffer's first one (dropped by
//     compaction before the output started, or before the stream) are staged as zero.  16-byte vector loads for the
//     aligned middle, single samples for the head and tail (the buffers keep stream offsets modulo 16).
//   * oscillator after the filter: y[m] = exp(-2 pi i (delta mD mod 2^32) / 2^32) * sum_j g[j] v[mD - j] with the complex
//     coefficients g[j] = h[j] exp(+2 pi i delta j / 2^32), built on the host in double.  This equals the definition up
//     to rounding and needs one rotation per output instead of one per input sample and output; the rotation comes from
//     the exact integer phase through a double sincospi, never from a running product.
//   * summation order: one warp per output, lane l adds the taps j = l, l + 32, ... in order, then a fixed xor-shuffle
//     tree.  A warp sums 32 consecutive outputs in turn and then rotates all 32 at once, one per lane.  Taps whose sample lies before the output's start are not added (adding their zero would change nothing), and
//     which ones they are depends on (m, start) only.  So each y[m] is bitwise the same whatever chunk, run or launch
//     computes it.
//   * results: tiles of TILE outputs go through shared memory and are written with consecutive threads on consecutive
//     outputs straight into the output's page-locked result ring (mapped), unless the run is resident.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/airband_b200.h"
#include "abg_internal.h"
#include "subband_dsp.cuh"

namespace {

constexpr int BLOCK = 256;
constexpr int WARPS = BLOCK / 32;
constexpr int CHUNK = 8192;  // input samples per work item
constexpr int TILE = 256;    // outputs per coalesced write to the ring
constexpr int PAD = 8;       // the staging origin is rounded down to a 16-byte boundary: up to 7 extra samples

__host__ __device__ constexpr size_t smem_bytes(int hist) {
    return sizeof(float2) * ((size_t)CHUNK + hist + PAD) + sizeof(float2) * TILE + sizeof(float) * 256;
}

__device__ __forceinline__ long long ceil_div(long long a, long long b) {  // a >= 0, b >= 1
    return (a + b - 1) / b;
}

template <int SFMT>
__device__ void subband_item(const SbCfg& cf, const SbRun& rn, int k, int c, unsigned char* smem) {
    constexpr int BPC = SFMT == ABG_SFMT_F32 ? 8 : SFMT == ABG_SFMT_S16 ? 4 : 2;  // bytes per complex sample
    constexpr int SPV = 16 / BPC;                                               // samples per 16-byte vector
    const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
    float2* sv = reinterpret_cast<float2*>(smem);
    float2* tile = sv + CHUNK + cf.hist + PAD;
    float* lut8 = reinterpret_cast<float*>(tile + TILE);
    if constexpr (SFMT == ABG_SFMT_U8) {
        static_assert(BLOCK == 256, "one thread per U8 code");
        sb_lut8_fill(lut8, tid);
        __syncthreads();
    }
    const float scale = cf.scale;

    // ---- stage samples [a_lo, a_hi) at sv[a - a_org] ----
    const long long sb = rn.s0 + (long long)k * cf.batch_samples;  // the batch's first sample
    const long long c0 = sb + (long long)c * CHUNK;
    const int clen = min(CHUNK, cf.batch_samples - c * CHUNK);
    const long long a_lo = c0 - cf.hist, a_hi = c0 + clen;
    const long long a_org = a_lo & ~(long long)(SPV - 1);  // floor, also for a_lo < 0
    long long v_lo = (a_lo + SPV - 1) & ~(long long)(SPV - 1), v_hi = a_hi & ~(long long)(SPV - 1);
    if (v_hi < v_lo) v_lo = v_hi = a_hi;  // no whole vector inside: all head
    // base is a multiple of SPV, so a vector lies wholly below or wholly inside the buffer
    const unsigned char* raw = rn.raw;
    const int n_head = (int)(v_lo - a_lo), n_tail = (int)(a_hi - v_hi), n_vec = (int)((v_hi - v_lo) / SPV);
    if (tid < n_head) {
        const long long a = a_lo + tid;
        sv[a - a_org] = a < rn.base ? make_float2(0.0f, 0.0f) : sb_level<SFMT>(raw + (a - rn.base) * BPC, scale, lut8);
    } else if (tid >= 32 && tid - 32 < n_tail) {
        const long long a = v_hi + (tid - 32);
        sv[a - a_org] = a < rn.base ? make_float2(0.0f, 0.0f) : sb_level<SFMT>(raw + (a - rn.base) * BPC, scale, lut8);
    }
#pragma unroll 4
    for (int i = tid; i < n_vec; i += BLOCK) {
        const long long a = v_lo + (long long)i * SPV;
        float2* dst = sv + (a - a_org);
        if (a < rn.base) {
#pragma unroll
            for (int s = 0; s < SPV; ++s) dst[s] = make_float2(0.0f, 0.0f);
        } else {
            sb_level_vec<SFMT>(__ldg(reinterpret_cast<const uint4*>(raw + (a - rn.base) * BPC)), scale, lut8, dst);
        }
    }
    __syncthreads();

    // ---- every output of the device ----
    for (int o = 0; o < cf.n_out; ++o) {
        const SbOut& so = cf.out[o];
        const long long D = so.decim;
        const int L = so.n_coeffs;
        const long long start = rn.s0 - rn.lead[o];
        const long long m_b0 = ceil_div(sb, D), m_lo = ceil_div(c0, D), m_hi = ceil_div(c0 + clen, D);
        float2* out = rn.ring_pos0[o] >= 0
                          ? reinterpret_cast<float2*>(so.ring + (size_t)((rn.ring_pos0[o] + k) % so.ring_cap) * so.entry_bytes)
                          : nullptr;
        const float2* g = so.coef;
        for (long long mt = m_lo; mt < m_hi; mt += TILE) {
            const int cnt = (int)min((long long)TILE, m_hi - mt);
            // warp w sums outputs 32w .. 32w + 31 of the tile one after another; lane q keeps output q's sum and rotates it
            for (int i0 = warp * 32; i0 < cnt; i0 += WARPS * 32) {
                const int nq = min(32, cnt - i0);
                float yr = 0.0f, yi = 0.0f;
                for (int q = 0; q < nq; ++q) {
                    const long long x = (mt + i0 + q) * D;  // absolute index of the output's newest sample
                    const float2* vx = sv + (x - a_org);
                    const int jmax = (int)min((long long)L, x - start + 1);
                    float ar = 0.0f, ai = 0.0f;
#pragma unroll 4
                    for (int j = lane; j < jmax; j += 32) sb_tap(__ldg(g + j), vx[-j], ar, ai);
                    sb_xor_tree(ar, ai);
                    if (lane == q) {
                        yr = ar;
                        yi = ai;
                    }
                }
                if (lane < nq) {
                    tile[i0 + lane] = sb_rotate(yr, yi, so.delta, (mt + i0 + lane) * D);
                }
            }
            __syncthreads();
            if (out)
                for (int i = tid; i < cnt; i += BLOCK) out[mt - m_b0 + i] = tile[i];
            __syncthreads();
        }
    }
}

__global__ void __launch_bounds__(BLOCK, 2) abg_subband_kernel(const SbArgs a) {
    extern __shared__ __align__(16) unsigned char smem[];
    const SbCfg& cf = a.cfg[blockIdx.y];
    const SbRun& rn = a.run[blockIdx.y];
    const int n_chunks = cf.n_chunks;
    const int item = blockIdx.x;
    if (item >= rn.n_batches * n_chunks) return;
    const int k = item / n_chunks, c = item % n_chunks;
    switch (cf.sfmt) {
        case ABG_SFMT_U8: subband_item<ABG_SFMT_U8>(cf, rn, k, c, smem); break;
        case ABG_SFMT_S8: subband_item<ABG_SFMT_S8>(cf, rn, k, c, smem); break;
        case ABG_SFMT_S16: subband_item<ABG_SFMT_S16>(cf, rn, k, c, smem); break;
        default: subband_item<ABG_SFMT_F32>(cf, rn, k, c, smem); break;
    }
}

}  // namespace

int abg_subband_chunks(int batch_samples) { return (batch_samples + CHUNK - 1) / CHUNK; }

cudaError_t abg_launch_subband(const SbArgs& a, int n_devices, int max_items, int max_hist, cudaStream_t s) {
    if (n_devices < 1 || max_items < 1) return cudaSuccess;
    const size_t smem = smem_bytes(max_hist);
    if (smem > 48 * 1024) {  // a host-side attribute of the current device, no launch
        const cudaError_t er = cudaFuncSetAttribute(abg_subband_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (er != cudaSuccess) return er;
    }
    abg_subband_kernel<<<dim3(max_items, n_devices, 1), BLOCK, smem, s>>>(a);
    return cudaGetLastError();
}
