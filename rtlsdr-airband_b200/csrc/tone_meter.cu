// CTCSS tone meter (abg_tone_meter_configure / abg_fetch_tone_meter): per channel and batch, the DFT of the channel's
// audio at each tone of the engine's list, its energy and its count of non-zero samples.  The definition is in
// include/airband_b200.h.
//
// The phase of sample aB + j splits into a part of the batch and a part of the sample in the batch:
//     S[c][k] = r_k(a) * sum_j y[c][aB + j] * T[j][k],   T[j][k] = exp(-2 pi i (delta_k j mod 2^32) / 2^32),
//     r_k(a)  = exp(-2 pi i (delta_k aB mod 2^32) / 2^32),
// so no oscillator runs per sample: T is built once on the host in double (wave_batch x 2K floats, stays in L2), the sums
// are one FP32 GEMM per run, [metered channel-batches x B] . [B x 2K], and r_k(a) is one double sincospi per (batch, tone)
// from its exact integer phase.
//
// One launch per run on stream B, after K2 and the mixers, before the tail copy overwrites wout[0, AGC_EXTRA).  Grid =
// (tiles of MT metered channels, tiles of ABG_TM_COLS table columns, batch of the run).  Channels of different devices
// share a tile; rows whose device ran fewer batches read as zero and write nothing, and a tile with no live row returns.
//   * register-tiled SIMT GEMM: each thread holds 2 rows x 4 columns; the B dimension goes through shared memory KC
//     samples at a time, the next stage's global loads in flight while the current one is multiplied.
//   * summation order: every accumulator adds its products in sample order j = 0 .. B-1, one fmaf each; E and active
//     are summed by lane l of the row's loading warp over j = l, l + 32, ... in order, then by a fixed xor-shuffle tree.
//     The order depends on (B, K) only, never on the run grouping, the tile or the other rows, so readings are bitwise
//     reproducible whenever the audio is.
//   * results go straight into the device's page-locked result ring (mapped); resident runs compute them and store nothing.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/airband_b200.h"
#include "abg_internal.h"

namespace {

constexpr int BLOCK = 256;
constexpr int MT = 32;            // metered channels (rows) per tile
constexpr int NT = ABG_TM_COLS;   // table columns per tile
constexpr int KC = 32;            // audio samples per shared-memory stage
constexpr int YS = KC + 4;        // row stride of the audio stage: float4-aligned, rows 4 apart on different banks
constexpr int ROWS_PER_WARP = MT / (BLOCK / 32);

__global__ void __launch_bounds__(BLOCK) abg_tone_meter_kernel(const TmArgs a) {
    __shared__ __align__(16) float ys[MT][YS];
    __shared__ __align__(16) float ts[KC][NT];
    __shared__ int s_g[MT], s_m[MT];  // global channel and device slot of each row; s_g < 0: no audio for this batch
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.z, col0 = blockIdx.y * NT;
    const int B = a.wave_batch;

    int live = 0;
    if (tid < MT) {
        const int i = blockIdx.x * MT + tid;
        int g = -1, m = -1;
        if (i < a.n_chan) {
            m = a.chan_dev[i];
            if (b < a.run[m].n_batches) g = a.cfg[m].g0 + (i - a.cfg[m].first);
        }
        s_g[tid] = g;
        s_m[tid] = m;
        live = g >= 0;
    }
    if (!__syncthreads_or(live)) return;

    // loaders: warp w stages rows w + 8 r (r < ROWS_PER_WARP), lane = sample of the stage; the table stage is 512 float4
    const float* yrow[ROWS_PER_WARP];
#pragma unroll
    for (int r = 0; r < ROWS_PER_WARP; ++r) {
        const int g = s_g[warp + 8 * r];
        yrow[r] = g >= 0 ? a.wout + (size_t)g * a.P + (size_t)b * B : nullptr;
    }
    const bool meter_energy = blockIdx.y == 0;
    float en[ROWS_PER_WARP];
    int act[ROWS_PER_WARP];
#pragma unroll
    for (int r = 0; r < ROWS_PER_WARP; ++r) { en[r] = 0.0f; act[r] = 0; }

    float yv[ROWS_PER_WARP];
    float4 tv[2];
    auto load = [&](int c0) {
        const int j = c0 + lane;
#pragma unroll
        for (int r = 0; r < ROWS_PER_WARP; ++r) yv[r] = (yrow[r] && j < B) ? __ldcg(yrow[r] + j) : 0.0f;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int idx = tid + BLOCK * q, k = idx / (NT / 4), n4 = idx % (NT / 4);
            tv[q] = c0 + k < B ? __ldg(reinterpret_cast<const float4*>(a.table + (size_t)(c0 + k) * a.n_cols + col0) + n4)
                               : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        }
    };

    const int tm = tid >> 4, tn = tid & 15;  // compute: rows 2 tm, 2 tm + 1; columns 4 tn .. 4 tn + 3 of the tile
    float acc[2][4];
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = 0.0f;

    load(0);
    for (int c0 = 0; c0 < B; c0 += KC) {
#pragma unroll
        for (int r = 0; r < ROWS_PER_WARP; ++r) {
            ys[warp + 8 * r][lane] = yv[r];
            if (meter_energy) {
                en[r] = fmaf(yv[r], yv[r], en[r]);
                act[r] += yv[r] != 0.0f;
            }
        }
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int idx = tid + BLOCK * q;
            reinterpret_cast<float4*>(&ts[idx / (NT / 4)][0])[idx % (NT / 4)] = tv[q];
        }
        __syncthreads();
        if (c0 + KC < B) load(c0 + KC);
#pragma unroll
        for (int kk = 0; kk < KC; kk += 4) {
            const float4 y0 = *reinterpret_cast<const float4*>(&ys[2 * tm][kk]);
            const float4 y1 = *reinterpret_cast<const float4*>(&ys[2 * tm + 1][kk]);
            const float yy[2][4] = {{y0.x, y0.y, y0.z, y0.w}, {y1.x, y1.y, y1.z, y1.w}};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float4 t = *reinterpret_cast<const float4*>(&ts[kk + q][4 * tn]);
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    acc[r][0] = fmaf(yy[r][q], t.x, acc[r][0]);
                    acc[r][1] = fmaf(yy[r][q], t.y, acc[r][1]);
                    acc[r][2] = fmaf(yy[r][q], t.z, acc[r][2]);
                    acc[r][3] = fmaf(yy[r][q], t.w, acc[r][3]);
                }
            }
        }
        __syncthreads();
    }

    // S = r_k(a) * (column 2k + i column 2k+1), straight into the ring entry [C][K][2]
    const int K = a.K;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = 2 * tm + r, g = s_g[row];
        if (g < 0) continue;
        const int m = s_m[row];
        const TmRun rn = a.run[m];
        if (rn.ring_pos0 < 0) continue;
        const TmCfg cf = a.cfg[m];
        const int c = g - cf.g0;
        const uint32_t base = (uint32_t)((rn.seq0 + (unsigned long long)b) * (unsigned long long)B);  // aB mod 2^32
        float* out = cf.ring + (size_t)((rn.ring_pos0 + b) % cf.ring_cap) * cf.n_channels * (2 * ABG_TONE_MAX + 2);
#pragma unroll
        for (int p = 0; p < 2; ++p) {
            const int k = (col0 + 4 * tn) / 2 + p;
            if (k >= K) continue;
            const uint32_t ph = a.delta[k] * base;
            double sn, cs;
            sincospi((double)(int32_t)ph * 0x1p-31, &sn, &cs);  // 2 pi * turns, turns in [-1/2, 1/2)
            const float rr = (float)cs, ri = (float)-sn;
            const float ar = acc[r][2 * p], ai = acc[r][2 * p + 1];
            float2 s;
            s.x = fmaf(rr, ar, -ri * ai);
            s.y = fmaf(rr, ai, ri * ar);
            reinterpret_cast<float2*>(out)[(size_t)c * K + k] = s;
        }
    }

    // E and active of the rows this warp staged: lane sums, then a fixed xor-shuffle tree
    if (!meter_energy) return;
#pragma unroll
    for (int r = 0; r < ROWS_PER_WARP; ++r) {
        float e = en[r];
        int n = act[r];
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) {
            e += __shfl_xor_sync(0xffffffffu, e, o);
            n += __shfl_xor_sync(0xffffffffu, n, o);
        }
        const int row = warp + 8 * r, g = s_g[row];
        if (lane != 0 || g < 0) continue;
        const int m = s_m[row];
        const TmRun rn = a.run[m];
        if (rn.ring_pos0 < 0) continue;
        const TmCfg cf = a.cfg[m];
        const int c = g - cf.g0;
        float* out = cf.ring + (size_t)((rn.ring_pos0 + b) % cf.ring_cap) * cf.n_channels * (2 * ABG_TONE_MAX + 2);
        out[(size_t)cf.n_channels * 2 * K + c] = e;
        reinterpret_cast<int32_t*>(out)[(size_t)cf.n_channels * (2 * K + 1) + c] = n;
    }
}

}  // namespace

cudaError_t abg_launch_tone_meter(const TmArgs& a, int max_batches, cudaStream_t s) {
    if (a.n_chan < 1 || max_batches < 1) return cudaSuccess;
    abg_tone_meter_kernel<<<dim3((a.n_chan + MT - 1) / MT, a.n_cols / NT, max_batches), BLOCK, 0, s>>>(a);
    return cudaGetLastError();
}
