// Carrier frequency meter (abg_carrier_configure / abg_fetch_carrier): per channel and batch, the lag-one correlation
// R = sum_j X_{j+1} * conj(X_j) and the energy E = sum_j |X_j|^2 of the bin value K1 wrote to iqin for the batch's frames.
// The definition is in include/airband_b200.h.
//
// One launch per run covers every metered device.  Work item = (device, batch of the run, group of up to 32 channels):
//   * iqin is time-major [P][Gp], so a row of the group's channels is one contiguous line.  The CTA's 256 threads are
//     CW channel lanes (CW = the group's channel count rounded up to a power of two) times S = 256 / CW row slices; slice
//     s sums, in frame order, E over rows [s*B/S, (s+1)*B/S) and R over the pairs that start there (it reads one row past
//     its end unless it is the batch's last slice: only pairs inside the batch count).
//   * the S slice sums are then added by a fixed binary tree in shared memory.  The order depends on B and the channel
//     count only, never on how batches are grouped into runs, so the sums are bitwise reproducible.
//   * the finished sums go straight into the device's page-locked result ring (mapped); resident runs compute them and
//     store nothing.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/airband_b200.h"
#include "abg_internal.h"

namespace {

constexpr int BLOCK = 256;
constexpr int GROUP = 32;  // channels per work item at most

__global__ void __launch_bounds__(BLOCK) abg_carrier_meter_kernel(const CarArgs a) {
    __shared__ float red[3][BLOCK];
    const CarCfg cf = a.cfg[blockIdx.y];
    const CarRun rn = a.run[blockIdx.y];
    const int groups = (cf.n_channels + GROUP - 1) / GROUP;
    const int item = blockIdx.x;
    if (item >= rn.n_batches * groups) return;
    const int k = item / groups, grp = item % groups;
    const int nc = min(GROUP, cf.n_channels - grp * GROUP);
    int cw = 1;
    while (cw < nc) cw <<= 1;
    const int S = BLOCK / cw, B = a.wave_batch;
    const int tid = threadIdx.x, c = tid & (cw - 1), s = tid / cw;
    const int ch = grp * GROUP + c;  // channel of the device

    float rr = 0.0f, ri = 0.0f, en = 0.0f;
    if (c < nc) {
        const int j0 = (int)((long long)s * B / S), j1 = (int)((long long)(s + 1) * B / S);
        const int jl = min(j1, B - 1);  // last row read: the pair (j1 - 1, j1) belongs to this slice when j1 < B
        const float2* col = a.iqin + ((size_t)ABG_AGC_EXTRA + (size_t)k * B) * a.Gp + cf.g0 + ch;
        if (j0 < j1) {
            float2 x = __ldcg(col + (size_t)j0 * a.Gp);
#pragma unroll 4
            for (int j = j0; j < jl; ++j) {
                const float2 y = __ldcg(col + (size_t)(j + 1) * a.Gp);
                en = fmaf(x.x, x.x, fmaf(x.y, x.y, en));
                rr = fmaf(y.x, x.x, fmaf(y.y, x.y, rr));   // Re(y * conj(x))
                ri = fmaf(y.y, x.x, fmaf(-y.x, x.y, ri));  // Im(y * conj(x))
                x = y;
            }
            if (jl < j1) en = fmaf(x.x, x.x, fmaf(x.y, x.y, en));  // the batch's last frame: energy only
        }
    }
    red[0][tid] = rr;
    red[1][tid] = ri;
    red[2][tid] = en;
    __syncthreads();
    for (int h = S / 2; h >= 1; h >>= 1) {
        if (s < h) {
#pragma unroll
            for (int q = 0; q < 3; ++q) red[q][tid] += red[q][tid + h * cw];
        }
        __syncthreads();
    }
    if (s == 0 && c < nc && rn.ring_pos0 >= 0) {
        float* out = cf.ring + (size_t)((rn.ring_pos0 + k) % cf.ring_cap) * 3 * cf.n_channels;
        out[2 * ch] = red[0][tid];
        out[2 * ch + 1] = red[1][tid];
        out[2 * cf.n_channels + ch] = red[2][tid];
    }
}

}  // namespace

int abg_carrier_items(int n_channels) { return (n_channels + GROUP - 1) / GROUP; }

cudaError_t abg_launch_carrier(const CarArgs& a, int n_devices, int max_items, cudaStream_t s) {
    if (n_devices < 1 || max_items < 1) return cudaSuccess;
    abg_carrier_meter_kernel<<<dim3(max_items, n_devices, 1), BLOCK, 0, s>>>(a);
    return cudaGetLastError();
}
