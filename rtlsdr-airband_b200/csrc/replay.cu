// History replay (abg_history_replay): the gather that feeds a device's I/Q history into the replay engine's input
// buffers, in place of abg_push's host->device copy.  The definition is in include/airband_b200.h.
//
// One launch per chunk moves, for every job, the next bytes of its window from the parent's history ring (stream byte b
// at b mod R, R % 16 == 0) to raw[cur] + fill of the job's device in the replay engine.  Work item = (slice of the job's
// bytes, job).  The destination is an arbitrary byte address and so is the source's ring position: they differ modulo 16
// whenever the window starts at a sample whose byte offset is not a multiple of 16 (hop 313 at 2.5 Msps).  So every
// thread owns one 16-byte aligned destination vector and builds it from the two aligned ring vectors it straddles: the
// shift k = (source byte) mod 16 is the same for every vector of a job, because R is a multiple of 16, and the second
// vector of the pair wraps with the ring.  The head and tail up to a 16-byte boundary of the destination go byte by byte.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "abg_internal.h"

namespace {

constexpr int BLOCK = 256;

// bytes [k, k + 16) of the 32-byte concatenation lo:hi, k in [0, 16)
__device__ __forceinline__ uint4 shift_pair(const uint4 lo, const uint4 hi, const unsigned k) {
    const unsigned ws = k >> 2, bs = (k & 3) * 8;
    // word-level shift by ws from selects, then a funnel shift by bs: no dynamically indexed array, so no local memory
    const uint32_t w0 = ws == 0 ? lo.x : ws == 1 ? lo.y : ws == 2 ? lo.z : lo.w;
    const uint32_t w1 = ws == 0 ? lo.y : ws == 1 ? lo.z : ws == 2 ? lo.w : hi.x;
    const uint32_t w2 = ws == 0 ? lo.z : ws == 1 ? lo.w : ws == 2 ? hi.x : hi.y;
    const uint32_t w3 = ws == 0 ? lo.w : ws == 1 ? hi.x : ws == 2 ? hi.y : hi.z;
    const uint32_t w4 = ws == 0 ? hi.x : ws == 1 ? hi.y : ws == 2 ? hi.z : hi.w;
    return make_uint4(__funnelshift_r(w0, w1, bs), __funnelshift_r(w1, w2, bs), __funnelshift_r(w2, w3, bs),
                      __funnelshift_r(w3, w4, bs));
}

__global__ void __launch_bounds__(BLOCK) abg_replay_gather_kernel(const RpGather* __restrict__ jobs) {
    const RpGather g = jobs[blockIdx.y];
    const unsigned long long n = g.n_bytes, R = g.ring_bytes;
    if (n == 0) return;
    const unsigned char* ring = g.ring;
    unsigned char* dst = g.dst;
    const unsigned long long p0 = g.src % R;  // ring position of dst[0]
    const unsigned long long head = min(n, (unsigned long long)((16 - ((uintptr_t)dst & 15)) & 15));
    const unsigned long long n_vec = (n - head) / 16, tail0 = head + n_vec * 16;
    const int tid = threadIdx.x;
    if (blockIdx.x == 0) {
        if ((unsigned long long)tid < head) {
            const unsigned long long p = p0 + tid;
            dst[tid] = ring[p >= R ? p - R : p];
        } else if (tid >= 32 && (unsigned long long)(tid - 32) < n - tail0) {
            const unsigned long long i = tail0 + (tid - 32), p = (p0 + i) % R;
            dst[i] = ring[p];
        }
    }
    const unsigned long long first = (p0 + head) % R;  // ring position of the first whole destination vector
    const unsigned k = (unsigned)(first & 15);
    const unsigned long long q_first = first - k;    // its aligned ring vector
    const unsigned long long stride = (unsigned long long)gridDim.x * BLOCK;
#pragma unroll 2
    for (unsigned long long v = (unsigned long long)blockIdx.x * BLOCK + tid; v < n_vec; v += stride) {
        unsigned long long q0 = q_first + v * 16;
        q0 = q0 >= R ? q0 % R : q0;
        const uint4 lo = __ldg(reinterpret_cast<const uint4*>(ring + q0));
        uint4 out = lo;
        if (k) {
            const unsigned long long q1 = q0 + 16 == R ? 0 : q0 + 16;
            out = shift_pair(lo, __ldg(reinterpret_cast<const uint4*>(ring + q1)), k);
        }
        *reinterpret_cast<uint4*>(dst + head + v * 16) = out;
    }
}

}  // namespace

cudaError_t abg_launch_replay_gather(const RpGather* jobs, int n_jobs, int blocks_per_job, cudaStream_t s) {
    if (n_jobs < 1 || blocks_per_job < 1) return cudaSuccess;
    abg_replay_gather_kernel<<<dim3(blocks_per_job, n_jobs, 1), BLOCK, 0, s>>>(jobs);
    return cudaGetLastError();
}
