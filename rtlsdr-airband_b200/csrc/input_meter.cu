// Input level meter (abg_input_meter_configure / abg_fetch_input_levels): per device and batch the histogram, peak and
// first and second moments of the I and Q levels of the raw samples the batch advanced over.  The definition is in
// include/airband_b200.h.
//
// One launch per run covers every metered device.  Work item = (device, batch of the run, chunk): a chunk is CHUNK
// consecutive bytes of the batch's byte range, counted from the batch's first byte, so the items depend on the batch
// only, never on how batches are grouped into runs.
//   * the range need not be 16-byte aligned (hop 313, S16 / F32 strides), but it starts on a sample and so does every
//     16-byte boundary inside it (a sample is 2, 4 or 8 bytes and the buffers keep stream offsets modulo 16).  Each
//     chunk therefore splits into a head of whole samples up to the first 16-byte boundary, 16-byte vectors, and a tail
//     of whole samples; every 16-byte vector starts with an I component.
//   * histogram: each warp counts into a private shared-memory sub-histogram (low-gain noise falls into a few codes, and
//     a single histogram would serialise the whole CTA on them), then the CTA adds its eight sub-histograms into the
//     batch's global histogram with integer atomics: order-free and exact.
//   * moments: 8-bit formats take sum and sum_sq from the batch's histogram and only accumulate sum_iq (an integer sum of
//     code products); S16 accumulates integer sums of the codes; F32 adds the float32 levels in double.  Each thread sums
//     its samples in a fixed order, a shuffle tree and the warp order fix the CTA's order, and the chunk sums go to
//     partial[batch][chunk].
//   * the CTA that arrives last at the batch's counter adds the chunk sums in chunk order, converts the integer sums once,
//     writes the reading straight into the device's page-locked result ring (mapped) unless the run is resident, and
//     resets the batch's histogram and counter for the next launch.
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/airband_b200.h"
#include "abg_internal.h"

namespace {

constexpr int BLOCK = 256;
constexpr int WARPS = BLOCK / 32;
constexpr int VECS = 8;                     // 16-byte vectors per thread and chunk
constexpr int CHUNK = BLOCK * 16 * VECS;    // bytes per work item
constexpr int HBINS = 512;                  // [I, Q] x 256

// clamp(floor((v + 1) * 128), 0, 255) in float32 without contraction (a NaN level counts in bin 0)
__device__ __forceinline__ int level_bin(float v) {
    const float t = floorf(__fmul_rn(__fadd_rn(v, 1.0f), 128.0f));
    return (int)fminf(fmaxf(t, 0.0f), 255.0f);
}

// Per-thread sums.  Integer formats: s/ss/iq are the centred integer codes' sums (8-bit: iq only); F32: the levels'.
template <int SFMT>
struct Acc {
    static constexpr bool INT8 = SFMT == ABG_SFMT_U8 || SFMT == ABG_SFMT_S8;
    using T = typename std::conditional<SFMT == ABG_SFMT_F32, double, long long>::type;
    T s[2] = {0, 0}, ss[2] = {0, 0}, iq = 0;
    float peak[2] = {0.0f, 0.0f};
    int iq8 = 0;  // 8-bit: at most 66 samples (64 from vectors, one head, one tail) of |u_I u_Q| <= 255^2 per thread and chunk

    __device__ __forceinline__ void code8(uint32_t cI, uint32_t cQ, uint32_t* hs) {
        if constexpr (SFMT == ABG_SFMT_U8) {
            atomicAdd(hs + cI, 1u);
            atomicAdd(hs + 256 + cQ, 1u);
            iq8 += (2 * (int)cI - 255) * (2 * (int)cQ - 255);
        } else {
            atomicAdd(hs + (cI ^ 0x80u), 1u);
            atomicAdd(hs + 256 + (cQ ^ 0x80u), 1u);
            iq8 += (int)(signed char)cI * (int)(signed char)cQ;
        }
    }
    __device__ __forceinline__ void word8(uint32_t w, uint32_t* hs) {  // two samples: I0 Q0 I1 Q1
        code8(w & 0xffu, (w >> 8) & 0xffu, hs);
        code8((w >> 16) & 0xffu, w >> 24, hs);
    }
    __device__ __forceinline__ void s16(int xI, int xQ, float scale, uint32_t* hs) {
        const float vI = __fmul_rn(scale, (float)xI), vQ = __fmul_rn(scale, (float)xQ);
        atomicAdd(hs + level_bin(vI), 1u);
        atomicAdd(hs + 256 + level_bin(vQ), 1u);
        peak[0] = fmaxf(peak[0], fabsf(vI));
        peak[1] = fmaxf(peak[1], fabsf(vQ));
        s[0] += xI; s[1] += xQ;
        ss[0] += (long long)(xI * xI); ss[1] += (long long)(xQ * xQ);  // |x| <= 32768: the product fits an int
        iq += (long long)xI * xQ;
    }
    __device__ __forceinline__ void f32(float xI, float xQ, float scale, uint32_t* hs) {
        const float vI = __fmul_rn(scale, xI), vQ = __fmul_rn(scale, xQ);
        atomicAdd(hs + level_bin(vI), 1u);
        atomicAdd(hs + 256 + level_bin(vQ), 1u);
        peak[0] = fmaxf(peak[0], fabsf(vI));
        peak[1] = fmaxf(peak[1], fabsf(vQ));
        const double dI = vI, dQ = vQ;
        s[0] = __dadd_rn(s[0], dI); s[1] = __dadd_rn(s[1], dQ);
        ss[0] = __dadd_rn(ss[0], __dmul_rn(dI, dI)); ss[1] = __dadd_rn(ss[1], __dmul_rn(dQ, dQ));
        iq = __dadd_rn(iq, __dmul_rn(dI, dQ));
    }
    // one sample at p (2, 4 or 8 bytes, aligned to its component size)
    __device__ __forceinline__ void sample(const unsigned char* p, float scale, uint32_t* hs) {
        if constexpr (INT8) {
            code8(p[0], p[1], hs);
        } else if constexpr (SFMT == ABG_SFMT_S16) {
            const short2 x = *reinterpret_cast<const short2*>(p);
            s16(x.x, x.y, scale, hs);
        } else {
            const float2 x = *reinterpret_cast<const float2*>(p);
            f32(x.x, x.y, scale, hs);
        }
    }
    // 16 bytes that start with an I component
    __device__ __forceinline__ void vec(uint4 q, float scale, uint32_t* hs) {
        if constexpr (INT8) {
            word8(q.x, hs); word8(q.y, hs); word8(q.z, hs); word8(q.w, hs);
        } else if constexpr (SFMT == ABG_SFMT_S16) {
            s16((short)(q.x & 0xffffu), (short)(q.x >> 16), scale, hs);
            s16((short)(q.y & 0xffffu), (short)(q.y >> 16), scale, hs);
            s16((short)(q.z & 0xffffu), (short)(q.z >> 16), scale, hs);
            s16((short)(q.w & 0xffffu), (short)(q.w >> 16), scale, hs);
        } else {
            f32(__uint_as_float(q.x), __uint_as_float(q.y), scale, hs);
            f32(__uint_as_float(q.z), __uint_as_float(q.w), scale, hs);
        }
    }
};

struct Smem {
    uint32_t hist[WARPS][HBINS];  // per-warp sub-histograms
    long long red[WARPS][5];      // per-warp sums (bit patterns of double for F32)
    float redp[WARPS][2];         // per-warp peaks
    int last;
};

// chunk sums travel through partial[] as 64-bit patterns
__device__ __forceinline__ long long to_bits(long long v) { return v; }
__device__ __forceinline__ long long to_bits(double v) { return __double_as_longlong(v); }
template <class T>
__device__ __forceinline__ T from_bits(long long w) {
    if constexpr (std::is_same<T, double>::value)
        return __longlong_as_double(w);
    else
        return w;
}

template <class T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

template <int SFMT>
__device__ void meter_item(const InmArgs& a, const InmCfg& cf, const InmRun& rn, int k, int c, Smem& sm) {
    using A = Acc<SFMT>;
    using T = typename A::T;
    constexpr int BPC = SFMT == ABG_SFMT_F32 ? 8 : SFMT == ABG_SFMT_S16 ? 4 : 2;  // bytes per complex sample
    auto& hs_all = sm.hist;
    T(&red)[WARPS][5] = *reinterpret_cast<T(*)[WARPS][5]>(&sm.red);
    auto& redp = sm.redp;
    int& last = sm.last;
    const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
    for (int i = tid; i < WARPS * HBINS / 4; i += BLOCK) reinterpret_cast<uint4*>(&hs_all[0][0])[i] = make_uint4(0, 0, 0, 0);
    __syncthreads();
    uint32_t* hs = hs_all[warp];

    const int batch_bytes = a.wave_batch * cf.hop_bytes;
    const unsigned char* batch = rn.raw + rn.first_byte + (unsigned long long)k * batch_bytes;
    const unsigned char* lo = batch + (size_t)c * CHUNK;
    const unsigned char* hi = batch + min(batch_bytes, (c + 1) * CHUNK);
    const unsigned char* v0 = reinterpret_cast<const unsigned char*>((reinterpret_cast<uintptr_t>(lo) + 15) & ~(uintptr_t)15);
    const unsigned char* v1 = reinterpret_cast<const unsigned char*>(reinterpret_cast<uintptr_t>(hi) & ~(uintptr_t)15);
    if (v1 < v0) v0 = v1 = hi;  // no 16-byte boundary pair inside: the whole chunk is head
    A acc;
    const float scale = cf.scale;
    // head, vectors, tail: each thread's samples in address order
    if (tid < (int)(v0 - lo) / BPC) acc.sample(lo + (size_t)tid * BPC, scale, hs);
    const int nvec = (int)(v1 - v0) / 16;
    const uint4* vp = reinterpret_cast<const uint4*>(v0);
#pragma unroll 2
    for (int i = tid; i < nvec; i += BLOCK) acc.vec(__ldg(vp + i), scale, hs);
    if (tid < (int)(hi - v1) / BPC) acc.sample(v1 + (size_t)tid * BPC, scale, hs);

    // chunk sums: shuffle tree per warp, then the warps in order
    T v[5] = {acc.s[0], acc.s[1], acc.ss[0], acc.ss[1], A::INT8 ? (T)acc.iq8 : acc.iq};
#pragma unroll
    for (int q = 0; q < 5; ++q) v[q] = warp_sum(v[q]);
    const float p0 = warp_max(acc.peak[0]), p1 = warp_max(acc.peak[1]);
    if (lane == 0) {
#pragma unroll
        for (int q = 0; q < 5; ++q) red[warp][q] = v[q];
        redp[warp][0] = p0;
        redp[warp][1] = p1;
    }
    __syncthreads();
    uint32_t* hist = cf.hist + (size_t)k * HBINS;
    for (int b = tid; b < HBINS; b += BLOCK) {
        uint32_t n = 0;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) n += hs_all[w][b];
        if (n) atomicAdd(hist + b, n);
    }
    long long* part = cf.partial + (size_t)k * cf.n_chunks * ABG_INM_PARTIAL;
    if (tid == 0) {
        T t[5] = {0, 0, 0, 0, 0};
        float pk[2] = {0.0f, 0.0f};
        for (int w = 0; w < WARPS; ++w) {
#pragma unroll
            for (int q = 0; q < 5; ++q) t[q] += red[w][q];
            pk[0] = fmaxf(pk[0], redp[w][0]);
            pk[1] = fmaxf(pk[1], redp[w][1]);
        }
        long long* mine = part + (size_t)c * ABG_INM_PARTIAL;
#pragma unroll
        for (int q = 0; q < 5; ++q) mine[q] = to_bits(t[q]);
        mine[5] = (long long)(((unsigned long long)__float_as_uint(pk[1]) << 32) | __float_as_uint(pk[0]));
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) last = atomicAdd(cf.counter + k, 1) == cf.n_chunks - 1;
    __syncthreads();
    if (!last) return;
    __threadfence();

    // ---- the batch's last CTA: finish the reading ----
    abg_input_levels* out =
        rn.ring_pos0 >= 0 ? reinterpret_cast<abg_input_levels*>(cf.ring + (size_t)((rn.ring_pos0 + k) % cf.ring_cap) * sizeof(abg_input_levels)) : nullptr;
    long long hsum[4] = {0, 0, 0, 0};  // 8-bit: sum u_I, sum u_Q, sum u_I^2, sum u_Q^2 from the histogram
    int hmax[2] = {0, 0};              // 8-bit: largest |u| of a code in use
    static_assert(BLOCK == 256, "thread t finishes bin t of both components");
#pragma unroll
    for (int comp = 0; comp < 2; ++comp) {
        const int code = tid, b = comp * 256 + code;
        const uint32_t n = __ldcg(hist + b);
        hist[b] = 0;
        if (out) out->hist[comp][code] = n;
        if constexpr (A::INT8) {
            const long long u = SFMT == ABG_SFMT_U8 ? 2 * code - 255 : code - 128;
            hsum[comp] = (long long)n * u;
            hsum[2 + comp] = (long long)n * u * u;
            hmax[comp] = n ? (int)(u < 0 ? -u : u) : 0;
        }
    }
    if constexpr (A::INT8) {
#pragma unroll
        for (int q = 0; q < 4; ++q) hsum[q] = warp_sum(hsum[q]);
        hmax[0] = __reduce_max_sync(0xffffffffu, hmax[0]);
        hmax[1] = __reduce_max_sync(0xffffffffu, hmax[1]);
        __syncthreads();  // red / redp are reused
        if (lane == 0) {
#pragma unroll
            for (int q = 0; q < 4; ++q) red[warp][q] = hsum[q];
            redp[warp][0] = (float)hmax[0];
            redp[warp][1] = (float)hmax[1];
        }
        __syncthreads();
    }
    if (tid != 0) return;
    T t[5] = {0, 0, 0, 0, 0};
    float pk[2] = {0.0f, 0.0f};
    for (int cc = 0; cc < cf.n_chunks; ++cc) {  // chunk order
        const long long* p = part + (size_t)cc * ABG_INM_PARTIAL;
#pragma unroll
        for (int q = 0; q < 5; ++q) {
            t[q] += from_bits<T>(__ldcg(p + q));
        }
        const unsigned long long pw = (unsigned long long)__ldcg(p + 5);
        pk[0] = fmaxf(pk[0], __uint_as_float((uint32_t)pw));
        pk[1] = fmaxf(pk[1], __uint_as_float((uint32_t)(pw >> 32)));
    }
    double sum[2], sq[2], iq;
    if constexpr (A::INT8) {
        long long h[4] = {0, 0, 0, 0};
        for (int w = 0; w < WARPS; ++w) {
#pragma unroll
            for (int q = 0; q < 4; ++q) h[q] += red[w][q];
            pk[0] = fmaxf(pk[0], redp[w][0]);
            pk[1] = fmaxf(pk[1], redp[w][1]);
        }
        // |v| grows with |u|: U8 (c - 127.5f) = u / 2 exactly, S8 u / 128 is exact
#pragma unroll
        for (int q = 0; q < 2; ++q) pk[q] = SFMT == ABG_SFMT_U8 ? __fdiv_rn(0.5f * pk[q], 127.5f) : pk[q] / 128.0f;
        const double d1 = SFMT == ABG_SFMT_U8 ? 255.0 : 128.0, d2 = d1 * d1;  // exact
        sum[0] = (double)h[0] / d1; sum[1] = (double)h[1] / d1;
        sq[0] = (double)h[2] / d2; sq[1] = (double)h[3] / d2;
        iq = (double)t[4] / d2;
    } else if constexpr (SFMT == ABG_SFMT_S16) {
        const double sc = (double)cf.scale, sc2 = sc * sc;
        sum[0] = (double)t[0] * sc; sum[1] = (double)t[1] * sc;
        sq[0] = (double)t[2] * sc2; sq[1] = (double)t[3] * sc2;
        iq = (double)t[4] * sc2;
    } else {
        sum[0] = t[0]; sum[1] = t[1]; sq[0] = t[2]; sq[1] = t[3]; iq = t[4];
    }
    if (out) {
        out->n_samples = (uint64_t)(batch_bytes / BPC);
        out->sum[0] = sum[0]; out->sum[1] = sum[1];
        out->sum_sq[0] = sq[0]; out->sum_sq[1] = sq[1];
        out->sum_iq = iq;
        out->peak[0] = pk[0]; out->peak[1] = pk[1];
    }
    cf.counter[k] = 0;
}

__global__ void __launch_bounds__(BLOCK) abg_input_meter_kernel(const InmArgs a) {
    __shared__ __align__(16) Smem sm;
    const InmCfg cf = a.cfg[blockIdx.y];
    const InmRun rn = a.run[blockIdx.y];
    const int item = blockIdx.x;
    if (item >= rn.n_batches * cf.n_chunks) return;
    const int k = item / cf.n_chunks, c = item % cf.n_chunks;
    switch (cf.sfmt) {
        case ABG_SFMT_U8: meter_item<ABG_SFMT_U8>(a, cf, rn, k, c, sm); break;
        case ABG_SFMT_S8: meter_item<ABG_SFMT_S8>(a, cf, rn, k, c, sm); break;
        case ABG_SFMT_S16: meter_item<ABG_SFMT_S16>(a, cf, rn, k, c, sm); break;
        default: meter_item<ABG_SFMT_F32>(a, cf, rn, k, c, sm); break;
    }
}

}  // namespace

int abg_input_meter_chunks(int batch_bytes) { return (batch_bytes + CHUNK - 1) / CHUNK; }

cudaError_t abg_launch_input_meter(const InmArgs& a, int n_devices, int max_items, cudaStream_t s) {
    if (n_devices < 1 || max_items < 1) return cudaSuccess;
    abg_input_meter_kernel<<<dim3(max_items, n_devices, 1), BLOCK, 0, s>>>(a);
    return cudaGetLastError();
}
