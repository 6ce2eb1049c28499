// K1 (tensor-core) — sample conversion + window + DFT of the configured bins as ONE integer GEMM on the Hopper tensor
// cores (wgmma.mma_async, 8-bit operands, S32 accumulators in registers), sm_90a.  Same inputs, same outputs as
// k1_pruned.cu / k1_fft.cu; replaces the same reference code (reference src/rtl_airband.cpp:402-455 convert+window, :460
// fftwf_execute, :483-489 bin extraction) for 8-bit sample formats (U8 / S8: RTL-SDR, file input).
//
// The reference transforms N points per frame and reads C bins.  Written out for one bin b of frame f,
//     X[f,b] = sum_n  level(raw[f*hop + n]) * window[n] * W_N^(n*b)            (level(u) = (u - 127.5)/127.5 for U8)
// is a dense contraction  [frames x 2N raw BYTES] x [2N x 2C coefficients]: the A operand is the device's raw byte
// stream itself (8-bit integers are exact tensor-core operands: no conversion instruction is ever executed), the B operand
// is window*twiddle quantised to ND signed 8-bit digits (ND = 4: 30-bit fixed point, |error| <= 2^-31 of the largest
// coefficient, below the FP32 FFT's own rounding), accumulated EXACTLY in S32 and recombined in the epilogue:
//     X = (Gmax / 2Q) * (2 * sum_d 256^(ND-1-d) * acc_d  -  255 * sum_k q_k)        (the -127.5 offset, folded out)
//
// Sliding windows without data movement: consecutive frames start hop_bytes apart (84 % overlap at N = 2048, hop 320).
// Column j (of hop_bytes/16) of a tile holds bytes [16j, 16j+16) of every hop-row r, rows 16 bytes apart.  That IS the
// canonical K-major no-swizzle operand layout (core matrix = 8 rows x 16 bytes), and the rows of frame f+q are the rows of
// frame f shifted by q*16 bytes, so the MMA for K bytes [q*hop_bytes + 32p, +32) takes columns 2p, 2p+1 with descriptor
// start address q*16 into them: every raw byte is fetched from HBM once and the tensor core reads it for each of the
// ~N/hop frames containing it.
//
// K order: column pair major.  The k-steps of pair p are q = 0, 1, ... while 32p + q*hop_bytes < K (7 or 6 of them at
// N = 2048, hop 320; 2 or 1 at N = 512), and they read nothing but the two columns 2p, 2p+1.  So the shared memory holds
// no whole tile: one ring of stages, each = one column pair of the tile (A: 2 columns x S bytes) + the coefficients of its
// k-steps (B: up to KBS k-steps of NC x 32 bytes, bulk-copied per k-step from the table in its natural k order).  Where
// pairs have at most 2 k-steps, a stage holds up to pps consecutive pairs with the same k-step count instead (N = 512:
// 6 pairs, 12 k-steps), so that the fixed cost of a stage (barrier round trip, copies) is paid for enough MMAs.  The
// integer sums are exact, so the K order changes no result bit.  A stage is released as soon as its MMAs have read it,
// and the ring runs on across tile and device boundaries: the producers never wait for a whole tile to drain.
//
// One CTA per SM, persistent, dynamic tile queue (tile = 128 consecutive frames of one device), warp-specialised:
//   warps 0-2   A producers: cp.async (LDGSTS) 16-byte chunks global -> the stage's columns, completing on the
//               stage's full barrier by themselves (cp.async.mbarrier.arrive.noinc): never a wait for a copy
//   warp 3      tile scheduler (atomic counter) + B loader (bulk copies (TMA) of the stage's k-steps out of L2)
//   warps 4-7   consumer warpgroup 0, frames 0-63 of the tile; warps 8-11 consumer warpgroup 1, frames 64-127: per stage
//               one m64nNCk32 wgmma per k-step into the register accumulators, the whole stage left in flight;
//               then the epilogue on them (digits recombined in int64, one double multiply, |X| with the reference's
//               rounding, rtl_airband.cpp:484) while the producers run ahead into the next tile
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include <algorithm>

#include "../../include/airband_b200.h"
#include "abg_internal.h"
#include "tc_ptx.cuh"

namespace {
using namespace tc;
extern long long* g_tc_trace;

constexpr int TC_THREADS = 384;
constexpr int TC_A_THREADS = 96;     // warps 0-2
constexpr int TC_CONSUMER_WARPS = 8;  // warps 4-11
constexpr int TC_CTRL_BYTES = 1024;
constexpr int TC_MAX_STAGES = 32;
constexpr int TC_INFO_SLOTS = 4;

struct TileInfo {
    const unsigned char* src;  // first byte of the tile's first frame
    int nf;                    // valid frames (1..128); <= 0: end of work
    int pos;                   // row of win/iqin of the first frame
    int gbase;                 // first channel index
    int nch;                   // channels
    int tab;                   // coefficient table
    int pad;
};

struct TcArgs {
    const K1Dev* devs;
    const int32_t* tab_of_dev;
    const signed char* btab;
    const long long* sq;
    float* win;
    float2* iqin;
    int* counter;
    int32_t* status;
    double cscale;
    int Gp, n_devices, tiles_per_dev, total_tiles;
    int K, hop_bytes, S, npairs;   // npairs: column pairs that hold K bytes of a frame (min(HC/2, K/32))
    int KBS, NSTG, pps;            // k-steps per pair and stage at most, stages in the ring, column pairs per stage at most
    int a_bytes, stage_bytes;      // A part of a stage (2 pps columns, 128-byte aligned); whole stage
    long long* trace;              // measurement aid (ABG_K1_TC_TRACE): clock64 stamps [cta][role 0..3][tile 0..15][event 0..3], or null
};

struct Ctrl {
    unsigned long long full[TC_MAX_STAGES], empty[TC_MAX_STAGES];
    unsigned long long info_full[TC_INFO_SLOTS], info_empty[TC_INFO_SLOTS];
    TileInfo info[TC_INFO_SLOTS];
};
static_assert(sizeof(Ctrl) <= TC_CTRL_BYTES, "control block too large");

// The stages of one tile, in the order every role walks them: pairs p .. p+np-1 with their k-steps q0 .. q0+nq-1.  One
// pair per stage (pps == 1), its k-steps cut into pieces of at most KBS only when K >> hop_bytes; or, where every pair has
// at most 2 k-steps (pps > 1), up to pps consecutive pairs with the same k-step count nk(p) = ceil((K - 32p) / hop_bytes).
// MMA j of a stage is pair g = j >> sh, k-step q = j & mk (pair major, B stored in that order).
struct StageSeq {
    int p, np, q0, nq, nk, sh, mk;
    __device__ __forceinline__ void start(const TcArgs& a) {  // pair p begins a stage
        nk = (a.K - 32 * p + a.hop_bytes - 1) / a.hop_bytes;
        q0 = 0;
        nq = min(a.KBS, nk);
        // pairs from p on that still have nk k-steps: 32 p' + (nk - 1) * hop_bytes < K
        np = min(min(a.pps, a.npairs - p), ((a.K - (nk - 1) * a.hop_bytes + 31) >> 5) - p);
        sh = np > 1 ? nq - 1 : 31;
        mk = np > 1 ? nq - 1 : -1;
    }
    __device__ __forceinline__ void first(const TcArgs& a) {
        p = 0;
        start(a);
    }
    __device__ __forceinline__ bool next(const TcArgs& a) {  // false after the tile's last stage
        q0 += nq;
        if (q0 < nk) {
            nq = min(a.KBS, nk - q0);
            return true;
        }
        p += np;
        if (p >= a.npairs) return false;
        start(a);
        return true;
    }
};

// Every wait below is mbar_wait_spin: bounded inside one asm statement, traps instead of hanging (tc_ptx.cuh).
// ND digits of C2P outputs each: NCOL = the MMA's N (the plan's NC), NCOL / 2 accumulator registers per consumer thread;
// S8: signed samples (the A operand's type); GROUPED: stages of several pairs (pps > 1).
template <int ND, int C2P, bool S8, bool GROUPED>
__global__ void __launch_bounds__(TC_THREADS, 1) k1_tc_kernel(const TcArgs a) {
    constexpr int NCOL = (ND * C2P + 31) & ~31;
    constexpr int KSTEP_BYTES = NCOL * 32;  // B bytes of one k-step
    extern __shared__ __align__(1024) unsigned char smem[];
    Ctrl* c = reinterpret_cast<Ctrl*>(smem);
    const uint32_t ring = smem_u32(smem + TC_CTRL_BYTES);
    const uint32_t full0 = smem_u32(&c->full[0]), empty0 = smem_u32(&c->empty[0]);
    const int tid = threadIdx.x, lane = tid & 31;
    // warp-uniform as far as ptxas can tell: a role branch it cannot prove uniform makes it serialise the wgmma chain
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);

    if (tid == 0) {
        for (int i = 0; i < TC_MAX_STAGES; i++) {
            mbar_init(smem_u32(&c->full[i]), TC_A_THREADS + 1);  // every producer thread + the B loader's expect_tx
            mbar_init(smem_u32(&c->empty[i]), TC_CONSUMER_WARPS);
        }
        for (int i = 0; i < TC_INFO_SLOTS; i++) {
            mbar_init(smem_u32(&c->info_full[i]), 1);
            mbar_init(smem_u32(&c->info_empty[i]), TC_CONSUMER_WARPS);
        }
        fence_mbar_init();
    }
    __syncthreads();

// stage-level stamps of tile 3: event e of stage st (< 16) goes to slot 32 + 2*st + e of the role's 64-slot block (tiles 8..15 unused then);
// every lane of the warp stores the same stamp (a lane condition would put a divergent path between the consumers' MMAs)
#define TC_TRACE_STAGE(role, it, st, e)                                                                          \
    do {                                                                                                         \
        if (a.trace && (it) == 3 && (st) < 16) a.trace[((size_t)blockIdx.x * 4 + (role)) * 64 + 32 + 2 * (st) + (e)] = clock64(); \
    } while (0)
#define TC_TRACE(role, it, ev)                                                                                   \
    do {                                                                                                         \
        if (a.trace && (it) < 8 && (threadIdx.x & 31) == 0) a.trace[(((size_t)blockIdx.x * 4 + (role)) * 16 + (it)) * 4 + (ev)] = clock64(); \
    } while (0)
    if (warp < 3) {
        // ================= A producers =================
        // the stage's chunks in the order (block of 8 rows, column, row): a quarter warp writes 8 consecutive rows of one
        // column (conflict-free), a warp reads whole 32-byte sectors; thread t takes chunks t, t + 96, ...
        const int rr = tid & 7;
        uint32_t stg = 0, ph = 0;
        for (int it = 0;; ++it) {
            const int slot = it & (TC_INFO_SLOTS - 1);
            mbar_wait_spin(smem_u32(&c->info_full[slot]), (it / TC_INFO_SLOTS) & 1);
            const TileInfo ti = c->info[slot];
            if (ti.nf <= 0) break;
            if (warp == 0) TC_TRACE(0, it, 0);
            const int valid = (ti.nf - 1) * a.hop_bytes + a.K;  // bytes of the tile that exist in the device's buffer
            StageSeq u;
            u.first(a);
            do {
                mbar_wait_spin(empty0 + 8 * stg, ph ^ 1);
                const int first = u.q0 * a.hop_bytes + 32 * u.p;  // stage row 0 = hop-row q0 of the tile, column 0 = column 2p
                const unsigned char* src = ti.src + first;
                const int rem = valid - first, nrows = 127 + u.nq, ncol = 2 * u.np;
                const uint32_t dst = ring + stg * (uint32_t)a.stage_bytes;
                const int total = ((nrows + 7) >> 3) * 8 * ncol;
                for (int i = tid; i - tid < total; i += TC_A_THREADS) {  // warp-uniform: whole warps issue the copies
                    const int u8 = i >> 3, rb = u8 / ncol, c = u8 - rb * ncol, r = rb * 8 + rr, off = r * a.hop_bytes + 16 * c;
                    if (i < total && r < nrows && off < rem) cp_async16(dst + c * a.S + r * 16, src + off);
                }
                // the stage's full barrier gets this thread's arrival once its copies have landed: no wait here, so the
                // copies of as many stages as the ring has free stay in flight (the consumers make them visible to the
                // tensor core's proxy)
                cp_async_arrive_noinc(full0 + 8 * stg);
                if (++stg == (uint32_t)a.NSTG) stg = 0, ph ^= 1;
            } while (u.next(a));
            if (warp == 0) TC_TRACE(0, it, 3);
        }
    } else if (warp == 3) {
        // ================= tile scheduler + B loader (whole warp in lock-step, one elected lane issues the copies) =================
        const uint32_t leader = elect_one();
        const size_t tab_bytes = (size_t)a.K * NCOL;
        const int ks_per_row = a.hop_bytes / 32;  // k-step of (pair p, hop-row q) = q * ks_per_row + p
        auto publish = [&](int it) -> int {  // lane 0: claim the next tile and publish it in slot it % 4; returns its table, -1 = no more
            const int slot = it & (TC_INFO_SLOTS - 1);
            mbar_wait_spin(smem_u32(&c->info_empty[slot]), ((it / TC_INFO_SLOTS) & 1) ^ 1);
            TileInfo ti{};
            ti.nf = 0;
            ti.tab = -1;
            for (;;) {
                const int t = atomicAdd(a.counter, 1);
                if (t >= a.total_tiles) break;
                const int dev = t / a.tiles_per_dev, st = t - dev * a.tiles_per_dev;
                const K1Dev dv = a.devs[dev];
                const int f0 = st * 128;
                if (f0 >= dv.n_frames || dv.n_channels <= 0) continue;
                ti.src = dv.raw + dv.start_byte + (unsigned long long)f0 * dv.hop_bytes;
                ti.nf = min(128, dv.n_frames - f0);
                ti.pos = dv.pos0 + f0;
                ti.gbase = dv.g0;
                ti.nch = dv.n_channels;
                ti.tab = a.tab_of_dev[dev];
                break;
            }
            c->info[slot] = ti;
            mbar_arrive(smem_u32(&c->info_full[slot]));
            return ti.tab;
        };
        uint32_t stg = 0, ph = 0;
        int tab = lane == 0 ? publish(0) : 0;
        tab = __shfl_sync(0xffffffffu, tab, 0);
        for (int it = 0; tab >= 0; ++it) {
            int next_tab = lane == 0 ? publish(it + 1) : 0;  // the A producers start on tile it+1 while tile it's stages stream
            next_tab = __shfl_sync(0xffffffffu, next_tab, 0);
            const signed char* src = a.btab + (size_t)tab * tab_bytes;
            TC_TRACE(2, it, 0);
            StageSeq u;
            u.first(a);
            int st = 0;
            do {
                mbar_wait_spin(empty0 + 8 * stg, ph ^ 1);
                TC_TRACE_STAGE(2, it, st, 0);
                if (leader) {
                    // B block j = (pair g, k-step q) of the stage = table k-step (q0 + q) * ks_per_row + p + g
                    const uint32_t bar = full0 + 8 * stg, dst = ring + stg * (uint32_t)a.stage_bytes + (uint32_t)a.a_bytes;
                    mbar_arrive_expect_tx(bar, (uint32_t)(u.np * u.nq * KSTEP_BYTES));
                    for (int g = 0; g < u.np; g++)
                        for (int q = 0; q < u.nq; q++)
                            bulk_g2s(dst + (g * u.nq + q) * KSTEP_BYTES, src + (size_t)((u.q0 + q) * ks_per_row + u.p + g) * KSTEP_BYTES,
                                     (uint32_t)KSTEP_BYTES, bar);
                }
                TC_TRACE_STAGE(2, it, st, 1);
                st++;
                if (++stg == (uint32_t)a.NSTG) stg = 0, ph ^= 1;
            } while (u.next(a));
            TC_TRACE(2, it, 1);
            tab = next_tab;
        }
    } else if (warp >= 4) {
        // ================= consumers: MMA + epilogue, one warpgroup per 64 frames of the tile =================
        const int wg = (warp - 4) >> 2;
        const int wq = warp & 3;
        uint32_t acc[NCOL / 2];
        // descriptor words that never change: LBO in bits [16,30) of the low word, SBO in the high word.  A: the two
        // 16-byte K chunks are the stage's two columns (S apart); this warpgroup's 64 frames start 64 rows in.
        const uint64_t adesc0 = smem_desc_noswizzle(0, (uint32_t)a.S, 128u), bdesc0 = smem_desc_noswizzle(0, (uint32_t)NCOL * 16u, 128u);
        const uint64_t a_hi = adesc0 >> 32 << 32, b_hi = bdesc0 >> 32 << 32;
        const uint32_t a_lo0 = (uint32_t)adesc0 + (ring >> 4) + (uint32_t)(wg * 64);
        const uint32_t b_lo0 = (uint32_t)bdesc0 + ((ring + (uint32_t)a.a_bytes) >> 4);
        const uint32_t stage16 = (uint32_t)a.stage_bytes >> 4, pair16 = (uint32_t)a.S >> 3;
        uint32_t stg = 0, ph = 0, prev_empty = 0;
        for (int it = 0;; ++it) {
            const int slot = it & (TC_INFO_SLOTS - 1);
            mbar_wait_spin(smem_u32(&c->info_full[slot]), (it / TC_INFO_SLOTS) & 1);
            const TileInfo ti = c->info[slot];
            if (ti.nf <= 0) break;
            if (warp == 4) TC_TRACE(3, it, 0);
            StageSeq u;
            u.first(a);
            uint32_t accumulate = 0;  // the tile's first MMA overwrites the accumulators
            int st = 0;
            wgmma_fence_regs(acc);
            do {
                mbar_wait_spin(full0 + 8 * stg, ph);
                fence_proxy_async();  // the producers' cp.async writes (generic proxy) -> the wgmma operand reads (async proxy)
                if (warp == 4) TC_TRACE_STAGE(3, it, st, 0);
                // MMA j of the stage: pair g, k-step q = A rows q.. of the stage's columns 2g, 2g+1 (rows are 16 bytes apart),
                // B block j.  One commit group per MMA (the count is a run-time value; ptxas keeps a chain of groups in
                // flight across a run-time loop) and nothing but uniform address arithmetic between the MMAs: the chain runs
                // at the MMA latency, so every instruction in the loop shows in K1's time.
                const uint32_t a_lo = a_lo0 + stg * stage16, b_lo = b_lo0 + stg * stage16;
                const int n_mma = GROUPED ? u.np * u.nq : u.nq;
                for (int j = 0; j < n_mma; j++) {
                    const uint32_t a_off = GROUPED ? (uint32_t)(j >> u.sh) * pair16 + (uint32_t)(j & u.mk) : (uint32_t)j;
                    wgmma_fence_regs(acc);
                    wgmma_fence();
                    WgmmaI8<NCOL, S8>::mma(acc, a_hi | (a_lo + a_off), b_hi | (b_lo + j * (KSTEP_BYTES >> 4)), accumulate);
                    wgmma_commit();
                    wgmma_fence_regs(acc);
                    accumulate = 1;
                }
                // the stage before this one is no longer read once at most this stage's groups are in flight
                wgmma_wait_groups(n_mma);
                mbar_arrive_if(prev_empty, st > 0 && lane == 0);
                prev_empty = empty0 + 8 * stg;
                if (warp == 4) TC_TRACE_STAGE(3, it, st, 1);
                st++;
                if (++stg == (uint32_t)a.NSTG) stg = 0, ph ^= 1;
            } while (u.next(a));
            wgmma_wait<0>();
            wgmma_fence_regs(acc);
            if (lane == 0) mbar_arrive(prev_empty);
            if (warp == 4) TC_TRACE(1, it, 1);
            // epilogue: this thread holds columns 8j + 2 (lane % 4) + {0, 1} of frames r0 and r0 + 8, i.e. the real and
            // imaginary part of channel 4 jb + lane % 4 for every group jb of eight outputs, all ND digits of each
            constexpr long long MUL = S8 ? 1 : 2, OFF = S8 ? 0 : 255;
            const int r0 = wg * 64 + wq * 16 + (lane >> 2);
            const long long* sq = a.sq + (size_t)ti.tab * C2P;
#pragma unroll
            for (int jb = 0; jb < C2P / 8; jb++) {
                const int ch = 4 * jb + (lane & 3);
                const long long sq_re = __ldg(sq + 2 * ch), sq_im = __ldg(sq + 2 * ch + 1);
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    long long v[2];
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        v[e] = 0;
#pragma unroll
                        for (int d = 0; d < ND; d++) v[e] = (v[e] << 8) + (long long)(int32_t)acc[4 * (d * C2P / 8 + jb) + 2 * h + e];
                    }
                    const float xr = (float)((double)(MUL * v[0] - OFF * sq_re) * a.cscale);
                    const float xi = (float)((double)(MUL * v[1] - OFF * sq_im) * a.cscale);
                    const int row = r0 + 8 * h;
                    if (row < ti.nf && ch < ti.nch) {
                        const size_t o = (size_t)(ti.pos + row) * a.Gp + ti.gbase + ch;
                        a.win[o] = sqrtf(__fadd_rn(__fmul_rn(xr, xr), __fmul_rn(xi, xi)));  // rtl_airband.cpp:484
                        a.iqin[o] = make_float2(xr, xi);
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(smem_u32(&c->info_empty[slot]));
            if (warp == 4) TC_TRACE(1, it, 2);
        }
    }
}

template <int ND, int C2P, bool S8>
cudaError_t tc_launch_one(const TcArgs& args, int grid, size_t smem, cudaStream_t s) {
    auto kern = args.pps > 1 ? k1_tc_kernel<ND, C2P, S8, true> : k1_tc_kernel<ND, C2P, S8, false>;
    static AbgPerDeviceSize configured[2];  // per instantiation, per CUDA device
    cudaError_t e = configured[args.pps > 1].ensure(smem, [&]() {
        cudaError_t e2 = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e2 != cudaSuccess) return e2;
        cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        return cudaSuccess;
    });
    if (e != cudaSuccess) return e;
    kern<<<grid, TC_THREADS, smem, s>>>(args);
    return cudaGetLastError();
}
template <int ND, bool S8>
cudaError_t tc_launch_nd(const TcArgs& args, int C2p, int grid, size_t smem, cudaStream_t s) {
    switch (C2p) {
        case 8: return tc_launch_one<ND, 8, S8>(args, grid, smem, s);
        case 16: return tc_launch_one<ND, 16, S8>(args, grid, smem, s);
        case 24: return tc_launch_one<ND, 24, S8>(args, grid, smem, s);
        case 32: return tc_launch_one<ND, 32, S8>(args, grid, smem, s);
        case 40: return tc_launch_one<ND, 40, S8>(args, grid, smem, s);
        case 48: return tc_launch_one<ND, 48, S8>(args, grid, smem, s);
        case 56: return tc_launch_one<ND, 56, S8>(args, grid, smem, s);
        case 64: return tc_launch_one<ND, 64, S8>(args, grid, smem, s);
    }
    return cudaErrorInvalidValue;
}

long long* g_tc_trace = nullptr;
}  // namespace

// measurement aid: copy the clock64 stamps of the last traced launches (ABG_K1_TC_TRACE set) to the host; 256*4*16*4 values
int abg_k1tc_trace_dump(long long* out) {
    if (!g_tc_trace) return -1;
    cudaDeviceSynchronize();
    return cudaMemcpy(out, g_tc_trace, sizeof(long long) * 256 * 4 * 16 * 4, cudaMemcpyDeviceToHost) == cudaSuccess ? 0 : -1;
}

// Geometry of the tensor-core K1 for one launch group, or eligible == 0 when the group has to use the CUDA-core kernels.
// KBS = k-steps per ring stage at most (a column pair's, unless K >> hop_bytes), NSTB = stages in the ring.
int abg_k1tc_plan(int fft_size, int sfmt, int hop_bytes, int max_channels, int digits, K1TcPlan* p) {
    *p = K1TcPlan{};
    if (sfmt != ABG_SFMT_U8 && sfmt != ABG_SFMT_S8) return 0;  // 16/32-bit formats stay on the FP32 kernels
    if (hop_bytes % 32 != 0 || hop_bytes < 32) return 0;        // both 16-byte chunks of an MMA's K slice must lie in one hop-row
    if (digits != 3 && digits != 4) return 0;
    const int K = fft_size * 2;
    const int HC = hop_bytes / 16;
    const int halo = (K - 32) / hop_bytes;                      // extra hop-rows the last frame of a tile reaches into
    int rows = 128 + halo;
    if ((rows & 1) == 0) rows++;                                // odd 16-byte pitch: conflict-free transposed writes
    const int S = rows * 16;
    const int C2p = (2 * max_channels + 7) & ~7;
    const int NC = (digits * C2p + 31) & ~31;                   // the wgmma's N (a multiple of 32 keeps the instantiations few)
    if (NC > 256) return 0;
    if (K > 16384) return 0;
    const size_t kstep = (size_t)NC * 32;
    size_t cap = 200 * 1024;                                     // leaves room for K2's one-warp CTAs on the same SM (measured: best pipelined step)
    if (const char* ev = getenv("ABG_K1_TC_CAP_KB")) cap = std::min<size_t>(227, std::max(64, atoi(ev))) * 1024;
    int max_stages = TC_MAX_STAGES;
    if (const char* ev = getenv("ABG_K1_TC_STAGES")) max_stages = std::min(TC_MAX_STAGES, std::max(2, atoi(ev)));
    const size_t hard_cap = 227 * 1024;
    auto stage_bytes = [&](int pps, int kbs) { return (((size_t)2 * pps * S + 127) & ~(size_t)127) + (size_t)pps * kbs * kstep; };
    auto stages = [&](int pps, int kbs, size_t c) {
        return c > TC_CTRL_BYTES ? (int)std::min<size_t>(max_stages, (c - TC_CTRL_BYTES) / stage_bytes(pps, kbs)) : 0;
    };
    // A stage holds whole column pairs (pair 0 has the most k-steps: ceil(K / hop_bytes)).  Every stage costs a barrier round
    // trip, whatever its size, so where pairs have at most 2 k-steps they are grouped up to about 12 k-steps per stage (2
    // pairs per stage measured 10 % and 4 pairs 3 % below 6 on cfg5, N = 512); a
    // pair is cut only when whole pairs would leave fewer than 4 stages.
    const int kq = (K + hop_bytes - 1) / hop_bytes, npairs = std::min(HC / 2, K / 32);
    int pps = kq <= 2 ? std::max(1, std::min(12 / kq, npairs)) : 1, kbs = kq;
    while (pps > 1 && stages(pps, kbs, cap) < 4) pps--;
    while (kbs > 1 && stages(pps, kbs, cap) < 4) kbs = (kbs + 1) / 2;
    int nst = stages(pps, kbs, cap);
    if (nst < 2) nst = stages(pps, kbs, hard_cap);
    if (nst < 2) return 0;
    p->pps = pps;
    p->eligible = 1; p->K = K; p->HC = HC; p->S = S; p->NC = NC; p->ND = digits; p->C2p = C2p; p->KBS = kbs; p->NSTB = nst;
    p->acc_regs = NC / 2;  // S32 accumulators per consumer thread (m64nNC fragment)
    p->consumer_warpgroups = 2;
    p->smem_bytes = (int)(TC_CTRL_BYTES + (size_t)nst * stage_bytes(pps, kbs)); p->halo = halo;
    p->table_bytes = (size_t)K * NC;
    return 1;
}

// Coefficient table of one device for the plan: tab[K * NC] signed digits in the shared-memory image the MMA reads
// ([k-step][16-byte chunk][column][16 bytes]), sq[C2p] = sum over K of the quantised coefficient per output, and the scale
// that turns the recombined integer into the reference's float (returned through *cscale; identical for every table of
// the group).  wsc[n] = window[n] * 1/full-scale (reference src/rtl_airband.cpp:319-324,335-351).
void abg_k1tc_build_table(const K1TcPlan& p, int fft_size, int sfmt, const float* wsc, const int32_t* bins, int n_channels, signed char* tab,
                          long long* sq, double* cscale) {
    const int N = fft_size, K = p.K, NC = p.NC, ND = p.ND;
    double gmax = 0.0;
    for (int n = 0; n < N; n++) gmax = std::max(gmax, fabs((double)wsc[n]));
    if (gmax <= 0.0) gmax = 1.0;
    const double Q = ldexp(1.0, 8 * ND - 2);
    std::fill(tab, tab + (size_t)K * NC, (signed char)0);
    for (int o = 0; o < p.C2p; o++) sq[o] = 0;
    for (int c = 0; c < n_channels; c++) {
        const int b = bins[c] & (N - 1);
        for (int n = 0; n < N; n++) {
            const double th = 2.0 * M_PI * (double)(((long long)n * b) % N) / (double)N;
            const double w = (double)wsc[n], cs = cos(th) * w, sn = sin(th) * w;
            // (I + iQ) * w * (cos - i sin):  Re = I*cs + Q*sn,  Im = -I*sn + Q*cs
            const double coef[2][2] = {{cs, sn}, {-sn, cs}};  // [re/im output][I/Q input]
            for (int reim = 0; reim < 2; reim++)
                for (int comp = 0; comp < 2; comp++) {
                    const int o = 2 * c + reim;
                    const int kk = 2 * n + comp;
                    long long q = llround(coef[reim][comp] / gmax * Q);
                    sq[o] += q;
                    const int ks = kk >> 5, h = (kk >> 4) & 1, t = kk & 15;
                    for (int d = ND - 1; d >= 0; d--) {  // balanced base-256 digits, least significant first
                        long long dig = ((q + 128) & 255) - 128;
                        q = (q - dig) >> 8;
                        tab[((size_t)(ks * 2 + h) * NC + (size_t)(d * p.C2p + o)) * 16 + t] = (signed char)dig;
                    }
                }
        }
    }
    // U8: X = (gmax / 2Q) * (2v - 255 * sq);  S8: X = (gmax / Q) * v
    *cscale = (sfmt == ABG_SFMT_U8) ? gmax / (2.0 * Q) : gmax / Q;
}

cudaError_t abg_launch_k1_tc(const K1Launch& L, const K1TcPlan& p, const K1TcTables& T, int sm_count, cudaStream_t s) {
    TcArgs a{};
    a.devs = L.devs; a.tab_of_dev = T.tab_of_dev; a.btab = T.btab; a.sq = T.sq; a.win = L.win; a.iqin = L.iqin; a.counter = T.counter;
    a.status = T.status; a.cscale = T.cscale; a.Gp = L.Gp; a.n_devices = L.n_devices;
    a.tiles_per_dev = (L.max_frames + 127) / 128;
    a.total_tiles = a.tiles_per_dev * L.n_devices;
    a.K = p.K; a.hop_bytes = p.HC * 16; a.S = p.S; a.npairs = std::min(p.HC / 2, p.K / 32);
    a.KBS = p.KBS; a.NSTG = p.NSTB;
    a.pps = p.pps;
    a.a_bytes = (2 * p.pps * p.S + 127) & ~127;
    a.stage_bytes = a.a_bytes + p.pps * p.KBS * p.NC * 32;
    a.trace = nullptr;
    static long long* trace_buf = nullptr;  // measurement aid only: one process-wide buffer, dumped by abg_debug_k1tc_trace_dump()
    if (getenv("ABG_K1_TC_TRACE")) {
        if (!trace_buf) {
            cudaMalloc((void**)&trace_buf, sizeof(long long) * 256 * 4 * 16 * 4);
            cudaMemset(trace_buf, 0, sizeof(long long) * 256 * 4 * 16 * 4);
        }
        a.trace = trace_buf;
        g_tc_trace = trace_buf;
    }
    if (a.total_tiles <= 0) return cudaSuccess;
    const int grid = std::min(a.total_tiles, std::max(sm_count, 1));
    const bool s8 = L.sfmt == ABG_SFMT_S8;
    const size_t smem = (size_t)p.smem_bytes;
    if (p.ND == 3) return s8 ? tc_launch_nd<3, true>(a, p.C2p, grid, smem, s) : tc_launch_nd<3, false>(a, p.C2p, grid, smem, s);
    if (p.ND == 4) return s8 ? tc_launch_nd<4, true>(a, p.C2p, grid, smem, s) : tc_launch_nd<4, false>(a, p.C2p, grid, smem, s);
    return cudaErrorInvalidValue;
}
