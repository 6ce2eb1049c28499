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
// The raw tile is stored in shared memory "transposed by 16-byte chunk": column j (of hop_bytes/16) holds bytes
// [16j, 16j+16) of every hop-row r at AT[j][r], rows 16 bytes apart.  That IS the canonical K-major no-swizzle operand
// layout (core matrix = 8 rows x 16 bytes), and the rows of frame f+q are the rows of frame f shifted by q*16 bytes, so
// the MMA for K bytes [q*hop_bytes + 16j, +32) simply takes descriptor start address AT + j*S + q*16: every raw byte is
// fetched from HBM once and written to shared memory once, and the tensor core reads it for each of the ~N/hop frames
// containing it.
//
// One CTA per SM, persistent, dynamic tile queue (tile = 128 consecutive frames of one device), warp-specialised:
//   warps 0-2   A producers: cp.async (LDGSTS) 16-byte chunks global -> transposed tile, double-buffered
//   warp 3      tile scheduler (atomic counter) + B loader: the device's coefficient table streams through a ring of
//               bulk-copy (TMA) stages, one pass per tile, out of L2
//   warps 4-7   consumer warpgroup 0, frames 0-63 of the tile; warps 8-11 consumer warpgroup 1, frames 64-127: each
//               issues one m64nNCk32 wgmma per 32 bytes of K into its register accumulators, then runs the epilogue on
//               them (digits recombined in int64, one double multiply, |X| with the reference's rounding,
//               rtl_airband.cpp:484) while the producers fill the other A buffer
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
constexpr int TC_MAX_BSTAGES = 16;
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
    int K, hop_bytes, HC, S, NC, ND, C2p, KBS, NSTB, a_signed;
    int mul, off;
    uint16_t aoff[512];        // per k-step start-address offset of the A operand, 16-byte units (K <= 16384)
    int stage_in_row;          // every B stage's k-steps lie inside one hop-row (HC/2 is a multiple of KBS)
    long long* trace;          // measurement aid (ABG_K1_TC_TRACE): clock64 stamps [cta][role 0..3][tile 0..15][event 0..3], or null
    int dbg_skip;              // measurement aid (ABG_K1_TC_SKIP): 1 = do not copy coefficients, 2 = do not copy samples, 4 = issue no MMA (results invalid)
    int rotate;                // start every CTA's K loop at a different coefficient block (exact integer sums commute)
};

struct Ctrl {
    unsigned long long full_a[2], empty_a[2];
    unsigned long long full_b[TC_MAX_BSTAGES], empty_b[TC_MAX_BSTAGES];
    unsigned long long info_full[TC_INFO_SLOTS], info_empty[TC_INFO_SLOTS];
    TileInfo info[TC_INFO_SLOTS];
};
static_assert(sizeof(Ctrl) <= TC_CTRL_BYTES, "control block too large");

// Every wait below is mbar_wait_spin: bounded inside one asm statement, traps instead of hanging (tc_ptx.cuh).
// ND digits of C2P outputs each: NCOL = the MMA's N (the plan's NC), NCOL / 2 accumulator registers per consumer thread.
template <int ND, int C2P>
__global__ void __launch_bounds__(TC_THREADS, 1) k1_tc_kernel(const TcArgs a) {
    constexpr int NCOL = (ND * C2P + 31) & ~31;
    extern __shared__ __align__(1024) unsigned char smem[];
    Ctrl* c = reinterpret_cast<Ctrl*>(smem);
    unsigned char* abuf = smem + TC_CTRL_BYTES;
    const int abuf_bytes = a.HC * a.S;
    unsigned char* bring = smem + TC_CTRL_BYTES + ((2 * abuf_bytes + 127) & ~127);
    const int stage_bytes = a.KBS * NCOL * 32;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    if (tid == 0) {
        for (int i = 0; i < 2; i++) {
            mbar_init(smem_u32(&c->full_a[i]), TC_A_THREADS);
            mbar_init(smem_u32(&c->empty_a[i]), TC_CONSUMER_WARPS);
        }
        for (int i = 0; i < TC_MAX_BSTAGES; i++) {
            mbar_init(smem_u32(&c->full_b[i]), 1);
            mbar_init(smem_u32(&c->empty_b[i]), TC_CONSUMER_WARPS);
        }
        for (int i = 0; i < TC_INFO_SLOTS; i++) {
            mbar_init(smem_u32(&c->info_full[i]), 1);
            mbar_init(smem_u32(&c->info_empty[i]), TC_CONSUMER_WARPS);
        }
        fence_mbar_init();
    }
    __syncthreads();
    const int NKB = (a.K / 32) / a.KBS;  // B stages per tile
    // All CTAs stream the same (or a few) coefficient tables out of L2 at the same pace: starting each CTA at a different
    // block spreads the requests over the L2 slices (exact integer sums commute, so the K order is free).
    const int kb_rot = a.rotate ? (int)((blockIdx.x * 2654435761u >> 8) % (unsigned)NKB) : 0;

// stage-level stamps of tile 3: event e of stage st (< 16) goes to slot 32 + 2*st + e of the role's 64-slot block (tiles 8..15 unused then)
#define TC_TRACE_STAGE(role, it, st, e)                                                                          \
    do {                                                                                                         \
        if (a.trace && (it) == 3 && (st) < 16 && (threadIdx.x & 31) == 0) a.trace[((size_t)blockIdx.x * 4 + (role)) * 64 + 32 + 2 * (st) + (e)] = clock64(); \
    } while (0)
#define TC_TRACE(role, it, ev)                                                                                   \
    do {                                                                                                         \
        if (a.trace && (it) < 8 && (threadIdx.x & 31) == 0) a.trace[(((size_t)blockIdx.x * 4 + (role)) * 16 + (it)) * 4 + (ev)] = clock64(); \
    } while (0)
    if (warp < 3) {
        // ================= A producers =================
        for (int it = 0;; ++it) {
            const int slot = it & (TC_INFO_SLOTS - 1);
            mbar_wait_spin(smem_u32(&c->info_full[slot]), (it / TC_INFO_SLOTS) & 1);
            const TileInfo ti = c->info[slot];
            if (ti.nf <= 0) break;
            const int buf = it & 1;
            if (warp == 0) TC_TRACE(0, it, 0);
            mbar_wait_spin(smem_u32(&c->empty_a[buf]), ((it >> 1) & 1) ^ 1);
            if (warp == 0) TC_TRACE(0, it, 1);
            const uint32_t dst0 = smem_u32(abuf + buf * abuf_bytes);
            const int total_chunks = ((ti.nf - 1) * a.hop_bytes + a.K) >> 4;
            int r = tid / a.HC, j = tid - r * a.HC;
            const int dr = TC_A_THREADS / a.HC, dj = TC_A_THREADS - dr * a.HC;
            for (int i = tid; i < total_chunks; i += TC_A_THREADS) {
                if (!(a.dbg_skip & 2)) cp_async16(dst0 + j * a.S + r * 16, ti.src + (size_t)i * 16);
                r += dr;
                j += dj;
                if (j >= a.HC) {
                    j -= a.HC;
                    r++;
                }
            }
            if (warp == 0) TC_TRACE(0, it, 2);
            cp_async_wait_all();
            fence_proxy_async();
            mbar_arrive(smem_u32(&c->full_a[buf]));
            if (warp == 0) TC_TRACE(0, it, 3);
        }
    } else if (warp == 3) {
        // ================= tile scheduler + B loader (whole warp in lock-step, one elected lane issues the copies) =================
        const uint32_t leader = elect_one();
        const size_t tab_bytes = (size_t)a.K * NCOL;
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
        const uint32_t fb_bar0 = smem_u32(&c->full_b[0]), eb_bar0 = smem_u32(&c->empty_b[0]);
        uint32_t fb_bar = fb_bar0, eb_bar = eb_bar0, dst = smem_u32(bring);
        int tab = lane == 0 ? publish(0) : 0;
        tab = __shfl_sync(0xffffffffu, tab, 0);
        for (int it = 0; tab >= 0; ++it) {
            int next_tab = lane == 0 ? publish(it + 1) : 0;  // the A producers start on tile it+1 while tile it's coefficients stream
            next_tab = __shfl_sync(0xffffffffu, next_tab, 0);
            const signed char* src = a.btab + (size_t)tab * tab_bytes;
            TC_TRACE(2, it, 0);
            int kb = kb_rot;
            for (int kbi = 0; kbi < NKB; kbi++) {
                mbar_wait_spin(eb_bar, ph ^ 1);
                TC_TRACE_STAGE(2, it, kbi, 0);
                if (leader) {
                    if (a.dbg_skip & 1) {
                        mbar_arrive(fb_bar);
                    } else {
                        mbar_arrive_expect_tx(fb_bar, (uint32_t)stage_bytes);
                        bulk_g2s(dst, src + (size_t)kb * stage_bytes, (uint32_t)stage_bytes, fb_bar);
                    }
                }
                TC_TRACE_STAGE(2, it, kbi, 1);
                if (++kb == NKB) kb = 0;
                dst += (uint32_t)stage_bytes;
                fb_bar += 8;
                eb_bar += 8;
                if (++stg == (uint32_t)a.NSTB) stg = 0, ph ^= 1, dst = smem_u32(bring), fb_bar = fb_bar0, eb_bar = eb_bar0;
            }
            TC_TRACE(2, it, 1);
            tab = next_tab;
        }
    } else if (warp >= 4) {
        // ================= consumers: MMA + epilogue, one warpgroup per 64 frames of the tile =================
        const int wg = (warp - 4) >> 2;
        const int wq = warp & 3;
        uint32_t acc[NCOL / 2];
        const uint32_t a_signed = (uint32_t)a.a_signed;
        const bool issue = !(a.dbg_skip & 4);
        // descriptor words that never change: LBO in bits [16,30) of the low word, SBO in the high word
        const uint64_t adesc0 = smem_desc_noswizzle(0, (uint32_t)a.S, 128u), bdesc0 = smem_desc_noswizzle(0, (uint32_t)NCOL * 16u, 128u);
        const uint32_t a_hi = (uint32_t)(adesc0 >> 32), b_hi = (uint32_t)(bdesc0 >> 32);
        const uint32_t bstep16 = (uint32_t)(NCOL * 32) >> 4, stage16 = (uint32_t)stage_bytes >> 4;
        const uint32_t b_lo_ring = (uint32_t)bdesc0 + (smem_u32(bring) >> 4);
        uint32_t b_lo = b_lo_ring;
        const uint32_t fb_bar0 = smem_u32(&c->full_b[0]), eb_bar0 = smem_u32(&c->empty_b[0]);
        uint32_t fb_bar = fb_bar0, eb_bar = eb_bar0, prev_eb = 0;
        uint32_t stg = 0, ph = 0;
        const uint32_t a_step = 2u * ((uint32_t)a.S >> 4);
        const int spr_ks = a.HC / 2;       // k-steps per hop-row
        const int spr = spr_ks / a.KBS;    // stages per hop-row (exact when a.stage_in_row)
        auto mma = [&](uint32_t a_lo, uint32_t b_lo_, uint32_t accumulate) {
            if (issue)
                WgmmaI8<NCOL>::mma(acc, ((uint64_t)a_hi << 32) | a_lo, ((uint64_t)b_hi << 32) | b_lo_, accumulate, a_signed);
        };
        for (int it = 0;; ++it) {
            const int slot = it & (TC_INFO_SLOTS - 1);
            mbar_wait_spin(smem_u32(&c->info_full[slot]), (it / TC_INFO_SLOTS) & 1);
            const TileInfo ti = c->info[slot];
            if (ti.nf <= 0) break;
            const int buf = it & 1;
            if (warp == 4) TC_TRACE(3, it, 0);
            mbar_wait_spin(smem_u32(&c->full_a[buf]), (it >> 1) & 1);
            if (warp == 4) TC_TRACE(3, it, 1);
            // this warpgroup's 64 frames start 64 hop-rows (64 x 16 bytes) into the tile
            const uint32_t a_lo = (uint32_t)adesc0 + (smem_u32(abuf + buf * abuf_bytes) >> 4) + (uint32_t)(wg * 64);
            // Stage `kb` of the frame covers k-steps [kb*KBS, kb*KBS + KBS).  When every stage lies inside one hop-row
            // (a.stage_in_row) its A start offsets are base + ks * a_step with base following a two-level counter (columns
            // inside the row, then the next row): pure uniform arithmetic, nothing loaded per stage.
            int kb = kb_rot;
            uint32_t base = a_lo + a.aoff[kb_rot * a.KBS];
            int in_row = (kb_rot * a.KBS) % spr_ks / a.KBS;  // stage index inside its hop-row
            wgmma_fence_regs(acc);
            for (int kbi = 0; kbi < NKB; kbi++) {
                mbar_wait_spin(fb_bar, ph);
                if (warp == 4) TC_TRACE_STAGE(3, it, kbi, 0);
                wgmma_fence();
                if (a.stage_in_row) {
                    for (int ks = 0; ks < a.KBS; ks++) mma(base + ks * a_step, b_lo + ks * bstep16, (kbi | ks) ? 1u : 0u);
                } else {
                    for (int ks = 0; ks < a.KBS; ks++) mma(a_lo + a.aoff[kb * a.KBS + ks], b_lo + ks * bstep16, (kbi | ks) ? 1u : 0u);
                }
                wgmma_commit();
                // the stage before this one is no longer read once at most one group (this stage's) is in flight
                wgmma_wait<1>();
                if (kbi > 0 && lane == 0) mbar_arrive(prev_eb);
                prev_eb = eb_bar;
                if (warp == 4) TC_TRACE_STAGE(3, it, kbi, 1);
                // next stage of the frame (wrapping around to its start)
                if (++kb == NKB) {
                    kb = 0;
                    base = a_lo + a.aoff[0];
                    in_row = 0;
                } else if (++in_row == spr) {
                    in_row = 0;
                    base = base - (uint32_t)(spr - 1) * a.KBS * a_step + 1u;  // first column of the next hop-row (rows are 16 bytes apart)
                } else {
                    base += a.KBS * a_step;
                }
                b_lo += stage16;
                fb_bar += 8;
                eb_bar += 8;
                if (++stg == (uint32_t)a.NSTB) stg = 0, ph ^= 1, b_lo = b_lo_ring, fb_bar = fb_bar0, eb_bar = eb_bar0;
            }
            wgmma_wait<0>();
            wgmma_fence_regs(acc);
            if (lane == 0) {
                mbar_arrive(prev_eb);
                mbar_arrive(smem_u32(&c->empty_a[buf]));
            }
            if (warp == 4) TC_TRACE(1, it, 1);
            // epilogue: this thread holds columns 8j + 2 (lane % 4) + {0, 1} of frames r0 and r0 + 8, i.e. the real and
            // imaginary part of channel 4 jb + lane % 4 for every group jb of eight outputs, all ND digits of each
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
                    const float xr = (float)((double)(a.mul * v[0] - a.off * sq_re) * a.cscale);
                    const float xi = (float)((double)(a.mul * v[1] - a.off * sq_im) * a.cscale);
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

template <int ND, int C2P>
cudaError_t tc_launch_one(const TcArgs& args, int grid, size_t smem, cudaStream_t s) {
    auto kern = k1_tc_kernel<ND, C2P>;
    static AbgPerDeviceSize configured;  // per instantiation, per CUDA device
    cudaError_t e = configured.ensure(smem, [&]() {
        cudaError_t e2 = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e2 != cudaSuccess) return e2;
        cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        return cudaSuccess;
    });
    if (e != cudaSuccess) return e;
    kern<<<grid, TC_THREADS, smem, s>>>(args);
    return cudaGetLastError();
}
template <int ND>
cudaError_t tc_launch_nd(const TcArgs& args, int grid, size_t smem, cudaStream_t s) {
    switch (args.C2p) {
        case 8: return tc_launch_one<ND, 8>(args, grid, smem, s);
        case 16: return tc_launch_one<ND, 16>(args, grid, smem, s);
        case 24: return tc_launch_one<ND, 24>(args, grid, smem, s);
        case 32: return tc_launch_one<ND, 32>(args, grid, smem, s);
        case 40: return tc_launch_one<ND, 40>(args, grid, smem, s);
        case 48: return tc_launch_one<ND, 48>(args, grid, smem, s);
        case 56: return tc_launch_one<ND, 56>(args, grid, smem, s);
        case 64: return tc_launch_one<ND, 64>(args, grid, smem, s);
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
    int stage_target = 8192;
    if (const char* ev = getenv("ABG_K1_TC_STAGE_BYTES")) stage_target = std::max(1024, atoi(ev));
    if (K > 16384) return 0;
    int KBS = 1;
    while (KBS < 8 && KBS * 2 * NC * 32 <= stage_target) KBS <<= 1;  // power of two: divides K/32
    const int stage = KBS * NC * 32;
    const size_t base = TC_CTRL_BYTES + (((size_t)2 * HC * S + 127) & ~(size_t)127);
    size_t cap = 200 * 1024;                                     // leaves room for K2's one-warp CTAs on the same SM (measured: best pipelined step)
    if (const char* ev = getenv("ABG_K1_TC_CAP_KB")) cap = std::min<size_t>(227, std::max(64, atoi(ev))) * 1024;
    int max_stages = TC_MAX_BSTAGES;
    if (const char* ev = getenv("ABG_K1_TC_STAGES")) max_stages = std::min(TC_MAX_BSTAGES, std::max(2, atoi(ev)));
    const size_t hard_cap = 227 * 1024;
    int nstb = (int)std::min<size_t>(max_stages, base < cap ? (cap - base) / stage : 0);
    if (nstb < 2) nstb = (int)std::min<size_t>(max_stages, base < hard_cap ? (hard_cap - base) / stage : 0);
    if (nstb < 2) return 0;
    p->eligible = 1; p->K = K; p->HC = HC; p->S = S; p->NC = NC; p->ND = digits; p->C2p = C2p; p->KBS = KBS; p->NSTB = nstb;
    p->acc_regs = NC / 2;  // S32 accumulators per consumer thread (m64nNC fragment)
    p->consumer_warpgroups = 2;
    p->smem_bytes = (int)(base + (size_t)nstb * stage); p->halo = halo;
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
    a.K = p.K; a.hop_bytes = p.HC * 16; a.HC = p.HC; a.S = p.S; a.NC = p.NC; a.ND = p.ND; a.C2p = p.C2p; a.KBS = p.KBS; a.NSTB = p.NSTB;
    a.a_signed = (L.sfmt == ABG_SFMT_S8) ? 1 : 0;
    a.mul = a.a_signed ? 1 : 2;
    a.off = a.a_signed ? 0 : 255;
    a.rotate = 1;
    a.dbg_skip = 0;
    if (const char* ev = getenv("ABG_K1_TC_SKIP")) a.dbg_skip = atoi(ev);
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
    a.stage_in_row = ((p.HC / 2) % p.KBS == 0) ? 1 : 0;
    for (int ks = 0; ks < p.K / 32; ks++) {
        // K bytes [32ks, 32ks+32) of a frame are the two 16-byte columns j, j+1 of hop-row q
        const int k0 = ks * 32, q = k0 / a.hop_bytes, j = (k0 - q * a.hop_bytes) >> 4;
        a.aoff[ks] = (uint16_t)(j * (p.S >> 4) + q);
    }
    if (const char* ev = getenv("ABG_K1_TC_ROTATE")) a.rotate = atoi(ev) != 0;
    if (a.total_tiles <= 0) return cudaSuccess;
    const int grid = std::min(a.total_tiles, std::max(sm_count, 1));
    if (p.ND == 3) return tc_launch_nd<3>(a, grid, (size_t)p.smem_bytes, s);
    if (p.ND == 4) return tc_launch_nd<4>(a, grid, (size_t)p.smem_bytes, s);
    return cudaErrorInvalidValue;
}
