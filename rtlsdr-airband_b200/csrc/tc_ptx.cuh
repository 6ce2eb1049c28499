// Inline-PTX building blocks of the tensor-core K1 (k1_tc.cu) for sm_90a: mbarrier, cp.async / bulk copies, and the
// warpgroup MMA (wgmma.mma_async, 8-bit integer operands from shared memory, S32 accumulators in registers).
//
// Descriptor encoding follows the PTX ISA "Matrix Descriptor Format" table of the warpgroup MMA:
//   shared-memory descriptor (64 bit): [0,14) start address >> 4 | [16,30) leading byte offset >> 4 |
//       [32,46) stride byte offset >> 4 | [49,52) base offset | [62,64) swizzle mode (0 = none)
//   K-major operand without swizzle ("interleaved" canonical layout): 8 rows x 16 bytes form one 128-byte core
//   matrix; LBO = byte distance between the two 16-byte K chunks of one MMA (K = 32 bytes for 8-bit types),
//   SBO = byte distance between consecutive 8-row groups along M (or N).  8-bit operands must be K-major.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// one lane of a fully converged warp (the others get 0)
__device__ __forceinline__ uint32_t elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(pred)
        :
        : "memory");
    return pred;
}

// ---- mbarrier -------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// arrive only where `pred` holds, without a branch around it (keeps warp-uniform code between asynchronous MMAs)
__device__ __forceinline__ void mbar_arrive_if(uint32_t bar, bool pred) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %1, 0;\n\t@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}" ::"r"(bar), "r"((uint32_t)pred) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    return done != 0;
}
// non-blocking probe of a phase (test_wait never suspends the warp)
__device__ __forceinline__ bool mbar_test(uint32_t bar, uint32_t parity) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    return done != 0;
}
// Bounded wait: a barrier that never completes (a protocol bug) must not hang the GPU.  Returns false on time-out.
__device__ __forceinline__ bool mbar_wait(uint32_t bar, uint32_t parity, long long budget_cycles = (1ll << 31)) {
    if (mbar_try_wait(bar, parity)) return true;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > budget_cycles) return false;
    }
    return true;
}

// Spin inside ONE asm statement (so the compiler sees straight-line, warp-uniform code around it and keeps the role loops
// on the uniform datapath), bounded: a barrier that never completes is a protocol bug and must not hang the GPU, so after
// ~10^6 failed try_waits (each suspends up to the hardware's time limit) the kernel traps and the launch fails cleanly.
__device__ __forceinline__ void mbar_wait_spin(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t.reg .u32 n;\n\t"
        "mov.u32 n, 0;\n"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "add.u32 n, n, 1;\n\t"
        "setp.lt.u32 p, n, 0x100000;\n\t"
        "@p bra WAIT_LOOP;\n\t"
        "trap;\n"
        "WAIT_DONE:\n\t}"
        :
        : "r"(bar), "r"(parity)
        : "memory");
}

// Same contract, polling with the non-blocking test_wait: lower wake-up latency than the suspending try_wait, at the price
// of issue slots (use on the single-warp critical path of a pipeline only).
__device__ __forceinline__ void mbar_wait_poll(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t.reg .u32 n;\n\t"
        "mov.u32 n, 0;\n"
        "POLL_LOOP:\n\t"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra POLL_DONE;\n\t"
        "add.u32 n, n, 1;\n\t"
        "setp.lt.u32 p, n, 0x4000000;\n\t"
        "@p bra POLL_LOOP;\n\t"
        "trap;\n"
        "POLL_DONE:\n\t}"
        :
        : "r"(bar), "r"(parity)
        : "memory");
}

// ---- copies ---------------------------------------------------------------------------------------------------------
// 16-byte asynchronous copy global -> shared (LDGSTS), L2 only
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
// arrive on `bar` once every cp.async this thread issued so far has landed (the barrier's count includes this arrival)
__device__ __forceinline__ void cp_async_arrive_noinc(uint32_t bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
// generic-proxy writes (st.shared, cp.async) -> visible to the async proxy (wgmma operand reads, bulk copies)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// TMA bulk copy global -> shared, completion counted in bytes on an mbarrier
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes),
                 "r"(bar)
                 : "memory");
}

// ---- wgmma ----------------------------------------------------------------------------------------------------------
__host__ __device__ constexpr uint64_t smem_desc_noswizzle(uint32_t addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((addr >> 4) & 0x3FFFu) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32);
}
// accumulator registers may be written by wgmma.mma_async only after this (every warp of the warpgroup)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// wait until at most n (warp-uniform; 7 when larger) of the most recent groups are in flight
__device__ __forceinline__ void wgmma_wait_groups(int n) {
    switch (n) {
        case 0: wgmma_wait<0>(); break;
        case 1: wgmma_wait<1>(); break;
        case 2: wgmma_wait<2>(); break;
        case 3: wgmma_wait<3>(); break;
        case 4: wgmma_wait<4>(); break;
        case 5: wgmma_wait<5>(); break;
        case 6: wgmma_wait<6>(); break;
        default: wgmma_wait<7>(); break;
    }
}
// keeps the compiler from moving accesses of an accumulator register across the asynchronous MMAs that own it
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(uint32_t (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+r"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 32] * B[N x 32]^T for one warpgroup, both operands K-major in shared memory, A unsigned (S8 =
// false) or signed 8-bit, B signed 8-bit, S32 accumulators: thread t of the warpgroup holds d[4j + 2h + e] =
// D[16 (t / 32) + (t % 32) / 4 + 8h][8j + 2 (t % 4) + e].  acc == 0 overwrites D.
template <int N, bool S8>
struct WgmmaI8;
// accumulator operand lists, 8 registers at a time, and the matching register strings, 16 at a time
#define ABG_D8(i) "+r"(d[i]), "+r"(d[i + 1]), "+r"(d[i + 2]), "+r"(d[i + 3]), "+r"(d[i + 4]), "+r"(d[i + 5]), "+r"(d[i + 6]), "+r"(d[i + 7])
#define ABG_D16 ABG_D8(0), ABG_D8(8)
#define ABG_S16 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
#define ABG_D32 ABG_D16, ABG_D8(16), ABG_D8(24)
#define ABG_S32 ABG_S16 ", %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define ABG_D48 ABG_D32, ABG_D8(32), ABG_D8(40)
#define ABG_S48 ABG_S32 ", %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"
#define ABG_D64 ABG_D48, ABG_D8(48), ABG_D8(56)
#define ABG_S64 ABG_S48 ", %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define ABG_D80 ABG_D64, ABG_D8(64), ABG_D8(72)
#define ABG_S80 ABG_S64 ", %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79"
#define ABG_D96 ABG_D80, ABG_D8(80), ABG_D8(88)
#define ABG_S96 ABG_S80 ", %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
#define ABG_D112 ABG_D96, ABG_D8(96), ABG_D8(104)
#define ABG_S112 ABG_S96 ", %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111"
#define ABG_D128 ABG_D112, ABG_D8(112), ABG_D8(120)
#define ABG_S128 ABG_S112 ", %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
#define ABG_WGMMA_I8(N, R, P, A, B, S8, AT) \
    template <> \
    struct WgmmaI8<N, S8> { \
        static __device__ __forceinline__ void mma(uint32_t (&d)[R], uint64_t a, uint64_t b, uint32_t acc) { \
            asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " P ", 0;\n\t" \
                         "wgmma.mma_async.sync.aligned.m64n" #N "k32.s32." AT ".s8 {" ABG_S##R "}, " A ", " B ", p;\n\t}" \
                         : ABG_D##R \
                         : "l"(a), "l"(b), "r"(acc)); \
        } \
    };
#define ABG_WGMMA_I8_BOTH(N, R, P, A, B) ABG_WGMMA_I8(N, R, P, A, B, false, "u8") ABG_WGMMA_I8(N, R, P, A, B, true, "s8")
ABG_WGMMA_I8_BOTH(32, 16, "%18", "%16", "%17")
ABG_WGMMA_I8_BOTH(64, 32, "%34", "%32", "%33")
ABG_WGMMA_I8_BOTH(96, 48, "%50", "%48", "%49")
ABG_WGMMA_I8_BOTH(128, 64, "%66", "%64", "%65")
ABG_WGMMA_I8_BOTH(160, 80, "%82", "%80", "%81")
ABG_WGMMA_I8_BOTH(192, 96, "%98", "%96", "%97")
ABG_WGMMA_I8_BOTH(224, 112, "%114", "%112", "%113")
ABG_WGMMA_I8_BOTH(256, 128, "%130", "%128", "%129")
#undef ABG_WGMMA_I8_BOTH
#undef ABG_WGMMA_I8

}  // namespace tc
