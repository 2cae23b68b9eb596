// sm90_ptx.cuh -- thin inline-PTX wrappers for the Hopper (sm_90a) features the engine uses:
// mbarrier, TMA (cp.async.bulk[.tensor]) and warpgroup MMA (wgmma.mma_async, integer s8 x s8 -> s32).
// The descriptor bit layout follows the PTX ISA "wgmma matrix descriptor" table.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace bnm {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.b32 %0, 1, 0, P;\n\t}" : "=r"(pred));
    return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred P;\n\tmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\tselp.b32 %0, 1, 0, P;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// try_wait with a suspend-time hint (ns): the warp sleeps in hardware until the phase completes (or the hint
// expires) instead of re-issuing the probe -- waiting warps then cost no issue slots
__device__ __forceinline__ bool mbar_try_wait_hint(uint64_t *bar, uint32_t parity, uint32_t hint_ns) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred P;\n\tmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n\tselp.b32 %0, 1, 0, P;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity), "r"(hint_ns) : "memory");
    return ok != 0;
}
// Bounded wait: a wrong byte count / descriptor must not hang the GPU box.  On timeout the error word is
// set and the kernel traps (the host then reports a launch failure instead of spinning forever).
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity, int *err_flag = nullptr, int code = 1) {
    if (mbar_try_wait(bar, parity)) return;
    uint32_t spins = 0;
    while (!mbar_try_wait_hint(bar, parity, 20000u)) {
        if (++spins > (1u << 20)) {
            if (err_flag) *reinterpret_cast<volatile int *>(err_flag) = code;
            __threadfence_system();
            asm volatile("trap;");
        }
    }
}

// Long waits of a helper warp that shares its SM sub-partition with working warps (producer / issuer roles): every failed probe is
// followed by a sleep, so the waiting warp takes (almost) no issue slots from its neighbours.  Bounded like mbar_wait.
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t *bar, uint32_t parity, int *err_flag = nullptr, int code = 1, uint32_t sleep_ns = 400) {
    if (mbar_try_wait(bar, parity)) return;
    uint32_t spins = 0;
    while (!mbar_try_wait_hint(bar, parity, 20000u)) {
        __nanosleep(sleep_ns);
        if (++spins > (1u << 22)) {
            if (err_flag) *reinterpret_cast<volatile int *>(err_flag) = code;
            __threadfence_system();
            asm volatile("trap;");
        }
    }
}

// same, on a 32-bit shared-memory address held in a register (hot loops: no generic->shared conversion per call)
__device__ __forceinline__ bool mbar_try_wait_a(uint32_t bar_addr, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred P;\n\tmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\tselp.b32 %0, 1, 0, P;\n\t}"
                 : "=r"(ok) : "r"(bar_addr), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ bool mbar_try_wait_hint_a(uint32_t bar_addr, uint32_t parity, uint32_t hint_ns) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred P;\n\tmbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2, %3;\n\tselp.b32 %0, 1, 0, P;\n\t}"
                 : "=r"(ok) : "r"(bar_addr), "r"(parity), "r"(hint_ns) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait_a(uint32_t bar_addr, uint32_t parity, int *err_flag = nullptr, int code = 1) {
    if (mbar_try_wait_a(bar_addr, parity)) return;
    uint32_t spins = 0;
    while (!mbar_try_wait_hint_a(bar_addr, parity, 20000u)) {
        if (++spins > (1u << 20)) {
            if (err_flag) *reinterpret_cast<volatile int *>(err_flag) = code;
            __threadfence_system();
            asm volatile("trap;");
        }
    }
}
__device__ __forceinline__ void mbar_arrive_a(uint32_t bar_addr) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar_addr) : "memory");
}

// ---------------------------------------------------------------- fences / barriers
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const void *tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// 2D tiled load global -> smem, completion on mbarrier (complete_tx)
__device__ __forceinline__ void tma_load_2d(void *smem_dst, const void *tmap, int32_t c0, int32_t c1, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
// same with an L2 cache-policy operand (createpolicy-style 64-bit hint)
__device__ __forceinline__ void tma_load_2d_hint(void *smem_dst, const void *tmap, int32_t c0, int32_t c1, uint64_t *bar,
                                                 uint64_t policy) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint "
                 "[%0], [%1, {%3, %4}], [%2], %5;"
                 ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
                 "l"(policy) : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
// 1D bulk store smem -> global (bulk async-group completion)
__device__ __forceinline__ void bulk_store_1d(void *gmem_dst, const void *smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 ::"l"(reinterpret_cast<uint64_t>(gmem_dst)), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
// 1D bulk load global -> smem with mbarrier completion
__device__ __forceinline__ void bulk_load_1d(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(gmem_src)), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// ---------------------------------------------------------------- shared-memory matrix descriptor (wgmma)
// start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | base_offset [49,52) | layout_type [62,64)  (0 none, 1 128B, 2 64B, 3 32B).
// K-major operands: LBO = byte distance between core matrices adjacent in K (no-swizzle layouts only), SBO = between 8-row groups.
enum : uint64_t { GMMA_LAYOUT_NONE = 0, GMMA_LAYOUT_SW128 = 1 };
__host__ __device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint64_t layout) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32) | (layout << 62);
}

// ---------------------------------------------------------------- warpgroup MMA (all 128 threads of a warpgroup, .sync.aligned)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x N] (+)= A[64 x 32] * B[N x 32]^T, s8 x s8 -> s32, both operands K-major.  Accumulator fragment of thread t of warp w:
// d[4 j + 0, 1] = row 16 w + t / 4, columns 8 j + 2 (t % 4) + {0, 1}; d[4 j + 2, 3] = the same columns of row 16 w + t / 4 + 8.
// _ss: A from shared memory (descriptor); _rs: A from registers, a[0..3] = int8x4 of (row t/4, k 4 (t%4) ..), (row t/4 + 8, same k),
// (row t/4, k 16 + 4 (t%4) ..), (row t/4 + 8, k 16 + 4 (t%4) ..).
__device__ __forceinline__ void wgmma_ss_n16(uint32_t *d, uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p;\n\t}"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
                 : "l"(a_desc), "l"(b_desc), "r"(accumulate) : "memory");
}
__device__ __forceinline__ void wgmma_rs_n16(uint32_t *d, const uint32_t *a, uint64_t b_desc, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7}, {%8,%9,%10,%11}, %12, p;\n\t}"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate) : "memory");
}
__device__ __forceinline__ void wgmma_ss_n64(uint32_t *d, uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p;\n\t}"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
                 : "l"(a_desc), "l"(b_desc), "r"(accumulate) : "memory");
}
__device__ __forceinline__ void wgmma_rs_n64(uint32_t *d, const uint32_t *a, uint64_t b_desc, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p;\n\t}"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate) : "memory");
}

}  // namespace bnm
