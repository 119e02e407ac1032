/* mzcuda_common.cuh -- shared device helpers for the mz_strm_cuda kernels (sm_90a).
 *
 * Compiles two ways: with nvcc for the product (the only build that ships), and with g++ -DMZ_EMU
 * against tests/emu/cuda_emu.h so the kernel logic can be exercised on the CPU by the unit tests.
 */
#ifndef MZCUDA_COMMON_CUH
#define MZCUDA_COMMON_CUH

#include <stdint.h>

#ifdef MZ_EMU
#include "cuda_emu.h"
#define MZ_DYN_SMEM(name) uint8_t *name = emu_dyn_smem
/* The emulator's preemption and race-check hooks (tests/emu/cuda_emu.h defines them). Without them every access below is a plain
 * load or store. */
#ifndef MZ_EMU_ACCESS
#define MZ_EMU_ACCESS(p, bytes, kind, newval)
#define MZ_EMU_PREEMPT()
#endif
#else
#include <cuda_runtime.h>
#define MZ_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#define MZ_DYN_SMEM(name) extern __shared__ __align__(128) uint8_t name[]
#endif

#define MZ_FULL_MASK 0xffffffffu

namespace mzc {

__device__ __forceinline__ unsigned lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ unsigned warp_id() { return threadIdx.x >> 5; }

/* unaligned little-endian 32-bit load from a byte buffer whose base is 4-byte aligned and which is
 * readable for 4 bytes past (p & ~3) + 4 */
__device__ __forceinline__ uint32_t load32u(const uint8_t *base, uint32_t p) {
    const uint32_t *w = (const uint32_t *)(base + (p & ~3u));
    return __funnelshift_r(w[0], w[1], (p & 3u) * 8u);
}

/* streaming 128-bit global load that does not pollute L1 */
__device__ __forceinline__ uint4 ldg_stream(const uint4 *p) {
#ifdef MZ_EMU
    MZ_EMU_PREEMPT();
    return *p;
#else
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
#endif
}


/* Explicit shared-state-space accessors for the hot loops. Going through generic pointers derived from
 * `extern __shared__` makes nvcc re-derive the shared window base (S2R SR_CgaCtaId + LEA) at most uses;
 * one 32-bit shared address kept in a register and ld.shared/st.shared on it avoids that. Under the CPU
 * emulator the "address" is a byte offset into the emulated dynamic shared memory. */
struct Smem {
#ifdef MZ_EMU
    /* every access first passes MZ_EMU_ACCESS: a seeded preemption point and the shared-memory race check (cuda_emu.h) */
    uint8_t *b;
    __device__ __forceinline__ void init(uint8_t *base) { b = base; }
    __device__ __forceinline__ uint8_t *p(uint32_t off) const { return b + (int32_t)off; }
    __device__ __forceinline__ uint32_t ld32(uint32_t off) const { MZ_EMU_ACCESS(p(off), 4, EMU_ACC_READ, nullptr); return *(const uint32_t *)p(off); }
    __device__ __forceinline__ uint32_t ld16(uint32_t off) const { MZ_EMU_ACCESS(p(off), 2, EMU_ACC_READ, nullptr); return *(const uint16_t *)p(off); }
    __device__ __forceinline__ uint32_t ld8(uint32_t off) const { MZ_EMU_ACCESS(p(off), 1, EMU_ACC_READ, nullptr); return *p(off); }
    __device__ __forceinline__ void st32(uint32_t off, uint32_t v) const { MZ_EMU_ACCESS(p(off), 4, EMU_ACC_WRITE, &v); *(uint32_t *)p(off) = v; }
    __device__ __forceinline__ void st16(uint32_t off, uint32_t v) const {
        const uint16_t h = (uint16_t)v;
        MZ_EMU_ACCESS(p(off), 2, EMU_ACC_WRITE, &h);
        *(uint16_t *)p(off) = h;
    }
    __device__ __forceinline__ void red_or32(uint32_t off, uint32_t v) const { MZ_EMU_ACCESS(p(off), 4, EMU_ACC_ATOMIC, nullptr); *(uint32_t *)p(off) |= v; }
    __device__ __forceinline__ void red_add32(uint32_t off, uint32_t v) const { MZ_EMU_ACCESS(p(off), 4, EMU_ACC_ATOMIC, nullptr); *(uint32_t *)p(off) += v; }
    __device__ __forceinline__ void red_min32(uint32_t off, uint32_t v) const {
        MZ_EMU_ACCESS(p(off), 4, EMU_ACC_ATOMIC, nullptr);
        uint32_t *q = (uint32_t *)p(off);
        if (v < *q) *q = v;
    }
    __device__ __forceinline__ void st16_if(bool c, uint32_t off, uint32_t v) const { if (c) st16(off, v); }
    __device__ __forceinline__ void red_add32_if(bool c, uint32_t off, uint32_t v) const { if (c) red_add32(off, v); }
    __device__ __forceinline__ void red_or32_if(bool c, uint32_t off, uint32_t v) const { if (c) red_or32(off, v); }
    __device__ __forceinline__ uint2 ld64(uint32_t off) const { MZ_EMU_ACCESS(p(off), 8, EMU_ACC_READ, nullptr); return *(const uint2 *)p(off); }
    __device__ __forceinline__ void st64(uint32_t off, uint32_t x, uint32_t y) const {
        const uint2 v = make_uint2(x, y);
        MZ_EMU_ACCESS(p(off), 8, EMU_ACC_WRITE, &v);
        *(uint2 *)p(off) = v;
    }
    __device__ __forceinline__ void st128(uint32_t off, uint32_t x, uint32_t y, uint32_t z, uint32_t w) const {
        const uint4 v = make_uint4(x, y, z, w);
        MZ_EMU_ACCESS(p(off), 16, EMU_ACC_WRITE, &v);
        *(uint4 *)p(off) = v;
    }
    /* absolute forms: addr() folds the window base into a region base once, the *_a accessors then take that address as it is */
    __device__ __forceinline__ uint32_t addr(uint32_t off) const { return off; }
    __device__ __forceinline__ uint32_t ld32_a(uint32_t a) const { return ld32(a); }
    __device__ __forceinline__ uint32_t ld8_a(uint32_t a) const { return ld8(a); }
    __device__ __forceinline__ void red_or32_a(uint32_t a, uint32_t v) const { red_or32(a, v); }
    __device__ __forceinline__ void red_add32_a(uint32_t a, uint32_t v) const { red_add32(a, v); }
#else
    uint32_t b;
    __device__ __forceinline__ void init(uint8_t *base) {
        b = (uint32_t)__cvta_generic_to_shared(base);
        asm volatile("" : "+r"(b)); /* opaque: keep the address in a register instead of re-deriving it (S2R + LEA) at every use */
    }
    __device__ __forceinline__ uint32_t ld32(uint32_t off) const {
        uint32_t v;
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(b + off));
        return v;
    }
    __device__ __forceinline__ uint32_t ld16(uint32_t off) const {
        uint32_t v;
        asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(b + off));
        return v;
    }
    __device__ __forceinline__ uint32_t ld8(uint32_t off) const {
        uint32_t v;
        asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(b + off));
        return v;
    }
    __device__ __forceinline__ void st32(uint32_t off, uint32_t v) const { asm volatile("st.shared.u32 [%0], %1;" ::"r"(b + off), "r"(v) : "memory"); }
    __device__ __forceinline__ void st16(uint32_t off, uint32_t v) const { asm volatile("st.shared.u16 [%0], %1;" ::"r"(b + off), "r"(v) : "memory"); }
    __device__ __forceinline__ void red_or32(uint32_t off, uint32_t v) const { asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(b + off), "r"(v) : "memory"); }
    __device__ __forceinline__ void red_add32(uint32_t off, uint32_t v) const { asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(b + off), "r"(v) : "memory"); }
    __device__ __forceinline__ void red_min32(uint32_t off, uint32_t v) const { asm volatile("red.shared.min.u32 [%0], %1;" ::"r"(b + off), "r"(v) : "memory"); }
    /* predicated forms: one instruction under a predicate instead of a branch around an asm statement */
    __device__ __forceinline__ void st16_if(bool p, uint32_t off, uint32_t v) const {
        asm volatile("{\n.reg .pred q;\nsetp.ne.u32 q, %2, 0;\n@q st.shared.u16 [%0], %1;\n}" ::"r"(b + off), "r"(v), "r"((uint32_t)p) : "memory");
    }
    __device__ __forceinline__ void red_add32_if(bool p, uint32_t off, uint32_t v) const {
        asm volatile("{\n.reg .pred q;\nsetp.ne.u32 q, %2, 0;\n@q red.shared.add.u32 [%0], %1;\n}" ::"r"(b + off), "r"(v), "r"((uint32_t)p) : "memory");
    }
    __device__ __forceinline__ void red_or32_if(bool p, uint32_t off, uint32_t v) const {
        asm volatile("{\n.reg .pred q;\nsetp.ne.u32 q, %2, 0;\n@q red.shared.or.b32 [%0], %1;\n}" ::"r"(b + off), "r"(v), "r"((uint32_t)p) : "memory");
    }
    __device__ __forceinline__ uint2 ld64(uint32_t off) const {
        uint2 v;
        asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(b + off));
        return v;
    }
    __device__ __forceinline__ void st64(uint32_t off, uint32_t x, uint32_t y) const { asm volatile("st.shared.v2.u32 [%0], {%1,%2};" ::"r"(b + off), "r"(x), "r"(y) : "memory"); }
    __device__ __forceinline__ void st128(uint32_t off, uint32_t x, uint32_t y, uint32_t z, uint32_t w) const {
        asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(b + off), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
    }
    __device__ __forceinline__ uint32_t addr(uint32_t off) const { return b + off; }
    __device__ __forceinline__ uint32_t ld32_a(uint32_t a) const {
        uint32_t v;
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
        return v;
    }
    __device__ __forceinline__ uint32_t ld8_a(uint32_t a) const {
        uint32_t v;
        asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a));
        return v;
    }
    __device__ __forceinline__ void red_or32_a(uint32_t a, uint32_t v) const { asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
    __device__ __forceinline__ void red_add32_a(uint32_t a, uint32_t v) const { asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
#endif
    /* unaligned little-endian 32-bit load at byte offset `off + p` (region base `off` is 4-byte aligned) */
    __device__ __forceinline__ uint32_t ld32u(uint32_t off, uint32_t p) const {
        uint32_t a = off + (p & ~3u);
        return __funnelshift_r(ld32(a), ld32(a + 4), (p & 3u) * 8u);
    }
};

/* named barrier over the first `nthreads` threads' worth of warps (id 1..15; 0 is __syncthreads) */
__device__ __forceinline__ void bar_sync(int id, int nthreads) {
#ifdef MZ_EMU
    emu_named_barrier(id, nthreads);
#else
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
#endif
}

/* warp inclusive scan (sum) */
__device__ __forceinline__ uint32_t warp_incl_sum(uint32_t v) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t n = __shfl_up_sync(MZ_FULL_MASK, v, d);
        if (lane_id() >= (unsigned)d) v += n;
    }
    return v;
}

__device__ __forceinline__ uint32_t warp_incl_max(uint32_t v) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t n = __shfl_up_sync(MZ_FULL_MASK, v, d);
        if (lane_id() >= (unsigned)d) v = v > n ? v : n;
    }
    return v;
}

/* v << s with PTX semantics: a shift amount of 32 or more (also a "negative" one that wrapped) gives 0 */
__device__ __forceinline__ uint32_t shl_clamp(uint32_t v, uint32_t s) {
#ifdef MZ_EMU
    return s >= 32u ? 0u : v << s;
#else
    uint32_t r;
    asm("shl.b32 %0, %1, %2;" : "=r"(r) : "r"(v), "r"(s));
    return r;
#endif
}
__device__ __forceinline__ uint32_t shr_clamp(uint32_t v, uint32_t s) {
#ifdef MZ_EMU
    return s >= 32u ? 0u : v >> s;
#else
    uint32_t r;
    asm("shr.u32 %0, %1, %2;" : "=r"(r) : "r"(v), "r"(s));
    return r;
#endif
}
/* byte k (0..3, a constant) of a word */
#define MZ_BYTE(x, k) __byte_perm((x), 0u, 0x4440u + (k))

#ifndef MZ_EMU
/* ---- mbarrier + TMA bulk copy (cp.async.bulk; SASS: UBLKCP) ------------------------------------ */
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t phase) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(phase)
        : "memory");
}
/* global -> shared bulk copy; dst, src 16-byte aligned, bytes multiple of 16 */
__device__ __forceinline__ void tma_load_1d(void *smem_dst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
/* shared -> global bulk copy (bulk async-group completion) */
__device__ __forceinline__ void tma_store_1d(void *gdst, const void *smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
#endif

} // namespace mzc
#endif
