/* cuda_emu.h -- minimal single-OS-thread CUDA execution-model emulator (TEST INFRASTRUCTURE ONLY).
 *
 * Purpose: test the kernels on machines without a GPU, where a GPU run is slow or unavailable. This header
 * lets the kernel SOURCES under minizip-ng_b200/csrc/ be compiled with g++ (-DMZ_EMU) and run on the
 * CPU with CUDA semantics that matter for logic bugs: a CTA's threads are fibers that run until they
 * hit __syncthreads() or a warp collective; shared memory, atomics, shuffles and ballots behave as on
 * the device for race-free code. It is never linked into the product library and never used as a
 * fallback: the product .so is built by nvcc only and fails loudly without a GPU.
 *
 * Not modelled: real concurrency, memory-ordering, bank conflicts, timing, TMA/mbarrier (kernels
 * guard their PTX with #ifndef MZ_EMU and use a plain copy under emulation).
 *
 * Seeded schedules (MZ_EMU_SCHED=<seed>, unset or 0 = the fixed schedule: tid order, blockIdx order, 0xCD fill):
 *  - every scheduler pass runs the runnable fibers of a CTA in a fresh seeded permutation;
 *  - before every Smem accessor, emulated atomic and ldg_stream a fiber yields with a small seeded probability
 *    (EMU_PREEMPT_ONE_IN), so lanes of one warp interleave between two shared accesses as they can on Volta and later;
 *  - each launch visits its CTAs in a seeded permutation of blockIdx;
 *  - at every CTA, dynamic shared memory and all static __shared__ storage (the mz_emu_shared section) are filled
 *    with seeded random bytes, so a read of shared memory nobody wrote gives seed-dependent output.
 *
 * Shared-memory race checker (MZ_EMU_RACE=1; most useful together with a seed):
 *  - shadow state per 4-byte word of the CTA's dynamic shared memory and of the static __shared__ storage records the
 *    last write (thread, plain or atomic, byte mask) and up to EMU_RACE_READERS reads since it;
 *  - happens-before comes only from a block barrier, from a named barrier in which both threads' whole warps took
 *    part, and from a warp barrier or warp collective of one warp whose mask holds both lanes (all transitively);
 *  - reported: a plain write followed by a read or a write of an overlapping byte by another thread, and a read
 *    followed by a write (plain or atomic) by another thread, with no such edge between them. Atomic against
 *    atomic is never reported, and neither is an atomic followed by a plain read. A plain write that leaves the
 *    bytes as they are (several threads storing the same value, an idiom the kernels use) is allowed;
 *  - the report names the launch, the block, the word and both threads, then aborts;
 *  - coverage: only the Smem accessors (mzcuda_common.cuh) and the emulated atomics are seen. Shared memory read or
 *    written through raw pointers or array indexing (staging through uint8_t pointers, static __shared__ arrays,
 *    inflate's table structs) is invisible to it; poisoning still covers those. When more than EMU_RACE_READERS
 *    threads read a word concurrently, only that many reads are kept for the check against the next write.
 */
#ifndef CUDA_EMU_H
#define CUDA_EMU_H
#ifndef MZ_EMU
#error "cuda_emu.h is for -DMZ_EMU host builds only"
#endif

#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __restrict__
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))
/* static __shared__ variables live in one section so that the scheduler can poison them at every CTA and the race checker can
 * map their addresses (cuda_emu.cc, __start_/__stop_mz_emu_shared) */
#define __shared__ static __attribute__((section("mz_emu_shared")))
#define __constant__ static

struct emu_dim3 {
    unsigned x, y, z;
    emu_dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {}
};
typedef emu_dim3 dim3;
struct uint4 { uint32_t x, y, z, w; };
struct uint2 { uint32_t x, y; };
static inline uint4 make_uint4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) { uint4 r = {a, b, c, d}; return r; }
static inline uint2 make_uint2(uint32_t a, uint32_t b) { uint2 r = {a, b}; return r; }

extern emu_dim3 threadIdx, blockIdx, blockDim, gridDim;
extern uint8_t *emu_dyn_smem;
static const int warpSize = 32;

/* ---- fibers ------------------------------------------------------------------------------- */
struct emu_fiber {
    void *sp;          /* saved stack pointer */
    void *stack;
    int done;
    int wait_block;    /* waiting at __syncthreads */
    int tid;
};

extern "C" void emu_switch(void **save_sp, void *load_sp);
void emu_yield(void);
void emu_run_block(unsigned nthreads, void (*entry)(void *), void *arg, size_t dyn_smem);

struct emu_warp_state {
    uint64_t slot[32];
    unsigned arrived;   /* lanes waiting at a warp barrier */
    unsigned want[32];  /* the mask each waiting lane named (its own bit included) */
    unsigned gen[32];   /* per lane: bumped when its warp barrier releases it */
    unsigned live_mask; /* lanes that exist and have not exited */
};
extern emu_warp_state *emu_cur_warp(void);
extern int emu_lane(void);
void emu_block_barrier(void);
void emu_named_barrier(int id, int nthreads);
void emu_warp_barrier(unsigned mask);

/* seeded schedules and the race checker (cuda_emu.cc) */
extern int emu_sched_on, emu_race_on, emu_hooks_on; /* emu_hooks_on = either: one test on the hot path when both are off */
void emu_preempt_slow(void);
static inline void emu_preempt(void) {
    if (emu_sched_on) emu_preempt_slow();
}
enum { EMU_ACC_READ = 0, EMU_ACC_WRITE = 1, EMU_ACC_ATOMIC = 2 };
void emu_access_slow(const void *p, unsigned bytes, int kind, const void *newval);
/* one shared-memory access through an Smem accessor or an atomic: a possible preemption point, then the race check. newval is
 * the bytes a plain write is about to store. */
static inline void emu_access(const void *p, unsigned bytes, int kind, const void *newval = nullptr) {
    if (__builtin_expect(emu_hooks_on, 0)) emu_access_slow(p, bytes, kind, newval);
}

/* the hooks as the Smem accessors and ldg_stream call them (mzcuda_common.cuh) */
#define MZ_EMU_ACCESS(p, bytes, kind, newval) emu_access((p), (bytes), (kind), (newval))
#define MZ_EMU_PREEMPT() emu_preempt()

static inline void __syncthreads() { emu_block_barrier(); }
static inline void __syncwarp(unsigned mask = 0xffffffffu) { emu_warp_barrier(mask); }
static inline void __threadfence() {}
static inline void __threadfence_block() {}

/* exchange: every participating lane publishes v, then reads after a warp barrier */
static inline uint64_t emu_exchange(unsigned mask, uint64_t v, int src_lane) {
    emu_warp_state *w = emu_cur_warp();
    w->slot[emu_lane()] = v;
    emu_warp_barrier(mask);
    uint64_t r = w->slot[src_lane & 31];
    emu_warp_barrier(mask);
    return r;
}

template <typename T> static inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
    uint64_t u = 0;
    memcpy(&u, &v, sizeof(T));
    int lane = emu_lane();
    int base = lane & ~(width - 1);
    u = emu_exchange(mask, u, base + (src & (width - 1)));
    T r;
    memcpy(&r, &u, sizeof(T));
    return r;
}
template <typename T> static inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    int lane = emu_lane();
    int src = lane - (int)delta;
    uint64_t u = 0;
    memcpy(&u, &v, sizeof(T));
    uint64_t got = emu_exchange(mask, u, src < (lane & ~(width - 1)) ? lane : src);
    T r;
    memcpy(&r, &got, sizeof(T));
    return r;
}
template <typename T> static inline T __shfl_down_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    int lane = emu_lane();
    int src = lane + (int)delta;
    uint64_t u = 0;
    memcpy(&u, &v, sizeof(T));
    uint64_t got = emu_exchange(mask, u, src > (lane | (width - 1)) ? lane : src);
    T r;
    memcpy(&r, &got, sizeof(T));
    return r;
}
template <typename T> static inline T __shfl_xor_sync(unsigned mask, T v, int lanemask, int width = 32) {
    (void)width;
    uint64_t u = 0;
    memcpy(&u, &v, sizeof(T));
    uint64_t got = emu_exchange(mask, u, emu_lane() ^ lanemask);
    T r;
    memcpy(&r, &got, sizeof(T));
    return r;
}
static inline unsigned __ballot_sync(unsigned mask, int pred) {
    emu_warp_state *w = emu_cur_warp();
    w->slot[emu_lane()] = pred ? 1 : 0;
    emu_warp_barrier(mask);
    unsigned r = 0;
    for (int i = 0; i < 32; i++)
        if ((mask >> i) & 1 & (unsigned)w->slot[i]) r |= 1u << i;
    emu_warp_barrier(mask);
    return r;
}
static inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
static inline int __all_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) == (mask & emu_cur_warp()->live_mask); }
static inline unsigned __match_any_sync(unsigned mask, unsigned v) {
    emu_warp_state *w = emu_cur_warp();
    w->slot[emu_lane()] = v;
    emu_warp_barrier(mask);
    unsigned r = 0;
    for (int i = 0; i < 32; i++)
        if (((mask >> i) & 1) && (unsigned)w->slot[i] == v) r |= 1u << i;
    emu_warp_barrier(mask);
    return r;
}
static inline unsigned __reduce_add_sync(unsigned mask, unsigned v) {
    emu_warp_state *w = emu_cur_warp();
    w->slot[emu_lane()] = v;
    emu_warp_barrier(mask);
    unsigned r = 0;
    for (int i = 0; i < 32; i++)
        if ((mask >> i) & 1) r += (unsigned)w->slot[i];
    emu_warp_barrier(mask);
    return r;
}
static inline unsigned __reduce_max_sync(unsigned mask, unsigned v) {
    emu_warp_state *w = emu_cur_warp();
    w->slot[emu_lane()] = v;
    emu_warp_barrier(mask);
    unsigned r = 0;
    for (int i = 0; i < 32; i++)
        if ((mask >> i) & 1) r = std::max(r, (unsigned)w->slot[i]);
    emu_warp_barrier(mask);
    return r;
}
static inline unsigned __reduce_min_sync(unsigned mask, unsigned v) {
    emu_warp_state *w = emu_cur_warp();
    w->slot[emu_lane()] = v;
    emu_warp_barrier(mask);
    unsigned r = 0xffffffffu;
    for (int i = 0; i < 32; i++)
        if ((mask >> i) & 1) r = std::min(r, (unsigned)w->slot[i]);
    emu_warp_barrier(mask);
    return r;
}
static inline unsigned __reduce_or_sync(unsigned mask, unsigned v) {
    emu_warp_state *w = emu_cur_warp();
    w->slot[emu_lane()] = v;
    emu_warp_barrier(mask);
    unsigned r = 0;
    for (int i = 0; i < 32; i++)
        if ((mask >> i) & 1) r |= (unsigned)w->slot[i];
    emu_warp_barrier(mask);
    return r;
}
static inline unsigned __reduce_xor_sync(unsigned mask, unsigned v) {
    emu_warp_state *w = emu_cur_warp();
    w->slot[emu_lane()] = v;
    emu_warp_barrier(mask);
    unsigned r = 0;
    for (int i = 0; i < 32; i++)
        if ((mask >> i) & 1) r ^= (unsigned)w->slot[i];
    emu_warp_barrier(mask);
    return r;
}
static inline unsigned __activemask() { return emu_cur_warp()->live_mask; }

/* ---- intrinsics ------------------------------------------------------------------------------ */
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }
static inline int __clz(int v) { return v == 0 ? 32 : __builtin_clz((unsigned)v); }
static inline int __clzll(long long v) { return v == 0 ? 64 : __builtin_clzll((unsigned long long)v); }
static inline int __ffs(int v) { return __builtin_ffs(v); }
static inline int __ffsll(long long v) { return __builtin_ffsll(v); }
static inline unsigned __brev(unsigned v) {
    unsigned r = 0;
    for (int i = 0; i < 32; i++) { r = (r << 1) | (v & 1); v >>= 1; }
    return r;
}
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned shift) {
    uint64_t v = ((uint64_t)hi << 32) | lo;
    return (unsigned)(v >> (shift & 31));
}
static inline unsigned __funnelshift_rc(unsigned lo, unsigned hi, unsigned shift) { /* clamped at 32 */
    if (shift >= 32) return hi;
    return shift ? (lo >> shift) | (hi << (32 - shift)) : lo;
}
static inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned shift) {
    uint64_t v = ((uint64_t)hi << 32) | lo;
    return (unsigned)((v << (shift & 31)) >> 32);
}
static inline unsigned __byte_perm(unsigned a, unsigned b, unsigned s) {
    uint64_t v = ((uint64_t)b << 32) | a;
    unsigned r = 0;
    for (int i = 0; i < 4; i++) r |= (unsigned)((v >> (8 * ((s >> (4 * i)) & 7))) & 0xff) << (8 * i);
    return r;
}
#define __log2f(x) log2f(x)
#define __exp2f(x) exp2f(x)
#define __powf(a, b) powf(a, b)
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((uint64_t)a * b) >> 32); }
template <typename T> static inline T __ldg(const T *p) { return *p; }

/* an emulated atomic is a plain read-modify-write that no other fiber can split: the preemption point comes before it */
template <typename T> static inline T atomicAdd(T *p, T v) { emu_access(p, sizeof(T), EMU_ACC_ATOMIC); T o = *p; *p = o + v; return o; }
template <typename T> static inline T atomicOr(T *p, T v) { emu_access(p, sizeof(T), EMU_ACC_ATOMIC); T o = *p; *p = o | v; return o; }
template <typename T> static inline T atomicXor(T *p, T v) { emu_access(p, sizeof(T), EMU_ACC_ATOMIC); T o = *p; *p = o ^ v; return o; }
template <typename T> static inline T atomicMax(T *p, T v) { emu_access(p, sizeof(T), EMU_ACC_ATOMIC); T o = *p; if (v > o) *p = v; return o; }
template <typename T> static inline T atomicMin(T *p, T v) { emu_access(p, sizeof(T), EMU_ACC_ATOMIC); T o = *p; if (v < o) *p = v; return o; }
template <typename T> static inline T atomicExch(T *p, T v) { emu_access(p, sizeof(T), EMU_ACC_ATOMIC); T o = *p; *p = v; return o; }
template <typename T> static inline T atomicCAS(T *p, T c, T v) { emu_access(p, sizeof(T), EMU_ACC_ATOMIC); T o = *p; if (o == c) *p = v; return o; }

/* ---- launch ---------------------------------------------------------------------------------- */
template <typename F> struct emu_thunk {
    F f;
    static void call(void *p) { (*(F *)p)(); }
};

/* one kernel at a time: the emulator's state (fibers, the built-in index variables, shared memory) is global, while the product
 * launches from several host threads (the zip writer's round workers) */
void emu_launch_lock(void);
void emu_launch_unlock(void);
/* the order in which a launch visits its CTAs (linear block indices): 0..n-1, or a seeded permutation of it */
const std::vector<uint64_t> &emu_block_order(uint64_t nblocks);
template <typename F> static inline void emu_launch(dim3 grid, dim3 block, size_t smem, F body) {
    emu_launch_lock();
    gridDim = grid;
    blockDim = block;
    for (uint64_t b : emu_block_order((uint64_t)grid.x * grid.y * grid.z)) {
        blockIdx = emu_dim3((unsigned)(b % grid.x), (unsigned)(b / grid.x % grid.y), (unsigned)(b / grid.x / grid.y));
        emu_run_block(block.x * block.y * block.z, &emu_thunk<F>::call, &body, smem);
    }
    emu_launch_unlock();
}
/* MZ_LAUNCH(kernel, grid, block, smem, stream, args...) */
#define MZ_LAUNCH(kernel, grid, block, smem, stream, ...) emu_launch((grid), (block), (smem), [&]() { kernel(__VA_ARGS__); })

#endif
