/* emu_sched_selftest.cc -- toy kernels with one planted defect each, and their corrected twins, for the emulator's seeded
 * schedules and shared-memory race checker (cuda_emu.h). TEST INFRASTRUCTURE ONLY: built with cuda_emu.cc by
 * tests/test_emu_schedules.py, which shows that every defect is reported by the checker or gives output that differs
 * between seeds, and that every twin runs clean with the same output under every seed. */
#define MZ_EMU 1
#include "../../minizip-ng_b200/csrc/mzcuda_common.cuh"

using namespace mzc;

/* a write and a read of other threads' words with no __syncthreads between them */
static void toy_no_sync(int fixed, uint32_t *out) {
    MZ_DYN_SMEM(smem);
    Smem sm;
    sm.init(smem);
    const uint32_t t = threadIdx.x;
    sm.st32(4 * t, t * 7 + 1);
    if (fixed) __syncthreads();
    out[t] = sm.ld32(4 * ((t + 1) % blockDim.x));
}

/* a counter every thread bumps with a plain load and store instead of an atomic */
static void toy_plain_counter(int fixed, uint32_t *out) {
    MZ_DYN_SMEM(smem);
    Smem sm;
    sm.init(smem);
    if (threadIdx.x == 0) sm.st32(0, 0);
    __syncthreads();
    if (fixed) sm.red_add32(0, 1);
    else sm.st32(0, sm.ld32(0) + 1);
    __syncthreads();
    if (threadIdx.x == 0) out[0] = sm.ld32(0);
}

/* three warps meet at named barriers sized for two: the writing warp is not always among them */
static void toy_named_barrier_short(int fixed, uint32_t *out) {
    MZ_DYN_SMEM(smem);
    Smem sm;
    sm.init(smem);
    const uint32_t lane = lane_id(), warp = warp_id(), n = fixed ? 96 : 64;
    uint32_t acc = 0;
    for (uint32_t it = 0; it < 2; it++) {
        if (warp == 2) sm.st32(4 * lane, it * 100 + lane);
        bar_sync(1, n);
        if (warp == 0) acc += sm.ld32(4 * lane);
        bar_sync(1, n);
    }
    if (warp == 0) out[lane] = acc;
}

/* a __syncwarp whose mask leaves out the lane that wrote the word another lane reads */
static void toy_syncwarp_mask(int fixed, uint32_t *out) {
    MZ_DYN_SMEM(smem);
    Smem sm;
    sm.init(smem);
    const uint32_t lane = lane_id();
    sm.st32(4 * lane, lane * 3 + 5);
    if (fixed) __syncwarp();
    else if (lane != 31) __syncwarp(0x7fffffffu);
    out[lane] = sm.ld32(4 * ((lane + 1) & 31));
}

/* a read of a dynamic shared word nobody wrote: the last thread's store is missing */
static void toy_unwritten_dynamic(int fixed, uint32_t *out) {
    MZ_DYN_SMEM(smem);
    Smem sm;
    sm.init(smem);
    const uint32_t t = threadIdx.x;
    if (fixed || t != blockDim.x - 1) sm.st32(4 * t, t);
    __syncthreads();
    out[t] = sm.ld32(4 * ((t + 1) % blockDim.x));
}

/* the same through a static __shared__ array, which the race checker does not see but the poisoning reaches */
static void toy_unwritten_static(int fixed, uint32_t *out) {
    __shared__ uint32_t s_tab[32];
    const uint32_t t = threadIdx.x;
    if (fixed || t != 31) s_tab[t] = t * 11;
    __syncthreads();
    out[t] = s_tab[(t + 1) & 31];
}

/* block 1 reads a global word that block 0 writes: right only when block 0 runs first */
static void toy_cta_order(int fixed, uint32_t *out) {
    if (threadIdx.x != 0) return;
    if (blockIdx.x == 0) out[0] = 42;
    else out[1] = fixed ? 42 : out[0];
}

extern "C" {
/* runs one toy, its defect planted (fixed = 0) or corrected (fixed = 1); out holds 64 words, zeroed first. Returns -1 for an
 * unknown name. */
int emu_selftest(const char *name, int fixed, uint32_t *out) {
    memset(out, 0, 64 * 4);
    if (!strcmp(name, "no_sync")) MZ_LAUNCH(toy_no_sync, dim3(1), dim3(64), 256, 0, fixed, out);
    else if (!strcmp(name, "plain_counter")) MZ_LAUNCH(toy_plain_counter, dim3(1), dim3(64), 16, 0, fixed, out);
    else if (!strcmp(name, "named_barrier_short")) MZ_LAUNCH(toy_named_barrier_short, dim3(1), dim3(96), 128, 0, fixed, out);
    else if (!strcmp(name, "syncwarp_mask")) MZ_LAUNCH(toy_syncwarp_mask, dim3(1), dim3(32), 128, 0, fixed, out);
    else if (!strcmp(name, "unwritten_dynamic")) MZ_LAUNCH(toy_unwritten_dynamic, dim3(1), dim3(32), 128, 0, fixed, out);
    else if (!strcmp(name, "unwritten_static")) MZ_LAUNCH(toy_unwritten_static, dim3(1), dim3(32), 0, 0, fixed, out);
    else if (!strcmp(name, "cta_order")) MZ_LAUNCH(toy_cta_order, dim3(2), dim3(32), 0, 0, fixed, out);
    else return -1;
    return 0;
}
}
