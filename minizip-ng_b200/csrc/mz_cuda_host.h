/* mz_cuda_host.h -- helpers shared by the host-side C files (mz_zip_cuda.c, mz_strm_cuda.c). Internal: static inline, not
 * installed, exports nothing. */
#ifndef MZ_CUDA_HOST_H
#define MZ_CUDA_HOST_H

#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "mz_abi.h"
#include "mz_cuda_batch.h"

/* MZ_OK, or MZ_SUPPORT_ERROR with a message on stderr naming the caller (`who`) when there is no usable GPU */
static inline int32_t mzh_gpu_required(const char *who) {
    if (mz_cuda_init() == MZ_OK)
        return MZ_OK;
    fprintf(stderr, "%s: no usable sm_90 GPU (%s); there is no CPU fallback\n", who, mz_cuda_last_error());
    return MZ_SUPPORT_ERROR;
}

/* a buffer in a table of staging or scratch buffers: where its pointer lives, its size, and whether it is page-locked host memory
 * (mz_cuda_host_alloc) or device memory (mz_cuda_malloc). MZH_DEV / MZH_PIN build one from the pointer variable itself. */
typedef struct mzh_piece_s {
    void **p;
    size_t size;
    int pinned;
} mzh_piece;

#define MZH_DEV(ptr, bytes) ((mzh_piece){(void **)&(ptr), (size_t)(bytes), 0})
#define MZH_PIN(ptr, bytes) ((mzh_piece){(void **)&(ptr), (size_t)(bytes), 1})

/* frees every piece of t[0, n) (NULL ones too) with the call that matches it, and sets its pointer to NULL */
static inline void mzh_free(const mzh_piece *t, int n) {
    for (int i = 0; i < n; i++) {
        if (t[i].pinned)
            mz_cuda_host_free(*t[i].p);
        else
            mz_cuda_free(*t[i].p);
        *t[i].p = NULL;
    }
}

/* one allocation per piece of t[0, n); a zero-byte piece is left NULL. All or nothing: 1, or 0 with every pointer NULL. Separate
 * allocations keep each buffer its own block, so an overrun of one is not hidden inside the next. */
static inline int mzh_alloc(const mzh_piece *t, int n) {
    for (int i = 0; i < n; i++)
        *t[i].p = NULL;
    for (int i = 0; i < n; i++) {
        if (!t[i].size)
            continue;
        *t[i].p = t[i].pinned ? mz_cuda_host_alloc(t[i].size) : mz_cuda_malloc(t[i].size);
        if (!*t[i].p) {
            mzh_free(t, n);
            return 0;
        }
    }
    return 1;
}

/* one device allocation carved into the pieces of t[0, n) in table order, each 256-byte aligned (the pinned flag is not used).
 * Returns the allocation (free it with mz_cuda_free), NULL when it fails. */
static inline uint8_t *mzh_carve(const mzh_piece *t, int n) {
    size_t total = 0;
    for (int i = 0; i < n; i++)
        total += (t[i].size + 255) & ~(size_t)255;
    uint8_t *p = (uint8_t *)mz_cuda_malloc(total ? total : 256);
    if (!p)
        return NULL;
    size_t o = 0;
    for (int i = 0; i < n; i++) {
        *t[i].p = p + o;
        o += (t[i].size + 255) & ~(size_t)255;
    }
    return p;
}

/* bytes per round from MZ_CUDA_ZIP_ROUND_MB (in MiB); dflt_mb when it is unset, empty or not a positive number */
static inline size_t mzh_round_bytes(size_t dflt_mb) {
    const char *v = getenv("MZ_CUDA_ZIP_ROUND_MB");
    const long long mb = v && *v ? atoll(v) : 0;
    return (mb > 0 ? (size_t)mb : dflt_mb) << 20;
}

/* chunks of 64 KiB per round of the device-memory writers (mz_zip_cuda_write_device / update_device, mz_cuda_gzip_compress_device):
 * mzh_round_bytes(1024) of them; at most 32768 (the place scan is 32-bit) and at most nch */
static inline uint64_t mzh_round_chunks(uint64_t nch) {
    uint64_t R = (uint64_t)mzh_round_bytes(1024) / 65536;
    if (R < 1)
        R = 1;
    if (R > 32768)
        R = 32768;
    if (R > nch)
        R = nch ? nch : 1;
    return R;
}

#endif
