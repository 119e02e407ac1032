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

/* one device allocation carved into n pieces of sz[i] bytes, each 256-byte aligned: *out[i] gets piece i. Returns the
 * allocation (free it with mz_cuda_free), NULL when it fails. */
static inline uint8_t *mzh_carve(const size_t *sz, void **out[], int n) {
    size_t total = 0;
    for (int i = 0; i < n; i++)
        total += (sz[i] + 255) & ~(size_t)255;
    uint8_t *p = (uint8_t *)mz_cuda_malloc(total ? total : 256);
    if (!p)
        return NULL;
    size_t o = 0;
    for (int i = 0; i < n; i++) {
        *out[i] = p + o;
        o += (sz[i] + 255) & ~(size_t)255;
    }
    return p;
}

/* chunks of 64 KiB per round of the device-memory writers (mz_zip_cuda_write_device / update_device, mz_cuda_gzip_compress_device):
 * MZ_CUDA_ZIP_ROUND_MB, 1024 when unset, empty, not a positive number; at most 32768 (the place scan is 32-bit) and at most nch */
static inline uint64_t mzh_round_chunks(uint64_t nch) {
    const char *v = getenv("MZ_CUDA_ZIP_ROUND_MB");
    const long long mb = v && *v ? atoll(v) : 0;
    uint64_t R = ((uint64_t)(mb > 0 ? mb : 1024) << 20) / 65536;
    if (R < 1)
        R = 1;
    if (R > 32768)
        R = 32768;
    if (R > nch)
        R = nch ? nch : 1;
    return R;
}

#endif
