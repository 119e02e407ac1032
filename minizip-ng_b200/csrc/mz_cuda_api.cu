/* mz_cuda_api.cu -- the thin extern "C" shim between the C host side and the sm_90a kernels.
 * Declares nothing new: every entry point is documented in include/mz_cuda_batch.h. */
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdio.h>
#include <string.h>

#include <mutex>
#include <vector>

#include "../../include/mz_cuda_batch.h"
#include "concat_kernel.cuh"
#include "crc32_kernel.cuh"
#include "deflate_kernel.cuh"
#include "gzip_kernel.cuh"
#include <cstdlib>
#include <cstdio>
#include "inflate_kernel.cuh"
#include "inflate_spec_kernel.cuh"
#include "sha256_kernel.cuh"
#include "wzaes_kernel.cuh"
#include "zipdir_kernel.cuh"
#include "zipcd_kernel.cuh"
#include "zipwr_kernel.cuh"
#include "zipsel_kernel.cuh"
#include "zipup_kernel.cuh"
#include "../../include/mz_zip_cuda.h"

#define MZ_OK 0
#define MZ_MEM_ERROR (-4)
#define MZ_FORMAT_ERROR (-103)
#define MZ_PARAM_ERROR (-102)
#define MZ_INTERNAL_ERROR (-104)
#define MZ_SUPPORT_ERROR (-109)

using namespace mzc;

static_assert(sizeof(mz_cuda_inflate_job) == sizeof(InflateJob), "job layout");
static_assert(sizeof(mz_cuda_inflate_state) == sizeof(InflateState), "state layout");
static_assert(sizeof(mz_cuda_spec_summary) == sizeof(SpecSummary), "summary layout");
static_assert(sizeof(mz_cuda_zip_ent) == sizeof(ZipEnt) && sizeof(mz_cuda_zip_ent) == 64, "zip entry layout");
static_assert(sizeof(mz_cuda_zip_round) == sizeof(ZipRound), "zip round layout");
static_assert(sizeof(mz_cuda_zip_dev_entry) == sizeof(ZipDevEnt) && sizeof(mz_cuda_zip_dev_entry) == 72 &&
                  offsetof(mz_cuda_zip_dev_entry, status) == offsetof(ZipDevEnt, status) && offsetof(ZipDevEnt, status) == 68,
              "device zip entry layout");
static_assert(sizeof(mz_cuda_zip_dev_item) == sizeof(ZwItem) && sizeof(ZwItem) == 40 && sizeof(mz_cuda_zip_wr_count) == sizeof(ZwCount) &&
                  sizeof(mz_cuda_zip_wr) == sizeof(ZwCall) && offsetof(mz_cuda_zip_wr, entries) == offsetof(ZwCall, entries) &&
                  offsetof(mz_cuda_zip_wr, comment) == offsetof(ZwCall, comment) &&
                  MZ_CUDA_ZIP_WR_TILE == ZC_TILE,
              "device zip writer layout");
static_assert(sizeof(mz_cuda_zip_sel_count) == sizeof(ZsCount) && sizeof(ZsCount) == 56 && sizeof(mz_cuda_zip_sel) == sizeof(ZsCall) &&
                  offsetof(mz_cuda_zip_sel, scratch) == offsetof(ZsCall, scratch),
              "device zip selection layout");
static_assert(sizeof(mz_cuda_zip_up_count) == sizeof(ZuCount) && sizeof(mz_cuda_zip_up) == sizeof(ZuCall) &&
                  offsetof(mz_cuda_zip_up, entries) == offsetof(ZuCall, entries) && MZ_CUDA_ZIP_UP_INFO == ZU_NINFO,
              "device zip update layout");

namespace {

struct DeviceCtx {
    bool ready = false;
    int sm_count = 0;
    CrcConsts *d_consts = nullptr;
    uint32_t *d_crc_scratch = nullptr; /* residues for mz_cuda_crc32_device */
    uint32_t *d_work = nullptr;        /* ring of work-counter pairs for dynamically scheduled launches */
    uint32_t *d_aes = nullptr;         /* K8 tables: 256 words of T-table, then the S-box (256 bytes); made on first use */
    unsigned work_next = 0;
    size_t crc_scratch_n = 0;
};

constexpr int kMaxDev = 16;
/* work-counter pairs for dynamically scheduled launches. A launch takes the next pair of the ring; the kernel's last CTA
 * leaves it zeroed, so a pair is only ever shared if more than kWorkRing launches are in flight on one device at once
 * (the driver's launch queue is far shorter). */
constexpr unsigned kWorkRing = 4096;
DeviceCtx g_dev[kMaxDev];
std::mutex g_mu;
std::mutex g_crc_mu;
CrcConsts g_consts;
bool g_consts_ready = false;
thread_local char g_err[256] = "";

int32_t fail(cudaError_t e, const char *what) {
    snprintf(g_err, sizeof(g_err), "%s: %s", what, cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? MZ_MEM_ERROR : MZ_INTERNAL_ERROR;
}
#define CK(call)                                       \
    do {                                               \
        cudaError_t e_ = (call);                       \
        if (e_ != cudaSuccess) return fail(e_, #call); \
    } while (0)

int32_t get_ctx(DeviceCtx **out) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) {
        snprintf(g_err, sizeof(g_err), "no CUDA device: %s", cudaGetErrorString(e));
        return MZ_SUPPORT_ERROR;
    }
    if (dev < 0 || dev >= kMaxDev) return MZ_PARAM_ERROR;
    DeviceCtx &c = g_dev[dev];
    if (!c.ready) {
        std::lock_guard<std::mutex> lk(g_mu);
        if (!c.ready) {
            if (!g_consts_ready) {
                crc_consts_init(g_consts);
                g_consts_ready = true;
            }
            cudaDeviceProp prop;
            CK(cudaGetDeviceProperties(&prop, dev));
            if (prop.major != 9 || prop.minor != 0) {
                snprintf(g_err, sizeof(g_err), "device %d is sm_%d%d; this library is built for sm_90a only", dev, prop.major, prop.minor);
                return MZ_SUPPORT_ERROR;
            }
            c.sm_count = prop.multiProcessorCount;
            CK(cudaMalloc(&c.d_consts, sizeof(CrcConsts)));
            CK(cudaMemcpy(c.d_consts, &g_consts, sizeof(CrcConsts), cudaMemcpyHostToDevice));
            CK(cudaFuncSetAttribute(deflate_chunks_kernel<2, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, DF_SMEM_BYTES));
            CK(cudaFuncSetAttribute(deflate_chunks_kernel<1, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, DF_SMEM_BYTES));
            CK(cudaFuncSetAttribute(deflate_chunks_kernel<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, DF_SMEM_BYTES));
            CK(cudaFuncSetAttribute(deflate_chunks_kernel<1, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, DFH_SMEM_BYTES));
            CK(cudaFuncSetAttribute(crc32_segments_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CRC_SMEM_BYTES));
            CK(cudaFuncSetAttribute(inflate_streams_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, INF_SMEM_BYTES));
            CK(cudaFuncSetAttribute(inflate_spec_resolve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SPEC_RESOLVE_SMEM));
            CK(cudaFuncSetAttribute(inflate_spec_compose_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SPEC_COMPOSE_SMEM));
            CK(cudaFuncSetAttribute(inflate_spec_link_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536));
            CK(cudaFuncSetAttribute(inflate_spec_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SPEC_MAX_SEGMENTS * 16));
            CK(cudaMalloc(&c.d_work, kWorkRing * 2 * sizeof(uint32_t)));
            CK(cudaMemset(c.d_work, 0, kWorkRing * 2 * sizeof(uint32_t)));
            c.ready = true;
        }
    }
    *out = &c;
    return MZ_OK;
}

uint64_t pick_crc_seg(uint64_t len, int sm_count) {
    /* aim for >= 4 segments per resident warp, segments between 4 KiB and 64 KiB */
    uint64_t warps = (uint64_t)sm_count * (CRC_THREADS / 32);
    uint64_t seg = 65536;
    while (seg > 4096 && len / seg < warps * 2) seg >>= 1;
    return seg;
}

/* the join's persistent grid: as many CTAs as are resident, and no more than one warp per slot */
uint32_t gather_grid(uint32_t nchunks, int sm_count) {
    const uint32_t need = (nchunks + GATHER_THREADS / 32 - 1) / (GATHER_THREADS / 32), resident = (uint32_t)sm_count * GATHER_CTAS_PER_SM;
    return need < resident ? need : resident;
}

} // namespace

extern "C" {

const char *mz_cuda_last_error(void) { return g_err; }

int32_t mz_cuda_init(void) {
    DeviceCtx *c;
    return get_ctx(&c);
}

int32_t mz_cuda_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

int32_t mz_cuda_set_device(int32_t ordinal) {
    CK(cudaSetDevice(ordinal));
    return MZ_OK;
}

int32_t mz_cuda_get_device(void) {
    int d = -1;
    if (cudaGetDevice(&d) != cudaSuccess) return -1;
    return d;
}

int32_t mz_cuda_sm_count(void) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    return err ? err : c->sm_count;
}

void *mz_cuda_malloc(size_t bytes) {
    void *p = nullptr;
    if (cudaMalloc(&p, bytes ? bytes : 16) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    return p;
}
void mz_cuda_free(void *p) {
    if (p) cudaFree(p);
}
void *mz_cuda_host_alloc(size_t bytes) {
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 16, cudaHostAllocDefault) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    return p;
}
void mz_cuda_host_free(void *p) {
    if (p) cudaFreeHost(p);
}
int32_t mz_cuda_memcpy_h2d(void *d, const void *h, size_t n, void *stream) {
    CK(cudaMemcpyAsync(d, h, n, cudaMemcpyHostToDevice, (cudaStream_t)stream));
    return MZ_OK;
}
int32_t mz_cuda_memcpy_d2h(void *h, const void *d, size_t n, void *stream) {
    CK(cudaMemcpyAsync(h, d, n, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    return MZ_OK;
}
int32_t mz_cuda_memcpy_d2d(void *d, const void *s, size_t n, void *stream) {
    CK(cudaMemcpyAsync(d, s, n, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return MZ_OK;
}
int32_t mz_cuda_host_is_pinned(const void *h) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, h) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return a.type == cudaMemoryTypeHost ? 1 : 0;
}
int32_t mz_cuda_memset(void *d, int v, size_t n, void *stream) {
    CK(cudaMemsetAsync(d, v, n, (cudaStream_t)stream));
    return MZ_OK;
}
int32_t mz_cuda_stream_sync(void *stream) {
    CK(cudaStreamSynchronize((cudaStream_t)stream));
    return MZ_OK;
}
void *mz_cuda_stream_create(void) {
    cudaStream_t s = nullptr;
    if (cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess) return nullptr;
    return s;
}
void mz_cuda_stream_destroy(void *s) {
    if (s) cudaStreamDestroy((cudaStream_t)s);
}
void *mz_cuda_event_create(void) {
    cudaEvent_t e = nullptr;
    if (cudaEventCreate(&e) != cudaSuccess) return nullptr;
    return e;
}
void mz_cuda_event_destroy(void *e) {
    if (e) cudaEventDestroy((cudaEvent_t)e);
}
int32_t mz_cuda_event_record(void *e, void *stream) {
    CK(cudaEventRecord((cudaEvent_t)e, (cudaStream_t)stream));
    return MZ_OK;
}
int32_t mz_cuda_event_sync(void *e) {
    CK(cudaEventSynchronize((cudaEvent_t)e));
    return MZ_OK;
}
int32_t mz_cuda_event_query(void *e) { /* 1 = everything recorded before it has finished, 0 = not yet, < 0 = error */
    const cudaError_t r = cudaEventQuery((cudaEvent_t)e);
    if (r == cudaSuccess) return 1;
    if (r == cudaErrorNotReady) {
        cudaGetLastError();
        return 0;
    }
    return fail(r, "cudaEventQuery");
}
float mz_cuda_event_elapsed_ms(void *a, void *b) {
    float ms = -1.f;
    if (cudaEventSynchronize((cudaEvent_t)b) != cudaSuccess) return -1.f;
    if (cudaEventElapsedTime(&ms, (cudaEvent_t)a, (cudaEvent_t)b) != cudaSuccess) return -1.f;
    return ms;
}

/* ---- CRC ------------------------------------------------------------------------------------------ */
int32_t mz_cuda_crc32_segments(const void *d_in, uint64_t total_len, uint64_t seg_size, const uint64_t *d_off, const uint32_t *d_len,
                               uint32_t nseg, uint32_t *d_residue, uint32_t *d_crc, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (nseg == 0) return MZ_OK;
    if (!d_residue || (!d_off && seg_size == 0) || (d_off && !d_len)) return MZ_PARAM_ERROR;
    CrcParams P;
    P.in = (const uint8_t *)d_in;
    P.in_off = d_off;
    P.in_len = d_len;
    P.total_len = total_len;
    P.seg_size = seg_size;
    P.nseg = nseg;
    P.consts = c->d_consts;
    P.out_residue = d_residue;
    P.out_crc = d_crc;
    P.init_len = d_off ? 0 : seg_size; /* every segment but perhaps the last has seg_size bytes */
    P.init = d_off ? 0u : crc_init_term(g_consts, seg_size);
    uint32_t warps_per_cta = CRC_THREADS / 32;
    uint32_t grid = (nseg + warps_per_cta - 1) / warps_per_cta;
    if (grid > (uint32_t)c->sm_count) grid = (uint32_t)c->sm_count;
    MZ_LAUNCH(crc32_segments_kernel, dim3(grid), dim3(CRC_THREADS), CRC_SMEM_BYTES, (cudaStream_t)stream, P);
    CK(cudaGetLastError());
    return MZ_OK;
}

int32_t mz_cuda_crc32_fold(const uint32_t *d_residue, uint32_t nseg, uint64_t seg_size, uint64_t total_len, uint32_t *d_out2, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    MZ_LAUNCH(crc32_fold_kernel, dim3(1), dim3(CRCF_THREADS), 0, (cudaStream_t)stream, d_residue, nseg, seg_size, total_len, c->d_consts, d_out2);
    CK(cudaGetLastError());
    return MZ_OK;
}

int32_t mz_cuda_crc32_device(const void *d_in, uint64_t len, uint32_t value, uint32_t *crc) {
    return mz_cuda_crc32_device_stream(d_in, len, value, crc, nullptr);
}

int32_t mz_cuda_crc32_device_stream(const void *d_in, uint64_t len, uint32_t value, uint32_t *crc, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (len == 0) {
        *crc = value;
        return MZ_OK;
    }
    uint64_t seg = pick_crc_seg(len, c->sm_count);
    uint64_t nseg64 = (len + seg - 1) / seg;
    while (nseg64 > 0x7fffffffull) {
        seg <<= 1;
        nseg64 = (len + seg - 1) / seg;
    }
    uint32_t nseg = (uint32_t)nseg64;
    /* the residue scratch is per device: threads sharing a device take turns for the whole operation */
    std::lock_guard<std::mutex> crc_turn(g_crc_mu);
    {
        std::lock_guard<std::mutex> lk(g_mu);
        if (c->crc_scratch_n < (size_t)nseg + 2) {
            if (c->d_crc_scratch) cudaFree(c->d_crc_scratch);
            c->d_crc_scratch = nullptr;
            c->crc_scratch_n = 0;
            CK(cudaMalloc(&c->d_crc_scratch, ((size_t)nseg + 2) * 4));
            c->crc_scratch_n = (size_t)nseg + 2;
        }
    }
    uint32_t *d_res = c->d_crc_scratch, *d_out2 = c->d_crc_scratch + nseg;
    err = mz_cuda_crc32_segments(d_in, len, seg, nullptr, nullptr, nseg, d_res, nullptr, stream);
    if (err) return err;
    err = mz_cuda_crc32_fold(d_res, nseg, seg, len, d_out2, stream);
    if (err) return err;
    uint32_t h[2];
    CK(cudaMemcpyAsync(h, d_out2, 8, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    CK(cudaStreamSynchronize((cudaStream_t)stream));
    /* chain the running value: crc(v, D) = ~((~v) x^(8|D|) + R(D)) */
    *crc = ~(gf2_mulmod(~value, gf2_xpow(g_consts.x2n, 8ull * len)) ^ h[0]);
    return MZ_OK;
}

uint32_t mz_cuda_crc32_combine(uint32_t crc_a, uint32_t crc_b, uint64_t len_b) {
    if (!g_consts_ready) {
        std::lock_guard<std::mutex> lk(g_mu);
        if (!g_consts_ready) {
            crc_consts_init(g_consts);
            g_consts_ready = true;
        }
    }
    if (len_b == 0) return crc_a; /* zlib's crc32_combine convention for the degenerate case */
    /* crc(A||B) = crc(A) x^(8|B|) + crc(B): the init/xorout terms cancel (both sides carry them once) */
    return gf2_mulmod(crc_a, gf2_xpow(g_consts.x2n, 8ull * len_b)) ^ crc_b;
}

/* ---- DEFLATE ---------------------------------------------------------------------------------------- */
uint64_t mz_cuda_deflate_slot_bound(uint32_t chunk_size) { return deflate_slot_bound(chunk_size); }

int32_t mz_cuda_deflate_chunks(const void *d_in, uint64_t total_len, uint32_t chunk_size, const uint64_t *d_off, const uint32_t *d_len,
                               const uint8_t *d_flags, uint32_t nchunks, uint32_t last_flags, int32_t level, void *d_slots,
                               uint64_t slot_stride, uint32_t *d_out_len, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (nchunks == 0) return MZ_OK;
    if (level < 0 || level > 9 || !d_slots || !d_out_len || (slot_stride & 15) || ((uintptr_t)d_slots & 15)) return MZ_PARAM_ERROR;
    if (!d_off) {
        if (chunk_size == 0 || chunk_size > MZ_CUDA_CHUNK_MAX || slot_stride < deflate_slot_bound(chunk_size)) return MZ_PARAM_ERROR;
        uint64_t need = total_len == 0 ? 1 : (total_len + chunk_size - 1) / chunk_size;
        if (need != nchunks) return MZ_PARAM_ERROR;
    } else if (!d_len) {
        return MZ_PARAM_ERROR;
    }
    DeflateParams P;
    P.in = (const uint8_t *)d_in;
    P.in_off = d_off;
    P.in_len = d_len;
    P.flags = d_flags;
    P.total_len = total_len;
    P.chunk_size = chunk_size;
    P.nchunks = nchunks;
    P.last_flags = last_flags;
    P.level = level;
    P.out = (uint8_t *)d_slots;
    P.slot_stride = slot_stride;
    P.out_len = d_out_len;
    {
        std::lock_guard<std::mutex> lk(g_mu);
        P.work_counter = c->d_work + 2 * (c->work_next++ % kWorkRing);
    }
    const uint32_t resident = (uint32_t)c->sm_count * 2u; /* two 512-thread CTAs of 111 KB shared memory per SM */
    uint32_t grid = nchunks < resident ? nchunks : resident;
    if (deflate_stride_for_level(level) == 2)
        MZ_LAUNCH((deflate_chunks_kernel<2, false>), dim3(grid), dim3(DF_THREADS), DF_SMEM_BYTES, (cudaStream_t)stream, P);
    else if (!deflate_lazy_for_level(level))
        MZ_LAUNCH((deflate_chunks_kernel<1, false>), dim3(grid), dim3(DF_THREADS), DF_SMEM_BYTES, (cudaStream_t)stream, P);
    else if (!deflate_hist_for_level(level))
        MZ_LAUNCH((deflate_chunks_kernel<1, true>), dim3(grid), dim3(DF_THREADS), DF_SMEM_BYTES, (cudaStream_t)stream, P);
    else { /* the history variant: 208 KiB of shared memory, one CTA per SM */
        const uint32_t grid1 = nchunks < (uint32_t)c->sm_count ? nchunks : (uint32_t)c->sm_count;
        MZ_LAUNCH((deflate_chunks_kernel<1, true, true>), dim3(grid1), dim3(DF_THREADS), DFH_SMEM_BYTES, (cudaStream_t)stream, P);
    }
    CK(cudaGetLastError());
    return MZ_OK;
}

#if defined(MZ_DF_PHASES) && !defined(MZ_EMU)
/* Only in the instrumented library (`make phases`): copy the deflate kernel's per-CTA phase counters, `rows` rows of DF_PH_COLS
 * u64 each (at most DF_PH_ROWS), to host memory and zero them on the device. Synchronises the device. */
int32_t mz_cuda_deflate_phases(uint64_t *host, uint32_t rows) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (!host || rows > (uint32_t)DF_PH_ROWS) return MZ_PARAM_ERROR;
    static unsigned long long zero[DF_PH_ROWS][DF_PH_COLS];
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpyFromSymbol(host, g_df_phases, (size_t)rows * DF_PH_COLS * sizeof(uint64_t)));
    CK(cudaMemcpyToSymbol(g_df_phases, zero, sizeof(zero)));
    return MZ_OK;
}
#endif

int32_t mz_cuda_concat(const void *d_slots, uint64_t slot_stride, const uint32_t *d_out_len, uint32_t nchunks, uint64_t *d_offsets,
                       void *d_dst, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    MZ_LAUNCH(scan_lengths_kernel, dim3(1), dim3(SCAN_THREADS), 0, (cudaStream_t)stream, d_out_len, nchunks, (uint64_t)0, d_offsets);
    if (nchunks) MZ_LAUNCH(gather_slots_kernel, dim3(gather_grid(nchunks, c->sm_count)), dim3(GATHER_THREADS), 0, (cudaStream_t)stream, (const uint8_t *)d_slots,
                           slot_stride, d_out_len, (const uint64_t *)d_offsets, nchunks, (uint8_t *)d_dst);
    CK(cudaGetLastError());
    return MZ_OK;
}

int32_t mz_cuda_gather(const void *d_slots, uint64_t slot_stride, const uint32_t *d_out_len, uint32_t nchunks, const uint64_t *d_offsets, void *d_dst,
                       void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (nchunks == 0) return MZ_OK;
    MZ_LAUNCH(gather_slots_kernel, dim3(gather_grid(nchunks, c->sm_count)), dim3(GATHER_THREADS), 0, (cudaStream_t)stream, (const uint8_t *)d_slots, slot_stride,
              d_out_len, d_offsets, nchunks, (uint8_t *)d_dst);
    CK(cudaGetLastError());
    return MZ_OK;
}

int32_t mz_cuda_scatter_blobs(const void *d_blob, const uint32_t *d_blob_off, const uint64_t *d_dst_off, uint32_t n, void *d_dst, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (n == 0) return MZ_OK;
    uint32_t grid = (n + 7) / 8;
    if (grid > (uint32_t)c->sm_count * 8u) grid = (uint32_t)c->sm_count * 8u;
    MZ_LAUNCH(scatter_blobs_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, (const uint8_t *)d_blob, d_blob_off, d_dst_off, n, (uint8_t *)d_dst);
    CK(cudaGetLastError());
    return MZ_OK;
}

int32_t mz_cuda_inflate_streams(const mz_cuda_inflate_job *d_jobs, mz_cuda_inflate_state *d_states, uint32_t nstreams, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (nstreams == 0) return MZ_OK;
    uint32_t maxgrid = (uint32_t)c->sm_count * 32u; /* 32 single-warp CTAs (6.4 KB of tables each) per SM */
    uint32_t grid = nstreams < maxgrid ? nstreams : maxgrid;
    uint32_t *counter;
    {
        std::lock_guard<std::mutex> lk(g_mu);
        counter = c->d_work + 2 * (c->work_next++ % kWorkRing);
    }
    MZ_LAUNCH(inflate_streams_kernel, dim3(grid), dim3(INF_THREADS), INF_SMEM_BYTES, (cudaStream_t)stream, (const InflateJob *)d_jobs,
              (InflateState *)d_states, nstreams, counter);
    CK(cudaGetLastError());
    return MZ_OK;
}

/* ---- K9: zip entries ---------------------------------------------------------------------------------------- */
namespace {
int32_t zip_launch(const mz_cuda_zip_round *r, void *stream, int which) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (!r) return MZ_PARAM_ERROR;
    if (r->n == 0) return MZ_OK;
    if (!r->buf || !r->ent || !r->status || !r->data_off) return MZ_PARAM_ERROR;
    ZipRound R;
    memcpy(&R, r, sizeof(R));
    const uint32_t cap = (uint32_t)c->sm_count * 8u;
    if (which == 0) {
        if (!r->jobs || !r->seg_off || !r->seg_len || !r->seg_len64 || !r->salt || !r->coff || !r->clen) return MZ_PARAM_ERROR;
        MZ_LAUNCH(zip_locate_kernel, dim3((r->n + 255) / 256), dim3(256), 0, (cudaStream_t)stream, R);
    } else if (which == 1) {
        if (!r->out) return MZ_PARAM_ERROR;
        const uint32_t g = (r->n + 7) / 8;
        MZ_LAUNCH(zip_stored_kernel, dim3(g < cap ? g : cap), dim3(256), 0, (cudaStream_t)stream, R);
    } else {
        if (!r->states || !r->crc || !r->clen) return MZ_PARAM_ERROR;
        MZ_LAUNCH(zip_verify_kernel, dim3((r->n + 255) / 256), dim3(256), 0, (cudaStream_t)stream, R);
    }
    CK(cudaGetLastError());
    return MZ_OK;
}
} // namespace

int32_t mz_cuda_zip_locate(const mz_cuda_zip_round *r, void *stream) { return zip_launch(r, stream, 0); }
int32_t mz_cuda_zip_copy_stored(const mz_cuda_zip_round *r, void *stream) { return zip_launch(r, stream, 1); }
int32_t mz_cuda_zip_verify(const mz_cuda_zip_round *r, void *stream) { return zip_launch(r, stream, 2); }

/* ---- K10: the central directory on the device ------------------------------------------------------------------ */
extern "C++" {
namespace {
/* the parse's scratch (19 arrays at most, sized by the summaries read back between stages): freed when the call returns, after
 * the stream has drained. A fixed table, so nothing can throw through the C entry point. */
struct ZcScratch {
    cudaStream_t s;
    void *p[24];
    int n = 0;
    explicit ZcScratch(cudaStream_t st) : s(st) {}
    ~ZcScratch() {
        cudaStreamSynchronize(s);
        for (int i = 0; i < n; i++) cudaFree(p[i]);
    }
    template <class T> T *get(uint64_t cnt) {
        void *q = nullptr;
        if (n == 24 || cudaMalloc(&q, cnt ? cnt * sizeof(T) : 16) != cudaSuccess) {
            cudaGetLastError();
            return nullptr;
        }
        p[n++] = q;
        return (T *)q;
    }
};

/* out[i] = in[0] + ... + in[i-1] for i = 0..n */
template <typename T> int32_t zc_scan(const T *in, uint64_t n, T *out, ZcScratch &w) {
    const uint64_t nb = n / ZC_TILE + 1;
    T *part = w.get<T>(nb);
    if (!part) return MZ_MEM_ERROR;
    MZ_LAUNCH(zc_scan_reduce_kernel<T>, dim3((uint32_t)nb), dim3(ZC_THREADS), 0, w.s, in, n, part);
    MZ_LAUNCH(zc_scan_parts_kernel<T>, dim3(1), dim3(ZC_THREADS), 0, w.s, part, (uint32_t)nb);
    MZ_LAUNCH(zc_scan_apply_kernel<T>, dim3((uint32_t)nb), dim3(ZC_THREADS), 0, w.s, in, n, (const T *)part, out);
    CK(cudaGetLastError());
    return MZ_OK;
}

int32_t zc_read_summary(ZcSummary *h, const ZcSummary *d, cudaStream_t s) {
    CK(cudaMemcpyAsync(h, d, sizeof(*h), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return MZ_OK;
}

uint32_t zc_grid(uint64_t n) { return (uint32_t)((n + ZC_THREADS - 1) / ZC_THREADS); }
} // namespace
} // extern "C++"

int32_t mz_cuda_zip_parse_directory(const void *d_archive, uint64_t len, mz_cuda_zip_dir *dir, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (!dir || (!d_archive && len)) return MZ_PARAM_ERROR;
    const cudaStream_t s = (cudaStream_t)stream;
    const uint8_t *buf = (const uint8_t *)d_archive;
    dir->err = dir->refuse = MZ_OK;
    dir->count = dir->njobs = dir->nsha = 0;
    dir->cd_off = dir->out_bytes = dir->bytes_in = dir->bytes_out = 0;
    memset(dir->na, 0, sizeof(dir->na));
    memset(dir->max_clen, 0, sizeof(dir->max_clen));
    dir->ent = nullptr;
    dir->sha_expect = nullptr;
    ZcScratch w(s);
    ZcSummary h;
    memset(&h, 0, sizeof(h));
    h.refuse_idx = 0xffffffffu;
    ZcSummary *S = w.get<ZcSummary>(1);
    if (!S) return MZ_MEM_ERROR;
    CK(cudaMemcpyAsync(S, &h, sizeof(h), cudaMemcpyHostToDevice, s));
    /* 1. end records */
    MZ_LAUNCH(zc_end_kernel, dim3(1), dim3(ZC_THREADS), 0, s, buf, len, S);
    CK(cudaGetLastError());
    if ((err = zc_read_summary(&h, S, s))) return err;
    if (h.err) {
        dir->err = h.err;
        return MZ_OK;
    }
    dir->cd_off = h.cd_off;
    const uint64_t cd_size = h.cd_size, count = h.count;
    /* Candidate ranks, the word prefix and the candidate count are 32-bit. Two PK\1\2 signatures cannot overlap (no proper suffix of
     * the signature is a prefix of it), so candidates lie at least 4 bytes apart and a directory below 16 GiB has fewer than
     * 2^32 - 2 of them: every rank stays below ZC_BRK. */
    if (cd_size >= (1ull << 34)) return MZ_SUPPORT_ERROR;
    const uint8_t *cd = buf + h.cd_off;
    /* 2. candidates */
    const uint64_t W = (cd_size + 31) / 32;
    uint32_t ncand = 0, *bits = nullptr, *wpre = nullptr;
    if (cd_size) {
        uint32_t *wcount = w.get<uint32_t>(W);
        bits = w.get<uint32_t>(W);
        wpre = w.get<uint32_t>(W + 1);
        if (!wcount || !bits || !wpre) return MZ_MEM_ERROR;
        MZ_LAUNCH(zc_cand_kernel, dim3(zc_grid(cd_size)), dim3(ZC_THREADS), 0, s, cd, cd_size, bits, wcount);
        CK(cudaGetLastError());
        if ((err = zc_scan(wcount, W, wpre, w))) return err;
        CK(cudaMemcpyAsync(&ncand, wpre + W, 4, cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
    }
    /* 3. the chain from the first record */
    const uint32_t slots = (uint32_t)(count < ncand ? count : ncand);
    uint64_t *rpos = nullptr;
    if (ncand) {
        uint64_t *cpos = w.get<uint64_t>(ncand);
        uint32_t *succ = w.get<uint32_t>(ncand), *ja = w.get<uint32_t>(ncand), *jb = w.get<uint32_t>(ncand), *mark = w.get<uint32_t>(ncand);
        uint32_t *midx = w.get<uint32_t>((uint64_t)ncand + 1);
        rpos = w.get<uint64_t>(slots);
        if (!cpos || !succ || !ja || !jb || !mark || !midx || !rpos) return MZ_MEM_ERROR;
        MZ_LAUNCH(zc_link_kernel, dim3(zc_grid(cd_size)), dim3(ZC_THREADS), 0, s, cd, cd_size, (const uint32_t *)bits, (const uint32_t *)wpre, cpos, succ,
                  ja, mark);
        for (uint32_t k = 0; (1ull << k) < ncand; k++) {
            MZ_LAUNCH(zc_double_kernel, dim3(zc_grid(ncand)), dim3(ZC_THREADS), 0, s, ncand, mark, (const uint32_t *)ja, jb);
            std::swap(ja, jb);
        }
        CK(cudaGetLastError());
        if ((err = zc_scan(mark, ncand, midx, w))) return err;
        MZ_LAUNCH(zc_place_kernel, dim3(zc_grid(ncand)), dim3(ZC_THREADS), 0, s, ncand, (const uint32_t *)mark, (const uint32_t *)midx,
                  (const uint64_t *)cpos, (const uint32_t *)succ, (uint64_t)slots, rpos, S);
        CK(cudaGetLastError());
        if ((err = zc_read_summary(&h, S, s))) return err;
    }
    /* where the chain itself ends the list, as the host loop would: a record that does not fit or has no signature, more records
     * than the end record counts, or fewer */
    const uint32_t n = (uint32_t)(h.nchain < count ? h.nchain : count);
    int32_t limit_code = MZ_OK;
    if (h.nchain == 0 ? cd_size != 0 : (h.nchain > count || h.term == ZC_BRK || h.nchain < count)) limit_code = MZ_FORMAT_ERROR;
    /* 4. records */
    ZcRec *rec = nullptr;
    uint64_t *roff = nullptr;
    ZcCount *pre = nullptr;
    if (n) {
        ZcCount *cnt = w.get<ZcCount>(n);
        rec = w.get<ZcRec>(n);
        roff = w.get<uint64_t>(n);
        pre = w.get<ZcCount>((uint64_t)n + 1);
        if (!cnt || !rec || !roff || !pre) return MZ_MEM_ERROR;
        MZ_LAUNCH(zc_records_kernel, dim3(zc_grid(n)), dim3(ZC_THREADS), 0, s, buf, h.cd_off, h.shift, (const uint64_t *)rpos, n, dir->have_password,
                  dir->password_long, rec, roff, cnt, S);
        CK(cudaGetLastError());
        if ((err = zc_scan(cnt, n, pre, w))) return err;
        MZ_LAUNCH(zc_finish_kernel, dim3(zc_grid(n)), dim3(ZC_THREADS), 0, s, (const ZcRec *)rec, (const uint64_t *)roff, (const ZcCount *)pre, n,
                  limit_code, S);
        CK(cudaGetLastError());
        if ((err = zc_read_summary(&h, S, s))) return err;
    } else {
        h.nacc = 0;
        h.refuse = limit_code;
    }
    const uint32_t m = h.nacc;
    dir->count = m;
    dir->refuse = h.refuse;
    dir->out_bytes = h.out;
    dir->bytes_in = h.cin;
    dir->bytes_out = h.cout;
    dir->njobs = h.job;
    dir->nsha = h.sha;
    for (int k = 0; k < 4; k++) {
        dir->na[k] = h.a[k];
        dir->max_clen[k] = h.max_clen[k];
    }
    const bool fits = dir->max_entries >= m && (!dir->decode || dir->out_cap >= h.out); /* otherwise MZ_BUF_ERROR: nothing listed */
    const bool own = fits && !dir->entries && dir->alloc_entries && m;
    if (own) CK(cudaMalloc(&dir->entries, (size_t)m * sizeof(ZipDevEnt)));
    const bool pub = fits && dir->entries, dec = fits && dir->decode;
    if (!m || (!pub && !dec)) return MZ_OK;
    /* 5. extents, tables */
    const uint64_t *key = roff;
    if (h.unsorted) {
        if (m > (1u << 31)) return MZ_SUPPORT_ERROR;
        uint32_t np = 1;
        while (np < m) np <<= 1;
        uint64_t *sorted = w.get<uint64_t>(np);
        if (!sorted) return MZ_MEM_ERROR;
        MZ_LAUNCH(zc_pad_kernel, dim3(zc_grid(np)), dim3(ZC_THREADS), 0, s, (const uint64_t *)roff, m, sorted, np);
        for (uint64_t k = 2; k <= np; k <<= 1)
            for (uint32_t j = (uint32_t)(k >> 1); j; j >>= 1) MZ_LAUNCH(zc_bitonic_kernel, dim3(zc_grid(np)), dim3(ZC_THREADS), 0, s, sorted, np, (uint32_t)k, j);
        CK(cudaGetLastError());
        key = sorted;
    }
    ZipEnt *ent = nullptr;
    uint8_t *sha = nullptr;
    if (dec) {
        CK(cudaMalloc(&ent, (size_t)m * sizeof(ZipEnt)));
        if (cudaMalloc(&sha, (size_t)(h.sha ? h.sha : 1) * 32) != cudaSuccess) {
            cudaFree(ent);
            return fail(cudaErrorMemoryAllocation, "cudaMalloc");
        }
    }
    MZ_LAUNCH(zc_fill_kernel, dim3(zc_grid(m)), dim3(ZC_THREADS), 0, s, (const ZcRec *)rec, (const ZcCount *)pre, key, m, h.cd_off, buf,
              pub ? (ZipDevEnt *)dir->entries : nullptr, ent, sha);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        cudaFree(ent);
        cudaFree(sha);
        return fail(e, "zc_fill_kernel");
    }
    dir->ent = (mz_cuda_zip_ent *)ent;
    dir->sha_expect = sha;
    return MZ_OK;
}

int32_t mz_cuda_zip_statuses(const uint32_t *d_status, uint32_t n, void *d_entries, uint32_t *d_first, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (n == 0) return MZ_OK;
    if (!d_status || !d_entries || !d_first) return MZ_PARAM_ERROR;
    MZ_LAUNCH(zc_status_kernel, dim3(zc_grid(n)), dim3(ZC_THREADS), 0, (cudaStream_t)stream, d_status, n, (ZipDevEnt *)d_entries, d_first);
    CK(cudaGetLastError());
    return MZ_OK;
}

/* ---- K11: a zip archive written into device memory -------------------------------------------------------------- */
extern "C++" {
namespace {
ZwCall zw_call(const mz_cuda_zip_wr *w) {
    ZwCall W;
    memcpy(&W, w, sizeof(W));
    return W;
}
/* out[i] = in[0] + ... + in[i-1] for i = 0..n, with the tiles' sums in part (n / ZC_TILE + 1 of them) */
template <typename T> int32_t zw_scan(const T *in, uint64_t n, T *out, T *part, cudaStream_t s) {
    const uint64_t nb = n / ZC_TILE + 1;
    MZ_LAUNCH(zc_scan_reduce_kernel<T>, dim3((uint32_t)nb), dim3(ZC_THREADS), 0, s, in, n, part);
    MZ_LAUNCH(zc_scan_parts_kernel<T>, dim3(1), dim3(ZC_THREADS), 0, s, part, (uint32_t)nb);
    MZ_LAUNCH(zc_scan_apply_kernel<T>, dim3((uint32_t)nb), dim3(ZC_THREADS), 0, s, in, n, (const T *)part, out);
    CK(cudaGetLastError());
    return MZ_OK;
}
} // namespace
} // extern "C++"

int32_t mz_cuda_zip_wr_items(const mz_cuda_zip_wr *w, uint32_t data_null, uint32_t names_null, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (!w || !w->cnt || !w->pre || !w->part || !w->bad || (w->n && !w->items)) return MZ_PARAM_ERROR;
    const ZwCall W = zw_call(w);
    const cudaStream_t s = (cudaStream_t)stream;
    if (W.n) MZ_LAUNCH(zw_items_kernel, dim3((W.n + ZW_THREADS - 1) / ZW_THREADS), dim3(ZW_THREADS), 0, s, W, data_null, names_null);
    CK(cudaGetLastError());
    return zw_scan<ZwCount>(W.cnt, W.n, W.pre, (ZwCount *)W.part, s);
}

int32_t mz_cuda_zip_wr_chunks(const mz_cuda_zip_wr *w, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (!w || !w->c_off || !w->c_len || !w->c_flags || !w->c_item || (w->sha && (!w->e_off || !w->e_len))) return MZ_PARAM_ERROR;
    if (w->nch == 0) return MZ_OK;
    const uint64_t g = (w->nch + ZW_THREADS - 1) / ZW_THREADS;
    if (g > 0x7fffffffull) return MZ_SUPPORT_ERROR;
    MZ_LAUNCH(zw_chunks_kernel, dim3((uint32_t)g), dim3(ZW_THREADS), 0, (cudaStream_t)stream, zw_call(w));
    CK(cudaGetLastError());
    return MZ_OK;
}

int32_t mz_cuda_zip_wr_place(const mz_cuda_zip_wr *w, uint64_t c0, uint32_t m, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (!w || !w->out_len || !w->S || !w->dst || !w->glen || !w->part || m > 32768u || c0 + m > w->nch) return MZ_PARAM_ERROR;
    if (m == 0) return MZ_OK;
    const cudaStream_t s = (cudaStream_t)stream;
    const uint32_t nb = m / ZC_TILE + 1;
    uint32_t *part = (uint32_t *)w->part;
    /* the round's stream bytes fit 32 bits: at most 32768 chunks of mz_cuda_deflate_slot_bound(65536) each */
    MZ_LAUNCH(zc_scan_reduce_kernel<uint32_t>, dim3(nb), dim3(ZC_THREADS), 0, s, (const uint32_t *)w->out_len + c0, (uint64_t)m, part);
    MZ_LAUNCH(zc_scan_parts_kernel<uint32_t>, dim3(1), dim3(ZC_THREADS), 0, s, part, nb);
    MZ_LAUNCH(zw_place_kernel, dim3(nb), dim3(ZC_THREADS), 0, s, zw_call(w), c0, m, (const uint32_t *)part);
    CK(cudaGetLastError());
    return MZ_OK;
}

int32_t mz_cuda_zip_wr_entries(const mz_cuda_zip_wr *w, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (!w || !w->e_lh || !w->e_csize || !w->e_cd || !w->e_cdpre || !w->e_coff || !w->e_crc || !w->max_csize || !w->residue || !w->S) return MZ_PARAM_ERROR;
    const ZwCall W = zw_call(w);
    const cudaStream_t s = (cudaStream_t)stream;
    const uint32_t per = ZW_THREADS / 32;
    if (W.n) MZ_LAUNCH(zw_entries_kernel, dim3((W.n + per - 1) / per), dim3(ZW_THREADS), 0, s, W, (const CrcConsts *)c->d_consts);
    CK(cudaGetLastError());
    return zw_scan<uint64_t>(W.e_cd, W.n, W.e_cdpre, (uint64_t *)W.part, s);
}

int32_t mz_cuda_zip_wr_emit(const mz_cuda_zip_wr *w, uint64_t cd_off, uint64_t cd_size, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (!w || !w->archive || (w->sha && !w->digest) || (w->aes && (!w->salt || !w->keys || !w->mac))) return MZ_PARAM_ERROR;
    const ZwCall W = zw_call(w);
    const cudaStream_t s = (cudaStream_t)stream;
    const uint32_t per = ZW_THREADS / 32;
    if (W.n) MZ_LAUNCH(zw_emit_kernel, dim3((W.n + per - 1) / per), dim3(ZW_THREADS), 0, s, W, cd_off);
    MZ_LAUNCH(zw_end_kernel, dim3(1), dim3(ZW_THREADS), 0, s, W, cd_off, cd_size);
    CK(cudaGetLastError());
    return MZ_OK;
}

/* ---- K13: an archive in device memory updated on the device ------------------------------------------------------ */
extern "C++" {
namespace {
ZuCall zu_call(const mz_cuda_zip_up *u) {
    ZuCall U;
    memcpy(&U, u, sizeof(U));
    return U;
}
} // namespace
} // extern "C++"

int32_t mz_cuda_zip_up_counts(const mz_cuda_zip_up *u, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (!u || !u->cnt || !u->pre || !u->part || !u->info || !u->src || (u->n && (!u->dir || (u->count && !u->ent)))) return MZ_PARAM_ERROR;
    const ZuCall U = zu_call(u);
    const cudaStream_t s = (cudaStream_t)stream;
    const uint32_t g = (U.n + ZU_THREADS - 1) / ZU_THREADS;
    if (U.n) MZ_LAUNCH(zu_counts_kernel, dim3(g), dim3(ZU_THREADS), 0, s, U);
    CK(cudaGetLastError());
    if ((err = zw_scan<ZuCount>(U.cnt, U.n, U.pre, (ZuCount *)U.part, s))) return err;
    if (U.n) MZ_LAUNCH(zu_layout_kernel, dim3(g), dim3(ZU_THREADS), 0, s, U);
    MZ_LAUNCH(zu_comment_kernel, dim3(1), dim3(ZU_THREADS), 0, s, U);
    CK(cudaGetLastError());
    return MZ_OK;
}

int32_t mz_cuda_zip_up_copy(const mz_cuda_zip_up *u, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (!u || !u->pre || !u->archive || (u->n && (!u->src || (u->count && !u->ent)))) return MZ_PARAM_ERROR;
    if (u->n == 0) return MZ_OK;
    const uint32_t per = ZU_THREADS / 32, g = (u->n + per - 1) / per, cap = (uint32_t)c->sm_count * 8u;
    MZ_LAUNCH(zu_copy_kernel, dim3(g < cap ? g : cap), dim3(ZU_THREADS), 0, (cudaStream_t)stream, zu_call(u));
    CK(cudaGetLastError());
    return MZ_OK;
}

int32_t mz_cuda_zip_up_records(const mz_cuda_zip_up *u, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (!u || !u->pre || !u->info || !u->archive || (u->n && (!u->dir || (u->count && !u->ent)))) return MZ_PARAM_ERROR;
    if (u->n == 0) return MZ_OK;
    const uint32_t per = ZU_THREADS / 32;
    MZ_LAUNCH(zu_records_kernel, dim3((u->n + per - 1) / per), dim3(ZU_THREADS), 0, (cudaStream_t)stream, zu_call(u));
    CK(cudaGetLastError());
    return MZ_OK;
}

/* ---- K12: random access to an archive in device memory ----------------------------------------------------------- */
int32_t mz_cuda_zip_name_index(const void *d_archive, const void *d_entries, uint32_t n, uint64_t *d_table, uint32_t P, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (n == 0) return MZ_OK;
    if (!d_archive || !d_entries || !d_table || P < 2ull * n || (P & (P - 1))) return MZ_PARAM_ERROR;
    MZ_LAUNCH(zs_index_kernel, dim3((n + ZS_THREADS - 1) / ZS_THREADS), dim3(ZS_THREADS), 0, (cudaStream_t)stream, (const uint8_t *)d_archive,
              (const ZipDevEnt *)d_entries, n, (unsigned long long *)d_table, P);
    CK(cudaGetLastError());
    return MZ_OK;
}

int32_t mz_cuda_zip_name_lookup(const void *d_archive, const void *d_entries, const uint64_t *d_table, uint32_t P, const void *d_names,
                                const uint64_t *d_name_off, const uint32_t *d_name_len, uint32_t nq, uint8_t ignore_case, uint32_t *d_index,
                                void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (nq == 0) return MZ_OK;
    if (!d_names || !d_name_off || !d_name_len || !d_index || (P & (P - 1)) || (P && (!d_archive || !d_entries || !d_table))) return MZ_PARAM_ERROR;
    MZ_LAUNCH(zs_lookup_kernel, dim3((nq + ZS_THREADS - 1) / ZS_THREADS), dim3(ZS_THREADS), 0, (cudaStream_t)stream, (const uint8_t *)d_archive,
              (const ZipDevEnt *)d_entries, (const unsigned long long *)d_table, P, (const uint8_t *)d_names, d_name_off, d_name_len, nq,
              (uint32_t)(ignore_case != 0), d_index);
    CK(cudaGetLastError());
    return MZ_OK;
}

extern "C++" {
namespace {
ZsCall zs_call(const mz_cuda_zip_sel *c) {
    ZsCall C;
    memcpy(&C, c, sizeof(C));
    return C;
}
} // namespace
} // extern "C++"

int32_t mz_cuda_zip_sel_counts(const mz_cuda_zip_sel *sc, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (!sc || !sc->cnt || !sc->pre || !sc->part || (sc->n && (!sc->select || (sc->count && !sc->ent)))) return MZ_PARAM_ERROR;
    const ZsCall C = zs_call(sc);
    const cudaStream_t s = (cudaStream_t)stream;
    if (C.n) MZ_LAUNCH(zs_count_kernel, dim3((C.n + ZS_THREADS - 1) / ZS_THREADS), dim3(ZS_THREADS), 0, s, C);
    CK(cudaGetLastError());
    return zw_scan<ZsCount>(C.cnt, C.n, C.pre, (ZsCount *)C.part, s);
}

int32_t mz_cuda_zip_sel_fill(const mz_cuda_zip_sel *sc, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (!sc || !sc->pre || (sc->sel && sc->n && (!sc->select || (sc->count && !sc->ent)))) return MZ_PARAM_ERROR;
    const ZsCall C = zs_call(sc);
    MZ_LAUNCH(zs_fill_kernel, dim3(C.n / ZS_THREADS + 1), dim3(ZS_THREADS), 0, (cudaStream_t)stream, C);
    CK(cudaGetLastError());
    return MZ_OK;
}

int32_t mz_cuda_zip_sel_gather(const mz_cuda_zip_sel *sc, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (!sc || !sc->pre || (sc->n && (!sc->select || !sc->archive || !sc->scratch || (sc->count && !sc->ent)))) return MZ_PARAM_ERROR;
    if (sc->n == 0) return MZ_OK;
    const uint32_t per = ZS_THREADS / 32, g = (sc->n + per - 1) / per, cap = (uint32_t)c->sm_count * 8u;
    MZ_LAUNCH(zs_gather_kernel, dim3(g < cap ? g : cap), dim3(ZS_THREADS), 0, (cudaStream_t)stream, zs_call(sc));
    CK(cudaGetLastError());
    return MZ_OK;
}

int32_t mz_cuda_zip_sel_status(const uint32_t *d_status, const uint32_t *d_select, uint32_t n, uint32_t count, int32_t *d_out, uint64_t *d_first,
                               void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (n == 0) return MZ_OK;
    if (!d_status || !d_select || !d_first) return MZ_PARAM_ERROR;
    MZ_LAUNCH(zs_status_kernel, dim3((n + ZS_THREADS - 1) / ZS_THREADS), dim3(ZS_THREADS), 0, (cudaStream_t)stream, d_status, d_select, n, count,
              d_out, (unsigned long long *)d_first);
    CK(cudaGetLastError());
    return MZ_OK;
}

/* ---- K14: a gzip member written into device memory ---------------------------------------------------------------- */
int32_t mz_cuda_gzip_place(const uint32_t *d_out_len, uint64_t c0, uint32_t m, uint64_t *d_S, uint64_t *d_dst, uint32_t *d_glen, uint64_t head,
                           uint64_t cap, uint32_t *d_part, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (!d_out_len || !d_S || !d_dst || !d_glen || !d_part || m > 32768u) return MZ_PARAM_ERROR;
    if (m == 0) return MZ_OK;
    const cudaStream_t s = (cudaStream_t)stream;
    const uint32_t nb = m / ZC_TILE + 1;
    /* the round's stream bytes fit 32 bits: at most 32768 chunks of mz_cuda_deflate_slot_bound(65536) each */
    MZ_LAUNCH(zc_scan_reduce_kernel<uint32_t>, dim3(nb), dim3(ZC_THREADS), 0, s, d_out_len + c0, (uint64_t)m, d_part);
    MZ_LAUNCH(zc_scan_parts_kernel<uint32_t>, dim3(1), dim3(ZC_THREADS), 0, s, d_part, nb);
    MZ_LAUNCH(gz_place_kernel, dim3(nb), dim3(ZC_THREADS), 0, s, d_out_len, c0, m, (const uint32_t *)d_part, d_S, d_dst, d_glen, head, cap);
    CK(cudaGetLastError());
    return MZ_OK;
}

int32_t mz_cuda_gzip_trailer(const uint64_t *d_S_end, const uint32_t *d_crc, uint64_t len, uint64_t head, void *d_out, uint64_t cap,
                             uint64_t *d_total, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (!d_S_end || !d_crc || !d_total || (!d_out && cap)) return MZ_PARAM_ERROR;
    MZ_LAUNCH(gz_trailer_kernel, dim3(1), dim3(32), 0, (cudaStream_t)stream, d_S_end, d_crc, len, head, (uint8_t *)d_out, cap, d_total);
    CK(cudaGetLastError());
    return MZ_OK;
}

/* workspace carving for K6 (all pieces 256-byte aligned) */
static inline uint64_t al256(uint64_t v) { return (v + 255) & ~255ull; }
uint64_t mz_cuda_inflate_spec_workspace_bytes(uint32_t max_segments) {
    const uint64_t m = max_segments;
    return al256(m * sizeof(SpecSeg)) + al256(m * sizeof(InflateState)) + al256(m * 8) + al256(m * SPEC_RING * 2) + al256(m * 32768) + al256((uint64_t)SPEC_GROUPS * 65536) +
           al256((uint64_t)SPEC_GROUPS * 32768) + 256 + 256;
}

int32_t mz_cuda_inflate_spec_round(const void *d_in, uint64_t in_base, uint64_t in_avail, uint32_t in_final, uint64_t start_bit,
                                   uint64_t seg_bytes, uint32_t nseg, void *d_out, uint64_t out_base, uint64_t out_pos,
                                   uint64_t out_end, void *d_workspace, uint32_t max_segments, mz_cuda_spec_summary *d_summary,
                                   void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (nseg == 0 || nseg > max_segments || max_segments > SPEC_MAX_SEGMENTS || seg_bytes < 64 || ((uintptr_t)d_in & 3) || !d_workspace || !d_summary) return MZ_PARAM_ERROR;
    SpecParams P;
    P.in = (const uint8_t *)d_in;
    P.in_base = in_base;
    P.in_avail = in_avail;
    P.start_bit = start_bit;
    P.seg_bits = seg_bytes * 8;
    P.out = (uint8_t *)d_out;
    P.out_base = out_base;
    P.out_pos = out_pos;
    P.out_end = out_end;
    P.in_final = in_final;
    P.nseg = nseg;
    uint8_t *w = (uint8_t *)(((uintptr_t)d_workspace + 255) & ~(uintptr_t)255);
    const uint64_t m = max_segments;
    P.seg = (SpecSeg *)w;            w += al256(m * sizeof(SpecSeg));
    P.states = (InflateState *)w;    w += al256(m * sizeof(InflateState));
    P.chain = (uint32_t *)w;         w += al256(m * 8);
    P.rings = (uint16_t *)w;         w += al256(m * SPEC_RING * 2);
    P.wins = w;                      w += al256(m * 32768);
    P.gmaps = (uint16_t *)w;         w += al256((uint64_t)SPEC_GROUPS * 65536);
    P.gwins = w;                     w += al256((uint64_t)SPEC_GROUPS * 32768);
    P.work = (uint32_t *)w;
    P.summary = (SpecSummary *)d_summary;
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t maxgrid = (uint32_t)c->sm_count * 32u;
    const uint32_t grid = nseg < maxgrid ? nseg : maxgrid;
    CK(cudaMemsetAsync(P.work, 0, 16, s));
    const bool trace = getenv("MZ_CUDA_TRACE") != nullptr; /* per-kernel times of the round on stderr (debug aid, serialises) */
    cudaEvent_t ev[6];
    if (trace)
        for (int i = 0; i < 6; i++) CK(cudaEventCreate(&ev[i]));
    if (trace) CK(cudaEventRecord(ev[0], s));
    MZ_LAUNCH(inflate_spec_find_kernel, dim3(grid), dim3(INF_THREADS), SPEC_FIND_SMEM, s, P);
    if (trace) CK(cudaEventRecord(ev[1], s));
    MZ_LAUNCH(inflate_spec_scan_kernel, dim3(grid), dim3(INF_THREADS), INF_SMEM_BYTES, s, P);
    if (trace) CK(cudaEventRecord(ev[2], s));
    MZ_LAUNCH(inflate_spec_chain_kernel, dim3(1), dim3(SPEC_CHAIN_THREADS), (size_t)nseg * 16, s, P);
    if (trace) CK(cudaEventRecord(ev[3], s));
    MZ_LAUNCH(inflate_spec_compose_kernel, dim3(SPEC_GROUPS), dim3(SPEC_RESOLVE_THREADS), SPEC_COMPOSE_SMEM, s, P);
    MZ_LAUNCH(inflate_spec_link_kernel, dim3(1), dim3(SPEC_RESOLVE_THREADS), 65536, s, P);
    MZ_LAUNCH(inflate_spec_resolve_kernel, dim3(SPEC_GROUPS), dim3(SPEC_RESOLVE_THREADS), SPEC_RESOLVE_SMEM, s, P);
    if (trace) CK(cudaEventRecord(ev[4], s));
    MZ_LAUNCH(inflate_spec_emit_kernel, dim3(grid), dim3(INF_THREADS), INF_SMEM_BYTES, s, P);
    if (trace) CK(cudaEventRecord(ev[5], s));
    CK(cudaGetLastError());
    if (trace) {
        CK(cudaEventSynchronize(ev[5]));
        float t[5];
        for (int i = 0; i < 5; i++) CK(cudaEventElapsedTime(&t[i], ev[i], ev[i + 1]));
        fprintf(stderr, "mz_cuda: K6 kernels ms: find %.3f scan %.3f chain %.3f compose+link+resolve %.3f emit %.3f (%u segments)\n", t[0], t[1], t[2], t[3], t[4], nseg);
        for (int i = 0; i < 6; i++) cudaEventDestroy(ev[i]);
    }
    return MZ_OK;
}

int32_t mz_cuda_sha256_batch(const void *d_in, const uint64_t *d_off, const uint64_t *d_len, uint32_t n, void *d_digest, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    if (n == 0) return MZ_OK;
    if (!d_in || !d_off || !d_len || !d_digest || ((uintptr_t)d_digest & 3)) return MZ_PARAM_ERROR;
    Sha256Params P;
    P.in = (const uint8_t *)d_in;
    P.off = d_off;
    P.len = d_len;
    P.n = n;
    P.digest = (uint8_t *)d_digest;
    uint32_t blocks = (n + SHA_THREADS - 1) / SHA_THREADS;
    const uint32_t cap = (uint32_t)c->sm_count * 16u;
    if (blocks > cap) blocks = cap;
    MZ_LAUNCH(sha256_batch_kernel, dim3(blocks), dim3(SHA_THREADS), 0, (cudaStream_t)stream, P);
    CK(cudaGetLastError());
    return MZ_OK;
}

/* ---- K8: WinZip AES for a batch of entries ------------------------------------------------------------------- */
namespace {
/* FIPS 197 4.2 / 5.1.1: S[x] = affine(inverse of x in GF(2^8) mod x^8 + x^4 + x^3 + x + 1); T[x] = (2 S, S, S, 3 S) */
int32_t aes_tables(DeviceCtx *c) {
    if (c->d_aes) return MZ_OK;
    std::lock_guard<std::mutex> lk(g_mu);
    if (c->d_aes) return MZ_OK;
    uint32_t h[256 + 64];
    uint8_t sbox[256];
    uint8_t p = 1, q = 1;
    do { /* p runs over the multiplicative group (generator 3), q over the inverses */
        p = (uint8_t)(p ^ (p << 1) ^ ((p & 0x80) ? 0x1b : 0));
        q ^= (uint8_t)(q << 1);
        q ^= (uint8_t)(q << 2);
        q ^= (uint8_t)(q << 4);
        if (q & 0x80) q ^= 0x09;
        const uint8_t x = (uint8_t)(q ^ (uint8_t)((q << 1) | (q >> 7)) ^ (uint8_t)((q << 2) | (q >> 6)) ^ (uint8_t)((q << 3) | (q >> 5)) ^ (uint8_t)((q << 4) | (q >> 4)));
        sbox[p] = (uint8_t)(x ^ 0x63);
    } while (p != 1);
    sbox[0] = 0x63;
    for (int i = 0; i < 256; i++) {
        const uint32_t s1 = sbox[i], s2 = ((s1 << 1) ^ ((s1 & 0x80) ? 0x11b : 0)) & 0xff, s3 = s2 ^ s1;
        h[i] = (s2 << 24) | (s1 << 16) | (s1 << 8) | s3;
    }
    memcpy(h + 256, sbox, 256);
    uint32_t *d = nullptr;
    CK(cudaMalloc(&d, sizeof(h)));
    CK(cudaMemcpy(d, h, sizeof(h), cudaMemcpyHostToDevice));
    c->d_aes = d;
    return MZ_OK;
}
bool wz_strength(uint32_t strength, uint32_t *key_len, uint32_t *salt_len) {
    if (strength < 1 || strength > 3) return false;
    *key_len = 8 * strength + 8;   /* MZ_AES_KEY_LENGTH, mz_strm_wzaes.c:19 */
    *salt_len = 4 * strength + 4;  /* MZ_AES_SALT_LENGTH, :21 */
    return true;
}
} // namespace

int32_t mz_cuda_wzaes_derive(const void *d_password, uint32_t pw_len, const void *d_salts, uint32_t n, uint32_t strength, void *d_keys, void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    WzDeriveParams P;
    if (!wz_strength(strength, &P.key_len, &P.salt_len) || pw_len > 128) return MZ_PARAM_ERROR;
    if (n == 0) return MZ_OK;
    if (!d_password || !d_salts || !d_keys) return MZ_PARAM_ERROR;
    P.password = (const uint8_t *)d_password;
    P.pw_len = pw_len;
    P.salts = (const uint8_t *)d_salts;
    P.iterations = 1000; /* MZ_AES_KEYING_ITERATIONS, mz_strm_wzaes.c:20 */
    P.n = n;
    P.keys = (uint8_t *)d_keys;
    const uint32_t threads = n * ((2 * P.key_len + 2 + 19) / 20);
    uint32_t blocks = (threads + 127) / 128;
    const uint32_t cap = (uint32_t)c->sm_count * 16u;
    if (blocks > cap) blocks = cap;
    MZ_LAUNCH(wzaes_derive_kernel, dim3(blocks), dim3(128), 0, (cudaStream_t)stream, P);
    CK(cudaGetLastError());
    return MZ_OK;
}

int32_t mz_cuda_wzaes_ctr(void *d_data, const uint64_t *d_off, const uint64_t *d_len, uint32_t n, uint64_t max_len, const void *d_keys, uint32_t strength,
                          void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    WzCtrParams P;
    uint32_t salt_len;
    if (!wz_strength(strength, &P.key_len, &salt_len)) return MZ_PARAM_ERROR;
    if (n == 0 || max_len == 0) return MZ_OK;
    if (!d_data || !d_off || !d_len || !d_keys) return MZ_PARAM_ERROR;
    err = aes_tables(c);
    if (err) return err;
    P.data = (uint8_t *)d_data;
    P.off = d_off;
    P.len = d_len;
    P.n = n;
    P.parts = (uint32_t)((max_len + WZ_CTR_PART - 1) / WZ_CTR_PART);
    if (P.parts > 65535) return MZ_PARAM_ERROR; /* entries up to 4 GiB */
    P.keys = (const uint8_t *)d_keys;
    P.te0 = c->d_aes;
    P.sbox = (const uint8_t *)(c->d_aes + 256);
    const uint32_t gx = n < (uint32_t)c->sm_count * 64u ? n : (uint32_t)c->sm_count * 64u;
    MZ_LAUNCH(wzaes_ctr_kernel, dim3(gx, P.parts), dim3(WZ_CTR_THREADS), 0, (cudaStream_t)stream, P);
    CK(cudaGetLastError());
    return MZ_OK;
}

int32_t mz_cuda_wzaes_hmac(const void *d_data, const uint64_t *d_off, const uint64_t *d_len, uint32_t n, const void *d_keys, uint32_t strength, void *d_mac,
                           void *stream) {
    DeviceCtx *c;
    int32_t err = get_ctx(&c);
    if (err) return err;
    WzHmacParams P;
    uint32_t salt_len;
    if (!wz_strength(strength, &P.key_len, &salt_len)) return MZ_PARAM_ERROR;
    if (n == 0) return MZ_OK;
    if (!d_data || !d_off || !d_len || !d_keys || !d_mac) return MZ_PARAM_ERROR;
    P.data = (const uint8_t *)d_data;
    P.off = d_off;
    P.len = d_len;
    P.n = n;
    P.keys = (const uint8_t *)d_keys;
    P.mac = (uint8_t *)d_mac;
    uint32_t blocks = (n + 127) / 128;
    const uint32_t cap = (uint32_t)c->sm_count * 16u;
    if (blocks > cap) blocks = cap;
    MZ_LAUNCH(wzaes_hmac_kernel, dim3(blocks), dim3(128), 0, (cudaStream_t)stream, P);
    CK(cudaGetLastError());
    return MZ_OK;
}

/* ---- multi-GPU --------------------------------------------------------------------------------------------- */
int32_t mz_cuda_ipc_export(const void *dptr, void *handle64) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    CK(cudaIpcGetMemHandle((cudaIpcMemHandle_t *)handle64, (void *)dptr));
    return MZ_OK;
}
int32_t mz_cuda_ipc_open(const void *handle64, void **dptr) {
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, sizeof(h));
    CK(cudaIpcOpenMemHandle(dptr, h, cudaIpcMemLazyEnablePeerAccess));
    return MZ_OK;
}
int32_t mz_cuda_ipc_close(void *dptr) {
    CK(cudaIpcCloseMemHandle(dptr));
    return MZ_OK;
}
int32_t mz_cuda_memcpy_peer(void *dst, const void *src, size_t bytes, void *stream) {
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, (cudaStream_t)stream)); /* UVA: the driver routes it over NVLink on a copy engine */
    return MZ_OK;
}
int32_t mz_cuda_stream_wait_event(void *stream, void *event) {
    CK(cudaStreamWaitEvent((cudaStream_t)stream, (cudaEvent_t)event, 0));
    return MZ_OK;
}

uint64_t mz_cuda_gather_region_bound(uint64_t shard_len) {
    const uint64_t nch = shard_len == 0 ? 1 : (shard_len + MZ_CUDA_CHUNK_MAX - 1) / MZ_CUDA_CHUNK_MAX;
    return (nch * deflate_slot_bound(MZ_CUDA_CHUNK_MAX) + 255) & ~255ull;
}

namespace {
struct ShardCtx { /* per shard slot (= per device in real use), grown on demand, kept for the life of the process */
    int device = -1;
    cudaStream_t compute = nullptr, copy = nullptr;
    cudaEvent_t ev[2] = {nullptr, nullptr};
    uint8_t *d_slots = nullptr;
    uint32_t *d_out_len = nullptr, *d_residue = nullptr, *d_chunk_crc = nullptr, *d_crc2 = nullptr, *d_rows = nullptr;
    uint64_t *d_offsets = nullptr;
    uint64_t *h_total = nullptr; /* pinned: [2] joined bytes of the piece in flight */
    uint32_t *h_crc = nullptr;   /* pinned: [2][2] */
    uint32_t cap_chunks = 0;
};
ShardCtx g_shard[kMaxDev];
std::mutex g_shard_mu;
}

int32_t mz_cuda_deflate_sharded(const mz_cuda_shard *sh, int32_t ndev, int32_t level, int32_t pieces, uint64_t *region_off, uint64_t *stream_len,
                                uint32_t *crc32) {
    if (!sh || ndev < 1 || ndev > kMaxDev || level < 0 || level > 9 || !region_off || !stream_len) return MZ_PARAM_ERROR;
    if (pieces < 1) pieces = 1;
    std::lock_guard<std::mutex> lk(g_shard_mu);
    int prev_dev = 0;
    cudaGetDevice(&prev_dev);
    const uint64_t stride = deflate_slot_bound(MZ_CUDA_CHUNK_MAX);
    std::vector<uint32_t> nch(ndev), chunk_base(ndev);
    uint64_t roff = 0;
    uint32_t cb = 0;
    for (int i = 0; i < ndev; i++) {
        if (sh[i].device < 0 || sh[i].device >= kMaxDev || !sh[i].d_gathered || ((uintptr_t)sh[i].d_in & 15) || ((uintptr_t)sh[i].d_gathered & 15)) return MZ_PARAM_ERROR;
        if (i + 1 < ndev && (sh[i].len == 0 || sh[i].len % MZ_CUDA_CHUNK_MAX)) return MZ_PARAM_ERROR;
        nch[i] = (uint32_t)(sh[i].len == 0 ? 1 : (sh[i].len + MZ_CUDA_CHUNK_MAX - 1) / MZ_CUDA_CHUNK_MAX);
        region_off[i] = roff;
        roff += mz_cuda_gather_region_bound(sh[i].len);
        chunk_base[i] = cb;
        cb += nch[i];
    }
    for (int i = 0; i < ndev; i++)
        if (sh[i].gathered_cap < roff) return MZ_PARAM_ERROR;
    /* contexts, scratch, peer access */
    for (int i = 0; i < ndev; i++) {
        CK(cudaSetDevice(sh[i].device));
        DeviceCtx *c;
        int32_t err = get_ctx(&c);
        if (err) return err;
        ShardCtx &x = g_shard[i];
        if (x.compute && x.device != sh[i].device) return MZ_PARAM_ERROR; /* slot i stays with the device it was first used with */
        if (!x.compute) {
            x.device = sh[i].device;
            CK(cudaStreamCreateWithFlags(&x.compute, cudaStreamNonBlocking));
            CK(cudaStreamCreateWithFlags(&x.copy, cudaStreamNonBlocking));
            CK(cudaEventCreateWithFlags(&x.ev[0], cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&x.ev[1], cudaEventDisableTiming));
            CK(cudaHostAlloc((void **)&x.h_total, 16, cudaHostAllocDefault));
            CK(cudaHostAlloc((void **)&x.h_crc, 16, cudaHostAllocDefault));
            CK(cudaMalloc(&x.d_crc2, 16));
        }
        const uint32_t need = (nch[i] + (uint32_t)pieces - 1) / (uint32_t)pieces + 1; /* chunks of the largest piece */
        if (x.cap_chunks < need || !x.d_rows) {
            cudaFree(x.d_slots); cudaFree(x.d_out_len); cudaFree(x.d_residue); cudaFree(x.d_chunk_crc); cudaFree(x.d_offsets); cudaFree(x.d_rows);
            x.cap_chunks = 0;
            CK(cudaMalloc(&x.d_slots, (size_t)need * stride));
            CK(cudaMalloc(&x.d_out_len, (size_t)need * 4));
            CK(cudaMalloc(&x.d_residue, (size_t)need * 4));
            CK(cudaMalloc(&x.d_chunk_crc, (size_t)need * 4));
            CK(cudaMalloc(&x.d_offsets, ((size_t)need + 1) * 8));
            CK(cudaMalloc(&x.d_rows, (size_t)need * 12));
            x.cap_chunks = need;
        }
        for (int j = 0; j < ndev; j++)
            if (j != i && sh[j].device != sh[i].device) {
                cudaError_t e = cudaDeviceEnablePeerAccess(sh[j].device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return fail(e, "cudaDeviceEnablePeerAccess");
                cudaGetLastError();
            }
    }
    std::vector<uint64_t> base(ndev, 0);            /* bytes of device i's stream produced so far */
    std::vector<uint32_t> crc_dev(ndev, 0);
    std::vector<uint64_t> done_len(ndev, 0);        /* input bytes folded into crc_dev */
    auto piece_range = [&](int i, int k, uint32_t &c0, uint32_t &c1) {
        c0 = (uint32_t)((uint64_t)nch[i] * k / pieces);
        c1 = (uint32_t)((uint64_t)nch[i] * (k + 1) / pieces);
    };
    /* finish piece k of device i: learn its size, send it (and its rows) to every other device on the copy stream */
    auto finish = [&](int i, int k) -> int32_t {
        ShardCtx &x = g_shard[i];
        CK(cudaSetDevice(sh[i].device));
        CK(cudaEventSynchronize(x.ev[k & 1]));
        uint32_t c0, c1;
        piece_range(i, k, c0, c1);
        const uint64_t L = x.h_total[k & 1];
        const uint64_t in0 = (uint64_t)c0 * MZ_CUDA_CHUNK_MAX;
        const uint64_t inl = ((uint64_t)c1 * MZ_CUDA_CHUNK_MAX < sh[i].len ? (uint64_t)c1 * MZ_CUDA_CHUNK_MAX : sh[i].len) - (in0 < sh[i].len ? in0 : sh[i].len);
        const uint32_t pc = x.h_crc[(k & 1) * 2 + 1];
        if (inl) {
            crc_dev[i] = done_len[i] == 0 ? pc : mz_cuda_crc32_combine(crc_dev[i], pc, inl);
            done_len[i] += inl;
        }
        if (c1 > c0) {
            const uint8_t *src = (const uint8_t *)sh[i].d_gathered + region_off[i] + base[i];
            for (int j = 0; j < ndev; j++) {
                if (j == i) continue;
                CK(cudaMemcpyPeerAsync((uint8_t *)sh[j].d_gathered + region_off[i] + base[i], sh[j].device, src, sh[i].device, (size_t)L, x.copy));
                if (sh[j].d_rows && sh[i].d_rows)
                    CK(cudaMemcpyPeerAsync(sh[j].d_rows + 3ull * (chunk_base[i] + c0), sh[j].device, sh[i].d_rows + 3ull * (chunk_base[i] + c0), sh[i].device,
                                           (size_t)(c1 - c0) * 12, x.copy));
            }
        }
        base[i] += L;
        return MZ_OK;
    };
    for (int k = 0; k <= pieces; k++) {
        if (k < pieces) {
            for (int i = 0; i < ndev; i++) { /* compression of piece k: does not depend on where the piece will land */
                ShardCtx &x = g_shard[i];
                CK(cudaSetDevice(sh[i].device));
                uint32_t c0, c1;
                piece_range(i, k, c0, c1);
                if (c1 == c0) continue;
                const uint64_t in0 = (uint64_t)c0 * MZ_CUDA_CHUNK_MAX;
                const uint64_t inl = ((uint64_t)c1 * MZ_CUDA_CHUNK_MAX < sh[i].len ? (uint64_t)c1 * MZ_CUDA_CHUNK_MAX : sh[i].len) - in0;
                const uint32_t lastf = (i == ndev - 1 && k == pieces - 1) ? MZ_CUDA_FLAG_FINAL : 0u;
                int32_t err = mz_cuda_deflate_chunks((const uint8_t *)sh[i].d_in + in0, inl, MZ_CUDA_CHUNK_MAX, nullptr, nullptr, nullptr, c1 - c0, lastf, level,
                                                     x.d_slots, stride, x.d_out_len, x.compute);
                if (!err) err = mz_cuda_crc32_segments((const uint8_t *)sh[i].d_in + in0, inl, MZ_CUDA_CHUNK_MAX, nullptr, nullptr, c1 - c0, x.d_residue, x.d_chunk_crc, x.compute);
                if (!err) err = mz_cuda_crc32_fold(x.d_residue, c1 - c0, MZ_CUDA_CHUNK_MAX, inl, x.d_crc2, x.compute);
                if (err) return err;
            }
        }
        if (k > 0)
            for (int i = 0; i < ndev; i++) {
                int32_t err = finish(i, k - 1);
                if (err) return err;
            }
        if (k < pieces) {
            for (int i = 0; i < ndev; i++) { /* join piece k straight into the device's own region of its gathered buffer */
                ShardCtx &x = g_shard[i];
                CK(cudaSetDevice(sh[i].device));
                uint32_t c0, c1;
                piece_range(i, k, c0, c1);
                x.h_total[k & 1] = 0;
                if (c1 > c0) {
                    uint8_t *dst = (uint8_t *)sh[i].d_gathered + region_off[i] + base[i];
                    const uint64_t in0 = (uint64_t)c0 * MZ_CUDA_CHUNK_MAX;
                    const uint64_t inl = ((uint64_t)c1 * MZ_CUDA_CHUNK_MAX < sh[i].len ? (uint64_t)c1 * MZ_CUDA_CHUNK_MAX : sh[i].len) - in0;
                    int32_t err = mz_cuda_concat(x.d_slots, stride, x.d_out_len, c1 - c0, x.d_offsets, dst, x.compute);
                    if (err) return err;
                    if (sh[i].d_rows) {
                        MZ_LAUNCH(pack_rows_kernel, dim3((c1 - c0 + 255) / 256), dim3(256), 0, x.compute, (const uint32_t *)x.d_chunk_crc, (const uint32_t *)x.d_out_len,
                                  c1 - c0, inl, (uint32_t)MZ_CUDA_CHUNK_MAX, sh[i].d_rows + 3ull * (chunk_base[i] + c0));
                        CK(cudaGetLastError());
                    }
                    CK(cudaMemcpyAsync(&x.h_total[k & 1], x.d_offsets + (c1 - c0), 8, cudaMemcpyDeviceToHost, x.compute));
                    CK(cudaMemcpyAsync(&x.h_crc[(k & 1) * 2], x.d_crc2, 8, cudaMemcpyDeviceToHost, x.compute));
                }
                CK(cudaEventRecord(x.ev[k & 1], x.compute));
                CK(cudaStreamWaitEvent(x.copy, x.ev[k & 1], 0)); /* the copies of this piece (issued later) follow its join */
            }
        }
    }
    uint32_t crc = 0;
    uint64_t folded = 0;
    for (int i = 0; i < ndev; i++) {
        ShardCtx &x = g_shard[i];
        CK(cudaSetDevice(sh[i].device));
        CK(cudaStreamSynchronize(x.copy));
        CK(cudaStreamSynchronize(x.compute));
        stream_len[i] = base[i];
        if (done_len[i]) {
            crc = folded == 0 ? crc_dev[i] : mz_cuda_crc32_combine(crc, crc_dev[i], done_len[i]);
            folded += done_len[i];
        }
    }
    if (crc32) *crc32 = crc;
    cudaSetDevice(prev_dev);
    return MZ_OK;
}

} /* extern "C" */
