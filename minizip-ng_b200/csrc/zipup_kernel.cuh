/* zipup_kernel.cuh -- K13: a zip archive in device memory updated on the device: kept entries moved as raw bytes, their directory
 * records rewritten (mz_zip_cuda_update_device, include/mz_zip_cuda.h; launches: mz_cuda_zip_up_* in mz_cuda_api.cu).
 *
 * The source's directory is parsed by K10 (its public table gives every accepted entry's local header, extent, sizes and record).
 * Slot i of the output keeps entry keep[i] (or entry i). K13 adds:
 *   counts  one thread per slot: the extent, the directory record without its zip64 (0x0001) fields, the plain and stored bytes
 *           and the 16-byte output slot, scanned with K10's templated scan kernels. The scanned extents are the new local-header
 *           offsets;
 *   layout  one thread per slot, after the scan: the first slot whose new offset reaches 0xffffffff (K11's zip64 rule, zw_emit_kernel).
 *           Offsets grow with the slot, so every slot from there on gets the 28-byte zip64 field and record i lies at
 *           pre[i].cd + 28 x max(0, i - first). Also: a keep index out of range, a slot whose bytes would move or whose extent
 *           holds more than its header, data and descriptor (in place either is an error), a record whose extra field would pass 65535 bytes; and one CTA finds the end record's comment (the last end
 *           record signature in the tail, as zc_end_kernel finds it);
 *   copy    one warp per slot copies its extent to its new offset: head bytes until the destination is 16-byte aligned, then 16-byte
 *           stores, each joined from two aligned 16-byte source loads (one from the next lane by a shuffle) by funnel shifts, then
 *           the ragged tail. A slot whose destination is its source (in place) is skipped, and nothing at or past cap is stored;
 *   records one warp per slot: the kept record (fixed fields, name, zip64 field when needed, every other extra field in order, the
 *           file comment) at its new place, and its mz_cuda_zip_dev_entry row.
 * The new entries, the directory's second part and the end records are K11's (zipwr_kernel.cuh), started at the bases K13 gives.
 * No CTA waits on another, so the kernels also run on the CPU emulator.
 */
#ifndef MZ_ZIPUP_KERNEL_CUH
#define MZ_ZIPUP_KERNEL_CUH

#include "mzcuda_common.cuh"
#include "zipcd_kernel.cuh"
#include "zipwr_kernel.cuh"

namespace mzc {

constexpr uint32_t ZU_THREADS = 256;
constexpr uint64_t ZU_Z64 = 0xffffffffull; /* an offset from here on needs the zip64 field */

struct ZuCount { /* mirror of mz_cuda_zip_up_count: per slot, scanned */
    uint64_t ext, cd, out16, bytes, stored;
    __device__ __forceinline__ ZuCount operator+(const ZuCount &o) const {
        ZuCount r;
        r.ext = ext + o.ext;
        r.cd = cd + o.cd;
        r.out16 = out16 + o.out16;
        r.bytes = bytes + o.bytes;
        r.stored = stored + o.stored;
        return r;
    }
};

/* info words (mz_cuda_zip_up.info), ~0 before counts */
enum { ZU_FIRST64 = 0, ZU_BADKEEP, ZU_MOVED, ZU_XLEN, ZU_EOCD, ZU_CLEN, ZU_NINFO };

struct ZuCall { /* mirror of mz_cuda_zip_up */
    const uint8_t *src;
    const ZipDevEnt *ent;
    uint32_t count, n;
    const uint32_t *keep;
    const uint8_t *dir;
    uint64_t dir_off, src_len;
    ZuCount *cnt, *pre;
    void *part;
    unsigned long long *info;
    uint8_t *archive;
    uint64_t cap, cd_off;
    void *entries;
};

__device__ __forceinline__ uint32_t zu_index(const ZuCall &U, uint32_t i) { return U.keep ? U.keep[i] : i; }
/* the source record of entry e (dir holds the source's bytes from dir_off on) */
__device__ __forceinline__ const uint8_t *zu_rec(const ZuCall &U, const ZipDevEnt &e) { return U.dir + (e.name_off - 46 - U.dir_off); }

/* bytes of the extra field xf[0, xlen) that are not zip64 fields: fields are walked by their stated lengths; a field cut by the
 * end of the extra field, and bytes too few for a field header, are kept as they are */
__device__ __forceinline__ uint32_t zu_kept_xlen(const uint8_t *xf, uint32_t xlen) {
    uint32_t drop = 0;
    for (uint32_t xo = 0; xo + 4 <= xlen;) {
        const uint32_t xs = zc_u16(xf + xo + 2), fl = 4 + xs < xlen - xo ? 4 + xs : xlen - xo;
        if (zc_u16(xf + xo) == 0x0001) drop += fl;
        xo += 4 + xs;
    }
    return xlen - drop;
}

__global__ void __launch_bounds__(ZU_THREADS) zu_counts_kernel(ZuCall U) {
    const uint32_t i = blockIdx.x * ZU_THREADS + threadIdx.x;
    if (i >= U.n) return;
    const uint32_t idx = zu_index(U, i);
    ZuCount c = zc_zero<ZuCount>();
    if (idx >= U.count) {
        atomicMin(&U.info[ZU_BADKEEP], (unsigned long long)i);
    } else {
        const ZipDevEnt e = U.ent[idx];
        const uint8_t *r = zu_rec(U, e);
        const uint32_t nlen = zc_u16(r + 28), xlen = zc_u16(r + 30), clen = zc_u16(r + 32);
        c.ext = e.extent;
        c.cd = 46ull + nlen + zu_kept_xlen(r + 46 + nlen, xlen) + clen;
        c.out16 = (e.usize + 15) & ~15ull;
        c.bytes = e.usize;
        c.stored = e.csize;
    }
    U.cnt[i] = c;
}

__global__ void __launch_bounds__(ZU_THREADS) zu_layout_kernel(ZuCall U) {
    const uint32_t i = blockIdx.x * ZU_THREADS + threadIdx.x;
    if (i >= U.n) return;
    const uint64_t off = U.pre[i].ext;
    if (off >= ZU_Z64 && (i == 0 || U.pre[i - 1].ext < ZU_Z64)) atomicMin(&U.info[ZU_FIRST64], (unsigned long long)i);
    const uint32_t idx = zu_index(U, i);
    if (idx >= U.count) return;
    const ZipDevEnt e = U.ent[idx];
    /* in place the kept bytes must not move, and the entries must tile the source with no gaps: an extent holds its local header,
     * the stored bytes and, with flag bit 3, a data descriptor (12 or 20 bytes, 16 or 24 with its signature) and nothing more */
    const uint8_t *lh = U.src + e.local_off;
    const uint64_t body = 30ull + zc_u16(lh + 26) + zc_u16(lh + 28) + e.csize, rest = e.extent - body;
    const bool tiles = e.extent >= body && (rest == 0 || ((zc_u16(lh + 6) & 8u) && (rest == 12 || rest == 16 || rest == 20 || rest == 24)));
    if (off != e.local_off || !tiles) atomicMin(&U.info[ZU_MOVED], (unsigned long long)i);
    if (off >= ZU_Z64) {
        const uint8_t *r = zu_rec(U, e);
        const uint32_t nlen = zc_u16(r + 28);
        if (zu_kept_xlen(r + 46 + nlen, zc_u16(r + 30)) + 28 > 65535u) atomicMin(&U.info[ZU_XLEN], (unsigned long long)i);
    }
}

/* one CTA: the end record's position and its comment length (clamped to the bytes behind it) */
__global__ void __launch_bounds__(ZU_THREADS) zu_comment_kernel(ZuCall U) {
    __shared__ uint64_t red[ZU_THREADS];
    const uint64_t len = U.src_len, tl = len < ZC_TAIL ? len : ZC_TAIL, base = len - tl;
    uint64_t best = 0;
    for (uint64_t i = threadIdx.x; i + 22 <= tl; i += ZU_THREADS) {
        const uint8_t *q = U.src + base + i;
        if (q[0] == 0x50 && q[1] == 0x4b && q[2] == 0x05 && q[3] == 0x06) best = i + 1;
    }
    red[threadIdx.x] = best;
    __syncthreads();
    for (uint32_t h = ZU_THREADS / 2; h; h >>= 1) {
        if (threadIdx.x < h && red[threadIdx.x + h] > red[threadIdx.x]) red[threadIdx.x] = red[threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x || !red[0]) return;
    const uint64_t eocd = base + red[0] - 1, room = len - eocd - 22;
    const uint64_t clen = zc_u16(U.src + eocd + 20);
    U.info[ZU_EOCD] = eocd;
    U.info[ZU_CLEN] = clen < room ? clen : room;
}

/* the 16 bytes at byte offset sh (0..15) of the 32 bytes c:n */
__device__ __forceinline__ uint4 zu_join(const uint4 &c, const uint4 &n, uint32_t sh) {
    const uint32_t q = sh >> 2, r = (sh & 3u) * 8u;
    uint32_t x0, x1, x2, x3, x4;
    if (q == 0) { x0 = c.x; x1 = c.y; x2 = c.z; x3 = c.w; x4 = n.x; }
    else if (q == 1) { x0 = c.y; x1 = c.z; x2 = c.w; x3 = n.x; x4 = n.y; }
    else if (q == 2) { x0 = c.z; x1 = c.w; x2 = n.x; x3 = n.y; x4 = n.z; }
    else { x0 = c.w; x1 = n.x; x2 = n.y; x3 = n.z; x4 = n.w; }
    return make_uint4(__funnelshift_r(x0, x1, r), __funnelshift_r(x1, x2, r), __funnelshift_r(x2, x3, r), __funnelshift_r(x3, x4, r));
}

/* one warp per slot. Source loads are aligned 16-byte blocks that hold at least one byte of the extent, so they stay inside the
 * 16-byte aligned granules of the source allocation; the extent ends at or before the directory. */
__global__ void __launch_bounds__(ZU_THREADS) zu_copy_kernel(ZuCall U) {
    const uint32_t warp = (blockIdx.x * ZU_THREADS + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const uint32_t nwarps = (gridDim.x * ZU_THREADS) >> 5;
    for (uint32_t i = warp; i < U.n; i += nwarps) {
        const uint32_t idx = zu_index(U, i);
        if (idx >= U.count) continue;
        const ZipDevEnt &e = U.ent[idx];
        const uint64_t pos = U.pre[i].ext;
        const uint8_t *s = U.src + e.local_off;
        uint8_t *d = U.archive + pos;
        if (d == s || pos >= U.cap) continue;
        uint64_t len = e.extent < U.cap - pos ? e.extent : U.cap - pos;
        uint32_t head = (uint32_t)(-(uintptr_t)d & 15u);
        if (head > len) head = (uint32_t)len;
        if (lane < head) d[lane] = s[lane];
        s += head;
        d += head;
        len -= head;
        const uint4 *a = (const uint4 *)((uintptr_t)s & ~(uintptr_t)15);
        const uint32_t sh = (uint32_t)((uintptr_t)s & 15);
        const uint64_t blocks = len >> 4, loads = blocks + (sh && blocks ? 1 : 0);
        for (uint64_t k0 = 0; k0 < blocks; k0 += 32) {
            const uint64_t k = k0 + lane;
            const uint4 z = make_uint4(0, 0, 0, 0);
            const uint4 c = k < loads ? a[k] : z;
            uint4 n;
            n.x = __shfl_down_sync(MZ_FULL_MASK, c.x, 1);
            n.y = __shfl_down_sync(MZ_FULL_MASK, c.y, 1);
            n.z = __shfl_down_sync(MZ_FULL_MASK, c.z, 1);
            n.w = __shfl_down_sync(MZ_FULL_MASK, c.w, 1);
            if (lane == 31) n = k + 1 < loads ? a[k + 1] : z;
            if (k < blocks) ((uint4 *)d)[k] = sh ? zu_join(c, n, sh) : c;
        }
        for (uint64_t k = (blocks << 4) + lane; k < len; k += 32) d[k] = s[k];
    }
}

/* one warp per slot: the kept record at cd_off + pre.cd + 28 x (slots in front that carry a zip64 field), and its row */
__global__ void __launch_bounds__(ZU_THREADS) zu_records_kernel(ZuCall U) {
    const uint32_t i = blockIdx.x * (ZU_THREADS / 32) + warp_id();
    const unsigned lane = lane_id();
    if (i >= U.n) return;
    const ZipDevEnt e = U.ent[zu_index(U, i)];
    const ZwOut o{U.archive, U.cap};
    const uint64_t f = U.info[ZU_FIRST64] < U.n ? U.info[ZU_FIRST64] : U.n;
    const bool z64 = i >= f;
    const uint64_t lh = U.pre[i].ext, cd = U.cd_off + U.pre[i].cd + 28ull * (z64 ? i - f : 0);
    const uint8_t *r = zu_rec(U, e);
    const uint32_t nlen = zc_u16(r + 28), xlen = zc_u16(r + 30), clen = zc_u16(r + 32);
    const uint8_t *xf = r + 46 + nlen;
    const uint32_t kept = zu_kept_xlen(xf, xlen);
    /* fixed fields: copied, but version needed (6), sizes (20, 24), extra length (30), disk (34) and offset (42) */
    for (uint32_t b = lane; b < 46; b += 32)
        if (!((b >= 6 && b < 8) || (b >= 20 && b < 28) || (b >= 30 && b < 32) || (b >= 34 && b < 36) || b >= 42)) o.b(cd + b, r[b]);
    if (lane == 0) {
        const uint32_t ver = zc_u16(r + 6);
        const bool had64 = kept != xlen; /* a zip64 field is dropped */
        uint32_t nv = ver;
        if (z64 && nv < 45) nv = 45;
        else if (!z64 && had64 && ver == 45 && !e.aes) nv = 20; /* 45 only for the zip64 field it loses */
        o.u16(cd + 6, nv);
        o.u32(cd + 20, z64 ? 0xffffffffu : (uint32_t)e.csize);
        o.u32(cd + 24, z64 ? 0xffffffffu : (uint32_t)e.usize);
        o.u16(cd + 30, kept + (z64 ? 28 : 0));
        o.u16(cd + 34, 0); /* an accepted record is on disk 0 (K10 refuses others); 0xffff would need the zip64 field */
        o.u32(cd + 42, z64 ? 0xffffffffu : (uint32_t)lh);
        if (z64) { /* as zw_emit_kernel: uncompressed, compressed, header offset */
            const uint64_t x = cd + 46 + nlen;
            o.u16(x, 1);
            o.u16(x + 2, 24);
            o.u64(x + 4, e.usize);
            o.u64(x + 12, e.csize);
            o.u64(x + 20, lh);
        }
    }
    for (uint32_t k = lane; k < nlen; k += 32) o.b(cd + 46 + k, r[46 + k]);
    /* the other extra fields in order; the hash field's digest moves with its field */
    const uint64_t sha_src = e.has_sha ? e.sha_off - 8 - (e.name_off + nlen) : ~0ull; /* its field's offset in the source extra field */
    uint64_t p = cd + 46 + nlen + (z64 ? 28 : 0), sha_off = 0;
    uint32_t xo = 0;
    while (xo + 4 <= xlen) {
        const uint32_t xs = zc_u16(xf + xo + 2), fl = 4 + xs < xlen - xo ? 4 + xs : xlen - xo;
        if (zc_u16(xf + xo) != 0x0001) {
            if (xo == sha_src) sha_off = p + 8;
            for (uint32_t k = lane; k < fl; k += 32) o.b(p + k, xf[xo + k]);
            p += fl;
        }
        xo += 4 + xs;
    }
    if (xo < xlen) { /* bytes too few for a field header */
        for (uint32_t k = lane; k < xlen - xo; k += 32) o.b(p + k, xf[xo + k]);
        p += xlen - xo;
    }
    for (uint32_t k = lane; k < clen; k += 32) o.b(p + k, xf[xlen + k]);
    if (U.entries && lane == 0) { /* the row mz_zip_cuda_extract_device lists for this entry of the output */
        ZipDevEnt d = e;
        d.local_off = lh;
        d.out_off = U.pre[i].out16;
        d.name_off = cd + 46;
        d.sha_off = e.has_sha ? sha_off : 0;
        d.status = 0;
        ((ZipDevEnt *)U.entries)[i] = d;
    }
}

} // namespace mzc
#endif
