/* zipwr_kernel.cuh -- K11: a zip archive written into device memory from entries held in device memory
 * (mz_zip_cuda_write_device, include/mz_zip_cuda.h; launches: mz_cuda_zip_wr_* in mz_cuda_api.cu).
 *
 * The native host writer (za_prepare / mz_zip_cuda_write_archive_aes in mz_zip_cuda.c) lays every entry out as
 *     local header | [salt | verifier] | DEFLATE stream | [authentication code]
 * and builds headers, CRCs and the central directory on the host. Here every step runs on the device:
 *   items    one thread per item: validation (the first invalid item by an atomic min over index << 1 | kind), and the entry's
 *            counts: chunks, fixed overhead (header + salt + verifier + authentication code: it does not depend on compression),
 *            plain bytes, slot bound, directory record size without zip64. One scan (per-tile sums, one CTA over the sums, per-tile
 *            apply, the K10 scan kernels) makes OV(e), the overhead of the entries in front of e, known before any chunk is
 *            compressed;
 *   chunks   one thread per chunk of the global chunk list: the {off, len, flags} rows K2+K3 and K1 take (binary search for the
 *            chunk's entry in the scanned chunk counts); FINAL on an entry's last chunk, DICT on the others' successors;
 *   place    per round, after K2+K3 and K1: an exclusive scan of the round's stream lengths carried in from the previous round by
 *            S[c0] in device memory gives S(c), the stream bytes in front of chunk c; its destination is OV(e) + header(e) + S(c),
 *            and a chunk whose bytes would pass `cap` gets copy length 0. K4 gathers straight into the archive;
 *   entries  one warp per entry: the CRC fold of the entry's chunk residues (each lane Horner-folds a run of full chunks by
 *            x^(8 * 65536), a shuffle tree joins the runs, the last chunk joins by its own length -- as crc32_fold_kernel does for
 *            one buffer), the local-header offset OV(e) + S(first chunk), the stream length, and the directory record size, which
 *            grows by the zip64 field when the offset reaches 0xffffffff; an entry whose stored size reaches 0xffffffff lowers `bad`
 *            (the host writer returns MZ_INTERNAL_ERROR for it). A second scan lays the directory out;
 *   emit     one warp per entry, after K8 encrypted the streams in place (AES): local header, salt and verifier, authentication
 *            code, directory record and the public table row; then one thread writes the end records.
 * The bases lh_base, cd_base, out_base, n_base and the comment place the new entries behind entries already in the archive
 * (mz_zip_cuda_update_device, zipup_kernel.cuh): local headers (and so the zip64 decision) see absolute offsets, the new records
 * follow cd_base bytes of kept records, the end records count n_base + n entries. All are 0 or empty for write_device.
 * No CTA waits on another, so the kernels also run on the CPU emulator. Every archive byte is written only below `cap`.
 * The layout rules are those of the host writer, written a second time here on purpose: the host writer serves host-resident
 * entries and is the reference the device output is compared with byte for byte.
 */
#ifndef MZ_ZIPWR_KERNEL_CUH
#define MZ_ZIPWR_KERNEL_CUH

#include "crc32_kernel.cuh"
#include "deflate_kernel.cuh"
#include "mzcuda_common.cuh"
#include "zipcd_kernel.cuh"

namespace mzc {

constexpr uint32_t ZW_THREADS = 256;
constexpr uint64_t ZW_CHUNK = 65536;

struct ZwItem { /* mirror of mz_cuda_zip_dev_item */
    uint64_t data_off, size, name_off;
    uint32_t name_len, dos_date, external_fa, reserved;
};

struct ZwCount { /* mirror of mz_cuda_zip_wr_count: per item, scanned */
    uint64_t chunks, overhead, bytes, out16, bound, cd;
    __device__ __forceinline__ ZwCount operator+(const ZwCount &o) const {
        ZwCount r;
        r.chunks = chunks + o.chunks;
        r.overhead = overhead + o.overhead;
        r.bytes = bytes + o.bytes;
        r.out16 = out16 + o.out16;
        r.bound = bound + o.bound;
        r.cd = cd + o.cd;
        return r;
    }
};

struct ZwCall { /* mirror of mz_cuda_zip_wr */
    const uint8_t *data, *names;
    const ZwItem *items;
    uint32_t n, aes, sha, dos_now;
    uint8_t *archive;
    uint64_t cap;
    unsigned long long *bad;
    ZwCount *cnt, *pre;
    void *part;
    uint64_t nch;
    uint64_t *c_off;
    uint32_t *c_len;
    uint8_t *c_flags;
    uint32_t *c_item, *out_len, *residue, *glen;
    uint64_t *S, *dst;
    uint64_t *e_lh, *e_csize, *e_cd, *e_cdpre, *e_coff, *e_off, *e_len;
    uint32_t *e_crc;
    unsigned long long *max_csize;
    const uint8_t *digest, *salt, *keys, *mac;
    void *entries;
    uint64_t lh_base, cd_base, out_base; /* in front of the new entries: archive bytes, directory bytes, output slots */
    uint32_t n_base, comment_len;         /* entries in front; the end record's comment */
    const uint8_t *comment;
};

__device__ __forceinline__ uint32_t zw_salt_len(uint32_t aes) { return aes ? 4 * aes + 4 : 0; }
__device__ __forceinline__ uint32_t zw_xf(const ZwCall &W) { return (W.aes ? 11u : 0u) + (W.sha ? 40u : 0u); }
/* local header, name, extra field, salt and verifier: the bytes in front of the entry's stream */
__device__ __forceinline__ uint64_t zw_head(const ZwCall &W, uint32_t nlen) { return 30ull + nlen + zw_xf(W) + (W.aes ? zw_salt_len(W.aes) + 2 : 0); }

/* ---- items ------------------------------------------------------------------------------------------------------------- */
/* bad: lowered to index << 1 | kind of the first invalid item (kind 0 = MZ_PARAM_ERROR: name or pointers, 1 = MZ_SUPPORT_ERROR:
 * size), the host writer's per-item order (mz_zip_cuda_write_archive_aes) */
__global__ void __launch_bounds__(ZW_THREADS) zw_items_kernel(ZwCall W, uint32_t data_null, uint32_t names_null) {
    const uint32_t i = blockIdx.x * ZW_THREADS + threadIdx.x;
    if (i >= W.n) return;
    const ZwItem it = W.items[i];
    bool param = it.name_len == 0 || it.name_len > 65535 || names_null || (it.size && data_null) || it.data_off + it.size < it.data_off ||
                 it.name_off + it.name_len < it.name_off;
    for (uint32_t k = 0; !param && k < it.name_len; k++)
        if (W.names[it.name_off + k] == 0) param = true;
    const bool support = it.size >= 0xffff0000ull;
    ZwCount c = zc_zero<ZwCount>();
    if (param || support) {
        atomicMin(W.bad, ((unsigned long long)i << 1) | (param ? 0ull : 1ull));
    } else {
        const uint64_t nch = it.size ? (it.size + ZW_CHUNK - 1) / ZW_CHUNK : 1;
        const uint32_t last = (uint32_t)(it.size - (nch - 1) * ZW_CHUNK);
        c.chunks = nch;
        c.overhead = zw_head(W, it.name_len) + (W.aes ? 10 : 0);
        c.bytes = it.size;
        c.out16 = (it.size + 15) & ~15ull;
        c.bound = (nch - 1) * deflate_slot_bound((uint32_t)ZW_CHUNK) + deflate_slot_bound(last);
        c.cd = 46ull + it.name_len + zw_xf(W);
    }
    W.cnt[i] = c;
}

/* ---- chunks: one thread per chunk of the global list --------------------------------------------------------------------- */
__global__ void __launch_bounds__(ZW_THREADS) zw_chunks_kernel(ZwCall W) {
    const uint64_t c = (uint64_t)blockIdx.x * ZW_THREADS + threadIdx.x;
    if (c >= W.nch) return;
    uint32_t lo = 0, hi = W.n; /* the entry e with pre[e].chunks <= c < pre[e + 1].chunks */
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (W.pre[mid].chunks <= c) lo = mid; else hi = mid;
    }
    const uint32_t e = lo;
    const ZwItem it = W.items[e];
    const uint64_t k = c - W.pre[e].chunks, nk = W.pre[e + 1].chunks - W.pre[e].chunks;
    const uint64_t rem = it.size - k * ZW_CHUNK;
    W.c_off[c] = it.data_off + k * ZW_CHUNK;
    W.c_len[c] = rem < ZW_CHUNK ? (uint32_t)rem : (uint32_t)ZW_CHUNK;
    W.c_flags[c] = (uint8_t)((k + 1 == nk ? DF_FLAG_FINAL : 0u) | (k > 0 ? DF_FLAG_DICT : 0u));
    W.c_item[c] = e;
    if (k == 0 && W.sha) { /* K7's segments: the entry's plain bytes */
        W.e_off[e] = it.data_off;
        W.e_len[e] = it.size;
    }
}

/* ---- place: the round's chunks (zc_round_place_kernel) ------------------------------------------------------------------- */
/* chunk c's destination in front of S(c): OV(e) and the header of its entry e */
struct ZwPlaceBase {
    ZwCall W;
    __device__ __forceinline__ uint64_t operator()(uint64_t c) const {
        const uint32_t e = W.c_item[c];
        return W.lh_base + W.pre[e].overhead + zw_head(W, W.items[e].name_len);
    }
};

/* ---- entries: one warp per entry ----------------------------------------------------------------------------------------- */
__global__ void __launch_bounds__(ZW_THREADS) zw_entries_kernel(ZwCall W, const CrcConsts *cc) {
    const uint32_t e = blockIdx.x * (ZW_THREADS / 32) + warp_id();
    const unsigned lane = lane_id();
    if (e >= W.n) return;
    const uint64_t first = W.pre[e].chunks, last = W.pre[e + 1].chunks - 1;
    const uint64_t size = W.items[e].size;
    /* full chunks [first, last): lane l Horner-folds run l of `per` of them, right-aligned so that the zero padding is in front */
    const uint64_t nfull = last - first, per = (nfull + 31) / 32, lead = per * 32 - nfull;
    const uint32_t m1 = gf2_xpow(cc->x2n, 8 * ZW_CHUNK);
    uint32_t acc = 0;
    for (uint64_t k = 0; k < per; k++) {
        const uint64_t j = (uint64_t)lane * per + k;
        acc = gf2_mulmod(acc, m1) ^ (j >= lead ? W.residue[first + j - lead] : 0u);
    }
    uint32_t mul = gf2_xpow(cc->x2n, 8 * ZW_CHUNK * (per ? per : 1));
    for (uint32_t st = 1; st < 32; st <<= 1) { /* lanes l, l + st hold adjacent groups of st runs: join them */
        const uint32_t other = __shfl_down_sync(MZ_FULL_MASK, acc, st);
        if ((lane & (2 * st - 1)) == 0) acc = gf2_mulmod(acc, mul) ^ other;
        mul = gf2_mulmod(mul, mul);
    }
    if (lane) return;
    const uint64_t last_len = size - nfull * ZW_CHUNK;
    const uint32_t r = gf2_mulmod(acc, gf2_xpow(cc->x2n, 8 * last_len)) ^ W.residue[last];
    const uint32_t crc = size ? ~(gf2_mulmod(0xffffffffu, gf2_xpow(cc->x2n, 8 * size)) ^ r) : 0u;
    const uint64_t lh = W.lh_base + W.pre[e].overhead + W.S[first], csize = W.S[last + 1] - W.S[first];
    W.e_lh[e] = lh;
    W.e_csize[e] = csize;
    W.e_crc[e] = crc;
    W.e_coff[e] = lh + zw_head(W, W.items[e].name_len);
    W.e_cd[e] = W.cnt[e].cd + (lh >= 0xffffffffull ? 28 : 0);
    if (W.aes) atomicMax(W.max_csize, (unsigned long long)csize);
    /* the local header stores the stored size in 32 bits: an entry just below 4 GiB whose stream grew past them (stored blocks of
     * incompressible data) is refused, as the host writer refuses it; bad is still ~0 after a validation that passed */
    if (csize + (W.aes ? zw_salt_len(W.aes) + 2 + 10 : 0) >= 0xffffffffull) atomicMin(W.bad, (unsigned long long)e << 1);
}

/* ---- emit ---------------------------------------------------------------------------------------------------------------- */
struct ZwOut { /* little-endian stores that never reach `cap` */
    uint8_t *a;
    uint64_t cap;
    __device__ __forceinline__ void b(uint64_t p, uint32_t v) const {
        if (p < cap) a[p] = (uint8_t)v;
    }
    __device__ __forceinline__ void u16(uint64_t p, uint32_t v) const { b(p, v); b(p + 1, v >> 8); }
    __device__ __forceinline__ void u32(uint64_t p, uint32_t v) const { u16(p, v); u16(p + 2, v >> 16); }
    __device__ __forceinline__ void u64(uint64_t p, uint64_t v) const { u32(p, (uint32_t)v); u32(p + 4, (uint32_t)(v >> 32)); }
};

/* the AES extra field (id 0x9901, AE-1, vendor "AE", strength, real method 8) and the hash extra field (id 0x1a51, SHA-256, 32
 * bytes), written by lanes 0..10 and 0..39 of a warp */
__device__ __forceinline__ uint64_t zw_fields(const ZwOut &o, uint64_t p, const ZwCall &W, uint32_t e, unsigned lane) {
    if (W.aes) { /* 01 99 07 00 01 00 'A' 'E' strength 08 00 */
        if (lane < 11) o.b(p + lane, lane < 8 ? (uint32_t)(0x4541000100079901ull >> (8 * lane)) : lane == 8 ? W.aes : lane == 9 ? 8u : 0u);
        p += 11;
    }
    if (W.sha) { /* 51 1a 24 00 17 00 20 00, digest */
        for (uint32_t k = lane; k < 40; k += 32) o.b(p + k, k < 8 ? (uint32_t)(0x0020001700241a51ull >> (8 * k)) : W.digest[(uint64_t)e * 32 + k - 8]);
        p += 40;
    }
    return p;
}

__global__ void __launch_bounds__(ZW_THREADS) zw_emit_kernel(ZwCall W, uint64_t cd_off) {
    const uint32_t e = blockIdx.x * (ZW_THREADS / 32) + warp_id();
    const unsigned lane = lane_id();
    if (e >= W.n) return;
    const ZwOut o{W.archive, W.cap};
    const ZwItem it = W.items[e];
    const uint32_t nlen = it.name_len, xf = zw_xf(W), slen = zw_salt_len(W.aes);
    const uint64_t lh = W.e_lh[e], csize = W.e_csize[e], stored = csize + (W.aes ? slen + 2 + 10 : 0);
    const uint32_t crc = W.e_crc[e], date = it.dos_date ? it.dos_date : W.dos_now;
    const uint32_t fa = it.external_fa ? it.external_fa : (0100644u << 16);
    const bool z64 = lh >= 0xffffffffull;
    const uint64_t cd = cd_off + W.cd_base + W.e_cdpre[e];
    if (lane == 0) {
        o.u32(lh, 0x04034b50u);                           /* local header (za_prepare) */
        o.u16(lh + 4, W.aes ? 51 : 20);
        o.u16(lh + 6, (1u << 11) | (W.aes ? 1u : 0u));
        o.u16(lh + 8, W.aes ? 99 : 8);
        o.u32(lh + 10, date);
        o.u32(lh + 14, crc);
        o.u32(lh + 18, (uint32_t)stored);
        o.u32(lh + 22, (uint32_t)it.size);
        o.u16(lh + 26, nlen);
        o.u16(lh + 28, xf);
    } else if (lane == 1) {
        o.u32(cd, 0x02014b50u);                           /* directory record (mz_zip_cuda_write_archive_aes) */
        o.u16(cd + 4, (3u << 8) | 45u);
        o.u16(cd + 6, W.aes ? 51 : (z64 ? 45 : 20));
        o.u16(cd + 8, (1u << 11) | (W.aes ? 1u : 0u));
        o.u16(cd + 10, W.aes ? 99 : 8);
        o.u32(cd + 12, date);
        o.u32(cd + 16, crc);
        o.u32(cd + 20, z64 ? 0xffffffffu : (uint32_t)stored);
        o.u32(cd + 24, z64 ? 0xffffffffu : (uint32_t)it.size);
        o.u16(cd + 28, nlen);
        o.u16(cd + 30, xf + (z64 ? 28 : 0));
        o.u32(cd + 32, 0);                                /* comment length, disk number start */
        o.u16(cd + 36, 0);                                /* internal attributes */
        o.u32(cd + 38, fa);
        o.u32(cd + 42, z64 ? 0xffffffffu : (uint32_t)lh);
        if (z64) {                                        /* zip64 field: uncompressed, compressed, header offset */
            const uint64_t x = cd + 46 + nlen;
            o.u16(x, 1);
            o.u16(x + 2, 24);
            o.u64(x + 4, it.size);
            o.u64(x + 12, stored);
            o.u64(x + 20, lh);
        }
    }
    for (uint32_t k = lane; k < nlen; k += 32) {
        const uint8_t ch = W.names[it.name_off + k];
        o.b(lh + 30 + k, ch);
        o.b(cd + 46 + k, ch);
    }
    uint64_t p = zw_fields(o, lh + 30 + nlen, W, e, lane);
    zw_fields(o, cd + 46 + nlen + (z64 ? 28 : 0), W, e, lane);
    if (W.aes) {
        if (lane < slen) o.b(p + lane, W.salt[(uint64_t)e * 16 + lane]);
        if (lane < 2) o.b(p + slen + lane, W.keys[(uint64_t)e * ZD_KEYREC + 64 + lane]);
        if (lane < 10) o.b(W.e_coff[e] + csize + lane, W.mac[(uint64_t)e * 20 + lane]);
    }
    if (W.entries && lane == 0) { /* the row mz_zip_cuda_extract_device lists for this entry */
        ZipDevEnt d;
        d.local_off = lh;
        d.csize = stored;
        d.usize = it.size;
        d.out_off = W.out_base + W.pre[e].out16;
        d.name_off = cd + 46;
        d.extent = (e + 1 < W.n ? W.e_lh[e + 1] : cd_off) - lh;
        d.sha_off = W.sha ? cd + 46 + nlen + (z64 ? 28 : 0) + (W.aes ? 11 : 0) + 8 : 0;
        d.crc = crc;
        d.name_len = nlen;
        d.method = 8;
        d.aes = (uint8_t)W.aes;
        d.has_sha = (uint8_t)(W.sha ? 1 : 0);
        d.status = 0;
        ((ZipDevEnt *)W.entries)[e] = d;
    }
}

/* the end records behind the directory (zip64 end record and locator when the directory starts at 0xffffffff or later or there
 * are 0xffff entries or more), written by thread 0; the comment (up to 65535 bytes) by the whole CTA */
__global__ void __launch_bounds__(ZW_THREADS) zw_end_kernel(ZwCall W, uint64_t cd_off, uint64_t cd_size) {
    const ZwOut o{W.archive, W.cap};
    const uint64_t n = (uint64_t)W.n_base + W.n;
    uint64_t q = cd_off + cd_size;
    const uint64_t z = cd_off >= 0xffffffffull || n >= 0xffffu ? 76 : 0;
    for (uint32_t k = threadIdx.x; k < W.comment_len; k += ZW_THREADS) o.b(q + z + 22 + k, W.comment[k]);
    if (threadIdx.x) return;
    if (z) {
        o.u32(q, 0x06064b50u);
        o.u64(q + 4, 44);
        o.u16(q + 12, (3u << 8) | 45u);
        o.u16(q + 14, 45);
        o.u64(q + 16, 0);
        o.u64(q + 24, n);
        o.u64(q + 32, n);
        o.u64(q + 40, cd_size);
        o.u64(q + 48, cd_off);
        o.u32(q + 56, 0x07064b50u);
        o.u32(q + 60, 0);
        o.u64(q + 64, cd_off + cd_size);
        o.u32(q + 72, 1);
        q += 76;
    }
    o.u32(q, 0x06054b50u);
    o.u32(q + 4, 0);
    o.u16(q + 8, n >= 0xffffu ? 0xffffu : (uint32_t)n);
    o.u16(q + 10, n >= 0xffffu ? 0xffffu : (uint32_t)n);
    o.u32(q + 12, (uint32_t)cd_size);
    o.u32(q + 16, cd_off >= 0xffffffffull ? 0xffffffffu : (uint32_t)cd_off);
    o.u16(q + 20, W.comment_len);
}

} // namespace mzc
#endif
