/* mz_zip_cuda.c -- batch zip-entry writer on the reference's raw-entry seam (include/mz_zip_cuda.h).
 *
 * What it replaces, per entry, in the reference: mz_zip_entry_write_open(raw = 0) creating a mz_stream_zlib
 * (mz_zip.c:1771-1773), the caller's write loop feeding it (mz_zip_rw.c:1424-1480), the CRC accumulation
 * (mz_zip.c:2062-2064) and mz_zip_entry_close (mz_zip.c:2116-2160). Here the codec work of MANY entries is one
 * K2+K3 launch + one K1 launch + one K4 launch per round, and the container calls run with raw = 1.
 */
#define _GNU_SOURCE /* qsort_r */
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <sys/random.h>

#include "mz_abi.h"
#include "mz_cuda_batch.h"
#include "mz_cuda_host.h"
#include "mz_zip_cuda.h"

#define ZC_CHUNK 65536u

/* mz_zip.h:25-51 (mz_zip_file): the raw seam takes this struct by pointer and copies it (mz_zip.c:1939) */
typedef struct zc_file_info_s {
    uint16_t version_madeby;
    uint16_t version_needed;
    uint16_t flag;
    uint16_t compression_method;
    time_t modified_date;
    time_t accessed_date;
    time_t creation_date;
    uint32_t crc;
    int64_t compressed_size;
    int64_t uncompressed_size;
    uint16_t filename_size;
    uint16_t extrafield_size;
    uint16_t comment_size;
    uint32_t disk_number;
    int64_t disk_offset;
    uint16_t internal_fa;
    uint32_t external_fa;
    const char *filename;
    const uint8_t *extrafield;
    const char *comment;
    const char *linkname;
    uint16_t zip64;
    uint16_t aes_version;
    uint8_t aes_strength;
    uint16_t pk_verify;
} zc_file_info;

/* the container stays the reference's: these come from the host program (mz_zip.c:1915, 2056, 2272) */
extern int32_t mz_zip_entry_write_open(void *handle, const void *file_info, int16_t compress_level, uint8_t raw, const char *password)
    __attribute__((weak));
extern int32_t mz_zip_entry_write(void *handle, const void *buf, int32_t len) __attribute__((weak));
extern int32_t mz_zip_entry_close_raw(void *handle, int64_t uncompressed_size, uint32_t crc32) __attribute__((weak));
/* reader side (mz_zip.h:115-172) */
extern int32_t mz_zip_goto_first_entry(void *handle) __attribute__((weak));
extern int32_t mz_zip_goto_next_entry(void *handle) __attribute__((weak));
extern int32_t mz_zip_entry_get_info(void *handle, zc_file_info **file_info) __attribute__((weak));
extern int32_t mz_zip_entry_read_open(void *handle, uint8_t raw, const char *password) __attribute__((weak));
extern int32_t mz_zip_entry_read(void *handle, void *buf, int32_t len) __attribute__((weak));
extern int32_t mz_zip_entry_close(void *handle) __attribute__((weak));

uint32_t mz_zip_cuda_abi_file_info_size(void) {
    return (uint32_t)sizeof(zc_file_info);
}

static double now_ms(void) {
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (double)ts.tv_sec * 1e3 + (double)ts.tv_nsec * 1e-6;
}

typedef struct zc_bufs_s {
    size_t round_bytes;
    uint32_t max_chunks;
    int with_join; /* d_out / h_out exist (the native writer assembles its own region instead) */
    uint64_t stride;
    uint8_t *h_in, *d_in, *d_slots, *d_out, *h_out;
    uint64_t *h_off, *d_off, *d_joined_off, *h_joined_off;
    uint32_t *h_len, *d_len, *d_out_len, *d_residue, *d_crc, *h_crc;
    uint8_t *h_flags, *d_flags;
    uint64_t *h_eoff, *d_eoff, *h_elen, *d_elen; /* per ENTRY: offset / size of the plain bytes (K7) */
    uint8_t *d_digest, *h_digest;                 /* per entry: 32 bytes */
} zc_bufs;

#define ZC_PIECES 23
/* b's buffers for its capacities into t; returns their number */
static int zc_pieces(zc_bufs *b, mzh_piece *t) {
    const size_t mc = b->max_chunks, join = b->with_join ? mc * b->stride : 0;
    int n = 0;
    t[n++] = MZH_PIN(b->h_in, b->round_bytes + 64);
    t[n++] = MZH_DEV(b->d_in, b->round_bytes + 64);
    t[n++] = MZH_DEV(b->d_slots, mc * b->stride);
    t[n++] = MZH_DEV(b->d_out, join);
    t[n++] = MZH_PIN(b->h_out, join);
    t[n++] = MZH_PIN(b->h_off, mc * 8);
    t[n++] = MZH_DEV(b->d_off, mc * 8);
    t[n++] = MZH_DEV(b->d_joined_off, (mc + 1) * 8);
    t[n++] = MZH_PIN(b->h_joined_off, (mc + 1) * 8);
    t[n++] = MZH_PIN(b->h_len, mc * 4);
    t[n++] = MZH_DEV(b->d_len, mc * 4);
    t[n++] = MZH_DEV(b->d_out_len, mc * 4);
    t[n++] = MZH_DEV(b->d_residue, mc * 4);
    t[n++] = MZH_DEV(b->d_crc, mc * 4);
    t[n++] = MZH_PIN(b->h_crc, mc * 4);
    t[n++] = MZH_PIN(b->h_flags, mc);
    t[n++] = MZH_DEV(b->d_flags, mc);
    t[n++] = MZH_PIN(b->h_eoff, mc * 8); /* an entry has at least one chunk */
    t[n++] = MZH_DEV(b->d_eoff, mc * 8);
    t[n++] = MZH_PIN(b->h_elen, mc * 8);
    t[n++] = MZH_DEV(b->d_elen, mc * 8);
    t[n++] = MZH_DEV(b->d_digest, mc * 32);
    t[n++] = MZH_PIN(b->h_digest, mc * 32);
    return n;
}

static void zc_free(zc_bufs *b) {
    mzh_piece t[ZC_PIECES];
    mzh_free(t, zc_pieces(b, t));
    memset(b, 0, sizeof(*b));
}

static int zc_alloc(zc_bufs *b, size_t round_bytes, uint32_t max_chunks, int with_join) {
    mzh_piece t[ZC_PIECES];
    memset(b, 0, sizeof(*b));
    b->round_bytes = round_bytes;
    b->max_chunks = max_chunks;
    b->with_join = with_join;
    b->stride = mz_cuda_deflate_slot_bound(ZC_CHUNK);
    return mzh_alloc(t, zc_pieces(b, t));
}

static uint32_t chunks_of(int64_t size) {
    return size <= 0 ? 1u : (uint32_t)(((uint64_t)size + ZC_CHUNK - 1) / ZC_CHUNK);
}

/* one round = consecutive entries that fit the staging buffers; prepared (packed, compressed, downloaded) by a
 * worker thread while the caller's thread hands the previous round to the container */
typedef struct zc_round_s {
    zc_bufs b;
    const mz_cuda_zip_item *items;
    uint32_t count, first, last, nch;
    int16_t level;
    uint32_t flags;
    int32_t device, err;
    double pack_ms, gpu_ms;
} zc_round;

static void *zc_prepare(void *arg) {
    zc_round *r = (zc_round *)arg;
    zc_bufs *b = &r->b;
    int32_t err = mz_cuda_set_device(r->device);
    double t0 = now_ms();
    uint32_t last = r->first, nch = 0;
    size_t pos = 0;
    while (last < r->count) {
        const size_t need = ((size_t)r->items[last].size + 15) & ~(size_t)15;
        const uint32_t c = chunks_of(r->items[last].size);
        if (last > r->first && (pos + need > b->round_bytes || nch + c > b->max_chunks))
            break;
        if (r->items[last].size > 0)
            memcpy(b->h_in + pos, r->items[last].data, (size_t)r->items[last].size);
        b->h_eoff[last - r->first] = pos;
        b->h_elen[last - r->first] = (uint64_t)r->items[last].size;
        int64_t left = r->items[last].size;
        for (uint32_t k = 0; k < c; k++) {
            const uint32_t n = left > (int64_t)ZC_CHUNK ? ZC_CHUNK : (uint32_t)left;
            b->h_off[nch] = pos + (uint64_t)k * ZC_CHUNK;
            b->h_len[nch] = n;
            b->h_flags[nch] = (k + 1 == c ? 1u : 0u) | (k > 0 ? 2u : 0u); /* BFINAL on the entry's last chunk; later chunks of an entry may refer back into the one before (MZ_CUDA_FLAG_DICT) */
            left -= n;
            nch++;
        }
        pos += need;
        last++;
    }
    r->last = last;
    r->nch = nch;
    if (!err) err = mz_cuda_memcpy_h2d(b->d_in, b->h_in, pos + 16, NULL);
    if (!err) err = mz_cuda_memcpy_h2d(b->d_off, b->h_off, (size_t)nch * 8, NULL);
    if (!err) err = mz_cuda_memcpy_h2d(b->d_len, b->h_len, (size_t)nch * 4, NULL);
    if (!err) err = mz_cuda_memcpy_h2d(b->d_flags, b->h_flags, nch, NULL);
    double t1 = now_ms();
    /* device: compress, checksum, join; download */
    if (!err) err = mz_cuda_deflate_chunks(b->d_in, 0, 0, b->d_off, b->d_len, b->d_flags, nch, 0, r->level, b->d_slots, b->stride, b->d_out_len, NULL);
    if (!err) err = mz_cuda_crc32_segments(b->d_in, 0, 0, b->d_off, b->d_len, nch, b->d_residue, b->d_crc, NULL);
    if (!err) err = mz_cuda_concat(b->d_slots, b->stride, b->d_out_len, nch, b->d_joined_off, b->d_out, NULL);
    if (!err && (r->flags & MZ_ZIP_CUDA_HASH_SHA256)) { /* K7: SHA-256 of every entry's plain bytes */
        const uint32_t ne = last - r->first;
        err = mz_cuda_memcpy_h2d(b->d_eoff, b->h_eoff, (size_t)ne * 8, NULL);
        if (!err) err = mz_cuda_memcpy_h2d(b->d_elen, b->h_elen, (size_t)ne * 8, NULL);
        if (!err) err = mz_cuda_sha256_batch(b->d_in, b->d_eoff, b->d_elen, ne, b->d_digest, NULL);
        if (!err) err = mz_cuda_memcpy_d2h(b->h_digest, b->d_digest, (size_t)ne * 32, NULL);
    }
    if (!err) err = mz_cuda_memcpy_d2h(b->h_joined_off, b->d_joined_off, ((size_t)nch + 1) * 8, NULL);
    if (!err) err = mz_cuda_memcpy_d2h(b->h_crc, b->d_crc, (size_t)nch * 4, NULL);
    if (!err) err = mz_cuda_stream_sync(NULL);
    if (!err) err = mz_cuda_memcpy_d2h(b->h_out, b->d_out, (size_t)b->h_joined_off[nch], NULL);
    if (!err) err = mz_cuda_stream_sync(NULL);
    r->pack_ms = t1 - t0;
    r->gpu_ms = now_ms() - t1;
    r->err = err;
    return NULL;
}

int32_t mz_zip_cuda_add_buffers(void *zip_handle, const mz_cuda_zip_item *items, uint32_t count, int16_t level, mz_cuda_zip_stats *stats) {
    return mz_zip_cuda_add_buffers_ex(zip_handle, items, count, level, 0, stats);
}

int32_t mz_zip_cuda_add_buffers_ex(void *zip_handle, const mz_cuda_zip_item *items, uint32_t count, int16_t level, uint32_t flags,
                                   mz_cuda_zip_stats *stats) {
    zc_round rd[2];
    int32_t err = MZ_OK;
    mz_cuda_zip_stats st;
    memset(&st, 0, sizeof(st));
    memset(rd, 0, sizeof(rd));
    if (!mz_zip_entry_write_open || !mz_zip_entry_write || !mz_zip_entry_close_raw)
        return MZ_SUPPORT_ERROR; /* no zip container in this process */
    if (!zip_handle || (!items && count))
        return MZ_PARAM_ERROR;
    if (level == MZ_COMPRESS_LEVEL_DEFAULT)
        level = 6;
    if (level < 0 || level > 9)
        return MZ_PARAM_ERROR;
    if (mzh_gpu_required("mz_zip_cuda"))
        return MZ_SUPPORT_ERROR;
    for (uint32_t i = 0; i < count; i++)
        if (!items[i].filename || items[i].size < 0 || (items[i].size > 0 && !items[i].data))
            return MZ_PARAM_ERROR;
    if (count == 0) {
        if (stats)
            *stats = st;
        return MZ_OK;
    }
    size_t round_bytes = mzh_round_bytes(256);
    /* an entry is never split over rounds: the round must hold the largest one */
    for (uint32_t i = 0; i < count; i++)
        if ((size_t)items[i].size + 16 > round_bytes)
            round_bytes = ((size_t)items[i].size + 16 + 65535) & ~(size_t)65535;
    /* chunks per round: full chunks by size plus one (partial or empty) chunk per entry; size the tables for the
     * densest window of the actual input (entries are packed at 16-byte aligned offsets) */
    uint32_t max_chunks = (uint32_t)(round_bytes / ZC_CHUNK) + 1;
    {
        uint32_t j = 0, ch = 0, best = 0;
        size_t bytes = 0;
        for (uint32_t i = 0; i < count; i++) {
            bytes += ((size_t)items[i].size + 15) & ~(size_t)15;
            ch += chunks_of(items[i].size);
            while (bytes > round_bytes) {
                bytes -= ((size_t)items[j].size + 15) & ~(size_t)15;
                ch -= chunks_of(items[j].size);
                j++;
            }
            if (ch > best)
                best = ch;
        }
        if (best + 1 > max_chunks)
            max_chunks = best + 1;
    }
    const int32_t device = mz_cuda_get_device();
    for (int k = 0; k < 2; k++) {
        if (!zc_alloc(&rd[k].b, round_bytes, max_chunks, 1)) {
            zc_free(&rd[0].b);
            return MZ_MEM_ERROR;
        }
        rd[k].items = items;
        rd[k].count = count;
        rd[k].level = level;
        rd[k].flags = flags;
        rd[k].device = device < 0 ? 0 : device;
    }
    /* round r is prepared by a worker while this thread feeds round r-1 to the container */
    int cur = 0;
    pthread_t th;
    rd[cur].first = 0;
    zc_prepare(&rd[cur]);
    while (err == MZ_OK) {
        zc_round *r = &rd[cur];
        err = r->err;
        if (err)
            break;
        int have_next = r->last < count, started = 0;
        if (have_next) {
            rd[cur ^ 1].first = r->last;
            started = pthread_create(&th, NULL, zc_prepare, &rd[cur ^ 1]) == 0;
            if (!started)
                zc_prepare(&rd[cur ^ 1]);
        }
        /* ---- container: the reference writes headers and copies the finished streams --------------------------- */
        double t2 = now_ms();
        const zc_bufs *b = &r->b;
        uint32_t c0 = 0;
        for (uint32_t i = r->first; i < r->last && err == MZ_OK; i++) {
            const uint32_t c = chunks_of(items[i].size);
            uint32_t crc = b->h_crc[c0];
            for (uint32_t k = 1; k < c; k++)
                crc = mz_cuda_crc32_combine(crc, b->h_crc[c0 + k], b->h_len[c0 + k]);
            if (items[i].size == 0)
                crc = 0;
            const uint8_t *comp = b->h_out + b->h_joined_off[c0];
            const uint64_t csize = b->h_joined_off[c0 + c] - b->h_joined_off[c0];
            zc_file_info fi;
            memset(&fi, 0, sizeof(fi));
            fi.version_madeby = (3u << 8) | 45u; /* MZ_HOST_SYSTEM_UNIX (mz.h:104), zip 4.5 as MZ_VERSION_MADEBY without extra codecs (mz_os.h:27-42) */
            /* MZ_ZIP_FLAG_UTF8 (mz.h:84) | MZ_ZIP_FLAG_DATA_DESCRIPTOR (mz.h:83): like the reference's own compressed
             * entries (mz_zip.c:1992) the sizes follow the data, so close_raw never seeks back to patch the header */
            fi.flag = (1u << 11) | (1u << 3);
            fi.compression_method = 8;           /* MZ_COMPRESS_METHOD_DEFLATE, mz.h:64 */
            fi.modified_date = items[i].modified_date ? (time_t)items[i].modified_date : time(NULL);
            fi.crc = crc;
            fi.compressed_size = (int64_t)csize;
            fi.uncompressed_size = items[i].size;
            fi.external_fa = items[i].external_fa ? items[i].external_fa : (0100644u << 16);
            fi.filename = items[i].filename;
            uint8_t xf[40];
            if (flags & MZ_ZIP_CUDA_HASH_SHA256) {
                /* MZ_ZIP_EXTENSION_HASH (mz.h:93): id, field length 4 + 32, algorithm MZ_HASH_SHA256 (mz.h:131), digest size, digest --
                 * the bytes mz_zip_writer_entry_close assembles (mz_zip_rw.c:1398-1408) */
                static const uint8_t head[8] = {0x51, 0x1a, 36, 0, 23, 0, 32, 0};
                memcpy(xf, head, 8);
                memcpy(xf + 8, b->h_digest + (size_t)(i - r->first) * 32, 32);
                fi.extrafield = xf;
                fi.extrafield_size = 40;
            }
            err = mz_zip_entry_write_open(zip_handle, &fi, level, 1, NULL);
            uint64_t done = 0;
            while (err == MZ_OK && done < csize) {
                const int32_t piece = csize - done > (1u << 30) ? (int32_t)(1u << 30) : (int32_t)(csize - done);
                const int32_t w = mz_zip_entry_write(zip_handle, comp + done, piece);
                if (w != piece)
                    err = w < 0 ? w : MZ_WRITE_ERROR;
                done += (uint64_t)piece;
            }
            if (err == MZ_OK)
                err = mz_zip_entry_close_raw(zip_handle, items[i].size, crc);
            st.bytes_in += (uint64_t)items[i].size;
            st.bytes_out += csize;
            c0 += c;
        }
        st.container_ms += now_ms() - t2;
        st.pack_ms += r->pack_ms;
        st.gpu_ms += r->gpu_ms;
        st.entries += r->last - r->first;
        st.rounds++;
        if (started)
            pthread_join(th, NULL);
        if (!have_next)
            break;
        cur ^= 1;
    }
    zc_free(&rd[0].b);
    zc_free(&rd[1].b);
    if (stats)
        *stats = st;
    return err;
}

/* ---- the native archive writer (mz_zip_cuda_write_archive) ------------------------------------------------------------- */
typedef struct za_meta_s { /* per entry of a round, filled by the worker */
    uint64_t csize, lh_rel; /* compressed bytes; offset of the local header inside the round's region */
    uint32_t crc, lh_size;
} za_meta;

typedef struct za_slot_s {
    zc_bufs b;
    uint32_t *h_out_len;               /* pinned: per chunk */
    uint64_t *h_dst_off, *d_dst_off;   /* per chunk: where its stream goes inside the region */
    uint64_t *h_hdr_off, *d_hdr_off;   /* per entry: where its local header goes */
    uint32_t *h_blob_off, *d_blob_off; /* per entry + 1: header bytes inside the blob */
    uint8_t *h_blob, *d_blob;
    size_t blob_cap;
    uint8_t *d_region, *h_region;
    size_t region_cap;
    za_meta *meta;
    /* the round in flight */
    const mz_cuda_zip_item *items;
    uint32_t first, last, nch;
    uint32_t flags;
    int16_t level;
    int32_t device, err;
    uint64_t region_len;
    double pack_ms, gpu_ms;
    void *stream; /* the slot's own CUDA stream: rounds of different slots (and devices) overlap */
    /* WinZip AES (flag MZ_ZIP_CUDA_AES): per entry a salt, derived keys, where its ciphertext lies in the region, its HMAC */
    const char *password;
    uint32_t strength, pw_len;
    uint8_t *h_salt, *d_salt, *h_keys, *d_keys, *d_pw, *h_mac, *d_mac;
    uint64_t *h_coff, *d_coff, *h_clen, *d_clen;
    pthread_t th;
    int running;
    int has_aes; /* the AES buffers exist (pool matching) */
} za_slot;

static void put16(uint8_t *p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); }
static void put32(uint8_t *p, uint32_t v) { put16(p, v); put16(p + 2, v >> 16); }
static void put64(uint8_t *p, uint64_t v) { put32(p, (uint32_t)v); put32(p + 4, (uint32_t)(v >> 32)); }

/* mz_zip_time_t_to_dos_date (mz_zip.c): local time, 2-second resolution, years from 1980 */
static uint32_t za_dos_date(int64_t t) {
    static __thread int64_t last_t = -1; /* archives carry few distinct dates: localtime_r once per run of equal ones */
    static __thread uint32_t last_v;
    if (t && t == last_t)
        return last_v;
    time_t tt = (time_t)(t ? t : time(NULL));
    struct tm tmv;
    if (!localtime_r(&tt, &tmv))
        return 0;
    int year = tmv.tm_year >= 1980 ? tmv.tm_year - 1980 : (tmv.tm_year >= 80 ? tmv.tm_year - 80 : 0);
    last_v = ((uint32_t)((tmv.tm_mday) + 32 * (tmv.tm_mon + 1) + 512 * year) << 16) |
             (uint32_t)(tmv.tm_sec / 2 + 32 * tmv.tm_min + 2048 * tmv.tm_hour);
    last_t = t;
    return last_v;
}

#define ZA_PIECES (ZC_PIECES + 22)
/* z's buffers for its capacities into t (zc_bufs' first); the WinZip AES ones have no bytes without has_aes */
static int za_pieces(za_slot *z, mzh_piece *t) {
    const size_t mc = z->b.max_chunks, aes = z->has_aes ? 1 : 0;
    int n = zc_pieces(&z->b, t);
    t[n++] = MZH_PIN(z->h_out_len, mc * 4);
    t[n++] = MZH_PIN(z->h_dst_off, mc * 8);
    t[n++] = MZH_DEV(z->d_dst_off, mc * 8);
    t[n++] = MZH_PIN(z->h_hdr_off, mc * 8);
    t[n++] = MZH_DEV(z->d_hdr_off, mc * 8);
    t[n++] = MZH_PIN(z->h_blob_off, (mc + 1) * 4);
    t[n++] = MZH_DEV(z->d_blob_off, (mc + 1) * 4);
    t[n++] = MZH_PIN(z->h_blob, z->blob_cap + 16);
    t[n++] = MZH_DEV(z->d_blob, z->blob_cap + 16);
    t[n++] = MZH_DEV(z->d_region, z->region_cap);
    t[n++] = MZH_PIN(z->h_region, z->region_cap);
    t[n++] = MZH_PIN(z->h_salt, aes * mc * 16);
    t[n++] = MZH_DEV(z->d_salt, aes * mc * 16);
    t[n++] = MZH_PIN(z->h_keys, aes * mc * MZ_CUDA_WZAES_KEYREC);
    t[n++] = MZH_DEV(z->d_keys, aes * mc * MZ_CUDA_WZAES_KEYREC);
    t[n++] = MZH_DEV(z->d_pw, aes * 256);
    t[n++] = MZH_PIN(z->h_mac, aes * mc * 20);
    t[n++] = MZH_DEV(z->d_mac, aes * mc * 20);
    t[n++] = MZH_PIN(z->h_coff, aes * mc * 8);
    t[n++] = MZH_DEV(z->d_coff, aes * mc * 8);
    t[n++] = MZH_PIN(z->h_clen, aes * mc * 8);
    t[n++] = MZH_DEV(z->d_clen, aes * mc * 8);
    return n;
}

static void za_free(za_slot *z) {
    mzh_piece t[ZA_PIECES];
    mzh_free(t, za_pieces(z, t));
    if (z->stream)
        mz_cuda_stream_destroy(z->stream);
    free(z->meta);
    memset(z, 0, sizeof(*z));
}

/* a new slot for the capacities and device set in *z */
static int za_alloc(za_slot *z) {
    mzh_piece t[ZA_PIECES];
    const uint32_t max_chunks = z->b.max_chunks;
    z->b.stride = mz_cuda_deflate_slot_bound(ZC_CHUNK);
    z->region_cap = (size_t)max_chunks * z->b.stride + z->blob_cap + 64;
    if (!mzh_alloc(t, za_pieces(z, t)))
        return 0;
    z->meta = (za_meta *)malloc((size_t)max_chunks * sizeof(za_meta));
    z->stream = mz_cuda_stream_create();
    if (!z->meta || !z->stream) {
        za_free(z);
        return 0;
    }
    return 1;
}

/* One round of extraction on the device (K9 locate, K8, K9 stored copy, K5, K1, K7, K9 verify): the slot's staging, its CUDA
 * stream, and the round in flight. Both extractors fill h_in and h_ent and call zr_run; mz_zip_cuda_extract_archive keeps up to
 * four slots in flight on their own threads and pools them between calls (like the native writer's), mz_zip_cuda_extract_all
 * runs one synchronously. mz_zip_cuda_extract_device and the reader carve the round arrays alone (zd_carve). */
typedef struct zr_slot_s {
    size_t in_cap, out_cap;
    uint32_t max_ent;
    int32_t device;
    uint8_t *h_in, *d_in, *h_out, *d_out;
    mz_cuda_zip_ent *h_ent, *d_ent;
    uint8_t *h_sha, *d_sha;
    uint32_t *h_status, *d_status;
    mz_cuda_inflate_job *d_job;
    mz_cuda_inflate_state *d_state;
    uint64_t *d_seg_off, *d_seg_len64, *d_data_off, *d_coff, *d_clen;
    uint32_t *d_seg_len, *d_residue, *d_crc;
    uint8_t *d_digest, *d_salt, *d_keys, *d_pw, *d_mac;
    void *stream;
    /* the round in flight */
    uint32_t first, last, n, njobs, nsha, na[4];
    uint64_t max_clen[4];
    size_t in_used, out_used;
    const char *password;
    int32_t err;
    double gpu_ms;
    pthread_t th;
    int running;
} zr_slot;

#define ZR_ROUND_PIECES 16
/* the arrays zr_launch uses for a round of m entries, digest_rows of them for K7's digests, into t; returns their number */
static int zr_round_pieces(zr_slot *z, size_t m, size_t digest_rows, mzh_piece *t) {
    int n = 0;
    t[n++] = MZH_DEV(z->d_status, m * 4);
    t[n++] = MZH_DEV(z->d_job, m * sizeof(mz_cuda_inflate_job));
    t[n++] = MZH_DEV(z->d_state, m * sizeof(mz_cuda_inflate_state));
    t[n++] = MZH_DEV(z->d_seg_off, m * 8);
    t[n++] = MZH_DEV(z->d_seg_len64, m * 8);
    t[n++] = MZH_DEV(z->d_data_off, m * 8);
    t[n++] = MZH_DEV(z->d_coff, m * 8);
    t[n++] = MZH_DEV(z->d_clen, m * 8);
    t[n++] = MZH_DEV(z->d_seg_len, m * 4);
    t[n++] = MZH_DEV(z->d_residue, m * 4);
    t[n++] = MZH_DEV(z->d_crc, m * 4);
    t[n++] = MZH_DEV(z->d_digest, digest_rows * 32);
    t[n++] = MZH_DEV(z->d_salt, m * 16);
    t[n++] = MZH_DEV(z->d_keys, m * MZ_CUDA_WZAES_KEYREC);
    t[n++] = MZH_DEV(z->d_pw, 256);
    t[n++] = MZH_DEV(z->d_mac, m * 20);
    return n;
}

#define ZR_PIECES (9 + ZR_ROUND_PIECES)
/* z's staging and round arrays for its capacities into t. in_cap: stored bytes of a round (+ 64 readable bytes past them); out_cap:
 * plain bytes (+ 512); max_ent: entries */
static int zr_pieces(zr_slot *z, mzh_piece *t) {
    const size_t m = z->max_ent;
    int n = 0;
    t[n++] = MZH_PIN(z->h_in, z->in_cap + 64);
    t[n++] = MZH_DEV(z->d_in, z->in_cap + 64);
    t[n++] = MZH_PIN(z->h_out, z->out_cap + 512);
    t[n++] = MZH_DEV(z->d_out, z->out_cap + 512);
    t[n++] = MZH_PIN(z->h_ent, m * sizeof(mz_cuda_zip_ent));
    t[n++] = MZH_DEV(z->d_ent, m * sizeof(mz_cuda_zip_ent));
    t[n++] = MZH_PIN(z->h_sha, m * 32);
    t[n++] = MZH_DEV(z->d_sha, m * 32);
    t[n++] = MZH_PIN(z->h_status, m * 4);
    return n + zr_round_pieces(z, m, m, t + n);
}

static void zr_free(zr_slot *z) {
    mzh_piece t[ZR_PIECES];
    mzh_free(t, zr_pieces(z, t));
    if (z->stream)
        mz_cuda_stream_destroy(z->stream);
    memset(z, 0, sizeof(*z));
}

/* a new slot for the capacities set in *z, with its own stream or none (mz_zip_cuda_extract_all) */
static int zr_alloc(zr_slot *z, int with_stream) {
    mzh_piece t[ZR_PIECES];
    if (!mzh_alloc(t, zr_pieces(z, t)))
        return 0;
    z->stream = with_stream ? mz_cuda_stream_create() : NULL;
    if (with_stream && !z->stream) {
        zr_free(z);
        return 0;
    }
    return 1;
}

/* Staging pool: a writer slot is ~130 MiB of page-locked and ~200 MiB of device memory, and making four of them costs more than half
 * a second -- as much as compressing 2 GiB. A process that writes or extracts archive after archive keeps up to eight idle slots of
 * each kind, writer (za_slot) and extractor (zr_slot), per device and matched by capacity; MZ_CUDA_ZIP_POOL=0 turns the pool off,
 * mz_zip_cuda_trim() empties it. */
#define ZA_POOL_MAX 8
enum { ZP_WRITER, ZP_EXTRACTOR };
typedef union zp_slot_u {
    za_slot w;
    zr_slot x;
} zp_slot;
static pthread_mutex_t g_zp_mu = PTHREAD_MUTEX_INITIALIZER;
static zp_slot g_zp[2][ZA_POOL_MAX];
static int g_zp_n[2];

static int zp_enabled(void) {
    const char *v = getenv("MZ_CUDA_ZIP_POOL");
    return !(v && v[0] == '0');
}

/* does the idle slot q serve the request r? Same device and capacities at least r's; a writer slot with the WinZip AES buffers
 * serves a plain request, not the reverse */
static int zp_serves(int kind, const zp_slot *q, const void *r) {
    if (kind == ZP_WRITER) {
        const za_slot *w = (const za_slot *)r;
        return q->w.device == w->device && q->w.b.round_bytes >= w->b.round_bytes && q->w.b.max_chunks >= w->b.max_chunks &&
               q->w.blob_cap >= w->blob_cap && (q->w.has_aes || !w->has_aes);
    }
    const zr_slot *x = (const zr_slot *)r;
    return q->x.device == x->device && q->x.in_cap >= x->in_cap && q->x.out_cap >= x->out_cap && q->x.max_ent >= x->max_ent;
}

static void zp_free(int kind, void *z) {
    if (kind == ZP_WRITER)
        za_free((za_slot *)z);
    else
        zr_free((zr_slot *)z);
}

/* *z (a za_slot or zr_slot) holds the request: its device and capacities. An idle slot that serves it replaces it, with the round in
 * flight cleared; else a new slot is made. 0 when that fails. */
static int zp_acquire(int kind, void *z) {
    const size_t size = kind == ZP_WRITER ? sizeof(za_slot) : sizeof(zr_slot);
    int hit = 0;
    pthread_mutex_lock(&g_zp_mu);
    for (int i = 0; i < g_zp_n[kind] && !hit; i++) {
        if ((hit = zp_serves(kind, &g_zp[kind][i], z))) {
            memcpy(z, &g_zp[kind][i], size);
            g_zp[kind][i] = g_zp[kind][--g_zp_n[kind]];
        }
    }
    pthread_mutex_unlock(&g_zp_mu);
    if (!hit)
        return kind == ZP_WRITER ? za_alloc((za_slot *)z) : zr_alloc((zr_slot *)z, 1);
    if (kind == ZP_WRITER) {
        za_slot *w = (za_slot *)z;
        w->items = NULL;
        w->first = w->last = w->nch = 0;
        w->err = 0;
        w->region_len = 0;
        w->pack_ms = w->gpu_ms = 0;
        w->running = 0;
        w->password = NULL;
    } else {
        zr_slot *x = (zr_slot *)z;
        x->running = 0;
        x->err = 0;
    }
    return 1;
}

/* *z back to the pool, or freed: the pool is off or full, or z has no staging, or no stream (mz_zip_cuda_extract_all) */
static void zp_release(int kind, void *z) {
    const size_t size = kind == ZP_WRITER ? sizeof(za_slot) : sizeof(zr_slot);
    const int whole = kind == ZP_WRITER ? ((za_slot *)z)->b.h_in != NULL : ((zr_slot *)z)->h_in && ((zr_slot *)z)->stream;
    int kept = 0;
    if (whole && zp_enabled()) {
        pthread_mutex_lock(&g_zp_mu);
        if (g_zp_n[kind] < ZA_POOL_MAX) {
            memcpy(&g_zp[kind][g_zp_n[kind]++], z, size);
            kept = 1;
        }
        pthread_mutex_unlock(&g_zp_mu);
    }
    if (kept)
        memset(z, 0, size);
    else
        zp_free(kind, z);
}

void mz_zip_cuda_trim(void) {
    const int32_t dev0 = mz_cuda_get_device();
    pthread_mutex_lock(&g_zp_mu);
    for (int kind = ZP_WRITER; kind <= ZP_EXTRACTOR; kind++) {
        for (int i = 0; i < g_zp_n[kind]; i++) {
            zp_slot *q = &g_zp[kind][i];
            mz_cuda_set_device(kind == ZP_WRITER ? q->w.device : q->x.device);
            zp_free(kind, q);
        }
        g_zp_n[kind] = 0;
    }
    pthread_mutex_unlock(&g_zp_mu);
    if (dev0 >= 0)
        mz_cuda_set_device(dev0);
}

/* the hash extra field of an entry (40 bytes) -- the bytes mz_zip_writer_entry_close assembles (mz_zip_rw.c:1398-1408) */
static void za_hash_field(uint8_t *xf, const uint8_t *digest) {
    static const uint8_t head[8] = {0x51, 0x1a, 36, 0, 23, 0, 32, 0};
    memcpy(xf, head, 8);
    memcpy(xf + 8, digest, 32);
}

/* the AES extra field of an entry (11 bytes): id 0x9901, size 7, AE version, vendor "AE", strength, the real method
 * (mz_zip.c:870-885) */
static void za_aes_field(uint8_t *xf, uint32_t strength) {
    const uint8_t f[11] = {0x01, 0x99, 7, 0, 1, 0, 'A', 'E', (uint8_t)strength, 8, 0};
    memcpy(xf, f, 11);
}

/* one round: pack, upload, compress + checksum (+ hash), lay the region out, assemble it on the device, download it */
static void *za_prepare(void *arg) {
    za_slot *z = (za_slot *)arg;
    zc_bufs *b = &z->b;
    int32_t err = mz_cuda_set_device(z->device);
    double t0 = now_ms();
    uint32_t nch = 0;
    size_t pos = 0;
    const uint32_t ne = z->last - z->first;
    for (uint32_t i = z->first; i < z->last; i++) {
        const mz_cuda_zip_item *it = &z->items[i];
        const uint32_t c = chunks_of(it->size);
        if (it->size > 0)
            memcpy(b->h_in + pos, it->data, (size_t)it->size);
        b->h_eoff[i - z->first] = pos;
        b->h_elen[i - z->first] = (uint64_t)it->size;
        int64_t left = it->size;
        for (uint32_t k = 0; k < c; k++) {
            const uint32_t n = left > (int64_t)ZC_CHUNK ? ZC_CHUNK : (uint32_t)left;
            b->h_off[nch] = pos + (uint64_t)k * ZC_CHUNK;
            b->h_len[nch] = n;
            b->h_flags[nch] = (k + 1 == c ? 1u : 0u) | (k > 0 ? 2u : 0u); /* FINAL | DICT, as above */
            left -= n;
            nch++;
        }
        pos += ((size_t)it->size + 15) & ~(size_t)15;
    }
    z->nch = nch;
    if (!err) err = mz_cuda_memcpy_h2d(b->d_in, b->h_in, pos + 16, z->stream);
    if (!err) err = mz_cuda_memcpy_h2d(b->d_off, b->h_off, (size_t)nch * 8, z->stream);
    if (!err) err = mz_cuda_memcpy_h2d(b->d_len, b->h_len, (size_t)nch * 4, z->stream);
    if (!err) err = mz_cuda_memcpy_h2d(b->d_flags, b->h_flags, nch, z->stream);
    double t1 = now_ms();
    const int aes = (z->flags & MZ_ZIP_CUDA_AES) != 0;
    const uint32_t slen = aes ? 4 * z->strength + 4 : 0; /* MZ_AES_SALT_LENGTH */
    if (!err && aes) { /* a fresh salt per entry (mz_strm_wzaes.c:85-86), then every entry's keys and password verifier by K8 */
        size_t got = 0;
        while (got < (size_t)ne * 16) {
            ssize_t k = getrandom(z->h_salt + got, (size_t)ne * 16 - got, 0);
            if (k <= 0) { err = MZ_INTERNAL_ERROR; break; }
            got += (size_t)k;
        }
        if (!err) err = mz_cuda_memcpy_h2d(z->d_salt, z->h_salt, (size_t)ne * 16, z->stream);
        if (!err) err = mz_cuda_memcpy_h2d(z->d_pw, z->password, z->pw_len ? z->pw_len : 1, z->stream);
        if (!err) err = mz_cuda_wzaes_derive(z->d_pw, z->pw_len, z->d_salt, ne, z->strength, z->d_keys, z->stream);
        if (!err) err = mz_cuda_memcpy_d2h(z->h_keys, z->d_keys, (size_t)ne * MZ_CUDA_WZAES_KEYREC, z->stream);
    }
    if (!err) err = mz_cuda_deflate_chunks(b->d_in, 0, 0, b->d_off, b->d_len, b->d_flags, nch, 0, z->level, b->d_slots, b->stride, b->d_out_len, z->stream);
    if (!err) err = mz_cuda_crc32_segments(b->d_in, 0, 0, b->d_off, b->d_len, nch, b->d_residue, b->d_crc, z->stream);
    if (!err && (z->flags & MZ_ZIP_CUDA_HASH_SHA256)) {
        err = mz_cuda_memcpy_h2d(b->d_eoff, b->h_eoff, (size_t)ne * 8, z->stream);
        if (!err) err = mz_cuda_memcpy_h2d(b->d_elen, b->h_elen, (size_t)ne * 8, z->stream);
        if (!err) err = mz_cuda_sha256_batch(b->d_in, b->d_eoff, b->d_elen, ne, b->d_digest, z->stream);
        if (!err) err = mz_cuda_memcpy_d2h(b->h_digest, b->d_digest, (size_t)ne * 32, z->stream);
    }
    if (!err) err = mz_cuda_memcpy_d2h(z->h_out_len, b->d_out_len, (size_t)nch * 4, z->stream);
    if (!err) err = mz_cuda_memcpy_d2h(b->h_crc, b->d_crc, (size_t)nch * 4, z->stream);
    if (!err) err = mz_cuda_stream_sync(z->stream);
    /* host: sizes, CRCs, local headers, the region's layout */
    uint64_t cur = 0, max_clen = 0;
    uint32_t c0 = 0, bo = 0;
    for (uint32_t e = 0; e < ne && !err; e++) {
        const mz_cuda_zip_item *it = &z->items[z->first + e];
        const uint32_t c = chunks_of(it->size);
        uint32_t crc = b->h_crc[c0];
        uint64_t csize = z->h_out_len[c0];
        for (uint32_t k = 1; k < c; k++) {
            crc = mz_cuda_crc32_combine(crc, b->h_crc[c0 + k], b->h_len[c0 + k]);
            csize += z->h_out_len[c0 + k];
        }
        if (it->size == 0)
            crc = 0;
        const size_t nlen = strlen(it->filename);
        const uint32_t xaes = aes ? 11u : 0u;
        const uint32_t xlen = xaes + ((z->flags & MZ_ZIP_CUDA_HASH_SHA256) ? 40u : 0u);
        const uint32_t lh = 30 + (uint32_t)nlen + xlen;
        const uint64_t stored = csize + (aes ? slen + 2 + 10 : 0); /* salt | verifier | ciphertext | authentication code */
        if (bo + lh + slen + 2 > z->blob_cap || stored >= 0xffffffffull) {
            err = MZ_INTERNAL_ERROR;
            break;
        }
        uint8_t *h = z->h_blob + bo;
        put32(h, 0x04034b50u);                       /* MZ_ZIP_MAGIC_LOCALHEADER */
        put16(h + 4, aes ? 51 : 20);                 /* version needed (mz_zip.c:703-725) */
        put16(h + 6, (1u << 11) | (aes ? 1u : 0u));  /* MZ_ZIP_FLAG_UTF8 (| MZ_ZIP_FLAG_ENCRYPTED); no data descriptor: everything is known */
        put16(h + 8, aes ? 99 : 8);                  /* MZ_COMPRESS_METHOD_DEFLATE, or _AES with the real method in the extra field (:728-733) */
        put32(h + 10, za_dos_date(it->modified_date));
        put32(h + 14, crc);                          /* AE-1 (MZ_AES_VERSION 1) keeps the CRC (mz_zip.c:2117-2121) */
        put32(h + 18, (uint32_t)stored);
        put32(h + 22, (uint32_t)it->size);
        put16(h + 26, (uint32_t)nlen);
        put16(h + 28, xlen);
        memcpy(h + 30, it->filename, nlen);
        if (aes)
            za_aes_field(h + 30 + nlen, z->strength);
        if (xlen > xaes)
            za_hash_field(h + 30 + nlen + xaes, b->h_digest + (size_t)e * 32);
        if (aes) { /* salt and password verifier travel with the header blob (mz_strm_wzaes.c:116-125) */
            memcpy(h + lh, z->h_salt + (size_t)e * 16, slen);
            memcpy(h + lh + slen, z->h_keys + (size_t)e * MZ_CUDA_WZAES_KEYREC + 64, 2);
        }
        z->h_blob_off[e] = bo;
        z->h_hdr_off[e] = cur;
        z->meta[e].csize = stored;
        z->meta[e].crc = crc;
        z->meta[e].lh_rel = cur;
        z->meta[e].lh_size = lh;
        bo += lh + (aes ? slen + 2 : 0);
        cur += lh + (aes ? slen + 2 : 0);
        if (aes) {
            z->h_coff[e] = cur;
            z->h_clen[e] = csize;
            if (csize > max_clen) max_clen = csize;
        }
        for (uint32_t k = 0; k < c; k++) {
            z->h_dst_off[c0 + k] = cur;
            cur += z->h_out_len[c0 + k];
        }
        if (aes)
            cur += 10; /* MZ_AES_AUTHCODE_SIZE */
        c0 += c;
    }
    z->h_blob_off[ne] = bo;
    z->region_len = cur;
    if (!err && cur > z->region_cap)
        err = MZ_INTERNAL_ERROR;
    /* device: streams and headers into place; the finished region comes down in one copy */
    if (!err) err = mz_cuda_memcpy_h2d(z->d_dst_off, z->h_dst_off, (size_t)nch * 8, z->stream);
    if (!err) err = mz_cuda_memcpy_h2d(z->d_hdr_off, z->h_hdr_off, (size_t)ne * 8, z->stream);
    if (!err) err = mz_cuda_memcpy_h2d(z->d_blob_off, z->h_blob_off, ((size_t)ne + 1) * 4, z->stream);
    if (!err) err = mz_cuda_memcpy_h2d(z->d_blob, z->h_blob, (size_t)bo + 16, z->stream);
    if (!err) err = mz_cuda_gather(b->d_slots, b->stride, b->d_out_len, nch, z->d_dst_off, z->d_region, z->stream);
    if (!err) err = mz_cuda_scatter_blobs(z->d_blob, z->d_blob_off, z->d_hdr_off, ne, z->d_region, z->stream);
    if (!err && aes) { /* the assembled streams become ciphertext in place; their HMACs follow them down */
        err = mz_cuda_memcpy_h2d(z->d_coff, z->h_coff, (size_t)ne * 8, z->stream);
        if (!err) err = mz_cuda_memcpy_h2d(z->d_clen, z->h_clen, (size_t)ne * 8, z->stream);
        if (!err) err = mz_cuda_wzaes_ctr(z->d_region, z->d_coff, z->d_clen, ne, max_clen, z->d_keys, z->strength, z->stream);
        if (!err) err = mz_cuda_wzaes_hmac(z->d_region, z->d_coff, z->d_clen, ne, z->d_keys, z->strength, z->d_mac, z->stream);
        if (!err) err = mz_cuda_memcpy_d2h(z->h_mac, z->d_mac, (size_t)ne * 20, z->stream);
    }
    if (!err) err = mz_cuda_memcpy_d2h(z->h_region, z->d_region, (size_t)cur, z->stream);
    if (!err) err = mz_cuda_stream_sync(z->stream);
    for (uint32_t e = 0; e < ne && !err && aes; e++) /* authentication code = the first 10 bytes of the HMAC (mz_strm_wzaes.c:243-247) */
        memcpy(z->h_region + z->h_coff[e] + z->h_clen[e], z->h_mac + (size_t)e * 20, 10);
    z->pack_ms = t1 - t0;
    z->gpu_ms = now_ms() - t1;
    z->err = err;
    return NULL;
}

typedef struct za_cd_s {
    uint8_t *p;
    size_t len, cap;
} za_cd;
static uint8_t *za_cd_room(za_cd *cd, size_t n) {
    if (cd->len + n > cd->cap) {
        size_t ncap = cd->cap ? cd->cap * 2 : (1u << 20);
        while (ncap < cd->len + n)
            ncap *= 2;
        uint8_t *q = (uint8_t *)realloc(cd->p, ncap);
        if (!q)
            return NULL;
        cd->p = q;
        cd->cap = ncap;
    }
    uint8_t *r = cd->p + cd->len;
    cd->len += n;
    return r;
}

static int32_t za_write(void *base, const uint8_t *p, uint64_t n) {
    while (n > 0) {
        const int32_t part = n > (1u << 30) ? (int32_t)(1u << 30) : (int32_t)n;
        if (mz_abi_base_write(base, p, part) != part)
            return MZ_WRITE_ERROR;
        p += part;
        n -= (uint64_t)part;
    }
    return MZ_OK;
}

int32_t mz_zip_cuda_write_archive(void *base_stream, const mz_cuda_zip_item *items, uint32_t count, int16_t level, uint32_t flags,
                                  mz_cuda_zip_stats *stats) {
    if (flags & MZ_ZIP_CUDA_AES)
        return MZ_PARAM_ERROR; /* needs a password: mz_zip_cuda_write_archive_aes */
    return mz_zip_cuda_write_archive_aes(base_stream, items, count, level, flags, NULL, 0, stats);
}

int32_t mz_zip_cuda_write_archive_aes(void *base_stream, const mz_cuda_zip_item *items, uint32_t count, int16_t level, uint32_t flags,
                                      const char *password, uint8_t aes_strength, mz_cuda_zip_stats *stats) {
    mz_cuda_zip_stats st;
    int32_t err = MZ_OK;
    memset(&st, 0, sizeof(st));
    if (!base_stream || (!items && count))
        return MZ_PARAM_ERROR;
    if (level == MZ_COMPRESS_LEVEL_DEFAULT)
        level = 6;
    if (level < 0 || level > 9)
        return MZ_PARAM_ERROR;
    const int aes = (flags & MZ_ZIP_CUDA_AES) != 0;
    if (aes_strength == 0)
        aes_strength = 3; /* MZ_AES_STRENGTH_256, the reference's default (mz_zip.c:2007-2009) */
    if (aes && (!password || strlen(password) > 128 || aes_strength > 3))
        return MZ_PARAM_ERROR; /* MZ_AES_PW_LENGTH_MAX, mz_strm_wzaes.c:77-79 */
    if (mzh_gpu_required("mz_zip_cuda"))
        return MZ_SUPPORT_ERROR;
    /* 64 MiB rounds, four in preparation: each round's entries are packed into pinned staging by its own worker thread (that copy is
     * the slowest stage of a round), and small rounds keep the page-locked allocations -- and the time to make them -- small */
    size_t round_bytes = mzh_round_bytes(64);
    size_t max_name = 0;
    for (uint32_t i = 0; i < count; i++) {
        if (!items[i].filename || items[i].size < 0 || (items[i].size > 0 && !items[i].data))
            return MZ_PARAM_ERROR;
        const size_t nl = strlen(items[i].filename);
        if (nl == 0 || nl > 65535)
            return MZ_PARAM_ERROR;
        if (nl > max_name)
            max_name = nl;
        if (items[i].size >= 0xffff0000ll)
            return MZ_SUPPORT_ERROR; /* zip64-sized ENTRIES take the per-entry path (mz_zip_cuda_add_buffers) */
        if ((size_t)items[i].size + 16 > round_bytes)
            round_bytes = ((size_t)items[i].size + 16 + 65535) & ~(size_t)65535;
    }
    /* rounds: consecutive entries that fit the staging buffers; boundaries depend on the sizes alone, so they are fixed up
     * front and several rounds can be prepared at once */
    uint32_t nrounds = 0, rcap = 16;
    uint32_t *rfirst = (uint32_t *)malloc((rcap + 1) * sizeof(uint32_t));
    uint32_t max_chunks = 1, max_entries = 1;
    size_t max_blob = 64;
    if (!rfirst)
        return MZ_MEM_ERROR;
    {
        uint32_t i = 0;
        while (i < count) {
            size_t bytes = 0, blob = 0;
            uint32_t ch = 0, j = i;
            while (j < count) {
                const size_t need = ((size_t)items[j].size + 15) & ~(size_t)15;
                if (j > i && bytes + need > round_bytes)
                    break;
                bytes += need;
                ch += chunks_of(items[j].size);
                blob += 30 + strlen(items[j].filename) + 40 + 11 + 18; /* header, name, hash field, AES field, salt + verifier */
                j++;
            }
            if (nrounds == rcap) {
                rcap *= 2;
                uint32_t *q = (uint32_t *)realloc(rfirst, (rcap + 1) * sizeof(uint32_t));
                if (!q) {
                    free(rfirst);
                    return MZ_MEM_ERROR;
                }
                rfirst = q;
            }
            rfirst[nrounds++] = i;
            if (ch > max_chunks) max_chunks = ch;
            if (j - i > max_entries) max_entries = j - i;
            if (blob > max_blob) max_blob = blob;
            i = j;
        }
        rfirst[nrounds] = count;
    }
    int32_t ndev = 1;
    const int32_t dev0 = mz_cuda_get_device() < 0 ? 0 : mz_cuda_get_device();
    if (flags & MZ_ZIP_CUDA_ALL_DEVICES) {
        ndev = mz_cuda_device_count();
        if (ndev < 1) ndev = 1;
        if (ndev > 8) ndev = 8;
    }
    const double t_setup0 = now_ms();
    const uint32_t want = ndev > 1 ? (uint32_t)ndev * 2 : 4u;
    const uint32_t nslots = want < nrounds ? want : (nrounds ? nrounds : 1);
    za_slot *slots = (za_slot *)calloc(nslots, sizeof(za_slot));
    za_cd cd = {NULL, 0, 0};
    if (!slots) {
        free(rfirst);
        return MZ_MEM_ERROR;
    }
    for (uint32_t k = 0; k < nslots && err == MZ_OK; k++) {
        za_slot *z = &slots[k];
        z->device = ndev > 1 ? (int32_t)(k % (uint32_t)ndev) : dev0;
        z->b.round_bytes = round_bytes;
        z->b.max_chunks = max_chunks + 1;
        z->blob_cap = max_blob;
        z->has_aes = aes;
        if (mz_cuda_set_device(z->device) != MZ_OK || !zp_acquire(ZP_WRITER, z)) {
            err = MZ_MEM_ERROR;
            break;
        }
        slots[k].items = items;
        slots[k].level = level;
        slots[k].flags = flags;
        slots[k].password = password;
        slots[k].pw_len = aes ? (uint32_t)strlen(password) : 0;
        slots[k].strength = aes_strength;
    }
    mz_cuda_set_device(dev0);
    uint64_t abs_off = 0;
    uint32_t issued = 0;
    st.setup_ms = now_ms() - t_setup0;
    for (uint32_t r = 0; r < nrounds && err == MZ_OK; r++) {
        /* keep every slot busy: rounds r .. r + nslots - 1 are in preparation */
        while (issued < nrounds && issued < r + nslots) {
            za_slot *z = &slots[issued % nslots];
            z->first = rfirst[issued];
            z->last = rfirst[issued + 1];
            z->running = pthread_create(&z->th, NULL, za_prepare, z) == 0;
            if (!z->running)
                za_prepare(z);
            issued++;
        }
        za_slot *z = &slots[r % nslots];
        if (z->running) {
            pthread_join(z->th, NULL);
            z->running = 0;
        }
        err = z->err;
        if (err)
            break;
        const double t2 = now_ms();
        err = za_write(base_stream, z->h_region, z->region_len);
        /* central directory records of the round (mz_zip.c:594-919 with local = 0) */
        for (uint32_t e = 0; e < z->last - z->first && err == MZ_OK; e++) {
            const mz_cuda_zip_item *it = &items[z->first + e];
            const za_meta *m = &z->meta[e];
            const uint64_t lh_off = abs_off + m->lh_rel;
            const int z64 = lh_off >= 0xffffffffull;
            const size_t nlen = strlen(it->filename);
            const uint32_t xhash = (flags & MZ_ZIP_CUDA_HASH_SHA256) ? 40u : 0u;
            const uint32_t xlen = (z64 ? 4u + 24u : 0u) + (aes ? 11u : 0u) + xhash;
            uint8_t *h = za_cd_room(&cd, 46 + nlen + xlen);
            if (!h) {
                err = MZ_MEM_ERROR;
                break;
            }
            put32(h, 0x02014b50u);                   /* MZ_ZIP_MAGIC_CENTRALHEADER */
            put16(h + 4, (3u << 8) | 45u);           /* made by: MZ_HOST_SYSTEM_UNIX, 4.5 */
            put16(h + 6, aes ? 51 : (z64 ? 45 : 20));
            put16(h + 8, (1u << 11) | (aes ? 1u : 0u));
            put16(h + 10, aes ? 99 : 8);
            put32(h + 12, za_dos_date(it->modified_date));
            put32(h + 16, m->crc);
            put32(h + 20, z64 ? 0xffffffffu : (uint32_t)m->csize); /* with a zip64 field both sizes move into it (mz_zip.c:519-548) */
            put32(h + 24, z64 ? 0xffffffffu : (uint32_t)it->size);
            put16(h + 28, (uint32_t)nlen);
            put16(h + 30, xlen);
            put16(h + 32, 0);                        /* comment */
            put16(h + 34, 0);                        /* disk number start */
            put16(h + 36, 0);                        /* internal attributes */
            put32(h + 38, it->external_fa ? it->external_fa : (0100644u << 16));
            put32(h + 42, z64 ? 0xffffffffu : (uint32_t)lh_off);
            memcpy(h + 46, it->filename, nlen);
            uint8_t *x = h + 46 + nlen;
            if (z64) {                               /* MZ_ZIP_EXTENSION_ZIP64: uncompressed, compressed, header offset */
                put16(x, 0x0001);
                put16(x + 2, 24);
                put64(x + 4, (uint64_t)it->size);
                put64(x + 12, m->csize);
                put64(x + 20, lh_off);
                x += 28;
            }
            if (aes) {
                za_aes_field(x, aes_strength);
                x += 11;
            }
            if (xhash)
                za_hash_field(x, z->b.h_digest + (size_t)e * 32);
            st.bytes_in += (uint64_t)it->size;
            st.bytes_out += m->csize;
        }
        abs_off += z->region_len;
        st.container_ms += now_ms() - t2;
        st.pack_ms += z->pack_ms;
        st.gpu_ms += z->gpu_ms;
        st.entries += z->last - z->first;
        st.rounds++;
    }
    for (uint32_t k = 0; k < nslots; k++)
        if (slots[k].running) {
            pthread_join(slots[k].th, NULL);
            slots[k].running = 0;
        }
    /* central directory + end records (mz_zip.c:1102-1234) */
    if (err == MZ_OK) {
        const uint64_t cd_off = abs_off, cd_size = cd.len;
        uint8_t tail[56 + 20 + 22];
        size_t tl = 0;
        err = za_write(base_stream, cd.p, cd.len);
        if (cd_off >= 0xffffffffull || count >= 0xffffu) {
            uint8_t *q = tail;
            put32(q, 0x06064b50u);                   /* MZ_ZIP_MAGIC_ENDHEADER64 */
            put64(q + 4, 44);
            put16(q + 12, (3u << 8) | 45u);
            put16(q + 14, 45);
            put32(q + 16, 0);
            put32(q + 20, 0);
            put64(q + 24, count);
            put64(q + 32, count);
            put64(q + 40, cd_size);
            put64(q + 48, cd_off);
            q += 56;
            put32(q, 0x07064b50u);                   /* MZ_ZIP_MAGIC_ENDLOCHEADER64 */
            put32(q + 4, 0);
            put64(q + 8, cd_off + cd_size);
            put32(q + 16, 1);
            tl = 76;
        }
        uint8_t *q = tail + tl;
        put32(q, 0x06054b50u);                       /* MZ_ZIP_MAGIC_ENDHEADER */
        put16(q + 4, 0);
        put16(q + 6, 0);
        put16(q + 8, count >= 0xffffu ? 0xffffu : count);
        put16(q + 10, count >= 0xffffu ? 0xffffu : count);
        put32(q + 12, (uint32_t)cd_size);
        put32(q + 16, cd_off >= 0xffffffffull ? 0xffffffffu : (uint32_t)cd_off);
        put16(q + 20, 0);
        tl += 22;
        if (err == MZ_OK)
            err = za_write(base_stream, tail, tl);
    }
    const double t_setup1 = now_ms();
    for (uint32_t k = 0; k < nslots; k++) {
        mz_cuda_set_device(slots[k].device);
        zp_release(ZP_WRITER, &slots[k]);
    }
    mz_cuda_set_device(dev0);
    st.setup_ms += now_ms() - t_setup1;
    free(slots);
    free(cd.p);
    free(rfirst);
    if (stats)
        *stats = st;
    return err;
}

/* ---- batch extraction ------------------------------------------------------------------------------------------ */
/* the round's launches on stream s, from the K9 table in z->d_ent (and digests in z->d_sha) over the stored bytes buf[0, buf_len)
 * (32 readable bytes past them) into out: locate, K8 per strength (decrypts buf in place), stored copy, K5, K1, K7, verify */
static int32_t zr_launch(zr_slot *z, uint8_t *buf, uint64_t buf_len, uint8_t *out, void *s) {
    const uint32_t n = z->n;
    int32_t err = MZ_OK;
    mz_cuda_zip_round R;
    memset(&R, 0, sizeof(R));
    R.buf = buf;
    R.buf_len = buf_len;
    R.out = out;
    R.ent = z->d_ent;
    R.n = n;
    R.jobs = z->d_job;
    R.states = z->d_state;
    R.seg_off = z->d_seg_off;
    R.seg_len64 = z->d_seg_len64;
    R.data_off = z->d_data_off;
    R.seg_len = z->d_seg_len;
    R.crc = z->d_crc;
    R.digest = z->d_digest;
    R.sha_expect = z->d_sha;
    R.salt = z->d_salt;
    R.coff = z->d_coff;
    R.clen = z->d_clen;
    R.keys = z->d_keys;
    R.mac = z->d_mac;
    R.status = z->d_status;
    if (!err) err = mz_cuda_zip_locate(&R, s);
    /* WinZip AES (mz_strm_wzaes.c): keys from password + salt, HMAC of the ciphertext, then the ciphertext becomes the compressed
     * stream in place; one pass per strength present, rows of a strength are contiguous from base */
    for (uint32_t st = 1, base = 0; st <= 3 && !err; base += z->na[st], st++) {
        if (!z->na[st])
            continue;
        const size_t pwl = strlen(z->password);
        err = mz_cuda_memcpy_h2d(z->d_pw, z->password, pwl ? pwl : 1, s);
        if (!err) err = mz_cuda_wzaes_derive(z->d_pw, (uint32_t)pwl, z->d_salt + (size_t)base * 16, z->na[st], st, z->d_keys + (size_t)base * MZ_CUDA_WZAES_KEYREC, s);
        if (!err) err = mz_cuda_wzaes_hmac(buf, z->d_coff + base, z->d_clen + base, z->na[st], z->d_keys + (size_t)base * MZ_CUDA_WZAES_KEYREC, st,
                                           z->d_mac + (size_t)base * 20, s);
        if (!err) err = mz_cuda_wzaes_ctr(buf, z->d_coff + base, z->d_clen + base, z->na[st], z->max_clen[st], z->d_keys + (size_t)base * MZ_CUDA_WZAES_KEYREC,
                                          st, s);
    }
    if (!err) err = mz_cuda_zip_copy_stored(&R, s);
    if (!err && z->njobs) {
        err = mz_cuda_memset(z->d_state, 0, (size_t)z->njobs * sizeof(mz_cuda_inflate_state), s);
        if (!err) err = mz_cuda_inflate_streams(z->d_job, z->d_state, z->njobs, s);
    }
    if (!err) err = mz_cuda_crc32_segments(out, 0, 0, z->d_seg_off, z->d_seg_len, n, z->d_residue, z->d_crc, s);
    if (!err && z->nsha) err = mz_cuda_sha256_batch(out, z->d_seg_off, z->d_seg_len64, n, z->d_digest, s);
    if (!err) err = mz_cuda_zip_verify(&R, s);
    return err;
}

/* the round's device work; on return h_status and h_out hold the results (z->err: a CUDA error, not an entry's) */
static void *zr_run(void *arg) {
    zr_slot *z = (zr_slot *)arg;
    const double t0 = now_ms();
    void *s = z->stream;
    const uint32_t n = z->n;
    int32_t err = mz_cuda_set_device(z->device);
    if (!err) err = mz_cuda_memcpy_h2d(z->d_in, z->h_in, z->in_used + 32, s); /* K5 reads up to 16 bytes past a stream */
    if (!err) err = mz_cuda_memcpy_h2d(z->d_ent, z->h_ent, (size_t)n * sizeof(mz_cuda_zip_ent), s);
    if (!err && z->nsha) err = mz_cuda_memcpy_h2d(z->d_sha, z->h_sha, (size_t)z->nsha * 32, s);
    if (!err) err = zr_launch(z, z->d_in, z->in_used, z->d_out, s);
    if (!err) err = mz_cuda_memcpy_d2h(z->h_status, z->d_status, (size_t)n * 4, s);
    if (!err) err = mz_cuda_memcpy_d2h(z->h_out, z->d_out, z->out_used, s);
    if (!err) err = mz_cuda_stream_sync(s);
    z->err = err;
    z->gpu_ms = now_ms() - t0;
    return NULL;
}

/* the round's verdict from the status words. archive_order (mz_zip_cuda_extract_archive): the first failing entry decides, as in
 * the reference's reader. Otherwise (mz_zip_cuda_extract_all, unchanged): locate errors first (there are none: its records point at
 * the data), then WinZip AES errors by strength and entry, then stream / CRC / hash errors by entry. */
static int32_t zr_verdict(const zr_slot *z, int archive_order) {
    if (archive_order) {
        for (uint32_t i = 0; i < z->n; i++)
            if (z->h_status[i])
                return -(int32_t)(z->h_status[i] & 0xffffu);
        return MZ_OK;
    }
    for (uint32_t i = 0; i < z->n; i++)
        if ((z->h_status[i] >> 24) == 1)
            return -(int32_t)(z->h_status[i] & 0xffffu);
    for (uint32_t st = 1; st <= 3; st++)
        for (uint32_t i = 0; i < z->n; i++)
            if (z->h_ent[i].aes == st && (z->h_status[i] >> 24) == 2)
                return -(int32_t)(z->h_status[i] & 0xffffu);
    for (uint32_t i = 0; i < z->n; i++)
        if (z->h_status[i])
            return -(int32_t)(z->h_status[i] & 0xffffu);
    return MZ_OK;
}

/* host-side description of an entry (both extractors) */
typedef struct zx_entry_s {
    uint64_t off, csize, usize, ext; /* extract_all: offset in the round's staging; native: absolute offset of the local header, extent */
    uint32_t crc, name_off;
    uint16_t method;
    uint8_t has_sha;
    uint8_t aes;     /* 0, or the WinZip AES strength 1..3: the stored bytes are salt | verifier | ciphertext | authentication code */
    uint8_t sha[32]; /* expected SHA-256 from the MZ_ZIP_EXTENSION_HASH extra field */
} zx_entry;

/* the records of entries [first, last) into z->h_ent / h_sha, with src_off[k] for entry first + k; plain bytes packed 16-byte aligned */
static void zr_table(zr_slot *z, const zx_entry *ent, uint32_t first, uint32_t last, const uint64_t *src_off, uint8_t flags) {
    const uint32_t n = last - first;
    uint32_t base[4] = {0, 0, 0, 0};
    memset(z->na, 0, sizeof(z->na));
    memset(z->max_clen, 0, sizeof(z->max_clen));
    for (uint32_t k = 0; k < n; k++)
        z->na[ent[first + k].aes & 3]++;
    base[2] = z->na[1];
    base[3] = z->na[1] + z->na[2];
    z->na[0] = 0;
    uint32_t fill[4] = {0, 0, 0, 0};
    size_t out = 0;
    z->n = n;
    z->njobs = z->nsha = 0;
    for (uint32_t k = 0; k < n; k++) {
        const zx_entry *e = &ent[first + k];
        mz_cuda_zip_ent *r = &z->h_ent[k];
        memset(r, 0, sizeof(*r));
        r->src_off = src_off[k];
        r->src_len = (flags & MZ_CUDA_ZIP_ENT_AT_DATA) ? e->csize : e->ext;
        r->csize = e->csize;
        r->usize = e->usize;
        r->out_off = out;
        r->crc = e->crc;
        r->method = e->method;
        r->aes = e->aes;
        r->flags = flags;
        r->job = e->method == 8 ? z->njobs++ : 0xffffffffu;
        r->aes_slot = e->aes ? base[e->aes] + fill[e->aes]++ : 0xffffffffu;
        if (e->aes) {
            const uint64_t clen = e->csize - (4u * e->aes + 4u + 12u);
            if (clen > z->max_clen[e->aes]) z->max_clen[e->aes] = clen;
        }
        r->sha_slot = 0xffffffffu;
        if (e->has_sha) {
            memcpy(z->h_sha + (size_t)z->nsha * 32, e->sha, 32);
            r->sha_slot = z->nsha++;
        }
        out += ((size_t)e->usize + 15) & ~(size_t)15;
    }
    z->out_used = out;
}

/* hands a verified round to the callback */
static int32_t zr_deliver(const zr_slot *z, const zx_entry *ent, const char *names, mz_cuda_zip_entry_cb cb, void *userdata, mz_cuda_zip_stats *st) {
    for (uint32_t k = 0; k < z->n; k++) {
        const zx_entry *e = &ent[z->first + k];
        if (cb) {
            const int32_t err = cb(userdata, names + e->name_off, z->h_out + z->h_ent[k].out_off, (int64_t)e->usize, e->crc);
            if (err)
                return err;
        }
        st->bytes_in += e->csize;
        st->bytes_out += e->usize;
    }
    return MZ_OK;
}

/* the hash extra field: {id u16, size u16, data}; MZ_ZIP_EXTENSION_HASH with algorithm SHA-256 (mz_zip_rw.c:478-510) */
static void zx_find_sha(zx_entry *e, const uint8_t *xf, uint32_t xlen) {
    e->has_sha = 0;
    for (uint32_t xo = 0; xf && xo + 4 <= xlen;) {
        const uint8_t *x = xf + xo;
        const uint32_t id = x[0] | (x[1] << 8), xs = x[2] | (x[3] << 8);
        if (xo + 4 + xs > xlen)
            break;
        if (id == 0x1a51 && xs >= 4 + 32 && (x[4] | (x[5] << 8)) == 23 && (x[6] | (x[7] << 8)) == 32) {
            memcpy(e->sha, x + 8, 32);
            e->has_sha = 1;
            break;
        }
        xo += 4 + xs;
    }
}

/* decode + checksum + deliver the entries collected in ent[0..n) (extract_all: one round at a time, synchronously) */
static int32_t zx_flush(zr_slot *z, const zx_entry *ent, uint32_t n, size_t comp_used, const char *names, const char *password, mz_cuda_zip_entry_cb cb,
                        void *userdata, mz_cuda_zip_stats *st) {
    if (n == 0)
        return MZ_OK;
    uint64_t *src = (uint64_t *)malloc((size_t)n * 8);
    if (!src)
        return MZ_MEM_ERROR;
    for (uint32_t i = 0; i < n; i++)
        src[i] = ent[i].off;
    const double t0 = now_ms();
    zr_table(z, ent, 0, n, src, MZ_CUDA_ZIP_ENT_AT_DATA);
    free(src);
    z->first = 0;
    z->last = n;
    z->in_used = comp_used;
    z->password = password;
    zr_run(z);
    const double t1 = now_ms();
    int32_t err = z->err ? z->err : zr_verdict(z, 0);
    if (err)
        return err;
    const double t2 = now_ms();
    err = zr_deliver(z, ent, names, cb, userdata, st);
    if (err)
        return err;
    st->gpu_ms += t1 - t0;
    st->container_ms += now_ms() - t2;
    st->entries += n;
    st->rounds++;
    return MZ_OK;
}

int32_t mz_zip_cuda_extract_all(void *zip_handle, mz_cuda_zip_entry_cb cb, void *userdata, mz_cuda_zip_stats *stats) {
    return mz_zip_cuda_extract_all_aes(zip_handle, NULL, cb, userdata, stats);
}

int32_t mz_zip_cuda_extract_all_aes(void *zip_handle, const char *password, mz_cuda_zip_entry_cb cb, void *userdata, mz_cuda_zip_stats *stats) {
    zr_slot z;
    mz_cuda_zip_stats st;
    int32_t err;
    memset(&st, 0, sizeof(st));
    if (!mz_zip_goto_first_entry || !mz_zip_goto_next_entry || !mz_zip_entry_get_info || !mz_zip_entry_read_open || !mz_zip_entry_read ||
        !mz_zip_entry_close)
        return MZ_SUPPORT_ERROR; /* no zip container in this process */
    if (!zip_handle)
        return MZ_PARAM_ERROR;
    if (mzh_gpu_required("mz_zip_cuda"))
        return MZ_SUPPORT_ERROR;
    const size_t comp_cap = mzh_round_bytes(128), out_cap = comp_cap * 4;
    const uint32_t max_entries = 65536;
    const size_t names_cap = (size_t)max_entries * 64;
    zx_entry *ent = (zx_entry *)malloc((size_t)max_entries * sizeof(zx_entry));
    char *names = (char *)malloc(names_cap);
    memset(&z, 0, sizeof(z));
    z.in_cap = comp_cap;
    z.out_cap = out_cap;
    z.max_ent = max_entries;
    if (!ent || !names || !zr_alloc(&z, 0)) {
        free(ent);
        free(names);
        return MZ_MEM_ERROR;
    }
    z.device = mz_cuda_get_device();
    uint32_t n = 0;
    size_t comp_used = 0, out_used = 0, names_used = 0;
    err = mz_zip_goto_first_entry(zip_handle);
    while (err == MZ_OK) {
        zc_file_info *fi = NULL;
        double t0 = now_ms();
        err = mz_zip_entry_get_info(zip_handle, &fi);
        if (err != MZ_OK)
            break;
        const int enc = (fi->flag & 1u) != 0;
        const uint32_t aes_over = enc ? 4u * fi->aes_strength + 4u + 12u : 0u; /* salt + verifier + authentication code */
        if (enc && fi->aes_version && !password) {
            err = MZ_PASSWORD_ERROR; /* encrypted and no password given */
            break;
        }
        if ((enc && (!fi->aes_version || fi->aes_strength < 1 || fi->aes_strength > 3 || strlen(password) > 128 ||
                     fi->compressed_size < (int64_t)aes_over)) ||
            (fi->compression_method != 0 && fi->compression_method != 8) || fi->compressed_size < 0 ||
            fi->uncompressed_size < 0 || fi->uncompressed_size > (1ll << 30) || fi->compressed_size > (1ll << 30)) {
            err = MZ_SUPPORT_ERROR; /* PKWARE-encrypted, another codec, or too large for the batch path */
            break;
        }
        if (fi->compression_method == 0 && fi->compressed_size - (int64_t)aes_over != fi->uncompressed_size) {
            err = MZ_FORMAT_ERROR;
            break;
        }
        const size_t csz = (size_t)fi->compressed_size, usz = (size_t)fi->uncompressed_size;
        const size_t cneed = (csz + 32 + 15) & ~(size_t)15, oneed = (usz + 15) & ~(size_t)15; /* K5 reads up to 16 bytes past a stream */
        const size_t nlen = strlen(fi->filename) + 1;
        if (cneed > z.in_cap || oneed > z.out_cap) { /* one entry larger than a round: not batched */
            err = MZ_SUPPORT_ERROR;
            break;
        }
        if (n == z.max_ent || comp_used + cneed > z.in_cap || out_used + oneed > z.out_cap || names_used + nlen > names_cap) {
            err = zx_flush(&z, ent, n, comp_used, names, password, cb, userdata, &st);
            if (err)
                break;
            n = 0;
            comp_used = out_used = names_used = 0;
        }
        zx_entry *e = &ent[n];
        e->off = comp_used;
        e->csize = csz;
        e->usize = usz;
        e->ext = csz;
        e->crc = fi->crc;
        e->method = fi->compression_method;
        e->name_off = (uint32_t)names_used;
        e->aes = enc ? fi->aes_strength : 0;
        zx_find_sha(e, fi->extrafield, fi->extrafield ? fi->extrafield_size : 0);
        memcpy(names + names_used, fi->filename, nlen);
        /* the compressed bytes, untouched, through the raw seam */
        if (csz) {
            err = mz_zip_entry_read_open(zip_handle, 1, NULL);
            size_t got = 0;
            while (err == MZ_OK && got < csz) {
                const int32_t want = csz - got > (1u << 30) ? (int32_t)(1u << 30) : (int32_t)(csz - got);
                const int32_t r = mz_zip_entry_read(zip_handle, z.h_in + comp_used + got, want);
                if (r <= 0) {
                    err = r < 0 ? r : MZ_READ_ERROR;
                    break;
                }
                got += (size_t)r;
            }
            const int32_t cerr = mz_zip_entry_close(zip_handle);
            if (err == MZ_OK && cerr != MZ_OK)
                err = cerr;
            if (err != MZ_OK)
                break;
        }
        memset(z.h_in + comp_used + csz, 0, cneed - csz);
        comp_used += cneed;
        out_used += oneed;
        names_used += nlen;
        n++;
        st.pack_ms += now_ms() - t0;
        err = mz_zip_goto_next_entry(zip_handle);
    }
    if (err == MZ_END_OF_LIST)
        err = zx_flush(&z, ent, n, comp_used, names, password, cb, userdata, &st);
    zr_free(&z);
    free(ent);
    free(names);
    if (stats)
        *stats = st;
    return err;
}

/* ---- the native archive extractor (mz_zip_cuda_extract_archive) ---------------------------------------------------------- */
static uint32_t get16(const uint8_t *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }
static uint32_t get32(const uint8_t *p) { return get16(p) | (get16(p + 2) << 16); }
static uint64_t get64(const uint8_t *p) { return (uint64_t)get32(p) | ((uint64_t)get32(p + 4) << 32); }

static int32_t zn_seek(void *base, int64_t off) {
    mz_stream *s = (mz_stream *)base;
    if (!s || !s->vtbl || !s->vtbl->seek)
        return MZ_PARAM_ERROR;
    return s->vtbl->seek(s, off, MZ_SEEK_SET) == MZ_OK ? MZ_OK : MZ_SEEK_ERROR;
}

/* n bytes at absolute offset off, in reads of at most 1 GiB (the vtbl takes int32_t sizes) */
static int32_t zn_read_at(void *base, int64_t off, uint8_t *p, uint64_t n) {
    int32_t err = zn_seek(base, off);
    while (err == MZ_OK && n > 0) {
        const int32_t part = n > (1u << 30) ? (int32_t)(1u << 30) : (int32_t)n;
        const int32_t r = mz_abi_base_read(base, p, part);
        if (r <= 0)
            return r < 0 ? r : MZ_READ_ERROR;
        p += r;
        n -= (uint64_t)r;
    }
    return err;
}

static int zn_cmp_off(const void *a, const void *b, void *ctx) {
    const zx_entry *e = (const zx_entry *)ctx;
    const uint64_t x = e[*(const uint32_t *)a].off, y = e[*(const uint32_t *)b].off;
    return x < y ? -1 : x > y;
}

/* The central directory, read with one base read and parsed here (mz_zip.c:131-200 end records, :947-1100 directory and the
 * correction for prepended data, :231 record layout): every entry's local-header offset, sizes, CRC, method, AES strength, expected
 * SHA-256, name; then every entry's extent (its offset up to the next higher one or the directory). */
static int32_t zn_read_directory(void *base, const char *password, zx_entry **out_ent, uint32_t *out_n, char **out_names, int32_t *out_refuse) {
    int32_t err, refuse = MZ_OK;
    int64_t size;
    uint8_t *tail = NULL, *cd = NULL;
    zx_entry *ent = NULL;
    char *names = NULL;
    *out_ent = NULL;
    *out_names = NULL;
    *out_n = 0;
    *out_refuse = MZ_OK;
    {
        mz_stream *s = (mz_stream *)base;
        if (!s || !s->vtbl || !s->vtbl->seek || !s->vtbl->tell || s->vtbl->seek(s, 0, MZ_SEEK_END) != MZ_OK)
            return MZ_SEEK_ERROR;
        size = s->vtbl->tell(s);
        if (size < 0)
            return MZ_TELL_ERROR;
    }
    /* the end record: the last signature within 64 KiB + 22 bytes of the end (mz_zip_search_eocd) */
    const int64_t tl = size < 65535 + 22 ? size : 65535 + 22;
    tail = (uint8_t *)malloc((size_t)tl + 1);
    if (!tail)
        return MZ_MEM_ERROR;
    err = zn_read_at(base, size - tl, tail, (uint64_t)tl);
    int64_t eocd = -1;
    for (int64_t i = tl - 22; err == MZ_OK && i >= 0; i--)
        if (get32(tail + i) == 0x06054b50u) {
            eocd = size - tl + i;
            break;
        }
    if (err == MZ_OK && eocd < 0)
        err = MZ_FORMAT_ERROR;
    uint64_t count = 0, cd_size = 0, cd_off = 0;
    int64_t eocd_pos = eocd;
    if (err == MZ_OK) {
        const uint8_t *q = tail + (eocd - (size - tl));
        const uint32_t disk = get16(q + 4), disk_cd = get16(q + 6), on_disk = get16(q + 8);
        count = get16(q + 10);
        cd_size = get32(q + 12);
        cd_off = get32(q + 16);
        if (disk != 0 || disk_cd != 0)
            err = MZ_SUPPORT_ERROR; /* split archive */
        else if (on_disk != count)
            err = MZ_FORMAT_ERROR;
        if (err == MZ_OK && (count == 0xffffu || cd_off == 0xffffffffu || cd_size == 0xffffffffu)) {
            /* zip64: the locator in front of the end record names the zip64 end record (mz_zip_search_zip64_eocd); with prepended
             * data the record sits right in front of the locator instead */
            uint8_t loc[20], z64[56];
            int found = 0;
            if (eocd >= 20 && zn_read_at(base, eocd - 20, loc, 20) == MZ_OK && get32(loc) == 0x07064b50u) {
                const uint64_t at[2] = {get64(loc + 8), (uint64_t)(eocd - 20 - 56)};
                for (int k = 0; k < 2 && !found; k++)
                    if (at[k] + 56 <= (uint64_t)eocd && zn_read_at(base, (int64_t)at[k], z64, 56) == MZ_OK && get32(z64) == 0x06064b50u) {
                        found = 1;
                        eocd_pos = (int64_t)at[k];
                    }
            }
            if (found) {
                if (get32(z64 + 16) != 0 || get32(z64 + 20) != 0)
                    err = MZ_SUPPORT_ERROR;
                else if (get64(z64 + 24) != get64(z64 + 32))
                    err = MZ_FORMAT_ERROR;
                count = get64(z64 + 32);
                cd_size = get64(z64 + 40);
                cd_off = get64(z64 + 48);
                if ((int64_t)cd_size < 0 || (int64_t)cd_off < 0)
                    err = MZ_FORMAT_ERROR;
            } else if (count == 0xffffu || cd_off == 0xffffffffu) {
                err = MZ_FORMAT_ERROR;
            }
        }
    }
    free(tail);
    /* prepended data (self-extracting archives): when the directory is not where the end record says, it is right in front of the
     * end record, and every recorded offset is off by the same shift (mz_zip.c:1066-1086) */
    int64_t shift = 0;
    if (err == MZ_OK) {
        uint8_t sig[4];
        if (cd_off > (uint64_t)eocd_pos || cd_size > (uint64_t)eocd_pos)
            err = MZ_FORMAT_ERROR;
        else if (cd_size && (zn_read_at(base, (int64_t)cd_off, sig, 4) != MZ_OK || get32(sig) != 0x02014b50u)) {
            const int64_t alt = eocd_pos - (int64_t)cd_size;
            if (zn_read_at(base, alt, sig, 4) == MZ_OK && get32(sig) == 0x02014b50u) {
                shift = alt - (int64_t)cd_off;
                cd_off = (uint64_t)alt;
            } else {
                err = MZ_FORMAT_ERROR;
            }
        }
        if (err == MZ_OK && cd_off + cd_size > (uint64_t)eocd_pos)
            cd_size = (uint64_t)eocd_pos - cd_off;
    }
    if (err == MZ_OK && cd_size / 46 < count)
        err = MZ_FORMAT_ERROR;
    if (err == MZ_OK) {
        cd = (uint8_t *)malloc(cd_size + 1);
        ent = (zx_entry *)malloc((size_t)(count ? count : 1) * sizeof(zx_entry));
        names = (char *)malloc(cd_size + count + 1);
        if (!cd || !ent || !names)
            err = MZ_MEM_ERROR;
    }
    if (err == MZ_OK)
        err = zn_read_at(base, (int64_t)cd_off, cd, cd_size);
    uint32_t n = 0;
    size_t nused = 0;
    /* A record that is malformed or names an entry this call refuses ends the list: the entries in front of it are extracted,
     * and then its error is returned -- what the reference's reader does when its walk reaches that entry. */
    for (uint64_t p = 0; err == MZ_OK && refuse == MZ_OK && p < cd_size;) {
        const uint8_t *h = cd + p;
        if (cd_size - p < 46 || get32(h) != 0x02014b50u || n >= count) {
            refuse = MZ_FORMAT_ERROR;
            break;
        }
        const uint32_t flag = get16(h + 8), nlen = get16(h + 28), xlen = get16(h + 30), clen = get16(h + 32);
        if (46ull + nlen + xlen + clen > cd_size - p) {
            refuse = MZ_FORMAT_ERROR;
            break;
        }
        zx_entry *e = &ent[n];
        memset(e, 0, sizeof(*e));
        uint32_t method = get16(h + 10);
        e->crc = get32(h + 16);
        e->csize = get32(h + 20);
        e->usize = get32(h + 24);
        e->off = get32(h + 42);
        uint32_t disk = get16(h + 34), aes_method = 0;
        const uint8_t *xf = h + 46 + nlen;
        for (uint32_t xo = 0; xo + 4 <= xlen;) {
            /* a field's length is clamped to what is left of the extra field, as mz_zip.c:321-322 does */
            const uint32_t id = get16(xf + xo), xs = get16(xf + xo + 2), xn = xo + 4 + xs > xlen ? xlen - xo - 4 : xs;
            const uint8_t *x = xf + xo + 4, *xe = x + xn;
            /* MZ_ZIP_EXTENSION_ZIP64: the saturated fields, in this order (mz_zip.c:325-343) */
            if (id == 0x0001) {
                if (e->usize == 0xffffffffu && x + 8 <= xe) { e->usize = get64(x); x += 8; }
                if (e->csize == 0xffffffffu && x + 8 <= xe) { e->csize = get64(x); x += 8; }
                if (e->off == 0xffffffffu && x + 8 <= xe) { e->off = get64(x); x += 8; }
                if (disk == 0xffffu && x + 4 <= xe) disk = get32(x);
            } else if (id == 0x9901 && xn == 7) { /* WinZip AES: version, "AE", strength, real method (mz_zip.c:415-440) */
                e->aes = x[4];
                aes_method = get16(x + 5);
                if (e->aes < 1 || e->aes > 3)
                    e->aes = 0xff;
            }
            xo += 4 + xs;
        }
        zx_find_sha(e, xf, xlen);
        const int enc = (flag & 1u) != 0;
        if (enc && method == 99 && e->aes)
            method = aes_method;
        e->method = (uint16_t)method;
        const uint64_t aes_over = enc && e->aes && e->aes != 0xff ? 4u * e->aes + 4u + 12u : 0u;
        if (enc && e->aes && !password) {
            refuse = MZ_PASSWORD_ERROR; /* encrypted and no password given */
        } else if ((enc && (!e->aes || e->aes == 0xff || strlen(password) > 128 || e->csize < aes_over)) || (!enc && e->aes) ||
                   (method != 0 && method != 8) || e->usize > (1ull << 30) || e->csize > (1ull << 30) || disk != 0) {
            refuse = MZ_SUPPORT_ERROR; /* PKWARE-encrypted, another codec, too large for the batch path, or on another disk */
        } else if (method == 0 && e->csize - aes_over != e->usize) {
            refuse = MZ_FORMAT_ERROR;
        } else {
            e->off += (uint64_t)shift;
            if (e->off + 30 > cd_off) /* the local header must lie in front of the directory */
                refuse = MZ_FORMAT_ERROR;
        }
        if (refuse != MZ_OK)
            break;
        if (!enc)
            e->aes = 0;
        e->name_off = (uint32_t)nused;
        memcpy(names + nused, h + 46, nlen);
        names[nused + nlen] = 0;
        nused += nlen + 1;
        p += 46ull + nlen + xlen + clen;
        n++;
    }
    free(cd);
    if (err == MZ_OK && refuse == MZ_OK && n != count)
        refuse = MZ_FORMAT_ERROR;
    /* extents: up to the next higher local-header offset or the directory, and never more than a header, the data and a
     * descriptor can take */
    uint32_t *ord = err == MZ_OK ? (uint32_t *)malloc((size_t)(n ? n : 1) * 4) : NULL;
    if (err == MZ_OK && !ord)
        err = MZ_MEM_ERROR;
    if (err == MZ_OK) {
        for (uint32_t i = 0; i < n; i++)
            ord[i] = i;
        qsort_r(ord, n, 4, zn_cmp_off, ent);
        for (uint32_t k = 0, j = 0; k < n; k++) {
            zx_entry *e = &ent[ord[k]];
            while (j < n && ent[ord[j]].off <= e->off)
                j++;
            const uint64_t end = j < n ? ent[ord[j]].off : cd_off;
            const uint64_t cap = 30u + 65535u + 65535u + e->csize + 24u;
            e->ext = end - e->off < cap ? end - e->off : cap;
        }
    }
    free(ord);
    if (err != MZ_OK) {
        free(ent);
        free(names);
        return err;
    }
    *out_ent = ent;
    *out_names = names;
    *out_n = n;
    *out_refuse = refuse;
    return MZ_OK;
}

/* a round's stored bytes into z->h_in: extents in directory order, packed; one base read per run of adjacent extents */
static int32_t zn_fill(zr_slot *z, void *base, const zx_entry *ent, uint64_t *src) {
    int32_t err = MZ_OK;
    size_t pos = 0, run_pos = 0;
    uint64_t run_off = 0, run_len = 0;
    for (uint32_t i = z->first; i < z->last && err == MZ_OK; i++) {
        const zx_entry *e = &ent[i];
        if (run_len && e->off != run_off + run_len) {
            err = zn_read_at(base, (int64_t)run_off, z->h_in + run_pos, run_len);
            run_len = 0;
        }
        if (!run_len) {
            run_off = e->off;
            run_pos = pos;
        }
        run_len += e->ext;
        src[i - z->first] = pos;
        pos += e->ext;
    }
    if (err == MZ_OK && run_len)
        err = zn_read_at(base, (int64_t)run_off, z->h_in + run_pos, run_len);
    memset(z->h_in + pos, 0, 64);
    z->in_used = pos;
    return err;
}

int32_t mz_zip_cuda_extract_archive(void *base_stream, const char *password, uint32_t flags, mz_cuda_zip_entry_cb cb, void *userdata,
                                    mz_cuda_zip_stats *stats) {
    mz_cuda_zip_stats st;
    memset(&st, 0, sizeof(st));
    if (!base_stream || (flags & ~MZ_ZIP_CUDA_ALL_DEVICES))
        return MZ_PARAM_ERROR;
    if (mzh_gpu_required("mz_zip_cuda"))
        return MZ_SUPPORT_ERROR;
    double t0 = now_ms();
    zx_entry *ent = NULL;
    char *names = NULL;
    uint32_t count = 0;
    int32_t refuse = MZ_OK;
    int32_t err = zn_read_directory(base_stream, password, &ent, &count, &names, &refuse);
    if (err) {
        if (stats)
            *stats = st;
        return err;
    }
    /* rounds: runs of entries in directory order whose extents fit the staging (32 MiB by default) and whose plain bytes fit four
     * times that; an entry larger than a round gets a round of its own size */
    const size_t round_bytes = mzh_round_bytes(32);
    const size_t out_round = round_bytes * 4;
    uint32_t nrounds = 0, rcap = 16, max_ent = 1;
    size_t max_in = 64, max_out = 64;
    uint32_t *rfirst = (uint32_t *)malloc((rcap + 1) * sizeof(uint32_t));
    uint64_t *src = NULL;
    if (!rfirst)
        err = MZ_MEM_ERROR;
    for (uint32_t i = 0; i < count && err == MZ_OK;) {
        size_t in = 0, out = 0;
        uint32_t j = i;
        while (j < count) {
            const size_t oneed = ((size_t)ent[j].usize + 15) & ~(size_t)15;
            if (j > i && (in + ent[j].ext > round_bytes || out + oneed > out_round))
                break;
            in += ent[j].ext;
            out += oneed;
            j++;
        }
        if (nrounds == rcap) {
            uint32_t *q = (uint32_t *)realloc(rfirst, (rcap * 2 + 1) * sizeof(uint32_t));
            if (!q) {
                err = MZ_MEM_ERROR;
                break;
            }
            rfirst = q;
            rcap *= 2;
        }
        rfirst[nrounds++] = i;
        if (in > max_in) max_in = in;
        if (out > max_out) max_out = out;
        if (j - i > max_ent) max_ent = j - i;
        i = j;
    }
    if (err == MZ_OK) {
        rfirst[nrounds] = count;
        /* staging is pooled by capacity: round it up so that similar archives share it */
        max_in = max_in > round_bytes ? (max_in + 65535) & ~(size_t)65535 : round_bytes;
        max_out = max_out > out_round ? (max_out + 65535) & ~(size_t)65535 : out_round;
        max_ent = (max_ent + 4095) & ~4095u;
        src = (uint64_t *)malloc((size_t)max_ent * 8);
        if (!src)
            err = MZ_MEM_ERROR;
    }
    st.pack_ms += now_ms() - t0;
    int32_t ndev = 1;
    const int32_t dev0 = mz_cuda_get_device() < 0 ? 0 : mz_cuda_get_device();
    if (flags & MZ_ZIP_CUDA_ALL_DEVICES) {
        ndev = mz_cuda_device_count();
        if (ndev < 1) ndev = 1;
        if (ndev > 8) ndev = 8;
    }
    const double t_setup0 = now_ms();
    /* an entry larger than a round makes every slot as large as it: then one slot per device, and it is not pooled */
    const int oversized = max_in > round_bytes || max_out > out_round;
    const uint32_t want = oversized ? (uint32_t)ndev : ndev > 1 ? (uint32_t)ndev * 2 : 4u;
    const uint32_t nslots = want < nrounds ? want : (nrounds ? nrounds : 1);
    zr_slot *slots = err == MZ_OK ? (zr_slot *)calloc(nslots, sizeof(zr_slot)) : NULL;
    if (err == MZ_OK && !slots)
        err = MZ_MEM_ERROR;
    for (uint32_t k = 0; k < nslots && err == MZ_OK && nrounds; k++) {
        zr_slot *z = &slots[k];
        z->device = ndev > 1 ? (int32_t)(k % (uint32_t)ndev) : dev0;
        z->in_cap = max_in;
        z->out_cap = max_out;
        z->max_ent = max_ent;
        if (mz_cuda_set_device(z->device) != MZ_OK || !zp_acquire(ZP_EXTRACTOR, z))
            err = MZ_MEM_ERROR;
        z->password = password;
    }
    mz_cuda_set_device(dev0);
    st.setup_ms = now_ms() - t_setup0;
    /* the caller's thread reads rounds ahead into free slots (the base stream is not thread-safe), each slot's worker runs the
     * device work on its own stream, and finished rounds are delivered in archive order. A base read that fails while reading ahead
     * stops the issuing; the rounds issued before it are still delivered, then its error is returned. */
    uint32_t issued = 0, stop = nrounds;
    int32_t read_err = MZ_OK;
    for (uint32_t r = 0; r < stop && err == MZ_OK; r++) {
        while (issued < stop && issued < r + nslots) {
            zr_slot *z = &slots[issued % nslots];
            const double t1 = now_ms();
            z->first = rfirst[issued];
            z->last = rfirst[issued + 1];
            read_err = zn_fill(z, base_stream, ent, src);
            if (read_err == MZ_OK)
                zr_table(z, ent, z->first, z->last, src, 0);
            st.pack_ms += now_ms() - t1;
            if (read_err) {
                stop = issued;
                break;
            }
            z->running = pthread_create(&z->th, NULL, zr_run, z) == 0;
            if (!z->running)
                zr_run(z);
            issued++;
        }
        if (r >= stop)
            break;
        zr_slot *z = &slots[r % nslots];
        if (z->running) {
            pthread_join(z->th, NULL);
            z->running = 0;
        }
        err = z->err ? z->err : zr_verdict(z, 1);
        if (err)
            break;
        const double t2 = now_ms();
        err = zr_deliver(z, ent, names, cb, userdata, &st);
        st.container_ms += now_ms() - t2;
        st.gpu_ms += z->gpu_ms;
        st.entries += z->n;
        st.rounds++;
    }
    for (uint32_t k = 0; slots && k < nslots; k++)
        if (slots[k].running) {
            pthread_join(slots[k].th, NULL);
            slots[k].running = 0;
        }
    if (err == MZ_OK)
        err = read_err;
    if (err == MZ_OK)
        err = refuse; /* the entry that ended the list (zn_read_directory), after every entry in front of it was delivered */
    const double t_setup1 = now_ms();
    for (uint32_t k = 0; slots && k < nslots; k++) {
        if (!slots[k].h_in)
            continue;
        mz_cuda_set_device(slots[k].device);
        if (oversized)
            zr_free(&slots[k]);
        else
            zp_release(ZP_EXTRACTOR, &slots[k]);
    }
    mz_cuda_set_device(dev0);
    st.setup_ms += now_ms() - t_setup1;
    free(slots);
    free(src);
    free(rfirst);
    free(ent);
    free(names);
    if (stats)
        *stats = st;
    return err;
}

/* ---- an archive in device memory (mz_zip_cuda_extract_device) ------------------------------------------------------------ */
/* zr_launch's arrays for a round of n entries (digest_rows of them for the digests), and the first-failure word, carved from one
 * device allocation (returned; NULL when it fails). The K9 table and the expected digests come from the directory parse. */
static uint8_t *zd_carve(zr_slot *z, uint32_t n, size_t digest_rows, uint32_t **first) {
    mzh_piece t[ZR_ROUND_PIECES + 1];
    const int k = zr_round_pieces(z, n ? n : 1, digest_rows, t);
    t[k] = MZH_DEV(*first, 4);
    return mzh_carve(t, k + 1);
}

int32_t mz_zip_cuda_extract_device(const void *d_archive, uint64_t len, const char *password, mz_cuda_zip_dev_entry *d_entries, uint32_t max_entries,
                                   uint32_t *count, void *d_out, uint64_t out_cap, uint64_t *out_bytes, mz_cuda_zip_stats *stats, void *stream) {
    mz_cuda_zip_stats st;
    memset(&st, 0, sizeof(st));
    if (stats)
        *stats = st;
    if (!count || !out_bytes || (!d_archive && len) || ((uintptr_t)d_out & 15) || (!d_entries && max_entries))
        return MZ_PARAM_ERROR;
    *count = 0;
    *out_bytes = 0;
    if (mzh_gpu_required("mz_zip_cuda"))
        return MZ_SUPPORT_ERROR;
    const double t0 = now_ms();
    mz_cuda_zip_dir dir;
    memset(&dir, 0, sizeof(dir));
    dir.have_password = password != NULL;
    dir.password_long = password && strlen(password) > 128;
    dir.entries = d_entries;
    dir.max_entries = max_entries;
    dir.decode = d_out != NULL;
    dir.out_cap = out_cap;
    int32_t err = mz_cuda_zip_parse_directory(d_archive, len, &dir, stream);
    if (err == MZ_OK && dir.err)
        err = dir.err; /* the archive as a whole */
    st.pack_ms = now_ms() - t0;
    if (err) {
        if (stats)
            *stats = st;
        return err;
    }
    *count = dir.count;
    *out_bytes = dir.out_bytes;
    st.entries = dir.count;
    st.bytes_in = dir.bytes_in;
    st.bytes_out = dir.bytes_out;
    if (max_entries < dir.count || (d_out && out_cap < dir.out_bytes))
        err = MZ_BUF_ERROR;
    else if (!d_out || !dir.count)
        err = dir.refuse;
    else {
        zr_slot z;
        memset(&z, 0, sizeof(z));
        z.n = dir.count;
        z.njobs = dir.njobs;
        z.nsha = dir.nsha;
        memcpy(z.na, dir.na, sizeof(z.na));
        memcpy(z.max_clen, dir.max_clen, sizeof(z.max_clen));
        z.password = password;
        z.d_ent = dir.ent;
        z.d_sha = (uint8_t *)dir.sha_expect;
        const double t1 = now_ms();
        /* K8 decrypts in place: AES entries are decoded from a copy of the bytes in front of the directory */
        const int aes = dir.na[1] || dir.na[2] || dir.na[3];
        uint8_t *buf = (uint8_t *)d_archive, *copy = NULL;
        uint32_t *d_first = NULL;
        uint8_t *work = zd_carve(&z, dir.count, dir.nsha ? dir.count : 1, &d_first);
        if (!work || (aes && !(copy = (uint8_t *)mz_cuda_malloc(dir.cd_off + 32))))
            err = MZ_MEM_ERROR;
        st.setup_ms = now_ms() - t1;
        const double t2 = now_ms();
        if (!err && copy) {
            err = mz_cuda_memcpy_d2d(copy, d_archive, dir.cd_off, stream);
            if (!err) err = mz_cuda_memset(copy + dir.cd_off, 0, 32, stream);
            buf = copy;
        }
        /* buf_len = cd_off: every stream ends at or before the directory, and behind cd_off lie at least one 46-byte directory
         * record and the 22-byte end record, so K5's 16-byte over-read and the stored copy's word reads stay inside [0, len) */
        if (!err) err = zr_launch(&z, buf, dir.cd_off, (uint8_t *)d_out, stream);
        if (!err) err = mz_cuda_memset(d_first, 0xff, 4, stream);
        if (!err) err = mz_cuda_zip_statuses(z.d_status, z.n, d_entries, d_first, stream);
        uint32_t first = 0xffffffffu, word = 0;
        if (!err) err = mz_cuda_memcpy_d2h(&first, d_first, 4, stream);
        if (!err) err = mz_cuda_stream_sync(stream);
        if (!err && first < z.n) {
            err = mz_cuda_memcpy_d2h(&word, z.d_status + first, 4, stream);
            if (!err) err = mz_cuda_stream_sync(stream);
            if (!err) err = -(int32_t)(word & 0xffffu);
        }
        if (!err) err = dir.refuse;
        st.gpu_ms = now_ms() - t2;
        st.rounds = 1;
        mz_cuda_stream_sync(stream);
        mz_cuda_free(copy);
        mz_cuda_free(work);
    }
    mz_cuda_free(dir.ent);
    mz_cuda_free(dir.sha_expect);
    if (stats)
        *stats = st;
    return err;
}

/* ---- an archive written into device memory (mz_zip_cuda_write_device) ---------------------------------------------------- */
/* ---- random access to an archive in device memory (mz_zip_cuda_reader_*) ------------------------------------------------- */
struct mz_zip_cuda_dev_reader {
    int32_t device;
    uint32_t count, P;                /* accepted entries; slots of the name index (0 when there are no entries) */
    const uint8_t *archive;
    uint64_t cd_off, max_clen[4];
    char *password;
    mz_cuda_zip_dev_entry *entries;   /* K10: the public table */
    mz_cuda_zip_ent *ent;             /* K10: the archive-wide K9 table (local header and extent in the archive) */
    void *sha;                        /* K10: expected digests, the rows sha_slot names */
    uint64_t *table;                  /* K12: the name index */
    /* a selection's round, kept between calls and grown when a selection needs more */
    uint32_t cap;                     /* slots the arrays below hold */
    uint8_t *work, *selw;             /* zd_carve's arrays; the counts, their scan, the selection's K9 table, the first-failure word */
    zr_slot z;
    mz_cuda_zip_sel_count *cnt, *pre;
    void *part;
    mz_cuda_zip_ent *sel;
    uint64_t *first;
    uint8_t *gbuf;                    /* gathered extents of a selection with WinZip AES entries, 32 zero bytes behind them */
    uint64_t gcap;
};

static int32_t zu_enter(const mz_zip_cuda_dev_reader *r, int32_t *prev) {
    *prev = mz_cuda_get_device();
    return *prev == r->device ? MZ_OK : mz_cuda_set_device(r->device);
}

static void zu_leave(const mz_zip_cuda_dev_reader *r, int32_t prev) {
    if (prev >= 0 && prev != r->device)
        mz_cuda_set_device(prev);
}

/* the round arrays for at least n slots (sized to a power of two, at least 256); MZ_OK or MZ_MEM_ERROR */
static int32_t zu_reserve(mz_zip_cuda_dev_reader *r, uint32_t n) {
    if (r->work && n <= r->cap)
        return MZ_OK;
    uint64_t cap = 256;
    while (cap < n)
        cap <<= 1;
    if (cap > 0xffffffffull)
        cap = 0xffffffffull;
    mz_cuda_free(r->work);
    mz_cuda_free(r->selw);
    r->work = r->selw = NULL;
    r->cap = 0;
    uint32_t *unused;
    const size_t m = (size_t)cap;
    r->work = zd_carve(&r->z, (uint32_t)cap, m, &unused);
    const mzh_piece t[5] = {MZH_DEV(r->cnt, m * sizeof(mz_cuda_zip_sel_count)), MZH_DEV(r->pre, (m + 1) * sizeof(mz_cuda_zip_sel_count)),
                            MZH_DEV(r->part, (m / MZ_CUDA_ZIP_WR_TILE + 1) * sizeof(mz_cuda_zip_sel_count)),
                            MZH_DEV(r->sel, m * sizeof(mz_cuda_zip_ent)), MZH_DEV(r->first, 8)};
    if (r->work)
        r->selw = mzh_carve(t, 5);
    if (!r->work || !r->selw) {
        mz_cuda_free(r->work);
        r->work = NULL;
        return MZ_MEM_ERROR;
    }
    r->cap = (uint32_t)cap;
    return MZ_OK;
}

int32_t mz_zip_cuda_reader_open(const void *d_archive, uint64_t len, const char *password, mz_zip_cuda_dev_reader **reader, uint32_t *count,
                                int32_t *refuse, mz_cuda_zip_stats *stats, void *stream) {
    mz_cuda_zip_stats st;
    memset(&st, 0, sizeof(st));
    if (stats)
        *stats = st;
    if (!reader || !count || !refuse || (!d_archive && len))
        return MZ_PARAM_ERROR;
    *reader = NULL;
    *count = 0;
    *refuse = MZ_OK;
    if (mzh_gpu_required("mz_zip_cuda"))
        return MZ_SUPPORT_ERROR;
    const double t0 = now_ms();
    mz_cuda_zip_dir dir;
    memset(&dir, 0, sizeof(dir));
    dir.have_password = password != NULL;
    dir.password_long = password && strlen(password) > 128;
    dir.max_entries = 0xffffffffu;
    dir.decode = 1;
    dir.out_cap = ~0ull;
    dir.alloc_entries = 1; /* the public table, allocated by the parse once it knows the count */
    int32_t err = mz_cuda_zip_parse_directory(d_archive, len, &dir, stream);
    if (err == MZ_OK && dir.err)
        err = dir.err; /* the archive as a whole */
    st.pack_ms = now_ms() - t0;
    mz_zip_cuda_dev_reader *r = NULL;
    if (!err && dir.count > (1u << 30))
        err = MZ_SUPPORT_ERROR; /* the name index holds 2 x count slots in 32 bits */
    if (!err && !(r = (mz_zip_cuda_dev_reader *)calloc(1, sizeof(*r))))
        err = MZ_MEM_ERROR;
    if (r)
        r->device = mz_cuda_get_device();
    if (!err && password && !(r->password = strdup(password)))
        err = MZ_MEM_ERROR;
    if (!err) {
        r->count = dir.count;
        r->archive = (const uint8_t *)d_archive;
        r->cd_off = dir.cd_off;
        memcpy(r->max_clen, dir.max_clen, sizeof(r->max_clen));
        r->entries = (mz_cuda_zip_dev_entry *)dir.entries;
        r->ent = dir.ent;
        r->sha = dir.sha_expect;
        dir.entries = NULL; /* the reader's now */
        dir.ent = NULL;
        dir.sha_expect = NULL;
        if (r->count) {
            r->P = 2;
            while (r->P < 2 * r->count)
                r->P <<= 1;
            const double t1 = now_ms();
            r->table = (uint64_t *)mz_cuda_malloc((size_t)r->P * 8);
            st.setup_ms = now_ms() - t1;
            if (!r->table)
                err = MZ_MEM_ERROR;
            const double t2 = now_ms();
            if (!err) err = mz_cuda_memset(r->table, 0xff, (size_t)r->P * 8, stream);
            if (!err) err = mz_cuda_zip_name_index(d_archive, r->entries, r->count, r->table, r->P, stream);
            if (!err) err = mz_cuda_stream_sync(stream);
            st.gpu_ms = now_ms() - t2;
        }
    }
    mz_cuda_free(dir.entries);
    mz_cuda_free(dir.ent);
    mz_cuda_free(dir.sha_expect);
    if (err) {
        mz_zip_cuda_reader_close(r);
        if (stats)
            *stats = st;
        return err;
    }
    st.entries = dir.count;
    st.bytes_in = dir.bytes_in;
    st.bytes_out = dir.bytes_out;
    *reader = r;
    *count = dir.count;
    *refuse = dir.refuse;
    if (stats)
        *stats = st;
    return MZ_OK;
}

const mz_cuda_zip_dev_entry *mz_zip_cuda_reader_entries(const mz_zip_cuda_dev_reader *reader) {
    return reader ? reader->entries : NULL;
}

int32_t mz_zip_cuda_reader_locate(mz_zip_cuda_dev_reader *r, const void *d_names, const uint64_t *d_name_off, const uint32_t *d_name_len,
                                  uint32_t n, uint8_t ignore_case, uint32_t *d_index, void *stream) {
    if (!r || (n && (!d_names || !d_name_off || !d_name_len || !d_index)))
        return MZ_PARAM_ERROR;
    int32_t prev;
    int32_t err = zu_enter(r, &prev);
    if (!err) err = mz_cuda_zip_name_lookup(r->archive, r->entries, r->table, r->P, d_names, d_name_off, d_name_len, n, ignore_case, d_index, stream);
    zu_leave(r, prev);
    return err;
}

int32_t mz_zip_cuda_reader_decode(mz_zip_cuda_dev_reader *r, const uint32_t *d_select, uint32_t nsel, void *d_out, uint64_t out_cap,
                                  uint64_t *out_bytes, uint64_t *d_out_off, int32_t *d_status, mz_cuda_zip_stats *stats, void *stream) {
    mz_cuda_zip_stats st;
    memset(&st, 0, sizeof(st));
    if (stats)
        *stats = st;
    if (!r || !out_bytes || (!d_select && nsel) || ((uintptr_t)d_out & 15))
        return MZ_PARAM_ERROR;
    *out_bytes = 0;
    int32_t prev;
    int32_t err = zu_enter(r, &prev);
    const double t0 = now_ms();
    if (!err && !(r->work && nsel <= r->cap)) {
        err = zu_reserve(r, nsel);
        st.setup_ms += now_ms() - t0;
    }
    /* 1. per-slot counts and their scan; the totals come back */
    mz_cuda_zip_sel sc;
    memset(&sc, 0, sizeof(sc));
    sc.archive = r->archive;
    sc.ent = r->ent;
    sc.count = r->count;
    sc.n = nsel;
    sc.select = d_select;
    sc.cnt = r->cnt;
    sc.pre = r->pre;
    sc.part = r->part;
    mz_cuda_zip_sel_count tot;
    memset(&tot, 0, sizeof(tot));
    if (!err) err = mz_cuda_zip_sel_counts(&sc, stream);
    if (!err) err = mz_cuda_memcpy_d2h(&tot, r->pre + nsel, sizeof(tot), stream);
    if (!err) err = mz_cuda_stream_sync(stream);
    st.pack_ms = now_ms() - t0 - st.setup_ms;
    if (!err) {
        *out_bytes = tot.out;
        st.entries = nsel;
        st.bytes_in = tot.cin;
        st.bytes_out = tot.cout;
        if (d_out && out_cap < tot.out)
            err = MZ_BUF_ERROR;
    }
    if (err || !d_out || !nsel) { /* sizing call, an empty selection, or an error: at most the offsets */
        sc.out_off = d_out_off;
        if (!err && d_out_off) err = mz_cuda_zip_sel_fill(&sc, stream);
        if (!err) err = mz_cuda_stream_sync(stream);
        zu_leave(r, prev);
        if (stats)
            *stats = st;
        return err;
    }
    /* 2. the selection's K9 table, and with WinZip AES entries every slot's extent gathered into scratch (K8 decrypts in place) */
    const int gather = tot.a[1] || tot.a[2] || tot.a[3];
    if (gather && tot.gather + 32 > r->gcap) {
        const double t1 = now_ms();
        mz_cuda_free(r->gbuf);
        r->gcap = 0;
        if (!(r->gbuf = (uint8_t *)mz_cuda_malloc(tot.gather + 32)))
            err = MZ_MEM_ERROR;
        else
            r->gcap = tot.gather + 32;
        st.setup_ms += now_ms() - t1;
    }
    const double t2 = now_ms();
    sc.gather = gather;
    sc.sel = r->sel;
    sc.out_off = d_out_off;
    sc.scratch = r->gbuf;
    if (!err) err = mz_cuda_zip_sel_fill(&sc, stream);
    if (!err && gather) {
        err = mz_cuda_memset(r->gbuf + tot.gather, 0, 32, stream);
        if (!err) err = mz_cuda_zip_sel_gather(&sc, stream);
    }
    /* 3. the round (K9 locate, K8, stored copy, K5, K1, K7, K9 verify), then each slot's status and the first failing slot */
    zr_slot *z = &r->z;
    z->n = nsel;
    z->njobs = tot.job;
    z->nsha = tot.sha;
    memcpy(z->na, tot.a, sizeof(z->na));
    z->na[0] = 0;
    memcpy(z->max_clen, r->max_clen, sizeof(z->max_clen)); /* the archive's largest ciphertext per strength: K8's bound */
    z->password = r->password;
    z->d_ent = r->sel;
    z->d_sha = (uint8_t *)r->sha;
    /* in place: buf_len = cd_off as extract_device reads it; gathered: the extents, 32 zero bytes behind them */
    if (!err) err = zr_launch(z, gather ? r->gbuf : (uint8_t *)r->archive, gather ? tot.gather : r->cd_off, (uint8_t *)d_out, stream);
    if (!err) err = mz_cuda_memset(r->first, 0xff, 8, stream);
    if (!err) err = mz_cuda_zip_sel_status(z->d_status, d_select, nsel, r->count, d_status, r->first, stream);
    uint64_t first = ~0ull;
    if (!err) err = mz_cuda_memcpy_d2h(&first, r->first, 8, stream);
    if (!err) err = mz_cuda_stream_sync(stream);
    if (!err && first != ~0ull)
        err = -(int32_t)(uint32_t)first;
    st.gpu_ms = now_ms() - t2;
    st.rounds = 1;
    mz_cuda_stream_sync(stream);
    zu_leave(r, prev);
    if (stats)
        *stats = st;
    return err;
}

void mz_zip_cuda_reader_close(mz_zip_cuda_dev_reader *r) {
    if (!r)
        return;
    int32_t prev;
    zu_enter(r, &prev);
    mz_cuda_free(r->entries);
    mz_cuda_free(r->ent);
    mz_cuda_free(r->sha);
    mz_cuda_free(r->table);
    mz_cuda_free(r->work);
    mz_cuda_free(r->selw);
    mz_cuda_free(r->gbuf);
    zu_leave(r, prev);
    free(r->password);
    free(r);
}

/* the argument checks of write_device, in the host writer's order: options, pointers, level, password and strength, the GPU; *level and
 * *aes_strength get their defaults */
static int32_t zw_args(const mz_cuda_zip_dev_item *d_items, uint32_t count, int16_t *level, uint32_t flags, const char *password,
                       uint8_t *aes_strength, uint64_t *archive_len) {
    if (flags & ~(MZ_ZIP_CUDA_HASH_SHA256 | MZ_ZIP_CUDA_AES))
        return MZ_PARAM_ERROR; /* MZ_ZIP_CUDA_ALL_DEVICES among them: the entries live on one device */
    if (!archive_len || (!d_items && count))
        return MZ_PARAM_ERROR;
    *archive_len = 0;
    if (*level == MZ_COMPRESS_LEVEL_DEFAULT)
        *level = 6;
    if (*level < 0 || *level > 9)
        return MZ_PARAM_ERROR;
    if (*aes_strength == 0)
        *aes_strength = 3;
    if ((flags & MZ_ZIP_CUDA_AES) && (!password || strlen(password) > 128 || *aes_strength > 3))
        return MZ_PARAM_ERROR;
    if (mzh_gpu_required("mz_zip_cuda"))
        return MZ_SUPPORT_ERROR;
    return MZ_OK;
}

/* what lies in front of the new entries: the kept entries of mz_zip_cuda_update_device; all zero for write_device */
typedef struct zw_front {
    uint64_t lh, cd, out;            /* archive bytes, directory bytes (zip64 fields included), 16-byte output slots */
    uint32_t n, comment_len;         /* entries; the end record's comment */
    const void *comment;             /* device; read when the end records are written */
    uint64_t bytes_in, bytes_out;    /* plain and stored bytes of those entries (stats) */
    /* called once the items passed and the call writes (before anything is written), and once the exact length fits cap (cd_off:
     * where the directory starts) */
    int32_t (*before)(void *ctx, void *stream);
    int32_t (*records)(void *ctx, uint64_t cd_off, void *stream);
    void *ctx;
} zw_front;

/* the body of write_device, behind f (arguments checked by zw_args; st zeroed) */
static int32_t zw_write(const zw_front *f, const void *d_data, const void *d_names, const mz_cuda_zip_dev_item *d_items, uint32_t count, int16_t level,
                        uint32_t flags, const char *password, uint8_t aes_strength, void *d_archive, uint64_t cap, uint64_t *archive_len,
                        mz_cuda_zip_dev_entry *d_entries, mz_cuda_zip_stats *stats_out, void *stream) {
    mz_cuda_zip_stats st;
    memset(&st, 0, sizeof(st));
    const int aes = (flags & MZ_ZIP_CUDA_AES) != 0;
    const double t0 = now_ms();
    mz_cuda_zip_wr w;
    memset(&w, 0, sizeof(w));
    w.data = d_data;
    w.names = d_names;
    w.items = d_items;
    w.n = count;
    w.aes = aes ? aes_strength : 0;
    w.sha = (flags & MZ_ZIP_CUDA_HASH_SHA256) != 0;
    w.dos_now = za_dos_date(0);
    w.archive = d_archive;
    w.cap = d_archive ? cap : 0;
    w.entries = d_entries ? d_entries + f->n : NULL;
    w.lh_base = f->lh;
    w.cd_base = f->cd;
    w.out_base = f->out;
    w.n_base = f->n;
    const size_t m = (size_t)count + 1, tiles = (size_t)count / MZ_CUDA_ZIP_WR_TILE + 1;
    /* 1. validation and per-item counts: the first invalid item and the totals come back */
    const mzh_piece p1[4] = {MZH_DEV(w.bad, 16), MZH_DEV(w.cnt, m * sizeof(mz_cuda_zip_wr_count)), MZH_DEV(w.pre, m * sizeof(mz_cuda_zip_wr_count)),
                             MZH_DEV(w.part, tiles * sizeof(mz_cuda_zip_wr_count))};
    double ts = now_ms();
    uint8_t *work1 = mzh_carve(p1, 4), *work2 = NULL;
    st.setup_ms += now_ms() - ts;
    if (!work1) {
        *stats_out = st;
        return MZ_MEM_ERROR;
    }
    int32_t err = mz_cuda_memset(w.bad, 0xff, 8, stream);
    if (!err) err = mz_cuda_zip_wr_items(&w, d_data == NULL, d_names == NULL, stream);
    uint64_t bad = ~0ull;
    mz_cuda_zip_wr_count tot;
    memset(&tot, 0, sizeof(tot));
    if (!err) err = mz_cuda_memcpy_d2h(&bad, w.bad, 8, stream);
    if (!err) err = mz_cuda_memcpy_d2h(&tot, w.pre + count, sizeof(tot), stream);
    if (!err) err = mz_cuda_stream_sync(stream);
    if (!err && bad != ~0ull)
        err = (bad & 1) ? MZ_SUPPORT_ERROR : MZ_PARAM_ERROR;
    if (!err && !d_archive) { /* sizing: the slot bound of every chunk, exact headers; the zip64 fields only when an offset can need them */
        const int big = f->lh + tot.overhead + tot.bound >= 0xffffffffull;
        *archive_len = f->lh + tot.overhead + tot.bound + f->cd + tot.cd + (big ? 28ull * count : 0) + 22 + f->comment_len +
                       (big || (uint64_t)f->n + count >= 0xffffu ? 76 : 0);
    }
    st.pack_ms = now_ms() - t0 - st.setup_ms; /* the scratch allocation is setup_ms */
    if (err || !d_archive) {
        mz_cuda_stream_sync(stream);
        mz_cuda_free(work1);
        *stats_out = st;
        return err;
    }
    if (f->before)
        err = f->before(f->ctx, stream);
    /* 2. scratch: the chunk table, a round of slots, per-entry arrays */
    w.nch = tot.chunks;
    const uint64_t R = mzh_round_chunks(w.nch);
    const uint64_t stride = mz_cuda_deflate_slot_bound(ZC_CHUNK);
    const size_t nch = (size_t)w.nch, n = count ? count : 1;
    const size_t ptiles = ((size_t)R > n ? (size_t)R : n) / MZ_CUDA_ZIP_WR_TILE + 1;
    uint8_t *slots = NULL, *pw = NULL;
    void *digest = NULL, *salt = NULL, *keys = NULL, *mac = NULL;
    void *part2 = NULL, *spare = NULL;
    const mzh_piece p2[26] = {MZH_DEV(w.c_off, nch * 8), MZH_DEV(w.c_len, nch * 4), MZH_DEV(w.c_flags, nch), MZH_DEV(w.c_item, nch * 4),
                              MZH_DEV(w.out_len, nch * 4), MZH_DEV(w.residue, nch * 4), MZH_DEV(w.glen, nch * 4), MZH_DEV(w.S, (nch + 1) * 8),
                              MZH_DEV(w.dst, nch * 8), MZH_DEV(w.e_lh, n * 8), MZH_DEV(w.e_csize, n * 8), MZH_DEV(w.e_cd, n * 8),
                              MZH_DEV(w.e_cdpre, (n + 1) * 8), MZH_DEV(w.e_coff, n * 8), MZH_DEV(w.e_off, n * 8), MZH_DEV(w.e_len, n * 8),
                              MZH_DEV(w.e_crc, n * 4), MZH_DEV(w.max_csize, 8), MZH_DEV(part2, ptiles * sizeof(mz_cuda_zip_wr_count)),
                              MZH_DEV(slots, (size_t)R * stride), MZH_DEV(digest, w.sha ? n * 32 : 32), MZH_DEV(salt, aes ? n * 16 : 16),
                              MZH_DEV(keys, aes ? n * MZ_CUDA_WZAES_KEYREC : 16), MZH_DEV(mac, aes ? n * 20 : 16), MZH_DEV(pw, 256),
                              MZH_DEV(spare, 16)};
    ts = now_ms();
    if (!err)
        work2 = mzh_carve(p2, 26);
    st.setup_ms += now_ms() - ts;
    if (!err && !work2)
        err = MZ_MEM_ERROR;
    w.part = part2;
    w.digest = digest;
    w.salt = salt;
    w.keys = keys;
    w.mac = mac;
    /* 3. the chunk table; SHA-256 of every entry (K7) */
    const double t1 = now_ms();
    if (!err) err = mz_cuda_memset(w.S, 0, 8, stream);
    if (!err) err = mz_cuda_memset(w.max_csize, 0, 8, stream);
    if (!err) err = mz_cuda_zip_wr_chunks(&w, stream);
    if (!err && w.sha) err = mz_cuda_sha256_batch(d_data ? d_data : digest, w.e_off, w.e_len, count, digest, stream);
    /* 4. rounds over the global chunk list: compress, checksum, place, gather into the archive; no host synchronisation between */
    for (uint64_t c0 = 0; !err && c0 < w.nch; c0 += R) {
        const uint32_t mr = (uint32_t)(w.nch - c0 < R ? w.nch - c0 : R);
        err = mz_cuda_deflate_chunks(d_data, 0, 0, w.c_off + c0, w.c_len + c0, w.c_flags + c0, mr, 0, level, slots, stride, w.out_len + c0, stream);
        if (!err) err = mz_cuda_crc32_segments(d_data, 0, 0, w.c_off + c0, w.c_len + c0, mr, w.residue + c0, NULL, stream);
        if (!err) err = mz_cuda_zip_wr_place(&w, c0, mr, stream);
        if (!err) err = mz_cuda_gather(slots, stride, w.glen + c0, mr, w.dst + c0, d_archive, stream);
        st.rounds++;
    }
    /* 5. per entry: CRC, sizes, offsets, directory layout; the exact length comes back */
    if (!err) err = mz_cuda_zip_wr_entries(&w, stream);
    uint64_t streams = 0, cd_size = 0, max_csize = 0;
    if (!err) err = mz_cuda_memcpy_d2h(&streams, w.S + w.nch, 8, stream);
    if (!err) err = mz_cuda_memcpy_d2h(&cd_size, w.e_cdpre + count, 8, stream);
    if (!err) err = mz_cuda_memcpy_d2h(&max_csize, w.max_csize, 8, stream);
    if (!err) err = mz_cuda_memcpy_d2h(&bad, w.bad, 8, stream);
    if (!err) err = mz_cuda_stream_sync(stream);
    const uint64_t cd_off = f->lh + tot.overhead + streams, ntot = (uint64_t)f->n + count;
    const uint64_t len = cd_off + f->cd + cd_size + 22 + f->comment_len + (cd_off >= 0xffffffffull || ntot >= 0xffffu ? 76 : 0);
    if (!err && bad != ~0ull)
        err = MZ_INTERNAL_ERROR; /* an entry's stored size does not fit its local header: what za_prepare returns for it */
    if (!err) {
        *archive_len = len;
        if (len > cap)
            err = MZ_BUF_ERROR;
    }
    /* 6. WinZip AES: fresh salts from the host, keys by K8, the streams encrypted in place, their HMACs; then headers, directory,
     * end records and the table */
    if (!err && aes && count) {
        uint8_t *h_salt = (uint8_t *)malloc((size_t)count * 16);
        size_t got = 0;
        if (!h_salt)
            err = MZ_MEM_ERROR;
        while (!err && got < (size_t)count * 16) {
            ssize_t k = getrandom(h_salt + got, (size_t)count * 16 - got, 0);
            if (k <= 0) { err = MZ_INTERNAL_ERROR; break; }
            got += (size_t)k;
        }
        const uint32_t pwl = (uint32_t)strlen(password);
        if (!err) err = mz_cuda_memcpy_h2d(salt, h_salt, (size_t)count * 16, stream);
        if (!err) err = mz_cuda_memcpy_h2d(pw, password, pwl ? pwl : 1, stream);
        if (!err) err = mz_cuda_stream_sync(stream); /* the pageable sources are freed below */
        free(h_salt);
        if (!err) err = mz_cuda_wzaes_derive(pw, pwl, salt, count, aes_strength, keys, stream);
        if (!err) err = mz_cuda_wzaes_ctr(d_archive, w.e_coff, w.e_csize, count, max_csize, keys, aes_strength, stream);
        if (!err) err = mz_cuda_wzaes_hmac(d_archive, w.e_coff, w.e_csize, count, keys, aes_strength, mac, stream);
    }
    if (!err && f->records) err = f->records(f->ctx, cd_off, stream);
    w.comment = f->comment;
    w.comment_len = f->comment_len;
    if (!err) err = mz_cuda_zip_wr_emit(&w, cd_off, f->cd + cd_size, stream);
    if (!err) err = mz_cuda_stream_sync(stream);
    st.gpu_ms = now_ms() - t1;
    if (!err || err == MZ_BUF_ERROR) {
        st.entries = f->n + count;
        st.bytes_in = f->bytes_in + tot.bytes;
        st.bytes_out = f->bytes_out + streams + (aes ? (uint64_t)count * (4u * aes_strength + 4u + 2u + 10u) : 0);
    }
    mz_cuda_stream_sync(stream);
    mz_cuda_free(work2);
    mz_cuda_free(work1);
    *stats_out = st;
    return err;
}

int32_t mz_zip_cuda_write_device(const void *d_data, const void *d_names, const mz_cuda_zip_dev_item *d_items, uint32_t count, int16_t level, uint32_t flags,
                                 const char *password, uint8_t aes_strength, void *d_archive, uint64_t cap, uint64_t *archive_len,
                                 mz_cuda_zip_dev_entry *d_entries, mz_cuda_zip_stats *stats, void *stream) {
    mz_cuda_zip_stats st;
    memset(&st, 0, sizeof(st));
    if (stats)
        *stats = st;
    int32_t err = zw_args(d_items, count, &level, flags, password, &aes_strength, archive_len);
    if (err)
        return err;
    zw_front f;
    memset(&f, 0, sizeof(f));
    err = zw_write(&f, d_data, d_names, d_items, count, level, flags, password, aes_strength, d_archive, cap, archive_len, d_entries, &st, stream);
    if (stats)
        *stats = st;
    return err;
}

/* ---- an archive in device memory updated on the device (mz_zip_cuda_update_device) ---------------------------------------- */
typedef struct zu_job {
    mz_cuda_zip_up u;
    uint64_t cd_off, src_len;   /* the source's directory; its length */
    int in_place;
    uint8_t *saved;             /* in place: the source's bytes from its directory on */
    uint64_t eocd;              /* the source's end record */
    zw_front *f;
} zu_job;

/* before anything is written: in place, save the source's directory and tail (the records and the comment are read from there);
 * then move the kept entries */
static int32_t zu_before(void *ctx, void *stream) {
    zu_job *j = (zu_job *)ctx;
    int32_t err = MZ_OK;
    if (j->in_place) {
        const uint64_t tail = j->src_len - j->cd_off;
        if (!(j->saved = (uint8_t *)mz_cuda_malloc(tail ? tail : 1)))
            return MZ_MEM_ERROR;
        if (tail) err = mz_cuda_memcpy_d2d(j->saved, (const uint8_t *)j->u.src + j->cd_off, tail, stream);
        j->u.dir = j->saved;
        j->f->comment = j->saved + (j->eocd + 22 - j->cd_off);
    }
    if (!err) err = mz_cuda_zip_up_copy(&j->u, stream);
    return err;
}

static int32_t zu_records(void *ctx, uint64_t cd_off, void *stream) {
    zu_job *j = (zu_job *)ctx;
    j->u.cd_off = cd_off;
    return mz_cuda_zip_up_records(&j->u, stream);
}

int32_t mz_zip_cuda_update_device(const void *d_src, uint64_t src_len, const uint32_t *d_keep, uint32_t nkeep, const void *d_data, const void *d_names,
                                  const mz_cuda_zip_dev_item *d_items, uint32_t count, int16_t level, uint32_t flags, const char *password,
                                  uint8_t aes_strength, void *d_archive, uint64_t cap, uint64_t *archive_len, mz_cuda_zip_dev_entry *d_entries,
                                  mz_cuda_zip_stats *stats, void *stream) {
    mz_cuda_zip_stats st;
    memset(&st, 0, sizeof(st));
    if (stats)
        *stats = st;
    /* 1. arguments: write_device's, then the source and the two buffers */
    int32_t err = zw_args(d_items, count, &level, flags, password, &aes_strength, archive_len);
    if (err)
        return err;
    if ((!d_src && src_len) || (!d_keep && nkeep))
        return MZ_PARAM_ERROR;
    const uintptr_t s0 = (uintptr_t)d_src, a0 = (uintptr_t)d_archive;
    const int in_place = d_archive && a0 == s0;
    if (in_place && d_keep)
        return MZ_PARAM_ERROR;
    if (d_archive && !in_place && cap && a0 < s0 + src_len && s0 < a0 + cap)
        return MZ_PARAM_ERROR; /* partly overlapping buffers */
    const double t0 = now_ms();
    /* 2. the source's directory (K10): nothing is decrypted, so it is parsed as if a password had been given */
    mz_cuda_zip_dir dir;
    memset(&dir, 0, sizeof(dir));
    dir.have_password = 1;
    dir.max_entries = 0xffffffffu;
    dir.alloc_entries = 1;
    err = mz_cuda_zip_parse_directory(d_src, src_len, &dir, stream);
    if (err == MZ_OK && dir.err)
        err = dir.err;
    if (err == MZ_OK && dir.refuse)
        err = dir.refuse; /* a refused record: the entries behind it are not dropped silently */
    const uint32_t n = d_keep ? nkeep : dir.count;
    zu_job j;
    memset(&j, 0, sizeof(j));
    zw_front f;
    memset(&f, 0, sizeof(f));
    j.f = &f;
    j.cd_off = dir.cd_off;
    j.src_len = src_len;
    j.in_place = in_place;
    mz_cuda_zip_up *u = &j.u;
    u->src = d_src;
    u->ent = dir.entries;
    u->count = dir.count;
    u->n = n;
    u->keep = d_keep;
    u->dir = (const uint8_t *)d_src + dir.cd_off;
    u->dir_off = dir.cd_off;
    u->src_len = src_len;
    u->archive = d_archive;
    u->cap = d_archive ? cap : 0;
    u->entries = d_entries;
    /* 3. kept counts, their scan and the layout facts; one readback */
    uint8_t *work = NULL;
    if (!err) {
        const size_t m = (size_t)n + 1;
        const mzh_piece t[4] = {MZH_DEV(u->cnt, m * sizeof(mz_cuda_zip_up_count)), MZH_DEV(u->pre, m * sizeof(mz_cuda_zip_up_count)),
                                MZH_DEV(u->part, ((size_t)n / MZ_CUDA_ZIP_WR_TILE + 1) * sizeof(mz_cuda_zip_up_count)),
                                MZH_DEV(u->info, 8 * MZ_CUDA_ZIP_UP_INFO)};
        const double ts = now_ms();
        work = mzh_carve(t, 4);
        st.setup_ms += now_ms() - ts;
        if (!work)
            err = MZ_MEM_ERROR;
    }
    mz_cuda_zip_up_count tot;
    memset(&tot, 0, sizeof(tot));
    uint64_t info[MZ_CUDA_ZIP_UP_INFO];
    memset(info, 0, sizeof(info));
    if (!err) err = mz_cuda_memset(u->info, 0xff, 8 * MZ_CUDA_ZIP_UP_INFO, stream);
    if (!err) err = mz_cuda_memset(u->info + 4, 0, 16, stream);
    if (!err) err = mz_cuda_zip_up_counts(u, stream);
    if (!err) err = mz_cuda_memcpy_d2h(&tot, u->pre + n, sizeof(tot), stream);
    if (!err) err = mz_cuda_memcpy_d2h(info, u->info, sizeof(info), stream);
    if (!err) err = mz_cuda_stream_sync(stream);
    /* 4. a keep index out of range; in place, kept bytes that would move or a directory that does not start where they end */
    if (!err && info[1] != ~0ull)
        err = MZ_PARAM_ERROR;
    if (!err && in_place && (info[2] != ~0ull || tot.ext != dir.cd_off))
        err = MZ_PARAM_ERROR;
    if (!err && info[3] != ~0ull)
        err = MZ_SUPPORT_ERROR; /* a kept record's extra field cannot take the zip64 field it needs */
    const uint64_t first64 = info[0] < n ? info[0] : n;
    f.lh = tot.ext;
    f.cd = tot.cd + 28ull * (n - first64);
    f.out = tot.out16;
    f.n = n;
    f.comment_len = (uint32_t)info[5];
    f.comment = (const uint8_t *)d_src + info[4] + 22;
    f.bytes_in = tot.bytes;
    f.bytes_out = tot.stored;
    f.before = zu_before;
    f.records = zu_records;
    f.ctx = &j;
    const double parse_ms = now_ms() - t0 - st.setup_ms, setup_ms = st.setup_ms;
    j.eocd = info[4];
    if ((uint64_t)n + count > 0xffffffffull && !err)
        err = MZ_PARAM_ERROR;
    /* 5. - 9. the items, [sizing], the save and the copy, the new entries, the records, the end records: write_device's body */
    if (!err)
        err = zw_write(&f, d_data, d_names, d_items, count, level, flags, password, aes_strength, d_archive, cap, archive_len, d_entries, &st, stream);
    st.pack_ms += parse_ms;
    st.setup_ms += setup_ms;
    if (err && j.saved) { /* put the source's directory and tail back: the source stays a valid archive */
        const uint64_t end = src_len < cap ? src_len : cap;
        if (end > j.cd_off) mz_cuda_memcpy_d2d((uint8_t *)d_src + j.cd_off, j.saved, end - j.cd_off, stream);
    }
    mz_cuda_stream_sync(stream);
    mz_cuda_free(j.saved);
    mz_cuda_free(work);
    mz_cuda_free(dir.entries);
    mz_cuda_free(dir.ent);
    mz_cuda_free(dir.sha_expect);
    if (stats)
        *stats = st;
    return err;
}
