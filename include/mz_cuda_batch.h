/* mz_cuda_batch.h -- device-pointer batch API of the H100 DEFLATE + CRC-32 backend (C ABI).
 *
 * ADDITIVE to the reference: minizip-ng has no batch interface (SURVEY.md section 8b "Beyond the vtbl").
 * It exists so that (a) the vtbl stream (mz_strm_cuda.h) has something to drive, (b) kernels can be
 * measured on device-resident buffers against the HBM roofline, (c) chunks / zip entries can be sharded
 * over GPUs. Plain pointers and sizes only; `stream` is a cudaStream_t passed as void* (NULL = default).
 * All functions return MZ_OK (0) or a negative MZ_* code (mz.h:21-47); MZ_CUDA_ERROR details are
 * available from mz_cuda_last_error().  Device pointers must belong to the CURRENT CUDA device.
 */
#ifndef MZ_CUDA_BATCH_H
#define MZ_CUDA_BATCH_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MZ_CUDA_CHUNK_MAX    65536u /* largest independent DEFLATE chunk */
#define MZ_CUDA_FLAG_FINAL   1u     /* chunk ends its stream (BFINAL, no sync marker) */
#define MZ_CUDA_FLAG_DICT    2u     /* the 32 KiB in front of the chunk (same buffer) are earlier bytes of the SAME stream: at levels 6-9 the
                                    * chunk may refer back into them (zlib's sliding window across our chunk boundaries). In `last_flags` of a
                                    * uniform partition it applies to every chunk: the buffer is one stream. */

/* ---- runtime ---------------------------------------------------------------------------------- */
int32_t mz_cuda_init(void);                 /* idempotent, thread-safe; MZ_SUPPORT_ERROR without a usable GPU */
int32_t mz_cuda_device_count(void);
int32_t mz_cuda_set_device(int32_t ordinal);
int32_t mz_cuda_get_device(void);           /* the calling thread's current device, -1 on failure */
const char *mz_cuda_last_error(void);
int32_t mz_cuda_sm_count(void);

void *mz_cuda_malloc(size_t bytes);         /* device memory; NULL on failure */
void mz_cuda_free(void *dptr);
void *mz_cuda_host_alloc(size_t bytes);     /* pinned host memory */
void mz_cuda_host_free(void *hptr);
int32_t mz_cuda_memcpy_h2d(void *dptr, const void *hptr, size_t bytes, void *stream);  /* async on stream */
int32_t mz_cuda_memcpy_d2h(void *hptr, const void *dptr, size_t bytes, void *stream);  /* async on stream */
int32_t mz_cuda_memcpy_d2d(void *dst, const void *src, size_t bytes, void *stream);
int32_t mz_cuda_memset(void *dptr, int value, size_t bytes, void *stream);
int32_t mz_cuda_host_is_pinned(const void *hptr);           /* 1 if page-locked and usable for async copies */
int32_t mz_cuda_stream_sync(void *stream);
void *mz_cuda_stream_create(void);
void mz_cuda_stream_destroy(void *stream);
void *mz_cuda_event_create(void);
void mz_cuda_event_destroy(void *event);
int32_t mz_cuda_event_record(void *event, void *stream);
int32_t mz_cuda_event_sync(void *event);
int32_t mz_cuda_event_query(void *event); /* 1 = complete, 0 = not yet, < 0 = MZ_* error */
float mz_cuda_event_elapsed_ms(void *start, void *stop); /* syncs on stop */

/* ---- K1: CRC-32 ---------------------------------------------------------------------------------
 * Segments: either a uniform partition (d_off = d_len = NULL: segment i = bytes [i*seg_size, ...) of
 * total_len) or explicit per-segment offsets/lengths (device arrays). d_residue[i] = pure residue
 * R(segment) (init 0, no final xor) -- the linear quantity that folds; d_crc[i] (optional) = the value
 * mz_crypt_crc32_update(0, segment, len) returns (mz_crypt.c:35). */
int32_t mz_cuda_crc32_segments(const void *d_in, uint64_t total_len, uint64_t seg_size, const uint64_t *d_off,
                               const uint32_t *d_len, uint32_t nseg, uint32_t *d_residue, uint32_t *d_crc, void *stream);
/* fold the residues of a UNIFORM partition: d_out2[0] = residue of the whole buffer, d_out2[1] = crc32(0, buffer) */
int32_t mz_cuda_crc32_fold(const uint32_t *d_residue, uint32_t nseg, uint64_t seg_size, uint64_t total_len, uint32_t *d_out2,
                           void *stream);
/* whole device buffer, synchronous: *crc = mz_crypt_crc32_update(value, buffer, len) */
int32_t mz_cuda_crc32_device(const void *d_in, uint64_t len, uint32_t value, uint32_t *crc);
/* same, enqueued on `stream` and synchronised on it only (the scratch buffer is shared: one caller per device at a time) */
int32_t mz_cuda_crc32_device_stream(const void *d_in, uint64_t len, uint32_t value, uint32_t *crc, void *stream);
/* host arithmetic: crc(A||B) from crc(A), crc(B), |B|  (the "polynomial combine" of the north star) */
uint32_t mz_cuda_crc32_combine(uint32_t crc_a, uint32_t crc_b, uint64_t len_b);

/* ---- K2+K3: DEFLATE encode of independent chunks --------------------------------------------------
 * Chunk i (<= MZ_CUDA_CHUNK_MAX bytes) is compressed into slot i = d_slots + i*slot_stride
 * (slot_stride >= mz_cuda_deflate_slot_bound(chunk size), multiple of 16; d_slots 16-byte aligned);
 * d_out_len[i] = bytes written. Every slot is a byte-aligned piece of raw RFC1951 data: non-final
 * chunks end with a sync-flush marker, chunks flagged FINAL end with BFINAL. Uniform partition when
 * d_off == NULL (then only the last chunk gets the FINAL bit of `last_flags`). level 0 = stored, 1 = candidates at every second
 * position, 2-3 = every position, 4-5 = + one-step lazy evaluation, 6-9 = + the previous 32 KiB as history (inside a chunk: its
 * first half for its second; with MZ_CUDA_FLAG_DICT also the bytes in front of the chunk). */
uint64_t mz_cuda_deflate_slot_bound(uint32_t chunk_size);
int32_t mz_cuda_deflate_chunks(const void *d_in, uint64_t total_len, uint32_t chunk_size, const uint64_t *d_off,
                               const uint32_t *d_len, const uint8_t *d_flags, uint32_t nchunks, uint32_t last_flags,
                               int32_t level, void *d_slots, uint64_t slot_stride, uint32_t *d_out_len, void *stream);
/* ---- K4: join slots into one contiguous stream ------------------------------------------------------
 * d_offsets: nchunks+1 uint64 (scratch/out): d_offsets[i] = position of chunk i in d_dst, [nchunks] = total. */
int32_t mz_cuda_concat(const void *d_slots, uint64_t slot_stride, const uint32_t *d_out_len, uint32_t nchunks,
                       uint64_t *d_offsets, void *d_dst, void *stream);

/* ---- multi-GPU: chunk-sharded DEFLATE, all-gather on the copy engines ---------------------------------------------------
 * Chunks are independent, so device r of N owns a contiguous chunk range; the only exchange is the all-gather of the joined
 * bitstreams and of the per-chunk {crc32, in_len, out_len} rows. It is done with peer-to-peer copies (cudaMemcpyPeerAsync /
 * IPC-mapped destinations): the copy engines move the bytes over NVLink while every SM keeps compressing -- an SM-based
 * collective cannot co-reside with the 2 x 111 KB deflate CTAs and serialises with them.
 *
 * (a) one process, N devices (a C host):  mz_cuda_deflate_sharded()
 * (b) one process per device (torchrun):  export / open IPC handles of the gathered buffers once, then mz_cuda_memcpy_peer(). */
typedef struct mz_cuda_shard {
    int32_t device;          /* CUDA ordinal */
    const void *d_in;        /* this device's shard of the input (on `device`), 16-byte aligned */
    uint64_t len;            /* bytes; every shard but the last must be a multiple of 64 KiB */
    void *d_gathered;        /* on `device`: receives EVERY device's joined stream; device r's stream starts at region_off[r] */
    uint64_t gathered_cap;
    uint32_t *d_rows;        /* on `device`: receives every device's rows {crc32, in_len, out_len} (3 x uint32 per chunk), in
                                global chunk order (device r's rows start at chunk index = sum of earlier devices' chunks) */
} mz_cuda_shard;
/* Compress + CRC + join every shard on its device (level 0..9, BFINAL on the globally last chunk) and all-gather: after the
 * call every device holds all streams and all rows. region_off[r], stream_len[r] (arrays of ndev, host) describe where device
 * r's stream lies in every gathered buffer: region_off[r] = sum over earlier devices of mz_cuda_gather_region_bound(len);
 * the rank-ordered concatenation of the N streams is ONE valid raw DEFLATE stream. *crc32 = CRC-32 of the whole input
 * (host fold of the per-device CRCs). `pieces` >= 1: each shard is compressed in that many pieces and a finished piece
 * travels while the next one is being compressed. Synchronous. */
uint64_t mz_cuda_gather_region_bound(uint64_t shard_len);
int32_t mz_cuda_deflate_sharded(const mz_cuda_shard *shards, int32_t ndev, int32_t level, int32_t pieces, uint64_t *region_off,
                                uint64_t *stream_len, uint32_t *crc32);
/* IPC: handle64 = 64 opaque bytes to hand to the other processes; open() maps a peer's allocation into this process (peer
 * access is enabled lazily); memcpy_peer() = cudaMemcpyAsync between any two device pointers of this process's address space
 * (own or IPC-mapped), executed by a copy engine. The exported pointer must come from mz_cuda_malloc(). */
int32_t mz_cuda_ipc_export(const void *dptr, void *handle64);
int32_t mz_cuda_ipc_open(const void *handle64, void **dptr);
int32_t mz_cuda_ipc_close(void *dptr);
int32_t mz_cuda_memcpy_peer(void *dst, const void *src, size_t bytes, void *stream);
int32_t mz_cuda_stream_wait_event(void *stream, void *event);

/* ---- K7: SHA-256 of independent buffers ----------------------------------------------------------------------
 * Message i = d_in[d_off[i] .. d_off[i] + d_len[i]); d_digest receives n x 32 bytes (the digest as the standard prints it).
 * This is the per-entry hash of the reference's zip writer / reader (MZ_ZIP_EXTENSION_HASH, mz_zip_rw.c:1339-1420, :410-450),
 * batched like the per-entry CRC. */
int32_t mz_cuda_sha256_batch(const void *d_in, const uint64_t *d_off, const uint64_t *d_len, uint32_t n, void *d_digest, void *stream);

/* K8: the arithmetic of WinZip AES entries (mz_strm_wzaes.c) for a batch of zip entries, every entry with its own salt.
 * strength = MZ_AES_STRENGTH_128 / _192 / _256 (1 / 2 / 3, mz.h:117-119): key 16 / 24 / 32 bytes, salt 8 / 12 / 16 bytes.
 *   derive: PBKDF2-HMAC-SHA1, 1000 iterations (mz_strm_wzaes.c:95-97) of the password with salt e (d_salts + 16 e) into the key
 *           record d_keys + MZ_CUDA_WZAES_KEYREC * e: encryption key at +0, authentication key at +32, 2-byte verifier at +64.
 *   ctr:    XOR entry e's bytes d_data[d_off[e] .. + d_len[e]) in place with the AES-CTR key stream of its encryption key
 *           (counter little-endian, first block 1, mz_strm_wzaes.c:147-171) -- encrypts and decrypts. max_len >= every d_len[e].
 *   hmac:   HMAC-SHA1 (authentication key) of entry e's bytes -> d_mac + 20 e; the entry stores the first 10 (:236-256). */
#define MZ_CUDA_WZAES_KEYREC 80
int32_t mz_cuda_wzaes_derive(const void *d_password, uint32_t pw_len, const void *d_salts, uint32_t n, uint32_t strength, void *d_keys, void *stream);
int32_t mz_cuda_wzaes_ctr(void *d_data, const uint64_t *d_off, const uint64_t *d_len, uint32_t n, uint64_t max_len, const void *d_keys, uint32_t strength,
                          void *stream);
int32_t mz_cuda_wzaes_hmac(const void *d_data, const uint64_t *d_off, const uint64_t *d_len, uint32_t n, const void *d_keys, uint32_t strength, void *d_mac,
                           void *stream);

/* K4 with caller-given destinations: slot i goes to d_dst + d_offsets[i] (no scan) -- the zip archive writer interleaves the
 * entries' streams with their local headers; and n small blobs (blob i = d_blob[d_blob_off[i] .. d_blob_off[i+1])) scattered to
 * d_dst + d_dst_off[i] (the headers themselves). */
int32_t mz_cuda_gather(const void *d_slots, uint64_t slot_stride, const uint32_t *d_out_len, uint32_t nchunks, const uint64_t *d_offsets,
                       void *d_dst, void *stream);
int32_t mz_cuda_scatter_blobs(const void *d_blob, const uint32_t *d_blob_off, const uint64_t *d_dst_off, uint32_t n, void *d_dst, void *stream);

/* ---- K5: DEFLATE decode of independent raw streams (resumable) ---------------------------------------- */
typedef struct mz_cuda_inflate_job {
    const void *d_in;    /* d_in[0] = stream byte `in_base`; readable (zero padded) 16 bytes past in_avail */
    uint64_t in_base;
    uint64_t in_avail;
    void *d_out;         /* d_out[0] = output byte `out_base`; keeps >= 32 KiB of history once out_pos > 0 */
    uint64_t out_base;
    uint64_t out_cap;
    uint32_t in_final;   /* no more input will follow */
    uint32_t flags;      /* MZ_CUDA_INFLATE_STOP_AT_BLOCK: return (why = 3) after the next completed block */
} mz_cuda_inflate_job;
#define MZ_CUDA_INFLATE_STOP_AT_BLOCK 1u

typedef struct mz_cuda_inflate_state {
    uint64_t in_bitpos;  /* consumed bits of the raw stream (TOTAL_IN = ceil(in_bitpos / 8) at END) */
    uint64_t out_pos;    /* produced bytes (TOTAL_OUT) */
    int32_t status;      /* 0 running, 1 end of stream, MZ_DATA_ERROR (-3), MZ_BUF_ERROR (-5) */
    int32_t why;         /* when running: 1 needs input, 2 needs output space, 3 stopped at a block boundary */
    uint32_t phase, last_block, stored_remaining, nlit, ndist, blocks;
    uint8_t lens[320];
} mz_cuda_inflate_state;

int32_t mz_cuda_inflate_streams(const mz_cuda_inflate_job *d_jobs, mz_cuda_inflate_state *d_states, uint32_t nstreams,
                                void *stream);

/* ---- K9: zip entries located, copied and verified on the device (csrc/zipdir_kernel.cuh) ------------------------------
 * A round = the stored bytes of n zip entries in one device buffer + one record per entry from the central directory. */
typedef struct mz_cuda_zip_ent {
    uint64_t src_off;   /* in the round's buffer: the entry's local header, or (MZ_CUDA_ZIP_ENT_AT_DATA) its stored bytes */
    uint64_t src_len;   /* the entry's extent: nothing of it lies past src_off + src_len */
    uint64_t csize;     /* stored bytes as recorded (WinZip AES: salt + verifier + ciphertext + authentication code) */
    uint64_t usize;     /* plain bytes as recorded */
    uint64_t out_off;   /* the plain bytes go to out + out_off (16-byte aligned) */
    uint32_t crc;       /* CRC-32 as recorded */
    uint32_t job;       /* DEFLATE entries: index of the entry's K5 job and state */
    uint32_t aes_slot;  /* WinZip AES entries: row of the K8 tables (salt, keys, MAC, ciphertext offset / length) */
    uint32_t sha_slot;  /* row of the expected SHA-256 digests, or 0xffffffff */
    uint16_t method;    /* 0 (STORE) or 8 (DEFLATE) */
    uint8_t aes;        /* 0, or the WinZip AES strength 1..3 */
    uint8_t flags;      /* MZ_CUDA_ZIP_ENT_AT_DATA */
    uint32_t pad;
} mz_cuda_zip_ent;
#define MZ_CUDA_ZIP_ENT_AT_DATA 1u

typedef struct mz_cuda_zip_round { /* device pointers; per entry unless noted */
    const void *buf;               /* the round's stored bytes, 32 readable bytes past buf_len */
    uint64_t buf_len;
    void *out;                     /* plain bytes */
    const mz_cuda_zip_ent *ent;
    uint32_t n, pad;
    mz_cuda_inflate_job *jobs;     /* per DEFLATE entry (written by locate) */
    const mz_cuda_inflate_state *states;
    uint64_t *seg_off, *seg_len64, *data_off; /* written by locate: the plain bytes' segment (K1 / K7), the stream's start in buf */
    uint32_t *seg_len;
    const uint32_t *crc;           /* K1 result over seg_* */
    const void *digest;            /* K7 result over seg_*, 32 bytes per entry (read only for entries with a sha_slot) */
    const void *sha_expect;        /* 32 bytes per sha_slot */
    void *salt;                    /* per aes_slot: 16 bytes (written by locate) */
    uint64_t *coff, *clen;         /* per aes_slot: ciphertext offset in buf and length (written by locate) */
    const void *keys, *mac;        /* per aes_slot: K8 key records and HMACs */
    uint32_t *status;              /* 0, or class << 24 | -MZ_code (1 locate, 2 AES, 3 stream / CRC / hash) */
} mz_cuda_zip_round;
/* locate: status, jobs, seg_*, data_off, salt / coff / clen. stored: STORE entries' bytes to out. verify: the final status words
 * (needs keys / mac for AES entries, states, crc, digest). */
int32_t mz_cuda_zip_locate(const mz_cuda_zip_round *round, void *stream);
int32_t mz_cuda_zip_copy_stored(const mz_cuda_zip_round *round, void *stream);
int32_t mz_cuda_zip_verify(const mz_cuda_zip_round *round, void *stream);

/* ---- K10: the central directory of an archive in device memory (csrc/zipcd_kernel.cuh) --------------------------------
 * The parse behind mz_zip_cuda_extract_device (include/mz_zip_cuda.h): end records, the record chain from the directory's first
 * record, each record's fields and refusal rules, extents and the output layout, all on the device; only a few scalars come back
 * (it synchronises on `stream` between its stages). On return: err = an error of the archive as a whole (then nothing else is
 * set); count = records accepted, refuse = the error of the record that ended the list (MZ_OK if none); the totals. The
 * tables fit when max_entries >= count and, with `decode` set, out_cap >= out_bytes; otherwise nothing more is written. When they
 * fit, `entries` (if not NULL) is filled (mz_cuda_zip_dev_entry, status 0) and, with `decode` set, `ent` (count K9 records: src_off = local header in the archive, src_len =
 * extent) and `sha_expect` (nsha expected digests, 32 bytes each, the K9 sha_slot rows) are allocated on the device and filled;
 * the caller frees them with mz_cuda_free. The function's own return value is MZ_OK or a CUDA / memory error. */
typedef struct mz_cuda_zip_dir {
    /* in */
    uint32_t have_password, password_long; /* a password was given; it is longer than 128 bytes */
    void *entries;                         /* device table of mz_cuda_zip_dev_entry, or NULL */
    uint32_t max_entries, decode;
    uint64_t out_cap;
    /* out */
    int32_t err, refuse;
    uint32_t count, njobs, nsha, na[4], pad; /* na[s]: entries of WinZip AES strength s */
    uint64_t cd_off, out_bytes, bytes_in, bytes_out, max_clen[4];
    mz_cuda_zip_ent *ent;
    void *sha_expect;
    /* in: with entries == NULL, allocate the public table (count rows) when it fits and set entries to it; the caller frees it
     * with mz_cuda_free (the reader of mz_zip_cuda_reader_open keeps it) */
    uint32_t alloc_entries, pad2;
} mz_cuda_zip_dir;
int32_t mz_cuda_zip_parse_directory(const void *d_archive, uint64_t len, mz_cuda_zip_dir *dir, void *stream);
/* after mz_cuda_zip_verify: each entry's status (0 or -MZ code) into the mz_cuda_zip_dev_entry table, and *d_first lowered to the
 * index of the first failing entry (the caller sets it to 0xffffffff first) */
int32_t mz_cuda_zip_statuses(const uint32_t *d_status, uint32_t n, void *d_entries, uint32_t *d_first, void *stream);

/* ---- K12: random access to an archive in device memory (csrc/zipsel_kernel.cuh) ---------------------------------------
 * The device half of the reader (mz_zip_cuda_reader_*, include/mz_zip_cuda.h). Name index: d_table holds P slots (a power of
 * two >= 2 x n, every slot ~0 before the build) of hash tag << 32 | entry index; the build inserts every one of the n entries of
 * the public table (names read from d_archive). Lookup: one thread per query (d_names + d_name_off[q], d_name_len[q] bytes);
 * d_index[q] = the smallest entry index whose name equals the query under mz_zip_path_compare(name, query, ignore_case), or
 * 0xffffffff. A lookup costs its probe length plus one compare per entry whose folded name hashes the same. P = 0: every query
 * misses. */
int32_t mz_cuda_zip_name_index(const void *d_archive, const void *d_entries, uint32_t n, uint64_t *d_table, uint32_t P, void *stream);
int32_t mz_cuda_zip_name_lookup(const void *d_archive, const void *d_entries, const uint64_t *d_table, uint32_t P, const void *d_names,
                                const uint64_t *d_name_off, const uint32_t *d_name_len, uint32_t nq, uint8_t ignore_case, uint32_t *d_index,
                                void *stream);
/* A selection of n slots, slot i = entry select[i] of the archive-wide K9 table ent (count rows, src_off / src_len = local header
 * and extent in the archive). count: per-slot counts and their exclusive scan pre[0..n] (part: scan scratch of n /
 * MZ_CUDA_ZIP_WR_TILE + 1 rows). fill: out_off[0..n] (if not NULL) and, with sel, the selection's K9 records (src_off in scratch
 * at pre.gather when gather is set, otherwise in the archive); an index >= count gets an inert record. gather: every valid
 * slot's extent to scratch + pre.gather. status: after mz_cuda_zip_verify, out[i] (if not NULL) = slot i's MZ code
 * (MZ_END_OF_LIST for an index >= count), *d_first (~0 before) lowered to slot << 32 | -code of the first failing slot. */
typedef struct mz_cuda_zip_sel_count { /* per slot; pre[i] = the sum over the slots in front of i */
    uint64_t out;       /* plain bytes rounded up to 16 */
    uint64_t cin, cout; /* stored and plain bytes */
    uint64_t gather;    /* extent rounded up to 16 */
    uint32_t job, sha;  /* DEFLATE (K5 job), an expected SHA-256 */
    uint32_t a[4];      /* a[s]: WinZip AES strength s */
} mz_cuda_zip_sel_count;
typedef struct mz_cuda_zip_sel {
    const void *archive;
    const mz_cuda_zip_ent *ent;
    uint32_t count, n;
    const uint32_t *select;
    mz_cuda_zip_sel_count *cnt, *pre;
    void *part;
    uint32_t gather, pad;
    mz_cuda_zip_ent *sel;
    uint64_t *out_off;
    void *scratch;
} mz_cuda_zip_sel;
int32_t mz_cuda_zip_sel_counts(const mz_cuda_zip_sel *c, void *stream);
int32_t mz_cuda_zip_sel_fill(const mz_cuda_zip_sel *c, void *stream);
int32_t mz_cuda_zip_sel_gather(const mz_cuda_zip_sel *c, void *stream);
int32_t mz_cuda_zip_sel_status(const uint32_t *d_status, const uint32_t *d_select, uint32_t n, uint32_t count, int32_t *d_out, uint64_t *d_first,
                               void *stream);

/* ---- K11: a zip archive written into device memory (csrc/zipwr_kernel.cuh) --------------------------------------------
 * The device half of mz_zip_cuda_write_device (include/mz_zip_cuda.h). One call state, device pointers unless noted; the host
 * carves the arrays and runs: items (validation, per-item counts and their exclusive scan pre[0..n]), chunks (the K2+K3 / K1
 * chunk table and K7's segments), per round K2+K3 + K1 over chunks [c0, c0 + m) then place (stream offsets S, destinations dst,
 * copy lengths glen: 0 for a chunk that would pass cap) then K4 mz_cuda_gather(slots, stride, glen + c0, m, dst + c0, archive),
 * entries (CRC fold, sizes, local-header offsets, directory record sizes and their scan e_cdpre[0..n]), [K8 over e_coff /
 * e_csize], emit (local headers, salts, verifiers, authentication codes, directory, end records, the mz_cuda_zip_dev_entry
 * table). `part`: scan scratch of (max(n, m) / MZ_CUDA_ZIP_WR_TILE + 1) x 48 bytes. A round holds at most 32768 chunks. */
#define MZ_CUDA_ZIP_WR_TILE 2048u
typedef struct mz_cuda_zip_wr_count { /* per item; pre[e] = the sum over the items in front of e */
    uint64_t chunks;    /* 64 KiB chunks (an empty entry has one) */
    uint64_t overhead;  /* local header + name + extra fields + salt + verifier + authentication code */
    uint64_t bytes;     /* plain bytes */
    uint64_t out16;     /* plain bytes rounded up to 16 (mz_zip_cuda_extract_device's output layout) */
    uint64_t bound;     /* mz_cuda_deflate_slot_bound of every chunk */
    uint64_t cd;        /* directory record without a zip64 field */
} mz_cuda_zip_wr_count;
typedef struct mz_cuda_zip_wr {
    const void *data, *names;
    const void *items;                     /* mz_cuda_zip_dev_item[n] */
    uint32_t n, aes, sha, dos_now;         /* aes: WinZip AES strength or 0; sha: hash fields; dos_now: the date of items with 0 */
    void *archive;
    uint64_t cap;
    uint64_t *bad;                         /* 1 word, ~0 before items: index << 1 | (0 = MZ_PARAM_ERROR, 1 = MZ_SUPPORT_ERROR) */
    mz_cuda_zip_wr_count *cnt, *pre;       /* n, n + 1 */
    void *part;
    uint64_t nch;                          /* host: pre[n].chunks */
    uint64_t *c_off;                       /* per chunk (nch) ... */
    uint32_t *c_len;
    uint8_t *c_flags;
    uint32_t *c_item, *out_len, *residue, *glen;
    uint64_t *S, *dst;                     /* S: nch + 1, S[0] = 0 */
    uint64_t *e_lh, *e_csize, *e_cd, *e_cdpre, *e_coff, *e_off, *e_len; /* per entry (e_cdpre: n + 1) */
    uint32_t *e_crc;
    uint64_t *max_csize;                   /* 1 word, 0 before entries */
    const void *digest, *salt, *keys, *mac; /* per entry: SHA-256 (sha), K8 salt / key record / HMAC (aes) */
    void *entries;                         /* mz_cuda_zip_dev_entry[n] or NULL */
    /* what lies in front of the new entries (mz_zip_cuda_update_device; all 0 for write_device): archive bytes (added to every
     * local-header offset, so the zip64 decision sees absolute offsets), directory bytes in front of the first new record, output
     * bytes in front of the first new row's out_off, entries (counted in the end records); the end record's comment (device) */
    uint64_t lh_base, cd_base, out_base;
    uint32_t n_base, comment_len;
    const void *comment;
} mz_cuda_zip_wr;
int32_t mz_cuda_zip_wr_items(const mz_cuda_zip_wr *w, uint32_t data_null, uint32_t names_null, void *stream);
int32_t mz_cuda_zip_wr_chunks(const mz_cuda_zip_wr *w, void *stream);
int32_t mz_cuda_zip_wr_place(const mz_cuda_zip_wr *w, uint64_t c0, uint32_t m, void *stream);
int32_t mz_cuda_zip_wr_entries(const mz_cuda_zip_wr *w, void *stream);
int32_t mz_cuda_zip_wr_emit(const mz_cuda_zip_wr *w, uint64_t cd_off, uint64_t cd_size, void *stream);

/* ---- K13: an archive in device memory updated on the device (csrc/zipup_kernel.cuh) ---------------------------------------
 * The device half of mz_zip_cuda_update_device (include/mz_zip_cuda.h). Slot i of n keeps entry keep[i] (keep NULL: entry i) of
 * the source's K10 public table ent (count rows). counts: per-slot counts, their exclusive scan pre[0..n] (pre[i].ext is slot i's
 * new local-header offset), then info: [0] the first slot whose offset needs the zip64 field (>= n: none), [1] the first keep index
 * >= count, [2] the first slot whose bytes move or whose extent holds more than its local header, stored bytes and data descriptor, [3] the first slot whose record would pass 65535 bytes of extra field, [4] / [5]
 * the source's end record and its comment length; [0..3] are ~0 before the call when nothing applies. `part`: scan scratch of
 * (n / MZ_CUDA_ZIP_WR_TILE + 1) counts. copy: every slot's extent (local header, stored bytes, descriptor) from src to archive +
 * pre[i].ext, stores below cap only; a slot whose destination is its source is skipped. records: slot i's directory record at
 * cd_off + pre[i].cd + 28 x (slots in front of i from info[0] on), its mz_cuda_zip_dev_entry row to entries[i] (if not NULL). The
 * records are read from dir + (record offset - dir_off): the source itself (dir = src + dir_off) or a saved copy of its tail. */
typedef struct mz_cuda_zip_up_count { /* per slot; pre[i] = the sum over the slots in front of i */
    uint64_t ext;       /* the entry's extent */
    uint64_t cd;        /* its directory record without zip64 fields */
    uint64_t out16;     /* plain bytes rounded up to 16 */
    uint64_t bytes;     /* plain bytes */
    uint64_t stored;    /* stored bytes */
} mz_cuda_zip_up_count;
#define MZ_CUDA_ZIP_UP_INFO 6
typedef struct mz_cuda_zip_up {
    const void *src;                       /* the source archive */
    const void *ent;                       /* its mz_cuda_zip_dev_entry table (K10) */
    uint32_t count, n;
    const uint32_t *keep;
    const void *dir;
    uint64_t dir_off, src_len;
    mz_cuda_zip_up_count *cnt, *pre;       /* n, n + 1 */
    void *part;
    uint64_t *info;                        /* MZ_CUDA_ZIP_UP_INFO words */
    void *archive;
    uint64_t cap, cd_off;
    void *entries;
} mz_cuda_zip_up;
int32_t mz_cuda_zip_up_counts(const mz_cuda_zip_up *u, void *stream);
int32_t mz_cuda_zip_up_copy(const mz_cuda_zip_up *u, void *stream);
int32_t mz_cuda_zip_up_records(const mz_cuda_zip_up *u, void *stream);

/* ---- K6: one long foreign stream, segment-speculative (csrc/inflate_spec_kernel.cuh) ------------------------
 * One ROUND decodes as much of the compressed window d_in[0..in_avail) as can be proven, starting at the block
 * boundary `start_bit` (absolute bit; the serial decoder's state must be at a block header), into
 * d_out[out_pos - out_base ...) up to absolute position out_end. 32 KiB of history before out_pos must be present
 * in d_out (as for K5). The summary says how far the round got; the caller continues from there with another
 * round or with mz_cuda_inflate_streams (which also owns every error / end-of-input decision: a round that
 * meets anything unusual just stops early). d_in must be 4-byte aligned with 16 readable bytes past in_avail. */
typedef struct mz_cuda_spec_summary {
    uint64_t end_bit;    /* absolute bit position reached (a block boundary, or the end of the stream) */
    uint64_t total_out;  /* bytes written from out_pos on */
    uint32_t nchain;     /* segments proven and emitted; 0 = no progress, use the serial decoder */
    int32_t status;      /* 0 running, 1 end of stream */
    uint32_t blocks;
    uint32_t flags;      /* != 0: internal cross-check failed, the round's output must be discarded */
    uint32_t candidates;
    uint32_t pad;
} mz_cuda_spec_summary;
uint64_t mz_cuda_inflate_spec_workspace_bytes(uint32_t max_segments);
int32_t mz_cuda_inflate_spec_round(const void *d_in, uint64_t in_base, uint64_t in_avail, uint32_t in_final, uint64_t start_bit,
                                   uint64_t seg_bytes, uint32_t nseg, void *d_out, uint64_t out_base, uint64_t out_pos,
                                   uint64_t out_end, void *d_workspace, uint32_t max_segments, mz_cuda_spec_summary *d_summary,
                                   void *stream);

#ifdef __cplusplus
}
#endif
#endif
