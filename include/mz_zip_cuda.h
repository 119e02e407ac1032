/* mz_zip_cuda.h -- batch zip-entry writer on the reference's RAW-entry seam (SURVEY.md 8f.1, config C4).
 *
 * The reference compresses a zip entry by pushing its bytes through mz_stream_zlib, one entry at a time
 * (mz_zip_entry_write_open -> mz_zip_entry_write -> mz_zip_entry_close, mz_zip.c:1915,2056,2269). This routine keeps
 * the container code exactly where it is and only moves the codec work: all entries of a batch are DEFLATE-compressed
 * and CRC'd on the GPU in ONE launch each (every entry its own raw stream: 64 KiB chunks joined by sync markers,
 * BFINAL on the entry's last chunk), then handed to the reference through its raw seam
 *     mz_zip_entry_write_open(handle, &file_info, level, raw = 1, NULL)     mz_zip.c:1915
 *     mz_zip_entry_write(handle, compressed, size)                          mz_zip.c:2056
 *     mz_zip_entry_close_raw(handle, uncompressed_size, crc32)              mz_zip.c:2272
 * so local headers, zip64 decisions and the central directory stay the reference's own code.
 *
 * Linking: the three functions above (plus nothing else) are taken from the HOST program, which links the
 * reference's mz_zip.c. They are declared weak here, so libmz_strm_cuda.so still loads in a process that has no
 * zip container (the call then returns MZ_SUPPORT_ERROR).
 */
#ifndef MZ_ZIP_CUDA_H
#define MZ_ZIP_CUDA_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct mz_cuda_zip_item {
    const char *filename;    /* utf-8, null terminated (stored with MZ_ZIP_FLAG_UTF8) */
    const void *data;        /* host memory, `size` bytes (may be NULL when size == 0) */
    int64_t size;
    int64_t modified_date;   /* unix time; 0 = now */
    uint32_t external_fa;    /* 0 = regular file 0644 */
    uint32_t reserved;
} mz_cuda_zip_item;

typedef struct mz_cuda_zip_stats {
    uint64_t bytes_in, bytes_out;
    uint32_t entries, rounds;
    double pack_ms, gpu_ms, container_ms; /* host packing + upload, device work + download, reference container calls */
    double setup_ms;                      /* native writer: creating and releasing the page-locked / device staging of the call */
} mz_cuda_zip_stats;

/* Append `count` entries to the zip that `zip_handle` (an open mz_zip writer, mz_zip.c:1237 mz_zip_open) is writing.
 * level: 0..9 or -1 (= 6), as mz_zip_entry_write_open takes it. Returns MZ_OK or the first error (MZ_* codes).
 * stats may be NULL. */
int32_t mz_zip_cuda_add_buffers(void *zip_handle, const mz_cuda_zip_item *items, uint32_t count, int16_t level,
                                mz_cuda_zip_stats *stats);

/* Same, with options. MZ_ZIP_CUDA_HASH_SHA256: every entry also gets the SHA-256 of its plain bytes, computed on the GPU in
 * the same round (K7) and stored in the MZ_ZIP_EXTENSION_HASH extra field (id 0x1a51: algorithm 23, digest size 32, digest)
 * exactly as the reference's zip writer stores it when built with a crypto provider (mz_zip_rw.c:1339-1420); the reference's
 * reader then verifies it on extraction (mz_zip_rw.c:410-450), and so does mz_zip_cuda_extract_all. */
#define MZ_ZIP_CUDA_HASH_SHA256 1u
int32_t mz_zip_cuda_add_buffers_ex(void *zip_handle, const mz_cuda_zip_item *items, uint32_t count, int16_t level, uint32_t flags,
                                   mz_cuda_zip_stats *stats);

/* ---- a whole archive, natively (scope row f1, "if the container is the limit") ------------------------------------------
 * With 100 000 small entries the reference's per-entry container calls (mz_zip_entry_write_open / _write / _close_raw: three
 * calls and ~28 us per entry) cost ten times the GPU work. This call writes the COMPLETE archive itself to `base_stream` (any
 * mz_stream object: file, buffered, memory): local headers (mz_zip.c:594-919 layout: no data descriptor -- sizes and CRC are
 * known before a byte is written --, UTF-8 flag, version 20, or 45 with a zip64 extra field), the entries' DEFLATE streams,
 * the central directory and the end records incl. the zip64 end record + locator when there are >= 65535 entries or the
 * directory starts beyond 4 GiB (mz_zip.c:1102-1234, zip64 rules :551-592). A round's region [header | stream | header | ...]
 * is assembled ON THE DEVICE (K4 gather with explicit destinations + a header scatter) and goes to base in one write.
 * MZ_ZIP_CUDA_ALL_DEVICES: rounds are prepared round-robin on every visible GPU (entries shard across the GPUs; the archive
 * itself is one serial byte stream written in order). Entries must be smaller than 4 GiB - 64 KiB. */
#define MZ_ZIP_CUDA_ALL_DEVICES 2u
int32_t mz_zip_cuda_write_archive(void *base_stream, const mz_cuda_zip_item *items, uint32_t count, int16_t level, uint32_t flags,
                                  mz_cuda_zip_stats *stats);
/* The native writer keeps the staging of finished calls (page-locked + device buffers, up to eight round slots per process) for
 * the next call; this frees them. MZ_CUDA_ZIP_POOL=0 in the environment turns the pool off. */
void mz_zip_cuda_trim(void);

/* The same archive with every entry WinZip-AES encrypted after compression (scope row f4, the part that follows the codec): what
 * the reference does per entry by stacking mz_stream_wzaes under the codec (mz_zip.c:1734-1741, mz_strm_wzaes.c) -- a random salt,
 * PBKDF2-HMAC-SHA1 (1000 iterations) of the password, AES in counter mode over the compressed stream, HMAC-SHA1 of the ciphertext
 * -- done for all entries of a round by three kernels (K8, include/mz_cuda_batch.h). Entry layout and headers as the reference
 * writes them: method 99 + the 0x9901 extra field (AE-1, strength, real method 8), flag bit 0, version needed 51, stored size =
 * salt + 2-byte verifier + ciphertext + 10-byte authentication code, CRC kept (mz_zip.c:703-733, :870-885).
 * flags must contain MZ_ZIP_CUDA_AES; aes_strength = 1 / 2 / 3 (AES-128 / 192 / 256; 0 = 3, the reference's default);
 * password up to 128 bytes. */
#define MZ_ZIP_CUDA_AES 4u
int32_t mz_zip_cuda_write_archive_aes(void *base_stream, const mz_cuda_zip_item *items, uint32_t count, int16_t level, uint32_t flags,
                                      const char *password, uint8_t aes_strength, mz_cuda_zip_stats *stats);

/* ---- batch extraction (scope row f2): the reverse direction ---------------------------------------------------
 * The reference extracts entry by entry: mz_zip_entry_read_open(raw=0) creates a mz_stream_zlib, the caller's loop
 * reads through it, mz_zip_entry_close compares the CRC (mz_zip_rw.c:818-909, mz_zip.c:2116-2128). Here the central
 * directory is still walked by the reference's own reader (mz_zip_goto_first_entry / _next_entry /
 * mz_zip_entry_get_info, mz_zip.c:2320-2400) and the compressed bytes are fetched through the raw seam
 * (mz_zip_entry_read_open(raw=1) / mz_zip_entry_read, mz_zip.c:1874,2031), but all entries of a round are inflated by
 * ONE K5 launch and checksummed by ONE K1 launch; the CRCs are compared with the headers on the host (MZ_CRC_ERROR on
 * the first mismatch, MZ_DATA_ERROR if a stream does not decode to exactly its recorded size). An entry that carries a
 * SHA-256 in a MZ_ZIP_EXTENSION_HASH extra field has that verified too (K7 over the round's plain bytes; MZ_CRC_ERROR on a
 * mismatch, as mz_zip_reader_entry_close reports it, mz_zip_rw.c:430-450).
 * `cb` is called once per entry in archive order with the plain bytes (valid during the call only); a non-zero return
 * stops the extraction and is returned. Entries that are encrypted, use another method than STORE/DEFLATE, or exceed
 * 1 GiB are not batched: the call returns MZ_SUPPORT_ERROR (use the per-entry stream path for such archives). */
typedef int32_t (*mz_cuda_zip_entry_cb)(void *userdata, const char *filename, const void *data, int64_t size, uint32_t crc32);
int32_t mz_zip_cuda_extract_all(void *zip_handle, mz_cuda_zip_entry_cb cb, void *userdata, mz_cuda_zip_stats *stats);

/* The same for archives whose entries are WinZip-AES encrypted (any strength; written by this library, by the reference or by
 * WinZip): the stored bytes still come through the raw seam (mz_zip_entry_read_open(raw = 1, password = NULL) hands out the
 * encrypted bytes, mz_zip.c:1727-1731), K8 derives every entry's keys from password + salt, the 2-byte verifier is compared
 * (MZ_PASSWORD_ERROR, mz_strm_wzaes.c:133-134), the HMAC-SHA1 of the ciphertext is compared with the stored authentication code
 * (MZ_CRC_ERROR, :252-254), the ciphertext is decrypted in place and decoded like any other entry. The HOST program's container
 * must be built with HAVE_WZAES (otherwise its reader refuses such entries before this code sees them). PKWARE-encrypted entries
 * return MZ_SUPPORT_ERROR; encrypted entries without a password MZ_PASSWORD_ERROR. */
int32_t mz_zip_cuda_extract_all_aes(void *zip_handle, const char *password, mz_cuda_zip_entry_cb cb, void *userdata, mz_cuda_zip_stats *stats);

/* ---- a whole archive, natively (scope row f2) ---------------------------------------------------------------------------
 * Extracts every entry of the archive readable from base_stream (any mz_stream: file, buffered, memory, mem64). The call needs no
 * mz_zip handle and no zip container in the process: it reads the end records (incl. zip64) and the whole central directory
 * itself, corrects for prepended data as the reference does (self-extracting archives), and reads each round's stored bytes with
 * one base read per run of adjacent entries. The device checks every local header (K9), decrypts (K8), inflates (K5), copies
 * STORE entries, and verifies CRC-32, SHA-256 (MZ_ZIP_EXTENSION_HASH) and the AES verifier and HMAC. Up to four rounds are in
 * flight, each on its own thread and CUDA stream; MZ_ZIP_CUDA_ALL_DEVICES sends them round-robin to every visible GPU.
 * `cb` as for mz_zip_cuda_extract_all: once per entry in central-directory order, on the caller's thread; a round is delivered
 * only when all its entries verified. Entries handled and errors: those of mz_zip_cuda_extract_all_aes (password may be NULL when
 * no entry is encrypted); MZ_FORMAT_ERROR for a missing or inconsistent end record, directory or local header; MZ_SUPPORT_ERROR
 * also for split archives. Errors of the archive as a whole (end records, directory location) are returned before anything is
 * delivered. Otherwise the first failing entry in directory order decides, as in the reference's reader: an entry the call refuses
 * (unsupported, no password, malformed record) ends the list, the entries in front of it are delivered, then its error is
 * returned; a decoding, CRC, hash, AES or local-header error in a round returns that round's first failing entry, and nothing of
 * that round is delivered; a base read error returns after the rounds read before it. Staging is pooled with the writer's
 * (MZ_CUDA_ZIP_POOL, mz_zip_cuda_trim); MZ_CUDA_ZIP_ROUND_MB sets the stored bytes per round (default 32; plain bytes up to four
 * times that). An entry larger than a round gets a round of its own size; the call then keeps one round slot per device instead of
 * four and does not pool it (an entry of 1 GiB needs about 1 GiB of page-locked input and output staging).
 * stats: pack_ms = directory parse and base reads (caller's thread), gpu_ms = upload to download summed over rounds,
 * container_ms = time in the callback, setup_ms = staging set-up and release; bytes_in / bytes_out = stored / plain bytes. */
int32_t mz_zip_cuda_extract_archive(void *base_stream, const char *password, uint32_t flags, mz_cuda_zip_entry_cb cb, void *userdata,
                                    mz_cuda_zip_stats *stats);

/* ---- an archive in device memory, extracted into device memory ------------------------------------------------------
 * The same extraction as mz_zip_cuda_extract_archive for an archive that already lies in device memory (d_archive, len bytes,
 * current device; no padding needed): the central directory is parsed on the device (K10), every accepted entry is decoded and
 * verified there (K9, K8, K5, K1, K7), and the plain bytes stay in device memory. Only a few scalars cross PCIe. Synchronous: the
 * work is enqueued on `stream` and the call synchronises on it before it returns. The archive is not modified (WinZip AES entries
 * are decrypted in a copy of the bytes in front of the directory).
 * Results and errors are those of mz_zip_cuda_extract_archive on the same bytes:
 *   - an error of the archive as a whole (end records, zip64 records, directory location, split archive) is returned first, with
 *     *count = 0 and nothing decoded;
 *   - *count = the directory records accepted; a refused record ends the list, the entries in front of it are decoded, then its
 *     error is returned; *out_bytes = the plain bytes of the accepted entries, each rounded up to 16;
 *   - d_out == NULL: list only: the table and *out_bytes are filled, nothing is decoded;
 *   - max_entries < *count, or d_out and out_cap < *out_bytes: MZ_BUF_ERROR with *count and *out_bytes set, nothing decoded or
 *     listed (call again with buffers that large; d_entries may be NULL with max_entries 0 for the first call). A truncated
 *     stream is also MZ_BUF_ERROR, as an entry's error: the caps then cover *count and *out_bytes;
 *   - otherwise every accepted entry is decoded and verified: local header, AES verifier and HMAC, DEFLATE end state and sizes,
 *     CRC-32, SHA-256. The first failing entry in directory order decides the return value; each entry's status is in the table.
 * A central directory of 16 GiB or more returns MZ_SUPPORT_ERROR (the device parse counts candidate records in 32 bits).
 * d_entries: device table, one row per accepted record in directory order. d_out: 16-byte aligned. stats (may be NULL):
 * entries / bytes_in / bytes_out of the accepted entries, pack_ms = the directory parse, gpu_ms = decode and verify, setup_ms =
 * scratch allocation; rounds = 1 when something was decoded. */
typedef struct mz_cuda_zip_dev_entry {
    uint64_t local_off; /* local header in the archive, after the prepended-data shift */
    uint64_t csize, usize;
    uint64_t out_off;   /* plain bytes at d_out + out_off: 16-byte aligned, packed in directory order */
    uint64_t name_off;  /* name bytes at d_archive + name_off (inside the central directory), name_len of them, not terminated */
    uint64_t extent;    /* bytes from local_off up to the next local header or the directory (capped) */
    uint64_t sha_off;   /* has_sha: the expected SHA-256 at d_archive + sha_off */
    uint32_t crc, name_len;
    uint16_t method;    /* 0 or 8 (an AES entry's real method) */
    uint8_t aes;        /* 0 or WinZip AES strength 1..3 */
    uint8_t has_sha;
    int32_t status;     /* after decoding: MZ_OK or this entry's error */
} mz_cuda_zip_dev_entry; /* 72 bytes */
int32_t mz_zip_cuda_extract_device(const void *d_archive, uint64_t len, const char *password, mz_cuda_zip_dev_entry *d_entries, uint32_t max_entries,
                                   uint32_t *count, void *d_out, uint64_t out_cap, uint64_t *out_bytes, mz_cuda_zip_stats *stats, void *stream);

/* ---- random access to an archive in device memory ----------------------------------------------------------------------
 * A reader parses the directory of an archive in device memory once and then looks entries up by name and decodes any chosen
 * subset of them, many times: what mz_zip_locate_entry (mz_zip.c:2414) and mz_zip_entry_read_* do entry by entry in the
 * reference, for batches of entries on the device (K10 at open, K12 for the name index and the selections, K9 / K8 / K5 / K1 / K7
 * for the decode, csrc/zipsel_kernel.cuh).
 *
 * open: parses the directory (K10, once) and builds the name index. An error of the archive as a whole is returned exactly as
 *   mz_zip_cuda_extract_device returns it, and no reader is created. Otherwise MZ_OK with *count = the records accepted and
 *   *refuse = the error that ended the list or MZ_OK (what extract_device returns after listing). The password (may be NULL) is
 *   copied. The archive must stay allocated and unchanged while the reader is open; the reader never writes it. A reader belongs
 *   to the device current at open and serves one call at a time; readers are independent of each other. stats (may be NULL):
 *   entries / bytes_in / bytes_out of the accepted entries, pack_ms = the directory parse, gpu_ms = the index build, setup_ms =
 *   the index allocation.
 * entries: the device table of the *count accepted records, row for row what extract_device lists (out_off included, status 0).
 * locate: enqueued on `stream`, no host synchronisation (its output can feed decode directly). Query q is the d_name_len[q] bytes
 *   at d_names + d_name_off[q], all in device memory. d_index[q] = the first accepted entry in directory order whose name compares
 *   equal to the query under mz_zip_path_compare(name, query, ignore_case) (mz_zip.c:2754): both taken as C strings (the bytes
 *   before the first NUL), '\\' equal to '/', with ignore_case only A-Z folded (tolower in the C locale; bytes >= 0x80 compare
 *   exactly). No match, or an empty query: 0xffffffff. Unlike the reference, whose walk continues past the records this library
 *   refuses, a name behind the record that ended the list is not found. Cost: a hash-table probe per query plus one compare per
 *   entry whose folded name hashes the same (all duplicates of a name).
 * decode: synchronous on `stream`. Slot i decodes entry d_select[i]; any selection is valid (repeats, any order, nsel = 0). The
 *   plain bytes are packed in selection order, each at a 16-byte aligned offset; d_out_off (optional, nsel + 1 values) receives
 *   the offsets and the total, *out_bytes the total.
 *   - MZ_PARAM_ERROR first: a NULL reader or out_bytes, d_select NULL with nsel > 0, d_out not 16-byte aligned;
 *   - d_out == NULL: sizing call: *out_bytes and d_out_off are set, nothing is decoded;
 *   - out_cap < *out_bytes: MZ_BUF_ERROR with *out_bytes set; nothing is written to d_out, d_out_off or d_status;
 *   - otherwise every slot is decoded and verified exactly as extract_device does it (local header, AES verifier and HMAC, DEFLATE
 *     end state and sizes, CRC-32, SHA-256): its bytes and status equal those extract_device gives that entry. An index >= count
 *     gets MZ_END_OF_LIST (what mz_zip_locate_entry returns for a missing name, so a miss from locate passes straight through)
 *     and no bytes. d_status (optional, nsel values) receives every slot's status; the return value is the status of the first
 *     failing slot in selection order, or MZ_OK.
 *   WinZip AES entries are decrypted in place by K8, so a selection that holds any is first gathered (every slot's extent) into
 *   scratch the reader owns; the same entry selected twice is decrypted once per slot. The reader keeps its scratch between calls
 *   and grows it only when a selection needs more. Host synchronisation: one readback of the selection's totals before the decode
 *   launches and one of the first failing slot after it. stats (may be NULL): entries / bytes_in / bytes_out of the valid slots,
 *   pack_ms = to the first readback, gpu_ms = decode and verify, setup_ms = scratch allocation (0 when the scratch fitted).
 * close: frees everything the reader allocated (NULL is a no-op).
 * Entries above 1 GiB are refused at open as extract_device refuses them. */
typedef struct mz_zip_cuda_dev_reader mz_zip_cuda_dev_reader;
int32_t mz_zip_cuda_reader_open(const void *d_archive, uint64_t len, const char *password, mz_zip_cuda_dev_reader **reader, uint32_t *count,
                                int32_t *refuse, mz_cuda_zip_stats *stats, void *stream);
const mz_cuda_zip_dev_entry *mz_zip_cuda_reader_entries(const mz_zip_cuda_dev_reader *reader);
int32_t mz_zip_cuda_reader_locate(mz_zip_cuda_dev_reader *reader, const void *d_names, const uint64_t *d_name_off, const uint32_t *d_name_len,
                                  uint32_t n, uint8_t ignore_case, uint32_t *d_index, void *stream);
int32_t mz_zip_cuda_reader_decode(mz_zip_cuda_dev_reader *reader, const uint32_t *d_select, uint32_t nsel, void *d_out, uint64_t out_cap,
                                  uint64_t *out_bytes, uint64_t *d_out_off, int32_t *d_status, mz_cuda_zip_stats *stats, void *stream);
void mz_zip_cuda_reader_close(mz_zip_cuda_dev_reader *reader);

/* ---- an archive written into device memory from entries in device memory ---------------------------------------------
 * The archive mz_zip_cuda_write_archive (flags with MZ_ZIP_CUDA_AES: mz_zip_cuda_write_archive_aes) writes for the same entries,
 * level, flags and dates, byte for byte (with AES only the random salts and what follows from them differ), built in device memory
 * from entries in device memory: d_items[count] (device), each naming its plain bytes at d_data + data_off and its name at d_names +
 * name_off. Validation, layout, local headers, CRC-32, the central directory and the end records are done on the device (K11 with
 * K2+K3, K1, K4, K7, K8); only scalars cross PCIe, and with AES the per-entry salts (from getrandom). Synchronous on `stream`.
 *   - flags: MZ_ZIP_CUDA_HASH_SHA256 and MZ_ZIP_CUDA_AES only (MZ_ZIP_CUDA_ALL_DEVICES: MZ_PARAM_ERROR); level 0..9 or -1 (= 6);
 *     password and aes_strength as for mz_zip_cuda_write_archive_aes, password ignored without MZ_ZIP_CUDA_AES.
 *   - errors: argument errors first, in the host writer's order; then the first invalid item in index order: MZ_PARAM_ERROR for its
 *     name (length 0 or above 65535, a NUL byte) or pointers (d_names NULL, d_data NULL with size > 0), MZ_SUPPORT_ERROR for a size
 *     of 0xffff0000 or more. Nothing is compressed or written then.
 *   - an entry just below 4 GiB whose stored size (compressed stream, with AES plus salt, verifier and authentication code) reaches
 *     0xffffffff cannot be described by its local header: MZ_INTERNAL_ERROR after compression, as mz_zip_cuda_write_archive returns.
 *   - d_archive == NULL: sizing call, MZ_OK with *archive_len = an upper bound of the archive's length; nothing is compressed.
 *   - cap smaller than the archive: MZ_BUF_ERROR with *archive_len = the exact length; bytes below cap may have been written.
 *     No byte at or beyond cap is ever written. On success *archive_len = the exact length.
 *   - d_data, d_names and d_items are only read; AES encrypts inside d_archive.
 *   - d_entries (optional, device): one mz_cuda_zip_dev_entry per item, the row mz_zip_cuda_extract_device lists for the archive.
 *   - chunks are compressed in rounds of MZ_CUDA_ZIP_ROUND_MB MiB of plain bytes (default 1024), so scratch is bounded; every call
 *     allocates its own.
 *   - stats: entries, bytes_in, bytes_out as the host writer counts them, rounds, pack_ms = validation and planning, gpu_ms =
 *     compression to the last kernel, setup_ms = scratch allocation. */
typedef struct mz_cuda_zip_dev_item {
    uint64_t data_off;    /* the entry's plain bytes at d_data + data_off (any alignment; items may share bytes) */
    uint64_t size;        /* below 0xffff0000, as mz_zip_cuda_write_archive */
    uint64_t name_off;    /* name at d_names + name_off: name_len bytes, no terminator */
    uint32_t name_len;    /* 1..65535, no NUL byte inside */
    uint32_t dos_date;    /* MS-DOS date/time exactly as the headers store it; 0 = the time of the call */
    uint32_t external_fa; /* 0 = regular file 0644, as mz_cuda_zip_item */
    uint32_t reserved;    /* 0 */
} mz_cuda_zip_dev_item;   /* 40 bytes */
int32_t mz_zip_cuda_write_device(const void *d_data, const void *d_names, const mz_cuda_zip_dev_item *d_items, uint32_t count, int16_t level, uint32_t flags,
                                 const char *password, uint8_t aes_strength, void *d_archive, uint64_t cap, uint64_t *archive_len,
                                 mz_cuda_zip_dev_entry *d_entries, mz_cuda_zip_stats *stats, void *stream);

/* ---- an archive in device memory updated on the device ----------------------------------------------------------------
 * Keeps, drops and appends entries of an archive in device memory without recompressing the kept ones: what the reference's append
 * mode (mz_zip_open with MZ_OPEN_MODE_APPEND, mz_zip.c:1445) and `minizip -e` (raw copies through mz_zip_writer_copy_from_reader,
 * mz_zip_rw.c:1731) do on the host, on the device (K10 parses the source, K13 moves the kept entries and rewrites their records,
 * K11 writes the new entries, csrc/zipup_kernel.cuh). Synchronous on `stream`.
 *   - output: (1) the kept entries of d_src[0, src_len), in keep order, each its raw extent (local header, stored bytes, any data
 *     descriptor: unchanged); (2) the count new entries, exactly as write_device lays them out; (3) the directory: the kept records,
 *     then the new ones; (4) a zip64 end record and locator when the directory starts at 0xffffffff or later or there are 65535
 *     entries or more (write_device's rule); (5) the end record with the source's archive comment. Data in front of the source's
 *     first entry (a self-extracting stub) is not carried over.
 *   - d_keep NULL (nkeep 0): every accepted entry, in directory order (append). Otherwise nkeep indices into the source's accepted
 *     entries (the rows extract_device and the reader list), any order, repeats allowed.
 *   - errors, in this order, and nothing is written when one of them is returned: (1) write_device's argument errors, then d_src NULL
 *     with src_len > 0, d_keep NULL with nkeep > 0, and overlapping buffers other than in place (below): MZ_PARAM_ERROR; (2) an error
 *     of the source as a whole, exactly as extract_device returns it (the parse runs as if a password had been given: nothing is
 *     decrypted); (3) a refused record (PKWARE encryption, another method, an entry above 1 GiB...): its code, not a shorter list;
 *     (4) a keep index >= the accepted count: MZ_PARAM_ERROR; in place, entries that do not tile [0, directory): MZ_PARAM_ERROR;
 *     a kept record that needs the zip64 field but whose extra field would pass 65535 bytes: MZ_SUPPORT_ERROR; (5) item errors, as
 *     write_device reports them.
 *   - kept WinZip AES entries are copied still encrypted: no password is needed for them. password and aes_strength apply to the
 *     new entries with MZ_ZIP_CUDA_AES only; flags as write_device (MZ_ZIP_CUDA_HASH_SHA256 allowed, MZ_ZIP_CUDA_ALL_DEVICES:
 *     MZ_PARAM_ERROR).
 *   - kept records: fixed fields, name, file comment and every extra field but zip64 (0x0001) unchanged and in order; the local-header
 *     offset becomes the entry's new one; the source's zip64 fields are dropped; when the new offset is 0xffffffff or more, sizes and
 *     offset are saturated and a 28-byte zip64 field follows the name, as write_device writes it. Version needed becomes at least
 *     45 with a zip64 field, and goes back to 20 for a non-AES record at 45 that loses its zip64 field. The disk number is written
 *     as 0. So a record write_device wrote comes out as write_device would write it at its new offset.
 *   - d_archive == NULL: sizing call, *archive_len = an upper bound. cap too small: MZ_BUF_ERROR with *archive_len = the exact length
 *     (bytes below cap may have been written). No byte at or beyond cap is ever written. d_entries (optional, device): the
 *     nkeep + count rows extract_device lists for the output.
 *   - in place: d_archive == d_src only with d_keep NULL and entries that tile [0, directory) exactly (no prepended data, no gaps).
 *     The kept bytes are not moved and writing starts at the old directory, as the reference's append does. The bytes from the
 *     source's directory to src_len are saved first; on any later error (MZ_BUF_ERROR, MZ_INTERNAL_ERROR, ...) they are put back, so
 *     a failed call leaves the source a valid archive.
 *   - stats: as write_device, entries / bytes_* over the whole output; pack_ms = the parse and planning. */
int32_t mz_zip_cuda_update_device(const void *d_src, uint64_t src_len, const uint32_t *d_keep, uint32_t nkeep, const void *d_data, const void *d_names,
                                  const mz_cuda_zip_dev_item *d_items, uint32_t count, int16_t level, uint32_t flags, const char *password,
                                  uint8_t aes_strength, void *d_archive, uint64_t cap, uint64_t *archive_len, mz_cuda_zip_dev_entry *d_entries,
                                  mz_cuda_zip_stats *stats, void *stream);

/* sizeof the mz_zip_file mirror this library was built with: the host asserts it equals sizeof(mz_zip_file) */
uint32_t mz_zip_cuda_abi_file_info_size(void);

#ifdef __cplusplus
}
#endif
#endif
