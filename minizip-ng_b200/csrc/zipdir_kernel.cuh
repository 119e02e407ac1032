/* zipdir_kernel.cuh -- K9: the device half of the zip extractor (include/mz_cuda_batch.h, mz_cuda_zip_*).
 *
 * A round is a run of zip entries whose stored bytes lie in one device buffer, plus a table with one record per entry
 * taken from the central directory. Three launches turn that into the arrays K8, K5, K1 and K7 take, and into one status
 * word per entry:
 *   locate  (one thread per entry): checks the local-header signature, skips the local name and extra field
 *           (mz_zip.c:947-1100 reads the same fields), checks that the data lies inside the entry's extent, and writes the
 *           entry's K5 job, its K1/K7 segment, and for WinZip AES entries its salt, ciphertext offset and length;
 *   stored  (one warp per entry): STORE entries' bytes to the output, from any source alignment;
 *   verify  (one thread per entry): locate result, AES verifier and HMAC, K5 end state and sizes, CRC-32, SHA-256.
 * A status word is 0, or class << 24 | -MZ_code: class 1 = locate, 2 = AES, 3 = stream / CRC / hash. The host reports
 * class 1 first, then class 2 by strength and entry, then class 3 by entry -- the order the reference's reader meets them.
 */
#ifndef MZ_ZIPDIR_KERNEL_CUH
#define MZ_ZIPDIR_KERNEL_CUH

#include "inflate_kernel.cuh"
#include "mzcuda_common.cuh"

namespace mzc {

constexpr uint32_t ZD_AT_DATA = 1u;  /* MZ_CUDA_ZIP_ENT_AT_DATA */
constexpr uint32_t ZD_NO_SHA = 0xffffffffu;
constexpr uint32_t ZD_KEYREC = 80;    /* MZ_CUDA_WZAES_KEYREC */

struct ZipEnt { /* mirror of mz_cuda_zip_ent */
    uint64_t src_off, src_len, csize, usize, out_off;
    uint32_t crc, job, aes_slot, sha_slot;
    uint16_t method;
    uint8_t aes, flags;
    uint32_t pad;
};

struct ZipRound { /* mirror of mz_cuda_zip_round */
    const uint8_t *buf;
    uint64_t buf_len;
    uint8_t *out;
    const ZipEnt *ent;
    uint32_t n, pad;
    InflateJob *jobs;
    const InflateState *states;
    uint64_t *seg_off, *seg_len64, *data_off;
    uint32_t *seg_len;
    const uint32_t *crc;
    const uint8_t *digest, *sha_expect;
    uint8_t *salt;
    uint64_t *coff, *clen;
    const uint8_t *keys, *mac;
    uint32_t *status;
};

__device__ __forceinline__ uint32_t zd_status(uint32_t cls, int32_t code) { return (cls << 24) | (uint32_t)(-code); }
__device__ __forceinline__ uint32_t zd_u16(const uint8_t *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }

__global__ void __launch_bounds__(256) zip_locate_kernel(ZipRound R) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= R.n) return;
    const ZipEnt e = R.ent[i];
    const uint32_t slen = e.aes ? 4u * e.aes + 4u : 0u; /* salt | verifier (2) | ciphertext | authentication code (10) */
    const uint64_t over = e.aes ? slen + 12u : 0u;
    bool ok = e.csize >= over && e.src_off <= R.buf_len && e.src_len <= R.buf_len - e.src_off;
    uint64_t data = e.src_off;
    if (ok && !(e.flags & ZD_AT_DATA)) {
        const uint8_t *h = R.buf + e.src_off;
        ok = e.src_len >= 30 && h[0] == 0x50 && h[1] == 0x4b && h[2] == 0x03 && h[3] == 0x04; /* MZ_ZIP_MAGIC_LOCALHEADER */
        if (ok) data = e.src_off + 30u + zd_u16(h + 26) + zd_u16(h + 28);
    }
    ok = ok && data >= e.src_off && data - e.src_off <= e.src_len && e.csize <= e.src_len - (data - e.src_off);
    const uint64_t stream = ok ? data + (e.aes ? slen + 2u : 0u) : 0u, slen_stream = ok ? e.csize - over : 0u;
    if (e.aes) {
        for (uint32_t k = 0; k < 16; k++) R.salt[(uint64_t)e.aes_slot * 16 + k] = ok && k < slen ? R.buf[data + k] : 0;
        R.coff[e.aes_slot] = stream;
        R.clen[e.aes_slot] = slen_stream;
    }
    if (e.method == 8) {
        InflateJob j;
        j.in = R.buf + stream;
        j.in_base = 0;
        j.in_avail = slen_stream;
        j.out = R.out + e.out_off;
        j.out_base = 0;
        j.out_cap = ok ? e.usize : 0u;
        j.in_final = 1;
        j.flags = 0;
        R.jobs[e.job] = j;
    }
    R.data_off[i] = ok ? stream : ~0ull;
    R.seg_off[i] = e.out_off;
    R.seg_len[i] = (uint32_t)e.usize;
    R.seg_len64[i] = e.usize;
    R.status[i] = ok ? 0u : zd_status(1, -103 /* MZ_FORMAT_ERROR */);
}

/* STORE entries: out[out_off ..) = buf[data_off ..). The destination is 16-byte aligned (the host's layout), the source is not:
 * every 4-byte destination word is two aligned source words joined by a funnel shift; the ragged tail is bytes. Reads stay
 * inside the aligned word after the entry's last byte (the round keeps 32 readable bytes past its end). */
__global__ void __launch_bounds__(256) zip_stored_kernel(ZipRound R) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i = warp; i < R.n; i += nwarps) {
        const ZipEnt &e = R.ent[i];
        const uint64_t src = R.data_off[i];
        if (e.method != 0 || src == ~0ull || e.usize == 0) continue;
        const uint8_t *s = R.buf + src;
        uint8_t *d = R.out + e.out_off;
        const uint32_t *w = (const uint32_t *)((uintptr_t)s & ~(uintptr_t)3);
        const uint32_t sh = (uint32_t)((uintptr_t)s & 3) * 8u;
        const uint64_t words = e.usize >> 2;
        for (uint64_t k = lane; k < words; k += 32) {
            const uint32_t lo = w[k], hi = sh ? w[k + 1] : 0u;
            ((uint32_t *)d)[k] = __funnelshift_r(lo, hi, sh);
        }
        for (uint64_t k = (words << 2) + lane; k < e.usize; k += 32) d[k] = s[k];
    }
}

__global__ void __launch_bounds__(256) zip_verify_kernel(ZipRound R) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= R.n || R.status[i]) return;
    const ZipEnt e = R.ent[i];
    const uint64_t stream = R.data_off[i];
    uint64_t slen_stream = e.csize;
    if (e.aes) {
        const uint8_t *k = R.keys + (uint64_t)e.aes_slot * ZD_KEYREC;
        const uint64_t clen = R.clen[e.aes_slot];
        if (k[64] != R.buf[stream - 2] || k[65] != R.buf[stream - 1]) {
            R.status[i] = zd_status(2, -108); /* MZ_PASSWORD_ERROR, mz_strm_wzaes.c:133-134 */
            return;
        }
        const uint8_t *m = R.mac + (uint64_t)e.aes_slot * 20, *a = R.buf + stream + clen;
        uint32_t diff = 0;
        for (int b = 0; b < 10; b++) diff |= (uint32_t)(m[b] ^ a[b]);
        if (diff) {
            R.status[i] = zd_status(2, -105); /* MZ_CRC_ERROR, :252-254 */
            return;
        }
        slen_stream = clen;
    }
    if (e.method == 8) {
        const InflateState &s = R.states[e.job];
        if (s.status != 1 || s.out_pos != e.usize || ((s.in_bitpos + 7) >> 3) != slen_stream) {
            R.status[i] = zd_status(3, s.status < 0 ? s.status : -3 /* MZ_DATA_ERROR */);
            return;
        }
    }
    const uint32_t crc = e.usize ? R.crc[i] : 0u;
    if (crc != e.crc) {
        R.status[i] = zd_status(3, -105);
        return;
    }
    if (e.sha_slot != ZD_NO_SHA) {
        const uint8_t *g = R.digest + (uint64_t)i * 32, *x = R.sha_expect + (uint64_t)e.sha_slot * 32;
        uint32_t diff = 0;
        for (int b = 0; b < 32; b++) diff |= (uint32_t)(g[b] ^ x[b]);
        if (diff) R.status[i] = zd_status(3, -105); /* hash mismatch -> MZ_CRC_ERROR (mz_zip_rw.c:444-447) */
    }
}

} // namespace mzc
#endif
