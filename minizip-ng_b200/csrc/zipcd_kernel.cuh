/* zipcd_kernel.cuh -- K10: the central directory of an archive in device memory, parsed on the device
 * (mz_zip_cuda_extract_device, include/mz_zip_cuda.h; launches: mz_cuda_zip_parse_directory in mz_cuda_api.cu).
 *
 * The host parse (zn_read_directory in mz_zip_cuda.c) walks the directory record by record. Here every step is parallel:
 *   end      one CTA: the last end-record signature in the tail (max-reduction over positions), then one thread applies the
 *            end-record, zip64 and prepended-data rules of the host parse and writes cd_off, cd_size, count, shift or an error;
 *   cand     one thread per directory byte: is a record with its bounds inside the directory at this position? A bitmap with a
 *            per-word prefix makes rank(p) one load and one popc;
 *   link     per candidate: its position and the rank of the candidate its lengths point to (or END / BREAK);
 *   double   forward pointer doubling from the first record: in round k every marked candidate marks its 2^k-th successor and
 *            the jump table is squared. What is reachable from position 0 is the true chain; a signature inside a name, extra
 *            field or comment is never reached. The chain is strictly increasing, so a record's index is its marked rank;
 *   place    the chain's positions in directory order, and how the chain ends;
 *   records  one thread per record: fixed fields, extra fields (zip64, WinZip AES, hash) and the refusal rules;
 *   finish   the first refused record, totals, whether local-header offsets are sorted, the largest AES ciphertext per strength;
 *   fill     extents (next higher local-header offset by binary search in the sorted offsets), the public table, the K9 table
 *            (zipdir_kernel.cuh) and the compact array of expected digests.
 * Scans are three launches (per-tile sums, one CTA over the sums, per-tile apply) and the sort of unsorted offsets is a bitonic
 * network, one launch per stage: no CTA ever waits on another, so the kernels also run on the CPU emulator.
 *
 * Reads stay inside [0, len): the tail scan reads 4 bytes at positions <= len - 22; the zip64 records are read only where the
 * host parse reads them (bounds checked against the end record's position); a directory position is read only when a whole
 * 46-byte record fits between it and cd_off + cd_size <= eocd_pos < len; extra fields are read inside their record.
 */
#ifndef MZ_ZIPCD_KERNEL_CUH
#define MZ_ZIPCD_KERNEL_CUH

#include "mzcuda_common.cuh"
#include "zipdir_kernel.cuh"

namespace mzc {

constexpr uint32_t ZC_THREADS = 256;
constexpr uint32_t ZC_ITEMS = 8; /* scan: elements per thread */
constexpr uint32_t ZC_TILE = ZC_THREADS * ZC_ITEMS;
constexpr uint32_t ZC_END = 0xffffffffu; /* successor: the record ends exactly at the end of the directory */
constexpr uint32_t ZC_BRK = 0xfffffffeu; /* successor: no valid record where the lengths point */
constexpr uint64_t ZC_TAIL = 65535u + 22u;

struct ZipDevEnt { /* mirror of mz_cuda_zip_dev_entry */
    uint64_t local_off, csize, usize, out_off, name_off, extent, sha_off;
    uint32_t crc, name_len;
    uint16_t method;
    uint8_t aes, has_sha;
    int32_t status;
};

struct ZcSummary { /* device side of the parse; the host reads it back between stages */
    int32_t err;        /* end records: MZ_OK or the archive's error */
    uint32_t unsorted;  /* finish: local-header offsets of the accepted records are not non-decreasing */
    uint64_t cd_off, cd_size, count, shift, eocd_pos;
    uint32_t nchain, term;           /* place: records reachable from position 0, successor of the last one */
    uint32_t refuse_idx, pad;        /* records: first record refused by its own fields */
    uint32_t nacc;                   /* finish: records accepted */
    int32_t refuse;                  /* finish: the error that ended the list, or MZ_OK */
    uint64_t out, cin, cout;         /* finish: totals of the accepted records */
    uint32_t job, sha, a[4];
    uint64_t max_clen[4];
};

struct ZcCount { /* per record, scanned: 16-byte output slots, stored and plain bytes, K5 jobs, digests, AES rows per strength */
    uint64_t out, cin, cout;
    uint32_t job, sha, a[4];
    __device__ __forceinline__ ZcCount operator+(const ZcCount &o) const {
        ZcCount r;
        r.out = out + o.out;
        r.cin = cin + o.cin;
        r.cout = cout + o.cout;
        r.job = job + o.job;
        r.sha = sha + o.sha;
        for (int k = 0; k < 4; k++) r.a[k] = a[k] + o.a[k];
        return r;
    }
};

struct ZcRec { /* per record, from the directory */
    uint64_t off, csize, usize, name_off, sha_off;
    uint32_t crc, name_len;
    uint16_t method;
    uint8_t aes, has_sha;
    int32_t code; /* MZ_OK, or why this record is refused */
};

__device__ __forceinline__ uint32_t zc_u16(const uint8_t *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }
__device__ __forceinline__ uint32_t zc_u32(const uint8_t *p) { return zc_u16(p) | (zc_u16(p + 2) << 16); }
__device__ __forceinline__ uint64_t zc_u64(const uint8_t *p) { return (uint64_t)zc_u32(p) | ((uint64_t)zc_u32(p + 4) << 32); }

/* ---- scans: out[i] = in[0] + ... + in[i-1] for i <= n (out has n + 1 entries) --------------------------------------- */
template <typename T> __device__ __forceinline__ T zc_zero() {
    T z;
    memset(&z, 0, sizeof(z));
    return z;
}

/* exclusive scan of v over the CTA; *total gets the CTA's sum */
template <typename T> __device__ __forceinline__ T zc_block_scan(T v, T *s, T *total) {
    const uint32_t t = threadIdx.x;
    s[t] = v;
    __syncthreads();
    for (uint32_t off = 1; off < ZC_THREADS; off <<= 1) {
        const T x = t >= off ? s[t - off] : zc_zero<T>();
        __syncthreads();
        if (t >= off) s[t] = s[t] + x;
        __syncthreads();
    }
    const T ex = t ? s[t - 1] : zc_zero<T>();
    *total = s[ZC_THREADS - 1];
    __syncthreads();
    return ex;
}

template <typename T> __global__ void __launch_bounds__(ZC_THREADS) zc_scan_reduce_kernel(const T *in, uint64_t n, T *part) {
    __shared__ T s[ZC_THREADS];
    const uint64_t b0 = (uint64_t)blockIdx.x * ZC_TILE + (uint64_t)threadIdx.x * ZC_ITEMS;
    T v = zc_zero<T>();
    for (uint32_t k = 0; k < ZC_ITEMS; k++)
        if (b0 + k < n) v = v + in[b0 + k];
    T tot;
    zc_block_scan(v, s, &tot);
    if (threadIdx.x == 0) part[blockIdx.x] = tot;
}

/* one CTA: the tiles' sums become their exclusive prefix */
template <typename T> __global__ void __launch_bounds__(ZC_THREADS) zc_scan_parts_kernel(T *part, uint32_t nb) {
    __shared__ T s[ZC_THREADS];
    const uint32_t per = (nb + ZC_THREADS - 1) / ZC_THREADS, b0 = threadIdx.x * per;
    T v = zc_zero<T>();
    for (uint32_t k = 0; k < per; k++)
        if (b0 + k < nb) v = v + part[b0 + k];
    T tot;
    T run = zc_block_scan(v, s, &tot);
    for (uint32_t k = 0; k < per; k++)
        if (b0 + k < nb) {
            const T x = part[b0 + k];
            part[b0 + k] = run;
            run = run + x;
        }
}

template <typename T> __global__ void __launch_bounds__(ZC_THREADS) zc_scan_apply_kernel(const T *in, uint64_t n, const T *part, T *out) {
    __shared__ T s[ZC_THREADS];
    const uint64_t b0 = (uint64_t)blockIdx.x * ZC_TILE + (uint64_t)threadIdx.x * ZC_ITEMS;
    T v = zc_zero<T>();
    for (uint32_t k = 0; k < ZC_ITEMS; k++)
        if (b0 + k < n) v = v + in[b0 + k];
    T tot;
    T run = part[blockIdx.x] + zc_block_scan(v, s, &tot);
    for (uint32_t k = 0; k < ZC_ITEMS; k++) {
        if (b0 + k > n) break;
        out[b0 + k] = run;
        if (b0 + k < n) run = run + in[b0 + k];
    }
}

/* ---- round placement (K11 and K14 place): the round's chunks [c0, c0 + m) of a stream cut into chunks --------------------- */
/* per tile of ZC_TILE chunks, with part[] the exclusive prefix of the tiles' stream bytes (zc_scan_reduce / zc_scan_parts over
 * out_len + c0): S(c) = S[c0] + the round's bytes in front of c; chunk c goes to base_of(c) + S(c), with copy length 0 when its
 * bytes would pass cap; S[c0 + m] carries the total into the next round */
template <class Base>
__global__ void __launch_bounds__(ZC_THREADS) zc_round_place_kernel(Base base_of, const uint32_t *out_len, uint64_t c0, uint32_t m, const uint32_t *part,
                                                                    uint64_t *S, uint64_t *dst, uint32_t *glen, uint64_t cap) {
    __shared__ uint64_t s[ZC_THREADS];
    const uint64_t base = S[c0];
    const uint32_t b0 = blockIdx.x * ZC_TILE + threadIdx.x * ZC_ITEMS;
    uint64_t v = 0;
    for (uint32_t k = 0; k < ZC_ITEMS; k++)
        if (b0 + k < m) v += out_len[c0 + b0 + k];
    uint64_t tot;
    uint64_t run = base + part[blockIdx.x] + zc_block_scan<uint64_t>(v, s, &tot);
    for (uint32_t k = 0; k < ZC_ITEMS; k++) {
        const uint32_t j = b0 + k;
        if (j > m) break;
        const uint64_t c = c0 + j;
        if (j) S[c] = run; /* S[c0] is the previous round's: read above by every thread, not written again */
        if (j == m) break;
        const uint32_t len = out_len[c];
        const uint64_t d = base_of(c) + run;
        dst[c] = d;
        glen[c] = d + len <= cap ? len : 0u;
        run += len;
    }
}

/* ---- end records ------------------------------------------------------------------------------------------------- */
__global__ void __launch_bounds__(ZC_THREADS) zc_end_kernel(const uint8_t *buf, uint64_t len, ZcSummary *S) {
    __shared__ uint64_t red[ZC_THREADS];
    const uint64_t tl = len < ZC_TAIL ? len : ZC_TAIL, base = len - tl;
    uint64_t best = 0; /* position + 1 of the last signature, 0 = none */
    for (uint64_t i = threadIdx.x; i + 22 <= tl; i += ZC_THREADS) {
        const uint8_t *q = buf + base + i;
        if (q[0] == 0x50 && q[1] == 0x4b && q[2] == 0x05 && q[3] == 0x06) best = i + 1;
    }
    red[threadIdx.x] = best;
    __syncthreads();
    for (uint32_t h = ZC_THREADS / 2; h; h >>= 1) {
        if (threadIdx.x < h && red[threadIdx.x + h] > red[threadIdx.x]) red[threadIdx.x] = red[threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x) return;
    /* from here on: zn_read_directory's rules, read for read */
    int32_t err = 0;
    uint64_t count = 0, cd_size = 0, cd_off = 0, eocd = 0, eocd_pos = 0, shift = 0;
    if (!red[0]) {
        err = -103;
    } else {
        eocd = base + red[0] - 1;
        eocd_pos = eocd;
        const uint8_t *q = buf + eocd;
        const uint32_t disk = zc_u16(q + 4), disk_cd = zc_u16(q + 6), on_disk = zc_u16(q + 8);
        count = zc_u16(q + 10);
        cd_size = zc_u32(q + 12);
        cd_off = zc_u32(q + 16);
        if (disk != 0 || disk_cd != 0)
            err = -109;
        else if (on_disk != count)
            err = -103;
        if (!err && (count == 0xffffu || cd_off == 0xffffffffu || cd_size == 0xffffffffu)) {
            const uint8_t *z64 = nullptr;
            if (eocd >= 20 && zc_u32(buf + eocd - 20) == 0x07064b50u) {
                const uint64_t at[2] = {zc_u64(buf + eocd - 20 + 8), eocd - 20 - 56};
                for (int k = 0; k < 2 && !z64; k++) /* the host's read fails at a negative offset */
                    if (at[k] + 56 <= eocd && (int64_t)at[k] >= 0 && zc_u32(buf + at[k]) == 0x06064b50u) {
                        z64 = buf + at[k];
                        eocd_pos = at[k];
                    }
            }
            if (z64) {
                if (zc_u32(z64 + 16) != 0 || zc_u32(z64 + 20) != 0)
                    err = -109;
                else if (zc_u64(z64 + 24) != zc_u64(z64 + 32))
                    err = -103;
                count = zc_u64(z64 + 32);
                cd_size = zc_u64(z64 + 40);
                cd_off = zc_u64(z64 + 48);
                if ((int64_t)cd_size < 0 || (int64_t)cd_off < 0)
                    err = -103;
            } else if (count == 0xffffu || cd_off == 0xffffffffu) {
                err = -103;
            }
        }
    }
    if (!err) {
        /* cd_off, alt <= eocd_pos, and at least 22 bytes lie behind eocd_pos: the 4-byte signature reads are inside */
        if (cd_off > eocd_pos || cd_size > eocd_pos) {
            err = -103;
        } else if (cd_size && zc_u32(buf + cd_off) != 0x02014b50u) {
            const uint64_t alt = eocd_pos - cd_size;
            if (zc_u32(buf + alt) == 0x02014b50u) {
                shift = alt - cd_off;
                cd_off = alt;
            } else {
                err = -103;
            }
        }
        if (!err && cd_off + cd_size > eocd_pos) cd_size = eocd_pos - cd_off;
    }
    if (!err && cd_size / 46 < count) err = -103;
    S->err = err;
    S->cd_off = cd_off;
    S->cd_size = cd_size;
    S->count = count;
    S->shift = shift;
    S->eocd_pos = eocd_pos;
}

/* ---- candidates --------------------------------------------------------------------------------------------------- */
/* a record at directory position p whose fixed part and lengths fit the directory (the host loop's first two checks) */
__device__ __forceinline__ bool zc_valid(const uint8_t *cd, uint64_t cd_size, uint64_t p) {
    if (p >= cd_size || cd_size - p < 46) return false;
    const uint8_t *h = cd + p;
    if (h[0] != 0x50 || h[1] != 0x4b || h[2] != 0x01 || h[3] != 0x02) return false;
    return 46ull + zc_u16(h + 28) + zc_u16(h + 30) + zc_u16(h + 32) <= cd_size - p;
}

__global__ void __launch_bounds__(ZC_THREADS) zc_cand_kernel(const uint8_t *cd, uint64_t cd_size, uint32_t *bits, uint32_t *wcount) {
    const uint64_t p = (uint64_t)blockIdx.x * ZC_THREADS + threadIdx.x;
    const uint32_t m = __ballot_sync(MZ_FULL_MASK, zc_valid(cd, cd_size, p));
    if ((threadIdx.x & 31) == 0 && p < cd_size) {
        bits[p >> 5] = m;
        wcount[p >> 5] = (uint32_t)__popc(m);
    }
}

__device__ __forceinline__ uint32_t zc_rank(const uint32_t *bits, const uint32_t *wpre, uint64_t p) {
    return wpre[p >> 5] + (uint32_t)__popc(bits[p >> 5] & ((1u << (p & 31)) - 1u));
}

__global__ void __launch_bounds__(ZC_THREADS) zc_link_kernel(const uint8_t *cd, uint64_t cd_size, const uint32_t *bits, const uint32_t *wpre,
                                                             uint64_t *cpos, uint32_t *succ, uint32_t *jump, uint32_t *mark) {
    const uint64_t p = (uint64_t)blockIdx.x * ZC_THREADS + threadIdx.x;
    if (p >= cd_size || !((bits[p >> 5] >> (p & 31)) & 1u)) return;
    const uint32_t r = zc_rank(bits, wpre, p);
    const uint8_t *h = cd + p;
    const uint64_t q = p + 46ull + zc_u16(h + 28) + zc_u16(h + 30) + zc_u16(h + 32);
    const uint32_t s = q == cd_size ? ZC_END : ((bits[q >> 5] >> (q & 31)) & 1u) ? zc_rank(bits, wpre, q) : ZC_BRK;
    cpos[r] = p;
    succ[r] = s;
    jump[r] = s;
    mark[r] = p == 0;
}

/* one doubling round. A candidate marked earlier in this same launch may pass its mark on too: it only ever marks nodes that
 * are reachable from the first record, so the result after ceil(log2 ncand) rounds is the same. */
__global__ void __launch_bounds__(ZC_THREADS) zc_double_kernel(uint32_t n, uint32_t *mark, const uint32_t *jin, uint32_t *jout) {
    const uint32_t c = blockIdx.x * ZC_THREADS + threadIdx.x;
    if (c >= n) return;
    const uint32_t j = jin[c];
    if (j < ZC_BRK && *(volatile uint32_t *)&mark[c]) mark[j] = 1;
    jout[c] = j < ZC_BRK ? jin[j] : j;
}

__global__ void __launch_bounds__(ZC_THREADS) zc_place_kernel(uint32_t n, const uint32_t *mark, const uint32_t *midx, const uint64_t *cpos,
                                                              const uint32_t *succ, uint64_t limit, uint64_t *rpos, ZcSummary *S) {
    const uint32_t c = blockIdx.x * ZC_THREADS + threadIdx.x;
    if (c == 0) S->nchain = midx[n];
    if (c >= n || !mark[c]) return;
    const uint32_t i = midx[c];
    if (i < limit) rpos[i] = cpos[c];
    if (i + 1 == midx[n]) S->term = succ[c];
}

/* ---- records --------------------------------------------------------------------------------------------------------- */
__global__ void __launch_bounds__(ZC_THREADS) zc_records_kernel(const uint8_t *buf, uint64_t cd_off, uint64_t shift, const uint64_t *rpos, uint32_t n,
                                                                uint32_t have_pw, uint32_t pw_long, ZcRec *rec, uint64_t *roff, ZcCount *cnt,
                                                                ZcSummary *S) {
    const uint32_t i = blockIdx.x * ZC_THREADS + threadIdx.x;
    if (i >= n) return;
    const uint8_t *h = buf + cd_off + rpos[i];
    const uint32_t flag = zc_u16(h + 8), nlen = zc_u16(h + 28), xlen = zc_u16(h + 30);
    uint32_t method = zc_u16(h + 10), disk = zc_u16(h + 34), aes_method = 0, aes = 0;
    ZcRec e;
    e.crc = zc_u32(h + 16);
    e.csize = zc_u32(h + 20);
    e.usize = zc_u32(h + 24);
    e.off = zc_u32(h + 42);
    e.name_off = cd_off + rpos[i] + 46;
    e.name_len = nlen;
    e.has_sha = 0;
    e.sha_off = 0;
    const uint8_t *xf = h + 46 + nlen;
    for (uint32_t xo = 0; xo + 4 <= xlen;) {
        const uint32_t id = zc_u16(xf + xo), xs = zc_u16(xf + xo + 2), xn = xo + 4 + xs > xlen ? xlen - xo - 4 : xs;
        const uint8_t *x = xf + xo + 4, *xe = x + xn;
        if (id == 0x0001) {
            if (e.usize == 0xffffffffu && x + 8 <= xe) { e.usize = zc_u64(x); x += 8; }
            if (e.csize == 0xffffffffu && x + 8 <= xe) { e.csize = zc_u64(x); x += 8; }
            if (e.off == 0xffffffffu && x + 8 <= xe) { e.off = zc_u64(x); x += 8; }
            if (disk == 0xffffu && x + 4 <= xe) disk = zc_u32(x);
        } else if (id == 0x9901 && xn == 7) {
            aes = x[4];
            aes_method = zc_u16(x + 5);
            if (aes < 1 || aes > 3) aes = 0xff;
        }
        xo += 4 + xs;
    }
    for (uint32_t xo = 0; xo + 4 <= xlen;) { /* zx_find_sha: unclamped lengths */
        const uint8_t *x = xf + xo;
        const uint32_t id = zc_u16(x), xs = zc_u16(x + 2);
        if (xo + 4 + xs > xlen) break;
        if (id == 0x1a51 && xs >= 4 + 32 && zc_u16(x + 4) == 23 && zc_u16(x + 6) == 32) {
            e.sha_off = (uint64_t)(x + 8 - buf);
            e.has_sha = 1;
            break;
        }
        xo += 4 + xs;
    }
    const bool enc = (flag & 1u) != 0;
    if (enc && method == 99 && aes) method = aes_method;
    const uint64_t aes_over = enc && aes && aes != 0xff ? 4u * aes + 4u + 12u : 0u;
    int32_t code = 0;
    if (enc && aes && !have_pw) {
        code = -108;
    } else if ((enc && (!aes || aes == 0xff || pw_long || e.csize < aes_over)) || (!enc && aes) || (method != 0 && method != 8) ||
               e.usize > (1ull << 30) || e.csize > (1ull << 30) || disk != 0) {
        code = -109;
    } else if (method == 0 && e.csize - aes_over != e.usize) {
        code = -103;
    } else {
        e.off += shift;
        if (e.off + 30 > cd_off) code = -103; /* the local header must lie in front of the directory */
    }
    if (!enc) aes = 0;
    e.method = (uint16_t)method;
    e.aes = (uint8_t)aes;
    e.code = code;
    rec[i] = e;
    roff[i] = e.off;
    ZcCount k = zc_zero<ZcCount>();
    k.out = (e.usize + 15) & ~15ull;
    k.cin = e.csize;
    k.cout = e.usize;
    k.job = method == 8;
    k.sha = e.has_sha;
    k.a[1] = aes == 1;
    k.a[2] = aes == 2;
    k.a[3] = aes == 3;
    cnt[i] = k;
    if (code) atomicMin(&S->refuse_idx, i);
}

/* limit / limit_code: where and how the chain itself ends the list (n and MZ_OK when it does not) */
__global__ void __launch_bounds__(ZC_THREADS) zc_finish_kernel(const ZcRec *rec, const uint64_t *roff, const ZcCount *pre, uint32_t limit,
                                                               int32_t limit_code, ZcSummary *S) {
    const uint32_t i = blockIdx.x * ZC_THREADS + threadIdx.x;
    const uint32_t ri = S->refuse_idx, nacc = ri < limit ? ri : limit;
    if (i == 0) {
        const ZcCount t = pre[nacc];
        S->nacc = nacc;
        S->refuse = ri < limit ? rec[ri].code : limit_code;
        S->out = t.out;
        S->cin = t.cin;
        S->cout = t.cout;
        S->job = t.job;
        S->sha = t.sha;
        for (int k = 0; k < 4; k++) S->a[k] = t.a[k];
    }
    if (i >= nacc) return;
    if (i + 1 < nacc && roff[i] > roff[i + 1]) S->unsorted = 1;
    const ZcRec &e = rec[i];
    if (e.aes) atomicMax((unsigned long long *)&S->max_clen[e.aes], (unsigned long long)(e.csize - (4u * e.aes + 4u + 12u)));
}

/* ---- sort and fill ------------------------------------------------------------------------------------------------ */
__global__ void __launch_bounds__(ZC_THREADS) zc_pad_kernel(const uint64_t *roff, uint32_t n, uint64_t *key, uint32_t np) {
    const uint32_t i = blockIdx.x * ZC_THREADS + threadIdx.x;
    if (i < np) key[i] = i < n ? roff[i] : ~0ull;
}

/* one stage (k, j) of the bitonic network over np = 2^m keys */
__global__ void __launch_bounds__(ZC_THREADS) zc_bitonic_kernel(uint64_t *key, uint32_t np, uint32_t k, uint32_t j) {
    const uint32_t i = blockIdx.x * ZC_THREADS + threadIdx.x, l = i ^ j;
    if (i >= np || l <= i) return;
    const uint64_t a = key[i], b = key[l];
    if ((i & k) == 0 ? a > b : a < b) {
        key[i] = b;
        key[l] = a;
    }
}

/* key: the n accepted local-header offsets, non-decreasing. Each entry's extent runs to the smallest offset strictly greater than
 * its own or to the directory, and never further than a header, its data and a descriptor can reach (the host parse's rule). */
__global__ void __launch_bounds__(ZC_THREADS, 4) zc_fill_kernel(const ZcRec *rec, const ZcCount *pre, const uint64_t *key, uint32_t n, uint64_t cd_off,
                                                             const uint8_t *buf, ZipDevEnt *pub, ZipEnt *ent, uint8_t *sha) {
    const uint32_t i = blockIdx.x * ZC_THREADS + threadIdx.x;
    if (i >= n) return;
    const ZcRec e = rec[i];
    const ZcCount p = pre[i];
    uint32_t lo = 0, hi = n; /* first key > e.off */
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (key[mid] <= e.off) lo = mid + 1; else hi = mid;
    }
    const uint64_t end = lo < n ? key[lo] : cd_off, cap = 30u + 65535u + 65535u + e.csize + 24u;
    const uint64_t ext = end - e.off < cap ? end - e.off : cap;
    if (pub) {
        ZipDevEnt d;
        d.local_off = e.off;
        d.csize = e.csize;
        d.usize = e.usize;
        d.out_off = p.out;
        d.name_off = e.name_off;
        d.extent = ext;
        d.sha_off = e.sha_off;
        d.crc = e.crc;
        d.name_len = e.name_len;
        d.method = e.method;
        d.aes = e.aes;
        d.has_sha = e.has_sha;
        d.status = 0;
        pub[i] = d;
    }
    if (ent) {
        const ZcCount t = pre[n];
        const uint32_t base = e.aes == 1 ? 0u : e.aes == 2 ? t.a[1] : t.a[1] + t.a[2]; /* rows grouped by strength, as zr_table lays them out */
        ZipEnt r;
        r.src_off = e.off;
        r.src_len = ext;
        r.csize = e.csize;
        r.usize = e.usize;
        r.out_off = p.out;
        r.crc = e.crc;
        r.job = e.method == 8 ? p.job : 0xffffffffu;
        r.aes_slot = e.aes ? base + (e.aes == 1 ? p.a[1] : e.aes == 2 ? p.a[2] : p.a[3]) : 0xffffffffu;
        r.sha_slot = e.has_sha ? p.sha : ZD_NO_SHA;
        r.method = e.method;
        r.aes = e.aes;
        r.flags = 0;
        r.pad = 0;
        ent[i] = r;
        if (e.has_sha)
            for (int b = 0; b < 32; b++) sha[(uint64_t)p.sha * 32 + b] = buf[e.sha_off + b];
    }
}

/* after K9 verify: each entry's status into the public table, and the first failing entry in directory order */
__global__ void __launch_bounds__(ZC_THREADS) zc_status_kernel(const uint32_t *status, uint32_t n, ZipDevEnt *pub, uint32_t *first) {
    const uint32_t i = blockIdx.x * ZC_THREADS + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = status[i];
    pub[i].status = s ? -(int32_t)(s & 0xffffu) : 0;
    if (s) atomicMin(first, i);
}

} // namespace mzc
#endif
