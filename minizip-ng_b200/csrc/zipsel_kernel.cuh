/* zipsel_kernel.cuh -- K12: random access to an archive in device memory (the reader of include/mz_zip_cuda.h,
 * mz_zip_cuda_reader_*; launches: mz_cuda_zip_name_* and mz_cuda_zip_sel_* in mz_cuda_api.cu).
 *
 * The reader parses the directory once (K10) and keeps its public table and its K9 table. K12 adds:
 *   index   one thread per accepted entry hashes its name (up to the first NUL, '\\' as '/', A-Z folded) and inserts its index
 *           into an open-addressing table of P >= 2 x count slots (a power of two, linear probing, atomicCAS). Every entry goes
 *           in, duplicates included, so the one table serves both case modes. A slot holds hash >> 32 << 32 | index;
 *   lookup  one thread per query hashes it the same way and walks the probe sequence to the first empty slot; a slot whose
 *           hash tag matches is compared byte for byte under the mode's rule (mz_zip_path_compare: the names as C strings,
 *           '\\' == '/', with ignore_case A-Z folded and bytes >= 0x80 exact), and the smallest matching index wins: the first
 *           match in directory order whatever order the insertions ran in. Cost per query: the probe length plus one compare
 *           per candidate whose folded name hashes the same (names that fold equal, and rare 64-bit collisions);
 *   count   one thread per selection slot: its 16-byte output slot, stored and plain bytes, bytes to gather, K5 job, AES row
 *           per strength and digest use, scanned with K10's templated scan kernels;
 *   fill    the selection's K9 records (mz_cuda_zip_ent) and the output offsets. An index >= count gets an inert record
 *           (no bytes, no job); the status pass marks it MZ_END_OF_LIST;
 *   gather  one warp per slot copies the slot's extent (local header, data, descriptor) from the archive to scratch, any
 *           source and destination alignment. Used when the selection holds WinZip AES entries: K8 decrypts in place, so
 *           the round then reads scratch and the caller's archive is never written;
 *   status  after K9 verify: each slot's status (MZ_END_OF_LIST for an index out of range) and the first failing slot with
 *           its code in one 64-bit word (slot << 32 | -code), lowered by atomicMin.
 * No CTA waits on another, so the kernels also run on the CPU emulator.
 */
#ifndef MZ_ZIPSEL_KERNEL_CUH
#define MZ_ZIPSEL_KERNEL_CUH

#include "mzcuda_common.cuh"
#include "zipcd_kernel.cuh"
#include "zipdir_kernel.cuh"

namespace mzc {

constexpr uint32_t ZS_THREADS = 256;
constexpr uint32_t ZS_MISS = 0xffffffffu;
constexpr uint64_t ZS_EMPTY = ~0ull;

struct ZsCount { /* mirror of mz_cuda_zip_sel_count: per selection slot, scanned */
    uint64_t out, cin, cout, gather;
    uint32_t job, sha, a[4];
    __device__ __forceinline__ ZsCount operator+(const ZsCount &o) const {
        ZsCount r;
        r.out = out + o.out;
        r.cin = cin + o.cin;
        r.cout = cout + o.cout;
        r.gather = gather + o.gather;
        r.job = job + o.job;
        r.sha = sha + o.sha;
        for (int k = 0; k < 4; k++) r.a[k] = a[k] + o.a[k];
        return r;
    }
};

struct ZsCall { /* mirror of mz_cuda_zip_sel */
    const uint8_t *archive;
    const ZipEnt *ent;
    uint32_t count, n;
    const uint32_t *select;
    ZsCount *cnt, *pre;
    void *part;
    uint32_t gather, pad;
    ZipEnt *sel;
    uint64_t *out_off;
    uint8_t *scratch;
};

/* ---- names ---------------------------------------------------------------------------------------------------------- */
/* the byte both compare modes agree on for hashing: '\\' as '/', A-Z folded */
__device__ __forceinline__ uint32_t zs_fold(uint32_t c, bool ic) {
    if (c == '\\') return '/';
    return ic && c - 'A' < 26u ? c + 32u : c;
}

/* length up to the first NUL and the 64-bit FNV-1a hash of the folded bytes */
__device__ __forceinline__ uint64_t zs_hash(const uint8_t *p, uint32_t len, uint32_t *cut) {
    uint64_t h = 0xcbf29ce484222325ull;
    uint32_t k = 0;
    for (; k < len; k++) {
        const uint32_t c = p[k];
        if (!c) break;
        h = (h ^ zs_fold(c, true)) * 0x100000001b3ull;
    }
    *cut = k;
    return h ^ (h >> 29);
}

__global__ void __launch_bounds__(ZS_THREADS) zs_index_kernel(const uint8_t *archive, const ZipDevEnt *pub, uint32_t n,
                                                              unsigned long long *table, uint32_t P) {
    const uint32_t i = blockIdx.x * ZS_THREADS + threadIdx.x;
    if (i >= n) return;
    uint32_t len;
    const uint64_t h = zs_hash(archive + pub[i].name_off, pub[i].name_len, &len);
    const unsigned long long v = (unsigned long long)(h >> 32 << 32 | i);
    for (uint32_t s = (uint32_t)h & (P - 1);; s = (s + 1) & (P - 1))
        if (atomicCAS(&table[s], (unsigned long long)ZS_EMPTY, v) == (unsigned long long)ZS_EMPTY) return;
}

__global__ void __launch_bounds__(ZS_THREADS) zs_lookup_kernel(const uint8_t *archive, const ZipDevEnt *pub, const unsigned long long *table,
                                                               uint32_t P, const uint8_t *names, const uint64_t *name_off, const uint32_t *name_len,
                                                               uint32_t nq, uint32_t ic, uint32_t *index) {
    const uint32_t q = blockIdx.x * ZS_THREADS + threadIdx.x;
    if (q >= nq) return;
    const uint8_t *b = names + name_off[q];
    uint32_t lb;
    const uint64_t h = zs_hash(b, name_len[q], &lb);
    uint32_t best = ZS_MISS;
    if (lb && P) {
        for (uint32_t s = (uint32_t)h & (P - 1);; s = (s + 1) & (P - 1)) {
            const uint64_t v = table[s];
            if (v == ZS_EMPTY) break;
            const uint32_t i = (uint32_t)v;
            if (v >> 32 != h >> 32 || i >= best) continue;
            const uint8_t *a = archive + pub[i].name_off;
            const uint32_t la = pub[i].name_len;
            uint32_t k = 0;
            for (; k < lb && k < la && a[k]; k++)
                if (zs_fold(a[k], ic) != zs_fold(b[k], ic)) break;
            if (k == lb && (k == la || !a[k])) best = i;
        }
    }
    index[q] = best;
}

/* ---- a selection ----------------------------------------------------------------------------------------------------- */
__global__ void __launch_bounds__(ZS_THREADS) zs_count_kernel(ZsCall C) {
    const uint32_t i = blockIdx.x * ZS_THREADS + threadIdx.x;
    if (i >= C.n) return;
    const uint32_t idx = C.select[i];
    ZsCount k = zc_zero<ZsCount>();
    if (idx < C.count) {
        const ZipEnt e = C.ent[idx];
        k.out = (e.usize + 15) & ~15ull;
        k.cin = e.csize;
        k.cout = e.usize;
        k.gather = (e.src_len + 15) & ~15ull;
        k.job = e.method == 8;
        k.sha = e.sha_slot != ZD_NO_SHA;
        k.a[1] = e.aes == 1;
        k.a[2] = e.aes == 2;
        k.a[3] = e.aes == 3;
    }
    C.cnt[i] = k;
}

/* C.sel == NULL: only the output offsets (a sizing call). C.gather: the round reads scratch, where slot i's extent lies at
 * pre[i].gather; otherwise it reads the archive in place. */
__global__ void __launch_bounds__(ZS_THREADS) zs_fill_kernel(ZsCall C) {
    const uint32_t i = blockIdx.x * ZS_THREADS + threadIdx.x;
    if (i > C.n) return;
    const ZsCount p = C.pre[i];
    if (C.out_off) C.out_off[i] = p.out;
    if (i == C.n || !C.sel) return;
    const uint32_t idx = C.select[i];
    ZipEnt r;
    if (idx < C.count) {
        const ZipEnt e = C.ent[idx];
        const ZsCount t = C.pre[C.n];
        const uint32_t base = e.aes == 1 ? 0u : e.aes == 2 ? t.a[1] : t.a[1] + t.a[2]; /* rows grouped by strength, as zc_fill_kernel */
        r = e;
        r.src_off = C.gather ? p.gather : e.src_off;
        r.out_off = p.out;
        r.job = e.method == 8 ? p.job : 0xffffffffu;
        r.aes_slot = e.aes ? base + (e.aes == 1 ? p.a[1] : e.aes == 2 ? p.a[2] : p.a[3]) : 0xffffffffu;
        /* sha_slot keeps pointing into the reader's table of expected digests */
    } else { /* inert: no bytes, no job; locate marks it, the status pass makes it MZ_END_OF_LIST */
        memset(&r, 0, sizeof(r));
        r.out_off = p.out;
        r.job = r.aes_slot = 0xffffffffu;
        r.sha_slot = ZD_NO_SHA;
    }
    C.sel[i] = r;
}

/* one warp per slot: scratch[pre.gather ..) = archive[src_off, src_off + src_len). The destination's head bytes go one by one
 * until it is word aligned; then every destination word is two aligned source words joined by a funnel shift, and the ragged
 * tail is bytes. The source word after the last byte is read: extents end at or before the directory, behind which lie at
 * least 68 bytes of the archive. */
__global__ void __launch_bounds__(ZS_THREADS) zs_gather_kernel(ZsCall C) {
    const uint32_t warp = (blockIdx.x * ZS_THREADS + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const uint32_t nwarps = (gridDim.x * ZS_THREADS) >> 5;
    for (uint32_t i = warp; i < C.n; i += nwarps) {
        const uint32_t idx = C.select[i];
        if (idx >= C.count) continue;
        const ZipEnt &e = C.ent[idx];
        const uint8_t *s = C.archive + e.src_off;
        uint8_t *d = C.scratch + C.pre[i].gather;
        uint64_t len = e.src_len;
        uint32_t head = (uint32_t)(-(uintptr_t)d & 3u);
        if (head > len) head = (uint32_t)len;
        if (lane < head) d[lane] = s[lane];
        s += head;
        d += head;
        len -= head;
        const uint32_t *w = (const uint32_t *)((uintptr_t)s & ~(uintptr_t)3);
        const uint32_t sh = (uint32_t)((uintptr_t)s & 3) * 8u;
        const uint64_t words = len >> 2;
        for (uint64_t k = lane; k < words; k += 32) {
            const uint32_t lo = w[k], hi = sh ? w[k + 1] : 0u;
            ((uint32_t *)d)[k] = __funnelshift_r(lo, hi, sh);
        }
        for (uint64_t k = (words << 2) + lane; k < len; k += 32) d[k] = s[k];
    }
}

/* after K9 verify: out (optional) = each slot's MZ code; *first lowered to slot << 32 | -code of the first failing slot */
__global__ void __launch_bounds__(ZS_THREADS) zs_status_kernel(const uint32_t *status, const uint32_t *select, uint32_t n, uint32_t count,
                                                               int32_t *out, unsigned long long *first) {
    const uint32_t i = blockIdx.x * ZS_THREADS + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = status[i];
    const int32_t code = select[i] >= count ? -100 /* MZ_END_OF_LIST */ : s ? -(int32_t)(s & 0xffffu) : 0;
    if (out) out[i] = code;
    if (code) atomicMin(first, (unsigned long long)i << 32 | (uint32_t)-code);
}

} // namespace mzc
#endif
