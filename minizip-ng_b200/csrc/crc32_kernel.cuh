/* crc32_kernel.cuh -- K1: slice-by-warp CRC-32 (poly 0xEDB88320 reflected) + GF(2) combine (sm_90a).
 *
 * Replaces the arithmetic behind mz_crypt_crc32_update (mz_crypt.c:35-92; table loop :81-90).
 *
 * Formulation. A buffer is the polynomial D(x) over GF(2); the "pure residue" R(D) = D(x) x^32 mod P
 * (CRC with init 0 / xorout 0) is linear, so
 *     crc(v, D) = ~( (~v) x^(8|D|) + R(D) )            (running update, mz_crypt.c:81,90 inversions)
 *     R(A||B)   = R(A) x^(8|B|) + R(B)                 (combine; what zlib calls crc32_combine)
 * One warp owns one segment (a chunk). It streams 512-byte rows with one coalesced 16-byte load per lane
 * and keeps 4 independent 32-bit states per lane, one per word slot of the row. Because consecutive words
 * of a slot are 512 bytes apart, the per-row step of every slot of every lane is the SAME linear map
 *     s <- s * x^4096 mod P  xor  w
 * done with four 256-entry tables (slice-by-4 on the state, not on the data). The tables are replicated
 * 32 times in shared memory, entry e of table k for lane l at word ((k*256+e)*32 + l), so every lookup of
 * every lane hits its own bank: 1 conflict-free LDS per input byte, 128 KiB of shared memory per CTA.
 * At the end of a segment the 128 slot states form a 512-byte string whose residue is the segment's:
 * each state is multiplied by x^(32*(128-slot)) (shift-xor multiply) and the warp xor-reduces.
 * Unaligned heads and sub-row tails go through the same row step as a right-aligned virtual row
 * (leading zeros do not change a pure residue).
 */
#ifndef MZ_CRC32_KERNEL_CUH
#define MZ_CRC32_KERNEL_CUH

#include "mzcuda_common.cuh"

namespace mzc {

constexpr uint32_t CRC_POLY = 0xEDB88320u;
constexpr int CRC_THREADS = 1024;
constexpr int CRC_ROW = 512;
constexpr int CRC_TABLE_WORDS = 4 * 256 * 32; /* 128 KiB */
constexpr int CRC_SMEM_BYTES = CRC_TABLE_WORDS * 4;
constexpr int CRC_UNROLL = 4; /* rows per load batch; the next batch is in flight while one is folded */

/* a(x) * b(x) mod P in the reflected representation (bit 31 = x^0). 32 shift-xor steps. */
__host__ __device__ inline uint32_t gf2_mulmod(uint32_t a, uint32_t b) {
    uint32_t p = 0;
    for (int i = 0; i < 32; i++) {
        p ^= b & (0u - ((a >> (31 - i)) & 1u)); /* coefficient of x^i in a */
        b = (b >> 1) ^ (CRC_POLY & (0u - (b & 1u)));
    }
    return p;
}

/* a(x) * x^32 mod P: 32 multiplications by x */
__host__ __device__ inline uint32_t gf2_mul_x32(uint32_t a) {
    for (int i = 0; i < 32; i++) a = (a >> 1) ^ (CRC_POLY & (0u - (a & 1u)));
    return a;
}

/* x^(2^k) mod P for k = 0..63, filled on the host once (crc_consts) */
struct CrcConsts {
    uint32_t x2n[64];      /* x^(2^k) */
    uint32_t slot_mul[128]; /* x^(32*(128-s)) for slot s = 4*lane + j */
    uint32_t row_tab[4][256]; /* T_k[v] = (v << 8k) * x^4096 */
};

__host__ __device__ inline uint32_t gf2_xpow(const uint32_t *x2n, uint64_t n) { /* x^n mod P */
    uint32_t p = 0x80000000u;
    for (int k = 0; n; n >>= 1, k++)
        if (n & 1) p = gf2_mulmod(x2n[k], p);
    return p;
}

inline void crc_consts_init(CrcConsts &c) {
    uint32_t p = 0x40000000u; /* x^1 */
    c.x2n[0] = p;
    for (int k = 1; k < 64; k++) c.x2n[k] = p = gf2_mulmod(p, p);
    for (int s = 0; s < 128; s++) c.slot_mul[s] = gf2_xpow(c.x2n, 32ull * (128 - s));
    uint32_t x4096 = gf2_xpow(c.x2n, 4096);
    for (int k = 0; k < 4; k++)
        for (uint32_t v = 0; v < 256; v++) c.row_tab[k][v] = gf2_mulmod(v << (8 * k), x4096);
}

struct CrcParams {
    const uint8_t *in;
    const uint64_t *in_off; /* per-segment offsets or NULL for a uniform partition */
    const uint32_t *in_len;
    uint64_t total_len;
    uint64_t seg_size; /* uniform partition */
    uint32_t nseg;
    const CrcConsts *consts; /* device copy */
    uint32_t *out_residue;   /* R(segment), per segment */
    uint32_t *out_crc;       /* optional: finalized crc32(0, segment) per segment */
    uint64_t init_len;       /* 0, or a segment length whose init term ~0 * x^(8 init_len) the caller computed once: init */
    uint32_t init;
};

/* the init term of crc32(0, .) over len bytes, ~0 * x^(8 len): a launch over a uniform partition passes it for seg_size */
inline uint32_t crc_init_term(const CrcConsts &c, uint64_t len) { return gf2_mulmod(0xffffffffu, gf2_xpow(c.x2n, 8ull * len)); }

/* one row step of a state: byte k of s picks entry k of this lane's copy of table k. The byte comes out of a PRMT and the
 * address of an IMAD by k128 = 128 (the stride between entries), which the compiler cannot turn into shifts and LEAs, so the
 * address arithmetic runs on the FMA pipe and the integer-ALU pipe is left with the byte extraction and the xors. */
#define MZ_CRC_STEP(s, w)                                                                                                    \
    (s) = sm.ld32_a(MZ_BYTE(s, 0) * k128 + a0) ^ sm.ld32_a(MZ_BYTE(s, 1) * k128 + a1) ^ sm.ld32_a(MZ_BYTE(s, 2) * k128 + a2) ^ \
          sm.ld32_a(MZ_BYTE(s, 3) * k128 + a3) ^ (w)

/* gather up to 16 bytes of a right-aligned virtual row: virtual byte index vb = lane*16 + i maps to
 * data[vb - (512 - n)] when that is >= 0 */
__device__ __forceinline__ uint4 crc_virtual_row(const uint8_t *data, uint32_t n, unsigned lane) {
    uint32_t w[4] = {0, 0, 0, 0};
    int shift = (int)CRC_ROW - (int)n;
#pragma unroll
    for (int i = 0; i < 16; i++) {
        int vb = (int)lane * 16 + i;
        if (vb >= shift) w[i >> 2] |= (uint32_t)data[vb - shift] << (8 * (i & 3));
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}

/* sum over the lane's slots j of s_j x^(32 (128 - 4 lane - j)): Horner over the four slots by x^32, then one multiplication by
 * the last slot's x^(32 (125 - 4 lane)) */
__device__ __forceinline__ uint32_t crc_warp_finalize(uint32_t s0, uint32_t s1, uint32_t s2, uint32_t s3, const CrcConsts *cc,
                                                      unsigned lane) {
    const uint32_t u = gf2_mul_x32(gf2_mul_x32(gf2_mul_x32(s0) ^ s1) ^ s2) ^ s3;
    return __reduce_xor_sync(MZ_FULL_MASK, gf2_mulmod(u, cc->slot_mul[4 * lane + 3]));
}

__global__ void __launch_bounds__(CRC_THREADS, 1) crc32_segments_kernel(CrcParams P) {
    MZ_DYN_SMEM(smem);
    uint32_t *tab = (uint32_t *)smem;
    const unsigned lane = lane_id();
    /* replicate the 4 KiB of tables 32 times, one copy per bank */
    for (uint32_t i = threadIdx.x; i < CRC_TABLE_WORDS; i += CRC_THREADS) tab[i] = (&P.consts->row_tab[0][0])[i >> 5];
    __syncthreads();
    Smem sm;
    sm.init(smem);
    const uint32_t a0 = sm.addr(lane * 4), a1 = a0 + 256 * 32 * 4, a2 = a1 + 256 * 32 * 4, a3 = a2 + 256 * 32 * 4;
    const uint32_t k128 = blockDim.x / (CRC_THREADS / 128); /* 128, opaque to the compiler */

    const uint32_t nwarps = gridDim.x * (CRC_THREADS / 32);
    for (uint32_t seg = blockIdx.x * (CRC_THREADS / 32) + warp_id(); seg < P.nseg; seg += nwarps) {
        uint64_t off;
        uint64_t len;
        if (P.in_off) {
            off = P.in_off[seg];
            len = P.in_len[seg];
        } else {
            off = (uint64_t)seg * P.seg_size;
            len = P.total_len - off < P.seg_size ? P.total_len - off : P.seg_size;
        }
        const uint8_t *p = P.in + off;
        uint32_t s0 = 0, s1 = 0, s2 = 0, s3 = 0;
        /* head: bytes up to the first 16-byte boundary, as a right-aligned virtual row */
        uint64_t head = (16 - ((uintptr_t)p & 15)) & 15;
        if (head > len) head = len;
        if (head) {
            uint4 w = crc_virtual_row(p, (uint32_t)head, lane);
            s0 = w.x; s1 = w.y; s2 = w.z; s3 = w.w; /* first row: states start at zero */
        }
        const uint8_t *q = p + head;
        uint64_t rows = (len - head) / CRC_ROW;
        const uint4 *rp = (const uint4 *)q + lane;
        uint64_t r = 0;
        if (rows >= CRC_UNROLL) {
            /* software pipeline: batch r + CRC_UNROLL is loaded before batch r is folded, so a warp always has rows in flight */
            uint4 w[CRC_UNROLL];
#pragma unroll
            for (int u = 0; u < CRC_UNROLL; u++) w[u] = ldg_stream(rp + (uint64_t)u * (CRC_ROW / 16));
            for (;; r += CRC_UNROLL) {
                const bool more = r + 2 * CRC_UNROLL <= rows;
                uint4 nx[CRC_UNROLL];
#pragma unroll
                for (int u = 0; u < CRC_UNROLL; u++) nx[u] = more ? ldg_stream(rp + (r + CRC_UNROLL + u) * (CRC_ROW / 16)) : w[u];
#pragma unroll
                for (int u = 0; u < CRC_UNROLL; u++) {
                    MZ_CRC_STEP(s0, w[u].x);
                    MZ_CRC_STEP(s1, w[u].y);
                    MZ_CRC_STEP(s2, w[u].z);
                    MZ_CRC_STEP(s3, w[u].w);
                }
                if (!more) break;
#pragma unroll
                for (int u = 0; u < CRC_UNROLL; u++) w[u] = nx[u];
            }
            r += CRC_UNROLL;
        }
        for (; r < rows; r++) {
            uint4 w = ldg_stream(rp + r * (CRC_ROW / 16));
            MZ_CRC_STEP(s0, w.x);
            MZ_CRC_STEP(s1, w.y);
            MZ_CRC_STEP(s2, w.z);
            MZ_CRC_STEP(s3, w.w);
        }
        const CrcConsts *cc = P.consts;
        uint32_t res = crc_warp_finalize(s0, s1, s2, s3, cc, lane);
        uint32_t tail = (uint32_t)(len - head - rows * CRC_ROW);
        if (tail) {
            uint4 w = crc_virtual_row(q + rows * CRC_ROW, tail, lane);
            uint32_t rt = crc_warp_finalize(w.x, w.y, w.z, w.w, cc, lane);
            if (lane == 0) res = gf2_mulmod(res, gf2_xpow(cc->x2n, 8ull * tail)) ^ rt;
        }
        if (lane == 0) {
            P.out_residue[seg] = res;
            if (P.out_crc) {
                const uint32_t init = P.init_len && len == P.init_len ? P.init : gf2_mulmod(0xffffffffu, gf2_xpow(cc->x2n, 8ull * len));
                P.out_crc[seg] = ~(init ^ res);
            }
        }
    }
}

/* Fold per-segment residues of a UNIFORM partition into one residue: R = sum_i R_i x^(8 * bytes after i).
 * Single CTA. Each thread Horner-folds a contiguous run, then a shared-memory tree combines the runs. */
constexpr int CRCF_THREADS = 1024;
__global__ void __launch_bounds__(CRCF_THREADS, 1)
crc32_fold_kernel(const uint32_t *residue, uint32_t nseg, uint64_t seg_size, uint64_t total_len, const CrcConsts *cc, uint32_t *out) {
    __shared__ uint32_t s_r[CRCF_THREADS];
    __shared__ uint32_t s_mul;
    const uint32_t tid = threadIdx.x;
    /* all segments but the last have seg_size bytes; put the ragged last segment aside */
    const uint32_t nfull = nseg ? nseg - 1 : 0;
    const uint64_t last_len = nseg ? total_len - (uint64_t)nfull * seg_size : 0;
    const uint32_t per = (nfull + CRCF_THREADS - 1) / CRCF_THREADS;
    const uint32_t m1 = gf2_xpow(cc->x2n, 8ull * seg_size);
    /* right-align the runs so that padding (zero residues) sits in FRONT and is harmless */
    const uint64_t padded = (uint64_t)per * CRCF_THREADS;
    const uint64_t lead = padded - nfull;
    uint32_t acc = 0;
    for (uint32_t k = 0; k < per; k++) {
        uint64_t j = (uint64_t)tid * per + k;
        uint32_t r = j >= lead ? residue[j - lead] : 0u;
        acc = gf2_mulmod(acc, m1) ^ r;
    }
    s_r[tid] = acc;
    if (tid == 0) s_mul = gf2_xpow(cc->x2n, 8ull * seg_size * per);
    __syncthreads();
    for (uint32_t stride = 1; stride < CRCF_THREADS; stride <<= 1) {
        uint32_t mul = s_mul;
        uint32_t v = 0;
        bool act = (tid % (2 * stride)) == (2 * stride - 1);
        if (act) v = gf2_mulmod(s_r[tid - stride], mul) ^ s_r[tid];
        __syncthreads();
        if (act) s_r[tid] = v;
        if (tid == 0) s_mul = gf2_mulmod(mul, mul);
        __syncthreads();
    }
    if (tid == 0) {
        uint32_t r = s_r[CRCF_THREADS - 1];
        if (nseg) r = gf2_mulmod(r, gf2_xpow(cc->x2n, 8ull * last_len)) ^ residue[nseg - 1];
        out[0] = r;                                                                  /* pure residue of the whole buffer */
        out[1] = ~(gf2_mulmod(0xffffffffu, gf2_xpow(cc->x2n, 8ull * total_len)) ^ r); /* crc32(0, buffer) */
    }
}

} // namespace mzc
#endif
