/* df_codes_v34.cuh -- the deflate kernel's code builder (phase D, block_build_codes) as it was in kernel v3.4, frozen
 * (TEST INFRASTRUCTURE ONLY). tests/emu/df_codes_pair.cuh runs it and today's block_build_codes on the same histograms, on the
 * CPU emulator and on the GPU, and the tests compare every code length, code word, bit count and header bit: a faster builder
 * must not change any of them. Do not edit this copy; the scratch layout (BB_*) is its own, the helpers it calls (cl_len,
 * cl_code, stage_put, len_extra_bits, dist_extra_bits, bar_sync) are the kernel's. */
#ifndef MZ_DF_CODES_V34_CUH
#define MZ_DF_CODES_V34_CUH

#include "deflate_kernel.cuh"

namespace mzc {
namespace v34 {

/* ---- D: block-parallel literal/length + distance codes ------------------------------------------------
 * Thread i < 288 owns literal/length symbol i (286 used), thread 288 + j owns distance symbol j (30 used);
 * both alphabets are warp aligned (warps 0-8 and warp 9). Called by threads 0..319 ONLY; they synchronise
 * among themselves on named barrier 1 so the other warps are not dragged through a dozen barriers.
 * bb = 512 words of shared scratch. Outputs lens (u8), codes (reversed code | len << 16 | extra bits << 20)
 * and bits (u8: code length + extra bits = what one entry of that symbol costs). */
enum { BB_STAT = 0 /* [2][4]: used,total,first */, BB_KRAFT = 8 /* [2 sweeps][2 alph][16] */, BB_K = 72 /* [2][16] */,
       BB_NEXT = 104 /* [2][16] */, BB_SLACK = 136 /* [2] */, BB_CNTW = 144 /* [2 bufs][10 warps][16] */,
       BB_NZ = 464 /* [10] ballots: length != 0 */, BB_ST = 474 /* [10] ballots: a run of equal lengths starts here */,
       BB_HSUM = 484 /* [10] header bits per warp */, BB_HDRBITS = 494 /* size of the block header in bits */ };

__device__ __forceinline__ void bb_count_lengths(uint32_t *cntw_row, uint32_t L, unsigned lane, unsigned &m) {
    if (lane < 16) cntw_row[lane] = 0;
    __syncwarp();
    m = __match_any_sync(MZ_FULL_MASK, L);
    if (L > 0 && lane == (unsigned)(__ffs((int)m) - 1)) cntw_row[L] = (uint32_t)__popc(m);
    __syncwarp();
}

__device__ inline void block_build_codes_v34(const uint32_t *hist_ll, const uint32_t *hist_lit2, const uint32_t *hist_d, uint8_t *lens_ll, uint8_t *lens_d,
                                         uint32_t *code_ll, uint32_t *code_d, uint8_t *bits_ll, uint8_t *bits_d, uint32_t *bb,
                                         uint32_t *stage, uint32_t hdrpos, uint32_t bfinal) {
    const uint32_t tid = threadIdx.x;
    const unsigned lane = lane_id(), w = warp_id();
    const int a = tid < 288 ? 0 : (tid < 320 ? 1 : 2);
    const uint32_t sym = a == 0 ? tid : tid - 288;
    const uint32_t nsym = a == 0 ? 286u : 30u;
    const int M = 15;
    const uint32_t one = 1u << M;
    const uint32_t w0 = a == 0 ? 0u : 9u; /* first warp of my alphabet */
    uint32_t c = (a < 2 && sym < nsym) ? (a == 0 ? hist_ll[sym] + (sym < 256 ? hist_lit2[sym] : 0u) : hist_d[sym]) : 0u;

    if (tid < 144) bb[tid] = (tid == BB_STAT + 2 || tid == BB_STAT + 6) ? 0xffffffffu : 0u;
    bar_sync(1, DF_BB_THREADS);
    if (a < 2) {
        uint32_t used_w = __reduce_add_sync(MZ_FULL_MASK, c ? 1u : 0u);
        uint32_t tot_w = __reduce_add_sync(MZ_FULL_MASK, c);
        uint32_t first_w = __reduce_min_sync(MZ_FULL_MASK, c ? sym : 0xffffffffu);
        if (lane == 0) {
            atomicAdd(&bb[BB_STAT + a * 4 + 0], used_w);
            atomicAdd(&bb[BB_STAT + a * 4 + 1], tot_w);
            atomicMin(&bb[BB_STAT + a * 4 + 2], first_w);
        }
    }
    bar_sync(1, DF_BB_THREADS);
    float ideal = 0.f;
    if (a < 2) {
        uint32_t used = bb[BB_STAT + a * 4 + 0], total = bb[BB_STAT + a * 4 + 1], fu = bb[BB_STAT + a * 4 + 2];
        if (used < 2) { /* force two coded symbols (a complete code needs them; zlib's inflate insists) */
            uint32_t d0 = used == 0 ? 0u : (fu == 0 ? 1u : 0u);
            uint32_t d1 = used == 0 ? 1u : d0;
            if ((sym == d0 || sym == d1) && c == 0) c = 1;
            total += 2 - used;
        }
        if (c) ideal = __log2f((float)total) - __log2f((float)c);
    }
    /* two sweeps of 16 candidate rounding offsets: coarse step 1/4 over [-3, 1), then step 1/64 */
    float lo = -3.0f, step = 0.25f;
    uint32_t slack[2] = {0, 0};
    for (int sweep = 0; sweep < 2; sweep++) {
        if (a < 2) {
#pragma unroll
            for (int cnd = 0; cnd < 16; cnd++) {
                uint32_t kr = 0;
                if (c) {
                    int l = (int)ceilf(ideal - (lo + step * (float)cnd));
                    l = l < 1 ? 1 : (l > M ? M : l);
                    kr = 1u << (M - l);
                }
                kr = __reduce_add_sync(MZ_FULL_MASK, kr);
                if (lane == 0) atomicAdd(&bb[BB_KRAFT + sweep * 32 + a * 16 + cnd], kr);
            }
        }
        bar_sync(1, DF_BB_THREADS);
        /* everyone derives both alphabets' choices (uniform): the largest feasible candidate */
        float lo_a = lo;
        for (int aa = 0; aa < 2; aa++) {
            int best = 0;
            for (int cnd = 1; cnd < 16; cnd++)
                if (bb[BB_KRAFT + sweep * 32 + aa * 16 + cnd] <= one) best = cnd;
            slack[aa] = one - bb[BB_KRAFT + sweep * 32 + aa * 16 + best];
            if (aa == a) lo_a = lo + step * (float)best;
        }
        /* lo is per alphabet from here on; the loop variable is private to the thread */
        lo = lo_a;
        step *= 0.0625f;
    }
    uint32_t L = 0;
    if (c) {
        int l = (int)ceilf(ideal - lo);
        L = (uint32_t)(l < 1 ? 1 : (l > M ? M : l));
    }
    /* exact Kraft completion: shorten codes (short ones first) until the sum is exactly 1 */
    unsigned m = 0;
    int buf = 0;
    for (int pass = 0; pass < 40; pass++) {
        if (slack[0] == 0 && slack[1] == 0) break;
        uint32_t *cntw = bb + BB_CNTW + buf * 160;
        if (a < 2) bb_count_lengths(cntw + w * 16, L, lane, m);
        bar_sync(1, DF_BB_THREADS);
        if (w == 0 || w == 9) { /* one warp per alphabet: lane = code length; the recurrence over lengths is uniform */
            const int aa = w == 0 ? 0 : 1;
            const uint32_t wa = aa == 0 ? 0u : 9u, wb = aa == 0 ? 9u : 10u;
            uint32_t tot = 0;
            if (lane >= 2 && lane <= (unsigned)M)
                for (uint32_t ww = wa; ww < wb; ww++) tot += cntw[ww * 16 + lane];
            uint32_t sl = slack[aa], myk = 0;
            for (int len = 2; len <= M; len++) {
                uint32_t t = __shfl_sync(MZ_FULL_MASK, tot, len);
                uint32_t can = sl >> (M - len);
                uint32_t k = t < can ? t : can;
                if (lane == (unsigned)len) myk = k;
                sl -= k << (M - len);
            }
            if (lane >= 2 && lane <= (unsigned)M) bb[BB_K + aa * 16 + lane] = myk;
            if (lane == 0) bb[BB_SLACK + aa] = sl;
        }
        bar_sync(1, DF_BB_THREADS);
        if (a < 2 && L >= 2) {
            uint32_t rank = (uint32_t)__popc(m & ((1u << lane) - 1));
            for (uint32_t ww = w0; ww < w; ww++) rank += cntw[ww * 16 + L];
            if (rank < bb[BB_K + a * 16 + L]) L -= 1;
        }
        slack[0] = bb[BB_SLACK + 0];
        slack[1] = bb[BB_SLACK + 1];
        buf ^= 1;
    }
    /* canonical codes: code = first code of its length + rank among equal lengths in symbol order */
    uint32_t *cntw = bb + BB_CNTW + buf * 160;
    if (a < 2) bb_count_lengths(cntw + w * 16, L, lane, m);
    bar_sync(1, DF_BB_THREADS);
    if (w == 0 || w == 9) {
        const int aa = w == 0 ? 0 : 1;
        const uint32_t wa = aa == 0 ? 0u : 9u, wb = aa == 0 ? 9u : 10u;
        uint32_t tot = 0;
        if (lane >= 1 && lane <= (unsigned)M)
            for (uint32_t ww = wa; ww < wb; ww++) tot += cntw[ww * 16 + lane];
        uint32_t code = 0, prev = 0, mycode = 0;
        for (int len = 1; len <= M; len++) {
            code = (code + prev) << 1;
            if (lane == (unsigned)len) mycode = code;
            prev = __shfl_sync(MZ_FULL_MASK, tot, len);
        }
        if (lane >= 1 && lane <= (unsigned)M) bb[BB_NEXT + aa * 16 + lane] = mycode;
    }
    bar_sync(1, DF_BB_THREADS);
    if (a < 2) {
        uint32_t cw = 0;
        if (L) {
            uint32_t rank = (uint32_t)__popc(m & ((1u << lane) - 1));
            for (uint32_t ww = w0; ww < w; ww++) rank += cntw[ww * 16 + L];
            uint32_t code = bb[BB_NEXT + a * 16 + L] + rank;
            cw = (__brev(code) >> (32 - L)) | (L << 16);
        }
        if (a == 0) {
            const uint32_t eb = sym >= 257 ? len_extra_bits(sym - 257) : 0u;
            lens_ll[sym] = (uint8_t)L; /* sym up to 287: entries 286, 287 get 0 */
            code_ll[sym] = cw | (eb << 20);
            bits_ll[sym] = (uint8_t)(L + eb);
        } else {
            lens_d[sym] = (uint8_t)L;  /* sym up to 31 */
            code_d[sym] = cw;          /* distance extra bits come from the entry, not the table */
            bits_d[sym] = (uint8_t)(L + dist_extra_bits(sym));
        }
    }
    /* ---- the block header, written straight into the (clean) staging buffer at bit hdrpos. One thread per code length;
     * runs of equal lengths are found from per-warp ballots (a run never crosses from the literal/length lengths into the
     * distance lengths: the RFC allows it, zlib never writes it, so neither do we). ---- */
    const unsigned nz = __ballot_sync(MZ_FULL_MASK, L != 0);
    if (lane == 0) bb[BB_NZ + w] = nz;
    bar_sync(1, DF_BB_THREADS);
    const uint32_t hlit = 256u + 32u - (uint32_t)__clz((int)bb[BB_NZ + 8]); /* the end-of-block symbol always has a code: >= 257 */
    const uint32_t hdw = bb[BB_NZ + 9];
    const uint32_t hdist = hdw ? 32u - (uint32_t)__clz((int)hdw) : 1u;
    const uint32_t nlen = a == 0 ? hlit : hdist;
    const bool valid = sym < nlen;
    const uint32_t prevL = sym == 0 ? 0xffu : (a == 0 ? lens_ll[sym - 1] : lens_d[sym - 1]);
    const unsigned st = __ballot_sync(MZ_FULL_MASK, (valid && prevL != L) || sym == nlen); /* + a sentinel start behind the last length */
    if (lane == 0) bb[BB_ST + w] = st;
    bar_sync(1, DF_BB_THREADS);
    uint32_t nb = 0, val = 0;
    if (valid) {
        uint32_t m = st & (0xffffffffu >> (31u - lane)), ww = w;
        while (m == 0) m = bb[BB_ST + --ww];                   /* symbol 0 starts a run: terminates inside my alphabet */
        const uint32_t s0 = (ww - w0) * 32u + 31u - (uint32_t)__clz((int)m);
        m = lane == 31 ? 0u : st & (0xfffffffeu << lane);
        ww = w;
        while (m == 0) m = bb[BB_ST + ++ww];                   /* the sentinel ends the last run */
        const uint32_t e0 = (ww - w0) * 32u + (uint32_t)__ffs((int)m) - 1u;
        const uint32_t k = sym - s0, R = e0 - s0;                /* my place in a run of R equal lengths */
        uint32_t cs = L, ev = 0, eb = 0;
        bool tok = true;
        if (L == 0) { /* zeros: 18 = 11..138 of them, 17 = 3..10, else one by one */
            const uint32_t full = (R / 138u) * 138u, rem = R - full;
            if (k < full) { tok = k % 138u == 0; cs = 18; ev = 127; eb = 7; }
            else if (rem >= 11) { tok = k == full; cs = 18; ev = rem - 11; eb = 7; }
            else if (rem >= 3) { tok = k == full; cs = 17; ev = rem - 3; eb = 3; }
        } else if (k > 0) { /* the length itself, then 16 = repeat it 3..6 times, else one by one */
            const uint32_t k1 = k - 1, rest = R - 1, full = (rest / 6u) * 6u, rem = rest - full;
            if (k1 < full) { tok = k1 % 6u == 0; cs = 16; ev = 3; eb = 2; }
            else if (rem >= 3) { tok = k1 == full; cs = 16; ev = rem - 3; eb = 2; }
        }
        if (tok) {
            const uint32_t cl = cl_len(cs);
            nb = cl + eb;
            val = cl_code(cs) | (ev << cl);
        }
    }
    const uint32_t incl = warp_incl_sum(nb);
    if (lane == 31) bb[BB_HSUM + w] = incl;
    bar_sync(1, DF_BB_THREADS);
    uint32_t off = incl - nb, total = 0;
    for (uint32_t ww = 0; ww < 10; ww++) {
        const uint32_t t = bb[BB_HSUM + ww];
        off += ww < w ? t : 0u;
        total += t;
    }
    if (nb) stage_put(stage, hdrpos + 17 + 57 + off, val, nb);
    if (tid == 0) {
        stage_put(stage, hdrpos, bfinal | (2u << 1) | ((hlit - 257u) << 3) | ((hdist - 1u) << 8) | (15u << 13), 17);
        bb[BB_HDRBITS] = 17 + 57 + total;
    }
    if (tid == 32) stage_put(stage, hdrpos + 17, (uint32_t)CL_ORDER57, 32);
    if (tid == 64) stage_put(stage, hdrpos + 17 + 32, (uint32_t)(CL_ORDER57 >> 32), 25);
}

} /* namespace v34 */
} /* namespace mzc */

#endif
