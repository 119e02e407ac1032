/* inflate_kernel.cuh -- K5: RFC1951 decode, one warp per independent stream (sm_90a).
 *
 * Replaces what zlib's inflate() does behind mz_stream_zlib_read (mz_strm_zlib.c:116-193): per block,
 * Huffman table build + symbol decode + LZ77 back-reference copy, with exact consumed-bytes accounting
 * (TOTAL_IN semantics, mz_strm_zlib.c:168-175) and zlib's error taxonomy (data error / truncated).
 *
 * Shape: block starts inside one foreign stream are only known by decoding, so ONE stream is walked serially by
 * one warp; parallelism comes from (a) many independent streams (zip entries) = many warps, (b) inside a warp:
 * table construction and match copies are warp-cooperative, the symbol loop runs uniformly in all lanes (lane 0
 * stores the literals), and (c) for one long
 * stream, the segment-speculative driver in inflate_spec_kernel.cuh, which runs this same decoder from guessed
 * block starts with a symbolic history. The decoder is RESUMABLE at symbol granularity through InflateState,
 * so the host can feed a long stream through a bounded device window (input refills, output drains) -- the
 * read path of the vtbl stream.
 *
 * v3 (instruction diet; the symbol loop is issue/latency bound, not memory bound):
 *   - 32-bit table entries carry {code length, extra-bit count, kind, base value}: no per-symbol base/extra
 *     arithmetic; 10-bit literal/length and 8-bit distance primary tables (5 KB per warp -> 32 warps per SM)
 *   - the bit reader merges aligned 32-bit words with the next word prefetched one refill ahead
 *   - input/output limits are turned into a token budget once, instead of four checks per symbol
 *   - one packed shuffle publishes {event, length, distance} to the warp
 *   - history is read where the output is written (template Out): final bytes in global memory, or the
 *     16-bit symbolic ring of the speculative pass
 */
#ifndef MZ_INFLATE_KERNEL_CUH
#define MZ_INFLATE_KERNEL_CUH

#include "mzcuda_common.cuh"

namespace mzc {

constexpr int INF_PB = 10;  /* primary lit/len table bits */
constexpr int INF_DB = 8;   /* primary distance table bits */
constexpr int INF_THREADS = 32;

enum { INF_ST_RUN = 0, INF_ST_END = 1, INF_ST_DATA_ERROR = -3, INF_ST_BUF_ERROR = -5 };
enum { INF_PH_HEADER = 0, INF_PH_CODES = 1, INF_PH_STORED = 2 };
enum { INF_WHY_NONE = 0, INF_WHY_INPUT = 1, INF_WHY_OUTPUT = 2, INF_WHY_BOUNDARY = 3 };
enum { INF_JOB_STOP_AT_BOUNDARY = 1 }; /* InflateJob.flags: return (why = BOUNDARY) after the next completed block */

struct InflateState {
    uint64_t in_bitpos;  /* absolute bit position in the raw deflate stream */
    uint64_t out_pos;    /* absolute bytes produced */
    int32_t status;      /* INF_ST_* */
    int32_t why;         /* INF_WHY_* when status == RUN */
    uint32_t phase;
    uint32_t last_block;
    uint32_t stored_remaining;
    uint32_t nlit, ndist;
    uint32_t blocks;     /* blocks completed */
    uint8_t lens[320];   /* current block's code lengths (lit/len then dist) */
};

struct InflateJob {
    const uint8_t *in;   /* device bytes; in[0] is absolute stream byte in_base; >= 16 readable bytes past in_avail */
    uint64_t in_base;
    uint64_t in_avail;   /* valid bytes at `in` */
    uint8_t *out;        /* out[0] is absolute output byte out_base; must hold 32 KiB of history if out_pos > 0 */
    uint64_t out_base;
    uint64_t out_cap;    /* bytes available at `out` */
    uint32_t in_final;   /* no more input will follow */
    uint32_t flags;      /* INF_JOB_* */
};

/* table entry: bits 0..3 code length (0 = not in the primary table), 4..7 extra bits, 8..9 kind, 16..31 value */
enum { INF_K_LIT = 0, INF_K_BASE = 1, INF_K_EOB = 2, INF_K_BAD = 3 };
enum { INF_ALPHA_PLAIN = 0, INF_ALPHA_LITLEN = 1, INF_ALPHA_DIST = 2 };

struct InfTables {
    uint32_t lit[1 << INF_PB];
    uint32_t dist[1 << INF_DB];
    uint16_t lsym[288];         /* symbols sorted by (len, sym) */
    uint16_t dsym[32];
    uint16_t lcount[16], dcount[16];
    uint32_t scratch[32];
    uint8_t lens[384];
};
constexpr int INF_SMEM_BYTES = ((int)sizeof(InfTables) + 15) / 16 * 16;
constexpr uint32_t INF_OFF_LIT = 0;                          /* byte offsets inside InfTables, for the explicit */
constexpr uint32_t INF_OFF_DIST = (1u << INF_PB) * 4u;        /* shared-space loads of the symbol loop */

__device__ __forceinline__ uint32_t inf_len_base(uint32_t s, uint32_t &eb) { /* s = sym - 257 in 0..28 */
    if (s < 8) { eb = 0; return 3 + s; }
    if (s == 28) { eb = 0; return 258; }
    eb = (s >> 2) - 1;
    return 3 + ((4 + (s & 3)) << eb);
}
__device__ __forceinline__ uint32_t inf_dist_base(uint32_t s, uint32_t &eb) { /* s in 0..29 */
    if (s < 4) { eb = 0; return 1 + s; }
    eb = (s >> 1) - 1;
    return 1 + ((2 + (s & 1)) << eb);
}
__device__ __forceinline__ uint32_t inf_entry(int alpha, uint32_t sym, uint32_t n) {
    if (alpha == INF_ALPHA_PLAIN) return n | (sym << 16);
    uint32_t eb, base;
    if (alpha == INF_ALPHA_LITLEN) {
        if (sym < 256) return n | (sym << 16);
        if (sym == 256) return n | (INF_K_EOB << 8);
        if (sym > 285) return n | (INF_K_BAD << 8);
        base = inf_len_base(sym - 257, eb);
    } else {
        if (sym > 29) return n | (INF_K_BAD << 8);
        base = inf_dist_base(sym, eb);
    }
    return n | (eb << 4) | (INF_K_BASE << 8) | (base << 16);
}

/* Build decode structures for one alphabet from code lengths. Warp-cooperative.
 * Returns <0 over-subscribed, >0 incomplete (unused code space), 0 complete. */
__device__ inline int inf_build(const uint8_t *lens, int n, uint16_t *count, uint16_t *sorted, uint32_t *table, int tbits, int alpha,
                                uint32_t *scratch) {
    const unsigned lane = lane_id();
    if (lane < 16) scratch[lane] = 0;
    for (int i = (int)lane; i < (1 << tbits); i += 32) table[i] = 0;
    __syncwarp();
    for (int i = (int)lane; i < n; i += 32) atomicAdd(&scratch[lens[i]], 1u);
    __syncwarp();
    uint32_t cnt = lane < 16 ? scratch[lane] : 0;
    __syncwarp();
    if (lane < 16) count[lane] = (uint16_t)cnt;
    /* Kraft check (uniform across the warp) */
    int left = 1;
    for (int len = 1; len <= 15; len++) {
        uint32_t c = __shfl_sync(MZ_FULL_MASK, cnt, len);
        left = (left << 1) - (int)c;
        if (left < 0) break;
    }
    if (left < 0) return left;
    /* lane = code length: first insert index and first canonical code of that length */
    uint32_t offs = 0, code = 0;
    if (lane >= 1 && lane < 16) {
        for (unsigned b = 1; b < lane; b++) offs += scratch[b];
        for (unsigned b = 1; b <= lane; b++) code = (code + (b == 1 ? 0u : scratch[b - 1])) << 1;
    }
    __syncwarp();
    if (lane < 16) {
        scratch[lane] = offs;       /* running insert index per length */
        scratch[16 + lane] = code;  /* running canonical code per length */
    }
    __syncwarp();
    for (int base = 0; base < n; base += 32) {
        int i = base + (int)lane;
        uint32_t l = i < n ? lens[i] : 0u;
        unsigned m = __match_any_sync(MZ_FULL_MASK, l);
        uint32_t rank = (uint32_t)__popc(m & ((1u << lane) - 1));
        if (l) {
            sorted[scratch[l] + rank] = (uint16_t)i;
            if ((int)l <= tbits) {
                uint32_t c = scratch[16 + l] + rank;
                uint32_t r = __brev(c) >> (32 - l);
                uint32_t ent = inf_entry(alpha, (uint32_t)i, l);
                for (uint32_t e = r; e < (1u << tbits); e += 1u << l) table[e] = ent;
            }
        }
        __syncwarp();
        if (l && rank == 0) {
            uint32_t k = (uint32_t)__popc(m);
            scratch[l] += k;
            scratch[16 + l] += k;
        }
        __syncwarp();
    }
    return left;
}

struct InfBits { /* LSB-first bit reader over aligned 32-bit words, next word prefetched; all state in 32-bit registers */
    const uint32_t *w0;  /* aligned word holding in[0] */
    uint64_t avail_bits;
    uint32_t lo, hi;     /* bit buffer: stream bits 0..31 in lo, 32..63 in hi; bits past `bc` are zero */
    uint32_t bc;         /* valid bits in hi:lo */
    uint32_t widx;       /* index (from w0) of the word held in `nxt` (not merged yet) */
    uint32_t wend;       /* first word index that must not be read */
    uint32_t nxt, skew;
    __device__ __forceinline__ void load() {
        nxt = 0;
        if (widx < wend) nxt = w0[widx];
    }
    __device__ __forceinline__ void init(const uint8_t *in, uint64_t avail_bytes, uint64_t rel_bitpos) {
        const uintptr_t a = (uintptr_t)in;
        w0 = (const uint32_t *)(a & ~(uintptr_t)3);
        skew = (uint32_t)(a & 3) * 8u;
        wend = (uint32_t)(((a & 3) + avail_bytes + 16) >> 2);
        avail_bits = avail_bytes * 8;
        const uint64_t abs = rel_bitpos + skew;
        widx = (uint32_t)(abs >> 5);
        load();
        lo = hi = 0; bc = 0;
        refill();
        drop((uint32_t)abs & 31u);
        refill();
    }
    __device__ __forceinline__ void refill() { /* keeps >= 32 valid bits; below 32 everything valid sits in lo and hi is 0 */
        if (bc < 32) {
            lo |= nxt << bc;
            hi = __funnelshift_rc(nxt, 0u, 32u - bc);
            bc += 32;
            widx++;
            load();
        }
    }
    __device__ __forceinline__ uint32_t peek(uint32_t n) const { return lo & ((1u << n) - 1u); }
    __device__ __forceinline__ void drop(uint32_t n) { /* n <= 31 */
        lo = __funnelshift_r(lo, hi, n);
        hi >>= n;
        bc -= n;
    }
    __device__ __forceinline__ uint32_t get(uint32_t n) { uint32_t v = peek(n); drop(n); refill(); return v; } /* n <= 16 */
    /* bits consumed so far, relative to in[0] */
    __device__ __forceinline__ uint64_t bitpos() const { return (uint64_t)widx * 32u - bc - skew; }
    __device__ __forceinline__ int64_t bits_left() const { return (int64_t)avail_bits - (int64_t)bitpos(); }
};

/* canonical bit-by-bit decode for codes longer than the primary table: takes the next 15 stream bits, returns
 * symbol | code length << 16, or -1. (Takes the bits by value so the bit reader never has to live in memory.) */
__device__ __noinline__ int inf_slow_decode(uint32_t bits, const uint16_t *count, const uint16_t *sorted) {
    int code = 0, first = 0, index = 0;
#pragma unroll 1
    for (int len = 1; len <= 15; len++) {
        code |= (int)((bits >> (len - 1)) & 1u);
        int c = count[len];
        if (code - c < first) return (int)sorted[index + (code - first)] | (len << 16);
        index += c;
        first += c;
        first <<= 1;
        code <<= 1;
    }
    return -1;
}

/* An incomplete set (zlib allows one code of length 1, and no distance code at all) leaves 1-bit patterns without a symbol:
 * mark them invalid with their bit, as zlib's tables do, so that decoding one consumes that bit and a truncated stream is told
 * from a corrupt one. l1 / l2: what inf_build returned for the literal/length and the distance set. Warp-cooperative. */
__device__ __forceinline__ void inf_mark_invalid(InfTables &T, int l1, int l2) {
    const unsigned lane = lane_id();
    if (l1 > 0)
        for (int i = (int)lane; i < (1 << INF_PB); i += 32)
            if (T.lit[i] == 0) T.lit[i] = 1u | (INF_K_BAD << 8);
    if (l2 > 0)
        for (int i = (int)lane; i < (1 << INF_DB); i += 32)
            if (T.dist[i] == 0) T.dist[i] = 1u | (INF_K_BAD << 8);
    __syncwarp();
}

/* Warp-cooperative: read a dynamic block header (the bits after BFINAL/BTYPE) and build both decode tables
 * (RFC1951 3.2.7; zlib's rules for incomplete sets). EVERY lane runs the same bit reader over the same bits
 * (uniform control flow, no broadcasts); shared memory is written by lane 0 or by lanes in parallel.
 * Returns 0 or an INF_ST_* error (the same in all lanes). Every check comes after all the bits it depends on, as
 * zlib's NEEDBITS does: a check that failed on bits past the input's end is a truncation, which the state save tells. */
__device__ __forceinline__ int inf_dynamic_header(InfBits &b, InfTables &T, uint32_t &nlit, uint32_t &ndist) {
    const unsigned lane = lane_id();
    nlit = b.get(5) + 257;
    ndist = b.get(5) + 1;
    const uint32_t hc = b.get(4) + 4;
    if (nlit > 286 || ndist > 30) return INF_ST_DATA_ERROR;
    if (lane < 19) T.lens[lane] = 0;
    __syncwarp();
    for (uint32_t i = 0; i < hc; i++) {
        uint32_t pos;
        switch (i) {
            case 0: pos = 16; break; case 1: pos = 17; break; case 2: pos = 18; break; case 3: pos = 0; break;
            case 4: pos = 8; break; case 5: pos = 7; break; case 6: pos = 9; break; case 7: pos = 6; break;
            case 8: pos = 10; break; case 9: pos = 5; break; case 10: pos = 11; break; case 11: pos = 4; break;
            case 12: pos = 12; break; case 13: pos = 3; break; case 14: pos = 13; break; case 15: pos = 2; break;
            case 16: pos = 14; break; case 17: pos = 1; break; default: pos = 15; break;
        }
        const uint32_t v = b.get(3);
        if (lane == 0) T.lens[pos] = (uint8_t)v;
    }
    __syncwarp();
    int left = inf_build(T.lens, 19, T.lcount, T.lsym, T.lit, 7, INF_ALPHA_PLAIN, T.scratch);
    __syncwarp();
    if (left != 0) return INF_ST_DATA_ERROR; /* code-length code must be complete */
    {
        uint32_t idx = 0, prev = 0;
        const uint32_t total = nlit + ndist;
        uint8_t *lens = T.lens + 32; /* decoded lengths, staged after the 19 cl lengths */
        while (idx < total) {
            const uint32_t e = T.lit[b.peek(7)];
            if (e == 0) return INF_ST_DATA_ERROR;
            b.drop(e & 15u);
            b.refill();
            const uint32_t sym = e >> 16;
            if (sym < 16) {
                if (lane == 0) lens[idx] = (uint8_t)sym;
                idx++;
                prev = sym;
            } else {
                uint32_t rep, val = 0;
                if (sym == 16) {
                    val = prev;
                    rep = 3 + b.get(2);
                } else if (sym == 17) rep = 3 + b.get(3);
                else rep = 11 + b.get(7);
                if ((sym == 16 && idx == 0) || idx + rep > total) return INF_ST_DATA_ERROR; /* after the extra bits */
                for (uint32_t r = lane; r < rep; r += 32) lens[idx + r] = (uint8_t)val;
                idx += rep;
                prev = val;
            }
        }
        if (b.bits_left() < 0) return INF_ST_BUF_ERROR;
        __syncwarp();
        if (lens[256] == 0) return INF_ST_DATA_ERROR; /* no end-of-block code */
    }
    /* move into place: lit/len lengths at T.lens[0..], distance lengths right after */
    uint8_t tmp[10];
    for (int k = 0; k < 10; k++) {
        uint32_t i = lane + 32 * k;
        tmp[k] = i < nlit + ndist ? T.lens[32 + i] : 0;
    }
    __syncwarp();
    for (int k = 0; k < 10; k++) {
        uint32_t i = lane + 32 * k;
        if (i < 320) T.lens[i] = tmp[k];
    }
    __syncwarp();
    int l1 = inf_build(T.lens, (int)nlit, T.lcount, T.lsym, T.lit, INF_PB, INF_ALPHA_LITLEN, T.scratch);
    __syncwarp();
    int l2 = inf_build(T.lens + nlit, (int)ndist, T.dcount, T.dsym, T.dist, INF_DB, INF_ALPHA_DIST, T.scratch);
    __syncwarp();
    /* zlib: incomplete sets are only allowed when there is a single code (of length 1) */
    uint32_t usedl = nlit - T.lcount[0], usedd = ndist - T.dcount[0];
    if (l1 < 0 || l2 < 0 || (l1 > 0 && !(usedl == 1 && T.lcount[1] == 1)) || (l2 > 0 && usedd != 0 && !(usedd == 1 && T.dcount[1] == 1)))
        return INF_ST_DATA_ERROR;
    inf_mark_invalid(T, l1, l2);
    return 0;
}

/* ---- where decoded data goes (and where history is read back from) -------------------------------------------
 * put(p, v) stores one element at absolute position p; cursor(dst, dist) prepares a match copy: src(i) is the element
 * at dst - dist + i, put(i, v) stores at dst + i (32-bit offsets, the 64-bit address arithmetic is done once). */
struct OutBytes { /* final bytes in global memory, indexed by absolute output position */
    uint8_t *base;
    struct Cursor {
        uint8_t *d;
        const uint8_t *s;
        __device__ __forceinline__ uint32_t src(uint32_t i) const { return s[i]; }
        __device__ __forceinline__ void put(uint32_t i, uint32_t v) const { d[i] = (uint8_t)v; }
    };
    __device__ __forceinline__ void put(uint64_t p, uint32_t v) const { base[p] = (uint8_t)v; }
    __device__ __forceinline__ Cursor cursor(uint64_t dst, uint32_t dist) const { Cursor c; c.d = base + dst; c.s = c.d - dist; return c; }
    static constexpr uint32_t reach_before_start = 0; /* distances may not reach before absolute position 0 */
};
struct OutBytesWin { /* like OutBytes, but positions below `floor` are read from a resolved 32 KiB window */
    uint8_t *base;
    const uint8_t *win; /* win[32768 - k] = the byte k positions before `floor` */
    uint64_t floor;
    struct Cursor {
        uint8_t *d;
        const uint8_t *s;  /* source in the output buffer */
        const uint8_t *ws; /* source in the window for offsets below `nwin` */
        uint32_t nwin;
        __device__ __forceinline__ uint32_t src(uint32_t i) const { return i < nwin ? ws[i] : s[i]; }
        __device__ __forceinline__ void put(uint32_t i, uint32_t v) const { d[i] = (uint8_t)v; }
    };
    __device__ __forceinline__ void put(uint64_t p, uint32_t v) const { base[p] = (uint8_t)v; }
    __device__ __forceinline__ Cursor cursor(uint64_t dst, uint32_t dist) const {
        Cursor c;
        c.d = base + dst;
        c.s = c.d - dist;
        const uint64_t first = dst - dist; /* may lie before the floor (never before floor - 32768) */
        c.nwin = first < floor ? (uint32_t)(floor - first) : 0u;
        c.ws = win + 32768 - c.nwin;
        return c;
    }
    static constexpr uint32_t reach_before_start = 0;
};
struct OutSymRing { /* 16-bit symbols in a 65536-entry ring: < 256 literal byte, 0x8000|i = byte i of the unknown 32 KiB window */
    uint16_t *ring;
    struct Cursor {
        uint16_t *ring;
        uint32_t d0, s0;
        __device__ __forceinline__ uint32_t src(uint32_t i) const { return ring[(s0 + i) & 65535u]; }
        __device__ __forceinline__ void put(uint32_t i, uint32_t v) const { ring[(d0 + i) & 65535u] = (uint16_t)v; }
    };
    __device__ __forceinline__ void put(uint64_t p, uint32_t v) const { ring[(uint32_t)p & 65535u] = (uint16_t)v; }
    __device__ __forceinline__ Cursor cursor(uint64_t dst, uint32_t dist) const { Cursor c; c.ring = ring; c.d0 = (uint32_t)dst; c.s0 = c.d0 - dist; return c; }
    static constexpr uint32_t reach_before_start = 32768; /* relative positions: the window before 0 is legal history */
};

/* warp-cooperative LZ77 copy; every source element of one round is final before the round starts */
template <class Out>
__device__ __forceinline__ void inf_copy_match(const Out &o, uint64_t dst, uint32_t len, uint32_t dist) {
    const unsigned lane = lane_id();
    const typename Out::Cursor c = o.cursor(dst, dist);
    __syncwarp(); /* lane 0's literal stores are history now */
    if (dist >= len) {
        if (lane < len) c.put(lane, c.src(lane)); /* most matches are shorter than a warp */
        for (uint32_t i = lane + 32; i < len; i += 32) c.put(i, c.src(i));
    } else if (dist >= 32) {
        for (uint32_t done = 0; done < len; done += 32) {
            const uint32_t i = done + lane;
            if (i < len) c.put(i, c.src(i));
            __syncwarp();
        }
    } else { /* short period: every source lies before dst */
        for (uint32_t i = lane; i < len; i += 32) c.put(i, c.src(i % dist));
    }
    __syncwarp();
}

/* what a run of tokens ended with (bits 28..31 of the packed word; bits 16..24 match length, bits 0..15 distance - 1) */
enum { INF_EV_BUDGET = 0, INF_EV_MATCH = 1, INF_EV_EOB = 2, INF_EV_NEED_IN = 3, INF_EV_NEED_OUT = 4, INF_EV_DATA_ERR = 5, INF_EV_BUF_ERR = 6 };

/* Decode tokens until something other than a literal happens. ALL lanes run this loop over the same bits: control
 * flow stays uniform (no divergence, no broadcast of the result), only lane 0 stores the literals. CAREFUL: the
 * output window may not hold the next token -- decode exactly one and un-read it if it does not fit. */
template <class Out, bool CAREFUL>
__device__ __forceinline__ uint32_t inf_run(const Smem &sm, const InfTables &T, InfBits &b, const Out &o, uint64_t &out_pos, uint64_t out_end,
                                            uint32_t &budget) {
    const bool writer = lane_id() == 0;
    while (budget) {
        budget--;
        InfBits saved;
        if (CAREFUL) saved = b;
        uint32_t e = sm.ld32(INF_OFF_LIT + ((b.lo & ((1u << INF_PB) - 1u)) << 2));
        if (e) {
            b.drop(e & 15u);
            b.refill();
        } else {
            const int sym = inf_slow_decode(b.lo, T.lcount, T.lsym);
            if (sym < 0) return INF_EV_DATA_ERR << 28;
            b.drop((uint32_t)sym >> 16);
            b.refill();
            e = inf_entry(INF_ALPHA_LITLEN, (uint32_t)sym & 0xffffu, 0);
        }
        if ((e & 0x300u) == 0) { /* INF_K_LIT */
            if (CAREFUL && out_pos >= out_end) { b = saved; return INF_EV_NEED_OUT << 28; }
            if (writer) o.put(out_pos, e >> 16);
            out_pos++;
            continue;
        }
        const uint32_t kind = (e >> 8) & 3u;
        if (kind == INF_K_EOB) return INF_EV_EOB << 28;
        if (kind == INF_K_BAD) return INF_EV_DATA_ERR << 28;
        uint32_t eb = (e >> 4) & 15u;
        const uint32_t mlen = (e >> 16) + b.peek(eb);
        b.drop(eb); /* >= 27 bits remain: enough for any distance code */
        uint32_t de = sm.ld32(INF_OFF_DIST + ((b.lo & ((1u << INF_DB) - 1u)) << 2));
        if (de) {
            b.drop(de & 15u);
            b.refill();
        } else {
            const int ds = inf_slow_decode(b.lo, T.dcount, T.dsym);
            if (ds < 0) return INF_EV_DATA_ERR << 28;
            b.drop((uint32_t)ds >> 16);
            b.refill();
            de = inf_entry(INF_ALPHA_DIST, (uint32_t)ds & 0xffffu, 0);
        }
        if (((de >> 8) & 3u) == INF_K_BAD) return INF_EV_DATA_ERR << 28;
        eb = (de >> 4) & 15u;
        const uint32_t mdist = (de >> 16) + b.peek(eb);
        b.drop(eb);
        b.refill();
        if (CAREFUL && out_pos + mlen > out_end) { b = saved; return INF_EV_NEED_OUT << 28; }
        return (INF_EV_MATCH << 28) | (mlen << 16) | (mdist - 1u);
    }
    return INF_EV_BUDGET << 28;
}

/* Decode one stream window with one warp. `o` receives the output; positions are the absolute out_pos of the
 * state. stop(pos): asked at every block boundary (absolute bit position); true = return with why = BOUNDARY
 * (also after every block when the job asks for it). */
struct StopAtBit { /* stop at the first block boundary at or after an absolute bit position */
    uint64_t bit;
    __device__ __forceinline__ bool operator()(uint64_t pos) const { return pos >= bit; }
};

template <class Out, class Stop>
__device__ __forceinline__ void inf_decode_window(const InflateJob &job, InflateState *st, InfTables &T, const Out &o, const Stop &stop) {
    const unsigned lane = lane_id();
    InfBits b; /* identical in every lane */
    Smem sm;
    sm.init(reinterpret_cast<uint8_t *>(&T));
    uint64_t out_pos = st->out_pos;
    uint32_t phase = st->phase, last = st->last_block, stored_rem = st->stored_remaining;
    uint32_t nlit = st->nlit, ndist = st->ndist, blocks = st->blocks;
    int status = INF_ST_RUN, why = INF_WHY_NONE;
    const uint64_t out_end = job.out_base + job.out_cap;
    const uint64_t start_bit = st->in_bitpos - job.in_base * 8;
    const bool stop_each_block = (job.flags & INF_JOB_STOP_AT_BOUNDARY) != 0;
    uint32_t budget = 0; /* tokens that are known to fit the input and output windows */
    b.init(job.in, job.in_avail, start_bit);
    if (phase == INF_PH_CODES) { /* resume inside a Huffman block: rebuild the tables */
        for (int i = (int)lane; i < 320; i += 32) T.lens[i] = st->lens[i];
        __syncwarp();
        const int l1 = inf_build(T.lens, (int)nlit, T.lcount, T.lsym, T.lit, INF_PB, INF_ALPHA_LITLEN, T.scratch);
        const int l2 = inf_build(T.lens + nlit, (int)ndist, T.dcount, T.dsym, T.dist, INF_DB, INF_ALPHA_DIST, T.scratch);
        __syncwarp();
        inf_mark_invalid(T, l1, l2);
    }
    while (status == INF_ST_RUN && why == INF_WHY_NONE) {
        if (phase == INF_PH_HEADER) {
            /* a dynamic header is at most 14 + 57 + 320*(7+7) bits ~ 570 bytes: wait for it unless final */
            if (!job.in_final && b.bits_left() < 8 * 1024) { why = INF_WHY_INPUT; break; }
            if (b.bits_left() < 3) { status = INF_ST_BUF_ERROR; break; }
            last = b.get(1);
            const uint32_t type = b.get(2);
            if (type == 0) {
                b.drop(b.bc & 7); /* to byte boundary */
                b.refill();
                if (b.bits_left() < 32) { status = INF_ST_BUF_ERROR; break; }
                const uint32_t len = b.get(16), nlen = b.get(16);
                if ((len ^ 0xffffu) != nlen) { status = INF_ST_DATA_ERROR; break; }
                stored_rem = len;
                phase = INF_PH_STORED;
            } else if (type == 1) {
                __syncwarp();
                for (int i = (int)lane; i < 288; i += 32) T.lens[i] = i < 144 ? 8 : (i < 256 ? 9 : (i < 280 ? 7 : 8));
                T.lens[288 + lane] = 5; /* 32 distance codes: 30 and 31 decode (all 5 bits) as invalid, as in zlib */
                nlit = 288; ndist = 32;
                __syncwarp();
                inf_build(T.lens, 288, T.lcount, T.lsym, T.lit, INF_PB, INF_ALPHA_LITLEN, T.scratch);
                inf_build(T.lens + 288, 32, T.dcount, T.dsym, T.dist, INF_DB, INF_ALPHA_DIST, T.scratch);
                __syncwarp();
                phase = INF_PH_CODES;
            } else if (type == 2) {
                __syncwarp();
                const int err = inf_dynamic_header(b, T, nlit, ndist);
                if (err) { status = err; break; }
                phase = INF_PH_CODES;
            } else {
                status = INF_ST_DATA_ERROR;
                break;
            }
            budget = 0;
        } else if (phase == INF_PH_STORED) {
            /* raw copy, bounded by the input and output windows */
            const uint64_t ib = b.bitpos() >> 3; /* byte aligned here */
            uint64_t in_left = job.in_avail > ib ? job.in_avail - ib : 0;
            uint64_t out_left = out_end - out_pos;
            uint32_t n = stored_rem;
            if (n > in_left) n = (uint32_t)in_left;
            if (n > out_left) n = (uint32_t)out_left;
            for (uint32_t i = lane; i < n; i += 32) o.put(out_pos + i, job.in[ib + i]);
            __syncwarp();
            out_pos += n;
            stored_rem -= n;
            b.init(job.in, job.in_avail, (ib + n) * 8);
            budget = 0;
            if (stored_rem == 0) {
                phase = INF_PH_HEADER;
                blocks++;
                if (last) status = INF_ST_END;
            } else if (out_pos >= out_end) {
                why = INF_WHY_OUTPUT;
            } else if (job.in_final) {
                status = INF_ST_BUF_ERROR;
            } else {
                why = INF_WHY_INPUT;
            }
        } else { /* INF_PH_CODES: tokens until the block ends or a window limit is reached */
            /* a short match's bytes are LOADED when it is decoded and STORED when the next match arrives (or the loop
             * ends): the history read is an L2 round trip, and an in-order warp would otherwise sit on it */
            typename Out::Cursor pend_c;
            uint32_t pend_len = 0, pend_val = 0;
            for (;;) {
                uint32_t pk = INF_EV_BUDGET << 28;
                if (budget == 0) {
                    bool careful = false;
                    const int64_t left = b.bits_left();
                    if (left < 0) pk = INF_EV_BUF_ERR << 28; /* ran past the end of the stream */
                    else {
                        /* a token reads at most 48 bits and writes at most 258 bytes */
                        const uint64_t nin = job.in_final ? (uint64_t)(left >> 6) + 1u : (left < 192 ? 0u : (uint64_t)(left - 128) >> 6);
                        const uint64_t room = out_end - out_pos;
                        if (nin == 0) pk = INF_EV_NEED_IN << 28;
                        else if (room < 512 || (job.in_final && left < 192)) careful = true; /* token by token near either end */
                        else {
                            uint64_t n = room >> 9;
                            if (n > nin) n = nin;
                            budget = n > 65536u ? 65536u : (uint32_t)n;
                        }
                    }
                    if (careful) {
                        const uint64_t before = out_pos;
                        budget = 1;
                        pk = inf_run<Out, true>(sm, T, b, o, out_pos, out_end, budget);
                        budget = 0;
                        if (b.bits_left() < 0) { out_pos = before; pk = INF_EV_BUF_ERR << 28; } /* the token lay past the end of the stream */
                    }
                }
                if (budget) pk = inf_run<Out, false>(sm, T, b, o, out_pos, out_end, budget);
                const uint32_t ev = pk >> 28;
                if (ev == INF_EV_MATCH) {
                    const uint32_t mlen = (pk >> 16) & 0x1ffu, mdist = (pk & 0xffffu) + 1u;
                    if (mdist > out_pos + Out::reach_before_start) { status = INF_ST_DATA_ERROR; break; } /* too far back */
                    if (pend_len) { /* the previous match's bytes become history before anything new is read */
                        if (lane < pend_len) pend_c.put(lane, pend_val);
                        pend_len = 0;
                    }
                    if (mlen <= 32 && mdist >= mlen) {
                        pend_c = o.cursor(out_pos, mdist);
                        __syncwarp(); /* lane 0's literals and the store above are visible to the loads below */
                        if (lane < mlen) pend_val = pend_c.src(lane); /* predicated load straight into the carried register: no use of the value here */
                        pend_len = mlen;
                    } else {
                        inf_copy_match(o, out_pos, mlen, mdist);
                    }
                    out_pos += mlen;
                    continue;
                }
                if (ev == INF_EV_BUDGET) continue;
                if (ev == INF_EV_EOB) {
                    if (b.bits_left() < 0) { status = INF_ST_BUF_ERROR; break; } /* the end-of-block code lay past the end */
                    phase = INF_PH_HEADER;
                    blocks++;
                    if (last) status = INF_ST_END;
                } else if (ev == INF_EV_NEED_IN) {
                    why = INF_WHY_INPUT;
                } else if (ev == INF_EV_NEED_OUT) {
                    why = INF_WHY_OUTPUT;
                } else if (ev == INF_EV_DATA_ERR) {
                    status = INF_ST_DATA_ERROR;
                } else {
                    status = INF_ST_BUF_ERROR;
                }
                break;
            }
            if (pend_len) {
                if (lane < pend_len) pend_c.put(lane, pend_val);
                __syncwarp();
            }
        }
        if (phase == INF_PH_HEADER && status == INF_ST_RUN && why == INF_WHY_NONE) { /* at a block boundary */
            if (stop_each_block || stop(job.in_base * 8 + b.bitpos())) why = INF_WHY_BOUNDARY;
        }
    }
    /* ---- save state ------------------------------------------------------------------------------- */
    __syncwarp();
    if (phase == INF_PH_CODES && status == INF_ST_RUN)
        for (int i = (int)lane; i < 320; i += 32) st->lens[i] = T.lens[i];
    if (lane == 0) {
        uint64_t bp = b.bitpos();
        if (status == INF_ST_END) bp = (bp + 7) & ~7ull; /* the partial last byte is consumed */
        if (bp > b.avail_bits) { /* the decoder read past the input's end: a truncated stream, whatever those bits made it decide */
            bp = b.avail_bits;
            if (status < 0) status = INF_ST_BUF_ERROR;
        }
        st->in_bitpos = job.in_base * 8 + bp;
        st->out_pos = out_pos;
        st->status = status;
        st->why = why;
        st->phase = phase;
        st->last_block = last;
        st->stored_remaining = stored_rem;
        st->nlit = nlit;
        st->ndist = ndist;
        st->blocks = blocks;
    }
    __syncwarp();
}

/* the next unit of work for this warp: streams differ a lot in length, so warps pull indices from a counter instead
 * of striding (a second stride would leave most of the GPU waiting for the unlucky warps) */
__device__ __forceinline__ uint32_t inf_next_work(uint32_t *counter) {
    uint32_t k = 0;
    if (lane_id() == 0) k = atomicAdd(counter, 1u);
    return __shfl_sync(MZ_FULL_MASK, k, 0);
}

__global__ void __launch_bounds__(INF_THREADS) inflate_streams_kernel(const InflateJob *jobs, InflateState *states, uint32_t nstreams,
                                                                      uint32_t *work_counter) {
    MZ_DYN_SMEM(smem);
    InfTables &T = *reinterpret_cast<InfTables *>(smem);
    for (;;) {
        const uint32_t sidx = inf_next_work(work_counter);
        if (sidx >= nstreams) {
            /* the last warp out puts the counter pair back to zero: the launch needs no memset, and the slot is clean for its
             * next user (work_counter[1] counts the warps that have left; every CTA is one warp) */
            if (lane_id() == 0 && atomicAdd(work_counter + 1, 1u) == gridDim.x - 1) {
                work_counter[0] = 0;
                work_counter[1] = 0;
            }
            break;
        }
        const InflateJob job = jobs[sidx];
        InflateState *st = &states[sidx];
        if (st->status != INF_ST_RUN) continue;
        OutBytes o;
        o.base = job.out - job.out_base; /* index with absolute positions */
        inf_decode_window(job, st, T, o, StopAtBit{~0ull});
    }
}

} // namespace mzc
#endif
