/* deflate_kernel.cuh -- K2+K3 (v3): per-chunk LZ77 match + dynamic-Huffman RFC1951 encode (sm_90a).
 *
 * Replaces, on the write path, what zlib's deflate() does behind mz_stream_zlib_write /
 * mz_stream_zlib_close (mz_strm_zlib.c:203-240, :243-264, :280-305).  The compressed bytes are NOT
 * zlib's; parity = the reference inflate (mz_stream_zlib_read) reproduces the input bit-exactly.
 *
 * Work decomposition (one CTA of 512 threads per chunk, two CTAs resident per SM, chunks pulled from a
 * work counter):
 *   chunk      <= 64 KiB of input = one output slot, byte-aligned at both ends
 *   unit       <= 32 KiB of a chunk: one LZ77 domain (matches never leave it) resident in shared memory
 *              (TMA bulk load), normally coded as ONE DEFLATE block
 *   batch      4096 consecutive positions of a unit = 512 threads x 8-byte spans
 *   A match    LOCKSTEP, every position: hash of 4 bytes -> table of 8192 32-bit keys.  Per batch:
 *              read the old key | barrier | red.min(key = (7-batch)<<16 | position) | barrier | read the new
 *              key.  So the candidate of p is the first position of p's own batch with the same hash
 *              if that lies before p, else the first such position of the latest earlier batch that
 *              had one -- a function of the data alone: the output is bit-reproducible.  All 32 lanes
 *              verify their candidate against the next 8 bytes in lockstep (length 4..8, 8 = "or more")
 *   W walk     every thread walks its own 8 positions (static, predicated; one-step lazy rule; lengths
 *              capped at 8 are extended byte-exact only when the match is actually taken); at most 2
 *              matches start in a span; results parked in shared memory (2 words per span)
 *   B cover    exclusive prefix-max of the spans' end positions in position order: a span drops / trims
 *              what an earlier span's overrunning match already covers
 *   T tokens   every span turns what it keeps into entries of ONE ordered token list (16-bit, one
 *              entry per code word: literal byte | length symbol + extra | distance), placed by a block
 *              scan; literal / length / distance histograms by shared-memory atomics on the way
 *   D codes    block-parallel length-limited prefix codes (10 warps, named barrier)
 *   E+F emit   two batches at a time, every thread looks up its two spans' code words, which give the spans' sizes; one warp
 *              scan of both + one barrier + the pair's 16 warp totals place every span, which then packs its bits at that offset
 *              into the staging buffer (aliases the hash table). The block's total comes from the histograms in D, so whether
 *              the block is stored is known before this pass
 *   G flush    staging -> global in 16-byte units; partial tail carried into the next block
 * Blocks that would not shrink are emitted as stored blocks. A unit with more entries than the list
 * holds is coded as two blocks (batch halves). A non-final chunk ends with an empty stored block
 * (00 00 FF FF after bit padding) so chunks join byte-wise; the final chunk carries BFINAL.
 */
#ifndef MZ_DEFLATE_KERNEL_CUH
#define MZ_DEFLATE_KERNEL_CUH

#include "mzcuda_common.cuh"

namespace mzc {

constexpr int DF_THREADS = 512;
constexpr int DF_WARPS = DF_THREADS / 32;
constexpr int DF_CHUNK_MAX = 65536;
constexpr int DF_UNIT = 32768;                  /* LZ77 domain */
constexpr int DF_SB = DF_UNIT;                  /* (name kept for the slot bound) */
constexpr int DF_SPAN = 8;                      /* positions per thread per batch */
constexpr int DF_BATCH = DF_THREADS * DF_SPAN;  /* 4096 */
constexpr int DF_NBATCH = DF_UNIT / DF_BATCH;   /* 8 */
constexpr int DF_MINMATCH = 4;
constexpr int DF_LOCKLEN = 8;                   /* lockstep verification depth */
constexpr int DF_HASH_BITS = 13;
constexpr int DF_HASH_ENTRIES = 1 << DF_HASH_BITS; /* u32 keys: 32 KiB */
constexpr int DF_STAGE_WORDS = DF_UNIT / 4 + 64;
constexpr int DF_HDR_WORDS = 96;

constexpr uint32_t DF_FLAG_FINAL = 1u; /* chunk ends the stream: BFINAL on its last block, no sync marker */
constexpr uint32_t DF_FLAG_DICT = 2u;  /* the 32 KiB in front of the chunk (same buffer) belong to the same DEFLATE stream: the chunk may refer back
                                        * into them. Only the history variant of the kernel (levels 6-9) looks at it. */

/* shared-memory carve-up (bytes); two CTAs per SM: <= 113 KiB each */
constexpr int DF_OFF_IN = 0;
constexpr int DF_OFF_HASH = DF_OFF_IN + DF_UNIT + 64;
constexpr int DF_OFF_STAGE = DF_OFF_HASH;       /* bit staging aliases the hash table (dead after the parse) */
constexpr int DF_OFF_REC = DF_OFF_HASH + DF_STAGE_WORDS * 4; /* span records: 4096 x 2 words */
constexpr int DF_OFF_SPN = DF_OFF_REC + DF_NBATCH * DF_THREADS * 8; /* u16 per span: match extent -> cover */
constexpr int DF_SPAN_BYTES = DF_NBATCH * DF_THREADS * 10;
constexpr int DF_OFF_HIST = DF_OFF_REC + DF_SPAN_BYTES;      /* u32[288 + 32] */
constexpr int DF_OFF_HIST2 = DF_OFF_HIST + (288 + 32) * 4;   /* u32[256]: second copy of the literal counts (odd lanes) */
constexpr int DF_OFF_CODE = DF_OFF_HIST2 + 256 * 4;          /* u32[288 + 32]: code | len << 16 | extra bits << 20 */
constexpr int DF_OFF_LENS = DF_OFF_CODE + (288 + 32) * 4;    /* u8[288 + 32] code lengths (header) */
constexpr int DF_OFF_BITS = DF_OFF_LENS + (288 + 32);        /* u8[288 + 32] code length + extra bits */
constexpr int DF_OFF_SCAN = DF_OFF_BITS + (288 + 32);        /* u32[256]: block-scan scratch */
constexpr int DF_OFF_BB = DF_OFF_SCAN + 256 * 4;             /* u32[512] code-builder scratch */
constexpr int DF_OFF_MISC = DF_OFF_BB + 512 * 4;             /* u32[32] + mbarrier */
constexpr int DF_OFF_SINK = DF_OFF_MISC + 32 * 4 + 16;       /* u32[32]: one word per lane, the target of atomics that have nothing to do
                                                              * (ptxas branches around a predicated ATOMS; a select on the address is one instruction) */
constexpr int DF_OFF_LSYM = DF_OFF_SINK + 32 * 4;            /* u16[256]: length - 3 -> length symbol (0..28) | extra value << 5; filled once per CTA */
constexpr int DF_SMEM_BYTES = DF_OFF_LSYM + 256 * 2;
/* u8[16 warps][256]: during the parse and M0, each warp's list of its spans with a capped match (batch << 5 | lane). It lies on the
 * histograms, code words, lengths and bits: dead from the emit pass of the unit before until the histograms are cleared after M0. */
constexpr int DF_OFF_CAPL = DF_OFF_HIST;
static_assert(DF_OFF_CAPL + DF_WARPS * DF_NBATCH * 32 <= DF_OFF_SCAN, "capped-span lists fit in front of the scan scratch");
constexpr uint32_t DF_ZERO_SYM = 286;                        /* literal/length symbol that never occurs: its table entries are all zero */
static_assert(DF_HASH_ENTRIES * 4 <= DF_STAGE_WORDS * 4, "hash fits the staging region");
/* The history variant (template parameter HIST, levels 6-9): the previous 32 KiB -- the chunk's first unit, or with DF_FLAG_DICT the
 * bytes in front of the chunk -- stay resident in FRONT of the unit (offsets -32768 .. -1 relative to the standard carve-up, which is
 * unchanged) and the hash table, now 2^14 keys that survive from unit to unit, lies BEHIND it instead of under the bit staging:
 * 32 KiB + DF_SMEM_BYTES + 64 KiB = 208 KiB, one CTA per SM. Positions in the keys and candidates are relative to the start of the
 * previous unit (0 .. 65535). */
constexpr int DFH_PREV = 32768;
constexpr int DFH_HASH_BITS = 14;
constexpr int DFH_OFF_HASH = (DF_SMEM_BYTES + 15) & ~15;
constexpr int DFH_SMEM_BYTES = DFH_PREV + DFH_OFF_HASH + (4 << DFH_HASH_BITS);
static_assert(DFH_SMEM_BYTES <= 227 * 1024, "shared memory budget of the history variant");
static_assert(DF_SMEM_BYTES <= 113 * 1024, "shared memory budget for two CTAs per SM");

enum { MISC_CHUNK = 3, MISC_CARRY = 8 /* 4 words */ };

struct DeflateParams {
    const uint8_t *in;       /* device base of the uncompressed bytes */
    const uint64_t *in_off;  /* per-chunk byte offset into `in`, or NULL for a uniform partition */
    const uint32_t *in_len;  /* per-chunk length (<= 65536), or NULL */
    const uint8_t *flags;    /* per-chunk DF_FLAG_*, or NULL */
    uint64_t total_len;      /* uniform partition: total bytes */
    uint32_t chunk_size;     /* uniform partition: bytes per chunk (<= 65536) */
    uint32_t nchunks;
    uint32_t last_flags;     /* uniform partition: flags of the last chunk */
    int32_t level;           /* 0 stored, 1..9 */
    uint8_t *out;            /* slot i at out + i * slot_stride (16-byte aligned) */
    uint64_t slot_stride;
    uint32_t *out_len;       /* per-chunk compressed bytes */
    uint32_t *work_counter;  /* pair {next chunk, CTAs done}, zero at launch and left zero: CTAs take chunks dynamically (NULL = static striding) */
};

__host__ __device__ inline uint64_t deflate_slot_bound(uint32_t chunk_size) {
    /* stored worst case: 5 bytes per block, up to 2 blocks per 32 KiB unit, + sync marker + slack */
    return (((uint64_t)chunk_size + 12ull * ((chunk_size + DF_SB - 1) / DF_SB + 1) + 64 + 15) & ~15ull);
}

/* ---- symbol mapping (RFC1951 3.2.5) without tables ------------------------------------------- */
__device__ __forceinline__ void length_symbol(uint32_t len, uint32_t &sym, uint32_t &ebits, uint32_t &eval) {
    /* sym is 0..28 (add 257 for the alphabet index). Branch-free: for l = len - 3 >= 8, e = floor(log2 l) - 2 extra bits and
     * sym = 4 (e + 1) + the two bits below the leading one; l < 8 and len == 258 are patched in by selects. */
    const uint32_t l = len - 3;
    const uint32_t msb = 31u - (uint32_t)__clz((int)(l | 4u)); /* 2..7 */
    uint32_t e = msb - 2;
    uint32_t sy = 4 * (e + 1) + ((l >> e) & 3u);
    uint32_t ev = l & ((1u << e) - 1u);
    sy = l < 8 ? l : sy;           /* (for 4 <= l < 8 the formula already gives l; below 4 it does not) */
    const bool top = len == 258;
    sym = top ? 28u : sy;
    ebits = top ? 0u : e;
    eval = top ? 0u : ev;
}
/* d = distance - 1 (0..32767); branch-free: m = floor(log2(d | 1)), eb = max(m - 1, 0), sym = 2m + bit */
__device__ __forceinline__ void dist_symbol0(uint32_t d, uint32_t &sym, uint32_t &ebits) {
    uint32_t m = 31u - (uint32_t)__clz((int)(d | 1u));
    ebits = m > 0 ? m - 1 : 0u;
    sym = 2 * m + ((d >> ebits) & 1u);
}
__device__ __forceinline__ uint32_t len_extra_bits(uint32_t lsym) { return (lsym < 8 || lsym >= 28) ? 0u : (lsym >> 2) - 1; }
__device__ __forceinline__ uint32_t dist_extra_bits(uint32_t dsym) { return dsym < 4 ? 0u : (dsym >> 1) - 1; }

/* byte address of the staging word that holds bit `pos`, from the region base: pos >> 5 by a high multiply, so that both steps run
 * on the FMA pipe (a shift and a mask would be two integer-ALU instructions; the emit pass is bound by that pipe). The bit offset in
 * the word needs no mask either where it feeds a funnel shift, which takes the amount modulo 32. */
__device__ __forceinline__ uint32_t stage_word(uint32_t base, uint32_t pos, uint32_t k4) { return base + __umulhi(pos, 1u << 27) * k4; }

/* OR `n` (<=32) bits of v into the staging bit string at bit position pos */
__device__ __forceinline__ void stage_put(uint32_t *stage, uint32_t pos, uint32_t v, uint32_t n) {
    if (n == 0) return;
    if (n < 32) v &= (1u << n) - 1;
    uint32_t w = pos >> 5, s = pos & 31;
    atomicOr(&stage[w], v << s);
    if (s + n > 32) atomicOr(&stage[w + 1], v >> (32 - s));
}

/* OR n (<= 32) bits of v into the staging bit string at bit position pos (explicit shared-space form) */
__device__ __forceinline__ void stage_or(const Smem &sm, uint32_t pos, uint32_t v, uint32_t n) {
    const uint32_t sh = pos & 31u, wa = DF_OFF_STAGE + ((pos >> 5) << 2);
    sm.red_or32(wa, v << sh);
    if (sh + n > 32) sm.red_or32(wa + 4, v >> (32 - sh));
}

/* per-thread bit packer: every completed 32-bit word goes out by red.or (words at run borders are shared) */
struct BitWriter {
    Smem sm;
    uint64_t acc;
    uint32_t nb, wa; /* wa = byte offset of the current staging word */
    __device__ __forceinline__ void init(const Smem &s, uint32_t bitoff) {
        sm = s; wa = DF_OFF_STAGE + (bitoff >> 5) * 4; nb = bitoff & 31; acc = 0;
    }
    __device__ __forceinline__ void put(uint32_t v, uint32_t n) {
        acc |= (uint64_t)v << nb;
        nb += n;
        if (nb >= 32) { /* short body: predicated, no divergence */
            sm.red_or32(wa, (uint32_t)acc);
            acc >>= 32; nb -= 32; wa += 4;
        }
    }
    /* position of the next bit, relative to the start of the staging buffer */
    __device__ __forceinline__ uint32_t bitpos() const { return ((wa - (uint32_t)DF_OFF_STAGE) << 3) + nb; }
    __device__ __forceinline__ void finish() { /* nb may exceed 32 after a gap left for a match */
        if (nb > 0) sm.red_or32(wa, (uint32_t)acc);
        if (nb > 32) sm.red_or32(wa + 4, (uint32_t)(acc >> 32));
    }
};

/* ---- opt-in per-phase cycle counters (compile with -DMZ_DF_PHASES: `make phases`, read by tools/deflate_phases.py) ---------------
 * Thread 0 of every CTA reads clock64() right after the barrier that ends a phase and adds the cycles since its previous reading to
 * column `phase` of the CTA's row of g_df_phases (column DF_PH_UNITS counts the units). After a barrier every thread of the CTA is
 * done with the phase before, so the deltas are the CTA's wall time per phase; no barrier is added. Inside D the same marks split
 * the phase at its named barriers (thread 0 takes part in D) into the DF_PH_D_* columns, whose sum is at most D's; the rest of D
 * is the header. DF_PH_D_PASSES + n counts the units whose Kraft completion ran n passes (the last bucket: 7 or more). The parse
 * is split the same way at the two barriers of each batch (DF_PH_P_*: (a) up to the first: loads, hashes, reads of the table as
 * earlier batches left it; (b) up to the second: the inserts; (c) thread 0's own rest of the batch: reads after the insert,
 * verification, walk, record stores -- a batch's (a) includes the wait for the other warps' (c) of the batch before). M0 has no
 * barrier inside: its DF_PH_M_* columns are thread 0's time in the capped-span index, the near-source test and the extension
 * (whatever is left of M0 is waiting at its closing barrier for the other warps). The count-and-emit pass is split at its barrier
 * per pair of batches (DF_PH_X_*: (i) up to the barrier: the spans' code words, sizes and the warp scan -- a pair's (i) includes
 * the wait for the other warps' (ii) of the pair before; (ii) thread 0's own emit of the pair; (iii) M3). Without the macro (the product
 * library) and on the emulator the marks compile to nothing. */
enum { DF_PH_LOAD, DF_PH_PARSE, DF_PH_M0, DF_PH_COVER, DF_PH_T_M1, DF_PH_D, DF_PH_EMIT, DF_PH_FLUSH, DF_PH_UNITS,
       DF_PH_D_STATS, DF_PH_D_SWEEP1, DF_PH_D_SWEEP2, DF_PH_D_KRAFT, DF_PH_D_CANON, DF_PH_D_PASSES,
       DF_PH_P_A = DF_PH_D_PASSES + 8, DF_PH_P_B, DF_PH_P_C, DF_PH_M_INDEX, DF_PH_M_NEAR, DF_PH_M_EXTEND, DF_PH_X_SCAN, DF_PH_X_EMIT,
       DF_PH_X_M3, DF_PH_COLS };
constexpr int DF_PH_ROWS = 1024;
#if defined(MZ_DF_PHASES) && !defined(MZ_EMU)
__device__ unsigned long long g_df_phases[DF_PH_ROWS][DF_PH_COLS];
#define DF_PHASE_BEGIN(t) unsigned long long t = clock64()
#define DF_PHASE(t, ph)                                                                        \
    do {                                                                                       \
        if (threadIdx.x == 0 && blockIdx.x < (unsigned)DF_PH_ROWS) {                           \
            const unsigned long long now_ = clock64();                                         \
            atomicAdd(&g_df_phases[blockIdx.x][ph], now_ - (t));                               \
            if ((ph) == DF_PH_LOAD) atomicAdd(&g_df_phases[blockIdx.x][DF_PH_UNITS], 1ull);   \
            (t) = now_;                                                                        \
        }                                                                                      \
    } while (0)
#define DF_PHASE_COUNT(col)                                                                                          \
    do {                                                                                                             \
        if (threadIdx.x == 0 && blockIdx.x < (unsigned)DF_PH_ROWS) atomicAdd(&g_df_phases[blockIdx.x][col], 1ull); \
    } while (0)
#else
#define DF_PHASE_BEGIN(t)
#define DF_PHASE(t, ph)
#define DF_PHASE_COUNT(col)
#endif

/* ---- D: block-parallel literal/length + distance codes ------------------------------------------------
 * Thread i < 288 owns literal/length symbol i (286 used), thread 288 + j owns distance symbol j (30 used);
 * both alphabets are warp aligned (warps 0-8 and warp 9). Called by threads 0..319 ONLY; they synchronise
 * among themselves on named barrier 1 so the other warps are not dragged through a dozen barriers.
 * bb = 512 words of shared scratch. Outputs lens (u8), codes (reversed code | len << 16 | extra bits << 20)
 * and bits (u8: code length + extra bits = what one entry of that symbol costs). */
constexpr int DF_BB_THREADS = 320;
enum { BB_STAT = 0 /* [2][4]: used,total,first */, BB_KRAFT = 8 /* [2 sweeps][2 alph][16] */, BB_SLACK = 136 /* [2] */,
       BB_CNTW = 144 /* [2 bufs][10 warps][16]: codes per length in a warp, then what a code's rank in its warp is set against */,
       BB_NZ = 464 /* [10] ballots: length != 0 */, BB_ST = 474 /* [10] ballots: a run of equal lengths starts here */,
       BB_HSUM = 484 /* [10] header bits per warp */, BB_HDRBITS = 494 /* size of the block header in bits */,
       BB_TOKBITS = 495 /* bits of the block's code words and extra bits, end of block left out */, BB_TOKW = 496 /* [10] the same per warp */ };

/* ---- block header (RFC 1951 3.2.7): HLIT/HDIST trimmed, code lengths run-length coded (symbols 16/17/18) under a STATIC
 * code-length code. A code chosen per block would save another 0.01-0.09 % of the input (tools/sim/lzsim hdr=0 vs hdr=3) and cost
 * a third code construction on the critical path. The static code is complete (Kraft sum exactly 1; zlib's inflate rejects
 * anything else) and gives every one of the 19 symbols a code, so any length 1..15 can be sent:
 *   3 bits: lengths 7 8 9 | 4 bits: 0 5 6 10 11 and run symbol 18 | 5 bits: 3 4 12 13, 16, 17 | 6 bits: 1 2 14 15.
 * Packed per symbol 0..18: CL_LENS 3 bits each; CL_CODE_* the canonical codes bit-reversed (sent LSB first), 6 bits each;
 * CL_ORDER57 the nineteen 3-bit lengths in the header's transmission order 16,17,18,0,8,7,9,6,10,5,11,4,12,3,13,2,14,1,15. */
constexpr uint64_t CL_LENS = 0x12ddad91b725bb4ull;
constexpr uint64_t CL_CODE_LO = 0x840013930ef3c6ull, CL_CODE_HI = 0xd5c7fdf6cb149ull;
constexpr uint64_t CL_ORDER57 = 0x1b6d6db248db92dull;
__device__ __forceinline__ uint32_t cl_len(uint32_t s) { return (uint32_t)(CL_LENS >> (3 * s)) & 7u; }
__device__ __forceinline__ uint32_t cl_code(uint32_t s) {
    return s < 10 ? (uint32_t)(CL_CODE_LO >> (6 * s)) & 63u : (uint32_t)(CL_CODE_HI >> (6 * (s - 10))) & 63u;
}

__device__ __forceinline__ void bb_count_lengths(uint32_t *cntw_row, uint32_t L, unsigned lane, unsigned &m) {
    if (lane < 16) cntw_row[lane] = 0;
    __syncwarp();
    m = __match_any_sync(MZ_FULL_MASK, L);
    if (L > 0 && lane == (unsigned)(__ffs((int)m) - 1)) cntw_row[L] = (uint32_t)__popc(m);
    __syncwarp();
}

__device__ inline void block_build_codes(const uint32_t *hist_ll, const uint32_t *hist_lit2, const uint32_t *hist_d, uint8_t *lens_ll, uint8_t *lens_d,
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
    DF_PHASE_BEGIN(d_t);

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
    DF_PHASE(d_t, DF_PH_D_STATS);
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
            uint32_t mine = 0; /* lane cnd < 16 keeps the warp's Kraft sum for candidate cnd */
#pragma unroll
            for (int cnd = 0; cnd < 16; cnd++) {
                uint32_t kr = 0;
                if (c) {
                    int l = (int)ceilf(ideal - (lo + step * (float)cnd));
                    l = l < 1 ? 1 : (l > M ? M : l);
                    kr = 1u << (M - l);
                }
                kr = __reduce_add_sync(MZ_FULL_MASK, kr);
                mine = lane == (unsigned)cnd ? kr : mine;
            }
            if (lane < 16) atomicAdd(&bb[BB_KRAFT + sweep * 32 + a * 16 + lane], mine); /* one shared atomic per warp and sweep */
        }
        bar_sync(1, DF_BB_THREADS);
        DF_PHASE(d_t, DF_PH_D_SWEEP1 + sweep);
        /* Every warp derives both alphabets' choices (uniform): the largest candidate in 1..15 whose Kraft sum is at most 1, else
         * 0. Lane l holds the sum of candidate l & 15 of alphabet l >> 4, so a ballot of "fits" and its highest bit per half give
         * the same `best` as scanning the candidates upwards and keeping the last that fits -- whatever the order of the sums.
         * (They do not decrease with the candidate anyway: lo + step * cnd is an exact binary fraction that grows with cnd, so
         * every length only shrinks.) */
        const uint32_t kl = bb[BB_KRAFT + sweep * 32 + lane];
        const unsigned fit = __ballot_sync(MZ_FULL_MASK, (lane & 15u) != 0 && kl <= one);
        const int best0 = (fit & 0xffffu) ? 31 - __clz((int)(fit & 0xffffu)) : 0;
        const int best1 = (fit >> 16) ? 31 - __clz((int)(fit >> 16)) : 0;
        slack[0] = one - __shfl_sync(MZ_FULL_MASK, kl, best0);
        slack[1] = one - __shfl_sync(MZ_FULL_MASK, kl, 16 + best1);
        /* lo is per alphabet from here on; the loop variable is private to the thread */
        lo = lo + step * (float)(a == 0 ? best0 : best1);
        step *= 0.0625f;
    }
    uint32_t L = 0;
    if (c) {
        int l = (int)ceilf(ideal - lo);
        L = (uint32_t)(l < 1 ? 1 : (l > M ? M : l));
    }
    /* exact Kraft completion: shorten codes (short ones first) until the sum is exactly 1. A pass that leaves no slack in either
     * alphabet also lays out the canonical codes (below), so the usual case -- one pass -- needs no second count and no more
     * barriers. */
    unsigned m = 0;
    int buf = 0, pass = 0;
    bool settled = false;
    for (; pass < 40; pass++) {
        if (slack[0] == 0 && slack[1] == 0) break;
        uint32_t *cntw = bb + BB_CNTW + buf * 160, *nxt = bb + BB_CNTW + (buf ^ 1) * 160;
        if (a < 2) bb_count_lengths(cntw + w * 16, L, lane, m);
        bar_sync(1, DF_BB_THREADS);
        if (w == 0 || w == 9) { /* one warp per alphabet: lane = code length; the recurrence over lengths is uniform */
            const int aa = w == 0 ? 0 : 1;
            const uint32_t wa = aa == 0 ? 0u : 9u, wb = aa == 0 ? 9u : 10u;
            const bool mine = lane >= 1 && lane <= (unsigned)M;
            uint32_t P[9], tot = 0; /* P[i] = the count in the warps before warp wa + i (all nine loads in flight at once) */
#pragma unroll
            for (int i = 0; i < 9; i++) {
                const uint32_t t = (mine && wa + i < wb) ? cntw[(wa + i) * 16 + lane] : 0u;
                P[i] = tot;
                tot += t;
            }
            uint32_t sl = slack[aa], myk = 0;
            for (int len = 2; len <= M; len++) {
                uint32_t t = __shfl_sync(MZ_FULL_MASK, tot, len);
                uint32_t can = sl >> (M - len);
                uint32_t k = t < can ? t : can;
                if (lane == (unsigned)len) myk = k;
                sl -= k << (M - len);
            }
            /* The codes per length after this pass: k[len] leave length len, k[len + 1] arrive from len + 1. Their canonical first
             * codes, in case this pass is the last. */
            const uint32_t kup = __shfl_down_sync(MZ_FULL_MASK, myk, 1);
            const uint32_t tot2 = mine ? tot - myk + kup : 0u;
            uint32_t code = 0, prev = 0, mycode = 0;
            for (int len = 1; len <= M; len++) {
                code = (code + prev) << 1;
                if (lane == (unsigned)len) mycode = code;
                prev = __shfl_sync(MZ_FULL_MASK, tot2, len);
            }
            /* Per warp ww and length: k - P (a code of that length in warp ww whose rank in its warp is below it is one of the
             * first k of its length in symbol order, the ones to shorten), and into the other buffer the first code of the length
             * after the pass + the codes of that length in the warps before ww after the pass: P - min(k, P) that stay and
             * min(k[len + 1], P[len + 1]) that arrive. */
#pragma unroll
            for (int i = 0; i < 9; i++) {
                const uint32_t Pup = __shfl_down_sync(MZ_FULL_MASK, P[i], 1);
                if (mine && wa + i < wb) {
                    cntw[(wa + i) * 16 + lane] = myk - P[i];
                    nxt[(wa + i) * 16 + lane] = mycode + P[i] - (myk < P[i] ? myk : P[i]) + (kup < Pup ? kup : Pup);
                }
            }
            if (lane == 0) bb[BB_SLACK + aa] = sl;
        }
        bar_sync(1, DF_BB_THREADS);
        if (a < 2 && L >= 2) {
            const int rank = __popc(m & ((1u << lane) - 1));
            if (rank < (int)cntw[w * 16 + L]) L -= 1;
        }
        slack[0] = bb[BB_SLACK + 0];
        slack[1] = bb[BB_SLACK + 1];
        buf ^= 1;
        if (slack[0] == 0 && slack[1] == 0) {
            settled = true;
            pass++;
            break;
        }
    }
    DF_PHASE(d_t, DF_PH_D_KRAFT);
    DF_PHASE_COUNT(DF_PH_D_PASSES + (pass < 7 ? pass : 7));
    /* canonical codes: code = first code of its length + rank among equal lengths in symbol order; the rows of cntw hold the
     * first code + the count in the warps before */
    uint32_t *cntw = bb + BB_CNTW + buf * 160;
    if (settled) { /* laid out by the last pass; only the rank in the warp is left */
        if (a < 2) m = __match_any_sync(MZ_FULL_MASK, L);
    } else { /* no pass ran, or none left both alphabets without slack */
        if (a < 2) bb_count_lengths(cntw + w * 16, L, lane, m);
        bar_sync(1, DF_BB_THREADS);
        if (w == 0 || w == 9) {
            const int aa = w == 0 ? 0 : 1;
            const uint32_t wa = aa == 0 ? 0u : 9u, wb = aa == 0 ? 9u : 10u;
            const bool mine = lane >= 1 && lane <= (unsigned)M;
            uint32_t tot = 0;
            if (mine)
                for (uint32_t ww = wa; ww < wb; ww++) {
                    const uint32_t t = cntw[ww * 16 + lane];
                    cntw[ww * 16 + lane] = tot;
                    tot += t;
                }
            uint32_t code = 0, prev = 0, mycode = 0;
            for (int len = 1; len <= M; len++) {
                code = (code + prev) << 1;
                if (lane == (unsigned)len) mycode = code;
                prev = __shfl_sync(MZ_FULL_MASK, tot, len);
            }
            if (mine)
                for (uint32_t ww = wa; ww < wb; ww++) cntw[ww * 16 + lane] += mycode;
        }
        bar_sync(1, DF_BB_THREADS);
    }
    if (a < 2) {
        uint32_t cw = 0;
        if (L) {
            const uint32_t code = cntw[w * 16 + L] + (uint32_t)__popc(m & ((1u << lane) - 1));
            cw = (__brev(code) >> (32 - L)) | (L << 16);
        }
        /* The block's token bits: count x (code length + extra bits) over both alphabets, end of block left out. The histograms
         * count exactly the symbols the emit pass writes, so this is the sum of the span sizes there. (The counts are read again:
         * c may hold a count forced to 1 above.) */
        uint32_t tb;
        if (a == 0) {
            const uint32_t eb = sym >= 257 ? len_extra_bits(sym - 257) : 0u;
            lens_ll[sym] = (uint8_t)L; /* sym up to 287: entries 286, 287 get 0 */
            code_ll[sym] = cw | (eb << 20);
            bits_ll[sym] = (uint8_t)(L + eb);
            tb = sym == 256 ? 0u : (hist_ll[sym] + (sym < 256 ? hist_lit2[sym] : 0u)) * (L + eb); /* (286, 287: count 0) */
        } else {
            lens_d[sym] = (uint8_t)L;  /* sym up to 31 */
            code_d[sym] = cw;          /* distance extra bits come from the entry, not the table */
            bits_d[sym] = (uint8_t)(L + dist_extra_bits(sym));
            tb = hist_d[sym] * (L + dist_extra_bits(sym)); /* (30, 31: count 0) */
        }
        tb = __reduce_add_sync(MZ_FULL_MASK, tb);
        if (lane == 0) bb[BB_TOKW + w] = tb;
    }
    /* ---- the block header, written straight into the (clean) staging buffer at bit hdrpos. One thread per code length;
     * runs of equal lengths are found from per-warp ballots (a run never crosses from the literal/length lengths into the
     * distance lengths: the RFC allows it, zlib never writes it, so neither do we). ---- */
    const unsigned nz = __ballot_sync(MZ_FULL_MASK, L != 0);
    if (lane == 0) bb[BB_NZ + w] = nz;
    bar_sync(1, DF_BB_THREADS);
    DF_PHASE(d_t, DF_PH_D_CANON);
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
        uint32_t tok = 0;
        for (uint32_t ww = 0; ww < 10; ww++) tok += bb[BB_TOKW + ww];
        bb[BB_TOKBITS] = tok;
    }
    if (tid == 32) stage_put(stage, hdrpos + 17, (uint32_t)CL_ORDER57, 32);
    if (tid == 64) stage_put(stage, hdrpos + 17 + 32, (uint32_t)(CL_ORDER57 >> 32), 25);
}

/* ---- A: match helpers ----------------------------------------------------------------------------------- */
/* in[q..] against in[c..] agree for 8 bytes already; extend to at most maxlen bytes (both inside the unit) */
__device__ __forceinline__ uint32_t extend_match8(const Smem &sm, uint32_t c, uint32_t q, uint32_t maxlen) {
    uint32_t len = 8;
    while (len < maxlen) {
        uint32_t x = sm.ld32u(DF_OFF_IN, q + len) ^ sm.ld32u(DF_OFF_IN, c + len);
        if (x) {
            len += (uint32_t)(__ffs((int)x) - 1) >> 3;
            break;
        }
        len += 4;
    }
    return len < maxlen ? len : maxlen;
}

/* p ? a : b as one SEL: left to itself, ptxas branches around the few instructions that compute a */
__device__ __forceinline__ uint32_t sel_u32(bool p, uint32_t a, uint32_t b) {
#ifdef MZ_EMU
    return p ? a : b;
#else
    uint32_t r;
    asm("{\n.reg .pred q;\nsetp.ne.u32 q, %3, 0;\nselp.b32 %0, %1, %2, q;\n}" : "=r"(r) : "r"(a), "r"(b), "r"((uint32_t)p));
    return r;
#endif
}

/* The constant 4 as a value the compiler cannot see (the kernel always runs DF_THREADS threads per CTA): an address `i * k4 + base`
 * stays one IMAD on the FMA pipe, where `i * 4 + base` would become a LEA on the integer-ALU pipe -- the pipe this kernel is bound
 * by. (A constant behind an inline-asm mov would not do: ptxas folds it.) */
__device__ __forceinline__ uint32_t opaque4() { return blockDim.x / (uint32_t)(DF_THREADS / 4); }

template <bool HIST>
__device__ __forceinline__ uint32_t hash_addr(uint32_t v, uint32_t k4) { /* byte offset of the key of 4-byte value v; k4 = opaque4() */
    /* the top bits of v * 2654435761 by a high multiply, then * 4: all on the FMA pipe (a shift and a mask would be two integer-ALU
     * instructions) */
    return (HIST ? DFH_OFF_HASH : DF_OFF_HASH) + __umulhi(v * 2654435761u, 1u << (HIST ? DFH_HASH_BITS : DF_HASH_BITS)) * k4;
}

/* span record (two words, parked in the token region during the parse):
 *   A = j0 | (L0 - 3) << 3 | (d0 - 1) << 11 | (lit & 63) << 26      first match: start offset, length, distance - 1
 *   B = j1 | (L1 - 3) << 3 | (d1 - 1) << 11 | (lit >> 6) << 26      second match; (L - 3) == 0 means none
 * lit = the span's positions coded as literals. */
__device__ __forceinline__ uint32_t rec_len(uint32_t r) { uint32_t l = (r >> 3) & 255u; return l ? l + 3 : 0u; }

/* What a span keeps once the cover is known, in final form (three words, computed once):
 *   F  = lit (bits 0-7: positions kept as literals) | ex << 8 (0..2 bytes that a match trimmed below 3 bytes leaves behind;
 *        they come first) | first such byte << 16 | second << 24
 *   MA, MB = the up to two matches, each whole or trimmed at the front: bit 31 valid | P (bits 0-2: the in-span position
 *        the match is ordered at: literals below it come first; 8 -> 0, then there are no literals) | (len - 3) << 4
 *        | (dist - 1) << 12; match_symbols() turns them into symbol form */
__device__ __forceinline__ uint32_t fin_len(uint32_t m) { return ((m >> 4) & 255u) + 3u; }
__device__ __forceinline__ uint32_t fin_dist(uint32_t m) { return ((m >> 12) & 0x7fffu) + 1u; }
template <bool ONEM>
__device__ __forceinline__ void span_classify(const Smem &sm, uint32_t A, uint32_t B, uint32_t q0, uint32_t cover, uint32_t &F, uint32_t &MA,
                                              uint32_t &MB) {
    const uint32_t lit = (A >> 26) | ((B >> 26) << 6);
    const uint32_t crel = cover > q0 ? cover - q0 : 0u;
    const uint32_t cr8 = crel < 8 ? crel : 8u;
    uint32_t ex = 0;
    MA = MB = 0; /* (scalars, not an array: an array of two ends up in local memory) */
#pragma unroll
    for (int r = 0; r < (ONEM ? 1 : 2); r++) {
        /* The match keeps what lies at or behind s = max(start, cover): Lf = end - s bytes, none when the cover reaches its end
         * (an empty record has end = start). Kept whole (s = start) it has at least 4; trimmed, 3 or more stay a match (ordered
         * at the cover's slot, min(s, 8) & 7) and 1 or 2 become the leftover literals. */
        const uint32_t R = r == 0 ? A : B;
        const uint32_t j = R & 7u, end = j + rec_len(R);
        const uint32_t s = j > crel ? j : crel;
        const uint32_t Lf = (end > s ? end : s) - s;
        const uint32_t P = (s < 8u ? s : 8u) & 7u;
        const uint32_t M = Lf >= 3 ? (((Lf << 4) + (0x80000000u - (3u << 4))) | P | ((R << 1) & (0x7fffu << 12))) : 0u;
        if (r == 0) MA = M;
        else MB = M;
        ex = Lf - 1u < 2u ? Lf : ex;
    }
    F = ((lit >> cr8) << cr8) | (ex << 8);
    if (ex) { /* rare: fetch the leftover bytes now, the write pass then needs nothing but F */
        const uint32_t p = DF_OFF_IN + q0 + crel;
        F |= sm.ld8(p) << 16;
        if (ex == 2) F |= sm.ld8(p + 1) << 24;
    }
}

/* final match record (P | len | dist form) -> symbol form, counting its two symbols on the way:
 *   bit 31 valid | P << 28 (3 bits; 8 -> 0: then the span has no literals, so the order does not matter)
 *   | distance extra value << 15 (13 bits) | distance symbol << 10 | length extra value << 5 | length symbol (0..28) */
__device__ __forceinline__ uint32_t match_symbols(const Smem &sm, uint32_t M) {
    uint32_t ds, db;
    const uint32_t lsv = sm.ld16(DF_OFF_LSYM + ((M >> 3) & 0x1feu)); /* length symbol | extra value << 5, by length - 3 */
    const uint32_t d = fin_dist(M) - 1;
    dist_symbol0(d, ds, db);
    sm.red_add32(DF_OFF_HIST + (257u + (lsv & 31u)) * 4, 1u);
    sm.red_add32(DF_OFF_HIST + (288u + ds) * 4, 1u);
    return 0x80000000u | ((M & 7u) << 28) | ((d & ((1u << db) - 1u)) << 15) | (ds << 10) | lsv;
}
/* bits a match costs (both code words with their extra bits); 0 for an empty record */
__device__ __forceinline__ uint32_t match_bits(const Smem &sm, uint32_t M) {
    const uint32_t n = sm.ld8(DF_OFF_BITS + 257u + (M & 31u)) + sm.ld8(DF_OFF_BITS + 288u + ((M >> 10) & 31u));
    return M ? n : 0u;
}
/* OR the <= 48 bits of a match (symbol form) into the staging bit string at bit position pos */
__device__ __forceinline__ void put_match_bits(const Smem &sm, uint32_t pos, uint32_t M) {
    const uint32_t cwl = sm.ld32(DF_OFF_CODE + (257u + (M & 31u)) * 4);
    const uint32_t cwd = sm.ld32(DF_OFF_CODE + (288u + ((M >> 10) & 31u)) * 4);
    const uint32_t cl = (cwl >> 16) & 15u, cd = (cwd >> 16) & 15u;
    const uint32_t v1 = (cwl & 0x7fffu) | (((M >> 5) & 31u) << cl);          /* <= 15 + 5 bits */
    const uint32_t n1 = cl + ((cwl >> 20) & 15u);
    const uint32_t v2 = (cwd & 0x7fffu) | (((M >> 15) & 0x1fffu) << cd);     /* <= 15 + 13 bits */
    const uint64_t V = (uint64_t)v1 | ((uint64_t)v2 << n1);
    const uint32_t lo = (uint32_t)V, hi = (uint32_t)(V >> 32);
    const uint32_t wa = stage_word(DF_OFF_STAGE, pos, opaque4());
    const uint32_t w0 = __funnelshift_l(0u, lo, pos), w1 = __funnelshift_l(lo, hi, pos), w2 = __funnelshift_l(hi, 0u, pos);
    sm.red_or32(wa, w0);
    sm.red_or32(wa + 4, w1);
    if (w2) sm.red_or32(wa + 8, w2);
}

/* The k-th (0-based) set bit over the eight ballot words bm[0..7] of this warp -> the span index b * 512 + warp * 32 + lane it
 * stands for; 0xffffffff when there are fewer. (Once or twice per unit and warp: a popcount walk + a 5-step binary search.) */
__device__ __forceinline__ uint32_t nth_parked(const uint32_t (&bm)[DF_NBATCH], uint32_t k, uint32_t warp) {
    uint32_t r = k, word = 0, bsel = 0;
    bool found = false;
#pragma unroll
    for (int b = 0; b < DF_NBATCH; b++) {
        const uint32_t c = (uint32_t)__popc(bm[b]);
        const bool here = !found && r < c;
        word = here ? bm[b] : word;
        bsel = here ? (uint32_t)b : bsel;
        found = found || here;
        r -= found ? 0u : c;
    }
    uint32_t base = 0;
#pragma unroll
    for (int st = 16; st; st >>= 1) {
        const uint32_t c = (uint32_t)__popc((word >> base) & ((1u << st) - 1u));
        const bool up = r >= c;
        r -= up ? c : 0u;
        base += up ? (uint32_t)st : 0u;
    }
    return found ? bsel * (uint32_t)DF_THREADS + warp * 32u + base : 0xffffffffu;
}

/* The count-and-emit pass, first half: a span's code words looked up once (a position that is not a literal looks up the
 * all-zero entry: no selects on the results). Their lengths, packed one per byte, and the sizes of the span's matches (added
 * to the byte of the slot they are ordered at) give every bit offset in the span by ONE multiplication per word: byte k of
 * w * 0x01010101 is the sum of bytes 0..k of w (no byte overflows: 8 x 15 + 2 x 48 < 256), and the top byte of P1 is the sum
 * of all eight. Kept for the write, no more: the four literal pairs packed for one OR each (at most the two literals of a pair
 * are in-band, and then they are adjacent: a match start covers its neighbour), the offsets of the slots (E0, E1: byte k = bits
 * before slot k), the 1 or 2 leftover bytes' code words (xv; they come first) with their bit count and both matches' offsets
 * (offs), the first match, the span's size (<= 30 + 216 bits; 0 only for a span that holds nothing). */
struct SpanBits {
    uint32_t v[4], E0, E1, offs, xv, MA, size;
};
template <bool ONEM>
__device__ __forceinline__ SpanBits span_bits(const Smem &sm, uint32_t sidx, uint32_t F, uint32_t MA, uint32_t MB, uint32_t code_base, uint32_t zero_ent,
                                              uint32_t k4) {
    SpanBits s;
    const uint2 x = sm.ld64(DF_OFF_IN + sidx * DF_SPAN);
    uint32_t xn = 0;
    s.xv = 0;
    const uint32_t ex = (F >> 8) & 3u;
    if (ex) {
        const uint32_t c0 = sm.ld32(DF_OFF_CODE + ((F >> 16) & 0xffu) * 4);
        s.xv = c0 & 0x7fffu;
        xn = (c0 >> 16) & 15u;
        if (ex == 2) {
            const uint32_t c1 = sm.ld32(DF_OFF_CODE + (F >> 24) * 4);
            s.xv |= (c1 & 0x7fffu) << xn;
            xn += (c1 >> 16) & 15u;
        }
    }
    uint32_t cw[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const uint32_t by = MZ_BYTE(j < 4 ? x.x : x.y, j & 3);
        cw[j] = sm.ld32_a(((F >> j) & 1u) ? by * k4 + code_base : zero_ent); /* code | length << 16 (a literal's entry has no extra-bits field) */
    }
    /* lengths, one per byte; a match leaves a gap of its size at its slot (slot 8 = none: the shifts clamp to 0) */
    const uint32_t nA = match_bits(sm, MA), nB = ONEM ? 0u : match_bits(sm, MB);
    const uint32_t sA = MA ? ((MA >> 28) & 7u) * 8u : 64u, sB = MB ? ((MB >> 28) & 7u) * 8u : 64u;
    const uint32_t L0 = __byte_perm(__byte_perm(cw[0], cw[1], 0x0062u), __byte_perm(cw[2], cw[3], 0x0062u), 0x5410u) + shl_clamp(nA, sA) + shl_clamp(nB, sB);
    const uint32_t L1 = __byte_perm(__byte_perm(cw[4], cw[5], 0x0062u), __byte_perm(cw[6], cw[7], 0x0062u), 0x5410u) + shl_clamp(nA, sA - 32u) + shl_clamp(nB, sB - 32u);
    const uint32_t P0 = L0 * 0x01010101u;                       /* inclusive sums of slots 0..3 */
    const uint32_t P1 = L1 * 0x01010101u + (P0 >> 24) * 0x01010101u;
    s.E0 = P0 << 8;
    s.E1 = __funnelshift_l(P0, P1, 8); /* exclusive: bits before slot k in byte k */
#pragma unroll
    for (int jj = 0; jj < 4; jj++) {
        const uint32_t c0 = cw[2 * jj], c1 = cw[2 * jj + 1];
        s.v[jj] = (c0 & 0xffffu) | ((c1 & 0xffffu) << (c0 >> 16));
    }
    /* the leftover bytes' bits | the first match's offset << 8 | the second's << 16 (each < 256) */
    s.offs = xn + (((shr_clamp(s.E0, sA) & 0xffu) + (shr_clamp(s.E1, sA - 32u) & 0xffu)) << 8) +
             (((shr_clamp(s.E0, sB) & 0xffu) + (shr_clamp(s.E1, sB - 32u) & 0xffu)) << 16);
    s.MA = MA;
    s.size = xn + (P1 >> 24);
    return s;
}
/* ... second half: the span's bits at bit position pos of the staging buffer. Two literals go out per OR of <= 30 bits; both
 * target words unconditionally (an OR of zero is cheaper than the branches around it). The first match is OR-ed in here, the
 * second one's position is parked next to its record (span sidx) for the M3 pass. */
template <bool ONEM>
__device__ __forceinline__ void span_emit(const Smem &sm, const SpanBits &s, uint32_t pos, uint32_t sidx, uint32_t stage_base, uint32_t k4) {
    const uint32_t xn = s.offs & 0xffu;
    if (xn) stage_or(sm, pos, s.xv, xn);
    pos += xn;
#pragma unroll
    for (int jj = 0; jj < 4; jj++) {
        const uint32_t pp = pos + MZ_BYTE(jj < 2 ? s.E0 : s.E1, 2 * (jj & 1));
        const uint32_t wa = stage_word(stage_base, pp, k4);
        sm.red_or32_a(wa, __funnelshift_l(0u, s.v[jj], pp));
        sm.red_or32_a(wa + 4, __funnelshift_l(s.v[jj], 0u, pp));
    }
    if (s.MA) put_match_bits(sm, pos + ((s.offs >> 8) & 0xffu), s.MA);
    if (!ONEM) sm.st32(DF_OFF_REC + sidx * 8, pos + (s.offs >> 16)); /* (only read back where MB != 0) */
}

/* ---- the kernel ------------------------------------------------------------------------------- */
template <int STRIDE, bool LAZY, bool HIST = false>
__global__ void __launch_bounds__(DF_THREADS, HIST ? 1 : 2) deflate_chunks_kernel(DeflateParams P) {
    MZ_DYN_SMEM(smem_raw);
    uint8_t *const smem = smem_raw + (HIST ? DFH_PREV : 0); /* the standard carve-up; the history variant keeps the previous unit in front of it */
    constexpr uint32_t CUR = HIST ? (uint32_t)DFH_PREV : 0u; /* position of the unit's byte 0 as keys and candidates count it */
    uint8_t *s_in = smem + DF_OFF_IN;
    uint32_t *s_stage = (uint32_t *)(smem + DF_OFF_STAGE);
    uint32_t *s_hist_ll = (uint32_t *)(smem + DF_OFF_HIST);
    uint32_t *s_hist_d = s_hist_ll + 288;
    uint32_t *s_code_ll = (uint32_t *)(smem + DF_OFF_CODE);
    uint32_t *s_code_d = s_code_ll + 288;
    uint8_t *s_lens_ll = smem + DF_OFF_LENS;
    uint8_t *s_lens_d = s_lens_ll + 288;
    uint8_t *s_bits_ll = smem + DF_OFF_BITS;
    uint8_t *s_bits_d = s_bits_ll + 288;
    uint32_t *s_scan = (uint32_t *)(smem + DF_OFF_SCAN);
    uint32_t *s_bb = (uint32_t *)(smem + DF_OFF_BB);
    uint32_t *s_misc = (uint32_t *)(smem + DF_OFF_MISC);
#ifndef MZ_EMU
    uint64_t *s_bar = (uint64_t *)(smem + DF_OFF_MISC + 32 * 4);
    uint32_t bar_phase = 0;
    if (threadIdx.x == 0) {
        mbar_init(s_bar, 1);
        mbar_fence_init();
    }
    __syncthreads();
#endif
    const uint32_t tid = threadIdx.x;
    const unsigned lane = lane_id(), warp = warp_id();
    Smem sm;
    sm.init(smem);
    if (tid < 256) { /* the length-symbol table (read first in the classify pass of the first unit, many barriers later) */
        uint32_t ls, lb, lv;
        length_symbol(tid + 3, ls, lb, lv);
        sm.st16(DF_OFF_LSYM + tid * 2, ls | (lv << 5));
    }
    /* ONEM = keep only the first match of a span (a second one becomes literals): every later phase then carries one match
     * record per span instead of two. Measured on the emulator: 3 % larger output on text at stride 2 (short matches are
     * common), so it is off; the switch stays for experiments. */
    constexpr bool ONEM = false;
    DF_PHASE_BEGIN(ph_t); /* (the chunk's set-up counts to the load of its first unit, its trailer to the flush of its last) */

    /* Chunks are handed out by an atomic counter: if another kernel holds some SMs, the resident CTAs simply
     * take more chunks instead of leaving a tail to late CTAs. */
    for (uint32_t chunk_static = blockIdx.x;; chunk_static += gridDim.x) {
        uint32_t chunk = chunk_static;
        if (P.work_counter) {
            if (tid == 0) s_misc[MISC_CHUNK] = atomicAdd(P.work_counter, 1u);
            __syncthreads();
            chunk = s_misc[MISC_CHUNK];
        }
        if (chunk >= P.nchunks) {
            /* the last CTA out puts the counter pair back to zero: the launch needs no memset, and the slot is clean for its
             * next user (work_counter[1] counts the CTAs that have left) */
            if (P.work_counter && tid == 0 && atomicAdd(P.work_counter + 1, 1u) == gridDim.x - 1) {
                P.work_counter[0] = 0;
                P.work_counter[1] = 0;
            }
            break;
        }
        /* ---- locate the chunk -------------------------------------------------------------- */
        uint64_t off;
        uint32_t len, flags;
        if (P.in_off) {
            off = P.in_off[chunk];
            len = P.in_len[chunk];
            flags = P.flags ? P.flags[chunk] : 0u;
        } else {
            off = (uint64_t)chunk * P.chunk_size;
            uint64_t rem = P.total_len - off;
            len = rem < P.chunk_size ? (uint32_t)rem : P.chunk_size;
            /* last_flags: FINAL belongs to the last chunk; DICT says the whole buffer is one stream, so it holds for every chunk */
            flags = P.flags ? P.flags[chunk] : ((chunk == P.nchunks - 1 ? P.last_flags & ~DF_FLAG_DICT : 0u) | (P.last_flags & DF_FLAG_DICT));
        }
        const bool dict = HIST && (flags & DF_FLAG_DICT) && off >= (uint64_t)DFH_PREV;
        uint8_t *gout = P.out + (uint64_t)chunk * P.slot_stride;

        uint32_t flushed = 0; /* bytes of this chunk already in global memory (multiple of 16) */
        uint32_t bitpos = 0;  /* valid bits in the staging buffer (incl. the carried tail); uniform across the CTA */
        const uint32_t nunits = (len + DF_UNIT - 1) / DF_UNIT;
        if (tid < 4) s_misc[MISC_CARRY + tid] = 0;

        if (len == 0) {
            /* no unit will run: staging is used directly */
            for (uint32_t i = tid; i < 64; i += DF_THREADS) s_stage[i] = 0;
            __syncthreads();
            if (flags & DF_FLAG_FINAL) {
                /* zlib's answer for an empty stream: one fixed-Huffman block holding only EOB = 03 00 */
                if (tid == 0) stage_put(s_stage, 0, 1u | (1u << 1), 3);
                bitpos = 10;
            }
            __syncthreads();
        }

        for (uint32_t u = 0; u < nunits; u++) {
            const uint32_t ustart = u * DF_UNIT;
            const uint32_t ulen = (ustart + DF_UNIT < len) ? (uint32_t)DF_UNIT : len - ustart;
            const uint8_t *gin = P.in + off + ustart;
            const bool last_unit = u == nunits - 1;
            const uint32_t nb = (ulen + DF_BATCH - 1) / DF_BATCH;

            /* ---- load the unit into shared memory, reset the hash table ------------------------------ */
            const uint32_t len16 = ulen & ~15u;
            bool bulk = false;
#ifndef MZ_EMU
            bulk = (((uintptr_t)gin) & 15) == 0 && len16 > 0;
            if (bulk && tid == 0) {
                fence_proxy_async(); /* earlier generic-proxy accesses of s_in are done (trailing __syncthreads) */
                mbar_expect_tx(s_bar, len16);
                tma_load_1d(s_in, gin, len16, s_bar);
            }
#endif
            if (!bulk) {
                if ((((uintptr_t)gin) & 15) == 0) {
                    for (uint32_t i = tid * 16; i < len16; i += DF_THREADS * 16) *(uint4 *)(s_in + i) = ldg_stream((const uint4 *)(gin + i));
                } else {
                    for (uint32_t i = tid; i < len16; i += DF_THREADS) s_in[i] = gin[i];
                }
            }
            for (uint32_t i = len16 + tid; i < ulen; i += DF_THREADS) s_in[i] = gin[i];
            for (uint32_t i = ulen + tid; i < ((ulen + 63) & ~15u) + 16 && i < DF_UNIT + 64; i += DF_THREADS) s_in[i] = 0; /* zero pad */
            if (P.level != 0) {
                if (!HIST) {
                    for (uint32_t i = tid; i < DF_HASH_ENTRIES / 4; i += DF_THREADS) sm.st128(DF_OFF_HASH + i * 16, ~0u, ~0u, ~0u, ~0u);
                } else if (u == 0) {
                    for (uint32_t i = tid; i < (1u << DFH_HASH_BITS) / 4; i += DF_THREADS) sm.st128(DFH_OFF_HASH + i * 16, ~0u, ~0u, ~0u, ~0u);
                    if (dict) { /* the 32 KiB in front of the chunk become the previous unit */
                        const uint8_t *gp = P.in + off - DFH_PREV;
                        if ((((uintptr_t)gp) & 15) == 0) {
                            for (uint32_t i = tid * 16; i < (uint32_t)DFH_PREV; i += DF_THREADS * 16) *(uint4 *)(smem - DFH_PREV + i) = ldg_stream((const uint4 *)(gp + i));
                        } else {
                            for (uint32_t i = tid; i < (uint32_t)DFH_PREV; i += DF_THREADS) smem[(int)i - DFH_PREV] = gp[i];
                        }
                    }
                } else {
                    /* the table lives on: what was the current unit is the previous one now (position - 32768, batch age + 8);
                     * what pointed into the unit before that is too far away and goes */
                    for (uint32_t i = tid; i < (1u << DFH_HASH_BITS) / 4; i += DF_THREADS) {
                        uint4 e = *(const uint4 *)(smem + DFH_OFF_HASH + i * 16);
                        e.x = (e.x != ~0u && (e.x & 0xffffu) >= (uint32_t)DFH_PREV) ? e.x + 0x78000u : ~0u;
                        e.y = (e.y != ~0u && (e.y & 0xffffu) >= (uint32_t)DFH_PREV) ? e.y + 0x78000u : ~0u;
                        e.z = (e.z != ~0u && (e.z & 0xffffu) >= (uint32_t)DFH_PREV) ? e.z + 0x78000u : ~0u;
                        e.w = (e.w != ~0u && (e.w & 0xffffu) >= (uint32_t)DFH_PREV) ? e.w + 0x78000u : ~0u;
                        *(uint4 *)(smem + DFH_OFF_HASH + i * 16) = e;
                    }
                }
            }
#ifndef MZ_EMU
            if (bulk) {
                mbar_wait(s_bar, bar_phase);
                bar_phase ^= 1;
            }
#endif
            __syncthreads();
            if (HIST && P.level != 0 && u == 0 && dict) {
                /* insert the dictionary's positions: keys (15 - batch) << 16 | position, older than anything the unit will add */
#pragma unroll 1
                for (uint32_t b = 0; b < (uint32_t)DF_NBATCH; b++) {
                    const uint32_t p0 = b * DF_BATCH + tid * DF_SPAN;
                    const uint2 x = sm.ld64((uint32_t)(DF_OFF_IN - DFH_PREV) + p0);
                    const uint32_t y = sm.ld32((uint32_t)(DF_OFF_IN - DFH_PREV) + p0 + 8); /* (the last span reads into the unit: loaded above) */
                    const uint32_t key0 = ((15u - b) << 16) | p0;
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const uint32_t v = j == 0 ? x.x : (j < 4 ? __funnelshift_r(x.x, x.y, 8 * j) : (j == 4 ? x.y : __funnelshift_r(x.y, y, 8 * (j - 4))));
                        sm.red_min32(hash_addr<true>(v, 4u), key0 + j);
                    }
                }
                __syncthreads();
            }
            DF_PHASE(ph_t, DF_PH_LOAD);

            uint32_t fF[DF_NBATCH], fA[DF_NBATCH];
            bool stored = (P.level == 0);
            const uint32_t bfinal = (last_unit && (flags & DF_FLAG_FINAL)) ? 1u : 0u;

            if (P.level != 0) {
                /* ---- A + W: batches ------------------------------------------------------------------ */
                DF_PHASE_BEGIN(p_t);
                uint32_t ncap = 0; /* the warp's capped spans so far (uniform in the warp) */
#pragma unroll 1
                for (uint32_t b = 0; b < nb; b++) {
                    const uint32_t q0 = b * DF_BATCH + tid * DF_SPAN;
                    uint32_t v[12], ha[8], lc[8]; /* lc: the key read before the batch's inserts, then the position's match record */
                    const uint32_t k4 = opaque4();
                    {
                        const uint2 x = sm.ld64(DF_OFF_IN + q0), y = sm.ld64(DF_OFF_IN + q0 + 8);
                        v[0] = x.x; v[4] = x.y; v[8] = y.x;
#pragma unroll
                        for (int k = 1; k < 4; k++) {
                            v[k] = __funnelshift_r(x.x, x.y, 8 * k);
                            v[4 + k] = __funnelshift_r(x.y, y.x, 8 * k);
                            v[8 + k] = __funnelshift_r(y.x, y.y, 8 * k);
                        }
                    }
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        ha[j] = hash_addr<HIST>(v[j], k4);
                        if (j % STRIDE == 0) lc[j] = sm.ld32(ha[j]); /* key of the latest earlier batch that holds this hash */
                    }
                    const uint32_t nvalid = ulen > q0 ? (ulen - q0 < 8 ? ulen - q0 : 8u) : 0u;
                    __syncthreads();
                    DF_PHASE(p_t, DF_PH_P_A);
                    const uint32_t key0 = ((uint32_t)(DF_NBATCH - 1 - b) << 16) | (CUR + q0);
                    /* positions at or behind the end of the unit (zero padding, stale bytes) are inserted as well: they lie behind
                     * every valid position, so they never win a bucket a valid position of this batch hashes to, are never
                     * "before" anybody, and no batch follows a short unit -- cheaper than a select per key */
#pragma unroll
                    for (int j = 0; j < 8; j++) sm.red_min32(ha[j], key0 + j);
                    __syncthreads();
                    DF_PHASE(p_t, DF_PH_P_B);
                    /* Verify, and turn each candidate into the position's match record (the span record's form below, 0 for none).
                     * The choice is made on the keys themselves: this batch's keys are the youngest, and my own insert makes the
                     * bucket's key at most mine, so a smaller key is an earlier position of this batch with the same hash; else the
                     * candidate is the key read before the batch (~0: none). Outside the history variant the key's age bits may
                     * stay in c: only the low five bits of the shift amount count, the address keeps bits 2-15, a present key
                     * lies before me, and distance - 1 (below 32768) is the low 15 bits of the key difference. */
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        if (j % STRIDE != 0) {
                            lc[j] = 0;
                            continue;
                        }
                        const uint32_t kp = key0 + j, kn = sm.ld32(ha[j]);
                        const uint32_t ck = kn < kp ? kn : lc[j];
                        const uint32_t c = HIST ? ck & 0xffffu : ck;
                        const uint32_t ca = DF_OFF_IN - CUR + (c & 0xfffcu);
                        const uint32_t w0 = sm.ld32(ca), w1 = sm.ld32(ca + 4), w2 = sm.ld32(ca + 8);
                        const uint32_t s = c << 3;
                        const uint32_t x0 = __funnelshift_r(w0, w1, s) ^ v[j];
                        const uint32_t x1 = __funnelshift_r(w1, w2, s) ^ v[j + 4];
                        /* (history variant: a candidate more than 32768 back is out of DEFLATE's reach) */
                        const bool reach = HIST ? c < CUR + q0 + j && c >= q0 + j : ck != 0xffffffffu;
                        /* length - 3 = 1 + the further bytes that agree (0..4); in place at bit 3: that count's bits 3-5 + 8 */
                        const uint32_t l3 = ((uint32_t)__clz((int)__brev(x1)) & ~7u) + 8u;
                        lc[j] = sel_u32(reach && x0 == 0, (((kp - ck - 1u) << 11) & (0x7fffu << 11)) + l3 + (uint32_t)j, 0u);
                    }
                    if (q0 + 16 > ulen) { /* unit tail: the zero padding must not be matched */
#pragma unroll
                        for (int j = 0; j < 8; j += STRIDE) {
                            const uint32_t room = ulen > q0 + j ? ulen - (q0 + j) : 0u;
                            const uint32_t l = rec_len(lc[j]);
                            lc[j] = l >= (uint32_t)DF_MINMATCH && l > room ? (room >= (uint32_t)DF_MINMATCH ? lc[j] - ((l - room) << 3) : 0u) : lc[j];
                        }
                    }
                    /* ---- W: walk the span: static and branch-free. A match whose lockstep length is the cap (8) reaches the end of
                     * the span whatever its true length is, so it is always the span's last token: it is extended once, after
                     * the walk ------------------------------------------------------------------------------------------------ */
                    uint32_t nxt = 0, lit = 0, mA = 0, mB = 0, span_end = 0;
                    if (STRIDE == 2 && !LAZY && !ONEM) {
                        /* Level 1: candidates only at even positions, lengths 0 or >= 4. The walk then takes the first even position
                         * with a match (A: before it, and after its end, every position is a literal until the next even one), and
                         * then the first even position at or behind A's end that has one (B, which runs past the span). The same
                         * tokens as the walk below, as two chains of selects and two masks. */
#pragma unroll
                        for (int j = 6; j >= 0; j -= 2) mA = lc[j] ? lc[j] : mA;
                        const uint32_t endA = (mA & 7u) + rec_len(mA);
#pragma unroll
                        for (int j = 6; j >= 2; j -= 2) mB = lc[j] && (uint32_t)j >= endA ? lc[j] : mB;
                        const uint32_t endB = (mB & 7u) + rec_len(mB);
                        /* positions under no match are literals (no match: end = start = 0) */
                        lit = ~(((1u << endA) - (1u << (mA & 7u))) | ((1u << endB) - (1u << (mB & 7u)))) & 0xffu;
                        span_end = mB ? endB : endA;
                    } else {
#pragma unroll
                        for (int j = 0; j < 8; j++) {
                            const bool take = nxt == (uint32_t)j;
                            if (j % STRIDE == 0) {
                                const uint32_t rec = lc[j], l = rec_len(rec);
                                bool ism = take && rec != 0;
                                /* (the length fields compare as the lengths do; 0 = none) */
                                if (LAZY && STRIDE == 1 && j < 7) ism = ism && !(((lc[j + 1] >> 3) & 255u) > ((rec >> 3) & 255u));
                                const bool first = mA == 0;
                                if (ONEM) ism = ism && first;
                                mA = (ism && first) ? rec : mA;
                                if (!ONEM) mB = (ism && !first) ? rec : mB;
                                lit |= (take && !ism) ? (1u << j) : 0u;
                                nxt = ism ? (uint32_t)j + l : (take ? (uint32_t)j + 1u : nxt);
                            } else {
                                lit |= take ? (1u << j) : 0u;
                                nxt = take ? (uint32_t)j + 1u : nxt;
                            }
                        }
                        const uint32_t last = mB ? mB : mA;
                        span_end = last ? (last & 7u) + rec_len(last) : 0u;
                    }
                    lit &= (1u << nvalid) - 1u;
                    {
                        /* a capped match (lockstep length 8) is the span's last token; its true length is found after the batches,
                         * by the M0 pass, 32 such matches at a time (inline it kept the warp busy for the 8 lanes that have one):
                         * the warp appends its capped spans to its list in batch and lane order */
                        const uint32_t last = mB ? mB : mA;
                        const bool cap = ((last >> 3) & 255u) == (uint32_t)(DF_LOCKLEN - 3);
                        const uint32_t capped = __ballot_sync(MZ_FULL_MASK, cap);
                        sm.st8_if(cap, DF_OFF_CAPL + warp * 256u + ncap + (uint32_t)__popc(capped & ((1u << lane) - 1u)), (b << 5) | lane);
                        ncap += (uint32_t)__popc(capped);
                        sm.st64(DF_OFF_REC + (b * DF_THREADS + tid) * 8, mA | ((lit & 63u) << 26), mB | ((lit >> 6) << 26));
                        /* start offset and end (relative to the span) of the span's last match (0 for none) */
                        sm.st16(DF_OFF_SPN + (b * DF_THREADS + tid) * 2, ((last & 7u) << 9) | span_end);
                    }
                    DF_PHASE(p_t, DF_PH_P_C);
                }
                DF_PHASE(ph_t, DF_PH_PARSE); /* (no barrier behind the last batch: warp 0's view; the walks left are uniform work) */
                /* ---- M0: true lengths of the capped matches ----------------------------------------------------------------- */
                {
                    DF_PHASE_BEGIN(m_t);
                    __syncwarp();
                    for (uint32_t k0 = 0; k0 < ncap; k0 += 32) {
                        const uint32_t k = k0 + lane;
                        const uint32_t e = k < ncap ? sm.ld8(DF_OFF_CAPL + warp * 256u + k) : 0u;
                        const uint32_t sidx = (e >> 5) * (uint32_t)DF_THREADS + warp * 32u + (e & 31u);
                        DF_PHASE(m_t, DF_PH_M_INDEX);
                        if (k < ncap) {
                            const uint2 r = sm.ld64(DF_OFF_REC + sidx * 8);
                            const bool second = (r.y & 0x03ffffffu) != 0;
                            const uint32_t w = second ? r.y : r.x, last = w & 0x03ffffffu;
                            const uint32_t j = last & 7u, q = sidx * DF_SPAN + j, c = q - ((last >> 11) & 0x7fffu) - 1u; /* (wraps below 0: into the previous unit) */
                            uint32_t maxlen = ulen - q;
                            maxlen = maxlen < 258 ? maxlen : 258u;
                            /* Runs and short periods (zeros, 16- / 24- / 32-bit fill patterns): the table's candidate is the FIRST occurrence
                             * of the 8 bytes in an earlier batch, thousands of positions back -- 11 to 13 distance extra bits per match
                             * where the same bytes lie 1..4 positions back for none. The 8 bytes at q themselves say whether that can
                             * be (period 4, 2 or 1: both words equal -- then one word 4, 2 or 1 back settles all 8 bytes; period 3: the bytes
                             * 3 further on repeat the first word -- then both words are compared), so text pays two loads and two compares here; then the nearest such source is taken if it carries at least as far. */
                            uint32_t l = 0, cb = c;
                            if (q >= 4) {
                                const uint32_t a0 = sm.ld32u(DF_OFF_IN, q), a1 = sm.ld32u(DF_OFF_IN, q + 4);
                                const bool p4 = a0 == a1, p3 = __funnelshift_r(a0, a1, 24) == a0;
                                if (p4 || p3) {
                                    uint32_t cn = c;
                                    if (p4) {
                                        if (a0 == sm.ld32u(DF_OFF_IN, q - 4)) cn = q - 4;
                                        if (a0 == sm.ld32u(DF_OFF_IN, q - 2)) cn = q - 2;
                                        if (a0 == sm.ld32u(DF_OFF_IN, q - 1)) cn = q - 1;
                                    } else if (a0 == sm.ld32u(DF_OFF_IN, q - 3) && a1 == sm.ld32u(DF_OFF_IN, q + 1)) {
                                        cn = q - 3; /* (the pre-test saw 7 bytes of the period; extend_match8 relies on all 8) */
                                    }
                                    if (cn != c) {
                                        /* Inside such a run EVERY span holds this match, and the cover would cut each down to the 64
                                         * bytes its thread adds (507 matches for 32 KiB of zeros). Only the anchors keep theirs -- the
                                         * run's first span (the 8 bytes in front of it do not continue the period) and every 32nd span
                                         * (a match of 258 reaches the next one); the others give the match back: its positions count as
                                         * literals again (emitted only if, against expectation, nothing covers them) and no walk is
                                         * spent on them. */
                                        const uint32_t pd = q - cn;
                                        if (q >= 12u && (sidx & 31u) != 0u && sm.ld32u(DF_OFF_IN, q - 8) == sm.ld32u(DF_OFF_IN, q - 8 - pd) &&
                                            sm.ld32u(DF_OFF_IN, q - 4) == sm.ld32u(DF_OFF_IN, q - 4 - pd)) {
                                            const uint32_t left = ulen - sidx * DF_SPAN, nval = left < 8u ? left : 8u;
                                            const uint32_t lit = ((r.x >> 26) | ((r.y >> 26) << 6) | (0xffu << j)) & ((1u << nval) - 1u);
                                            const uint32_t mA = second ? (r.x & 0x03ffffffu) : 0u; /* an earlier, short match of the span stays */
                                            sm.st64(DF_OFF_REC + sidx * 8, mA | ((lit & 63u) << 26), (lit >> 6) << 26);
                                            sm.st16(DF_OFF_SPN + sidx * 2, mA ? ((mA & 7u) << 9) | ((mA & 7u) + rec_len(mA)) : 0u);
                                            continue;
                                        }
                                        l = extend_match8(sm, cn, q, maxlen);
                                        cb = cn;
                                    }
                                }
                            }
                            DF_PHASE(m_t, DF_PH_M_NEAR);
                            if (l < 64u && l < maxlen) { /* (a near source that runs this far is good enough: skip the second walk) */
                                const uint32_t lf = extend_match8(sm, c, q, maxlen);
                                if (lf > l) {
                                    l = lf;
                                    cb = c;
                                }
                            }
                            sm.st32(DF_OFF_REC + sidx * 8 + (second ? 4u : 0u), (w & ~((255u << 3) | (0x7fffu << 11))) | ((l - 3) << 3) | ((q - cb - 1u) << 11));
                            sm.st16(DF_OFF_SPN + sidx * 2, (j << 9) | (j + l));
                            DF_PHASE(m_t, DF_PH_M_EXTEND);
                        }
                    }
                }
                __syncthreads(); /* S1: records visible; the hash table is dead */
                DF_PHASE(ph_t, DF_PH_M0);

                /* ---- staging := 0 (+ the carried tail), histograms := 0 ------------------------------ */
                for (uint32_t i = tid; i < DF_STAGE_WORDS / 4; i += DF_THREADS) {
                    if (i == 0) sm.st128(DF_OFF_STAGE, s_misc[MISC_CARRY], s_misc[MISC_CARRY + 1], s_misc[MISC_CARRY + 2], s_misc[MISC_CARRY + 3]);
                    else sm.st128(DF_OFF_STAGE + i * 16, 0, 0, 0, 0);
                }
                for (uint32_t i = tid; i < 288 + 32 + 256; i += DF_THREADS) s_hist_ll[i] = 0; /* + the second literal copy */

                /* ---- B: cover. For this pass thread T owns the 8 CONSECUTIVE spans 8T..8T+7 (64 positions), so one block
                 * scan is enough; everything else keeps the parse mapping (span b*512+t),
                 * whose shared-memory accesses are conflict-free. cover(span) = the largest end of a match of an earlier
                 * span. Runs: inside a long repeat every span holds a maximal match, and the plain rule would cut each of
                 * them down to the 8 bytes it adds to the cover. A span that lies wholly under the cover and whose match
                 * sticks out of it is PENDING; a later such span whose match starts at or before the pending one's cover
                 * takes its place (and its cover), so a run is coded by the last match that can still start at the cover. */
                {
                    uint32_t se[8];
                    if (tid * 8 < nb * DF_THREADS) {
                        const uint4 q = *(const uint4 *)(smem + DF_OFF_SPN + tid * 16);
                        se[0] = q.x & 0xffffu; se[1] = q.x >> 16; se[2] = q.y & 0xffffu; se[3] = q.y >> 16;
                        se[4] = q.z & 0xffffu; se[5] = q.z >> 16; se[6] = q.w & 0xffffu; se[7] = q.w >> 16;
                    } else {
#pragma unroll
                        for (int k = 0; k < 8; k++) se[k] = 0;
                    }
                    const uint32_t p0 = tid * 64;
                    uint32_t tmax = 0;
#pragma unroll
                    for (int k = 0; k < 8; k++) {
                        const uint32_t e = se[k] ? p0 + 8 * k + (se[k] & 511u) : 0u;
                        tmax = tmax > e ? tmax : e;
                    }
                    const uint32_t incl = warp_incl_max(tmax);
                    uint32_t cin = __shfl_up_sync(MZ_FULL_MASK, incl, 1);
                    if (lane == 0) cin = 0;
                    if (lane == 31) s_scan[warp] = incl;
                    __syncthreads(); /* S2 */
                    {
                        const uint32_t w = (lane < (unsigned)DF_WARPS && lane < warp) ? s_scan[lane] : 0u;
                        const uint32_t base = __reduce_max_sync(MZ_FULL_MASK, w);
                        cin = cin > base ? cin : base;
                    }
                    uint32_t run = cin, drop = 0, pcv = 0, pendk = 0;
                    bool alive = false;
                    uint32_t cv[8];
#pragma unroll
                    for (int k = 0; k < 8; k++) {
                        const uint32_t q0 = p0 + 8 * k;
                        const uint32_t ms = q0 + (se[k] >> 9), me = q0 + (se[k] & 511u);
                        const bool fc = run >= q0 + 8;
                        const bool strad = se[k] != 0 && ms < run && me > run;
                        const bool takes = fc && strad && alive && ms <= pcv;
                        drop |= takes ? 1u << pendk : 0u;
                        cv[k] = takes ? pcv : run;
                        pcv = (fc && strad && !takes) ? run : pcv;
                        pendk = (fc && strad) ? (uint32_t)k : pendk;
                        alive = fc && (strad || alive);
                        run = (se[k] != 0 && me > run) ? me : run;
                    }
#pragma unroll
                    for (int k = 0; k < 8; k++) cv[k] = ((drop >> k) & 1u) ? 0xffffu : cv[k];
                    *(uint4 *)(smem + DF_OFF_SPN + tid * 16) = make_uint4(cv[0] | (cv[1] << 16), cv[2] | (cv[3] << 16), cv[4] | (cv[5] << 16), cv[6] | (cv[7] << 16));
                }
                __syncthreads(); /* S3: covers visible */
                DF_PHASE(ph_t, DF_PH_COVER);

                /* ---- T: classify every span once -> final records; symbol counts. The first match of a span is turned into symbol
                 * form here (36 % of the spans have one); the second one (7 %) would keep the whole warp busy for two or three
                 * lanes, so it is parked in the record region (word 1 of the span's record, dead once it has been read) and the
                 * warp's ballots remember where: the M1 pass below works through them 32 at a time. -------------------------- */
                const uint32_t hist_lit = sm.addr((lane & 1u) ? (uint32_t)DF_OFF_HIST2 : (uint32_t)DF_OFF_HIST); /* two copies halve the same-address traffic */
                const uint32_t k4 = opaque4();
                const uint32_t sink = sm.addr(DF_OFF_SINK + lane * 4);
                uint32_t bmB[DF_NBATCH]; /* per batch: the lanes of this warp whose span has a second match (warp-uniform) */
#pragma unroll
                for (int b = 0; b < DF_NBATCH; b++) {
                    uint32_t F = 0, MA = 0, MB = 0;
                    bmB[b] = 0;
                    if ((uint32_t)b < nb) {
                        const uint32_t sidx = (uint32_t)b * DF_THREADS + tid;
                        const uint32_t q0 = sidx * DF_SPAN;
                        const uint2 r = sm.ld64(DF_OFF_REC + sidx * 8);
                        const uint32_t cover = sm.ld16(DF_OFF_SPN + sidx * 2);
                        span_classify<ONEM>(sm, r.x, r.y, q0, cover, F, MA, MB);
                        const uint32_t ex = (F >> 8) & 3u;
                        if (ex) {
                            sm.red_add32_a(hist_lit + ((F >> 16) & 0xffu) * 4, 1u);
                            if (ex == 2) sm.red_add32_a(hist_lit + (F >> 24) * 4, 1u);
                        }
                        const uint2 x = sm.ld64(DF_OFF_IN + q0);
#pragma unroll
                        for (int j = 0; j < 8; j++) {
                            const uint32_t by = MZ_BYTE(j < 4 ? x.x : x.y, j & 3);
                            sm.red_add32_a(((F >> j) & 1u) ? by * k4 + hist_lit : sink, 1u);
                        }
                        if (MA) MA = match_symbols(sm, MA);
                        if (!ONEM) {
                            bmB[b] = __ballot_sync(MZ_FULL_MASK, MB != 0);
                            sm.st32(DF_OFF_REC + sidx * 8 + 4, MB);
                        }
                    }
                    fF[b] = F; fA[b] = MA;
                }
                /* ---- M1: the parked second matches -> symbol form (+ their two symbol counts), one per lane ---------------- */
                if (!ONEM) {
                    uint32_t totB = 0;
#pragma unroll
                    for (int b = 0; b < DF_NBATCH; b++) totB += (uint32_t)__popc(bmB[b]);
                    __syncwarp();
                    for (uint32_t k0 = 0; k0 < totB; k0 += 32) {
                        const uint32_t sidx = nth_parked(bmB, k0 + lane, warp);
                        if (sidx != 0xffffffffu) {
                            const uint32_t a = DF_OFF_REC + sidx * 8 + 4;
                            sm.st32(a, match_symbols(sm, sm.ld32(a)));
                        }
                    }
                }
                if (tid == 0) sm.red_add32(DF_OFF_HIST + 256 * 4, 1u); /* end of block */
                __syncthreads(); /* S4 */
                DF_PHASE(ph_t, DF_PH_T_M1);
                /* ---- D: codes (10 warps on a named barrier; the rest wait here) ------------------------- */
#ifdef MZ_DF_CODES_HOOK /* test builds only (tests/emu/emu_df_codes.cc): record the histograms the builder is given */
                if (tid == 0) MZ_DF_CODES_HOOK(s_hist_ll, (const uint32_t *)(smem + DF_OFF_HIST2), s_hist_d);
#endif
                if (tid < DF_BB_THREADS)
                    block_build_codes(s_hist_ll, (const uint32_t *)(smem + DF_OFF_HIST2), s_hist_d, s_lens_ll, s_lens_d, s_code_ll, s_code_d, s_bits_ll, s_bits_d, s_bb,
                                      s_stage, bitpos, bfinal);
                __syncthreads(); /* S5 */
                DF_PHASE(ph_t, DF_PH_D);
                const uint32_t hdrbits = s_bb[BB_HDRBITS], tokbits = s_bb[BB_TOKBITS];
                const uint32_t eob = s_code_ll[256];
                const uint32_t dyn_bits = hdrbits + tokbits + ((eob >> 16) & 15u);
                const uint32_t stored_bits = (((bitpos + 3 + 7) & ~7u) - bitpos) + 32 + ulen * 8;
                if (dyn_bits >= stored_bits) {
                    stored = true;
                    /* take the header back out of the staging buffer (rare path) */
                    const uint32_t w0 = bitpos >> 5;
                    for (uint32_t i = tid; i <= (hdrbits + 31) / 32 + 1; i += DF_THREADS)
                        s_stage[w0 + i] = i == 0 ? s_stage[w0] & ((1u << (bitpos & 31u)) - 1u) : 0u;
                    __syncthreads();
                } else {
                    /* ---- E + F: count and emit, two batches at a time. span_bits() looks up a span's code words once and gives
                     * its size and every bit offset inside it. One warp scan covers both batches (the sizes packed in 16-bit
                     * halves: a warp's total per batch is at most 32 x 246 bits), the warp totals go to s_scan (one slot per batch
                     * pair and warp, never rewritten in a unit), and one barrier per pair places every span: spans of a batch are
                     * in stream order by thread, the second batch follows the first, and each pair starts where the one before
                     * ended (`run`). The spans are then written as span_emit() says. ------------------------------------------ */
                    const uint32_t code_base = sm.addr(DF_OFF_CODE), zero_ent = sm.addr(DF_OFF_CODE + DF_ZERO_SYM * 4), stage_base = sm.addr(DF_OFF_STAGE);
                    const uint32_t k4 = opaque4();
                    uint32_t run = bitpos + hdrbits; /* bit position of the pair's first span (uniform across the CTA) */
                    DF_PHASE_BEGIN(x_t);
#pragma unroll
                    for (int b = 0; b < DF_NBATCH; b += 2) {
                        if ((uint32_t)b >= nb) break; /* (uniform) */
                        const uint32_t s0 = (uint32_t)b * DF_THREADS + tid, s1 = s0 + DF_THREADS;
                        /* (a short unit may end after the first batch of a pair: the second then holds nothing; its record is stale) */
                        const uint32_t MB0 = ONEM ? 0u : sm.ld32(DF_OFF_REC + s0 * 8 + 4);
                        const uint32_t MB1 = (ONEM || (uint32_t)b + 1 >= nb) ? 0u : sm.ld32(DF_OFF_REC + s1 * 8 + 4);
                        const SpanBits A = span_bits<ONEM>(sm, s0, fF[b], fA[b], MB0, code_base, zero_ent, k4);
                        const SpanBits B = span_bits<ONEM>(sm, s1, fF[b + 1], fA[b + 1], MB1, code_base, zero_ent, k4);
                        const uint32_t sz = A.size | (B.size << 16);
                        const uint32_t incl = warp_incl_sum(sz);
                        if (lane == 31) s_scan[(b / 2) * DF_WARPS + warp] = incl;
                        __syncthreads(); /* one per pair: the pair's warp totals are visible */
                        DF_PHASE(x_t, DF_PH_X_SCAN);
                        const uint32_t wt = lane < (unsigned)DF_WARPS ? s_scan[(b / 2) * DF_WARPS + lane] : 0u;
                        const uint32_t wlo = wt & 0xffffu, whi = wt >> 16; /* (the sums over warps no longer fit 16 bits) */
                        const uint32_t totA = __reduce_add_sync(MZ_FULL_MASK, wlo);
                        const uint32_t ex = incl - sz; /* exclusive, per half (no borrow: each half of incl is at least its size) */
                        const uint32_t posA = run + __reduce_add_sync(MZ_FULL_MASK, lane < warp ? wlo : 0u) + (ex & 0xffffu);
                        const uint32_t posB = run + totA + __reduce_add_sync(MZ_FULL_MASK, lane < warp ? whi : 0u) + (ex >> 16);
                        run += totA + __reduce_add_sync(MZ_FULL_MASK, whi);
                        if (A.size) span_emit<ONEM>(sm, A, posA, s0, stage_base, k4);
                        if (B.size) span_emit<ONEM>(sm, B, posB, s1, stage_base, k4);
                        DF_PHASE(x_t, DF_PH_X_EMIT);
                    }
#ifdef MZ_EMU
                    if (run != bitpos + hdrbits + tokbits) { /* the spans' sizes must add up to what D counted from the histograms */
                        fprintf(stderr, "deflate: block %u, unit %u: emitted %u token bits, the histograms count %u\n", (unsigned)blockIdx.x, u,
                                run - bitpos - hdrbits, tokbits);
                        abort();
                    }
#endif
                    /* ---- M3: the parked second matches, one per lane ----------------------------------------------------- */
                    if (!ONEM) {
                        uint32_t totB = 0;
#pragma unroll
                        for (int b = 0; b < DF_NBATCH; b++) totB += (uint32_t)__popc(bmB[b]);
                        __syncwarp();
                        for (uint32_t k0 = 0; k0 < totB; k0 += 32) {
                            const uint32_t sidx = nth_parked(bmB, k0 + lane, warp);
                            if (sidx != 0xffffffffu) {
                                const uint2 r = sm.ld64(DF_OFF_REC + sidx * 8);
                                put_match_bits(sm, r.x, r.y);
                            }
                        }
                    }
                    DF_PHASE(x_t, DF_PH_X_M3);
                    if (tid == DF_THREADS - 1) stage_put(s_stage, bitpos + hdrbits + tokbits, eob & 0x7fffu, (eob >> 16) & 15u);
                    bitpos += dyn_bits;
                }
            } else {
                /* level 0: staging was never a hash table, but it still has to be clean */
                for (uint32_t i = tid; i < DF_STAGE_WORDS / 4; i += DF_THREADS) {
                    if (i == 0) sm.st128(DF_OFF_STAGE, s_misc[MISC_CARRY], s_misc[MISC_CARRY + 1], s_misc[MISC_CARRY + 2], s_misc[MISC_CARRY + 3]);
                    else sm.st128(DF_OFF_STAGE + i * 16, 0, 0, 0, 0);
                }
                __syncthreads();
            }
            if (stored) {
                /* stored block: header, pad to byte, LEN, ~LEN, raw bytes */
                const uint32_t p0 = (bitpos + 3 + 7) >> 3; /* byte index of LEN */
                if (tid == 0) {
                    stage_put(s_stage, bitpos, bfinal, 3);
                    stage_put(s_stage, p0 * 8, ulen, 16);
                    stage_put(s_stage, p0 * 8 + 16, ulen ^ 0xffffu, 16);
                }
                for (uint32_t i = tid * 4; i < ulen; i += DF_THREADS * 4) {
                    uint32_t v = load32u(s_in, i);
                    uint32_t n = ulen - i;
                    stage_put(s_stage, (p0 + 4 + i) * 8, v, n >= 4 ? 32 : n * 8);
                }
                bitpos = (p0 + 4 + ulen) * 8;
            }
            __syncthreads();
            DF_PHASE(ph_t, DF_PH_EMIT); /* (a stored block counts here) */
            /* ---- G: flush whole 16-byte units, carry the tail ------------------------------------ */
            {
                const uint32_t n16 = bitpos >> 7;
                const uint32_t used_words = (bitpos + 31) >> 5;
                /* (four copies in flight per thread; unrolled further, the copy sets the register count of the history variant,
                 * which has no limit below 128 from its launch bounds) */
#pragma unroll 4
                for (uint32_t i = tid; i < n16; i += DF_THREADS) ((uint4 *)(gout + flushed))[i] = ((const uint4 *)s_stage)[i];
                if (tid < 4) s_misc[MISC_CARRY + tid] = (n16 * 4 + tid < used_words) ? s_stage[n16 * 4 + tid] : 0u;
                bitpos -= n16 * 128;
                flushed += n16 * 16;
                if (HIST && u + 1 < nunits) /* this unit is the next one's history */
                    for (uint32_t i = tid; i < (uint32_t)DF_UNIT / 16; i += DF_THREADS) *(uint4 *)(smem - DFH_PREV + i * 16) = *(const uint4 *)(s_in + i * 16);
                __syncthreads();
                DF_PHASE(ph_t, DF_PH_FLUSH);
            }
        }


        /* ---- chunk trailer: the carried tail (< 16 bytes, in s_misc; for an empty chunk still in the staging buffer) plus the
         * sync-flush marker of a non-final chunk go out as two 16-byte units (the slot has the room) ------------------- */
        {
            if (tid < 8) {
                const uint32_t v = tid < 4 ? (len == 0 ? s_stage[tid] : s_misc[MISC_CARRY + tid]) : 0u;
                __syncwarp(0xffu);
                s_stage[tid] = v;
            }
            __syncthreads();
            if (flags & DF_FLAG_FINAL) {
                bitpos = (bitpos + 7) & ~7u;
            } else {
                /* empty stored block: BFINAL=0 BTYPE=00, pad, LEN=0000 NLEN=FFFF */
                const uint32_t p0 = (bitpos + 3 + 7) >> 3; /* <= 17 */
                if (tid == 0) stage_put(s_stage, (p0 + 2) * 8, 0xffffu, 16);
                bitpos = (p0 + 4) * 8;
            }
            __syncthreads();
            if (tid < 8) ((uint32_t *)(gout + flushed))[tid] = s_stage[tid];
            if (tid == 0) P.out_len[chunk] = flushed + (bitpos >> 3);
            __syncthreads();
            DF_PHASE(ph_t, DF_PH_FLUSH);
        }
    }
}

/* level -> match-finder configuration: 1 = candidates looked up at even positions only (every position is still
 * inserted), 2..3 = every position, 4..9 = every position + one-step lazy evaluation */
__host__ __device__ inline int deflate_stride_for_level(int level) { return level <= 1 ? 2 : 1; }
__host__ __device__ inline bool deflate_lazy_for_level(int level) { return level >= 4; }
/* 6..9: the history variant (previous 32 KiB as a dictionary, 2^14-key table that survives from unit to unit, one CTA per SM) */
__host__ __device__ inline bool deflate_hist_for_level(int level) { return level >= 6; }

} // namespace mzc
#endif
