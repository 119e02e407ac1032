/* mzoracle.c -- CPU oracle for the DEFLATE + CRC-32 hot path (TEST INFRASTRUCTURE ONLY).
 * See mzoracle.h for scope, sources restated and how the oracle is pinned. */
#include "mzoracle.h"

#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------------------------
 * CRC-32 (poly 0xEDB88320 reflected). Follows the loop at mz_crypt.c:81-90: invert, one table
 * step per byte, invert. The 256-entry table (mz_crypt.c:51-80) is generated, not copied: entry
 * n is n pushed through 8 shift/conditional-xor steps.
 * ---------------------------------------------------------------------------------------- */
static uint32_t g_crc_table[256];
static int g_crc_table_ready;

static void crc_table_init(void) {
    for (uint32_t n = 0; n < 256; n++) {
        uint32_t c = n;
        for (int k = 0; k < 8; k++)
            c = (c & 1) ? (0xEDB88320u ^ (c >> 1)) : (c >> 1);
        g_crc_table[n] = c;
    }
    g_crc_table_ready = 1;
}

uint32_t orc_crc32_update(uint32_t value, const uint8_t *buf, size_t size) {
    if (!g_crc_table_ready)
        crc_table_init();
    value = ~value;                                 /* mz_crypt.c:81 */
    while (size > 0) {                              /* mz_crypt.c:83-88 */
        value = (value >> 8) ^ g_crc_table[(value ^ *buf) & 0xFF];
        buf += 1;
        size -= 1;
    }
    return ~value;                                  /* mz_crypt.c:90 */
}

/* crc(A||B) = crc(A) * x^(8*len_b) + crc(B) over GF(2)[x]/P (the pre/post inversions cancel).
 * Multiplication by x^(8*len_b) by square-and-multiply on 32x32 bit matrices. */
static uint32_t gf2_matrix_times(const uint32_t *mat, uint32_t vec) {
    uint32_t sum = 0;
    while (vec) {
        if (vec & 1)
            sum ^= *mat;
        vec >>= 1;
        mat++;
    }
    return sum;
}

static void gf2_matrix_square(uint32_t *square, const uint32_t *mat) {
    for (int n = 0; n < 32; n++)
        square[n] = gf2_matrix_times(mat, mat[n]);
}

uint32_t orc_crc32_combine(uint32_t crc_a, uint32_t crc_b, uint64_t len_b) {
    uint32_t even[32], odd[32];
    if (len_b == 0)
        return crc_a;
    /* odd = operator for one zero bit */
    odd[0] = 0xEDB88320u;
    uint32_t row = 1;
    for (int n = 1; n < 32; n++) {
        odd[n] = row;
        row <<= 1;
    }
    gf2_matrix_square(even, odd); /* 2 bits */
    gf2_matrix_square(odd, even); /* 4 bits */
    do {
        gf2_matrix_square(even, odd); /* first pass: 8 bits = 1 byte */
        if (len_b & 1)
            crc_a = gf2_matrix_times(even, crc_a);
        len_b >>= 1;
        if (len_b == 0)
            break;
        gf2_matrix_square(odd, even);
        if (len_b & 1)
            crc_a = gf2_matrix_times(odd, crc_a);
        len_b >>= 1;
    } while (len_b != 0);
    return crc_a ^ crc_b;
}

uint32_t orc_adler32_update(uint32_t value, const uint8_t *buf, size_t size) {
    uint32_t a = value & 0xffff, b = (value >> 16) & 0xffff;
    while (size > 0) {
        size_t n = size > 5552 ? 5552 : size;
        size -= n;
        while (n--) {
            a += *buf++;
            b += a;
        }
        a %= 65521u;
        b %= 65521u;
    }
    return (b << 16) | a;
}

/* ------------------------------------------------------------------------------------------
 * RFC 1951 decoder.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    const uint8_t *in;
    size_t in_len;
    size_t pos;      /* next byte to load */
    uint64_t bitbuf; /* LSB-first */
    int bitcnt;
    int starved;     /* ran past end of input */
    uint8_t *out;
    size_t out_cap;
    size_t out_pos;
} orc_state;

static inline uint32_t need_bits(orc_state *s, int n) {
    while (s->bitcnt < n) {
        if (s->pos >= s->in_len) {
            s->starved = 1;
            return 0;
        }
        s->bitbuf |= (uint64_t)s->in[s->pos++] << s->bitcnt;
        s->bitcnt += 8;
    }
    return (uint32_t)(s->bitbuf & ((1ull << n) - 1));
}

static inline uint32_t get_bits(orc_state *s, int n) {
    if (n == 0)
        return 0;
    uint32_t v = need_bits(s, n);
    if (s->starved)
        return 0;
    s->bitbuf >>= n;
    s->bitcnt -= n;
    return v;
}

typedef struct {
    uint16_t count[16];  /* codes of each length */
    uint16_t symbol[288]; /* symbols ordered by code */
} orc_huff;

/* Canonical code from lengths (RFC1951 3.2.2). Returns 0 complete, >0 incomplete (unused
 * code space left), <0 over-subscribed. */
static int huff_build(orc_huff *h, const uint8_t *lens, int n) {
    uint16_t offs[16];
    memset(h->count, 0, sizeof(h->count));
    for (int i = 0; i < n; i++)
        h->count[lens[i]]++;
    if (h->count[0] == n)
        return 0; /* no codes: complete but empty; decoding any symbol fails */
    int left = 1;
    for (int len = 1; len <= 15; len++) {
        left <<= 1;
        left -= h->count[len];
        if (left < 0)
            return left;
    }
    offs[1] = 0;
    for (int len = 1; len < 15; len++)
        offs[len + 1] = offs[len] + h->count[len];
    for (int i = 0; i < n; i++)
        if (lens[i])
            h->symbol[offs[lens[i]]++] = (uint16_t)i;
    return left;
}

/* Decode one symbol bit by bit (codes are packed MSB-first, RFC1951 3.1.1). */
static int huff_decode(orc_state *s, const orc_huff *h) {
    int code = 0, first = 0, index = 0;
    for (int len = 1; len <= 15; len++) {
        code |= (int)get_bits(s, 1);
        if (s->starved)
            return -2;
        int count = h->count[len];
        if (code - count < first)
            return h->symbol[index + (code - first)];
        index += count;
        first += count;
        first <<= 1;
        code <<= 1;
    }
    return -1; /* ran out of codes */
}

static const uint16_t k_len_base[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                        31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
static const uint8_t k_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
static const uint16_t k_dist_base[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                         193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
static const uint8_t k_dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};

static int inflate_codes(orc_state *s, const orc_huff *lit, const orc_huff *dist) {
    for (;;) {
        int sym = huff_decode(s, lit);
        if (sym == -2)
            return ORC_BUF_ERROR;
        if (sym < 0)
            return ORC_DATA_ERROR;
        if (sym < 256) {
            if (s->out_pos >= s->out_cap)
                return ORC_BUF_ERROR;
            s->out[s->out_pos++] = (uint8_t)sym;
        } else if (sym == 256) {
            return ORC_OK;
        } else {
            sym -= 257;
            if (sym >= 29)
                return ORC_DATA_ERROR;
            uint32_t len = k_len_base[sym] + get_bits(s, k_len_extra[sym]);
            int dsym = huff_decode(s, dist);
            if (dsym == -2 || s->starved)
                return ORC_BUF_ERROR;
            if (dsym < 0 || dsym >= 30)
                return ORC_DATA_ERROR;
            uint32_t d = k_dist_base[dsym] + get_bits(s, k_dist_extra[dsym]);
            if (s->starved)
                return ORC_BUF_ERROR;
            if (d > s->out_pos)
                return ORC_DATA_ERROR; /* distance too far back */
            if (s->out_pos + len > s->out_cap)
                return ORC_BUF_ERROR;
            uint8_t *dst = s->out + s->out_pos;
            const uint8_t *src = dst - d;
            for (uint32_t i = 0; i < len; i++)
                dst[i] = src[i]; /* byte-serial on purpose: overlap replicates */
            s->out_pos += len;
        }
    }
}

static int inflate_stored(orc_state *s) {
    s->bitbuf >>= (s->bitcnt & 7); /* drop to byte boundary */
    s->bitcnt -= (s->bitcnt & 7);
    uint32_t len = get_bits(s, 16);
    uint32_t nlen = get_bits(s, 16);
    if (s->starved)
        return ORC_BUF_ERROR;
    if ((len ^ 0xffffu) != nlen)
        return ORC_DATA_ERROR;
    /* bitcnt is now a multiple of 8 and holds whole look-ahead bytes: give them back */
    while (s->bitcnt >= 8) {
        s->pos--;
        s->bitcnt -= 8;
    }
    s->bitbuf = 0;
    s->bitcnt = 0;
    if (s->pos + len > s->in_len) {
        s->starved = 1;
        return ORC_BUF_ERROR;
    }
    if (s->out_pos + len > s->out_cap)
        return ORC_BUF_ERROR;
    memcpy(s->out + s->out_pos, s->in + s->pos, len);
    s->pos += len;
    s->out_pos += len;
    return ORC_OK;
}

static int build_fixed(orc_huff *lit, orc_huff *dist) {
    uint8_t lens[288];
    int i = 0;
    for (; i < 144; i++) lens[i] = 8;
    for (; i < 256; i++) lens[i] = 9;
    for (; i < 280; i++) lens[i] = 7;
    for (; i < 288; i++) lens[i] = 8;
    huff_build(lit, lens, 288);
    for (i = 0; i < 32; i++) lens[i] = 5; /* codes 30 and 31 exist and are invalid when decoded, as in zlib */
    huff_build(dist, lens, 32);
    return 0;
}

static int read_dynamic(orc_state *s, orc_huff *lit, orc_huff *dist) {
    static const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    uint8_t lens[320];
    orc_huff clh;
    int nlen = (int)get_bits(s, 5) + 257;
    int ndist = (int)get_bits(s, 5) + 1;
    int ncode = (int)get_bits(s, 4) + 4;
    if (s->starved)
        return ORC_BUF_ERROR;
    if (nlen > 286 || ndist > 30)
        return ORC_DATA_ERROR;
    memset(lens, 0, sizeof(lens));
    for (int i = 0; i < ncode; i++)
        lens[order[i]] = (uint8_t)get_bits(s, 3);
    if (s->starved)
        return ORC_BUF_ERROR;
    if (huff_build(&clh, lens, 19) != 0)
        return ORC_DATA_ERROR; /* code length code must be complete */
    int idx = 0;
    while (idx < nlen + ndist) {
        int sym = huff_decode(s, &clh);
        if (sym == -2)
            return ORC_BUF_ERROR;
        if (sym < 0)
            return ORC_DATA_ERROR;
        if (sym < 16) {
            lens[idx++] = (uint8_t)sym;
        } else {
            int rep, val = 0;
            if (sym == 16) {
                val = idx ? lens[idx - 1] : 0;
                rep = 3 + (int)get_bits(s, 2);
            } else if (sym == 17) {
                rep = 3 + (int)get_bits(s, 3);
            } else {
                rep = 11 + (int)get_bits(s, 7);
            }
            if (s->starved)
                return ORC_BUF_ERROR; /* zlib decides on a repeat once its extra bits are in */
            if ((sym == 16 && idx == 0) || idx + rep > nlen + ndist)
                return ORC_DATA_ERROR;
            while (rep--)
                lens[idx++] = (uint8_t)val;
        }
    }
    if (lens[256] == 0)
        return ORC_DATA_ERROR; /* no end-of-block code */
    int err = huff_build(lit, lens, nlen);
    if (err < 0 || (err > 0 && !(nlen - lit->count[0] == 1 && lit->count[1] == 1)))
        return ORC_DATA_ERROR; /* incomplete only allowed for a single code of length 1 */
    err = huff_build(dist, lens + nlen, ndist);
    if (err < 0 || (err > 0 && !(ndist - dist->count[0] == 1 && dist->count[1] == 1)))
        return ORC_DATA_ERROR;
    return ORC_OK;
}

static int inflate_raw(orc_state *s, orc_block_info *blocks, size_t max_blocks, int64_t *nblocks) {
    orc_huff lit, dist;
    int last;
    do {
        uint64_t start_bit = (uint64_t)s->pos * 8 - (uint64_t)s->bitcnt;
        size_t out_before = s->out_pos;
        last = (int)get_bits(s, 1);
        int type = (int)get_bits(s, 2);
        if (s->starved)
            return ORC_BUF_ERROR;
        int err;
        if (type == 0) {
            err = inflate_stored(s);
        } else if (type == 1) {
            build_fixed(&lit, &dist);
            err = inflate_codes(s, &lit, &dist);
        } else if (type == 2) {
            err = read_dynamic(s, &lit, &dist);
            if (err == ORC_OK)
                err = inflate_codes(s, &lit, &dist);
        } else {
            err = ORC_DATA_ERROR;
        }
        if (err != ORC_OK)
            return err;
        if (nblocks) {
            if (blocks && (size_t)*nblocks < max_blocks) {
                blocks[*nblocks].start_bit = start_bit;
                blocks[*nblocks].out_bytes = s->out_pos - out_before;
                blocks[*nblocks].type = type;
                blocks[*nblocks].final = last;
            }
            (*nblocks)++;
        }
    } while (!last);
    /* give back whole unused look-ahead bytes; the partial final byte is consumed */
    while (s->bitcnt >= 8) {
        s->pos--;
        s->bitcnt -= 8;
    }
    s->bitbuf = 0;
    s->bitcnt = 0;
    return ORC_OK;
}

static int parse_gzip_header(orc_state *s) {
    const uint8_t *p = s->in;
    size_t n = s->in_len, i = 10;
    if (n < 10)
        return ORC_BUF_ERROR;
    if (p[0] != 0x1f || p[1] != 0x8b || p[2] != 8 || (p[3] & 0xe0))
        return ORC_DATA_ERROR;
    int flg = p[3];
    if (flg & 4) { /* FEXTRA */
        if (i + 2 > n) return ORC_BUF_ERROR;
        size_t xlen = p[i] | (p[i + 1] << 8);
        i += 2 + xlen;
    }
    if (flg & 8) { /* FNAME */
        while (i < n && p[i]) i++;
        i++;
    }
    if (flg & 16) { /* FCOMMENT */
        while (i < n && p[i]) i++;
        i++;
    }
    if (flg & 2)
        i += 2; /* FHCRC */
    if (i > n)
        return ORC_BUF_ERROR;
    s->pos = i;
    return ORC_OK;
}

static int inflate_any(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap, int wrap, size_t *consumed,
                       size_t *produced, orc_block_info *blocks, size_t max_blocks, int64_t *nblocks) {
    orc_state s;
    memset(&s, 0, sizeof(s));
    s.in = in;
    s.in_len = in_len;
    s.out = out;
    s.out_cap = out_cap;
    int err = ORC_OK;
    if (wrap == ORC_WRAP_GZIP) {
        err = parse_gzip_header(&s);
    } else if (wrap == ORC_WRAP_ZLIB) {
        if (in_len < 2)
            err = ORC_BUF_ERROR;
        else if ((in[0] & 0x0f) != 8 || (in[0] >> 4) > 7 || ((in[0] << 8) | in[1]) % 31 != 0 || (in[1] & 0x20))
            err = ORC_DATA_ERROR;
        else
            s.pos = 2;
    }
    if (err == ORC_OK)
        err = inflate_raw(&s, blocks, max_blocks, nblocks);
    if (err == ORC_OK && wrap == ORC_WRAP_GZIP) {
        if (s.pos + 8 > in_len) {
            err = ORC_BUF_ERROR;
        } else {
            const uint8_t *t = in + s.pos;
            uint32_t crc = t[0] | (t[1] << 8) | (t[2] << 16) | ((uint32_t)t[3] << 24);
            uint32_t isz = t[4] | (t[5] << 8) | (t[6] << 16) | ((uint32_t)t[7] << 24);
            s.pos += 8;
            if (crc != orc_crc32_update(0, out, s.out_pos) || isz != (uint32_t)s.out_pos)
                err = ORC_DATA_ERROR;
        }
    } else if (err == ORC_OK && wrap == ORC_WRAP_ZLIB) {
        if (s.pos + 4 > in_len) {
            err = ORC_BUF_ERROR;
        } else {
            const uint8_t *t = in + s.pos;
            uint32_t ad = ((uint32_t)t[0] << 24) | (t[1] << 16) | (t[2] << 8) | t[3];
            s.pos += 4;
            if (ad != orc_adler32_update(1, out, s.out_pos))
                err = ORC_DATA_ERROR;
        }
    }
    if (consumed)
        *consumed = s.pos;
    if (produced)
        *produced = s.out_pos;
    return err;
}

int orc_inflate(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap, int wrap, size_t *consumed,
                size_t *produced) {
    return inflate_any(in, in_len, out, out_cap, wrap, consumed, produced, NULL, 0, NULL);
}

int64_t orc_inflate_blocks(const uint8_t *in, size_t in_len, int wrap, orc_block_info *blocks, size_t max_blocks,
                           size_t *produced) {
    /* needs a real output buffer for back-references: grow until it fits */
    size_t cap = in_len * 8 + 65536;
    for (;;) {
        uint8_t *out = (uint8_t *)malloc(cap);
        if (!out)
            return ORC_MEM_ERROR;
        int64_t n = 0;
        size_t prod = 0, cons = 0;
        int err = inflate_any(in, in_len, out, cap, wrap, &cons, &prod, blocks, max_blocks, &n);
        free(out);
        if (err == ORC_BUF_ERROR && prod + 258 >= cap && cap < ((size_t)1 << 36)) {
            cap *= 4;
            continue;
        }
        if (produced)
            *produced = prod;
        return err == ORC_OK ? n : err;
    }
}

/* ------------------------------------------------------------------------------------------
 * RFC 1951 encoder (port-style CPU baseline and second stream producer).
 * Greedy hash-chain LZ77, 32 KiB window, min match 3, max 258; dynamic Huffman per block with
 * lengths from a heap-free two-queue Huffman build limited to 15 bits by the classic
 * "demote overflow" fix-up; code-length alphabet emitted without run-length symbols 16-18 when
 * that is shorter to implement -- still RFC-valid.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
    uint8_t *out;
    size_t cap, pos;
    uint64_t bitbuf;
    int bitcnt;
    int overflow;
} orc_bw;

static inline void bw_put(orc_bw *w, uint32_t v, int n) {
    w->bitbuf |= (uint64_t)v << w->bitcnt;
    w->bitcnt += n;
    while (w->bitcnt >= 8) {
        if (w->pos < w->cap)
            w->out[w->pos++] = (uint8_t)w->bitbuf;
        else
            w->overflow = 1;
        w->bitbuf >>= 8;
        w->bitcnt -= 8;
    }
}

static inline void bw_align(orc_bw *w) {
    if (w->bitcnt > 0)
        bw_put(w, 0, 8 - w->bitcnt);
}

static uint32_t rev_bits(uint32_t v, int n) {
    uint32_t r = 0;
    for (int i = 0; i < n; i++) {
        r = (r << 1) | (v & 1);
        v >>= 1;
    }
    return r;
}

/* Length-limited Huffman lengths. Simple O(n^2)-free approach: sort, two-queue tree build,
 * depth count, then Kraft repair to maxbits. */
typedef struct { uint32_t f; int s; } orc_fs;
static int fs_cmp(const void *a, const void *b) {
    const orc_fs *x = (const orc_fs *)a, *y = (const orc_fs *)b;
    if (x->f != y->f) return x->f < y->f ? -1 : 1;
    return x->s - y->s;
}

static void huff_lengths(const uint32_t *freq, int n, int maxbits, uint8_t *lens) {
    orc_fs leaves[288];
    int nl = 0;
    memset(lens, 0, (size_t)n);
    for (int i = 0; i < n; i++)
        if (freq[i]) {
            leaves[nl].f = freq[i];
            leaves[nl].s = i;
            nl++;
        }
    /* zlib's inflate wants at least a usable code; force two symbols */
    for (int i = 0; nl < 2 && i < n; i++) {
        int present = 0;
        for (int j = 0; j < nl; j++)
            if (leaves[j].s == i) present = 1;
        if (!present) {
            leaves[nl].f = 1;
            leaves[nl].s = i;
            nl++;
        }
    }
    qsort(leaves, (size_t)nl, sizeof(orc_fs), fs_cmp);
    /* two-queue build; nodes 0..nl-1 leaves, nl.. internal */
    uint64_t w[576];
    int parent[576];
    for (int i = 0; i < nl; i++) w[i] = leaves[i].f;
    int qa = 0, qb = nl, nn = nl;
    while ((nl - qa) + (nn - qb) >= 2) {
        int pick[2];
        for (int k = 0; k < 2; k++) {
            if (qa < nl && (qb >= nn || w[qa] <= w[qb]))
                pick[k] = qa++;
            else
                pick[k] = qb++;
        }
        w[nn] = w[pick[0]] + w[pick[1]];
        parent[pick[0]] = nn;
        parent[pick[1]] = nn;
        nn++;
    }
    int root = nn - 1;
    int depth[576];
    depth[root] = 0;
    for (int i = root - 1; i >= 0; i--)
        depth[i] = depth[parent[i]] + 1;
    /* clamp + Kraft repair */
    uint32_t kraft = 0; /* in units of 2^-maxbits */
    int L[288];
    for (int i = 0; i < nl; i++) {
        L[i] = depth[i] > maxbits ? maxbits : (depth[i] < 1 ? 1 : depth[i]);
        kraft += 1u << (maxbits - L[i]);
    }
    uint32_t one = 1u << maxbits;
    /* leaves[] ascending freq: lengthen the rarest symbols first while over-subscribed */
    while (kraft > one) {
        for (int i = 0; i < nl && kraft > one; i++)
            if (L[i] < maxbits) {
                kraft -= 1u << (maxbits - L[i] - 1);
                L[i]++;
            }
    }
    /* use up slack: shorten the most frequent symbols that fit */
    for (int i = nl - 1; i >= 0; i--)
        while (L[i] > 1 && kraft + (1u << (maxbits - L[i])) <= one) {
            kraft += 1u << (maxbits - L[i]);
            L[i]--;
        }
    for (int i = 0; i < nl; i++)
        lens[leaves[i].s] = (uint8_t)L[i];
}

static void huff_codes(const uint8_t *lens, int n, uint16_t *codes) {
    uint16_t bl_count[16] = {0}, next[16];
    for (int i = 0; i < n; i++) bl_count[lens[i]]++;
    bl_count[0] = 0;
    uint16_t code = 0;
    for (int b = 1; b <= 15; b++) {
        code = (uint16_t)((code + bl_count[b - 1]) << 1);
        next[b] = code;
    }
    for (int i = 0; i < n; i++)
        codes[i] = lens[i] ? (uint16_t)rev_bits(next[lens[i]]++, lens[i]) : 0;
}

static int len_symbol(int len) {
    for (int s = 28; s >= 0; s--)
        if (len >= k_len_base[s]) return s;
    return 0;
}
static int dist_symbol(int d) {
    for (int s = 29; s >= 0; s--)
        if (d >= k_dist_base[s]) return s;
    return 0;
}

typedef struct { uint16_t len; uint16_t dist; } orc_tok; /* dist==0 -> literal in len */

static void emit_block(orc_bw *w, const orc_tok *tok, size_t ntok, int final) {
    uint32_t lf[286] = {0}, df[30] = {0};
    for (size_t i = 0; i < ntok; i++) {
        if (tok[i].dist == 0) {
            lf[tok[i].len]++;
        } else {
            lf[257 + len_symbol(tok[i].len)]++;
            df[dist_symbol(tok[i].dist)]++;
        }
    }
    lf[256] = 1;
    uint8_t ll[288], dl[32];
    uint16_t lc[288], dc[32];
    huff_lengths(lf, 286, 15, ll);
    huff_lengths(df, 30, 15, dl);
    huff_codes(ll, 286, lc);
    huff_codes(dl, 30, dc);
    /* header: emit all 286 + 30 lengths literally through the code-length code */
    static const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    uint32_t cf[19] = {0};
    for (int i = 0; i < 286; i++) cf[ll[i]]++;
    for (int i = 0; i < 30; i++) cf[dl[i]]++;
    uint8_t cl[19];
    uint16_t cc[19];
    huff_lengths(cf, 19, 7, cl);
    huff_codes(cl, 19, cc);
    bw_put(w, (uint32_t)final, 1);
    bw_put(w, 2, 2);
    bw_put(w, 286 - 257, 5);
    bw_put(w, 30 - 1, 5);
    bw_put(w, 19 - 4, 4);
    for (int i = 0; i < 19; i++) bw_put(w, cl[order[i]], 3);
    for (int i = 0; i < 286; i++) bw_put(w, cc[ll[i]], cl[ll[i]]);
    for (int i = 0; i < 30; i++) bw_put(w, cc[dl[i]], cl[dl[i]]);
    for (size_t i = 0; i < ntok; i++) {
        if (tok[i].dist == 0) {
            bw_put(w, lc[tok[i].len], ll[tok[i].len]);
        } else {
            int ls = len_symbol(tok[i].len);
            bw_put(w, lc[257 + ls], ll[257 + ls]);
            bw_put(w, (uint32_t)(tok[i].len - k_len_base[ls]), k_len_extra[ls]);
            int ds = dist_symbol(tok[i].dist);
            bw_put(w, dc[ds], dl[ds]);
            bw_put(w, (uint32_t)(tok[i].dist - k_dist_base[ds]), k_dist_extra[ds]);
        }
    }
    bw_put(w, lc[256], ll[256]);
}

size_t orc_deflate_bound(size_t in_len) {
    return in_len + (in_len / 16383 + 1) * 5 + 1024;
}

int64_t orc_deflate(const uint8_t *in, size_t in_len, uint8_t *out, size_t out_cap, int level, int wrap) {
    orc_bw w;
    memset(&w, 0, sizeof(w));
    w.out = out;
    w.cap = out_cap;
    if (wrap == ORC_WRAP_GZIP) {
        static const uint8_t hdr[10] = {0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 0, 3};
        for (int i = 0; i < 10; i++) bw_put(&w, hdr[i], 8);
        if (level == 9) w.out[8] = 2;
        else if (level < 2) w.out[8] = 4;
    } else if (wrap == ORC_WRAP_ZLIB) {
        bw_put(&w, 0x78, 8);
        bw_put(&w, 0x9c, 8);
    }
    if (level == 0 || in_len == 0) {
        size_t pos = 0;
        do {
            size_t n = in_len - pos > 65535 ? 65535 : in_len - pos;
            int final = (pos + n == in_len);
            if (in_len == 0) { /* zlib emits a fixed block holding only EOB: 03 00 */
                bw_put(&w, 1, 1); bw_put(&w, 1, 2); bw_put(&w, 0, 7);
                break;
            }
            bw_put(&w, (uint32_t)final, 1);
            bw_put(&w, 0, 2);
            bw_align(&w);
            bw_put(&w, (uint32_t)n, 16);
            bw_put(&w, (uint32_t)(n ^ 0xffff), 16);
            for (size_t i = 0; i < n; i++) bw_put(&w, in[pos + i], 8);
            pos += n;
        } while (pos < in_len);
    } else {
        const int HB = 15;
        int max_chain = level <= 1 ? 4 : level <= 3 ? 16 : level <= 6 ? 64 : 256;
        int32_t *head = (int32_t *)malloc(sizeof(int32_t) << HB);
        int32_t *prev = (int32_t *)malloc(sizeof(int32_t) * 32768);
        const size_t TOKMAX = 65536;
        orc_tok *tok = (orc_tok *)malloc(sizeof(orc_tok) * TOKMAX);
        if (!head || !prev || !tok) { free(head); free(prev); free(tok); return ORC_MEM_ERROR; }
        memset(head, 0xff, sizeof(int32_t) << HB);
        size_t ntok = 0, pos = 0;
        while (pos < in_len) {
            int best_len = 0, best_dist = 0;
            if (pos + 3 <= in_len) {
                uint32_t h = ((uint32_t)in[pos] | ((uint32_t)in[pos + 1] << 8) | ((uint32_t)in[pos + 2] << 16)) * 0x9E3779B1u >> (32 - HB);
                int32_t cand = head[h];
                int chain = max_chain;
                size_t maxl = in_len - pos > 258 ? 258 : in_len - pos;
                while (cand >= 0 && pos - (size_t)cand <= 32768 && chain-- > 0) {
                    size_t l = 0;
                    while (l < maxl && in[cand + l] == in[pos + l]) l++;
                    if ((int)l > best_len) { best_len = (int)l; best_dist = (int)(pos - (size_t)cand); }
                    if (l == maxl) break;
                    int32_t nx = prev[cand & 32767];
                    if (nx >= cand) break;
                    cand = nx;
                }
                prev[pos & 32767] = head[h];
                head[h] = (int32_t)pos;
            }
            if (best_len >= 3 && !(best_len == 3 && best_dist > 4096)) {
                tok[ntok].len = (uint16_t)best_len;
                tok[ntok].dist = (uint16_t)best_dist;
                ntok++;
                for (int k = 1; k < best_len; k++) { /* keep the chains warm */
                    size_t p = pos + (size_t)k;
                    if (p + 3 <= in_len) {
                        uint32_t h = ((uint32_t)in[p] | ((uint32_t)in[p + 1] << 8) | ((uint32_t)in[p + 2] << 16)) * 0x9E3779B1u >> (32 - HB);
                        prev[p & 32767] = head[h];
                        head[h] = (int32_t)p;
                    }
                }
                pos += (size_t)best_len;
            } else {
                tok[ntok].len = in[pos];
                tok[ntok].dist = 0;
                ntok++;
                pos++;
            }
            if (ntok == TOKMAX || pos >= in_len) {
                emit_block(&w, tok, ntok, pos >= in_len);
                ntok = 0;
            }
        }
        free(head); free(prev); free(tok);
    }
    bw_align(&w);
    if (wrap == ORC_WRAP_GZIP) {
        uint32_t crc = orc_crc32_update(0, in, in_len);
        bw_put(&w, crc & 0xffff, 16); bw_put(&w, crc >> 16, 16);
        bw_put(&w, (uint32_t)in_len & 0xffff, 16); bw_put(&w, ((uint32_t)in_len) >> 16, 16);
    } else if (wrap == ORC_WRAP_ZLIB) {
        uint32_t ad = orc_adler32_update(1, in, in_len);
        bw_put(&w, ad >> 24, 8); bw_put(&w, (ad >> 16) & 0xff, 8); bw_put(&w, (ad >> 8) & 0xff, 8); bw_put(&w, ad & 0xff, 8);
    }
    if (w.overflow)
        return ORC_BUF_ERROR;
    return (int64_t)w.pos;
}
