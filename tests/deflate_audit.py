"""An independent look at every block the deflate kernel writes (TEST SUPPORT: no GPU, no product code).

decode() walks a raw DEFLATE stream (RFC 1951) block by block and returns what each block holds: its bit span, BFINAL and
BTYPE; for a stored block LEN, NLEN and the padding bits; for a Huffman block the header (HLIT, HDIST, HCLEN, the 19
code-length-code lengths, the 286 + 30 code lengths, the header size in bits) and the token list (a literal byte, or a
(length, distance) pair) up to the end of block. It rejects what zlib's inflate rejects: incomplete or over-subscribed codes
(zlib's exceptions kept: one code of length 1, no distance code at all), symbols 286/287 and distances 30/31, a distance
further back than the output, a bad NLEN, block type 3, a truncated stream. Bits are read through a byte-indexed window, so a
long stream costs linear time.

The check_* functions state the rules of minizip-ng_b200/csrc/deflate_kernel.cuh (line numbers cite that file) as
assertions on one output slot (= one chunk). The code lengths and header bits of a Huffman block are set against the kernel's
own code builder (block_build_codes, run through tests/emu/df_codes_pair.cuh on the emulator or on the GPU): given the
block's token histogram, every bit of the header is determined, and so is the choice between a stored and a Huffman block.
"""
import numpy as np

from deflate_craft import CL_ORDER, DBASE, DEXT, FIXED_DIST, FIXED_LIT, LBASE, LEXT

# ---- the kernel's constants (deflate_kernel.cuh) --------------------------------------------------------------------------------
DF_UNIT = 32768      # :47: one LZ77 domain = one block
DF_MINMATCH = 4      # :52
CL_LENS = 0x12ddad91b725bb4  # :253: the static code-length code, 3 bits per symbol 0..18
KERNEL_CL_LENS = [(CL_LENS >> (3 * s)) & 7 for s in range(19)]
FLAG_FINAL, FLAG_DICT = 1, 2  # :59-61

# ---- the builder's input and output layout (tests/emu/df_codes_pair.cuh) -------------------------------------------------------
HIST_WORDS = 288 + 32 + 256  # literal/length counts | distance counts | second copy of the literal counts
OUT_LENS, OUT_BITS, OUT_STAGE, OUT_HDRBITS = 320, 400, 480, 576


class DeflateError(ValueError):
    """the stream is one zlib's inflate rejects"""


# length 3..258 -> (symbol 0..28, extra bits); distance 1..32768 -> (symbol, extra bits)
LSYM = [None] * 259
for _s in range(29):
    for _l in range(LBASE[_s], min(LBASE[_s] + (1 << LEXT[_s]), 259)):
        LSYM[_l] = (_s, LEXT[_s])
LSYM[258] = (28, 0)
DSYM = [None] * 32769
for _s in range(30):
    for _d in range(DBASE[_s], min(DBASE[_s] + (1 << DEXT[_s]), 32769)):
        DSYM[_d] = (_s, DEXT[_s])


class Block:
    """one decoded block; fields that do not apply to its type stay None"""
    __slots__ = ("start", "end", "bfinal", "btype", "out_start", "out_end", "stored_len", "stored_nlen", "pad_bits", "hlit", "hdist",
                 "hclen", "cl_lens", "ll_lens", "d_lens", "hdr_bits", "tokens", "eob_pos")

    def __init__(self, **kw):
        for k in self.__slots__:
            setattr(self, k, kw.get(k))

    def __repr__(self):
        return "Block(bits %d..%d, BFINAL %d, BTYPE %d, out %d..%d)" % (self.start, self.end, self.bfinal, self.btype, self.out_start,
                                                                       self.out_end)


def _table(lens, kind):
    """(lookup list indexed by the next `maxbits` stream bits -> symbol << 4 | length, -1 for no code; maxbits) of a canonical code.
    kind: "codes" (must be complete), "lens" or "dists" (incomplete only as one code of length 1, as zlib allows)"""
    count = [0] * 16
    for n in lens:
        count[n] += 1
    count[0] = 0
    left = 1
    for n in range(1, 16):
        left = (left << 1) - count[n]
        if left < 0:
            raise DeflateError("over-subscribed %s code" % kind)
    maxb = max(lens) if any(lens) else 0
    if maxb == 0:
        if kind != "dists":
            raise DeflateError("empty %s code" % kind)
        return [-1], 0
    if left > 0 and (kind == "codes" or maxb != 1):
        raise DeflateError("incomplete %s code" % kind)
    nxt, code = [0] * 16, 0
    for n in range(1, 16):
        code = (code + count[n - 1]) << 1
        nxt[n] = code
    tab = [-1] * (1 << maxb)
    for sym, n in enumerate(lens):
        if n:
            c = nxt[n]
            nxt[n] += 1
            rev = int(format(c, "0%db" % n)[::-1], 2)
            ent = (sym << 4) | n
            for i in range(rev, 1 << maxb, 1 << n):
                tab[i] = ent
    return tab, maxb


_FIXED = None


def _fixed_tables():
    global _FIXED
    if _FIXED is None:
        _FIXED = (_table(FIXED_LIT, "lens"), _table(FIXED_DIST, "dists"))
    return _FIXED


def decode(data, window=b"", bit=0, until_final=True):
    """Walk the raw DEFLATE stream `data` from bit `bit`. `window` = the bytes in front of it (a preset dictionary / the stream so
    far). Stops after the block with BFINAL, or (until_final=False) also where a block ends at the last byte. Returns
    (blocks, plain bytes, end bit); raises DeflateError for what zlib rejects."""
    d = bytes(data)
    nbits = len(d) * 8
    out = bytearray(window)
    base = len(out)
    blocks = []
    p = bit

    def need(n):
        if p + n > nbits:
            raise DeflateError("truncated stream")

    def bits(n):
        nonlocal p
        need(n)
        q = p >> 3
        v = (int.from_bytes(d[q:q + 5], "little") >> (p & 7)) & ((1 << n) - 1)
        p += n
        return v

    while True:
        start = p
        bfinal = bits(1)
        btype = bits(2)
        blk = Block(start=start, bfinal=bfinal, btype=btype, out_start=len(out) - base)
        if btype == 0:
            pad = (-p) & 7
            blk.pad_bits = bits(pad) if pad else 0
            n, nn = bits(16), bits(16)
            blk.stored_len, blk.stored_nlen = n, nn
            if nn != n ^ 0xFFFF:
                raise DeflateError("invalid stored block lengths")
            need(8 * n)
            q = p >> 3
            out += d[q:q + n]
            p += 8 * n
        elif btype == 3:
            raise DeflateError("invalid block type")
        else:
            if btype == 1:
                (ltab, lmax), (dtab, dmax) = _fixed_tables()
            else:
                hlit, hdist, hclen = bits(5) + 257, bits(5) + 1, bits(4) + 4
                if hlit > 286 or hdist > 30:
                    raise DeflateError("too many length or distance symbols")
                cl = [0] * 19
                for i in range(hclen):
                    cl[CL_ORDER[i]] = bits(3)
                ctab, cmax = _table(cl, "codes")
                lens = []
                while len(lens) < hlit + hdist:
                    q = p >> 3
                    e = ctab[(int.from_bytes(d[q:q + 3], "little") >> (p & 7)) & ((1 << cmax) - 1)]
                    if e < 0:
                        raise DeflateError("invalid code lengths set")
                    need(e & 15)
                    p += e & 15
                    sym = e >> 4
                    if sym < 16:
                        lens.append(sym)
                        continue
                    if sym == 16:
                        if not lens:
                            raise DeflateError("invalid bit length repeat")
                        rep, v = 3 + bits(2), lens[-1]
                    elif sym == 17:
                        rep, v = 3 + bits(3), 0
                    else:
                        rep, v = 11 + bits(7), 0
                    if len(lens) + rep > hlit + hdist:
                        raise DeflateError("invalid bit length repeat")
                    lens += [v] * rep
                ll, dl = lens[:hlit], lens[hlit:]
                if ll[256] == 0:
                    raise DeflateError("invalid code -- missing end-of-block")
                (ltab, lmax), (dtab, dmax) = _table(ll, "lens"), _table(dl, "dists")
                blk.hlit, blk.hdist, blk.hclen, blk.cl_lens = hlit, hdist, hclen, cl
                blk.ll_lens, blk.d_lens = ll + [0] * (286 - hlit), dl + [0] * (30 - hdist)
                blk.hdr_bits = p - start
            lmask, dmask = (1 << lmax) - 1, (1 << dmax) - 1
            toks = []
            while True:
                q = p >> 3
                w = int.from_bytes(d[q:q + 8], "little") >> (p & 7)  # >= 57 bits: a whole token (<= 48 bits)
                e = ltab[w & lmask]
                if e < 0:
                    raise DeflateError("invalid literal/length code")
                n = e & 15
                sym = e >> 4
                if sym < 256:
                    p += n
                    if p > nbits:
                        raise DeflateError("truncated stream")
                    out.append(sym)
                    toks.append(sym)
                    continue
                if sym == 256:
                    blk.eob_pos = p
                    p += n
                    if p > nbits:
                        raise DeflateError("truncated stream")
                    break
                sym -= 257
                if sym >= 29:
                    raise DeflateError("invalid literal/length code")
                w >>= n
                eb = LEXT[sym]
                length = LBASE[sym] + (w & ((1 << eb) - 1))
                w >>= eb
                p += n + eb
                e = dtab[w & dmask]
                if e < 0 or (e >> 4) >= 30:
                    raise DeflateError("invalid distance code")
                n, ds = e & 15, e >> 4
                w >>= n
                eb = DEXT[ds]
                dist = DBASE[ds] + (w & ((1 << eb) - 1))
                p += n + eb
                if p > nbits:
                    raise DeflateError("truncated stream")
                if dist > len(out):
                    raise DeflateError("invalid distance too far back")
                if dist >= length:
                    s = len(out) - dist
                    out += out[s:s + length]
                else:
                    pat = out[-dist:]
                    out += (pat * (length // dist + 1))[:length]
                toks.append((length, dist))
            blk.tokens = toks
        blk.end = p
        blk.out_end = len(out) - base
        blocks.append(blk)
        if bfinal or (not until_final and p >= nbits - 7):
            break
    return blocks, bytes(out[base:]), p


def expand(tokens, window=b""):
    """the bytes a token list stands for"""
    out = bytearray(window)
    for t in tokens:
        if isinstance(t, int):
            out.append(t)
        else:
            length, dist = t
            for _ in range(length):
                out.append(out[-dist])
    return bytes(out[len(window):])


def histogram(tokens):
    """the block's symbol counts in the builder's input layout (DFC_HIST_WORDS): literal/length counts with the end of block's 1,
    distance counts at 288; the whole count in the first copy, the second literal copy (which the builder adds) left at zero"""
    ll = [0] * 288
    dd = [0] * 32
    for t in tokens:
        if isinstance(t, int):
            ll[t] += 1
        else:
            ll[257 + LSYM[t[0]][0]] += 1
            dd[DSYM[t[1]][0]] += 1
    ll[256] += 1
    h = np.zeros(HIST_WORDS, dtype=np.uint32)
    h[:288] = ll
    h[288:320] = dd
    return h


def merged(h):
    """a histogram with the second literal copy folded into the first (what the builder counts)"""
    h = np.array(h, dtype=np.uint32)
    h[:256] += h[320:576]
    h[320:576] = 0
    return h


class Built:
    """one row of the builder's output (df_codes_pair.cuh): code lengths, bits per symbol, header staging and size"""

    def __init__(self, row):
        row = np.ascontiguousarray(row, dtype=np.uint32)
        lens = row[OUT_LENS:OUT_BITS].view(np.uint8)
        bits = row[OUT_BITS:OUT_STAGE].view(np.uint8)
        self.ll_lens, self.d_lens = [int(x) for x in lens[:286]], [int(x) for x in lens[288:318]]
        self.ll_bits, self.d_bits = bits[:288].astype(np.int64), bits[288:320].astype(np.int64)
        self.stage = int.from_bytes(row[OUT_STAGE:OUT_HDRBITS].tobytes(), "little")
        self.hdr_bits = int(row[OUT_HDRBITS])
        self.hlit = max(i for i in range(286) if self.ll_lens[i]) + 1
        nz = [i for i in range(30) if self.d_lens[i]]
        self.hdist = nz[-1] + 1 if nz else 1

    def dyn_bits(self, h):
        """:1261-1263: the block's size as a Huffman block: header + every token's code word and extra bits + the end of block"""
        h = merged(h).astype(np.int64)
        tok = int((h[:288] * self.ll_bits).sum() - h[256] * self.ll_bits[256] + (h[288:320] * self.d_bits).sum())
        return self.hdr_bits + tok + self.ll_lens[256]


def stored_bits(start, ulen):
    """:1264: a stored block's size when it starts at bit `start` (only start mod 8 matters: the slot is flushed in 16-byte units)"""
    return (((start + 3 + 7) & ~7) - start) + 32 + ulen * 8


def posfin(blk):
    """the builder's header position for this block: its bit offset in the kernel's staging buffer (flushed in 128-bit units)"""
    return (blk.start & 127) | (blk.bfinal << 31)


# ---- a slot, decoded and checked --------------------------------------------------------------------------------------------------
class Slot:
    """one chunk's output slot: the input it stands for, its flags and level, its blocks. `window` = the bytes in front of the
    chunk that it may refer to (DF_FLAG_DICT at levels 6-9, :88-92 and :831), else empty."""

    def __init__(self, slot, chunk, level, flags, window=b""):
        self.slot, self.chunk, self.level, self.flags, self.window = bytes(slot), bytes(chunk), level, flags, bytes(window)
        self.final = bool(flags & FLAG_FINAL)
        self.blocks, out, self.end = decode(self.slot, self.window, until_final=self.final)
        assert out == self.chunk, "slot does not decode to its chunk"
        self.units = self.blocks if self.final else self.blocks[:-1]  # the blocks that carry the chunk's units (no sync marker)


def check_framing(s):
    """:839-849, :1377-1396"""
    b = s.blocks
    if s.final:
        # BFINAL on the last block only; zero bits up to the next byte, which is the slot's end (out_len)
        assert [x.bfinal for x in b] == [0] * (len(b) - 1) + [1], "BFINAL must be set on the last block only"
        pad = (-s.end) & 7
        assert (s.end + pad) // 8 == len(s.slot), "out_len is not the decoded end rounded up to a byte"
        if pad:
            assert s.slot[-1] >> (8 - pad) == 0, "pad bits after the final block are not zero"
        if not s.chunk:
            assert s.slot == b"\x03\x00", "an empty final chunk is 03 00 (:843-847)"
    else:
        # :1389-1392: an empty stored block, zero padded, ending the slot: ... 00 00 FF FF
        m = b[-1]
        assert not any(x.bfinal for x in b), "BFINAL in a non-final chunk"
        assert m.btype == 0 and m.stored_len == 0 and m.stored_nlen == 0xFFFF and m.pad_bits == 0, "no empty stored block at the end"
        assert m.end == 8 * len(s.slot) and s.slot[-4:] == b"\x00\x00\xff\xff", "the sync marker does not end the slot"
        assert s.slot[(m.start >> 3)] >> (m.start & 7) == 0
        assert m.out_start == len(s.chunk)


def check_partition(s):
    """:836, :851-856: one block per 32 KiB unit, in order; the last unit takes the rest. (The comment at :33-34 once promised a
    second block for a unit with too many entries; the code has no such path, so one block per unit is the rule.)"""
    n = len(s.chunk)
    if n == 0:
        if s.final:
            assert len(s.units) == 1 and s.units[0].btype == 1 and s.units[0].tokens == []
        else:
            assert s.units == []
        return
    nunits = (n + DF_UNIT - 1) // DF_UNIT
    assert len(s.units) == nunits, "%d blocks for %d units" % (len(s.units), nunits)
    for u, blk in enumerate(s.units):
        assert blk.btype in (0, 2), "block type %d: the kernel writes stored and dynamic blocks only" % blk.btype
        assert (blk.out_start, blk.out_end) == (u * DF_UNIT, min(n, (u + 1) * DF_UNIT)), "block %d covers %d..%d" % (
            u, blk.out_start, blk.out_end)
        if s.level == 0:
            assert blk.btype == 0, "level 0 writes stored blocks only"


def check_matches(s):
    """lengths 3..258: the parse finds matches of DF_MINMATCH (4, :52) or more, but a match whose front an earlier span's match
    already covers is trimmed, and 3 bytes left of it stay a match (:601-609); at levels 1-5 a match stays inside its unit (:10); at levels 6-9 it reaches back at most
    into the previous 32 KiB: the chunk's unit before, or with DF_FLAG_DICT (chunk offset >= 32 KiB) the bytes in front of the
    chunk (:88-92, :989)"""
    for u, blk in enumerate(s.units):
        if blk.btype != 2:
            continue
        pos = blk.out_start
        if s.level <= 5:
            lowest = u * DF_UNIT
        else:
            lowest = (u - 1) * DF_UNIT if u else -len(s.window)
        for t in blk.tokens:
            if isinstance(t, int):
                pos += 1
                continue
            length, dist = t
            assert DF_MINMATCH - 1 <= length <= 258, "match length %d" % length
            assert pos - dist >= lowest, "unit %d: match at %d, distance %d reaches before %d (level %d)" % (u, pos, dist, lowest, s.level)
            pos += length


def dynamic_hists(s):
    """[(block, histogram of its tokens)] for the slot's Huffman blocks"""
    return [(blk, histogram(blk.tokens)) for blk in s.units if blk.btype == 2]


def check_header(blk, built):
    """:246-253, :474-536: the static code-length code (HCLEN 19), HLIT/HDIST trimmed to the last used symbol, the code lengths
    the builder gives for the block's histogram, the header size the builder counts (BB_HDRBITS), and every header bit as the
    builder staged it"""
    assert blk.hclen == 19 and blk.cl_lens == KERNEL_CL_LENS, "code-length code is not the kernel's static one"
    assert (blk.hlit, blk.hdist) == (built.hlit, built.hdist), "HLIT/HDIST %d/%d, the builder's lengths give %d/%d" % (
        blk.hlit, blk.hdist, built.hlit, built.hdist)
    assert blk.ll_lens == built.ll_lens, "literal/length code lengths differ from the builder's for this histogram"
    assert blk.d_lens == built.d_lens, "distance code lengths differ from the builder's for this histogram"
    assert blk.hdr_bits == built.hdr_bits, "header of %d bits, the builder counts %d" % (blk.hdr_bits, built.hdr_bits)


def check_header_bits(slot_bytes, blk, built):
    """the header's bits in the stream are the ones the builder staged at the same bit offset"""
    n = built.hdr_bits
    got = (int.from_bytes(slot_bytes, "little") >> blk.start) & ((1 << n) - 1)
    want = (built.stage >> (blk.start & 127)) & ((1 << n) - 1)
    assert got == want, "header bits differ from the builder's staging"


def check_stored_rule(blk, ulen, h, built):
    """:1261-1265: a unit is stored iff its Huffman coding would take at least as many bits as the stored block at the same place.
    h = the unit's token histogram (the block's own for a Huffman block; for a stored block the parse from elsewhere)."""
    dyn, st = built.dyn_bits(h), stored_bits(blk.start, ulen)
    if blk.btype == 2:
        assert dyn < st, "Huffman block of %d bits where a stored one takes %d" % (dyn, st)
        assert blk.end - blk.start == dyn, "Huffman block is %d bits, the histogram and builder say %d" % (blk.end - blk.start, dyn)
    else:
        assert dyn >= st, "stored block of %d bits where the Huffman block takes %d" % (st, dyn)


def check_slot(s):
    """every rule that needs no code builder"""
    check_framing(s)
    check_partition(s)
    check_matches(s)


def check_codes(slots, builder, hists=None):
    """the header and stored-decision rules for every unit of `slots` ([Slot]). builder(hists, posfin) -> output rows (the "new"
    builder of df_codes_pair.cuh). hists: optional {(slot index, unit): histogram} of the same parse from elsewhere (the
    emulator's capture); a Huffman block's own tokens must give the same histogram, and a stored block is judged by it.
    Returns the number of units checked against the stored rule."""
    jobs = []  # (slot, unit, block, histogram)
    for i, s in enumerate(slots):
        if s.level == 0:
            continue
        for u, blk in enumerate(s.units):
            h = hists.get((i, u)) if hists is not None else None
            if blk.btype == 2:
                own = histogram(blk.tokens)
                if h is not None:
                    assert (merged(h) == own).all(), "slot %d unit %d: the block's tokens are not the parse the builder was given" % (i, u)
                h = own
            if h is not None:
                jobs.append((s, u, blk, h))
    if not jobs:
        return 0
    rows = builder(np.stack([j[3] for j in jobs]), np.array([posfin(j[2]) for j in jobs], dtype=np.uint32))
    for (s, u, blk, h), row in zip(jobs, rows):
        built = Built(row)
        if blk.btype == 2:
            check_header(blk, built)
            check_header_bits(s.slot, blk, built)
        check_stored_rule(blk, blk.out_end - blk.out_start, h, built)
    return len(jobs)
