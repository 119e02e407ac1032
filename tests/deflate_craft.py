"""Hand-built raw DEFLATE streams (RFC 1951) for decoder conformance tests.

Stream writes blocks bit by bit, so a test can state exactly what a stream holds: stored blocks with any LEN and NLEN, fixed
blocks with any symbol (286/287 and distances 30/31 included), and dynamic blocks whose code lengths, code-length code, HCLEN and
header encoding (plain lengths or repeat codes 16/17/18, or an explicit list of header operations) are given or derived. Stream
also keeps the bytes a correct decoder produces, as far as the stream is valid.

Tokens of a Huffman block:
  int 0..255                    a literal
  ("m", length, distance)       a match; symbols and extra bits follow from the values
  ("M", lsym, lext, dsym, dext) a match with its symbols and extra-bit values given (lsym 284 + 31 = length 258)
  ("s", sym)                    a bare literal/length symbol and nothing after it (286, 287, or 256 in the middle of a block)
EOB is written at the end of each block unless eob=False.
"""
import heapq

LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEXT = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193,
         12289, 16385, 24577, 32769, 49153]
DEXT = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13, 14, 14]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
CL_EXTRA = {16: (2, 3), 17: (3, 3), 18: (7, 11)}  # repeat code -> (extra bits, least count)
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 32


def len_sym(length):
    """(symbol, extra value) of a match length 3..258 as zlib writes it (258 is symbol 285)"""
    if length == 258:
        return 285, 0
    i = max(i for i in range(28) if LBASE[i] <= length)
    return 257 + i, length - LBASE[i]


def dist_sym(dist):
    i = max(i for i in range(30) if DBASE[i] <= dist)
    return i, dist - DBASE[i]


def canonical(lens):
    """RFC 1951 3.2.2 codes (as integers, MSB first) for a list of code lengths; 0 = unused"""
    count = [0] * 16
    for n in lens:
        count[n] += 1
    count[0] = 0
    code, nxt = 0, [0] * 16
    for b in range(1, 16):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    codes = []
    for n in lens:
        codes.append(nxt[n] & ((1 << n) - 1) if n else None)
        if n:
            nxt[n] += 1
    return codes


def huffman_lengths(freq, limit):
    """code lengths (at most `limit`) of a Huffman code for the symbols with freq > 0; one used symbol gets a partner so the code is
    complete"""
    used = [i for i, f in enumerate(freq) if f]
    if len(used) == 1:
        used.append(0 if used[0] else 1)
    f = [max(freq[i], 1) for i in used]
    while True:
        heap = [(f[k], k, [k]) for k in range(len(used))]
        heapq.heapify(heap)
        depth = [0] * len(used)
        n = len(used)
        while len(heap) > 1:
            a, b = heapq.heappop(heap), heapq.heappop(heap)
            for k in a[2] + b[2]:
                depth[k] += 1
            heapq.heappush(heap, (a[0] + b[0], n, a[2] + b[2]))
            n += 1
        if max(depth) <= limit:
            break
        f = [(x + 1) // 2 for x in f]  # flatten the frequencies until the tree is shallow enough
    lens = [0] * len(freq)
    for k, i in enumerate(used):
        lens[i] = depth[k]
    return lens


def chain_lengths(n_syms):
    """lengths 1, 2, ..., n-1, n-1: a complete code whose longest two codes are n-1 bits (n <= 16)"""
    return list(range(1, n_syms)) + [n_syms - 1]


def rle_ops(lens):
    """zlib-style header operations for a list of code lengths: (symbol, extra value) with repeat codes 16/17/18"""
    ops, i, prev = [], 0, None
    while i < len(lens):
        v = lens[i]
        run = 1
        while i + run < len(lens) and lens[i + run] == v:
            run += 1
        if v == 0 and run >= 3:
            n = min(run, 138)
            ops.append((18, n - 11) if n >= 11 else (17, n - 3))
        elif v != 0 and v == prev and run >= 3:
            n = min(run, 6)
            ops.append((16, n - 3))
        else:
            n = 1
            ops.append((v, 0))
        prev = v
        i += n
    return ops


def plain_ops(lens):
    return [(v, 0) for v in lens]


class Stream:
    def __init__(self):
        self.acc = 0
        self.nbits = 0
        self.out = bytearray()  # what a correct decoder produces (up to the first invalid token)
        self.valid = True

    # ---- bits ---------------------------------------------------------------------------------------------------------------
    def bits(self, value, n):
        assert 0 <= value < (1 << n) or n == 0
        self.acc |= value << self.nbits
        self.nbits += n

    def code(self, c, n):
        """a Huffman code: sent most significant bit first"""
        self.bits(int(format(c, "0%db" % n)[::-1], 2) if n else 0, n)

    def align(self):
        self.nbits = (self.nbits + 7) & ~7

    def bit_offset(self):
        return self.nbits & 7

    def getvalue(self):
        return self.acc.to_bytes((self.nbits + 7) // 8, "little")

    # ---- blocks -------------------------------------------------------------------------------------------------------------
    def stored(self, data, final=False, nlen=None, length=None):
        self.bits(int(final), 1)
        self.bits(0, 2)
        self.align()
        n = len(data) if length is None else length
        self.bits(n, 16)
        self.bits((n ^ 0xFFFF) if nlen is None else nlen, 16)
        for b in data:
            self.bits(b, 8)
        if nlen is not None and nlen != n ^ 0xFFFF:
            self.valid = False
        if self.valid:
            self.out += data
        return self

    def raw_block_type(self, btype, final=False):
        self.bits(int(final), 1)
        self.bits(btype, 2)
        if btype == 3:
            self.valid = False
        return self

    def fixed(self, tokens, final=False, eob=True):
        self.bits(int(final), 1)
        self.bits(1, 2)
        self._symbols(tokens, FIXED_LIT, FIXED_DIST, eob)
        return self

    def dynamic(self, tokens, litlens, distlens, final=False, ops=None, cl_lens=None, hclen=None, eob=True, header_only=False):
        """litlens / distlens: the lengths written (their sizes give HLIT and HDIST, 257..288 and 1..32). ops: "rle" (default),
        "plain" or a list of (symbol, extra value) header operations. cl_lens: 19 code-length-code lengths, derived from the
        operations by default; hclen: the number of them written (4..19), by default up to the last nonzero one in CL_ORDER."""
        nlit, ndist = len(litlens), len(distlens)
        all_lens = list(litlens) + list(distlens)
        if ops is None or ops == "rle":
            ops = rle_ops(all_lens)
        elif ops == "plain":
            ops = plain_ops(all_lens)
        if cl_lens is None:
            freq = [0] * 19
            for s, _ in ops:
                freq[s] += 1
            cl_lens = huffman_lengths(freq, 7)
        if hclen is None:
            hclen = max([4] + [k + 1 for k, s in enumerate(CL_ORDER) if cl_lens[s]])
        self.bits(int(final), 1)
        self.bits(2, 2)
        self.bits(nlit - 257, 5)
        self.bits(ndist - 1, 5)
        self.bits(hclen - 4, 4)
        for k in range(hclen):
            self.bits(cl_lens[CL_ORDER[k]], 3)
        cl_codes = canonical(cl_lens)
        for s, extra in ops:
            self.code(cl_codes[s], cl_lens[s])
            if s in CL_EXTRA:
                self.bits(extra, CL_EXTRA[s][0])
        if header_only:
            self.valid = False
            return self
        self._symbols(tokens, list(litlens) + [0] * (288 - nlit), list(distlens) + [0] * (32 - ndist), eob)
        return self

    def _symbols(self, tokens, llens, dlens, eob):
        lcodes, dcodes = canonical(llens), canonical(dlens)

        def put(codes, lens, sym):
            assert lens[sym], "symbol %d has no code" % sym
            self.code(codes[sym], lens[sym])
        for t in tokens:
            if isinstance(t, int):
                put(lcodes, llens, t)
                if self.valid:
                    self.out.append(t)
                continue
            if t[0] == "s":
                put(lcodes, llens, t[1])
                self.valid = False
                continue
            if t[0] == "m":
                (ls, le), (ds, de) = len_sym(t[1]), dist_sym(t[2])
            else:
                _, ls, le, ds, de = t
            put(lcodes, llens, ls)
            self.bits(le, LEXT[ls - 257] if ls < 286 else 0)
            put(dcodes, dlens, ds)
            self.bits(de, DEXT[ds])
            if ls >= 286 or ds >= 30:
                self.valid = False
                continue
            length, dist = LBASE[ls - 257] + le, DBASE[ds] + de
            if dist > len(self.out):
                self.valid = False
            if self.valid:
                for _ in range(length):
                    self.out.append(self.out[-dist])
        if eob:
            put(lcodes, llens, 256)


# ---- the conformance corpus -----------------------------------------------------------------------------------------------------
def text(n, seed=1):
    import random
    words = [b"inflate", b"the", b"block", b"of", b"code", b"length", b"stored", b"huffman", b"distance", b"window"]
    r, out = random.Random(seed), bytearray()
    while len(out) < n:
        out += r.choice(words) + b" "
    return bytes(out[:n])


def lengths_for(tokens):
    """Huffman code lengths (at most 15 bits) for the symbols a token list uses, EOB included; [0] when it has no match"""
    lf, df = [0] * 286, [0] * 30
    for t in tokens:
        if isinstance(t, int):
            lf[t] += 1
            continue
        (ls, _), (ds, _) = (len_sym(t[1]), dist_sym(t[2])) if t[0] == "m" else ((t[1], 0), (t[3], 0))
        lf[ls] += 1
        df[ds] += 1
    lf[256] += 1
    return huffman_lengths(lf, 15), (huffman_lengths(df, 15) if any(df) else [0])


def _every_length_distance():
    """every length symbol 257..285 and every distance symbol 0..29, each at its least and largest extra value"""
    toks = list(text(300)) + [("m", 258, 1)] * 130  # 33 KiB of history first
    for ls in range(257, 286):
        for le in sorted({0, (1 << LEXT[ls - 257]) - 1}):
            toks.append(("M", ls, le, 0, 0))
    for ds in range(30):
        for de in sorted({0, (1 << DEXT[ds]) - 1}):
            toks.append(("M", 284, 31, ds, de))
    return toks


def _long_codes(long_syms):
    """one dynamic block: its literal/length code has one code of each length 1..14 and two of 15 bits, on `long_syms`; its distance
    code over distances 1..256 has the same lengths (distance codes of 9..15 bits). Every code is used."""
    short = [s for s in list(b"etaoinsr") + [256, 257, 258, 259, 270, 285, ord("h"), ord("d")] if s not in long_syms][:14]
    order = short + list(long_syms)
    ll, dl = [0] * 286, [0] * 16
    for s, n in zip(order, chain_lengths(16)):
        ll[s] = n
    for s, n in zip(range(16), chain_lengths(16)):
        dl[s] = n
    lits = [s for s in order if s < 256]
    toks = [lits[i % len(lits)] for i in range(300)]
    for i, ls in enumerate(s for s in order if 256 < s):
        for ds in range(16):
            toks += [("M", ls, (1 << LEXT[ls - 257]) - 1 if i & 1 else 0, ds, (1 << DEXT[ds]) - 1 if i & 1 else 0)] + lits
    return Stream().dynamic(toks, ll, dl, final=True)


def valid_cases():
    """[(name, stream, plain bytes)]: streams zlib decodes"""
    cases = []

    def add(name, s):
        assert s.valid, name
        cases.append((name, s.getvalue(), bytes(s.out)))
    add("long-codes-literal-and-length", _long_codes([ord("z"), 270]))
    add("long-codes-eob-and-length", _long_codes([256, 285]))
    add("long-codes-literal-and-eob", _long_codes([ord("q"), 256]))
    toks = _every_length_distance()
    add("fixed-every-symbol-extreme", Stream().fixed(toks, final=True))
    ll, dl = lengths_for(toks)
    add("dynamic-every-symbol-extreme", Stream().dynamic(toks, ll, dl, final=True))
    add("dynamic-every-symbol-extreme-plain-header", Stream().dynamic(toks, ll, dl, final=True, ops="plain"))
    # degenerate code sets: one distance code of length 1 (incomplete), no distance code, EOB alone, HLIT 257 + HDIST 1
    ll = [0] * 258
    for c in (97, 98, 99, 256, 257):
        ll[c] = 3 if c != 97 else 1
    ll[97], ll[98], ll[99], ll[256], ll[257] = 1, 2, 3, 4, 4
    add("one-distance-code-of-length-1", Stream().dynamic([97, 98, 99, ("m", 3, 3), ("m", 3, 3), 97], ll, [0, 0, 1], final=True))
    add("one-distance-code-of-length-1-dist-1", Stream().dynamic([97, ("m", 3, 1), 98], ll, [1], final=True))
    add("no-distance-code", Stream().dynamic(list(b"abcabcabba"), [0] * 97 + [1, 2, 3] + [0] * 156 + [3], [0], final=True))
    add("eob-alone", Stream().dynamic([], [0] * 256 + [1], [0], final=True))
    add("eob-alone-then-stored", Stream().dynamic([], [0] * 256 + [1], [0]).stored(b"tail", final=True))
    ll = [8] * 252 + [0, 0, 0, 7, 7]  # lengths 7 and 8 only: HCLEN 6
    s = Stream().dynamic(list(range(252)) + [255, 255, 251], ll, [0], final=True)
    assert int.from_bytes(s.getvalue()[:3], "little") >> 13 & 15 == 2  # HCLEN - 4
    add("hlit257-hdist1-hclen6", s)
    # repeat codes: 16 x 6 and 18 x 138 (the most each repeats), and a 16 that runs from the literal/length lengths into the distances
    lens = [0] * 97 + [4] * 12 + [0] * 145 + [4] * 4  # 16 codes of 4 bits: literals a..l, 254, 255, EOB, length 3
    ops = [(18, 86), (4, 0), (16, 3), (16, 1), (4, 0), (18, 127), (17, 4), (4, 0), (16, 0), (1, 0)]
    add("repeat-16x6-18x138", Stream().dynamic(list(b"abcdefghijkl") * 5 + [254, 255, ("m", 3, 1)], lens, [1], final=True, ops=ops))
    ll = [0] * 97 + [4] * 14 + [0] * 145 + [4, 4]
    ops = [(18, 86), (4, 0), (16, 3), (16, 3), (4, 0), (18, 127), (17, 4), (4, 0), (16, 3), (16, 3), (16, 2)]
    add("repeat-across-lit-dist", Stream().dynamic(list(b"abcdefghijklmn") * 3 + [("m", 3, 1), ("m", 3, 4)], ll, [4] * 16, final=True,
                                                   ops=ops))
    ll = [0] * 97 + [4] * 14 + [0] * 145 + [4, 4, 0, 0]
    ops = [(18, 86), (4, 0), (16, 3), (16, 3), (4, 0), (18, 127), (17, 4), (4, 0), (4, 0), (17, 1), (1, 0), (1, 0)]
    add("zero-run-across-lit-dist", Stream().dynamic(list(b"abcdefghijklmn") * 3 + [("m", 3, 4), ("m", 3, 3)], ll, [0, 0, 1, 1],
                                                     final=True, ops=ops))
    t = text(3000)
    ll, dl = lengths_for(list(t))
    add("repeat-codes-zlib-style", Stream().dynamic(list(t), ll, dl, final=True))
    # stored blocks after a fixed block of 10 + 9k bits: the stored header at every bit offset; empty fixed blocks; a later final block
    big = text(65535, seed=7)
    for k in range(8):
        s = Stream().fixed([200] * k)
        add("stored-empty-at-bit-%d" % s.bit_offset(), s.stored(b"", final=True))
        s = Stream().fixed([200] * k)
        add("stored-65535-at-bit-%d" % s.bit_offset(), s.stored(big, final=True))
    add("empty-fixed", Stream().fixed([], final=True))
    add("empty-blocks-then-final", Stream().fixed([]).fixed([]).stored(b"").fixed([]).fixed([65], final=True))
    # matches at the edges: a distance equal to the bytes written so far, distances 1..3 at length 258
    toks = list(b"abcdefg") + [("m", 7, 7), ("m", 14, 14), ("m", 258, 28), ("m", 258, 1), 120, ("m", 258, 2), 121, ("m", 258, 3)]
    toks += [("m", 3, 1), ("m", 3, 2), ("m", 258, 552)]
    add("matches-at-the-edges-fixed", Stream().fixed(toks, final=True))
    ll, dl = lengths_for(toks)
    add("matches-at-the-edges-dynamic", Stream().dynamic(toks, ll, dl, final=True))
    # 300 blocks of mixed types
    import random
    r = random.Random(5)
    s = Stream()
    for i in range(300):
        toks = list(text(r.randrange(0, 10), seed=i))
        if len(s.out) + len(toks):
            toks.append(("m", 3 + r.randrange(100), 1 + r.randrange(len(s.out) + len(toks))))
        if i % 5 == 0:
            s.stored(text(r.randrange(0, 10), seed=i))
        elif i % 5 < 4 or i % 10 == 4:
            s.fixed(toks)
        else:
            ll, dl = lengths_for(toks)
            s.dynamic(toks, ll, dl, ops="plain" if i % 10 == 9 else "rle")
    add("300-mixed-blocks", s.fixed([65], final=True))
    return cases


def invalid_cases():
    """[(name, stream)]: streams zlib rejects with a data error"""
    cases = []

    def add(name, s):
        cases.append((name, s.getvalue()))
    t = text(600)
    good = lengths_for(list(t))[0][:257]
    hdr = dict(final=True, header_only=True)
    for nlit, ndist in ((287, 1), (288, 1), (257, 31), (257, 32)):
        add("hlit%d-hdist%d" % (nlit, ndist), Stream().dynamic([], good + [0] * (nlit - 257), [0] * ndist, **hdr))
    cl = huffman_lengths([1] * 19, 7)
    longest = cl.index(max(cl))
    add("cl-code-incomplete", Stream().dynamic([], good, [0], cl_lens=cl[:longest] + [0] + cl[longest + 1:], ops="plain", **hdr))
    add("cl-code-oversubscribed", Stream().dynamic([], good, [0], cl_lens=cl[:longest] + [1] + cl[longest + 1:], ops="plain", **hdr))
    add("cl-code-one-code", Stream().dynamic([], [0] * 257, [0], cl_lens=[0] * 18 + [1], ops="plain", **hdr))
    add("hclen4-no-eob", Stream().dynamic([], [0] * 257, [0], ops=[(18, 127), (18, 109)], hclen=4, cl_lens=[0] * 17 + [1, 1], **hdr))
    add("16-first", Stream().dynamic([], good, [0], ops=[(16, 0)] + rle_ops(good + [0])[1:], **hdr))
    add("18-past-hlit-hdist", Stream().dynamic([], good, [0], ops=rle_ops(good) + [(18, 0)], **hdr))
    add("16-past-hlit-hdist", Stream().dynamic([], good, [5, 5, 5], ops=rle_ops(good) + [(5, 0), (16, 0)], **hdr))
    add("no-eob-length", Stream().dynamic([], good[:256] + [0], [0], **hdr))
    longest = good.index(max(good))
    add("litlen-oversubscribed", Stream().dynamic([], good[:longest] + [1] + good[longest + 1:], [0], **hdr))
    add("litlen-incomplete", Stream().dynamic([], good[:longest] + [0] + good[longest + 1:], [0], **hdr))
    add("dist-oversubscribed", Stream().dynamic([], good, [1, 1, 1], **hdr))
    add("dist-incomplete-two-codes", Stream().dynamic([], good, [1, 2], **hdr))
    add("dist-one-code-of-length-2", Stream().dynamic([], good, [0, 2], **hdr))
    add("block-type-3", Stream().raw_block_type(3, final=True))
    add("block-type-3-after-fixed", Stream().fixed(list(b"ok")).raw_block_type(3, final=True))
    add("stored-bad-nlen", Stream().stored(b"abc", final=True, nlen=0xFFFF ^ 4))
    add("stored-bad-nlen-after-fixed", Stream().fixed(list(b"x")).stored(b"abc", final=True, nlen=0))
    for sym in (286, 287):
        add("fixed-symbol-%d" % sym, Stream().fixed(list(b"abc") + [("s", sym)], final=True))
        add("dynamic-symbol-%d" % sym, Stream().dynamic([], good + [0] * (sym - 257) + [8], [0], **hdr))
    for ds in (30, 31):
        add("fixed-distance-%d" % ds, Stream().fixed(list(b"abc") + [("M", 257, 0, ds, 0)], final=True))
        add("dynamic-distance-%d" % ds, Stream().dynamic([], good, [0] * (ds - 1) + [1, 1], **hdr))
    add("too-far-back-at-start-fixed", Stream().fixed([("m", 3, 1)], final=True))
    add("too-far-back-at-start-dynamic", Stream().dynamic([("m", 3, 1)], [0] * 256 + [1, 1], [1], final=True))
    add("too-far-back-after-100", Stream().fixed(list(t[:100]) + [("m", 3, 101)], final=True))
    add("too-far-back-after-600-stored", Stream().stored(t).fixed([("m", 258, 601)], final=True))
    return cases


def prefixes(n, sample=None, seed=0):
    """the lengths of the prefixes checked for an n-byte stream: every one for short streams; for long ones (and when `sample` is
    given) the first and last 64 and a seeded sample of the rest"""
    import random
    if sample is None and n <= 4096:
        return list(range(n))
    k = sample if sample is not None else 200
    edge = set(range(min(n, 64))) | set(range(max(0, n - 64), n))
    rest = sorted(set(range(n)) - edge)
    return sorted(edge | set(random.Random(seed * 7919 + n).sample(rest, min(k, len(rest)))))


# ---- zlib, the reference ------------------------------------------------------------------------------------------------------
END, DATA_ERROR, BUF_ERROR = 1, -3, -5


class ZlibTrace:
    """CPython's zlib fed one byte at a time: answers, for every prefix, the status (END, DATA_ERROR or BUF_ERROR for a truncated
    stream), the bytes delivered and the bytes consumed"""

    def __init__(self, stream):
        import zlib
        d = zlib.decompressobj(-15)
        self.n = len(stream)
        self.out = bytearray()
        self.delivered = [0]  # bytes delivered after feeding k bytes
        self.stop, self.status = None, BUF_ERROR  # the byte count at which zlib ended or failed
        for k in range(self.n):
            try:
                self.out += d.decompress(stream[k:k + 1])
            except zlib.error:
                self.stop, self.status = k + 1, DATA_ERROR
                break
            self.delivered.append(len(self.out))
            if d.eof:
                self.stop, self.status = k + 1, END
                break
        self.out = bytes(self.out)

    def at(self, k):
        """(status, delivered bytes, consumed) for the first k bytes"""
        if self.stop is None or k < self.stop:
            return BUF_ERROR, self.out[:self.delivered[k]], k
        return self.status, self.out[:self.delivered[self.stop - 1]] if self.status == DATA_ERROR else self.out, self.stop
