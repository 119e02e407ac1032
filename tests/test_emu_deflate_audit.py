"""Every block the deflate kernel writes, checked against the kernel's own rules (tests/deflate_audit.py) on the CPU emulator: the
kernel sources compressed by emushim.EmuLib.deflate, each output slot decoded by an independent block decoder, and every block
checked for framing, the one-block-per-unit partition, match lengths and reach, the code-length code, code lengths and header
bits the code builder gives for the block's histogram, and the stored-versus-dynamic decision. The histograms the builder was
given come from the same kernel sources built with the capture hook (tests/emu/emu_df_codes.cc), so stored units are judged
too. Levels 0, 1, 2, 4 and 6 are the kernel's four instantiations (deflate_kernel.cuh:1403-1408) plus stored-only; every input
runs as independent chunks and as one stream (FINAL | DICT).

The decoder itself is checked first: it must reproduce zlib's own streams token by token, accept every stream of
deflate_craft.valid_cases() and reject every one of invalid_cases()."""
import ctypes as C
import random
import zlib

import numpy as np
import pytest

import datagen
import deflate_audit as A
import deflate_craft
import test_emu_deflate_digests as digests
import test_emu_df_codes_equiv as codes_equiv

LEVELS = (0, 1, 2, 4, 6)
MODES = {"chunks": A.FLAG_FINAL, "stream": A.FLAG_FINAL | A.FLAG_DICT}
NEAR_WINDOW = (-60, -4)  # dyn_bits - stored_bits of the near-threshold unit: Huffman, but by less than 64 bits


# ---- the decoder against zlib ------------------------------------------------------------------------------------------------
def _zlib_stream(data, level, strategy=zlib.Z_DEFAULT_STRATEGY, flush_every=0):
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 9, strategy)
    if not flush_every:
        return c.compress(data) + c.flush()
    out = b""
    for i in range(0, len(data), flush_every):
        out += c.compress(data[i:i + flush_every]) + c.flush(zlib.Z_FULL_FLUSH)
    return out + c.flush()


@pytest.mark.parametrize("level", range(1, 10))
def test_decoder_reproduces_zlib_streams(level):
    data = datagen.mixed(300_000, 11) + bytes(5000) + datagen.text_like(40_000, 12)
    for strategy, flush in ((zlib.Z_DEFAULT_STRATEGY, 0), (zlib.Z_FIXED, 0), (zlib.Z_DEFAULT_STRATEGY, 70_001)):
        comp = _zlib_stream(data, level, strategy, flush)
        blocks, out, end = A.decode(comp)
        assert out == data and (end + 7) // 8 == len(comp)
        assert b"".join(A.expand(b.tokens, data[:b.out_start]) if b.tokens is not None else data[b.out_start:b.out_end]
                        for b in blocks) == data
        assert {b.btype for b in blocks} >= ({1} if strategy == zlib.Z_FIXED else {2})
        if flush:
            assert sum(1 for b in blocks if b.btype == 0 and b.stored_len == 0) >= len(data) // flush


def test_decoder_accepts_the_valid_crafted_streams():
    for name, stream, plain in deflate_craft.valid_cases():
        _, out, end = A.decode(stream)
        assert out == plain and (end + 7) // 8 == len(stream), name


def test_decoder_rejects_the_invalid_crafted_streams():
    for name, stream in deflate_craft.invalid_cases():
        with pytest.raises(A.DeflateError):
            A.decode(stream)
        with pytest.raises(zlib.error):
            zlib.decompress(stream, -15)
    # truncation: every proper prefix of a dynamic stream
    comp = _zlib_stream(datagen.text_like(3000, 3), 6)
    for k in range(len(comp)):
        with pytest.raises(A.DeflateError):
            A.decode(comp[:k])


# ---- the kernel on the emulator ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(built):
    return digests._emu()


@pytest.fixture(scope="module")
def codes(tmp_path_factory):
    path, log = codes_equiv.build(tmp_path_factory.mktemp("emu_df_codes"))
    assert path, log
    return with_capture(codes_equiv.load(path))


@pytest.fixture(scope="module")
def inputs(codes):
    return corpus(codes)


def with_capture(L):
    """the code-builder harness (test_emu_df_codes_equiv.load) with its explicit-chunk capture declared"""
    L.emu_df_capture_chunks.restype = C.c_uint32
    L.emu_df_capture_chunks.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p,
                                        C.c_void_p, C.c_uint32]
    return L


def emu_builder(L):
    """the kernel's code builder on the emulator ("new" output of df_codes_pair.cuh)"""
    def run(h, pf):
        h, pf = np.ascontiguousarray(h, dtype=np.uint32), np.ascontiguousarray(pf, dtype=np.uint32)
        old = np.zeros((len(h), L.emu_df_out_words()), dtype=np.uint32)
        new = np.zeros_like(old)
        L.emu_df_codes_pair(codes_equiv.ptr(h), codes_equiv.ptr(pf), len(h), codes_equiv.ptr(old), codes_equiv.ptr(new))
        return new
    return run


def chunk_table(n, chunk, flags):
    """(offsets, lengths, per-chunk flags) of the uniform partition the kernel makes of n bytes (deflate_kernel.cuh:824-830)"""
    k = max(1, (n + chunk - 1) // chunk)
    offs = [i * chunk for i in range(k)]
    lens = [min(chunk, n - o) for o in offs]
    fl = [(flags & A.FLAG_DICT) | (flags & A.FLAG_FINAL if i == k - 1 else 0) for i in range(k)]
    return offs, lens, fl


def capture(L, data, offs, lens, flags, level):
    """{(chunk, unit): the histogram the kernel's builder was given} for explicit chunks, on the emulator"""
    n = len(offs)
    cap = sum((ln + A.DF_UNIT - 1) // A.DF_UNIT for ln in lens) + 1
    h = np.zeros((cap, A.HIST_WORDS), dtype=np.uint32)
    tags = np.zeros(cap, dtype=np.uint32)
    o = (C.c_uint64 * n)(*offs)
    ln = (C.c_uint32 * n)(*lens)
    fl = (C.c_uint8 * n)(*flags)
    k = L.emu_df_capture_chunks(bytes(data), len(data), o, ln, fl, n, level, codes_equiv.ptr(h), codes_equiv.ptr(tags), cap)
    assert k <= cap
    return {(int(t) >> 8, int(t) & 255): h[i] for i, t in enumerate(tags[:k])}


def window_of(data, off, level, flags):
    """the bytes in front of a chunk that its matches may reach (deflate_kernel.cuh:831)"""
    return data[off - A.DF_UNIT:off] if level >= 6 and flags & A.FLAG_DICT and off >= A.DF_UNIT else b""


def slots_of(data, comp, out_len, offs, lens, flags, level):
    slots, pos = [], 0
    for o, ln, fl, k in zip(offs, lens, flags, out_len):
        slots.append(A.Slot(comp[pos:pos + k], data[o:o + ln], level, fl, window_of(data, o, level, fl)))
        pos += k
    assert pos == len(comp)
    return slots


# ---- the corpus --------------------------------------------------------------------------------------------------------------
def near_threshold_unit(L, seed=1):
    """32 KiB whose Huffman block is smaller than a stored one by less than 64 bits: random bytes with a run of r zeros in the
    middle, r found by bisection on dyn_bits - stored_bits (the builder's own count, from the captured histogram; it falls by
    about a bit per byte of the run once the run is matched)"""
    noise = np.random.default_rng(seed).integers(0, 256, A.DF_UNIT, dtype=np.uint8)
    build = emu_builder(L)

    def unit(r):
        u = noise.copy()
        u[16000:16000 + r] = 0
        return u.tobytes()

    def margin(r):
        d = unit(r)
        h = capture(L, d, [0], [len(d)], [A.FLAG_FINAL], 1)[(0, 0)]
        built = A.Built(build(h[None], np.zeros(1, dtype=np.uint32))[0])
        return built.dyn_bits(h) - A.stored_bits(0, len(d))

    lo, hi = 0, 4096
    assert margin(lo) > 0 > margin(hi)
    target = sum(NEAR_WINDOW) // 2
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if margin(mid) > target:
            lo = mid
        else:
            hi = mid
    for r in sorted(range(max(0, hi - 64), hi + 64), key=lambda r: abs(r - hi)):
        if NEAR_WINDOW[0] <= margin(r) <= NEAR_WINDOW[1]:
            return unit(r)
    raise AssertionError("no unit within %s bits of the stored size" % (NEAR_WINDOW,))


def edge_inputs(near):
    text = datagen.text_like(70_000, 77)
    out = {"len%d" % n: text[:n] for n in (0, 1, 3, 4, 5, 32767, 32768, 32769, 65535, 65536, 65537)}
    out["one-byte"] = b"x" * 100_000
    out["two-symbols"] = bytes(b"ab"[i] for i in np.random.default_rng(5).integers(0, 2, 90_000))
    r = random.Random(9)
    out["runs-258-259"] = b"".join(datagen.random_bytes(r.randrange(20, 60), i) + bytes([i & 255]) * (258 + (i & 1) + (i % 3 == 2))
                                   for i in range(300))
    out["period-32768"] = datagen.random_bytes(32768, 21) * 4 + datagen.random_bytes(1000, 22)
    out["random"] = datagen.random_bytes(150_000, 23)
    out["near-threshold"] = near + text[:32768] + near
    return out


def corpus(L):
    """[(name, data, chunk size)]"""
    items = [(k, v, 65536) for k, v in digests.inputs().items()]
    items += [(k, v, 65536) for k, v in edge_inputs(near_threshold_unit(L)).items()]
    items += [("text-ragged-40000", digests.inputs()["text"], 40000), ("runs-ragged-40000", digests.inputs()["runs"], 40000)]
    return items


def run_config(emu, L, data, chunk, level, flags):
    comp, out_len = emu.deflate(data, level=level, chunk=chunk, final=flags)
    offs, lens, fl = chunk_table(len(data), chunk, flags)
    slots = slots_of(data, comp, out_len, offs, lens, fl, level)
    for s in slots:
        A.check_slot(s)
    hists = None
    if level:
        cap = capture(L, data, offs, lens, fl, level)
        hists = {(i, u): h for (i, u), h in cap.items()}
        assert len(hists) == sum(len(s.units) for s in slots if s.chunk)  # (an empty chunk runs no unit)
    checked = A.check_codes(slots, emu_builder(L), hists)
    return slots, checked


@pytest.mark.parametrize("level", LEVELS)
def test_every_block_follows_the_kernel_rules(emu, codes, inputs, level):
    stats = {"blocks": 0, "stored": 0}
    for name, data, chunk in inputs:
        for mode, flags in list(MODES.items()) + ([("open", 0)] if name in ("len0", "len65537", "text") else []):
            try:
                slots, checked = run_config(emu, codes, data, chunk, level, flags)
            except AssertionError as e:
                raise AssertionError("%s, chunk %d, level %d, %s: %s" % (name, chunk, level, mode, e)) from e
            units = [b for s in slots for b in s.units]
            stats["blocks"] += len(units)
            stats["stored"] += sum(b.btype == 0 for b in units)
            if level:
                assert checked == sum(len(s.units) for s in slots if s.chunk)
    assert stats["blocks"] > 100
    if level:
        assert 0 < stats["stored"] < stats["blocks"]

