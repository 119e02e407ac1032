"""mz_cuda_gzip_compress_device / mz_cuda_gzip_decompress_device on the CPU: the real host C and kernel sources on the execution-model
emulator (tests/emu/libmz_strm_emu.so). Every device buffer is an allocation of exactly its size (plus guard bytes where a test says
so). A member the device writes must be what the vtbl stream writes with window bits 31 for the same bytes, and must read back through
CPython's gzip; a member the device decodes must give what the vtbl gives when it reads the same bytes from memory: return code,
plain bytes, and in_used against TOTAL_IN."""
import ctypes as C
import gzip
import hashlib
import os
import random
import struct
import subprocess
import sys
import zlib

import pytest

import datagen

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
MZ_OK, MZ_DATA_ERROR, MZ_BUF_ERROR, MZ_PARAM_ERROR = 0, -3, -5, -102


class GzipDevice:
    """ctypes driver of the two device calls and of the vtbl stream on one library (the emulator here, the product in the GPU twin)"""

    def __init__(self, lib):
        import cuharness
        self.pkg = cuharness.pkg()
        self.lib = lib
        self.t = cuharness.TestLib()

    def put(self, data, shift=0, slack=0):
        """an allocation of shift + len(data) + slack bytes (at least 1) with data at +shift and 0xab around it -> (base, ptr)"""
        n = shift + len(data) + slack
        base = self.lib.mz_cuda_malloc(max(1, n))
        assert base
        raw = b"\xab" * shift + bytes(data) + b"\xab" * slack
        if raw:
            assert self.lib.mz_cuda_memcpy_h2d(base, raw, len(raw), None) == 0
        return base, (base + shift if data or shift else None)

    def back(self, p, n):
        b = C.create_string_buffer(max(1, n))
        if n:
            assert self.lib.mz_cuda_memcpy_d2h(b, p, n, None) == 0
        return b.raw[:n]

    def compress(self, data, level=6, cap=None, slack=0):
        """-> (err, member, exact length, sizing bound, stats); the input is read back unchanged, the slack behind cap untouched"""
        L = self.lib
        base, d_in = self.put(data)
        n = C.c_uint64(0)
        try:
            err = L.mz_cuda_gzip_compress_device(d_in, len(data), level, None, 0, C.byref(n), None, None)
            if err:
                return err, b"", 0, 0, None
            bound = n.value
            size = bound if cap is None else cap
            obase, d_out = self.put(b"\xab" * size, slack=slack)
            st = self.pkg.GzipStats()
            err = L.mz_cuda_gzip_compress_device(d_in, len(data), level, obase, size, C.byref(n), C.byref(st), None)
            got = self.back(obase, size + slack)
            L.mz_cuda_free(obase)
            assert got[size:] == b"\xab" * slack, "written at or beyond cap"
            assert self.back(d_in, len(data)) == bytes(data), "input changed"
            return err, got[:min(n.value, size)], n.value, bound, st
        finally:
            L.mz_cuda_free(base)

    def decompress(self, member, cap, shift=0, slack=0):
        """-> (err, plain bytes, result, stats); the member is read back unchanged, the slack behind cap untouched"""
        L = self.lib
        base, d_in = self.put(member, shift=shift)
        obase, d_out = self.put(b"\xab" * cap, slack=slack)
        res, st = self.pkg.GzipResult(), self.pkg.GzipStats()
        try:
            err = L.mz_cuda_gzip_decompress_device(d_in, len(member), obase if cap else None, cap, C.byref(res), C.byref(st), None)
            got = self.back(obase, cap + slack)
            assert got[cap:] == b"\xab" * slack, "written at or beyond cap"
            assert self.back(base, shift + len(member))[shift:] == bytes(member), "input changed"
            return err, got[:min(res.out_len, cap)], res, st
        finally:
            L.mz_cuda_free(base)
            L.mz_cuda_free(obase)

    def vtbl_compress(self, data, level=6):
        out, info = self.t.compress(self.lib.mz_stream_cuda_create, data, level=level, window_bits=31, write_size=16384)
        assert info["close"] == 0, info
        return out

    def vtbl_decompress(self, member, out_cap):
        """the vtbl reading the member from memory -> (code, bytes, TOTAL_IN); an error that follows the last byte counts"""
        out, info = self.t.decompress(self.lib.mz_stream_cuda_create, member, out_cap, window_bits=31)
        code = info["read"] if info["read"] < 0 else (info["read_again"] if info["read_again"] < 0 else 0)
        return code, out, info["total_in"]


@pytest.fixture(scope="module")
def gz(built):
    r = subprocess.run(["make", "-s", "-C", EMU, "libmz_strm_emu.so"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    import cuharness
    return GzipDevice(cuharness.pkg().configure(C.CDLL(os.path.join(EMU, "libmz_strm_emu.so"))))


def compress_inputs():
    rnd = random.Random(11)
    return [("empty", b""), ("one", b"x"), ("65535", rnd.randbytes(65535)), ("65536", bytes(range(256)) * 256),
            ("65537", (b"abcdefgh" * 9000)[:65537]), ("random", datagen.random_bytes(200000, seed=3)), ("zeros", bytes(300000)),
            ("traps", datagen.near_period_traps()), ("text", datagen.text_like(150000, seed=9))]


def check_member(gz, data, level, member, n, bound):
    """CPython reads it back; the vtbl writes the same bytes (levels 0-9: every input here fits one vtbl batch)"""
    assert gzip.decompress(member) == data
    assert n == len(member) <= bound
    want = gz.vtbl_compress(data, level)
    assert member[:10] == want[:10]
    assert member == want


@pytest.mark.parametrize("level", [0, 1, 2, 4, 6, 9, -1])
def test_compress_matches_vtbl(gz, level):
    for name, data in compress_inputs():
        err, member, n, bound, st = gz.compress(data, level)
        assert err == MZ_OK, name
        check_member(gz, data, level, member, n, bound)
        assert st.bytes_in == len(data) and st.bytes_out == n and st.rounds == 1, name
        xfl = 2 if level == 9 else (4 if level in (0, 1) else 0)
        assert member[:10] == bytes([0x1f, 0x8b, 8, 0, 0, 0, 0, 0, xfl, 3]), name


def test_compress_empty_is_fixed_block(gz):
    err, member, _, _, _ = gz.compress(b"", 6)
    assert err == 0 and member[10:] == b"\x03\x00" + b"\0" * 8


@pytest.mark.parametrize("level", [1, 6, 9])
def test_compress_rounds_keep_one_stream(gz, monkeypatch, level):
    """1 MiB rounds over a few MiB of text: the history crosses the round boundaries, so the member is the one-round member and the
    vtbl's (its batch holds the whole input)"""
    data = datagen.text_like(3 * (1 << 20) + 12345, seed=21)
    err, one, _, _, st1 = gz.compress(data, level)
    assert err == 0 and st1.rounds == 1
    monkeypatch.setenv("MZ_CUDA_ZIP_ROUND_MB", "1")
    err, many, n, bound, st = gz.compress(data, level)
    assert err == 0 and st.rounds == 4 and many == one
    check_member(gz, data, level, many, n, bound)


def test_compress_levels_and_arguments(gz):
    L = gz.lib
    n = C.c_uint64(0)
    for bad in (-2, 10, 100):
        assert L.mz_cuda_gzip_compress_device(None, 0, bad, None, 0, C.byref(n), None, None) == MZ_PARAM_ERROR
    assert L.mz_cuda_gzip_compress_device(None, 5, 6, None, 0, C.byref(n), None, None) == MZ_PARAM_ERROR
    assert L.mz_cuda_gzip_compress_device(None, 0, 6, None, 0, None, None, None) == MZ_PARAM_ERROR


def test_compress_cap_too_small(gz):
    data = datagen.text_like(200000, seed=5)
    err, full, n, bound, _ = gz.compress(data, 6)
    assert err == 0
    # one byte short (only the trailer is missing), inside the stream (the chunk across cap is not copied), inside the header
    for cap in (n - 1, n - 9, n // 2, 5, 0):
        err, part, n2, _, _ = gz.compress(data, 6, cap=cap, slack=4096)
        assert (err, n2) == (MZ_BUF_ERROR, n), cap
        assert part[:min(cap, 10)] == full[:min(cap, 10)]
    err, again, _, _, _ = gz.compress(data, 6, cap=n, slack=4096)
    assert err == 0 and again == full


# ---- decode ------------------------------------------------------------------------------------------------------------------------
def same_as_vtbl(gz, member, cap=None, shift=0, want=None):
    """the device call and the vtbl on the same bytes: code, bytes and in_used / TOTAL_IN"""
    code, vout, total_in = gz.vtbl_decompress(member, (len(want) if want is not None else 1 << 20) + 4096)
    c = cap if cap is not None else (len(vout) if code == 0 else 1 << 20)
    err, out, res, st = gz.decompress(member, c, shift=shift, slack=64)
    assert err == code, (err, code)
    if code == 0:
        assert out == vout and res.in_used == total_in and res.out_len == len(out) and res.crc == zlib.crc32(out) and not res.out_full
        assert st.bytes_in == res.in_used and st.bytes_out == len(out)
        if want is not None:
            assert out == want
    elif code == MZ_BUF_ERROR and res.out_len and res.in_used:  # the trailer was cut short: TOTAL_IN counts what there is
        assert res.in_used == total_in == len(member)
    return err, out, res, st


def hand_header(flags, extra=b"", name=b"", comment=b"", mtime=0):
    h = bytes([0x1f, 0x8b, 8, flags]) + struct.pack("<I", mtime) + b"\x00\x03"
    if flags & 4:
        h += struct.pack("<H", len(extra)) + extra
    if flags & 8:
        h += name + b"\0"
    if flags & 16:
        h += comment + b"\0"
    if flags & 2:
        h += b"\x12\x34"  # FHCRC: skipped, not verified
    return h


def raw_deflate(data, level=6, strategy=zlib.Z_DEFAULT_STRATEGY):
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 9, strategy)
    return c.compress(data) + c.flush()


def member_of(data, header, body=None):
    return header + (raw_deflate(data) if body is None else body) + struct.pack("<II", zlib.crc32(data), len(data) & 0xffffffff)


def wbits31(data, level):
    c = zlib.compressobj(level, zlib.DEFLATED, 31)
    return c.compress(data) + c.flush()


def decode_inputs():
    text = datagen.text_like(120000, seed=31)
    rec = datagen.binary_records(90000)
    full = hand_header(4 | 8 | 16 | 2, extra=b"AB\x02\x00xy", name=b"file.txt", comment=b"a comment")
    return [
        ("cpython", gzip.compress(text, mtime=1700000000), text),
        ("cpython-name", _cpython_named(text), text),
        ("zlib1", wbits31(text, 1), text), ("zlib6", wbits31(rec, 6), rec), ("zlib9", wbits31(text, 9), text),
        ("fextra", member_of(text, hand_header(4, extra=b"\x01\x02\x03")), text),
        ("fname", member_of(text, hand_header(8, name=b"x" * 300)), text),
        ("fcomment", member_of(rec, hand_header(16, comment=b"c" * 5000)), rec),
        ("fhcrc", member_of(rec, hand_header(2)), rec),
        ("all-flags", member_of(text, full), text),
        ("header-over-4k", member_of(text, hand_header(4 | 8, extra=b"e" * 5000, name=b"n" * 3000)), text),
        ("stored", wbits31(text[:70000], 0), text[:70000]),
        ("fixed", member_of(text, hand_header(0), raw_deflate(text, 6, zlib.Z_FIXED)), text),
        ("empty-member", gzip.compress(b""), b""),
        ("one-byte", gzip.compress(b"z"), b"z"),
    ]


def _cpython_named(data):
    import io
    b = io.BytesIO()
    with gzip.GzipFile(filename="name.bin", mode="wb", fileobj=b, mtime=123) as f:
        f.write(data)
    return b.getvalue()


def test_decode_foreign_members(gz):
    for name, member, want in decode_inputs():
        err, _, res, _ = same_as_vtbl(gz, member, want=want)
        assert err == 0, name
        assert res.in_used == len(member), name


def test_decode_own_members(gz):
    for level in (0, 1, 6, 9):
        for name, data in compress_inputs():
            err, member, _, _, _ = gz.compress(data, level)
            assert err == 0
            err, out, res, _ = same_as_vtbl(gz, member, want=data)
            assert err == 0 and res.header_len == 10 and res.in_used == len(member), (level, name)


def test_decode_ignores_what_follows(gz):
    text = datagen.text_like(50000, seed=41)
    m = gzip.compress(text)
    for tail in (b"garbage!" * 10, gzip.compress(b"second member"), b"\0" * 1000, b"\x1f"):
        err, out, res, _ = same_as_vtbl(gz, m + tail, want=text)
        assert err == 0 and res.in_used == len(m)


def test_decode_misaligned_input(gz):
    text = datagen.text_like(100000, seed=42)
    for member in (gzip.compress(text), member_of(text, hand_header(8, name=b"abc"))):
        for shift in (1, 2, 3):
            err, out, res, _ = same_as_vtbl(gz, member, shift=shift, want=text)
            assert err == 0 and out == text


def test_decode_long_member_with_speculative_rounds(gz, monkeypatch):
    """a foreign level-6 stream of several MiB: K6 rounds run, and with MZ_CUDA_SPEC=0 K5 alone gives the same bytes"""
    text = datagen.text_like(6 << 20, seed=43)
    member = wbits31(text, 6)
    err, out, res, st = same_as_vtbl(gz, member, want=text)
    assert err == 0 and st.k6_rounds > 0 and res.in_used == len(member)
    monkeypatch.setenv("MZ_CUDA_SPEC", "0")
    err, out0, res0, st0 = gz.decompress(member, len(text))
    assert err == 0 and out0 == text and st0.k6_rounds == 0 and res0.in_used == res.in_used and res0.crc == res.crc


def test_decode_header_errors(gz):
    text = datagen.text_like(20000, seed=44)
    full = member_of(text, hand_header(4 | 8 | 16 | 2, extra=b"xyz", name=b"nm", comment=b"cm"))
    hlen = 10 + 2 + 3 + 3 + 3 + 2
    codes = set()
    for k in range(hlen + 1):  # every truncation of the header
        err, _, res, _ = same_as_vtbl(gz, full[:k])
        codes.add(err)
        assert err != 0 and res.out_len == 0
    assert codes == {MZ_BUF_ERROR}
    good = gzip.compress(text)
    for pos, val in ((0, 0x1e), (1, 0x8a), (2, 7), (2, 0), (3, 0x20), (3, 0x80)):  # magic, method, reserved flags
        bad = bytearray(good)
        bad[pos] = val
        err, _, _, _ = same_as_vtbl(gz, bytes(bad))
        assert err == MZ_DATA_ERROR, (pos, val)
    for short in (b"\x1f", b"\x1e", b"\x1e\x8b", b"\x1f\x8b\x08"):
        same_as_vtbl(gz, short)


def test_decode_trailer_and_stream_errors(gz):
    text = datagen.text_like(80000, seed=45)
    m = gzip.compress(text, mtime=0)
    for pos in (len(m) - 8, len(m) - 5, len(m) - 4, len(m) - 1):  # a flipped CRC byte, a flipped ISIZE byte
        bad = bytearray(m)
        bad[pos] ^= 0x40
        err, _, _, _ = same_as_vtbl(gz, bytes(bad))
        assert err == MZ_DATA_ERROR, pos
    rnd = random.Random(46)
    cuts = sorted(set([10, 11, 12, len(m) - 9, len(m) - 8, len(m) - 7, len(m) - 4, len(m) - 1] + rnd.sample(range(13, len(m) - 9), 12)))
    for k in cuts:  # truncation in the stream and in the trailer: zlib's truncated, MZ_BUF_ERROR
        err, _, _, _ = same_as_vtbl(gz, m[:k])
        assert err == MZ_BUF_ERROR, k
    for k in rnd.sample(range(12, len(m) - 9), 10):  # corrupt stream bytes: whatever the vtbl says
        bad = bytearray(m)
        bad[k] ^= 0xff
        same_as_vtbl(gz, bytes(bad))


def test_decode_output_full(gz):
    text = datagen.text_like(200000, seed=47)
    for member in (gzip.compress(text), wbits31(text, 0)):
        for cap in (len(text) - 1, len(text) // 2, 1000, 0):
            err, out, res, _ = gz.decompress(member, cap, slack=4096)
            assert (err, res.out_full) == (MZ_BUF_ERROR, 1), cap
            assert out == text[:len(out)] and len(out) <= cap
        err, out, res, _ = gz.decompress(member, len(text), slack=4096)
        assert err == 0 and out == text and not res.out_full


def test_decode_arguments(gz):
    L = gz.lib
    res = gz.pkg.GzipResult()
    assert L.mz_cuda_gzip_decompress_device(None, 10, None, 0, C.byref(res), None, None) == MZ_PARAM_ERROR
    assert L.mz_cuda_gzip_decompress_device(None, 0, None, 10, C.byref(res), None, None) == MZ_PARAM_ERROR
    assert L.mz_cuda_gzip_decompress_device(None, 0, None, 0, None, None, None) == MZ_PARAM_ERROR
    assert L.mz_cuda_gzip_decompress_device(None, 0, None, 0, C.byref(res), None, None) == MZ_BUF_ERROR


SCHED_BODY = (
    "import hashlib, datagen, gzip\n"
    "text = datagen.text_like(140000, seed=7)\n"
    "for lv in (1, 6):\n"
    "    err, m, _, _, _ = g.compress(text, lv)\n"
    "    print('c', lv, err, hashlib.sha256(m).hexdigest())\n"
    "    err, out, res, st = g.decompress(gzip.compress(text) if lv == 1 else m, len(text))\n"
    "    print('d', lv, err, res.in_used, hashlib.sha256(out).hexdigest())\n")


def test_schedules_and_race_checker(gz):
    """compress and decode under two fixed thread / block schedules with the shared-memory race checker: the default schedule's bytes"""
    def run(env):
        script = ("import ctypes as C, os, sys\nsys.path.insert(0, %r)\nimport cuharness, test_emu_device_gzip as t\n"
                  "g = t.GzipDevice(cuharness.pkg().configure(C.CDLL(%r)))\n" % (HERE, os.path.join(EMU, "libmz_strm_emu.so"))) + SCHED_BODY
        r = subprocess.run([sys.executable, "-c", script], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
        assert r.returncode == 0, r.stdout[-3000:]
        return [l for l in r.stdout.splitlines() if l[:2] in ("c ", "d ")]
    want = run(dict(os.environ))
    assert len(want) == 4 and all(l.split()[2] == "0" for l in want)
    for seed in (5, 23):
        assert run(dict(os.environ, MZ_EMU_SCHED=str(seed), MZ_EMU_RACE="1")) == want, seed
