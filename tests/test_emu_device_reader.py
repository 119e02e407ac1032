"""The device reader (mz_zip_cuda_reader_*) on the CPU: the real host C and kernel sources on the execution-model emulator
(tests/emu/libmz_strm_emu.so), every device buffer in an allocation of exactly its size. The reader is checked against
mz_zip_cuda_extract_device on the same bytes: open's code, count, refusal and table equal the list-only call's, and every
selection slot's bytes and status equal what extract_device gives that entry. Name lookup is checked against a Python restatement
of the reference's mz_zip_path_compare and, when oracle/_ref/libmzref.so is built, against the reference's mz_zip_locate_entry."""
import ctypes as C
import io
import os
import random
import struct
import subprocess
import sys
import threading
import zipfile
import zlib

import pytest

from test_emu_device_extract import DeviceExtractor, adversarial_cases, mutations, with_count
from test_emu_native_extract import (AES, EMU, HASH_SHA256, HERE, MZ_SUPPORT_ERROR, Extractor, corpus, edit_directory, malformed_cases,
                                     patch_zip64_end, py_zip, reorder_directory, zip64_directory)

MZ_BUF_ERROR, MZ_END_OF_LIST, MZ_PARAM_ERROR = -5, -100, -102
MISS = 0xffffffff
ROOT = os.path.dirname(HERE)


class DeviceReader:
    """ctypes driver of the reader on one library (the emulator here, the product in the GPU twin); every device buffer is an
    allocation of exactly its size"""

    def __init__(self, lib):
        import cuharness
        self.pkg = cuharness.pkg()
        self.lib = lib
        self.row = C.sizeof(self.pkg.ZipDevEntry)

    def put(self, data):
        p = self.lib.mz_cuda_malloc(max(1, len(data)))
        assert p
        if data:
            assert self.lib.mz_cuda_memcpy_h2d(p, bytes(data), len(data), None) == 0
        return p

    def get(self, p, n):
        b = C.create_string_buffer(max(1, n))
        if n:
            assert self.lib.mz_cuda_memcpy_d2h(b, p, n, None) == 0
        return b.raw[:n]

    def open(self, d_arc, n, password=None):
        """-> (err, handle, count, refuse)"""
        h, count, refuse = C.c_void_p(), C.c_uint32(0), C.c_int32(0)
        st = self.pkg.ZipStats()
        err = self.lib.mz_zip_cuda_reader_open(d_arc if n else None, n, password.encode() if password is not None else None, C.byref(h),
                                               C.byref(count), C.byref(refuse), C.byref(st), None)
        if err:
            assert not h.value and count.value == 0
        return err, h, count.value, refuse.value

    def table(self, h, count):
        return self.get(self.lib.mz_zip_cuda_reader_entries(h), count * self.row)

    def decode(self, h, sel, cap_delta=0, status=True, offsets=True):
        """-> (err, out_bytes, raw output, offsets, statuses); the output allocation holds exactly out_bytes + cap_delta bytes"""
        L = self.lib
        d_sel = self.put(struct.pack("<%dI" % len(sel), *sel)) if sel else None
        size = C.c_uint64(0)
        try:
            assert L.mz_zip_cuda_reader_decode(h, d_sel, len(sel), None, 0, C.byref(size), None, None, None, None) == 0
            n = size.value
            cap = max(0, n + cap_delta)
            d_out = L.mz_cuda_malloc(max(1, cap))
            assert L.mz_cuda_memset(d_out, 0, max(1, cap), None) == 0  # the padding between slots reads as zeros
            d_off = L.mz_cuda_malloc(8 * (len(sel) + 1)) if offsets else None
            d_st = L.mz_cuda_malloc(4 * max(1, len(sel))) if status else None
            try:
                err = L.mz_zip_cuda_reader_decode(h, d_sel, len(sel), d_out, cap, C.byref(size), d_off, d_st, None, None)
                assert size.value == n
                offs = list(struct.unpack("<%dQ" % (len(sel) + 1), self.get(d_off, 8 * (len(sel) + 1)))) if offsets else None
                sts = list(struct.unpack("<%di" % len(sel), self.get(d_st, 4 * len(sel)))) if status and sel else []
                return err, n, self.get(d_out, min(n, cap)), offs, sts
            finally:
                for p in (d_out, d_off, d_st):
                    if p:
                        L.mz_cuda_free(p)
        finally:
            if d_sel:
                L.mz_cuda_free(d_sel)

    def locate(self, h, names, ignore_case):
        """names: bytes each -> [index or MISS]"""
        L = self.lib
        if not names:
            assert L.mz_zip_cuda_reader_locate(h, None, None, None, 0, ignore_case, None, None) == 0
            return []
        offs, pos = [], 0
        for q in names:
            offs.append(pos)
            pos += len(q)
        d_names = self.put(b"".join(names))
        d_off = self.put(struct.pack("<%dQ" % len(names), *offs))
        d_len = self.put(struct.pack("<%dI" % len(names), *[len(q) for q in names]))
        d_idx = L.mz_cuda_malloc(4 * len(names))
        try:
            assert L.mz_zip_cuda_reader_locate(h, d_names, d_off, d_len, len(names), ignore_case, d_idx, None) == 0
            return list(struct.unpack("<%dI" % len(names), self.get(d_idx, 4 * len(names))))
        finally:
            for p in (d_names, d_off, d_len, d_idx):
                L.mz_cuda_free(p)


def listed(dx, archive, password=None):
    """extract_device list-only -> (err, count, raw table)"""
    L = dx.lib
    pw = password.encode() if password is not None else None
    d_arc = dx._dev(len(archive))
    if archive:
        assert L.mz_cuda_memcpy_h2d(d_arc, archive, len(archive), None) == 0
    count, nbytes = C.c_uint32(0), C.c_uint64(0)
    row = C.sizeof(dx.pkg.ZipDevEntry)
    try:
        err = L.mz_zip_cuda_extract_device(d_arc, len(archive), pw, None, 0, C.byref(count), None, 0, C.byref(nbytes), None, None)
        if err != MZ_BUF_ERROR:
            return err, count.value, b""
        n = count.value
        d_ent = dx._dev(n * row)
        err = L.mz_zip_cuda_extract_device(d_arc, len(archive), pw, d_ent, n, C.byref(count), None, 0, C.byref(nbytes), None, None)
        back = C.create_string_buffer(n * row)
        assert L.mz_cuda_memcpy_d2h(back, d_ent, n * row, None) == 0
        L.mz_cuda_free(d_ent)
        return err, n, back.raw
    finally:
        L.mz_cuda_free(d_arc)


class Case:
    """one archive: extract_device's view of it and an open reader over a device copy"""

    def __init__(self, ctx, archive, password=None):
        self.ctx, self.archive, self.password = ctx, archive, password
        dx, rd = ctx.dx, ctx.rd
        self.lerr, self.lcount, self.ltable = listed(dx, archive, password)
        self.xerr, self.xgot, self.xn, _ = dx.extract(archive, password=password)  # [(name, bytes, crc, status)]
        self.d_arc = rd.put(archive)
        self.err, self.h, self.count, self.refuse = rd.open(self.d_arc, len(archive), password)

    def close(self):
        if self.h:
            self.ctx.rd.lib.mz_zip_cuda_reader_close(self.h)
        self.ctx.rd.lib.mz_cuda_free(self.d_arc)

    def unchanged(self):
        assert self.ctx.rd.get(self.d_arc, len(self.archive)) == bytes(self.archive)

    def check_open(self):
        if self.err:  # an error of the archive as a whole: what extract_device returns, with nothing listed
            assert self.err == self.lerr and self.lcount == 0
            return False
        assert (self.count, self.refuse) == (self.lcount, self.lerr)  # listing returns what ended the list
        assert self.ctx.rd.table(self.h, self.count) == self.ltable
        return True

    def check_selection(self, sel, **kw):
        """every slot's bytes and status against extract_device's for that entry; the return is the first failing slot's status"""
        err, n, raw, offs, sts = self.ctx.rd.decode(self.h, sel, **kw)
        want = [self.xgot[i][3] if i < self.count else MZ_END_OF_LIST for i in sel]
        if kw.get("status", True):
            assert sts == want, (sts, want)
        assert err == next((s for s in want if s), 0)
        assert offs[0] == 0 and offs[-1] == n
        for k, i in enumerate(sel):
            size = len(self.xgot[i][1]) if i < self.count else 0  # the entry's recorded plain size
            assert offs[k + 1] - offs[k] == (size + 15) // 16 * 16, (k, i)
            if want[k] == 0:  # a failing entry's bytes are unspecified
                assert raw[offs[k]:offs[k] + size] == self.xgot[i][1], (k, i)
        self.unchanged()
        return err


class Ctx:
    def __init__(self, lib):
        self.lib = lib
        self.ex, self.dx, self.rd = Extractor(lib), DeviceExtractor(lib), DeviceReader(lib)


@pytest.fixture(scope="module")
def ctx(built):
    r = subprocess.run(["make", "-s", "-C", EMU, "libmz_strm_emu.so"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    import cuharness
    return Ctx(cuharness.pkg().configure(C.CDLL(os.path.join(EMU, "libmz_strm_emu.so"))))


def identity(ctx, archive, password=None, seed=0, selections=4):
    """open against list-only, decode(0..count-1) against the full extraction, then seeded selections"""
    c = Case(ctx, archive, password)
    try:
        if not c.check_open():
            return c.err
        err = c.check_selection(list(range(c.count)))
        assert (err or c.refuse) == c.xerr, (err, c.refuse, c.xerr)
        rng = random.Random(seed)
        n = c.count
        for _ in range(selections):
            k = rng.randrange(0, 2 * n + 3)
            sel = [rng.randrange(0, n + 2) if n else rng.randrange(0, 3) for _ in range(k)]
            c.check_selection(sel)
        if n:
            c.check_selection(list(reversed(range(n))))
            c.check_selection([n - 1])
            c.check_selection([0, 0, n - 1, 0])
        c.check_selection([])
        c.check_selection([n, MISS, 0x7fffffff])
        return err or c.refuse
    finally:
        c.close()


def test_zipfile_archives(ctx):
    files = corpus(12, 3000, seed=21)
    for comp in (zipfile.ZIP_STORED, zipfile.ZIP_DEFLATED):
        assert identity(ctx, py_zip(files, comp, dirs=("empty_dir/",)), seed=1) == 0


def test_data_descriptors_and_zip64_fields(ctx):
    files = corpus(7, 5000, seed=22)
    for a in (py_zip(files, stream=True), py_zip(files, force_zip64=True), zip64_directory(py_zip(files))):
        assert identity(ctx, a, seed=2) == 0


@pytest.mark.parametrize("flags", [0, HASH_SHA256])
def test_native_writer_archives(ctx, flags):
    assert identity(ctx, ctx.ex.write(corpus(9, 70000, seed=23), flags=flags), seed=3) == 0


@pytest.mark.parametrize("strength", [1, 2, 3])
def test_aes_archives(ctx, strength):
    a = ctx.ex.write(corpus(6, 4000, seed=24), flags=AES | HASH_SHA256, password="pw-%d" % strength, strength=strength)
    assert identity(ctx, a, password="pw-%d" % strength, seed=4) == 0  # the device archive is read back after every call
    assert identity(ctx, a, password="wrong", seed=5) == -108
    assert identity(ctx, a, seed=6) == -108


def test_mixed_aes_strengths_and_the_same_entry_twice(ctx):
    """one archive whose entries use all three strengths (the directories of three archives merged); an AES entry selected twice is
    decrypted once per slot"""
    files = corpus(4, 3000, seed=40)
    parts = [ctx.ex.write([("s%d/%s" % (s, n), d) for n, d in files], flags=AES, password="pw", strength=s) for s in (1, 2, 3)]
    a = merge_archives(parts)
    c = Case(ctx, a, "pw")
    try:
        assert c.check_open() and c.count == 12 and c.xerr == 0
        c.check_selection([0, 0, 5, 11, 5, 11, 0])
        c.check_selection([11, 4, 2, 9, 9, 1, 7, 3])
        c.check_selection(list(range(12)) * 2)
    finally:
        c.close()


def merge_archives(parts):
    """the local sections of several single-disk archives back to back, one directory (offsets shifted), one end record"""
    body, cds, n = b"", b"", 0
    for a in parts:
        e = a.rindex(b"PK\x05\x06")
        cnt, cd_size, cd_off = struct.unpack("<HII", a[e + 10:e + 20])
        cd = bytearray(a[cd_off:cd_off + cd_size])
        p = 0
        while p < len(cd):
            nl, xl, cl = struct.unpack("<HHH", cd[p + 28:p + 34])
            cd[p + 42:p + 46] = struct.pack("<I", struct.unpack("<I", cd[p + 42:p + 46])[0] + len(body))
            p += 46 + nl + xl + cl
        body += a[:cd_off]
        cds += bytes(cd)
        n += cnt
    return body + cds + struct.pack("<IHHHHIIH", 0x06054b50, 0, 0, n, n, len(cds), len(body), 0)


def test_zip64_end_prepended_data_and_reordered_directory(ctx):
    a = py_zip(corpus(8, 2000, seed=25))
    for b in (patch_zip64_end(a), b"\x7fSFX" * 250 + a, reorder_directory(a)):
        assert identity(ctx, b, seed=7) == 0


def test_malformed_archives(ctx):
    for name, (arc, codes) in malformed_cases(ctx.ex).items():
        assert identity(ctx, arc, seed=8, selections=1) in codes, name


def test_refusal_and_adversarial_signatures(ctx):
    a = py_zip(corpus(6, 3000, seed=26))
    b = edit_directory(a, lambda i, r: r[:8] + bytes([r[8] | 1]) + r[9:] if i == 3 else r)
    assert identity(ctx, b, seed=9) == MZ_SUPPORT_ERROR
    for arc in adversarial_cases((ctx.ex, ctx.dx)).values():
        identity(ctx, arc, seed=10, selections=1)
    assert identity(ctx, py_zip([]), seed=11) == 0
    assert identity(ctx, with_count(a, 1), seed=12) != 0
    assert identity(ctx, b"", seed=13) != 0


def test_random_directory_mutations(ctx):
    for k, arc in enumerate(mutations(1234, 120)):
        try:
            identity(ctx, arc, seed=k, selections=1)
        except AssertionError as x:
            raise AssertionError("mutation %d: %s" % (k, x)) from None


def test_sizing_short_caps_and_arguments(ctx):
    """the sizing call; out_cap one byte short: MZ_BUF_ERROR and guard-filled buffers untouched; argument errors"""
    rd, L = ctx.rd, ctx.lib
    a = ctx.ex.write(corpus(6, 3000, seed=30), flags=HASH_SHA256)
    c = Case(ctx, a)
    try:
        assert c.check_open()
        sel = [3, 1, 1, 7, 0]
        d_sel = rd.put(struct.pack("<5I", *sel))
        size, offs = C.c_uint64(0), L.mz_cuda_malloc(48)
        assert L.mz_zip_cuda_reader_decode(c.h, d_sel, 5, None, 0, C.byref(size), offs, None, None, None) == 0
        o = struct.unpack("<6Q", rd.get(offs, 48))
        want = [0]
        for i in sel:
            want.append(want[-1] + ((len(c.xgot[i][1]) + 15) // 16 * 16 if i < c.count else 0))
        assert list(o) == want and size.value == want[-1]
        n = size.value
        d_out, d_st = L.mz_cuda_malloc(n), L.mz_cuda_malloc(20)
        for p, nb in ((d_out, n), (offs, 48), (d_st, 20)):
            assert L.mz_cuda_memset(p, 0xab, nb, None) == 0
        assert L.mz_zip_cuda_reader_decode(c.h, d_sel, 5, d_out, n - 1, C.byref(size), offs, d_st, None, None) == MZ_BUF_ERROR
        assert size.value == n
        for p, nb in ((d_out, n), (offs, 48), (d_st, 20)):
            assert rd.get(p, nb) == b"\xab" * nb
        assert L.mz_zip_cuda_reader_decode(c.h, d_sel, 5, d_out + 1, n, C.byref(size), offs, d_st, None, None) == MZ_PARAM_ERROR
        assert L.mz_zip_cuda_reader_decode(c.h, None, 5, d_out, n, C.byref(size), offs, d_st, None, None) == MZ_PARAM_ERROR
        assert L.mz_zip_cuda_reader_decode(None, d_sel, 5, d_out, n, C.byref(size), offs, d_st, None, None) == MZ_PARAM_ERROR
        assert L.mz_zip_cuda_reader_decode(c.h, d_sel, 5, d_out, n, None, offs, d_st, None, None) == MZ_PARAM_ERROR
        assert L.mz_zip_cuda_reader_decode(c.h, d_sel, 5, d_out, n, C.byref(size), None, None, None, None) == MZ_END_OF_LIST  # slot 3: no entry 7
        for p in (d_sel, offs, d_out, d_st):
            L.mz_cuda_free(p)
        c.check_selection([5, 2], status=False)
        c.unchanged()
    finally:
        c.close()
    cnt, ref = C.c_uint32(0), C.c_int32(0)
    assert L.mz_zip_cuda_reader_open(None, 10, None, C.byref(C.c_void_p()), C.byref(cnt), C.byref(ref), None, None) == MZ_PARAM_ERROR
    L.mz_zip_cuda_reader_close(None)


def test_scratch_reuse(ctx):
    """small, large, then small selections on one reader give what fresh readers give"""
    a = ctx.ex.write(corpus(40, 3000, seed=31), flags=HASH_SHA256)
    b = ctx.ex.write(corpus(10, 2000, seed=32), flags=AES, password="pw", strength=2)
    for arc, pw in ((a, None), (b, "pw")):
        rng = random.Random(5)
        n = len(zipfile.ZipFile(io.BytesIO(arc)).infolist())
        sels = [[rng.randrange(n) for _ in range(3)], [rng.randrange(n) for _ in range(700)], [rng.randrange(n) for _ in range(2)]]
        c = Case(ctx, arc, pw)
        try:
            got = [ctx.rd.decode(c.h, s) for s in sels]
        finally:
            c.close()
        for s, g in zip(sels, got):
            f = Case(ctx, arc, pw)
            try:
                assert ctx.rd.decode(f.h, s) == g
            finally:
                f.close()


# ---- names ------------------------------------------------------------------------------------------------------------
def _lower(c):
    return c + 32 if 0x41 <= c <= 0x5a else c  # tolower in the C locale


def path_compare(p1, p2, ignore_case):
    """mz_zip_path_compare (mz_zip.c:2754) restated on byte strings read as C strings"""
    p1, p2 = p1 + b"\0", p2 + b"\0"
    i = 0
    while True:
        a, b = p1[i], p2[i]
        if (a == 0x5c and b == 0x2f) or (b == 0x5c and a == 0x2f):
            pass
        elif ignore_case:
            if _lower(a) != _lower(b):
                break
        elif a != b:
            break
        i += 1
        if p1[i] == 0 or p2[i] == 0:
            break
    return _lower(p1[i]) - _lower(p2[i]) if ignore_case else p1[i] - p2[i]


def oracle_locate(names, queries, ignore_case):
    """the first name in order that compares equal; an empty query finds nothing. Names are bucketed by C-string length (equality
    needs equal lengths) so the restatement runs only where it can match."""
    buckets = {}
    for i, n in enumerate(names):
        buckets.setdefault(len(n.split(b"\0")[0]), []).append(i)
    out = []
    for q in queries:
        qc = q.split(b"\0")[0]
        out.append(next((i for i in buckets.get(len(qc), []) if path_compare(names[i], qc, ignore_case) == 0), MISS) if qc else MISS)
    return out


def stored_archive(entries):
    """STORE entries with arbitrary name bytes (NULs, any length up to 65535), built directly; zip64 end records past 65534"""
    loc, cd, off = [], [], 0
    for name, data in entries:
        crc = zlib.crc32(data)
        loc.append(struct.pack("<IHHHHHIIIHH", 0x04034b50, 10, 0, 0, 0, 0, crc, len(data), len(data), len(name), 0) + name + data)
        cd.append(struct.pack("<IHHHHHHIIIHHHHHII", 0x02014b50, 20, 10, 0, 0, 0, 0, crc, len(data), len(data), len(name), 0, 0, 0, 0, 0, off) + name)
        off += len(loc[-1])
    body, cdb, n = b"".join(loc), b"".join(cd), len(entries)
    if n < 0xffff:
        return body + cdb + struct.pack("<IHHHHIIH", 0x06054b50, 0, 0, n, n, len(cdb), len(body), 0)
    z64 = struct.pack("<IQHHIIQQQQ", 0x06064b50, 44, 45, 45, 0, 0, n, n, len(cdb), len(body))
    return body + cdb + z64 + struct.pack("<IIQI", 0x07064b50, 0, len(body) + len(cdb), 1) + struct.pack(
        "<IHHHHIIH", 0x06054b50, 0, 0, 0xffff, 0xffff, 0xffffffff, 0xffffffff, 0)


def name_corpus(seed, nrand):
    rng = random.Random(seed)
    names = [b"a", b"ab", b"A", b"AB", b"dir/file.txt", b"dir\\file.txt", b"DIR/FILE.TXT", b"Dir\\File.Txt", b"dup", b"dup", b"DUP",
             "É.txt".encode(), "é.txt".encode(), "ÉTÉ/x".encode(), b"nul\0tail", b"nul", b"nul\0other", b"\0hidden", b"x" * 65535,
             b"x" * 65534 + b"X", b"a/b\\c/d", b"A\\B/C\\D", b"[bracket]", b"@^_`{", b"Z", b"z", b"\\", b"/"]
    alphabet = b"abcABC/\\._-0129\x80\xc3\xa9"
    for _ in range(nrand):
        names.append(bytes(rng.choice(alphabet) for _ in range(rng.randrange(1, 48))))
    return names


def name_queries(names, seed):
    rng = random.Random(seed)
    qs = [b"", b"\0", b"\0a", b"missing", b"a\0", b"ab\0zz", b"nul", b"nul\0", b"DUP", b"x" * 65535 + b"\0junk", b"X" * 65535, b"x" * 65536]
    for n in names:
        v = [n, n.upper(), n.lower(), n.swapcase(), n.replace(b"/", b"\\"), n.replace(b"\\", b"/"), n + b"!", n[:-1]]
        qs.extend(rng.sample(v, 4) if len(names) > 100 else v)
    return qs


def test_locate_against_path_compare(ctx):
    names = name_corpus(7, 2500)
    a = stored_archive([(n, b"%d" % i) for i, n in enumerate(names)])
    c = Case(ctx, a)
    try:
        assert c.check_open() and c.count == len(names)
        qs = name_queries(names, 8)
        for ic in (0, 1):
            assert ctx.rd.locate(c.h, qs, ic) == oracle_locate(names, qs, ic), ic
        assert ctx.rd.locate(c.h, [], 0) == []
        c.unchanged()
    finally:
        c.close()


def test_names_behind_a_refused_record_are_not_found(ctx):
    names = [b"one", b"two", b"three", b"four", b"two"]
    a = stored_archive([(n, b"x") for n in names])
    b = edit_directory(a, lambda i, r: r[:8] + bytes([r[8] | 1]) + r[9:] if i == 2 else r)  # record 2 encrypted: refused
    c = Case(ctx, b)
    try:
        assert c.check_open() and c.count == 2 and c.refuse == MZ_SUPPORT_ERROR
        assert ctx.rd.locate(c.h, [b"one", b"TWO", b"three", b"four"], 1) == [0, 1, MISS, MISS]
    finally:
        c.close()
    c = Case(ctx, stored_archive([]))
    try:
        assert c.check_open() and c.count == 0
        assert ctx.rd.locate(c.h, [b"a", b""], 0) == [MISS, MISS]
        assert c.check_selection([0, 3]) == MZ_END_OF_LIST
    finally:
        c.close()


@pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, "oracle/_ref/libmzref.so")), reason="oracle/_ref/libmzref.so is not built")
def test_locate_against_the_reference(ctx):
    """mz_zip_locate_entry of the reference's own reader over the same bytes (a memory stream), from the first entry each time"""
    ref = C.CDLL(os.path.join(ROOT, "oracle/_ref/libmzref.so"))
    vp, i32 = C.c_void_p, C.c_int32
    for name, res, args in (("mz_stream_mem_create", vp, []), ("mz_stream_mem_set_buffer", None, [vp, vp, i32]), ("mz_stream_mem_delete", None, [C.POINTER(vp)]),
                            ("mz_zip_create", vp, []), ("mz_zip_delete", None, [C.POINTER(vp)]), ("mz_zip_open", i32, [vp, vp, i32]),
                            ("mz_zip_close", i32, [vp]), ("mz_zip_goto_first_entry", i32, [vp]), ("mz_zip_goto_next_entry", i32, [vp]),
                            ("mz_zip_get_entry", C.c_int64, [vp]), ("mz_zip_locate_entry", i32, [vp, C.c_char_p, C.c_uint8])):
        f = getattr(ref, name)
        f.restype, f.argtypes = res, args
    names = name_corpus(9, 600)
    a = stored_archive([(n, b"") for n in names])
    keep = C.create_string_buffer(a, len(a))
    m = vp(ref.mz_stream_mem_create())
    ref.mz_stream_mem_set_buffer(m, keep, len(a))
    z = vp(ref.mz_zip_create())
    assert ref.mz_zip_open(z, m, 1) == 0
    pos, err = {}, ref.mz_zip_goto_first_entry(z)
    while err == 0:
        pos[ref.mz_zip_get_entry(z)] = len(pos)
        err = ref.mz_zip_goto_next_entry(z)
    assert len(pos) == len(names)
    qs = [q for q in name_queries(names, 10) if q.split(b"\0")[0]]  # the reference reads past an empty query's terminator
    c = Case(ctx, a)
    try:
        for ic in (0, 1):
            want = []
            for q in qs:
                assert ref.mz_zip_goto_first_entry(z) == 0
                want.append(pos[ref.mz_zip_get_entry(z)] if ref.mz_zip_locate_entry(z, q.split(b"\0")[0], ic) == 0 else MISS)
            assert ctx.rd.locate(c.h, qs, ic) == want, ic
    finally:
        c.close()
        ref.mz_zip_close(z)
        ref.mz_zip_delete(C.byref(z))
        ref.mz_stream_mem_delete(C.byref(m))


def test_locate_feeds_decode(ctx):
    """locate's output in device memory is the selection of decode, misses included (MZ_END_OF_LIST)"""
    rd, L = ctx.rd, ctx.lib
    files = corpus(10, 3000, seed=33)
    a = ctx.ex.write(files)
    c = Case(ctx, a)
    try:
        assert c.check_open()
        qs = [files[4][0].encode(), b"nope", files[0][0].upper().encode(), files[9][0].encode()]
        offs, pos = [], 0
        for q in qs:
            offs.append(pos)
            pos += len(q)
        d_names, d_off = rd.put(b"".join(qs)), rd.put(struct.pack("<4Q", *offs))
        d_len, d_idx = rd.put(struct.pack("<4I", *[len(q) for q in qs])), L.mz_cuda_malloc(16)
        assert L.mz_zip_cuda_reader_locate(c.h, d_names, d_off, d_len, 4, 1, d_idx, None) == 0
        size = C.c_uint64(0)
        assert L.mz_zip_cuda_reader_decode(c.h, d_idx, 4, None, 0, C.byref(size), None, None, None, None) == 0
        d_out, d_o, d_st = L.mz_cuda_malloc(size.value), L.mz_cuda_malloc(40), L.mz_cuda_malloc(16)
        assert L.mz_zip_cuda_reader_decode(c.h, d_idx, 4, d_out, size.value, C.byref(size), d_o, d_st, None, None) == MZ_END_OF_LIST
        raw, o = rd.get(d_out, size.value), struct.unpack("<5Q", rd.get(d_o, 40))
        assert struct.unpack("<4i", rd.get(d_st, 16)) == (0, MZ_END_OF_LIST, 0, 0)
        assert [raw[o[k]:o[k + 1]][:len(files[i][1])] for k, i in ((0, 4), (2, 0), (3, 9))] == [files[4][1], files[0][1], files[9][1]]
        for p in (d_names, d_off, d_len, d_idx, d_out, d_o, d_st):
            L.mz_cuda_free(p)
    finally:
        c.close()


def test_two_readers_on_two_threads(ctx):
    a = ctx.ex.write(corpus(12, 4000, seed=34), flags=HASH_SHA256)
    rng = random.Random(3)
    sels = [[rng.randrange(14) for _ in range(9)] for _ in range(3)]
    names = [b"d%d/f%04d.bin" % (i % 3, i) for i in range(12)] + [b"none"]

    def work(out):
        c = Case(ctx, a)
        try:
            out.append(([ctx.rd.decode(c.h, s) for s in sels], ctx.rd.locate(c.h, names, 0)))
        finally:
            c.close()
    serial = []
    work(serial)
    res = [[], []]
    ts = [threading.Thread(target=work, args=(res[k],)) for k in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert res[0] == serial and res[1] == serial


def _subprocess(lib_name, body, env):
    script = ("import ctypes as C, os, sys\nsys.path.insert(0, %r)\nimport cuharness, test_emu_device_reader as t\n"
              "ctx = t.Ctx(cuharness.pkg().configure(C.CDLL(%r)))\n" % (HERE, os.path.join(EMU, lib_name))) + body
    return subprocess.run([sys.executable, "-c", script], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)


SCHED_BODY = (
    "import hashlib\n"
    "from test_emu_native_extract import AES, HASH_SHA256, corpus, py_zip\n"
    "arcs = [(py_zip(corpus(6, 3000, seed=50)), None), (ctx.ex.write(corpus(6, 3000, seed=51), flags=HASH_SHA256), None),\n"
    "        (ctx.ex.write(corpus(5, 2000, seed=52), flags=AES, password='pw', strength=3), 'pw')]\n"
    "for k, (a, pw) in enumerate(arcs):\n"
    "    c = t.Case(ctx, a, pw)\n"
    "    sel = [0, 3, 3, 1, 9, 5, 2][:c.count + 2]\n"
    "    err, n, raw, offs, sts = ctx.rd.decode(c.h, sel)\n"
    "    good = b''.join(raw[offs[i]:offs[i + 1]] for i in range(len(sel)) if sts[i] == 0)\n"
    "    names = [n.encode() for n, _ in corpus(6, 10, seed=0)] + [b'X']\n"
    "    print('case', k, err, n, offs, sts, hashlib.sha256(good).hexdigest(), ctx.rd.locate(c.h, names, 1))\n"
    "    c.unchanged()\n"
    "    c.close()\n")


def test_schedules_and_race_checker(ctx):
    """the identity cases under three fixed thread / block schedules with the shared-memory race checker, each seed in its own
    process: the default schedule's results"""
    base = _subprocess("libmz_strm_emu.so", SCHED_BODY, dict(os.environ))
    assert base.returncode == 0, base.stdout[-3000:]
    want = [l for l in base.stdout.splitlines() if l.startswith("case")]
    assert len(want) == 3
    for seed in (3, 17, 101):
        r = _subprocess("libmz_strm_emu.so", SCHED_BODY, dict(os.environ, MZ_EMU_SCHED=str(seed), MZ_EMU_RACE="1"))
        assert r.returncode == 0, r.stdout[-3000:]
        assert [l for l in r.stdout.splitlines() if l.startswith("case")] == want, seed


def test_under_address_sanitizer(ctx, tmp_path):
    """malformed and mutated archives, out-of-range selections and short caps on the AddressSanitizer + UBSan build: no report"""
    r = subprocess.run(["make", "-s", "-C", EMU, "libmz_strm_emu_san.so"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], stdout=subprocess.PIPE, text=True).stdout.strip()
    if not os.path.isabs(asan):
        pytest.skip("libasan not found")
    arcs = [arc for arc, _ in malformed_cases(ctx.ex).values()] + mutations(99, 25)
    arcs.append(ctx.ex.write(corpus(5, 3000, seed=35), flags=AES, password="pw", strength=1))
    for k, arc in enumerate(arcs):
        (tmp_path / ("%03d.zip" % k)).write_bytes(arc)
    body = (
        "d = %r\n"
        "for f in sorted(os.listdir(d)):\n"
        "    a = open(os.path.join(d, f), 'rb').read()\n"
        "    d_arc = ctx.rd.put(a)\n"
        "    err, h, n, ref = ctx.rd.open(d_arc, len(a), 'pw')\n"
        "    if not err:\n"
        "        r1 = ctx.rd.decode(h, [0, n, n + 5, 0xffffffff, max(0, n - 1), 0])[0]\n"
        "        r2 = ctx.rd.decode(h, list(range(n)), cap_delta=-1)[0] if n else 0\n"
        "        ctx.rd.locate(h, [b'a', b'', b'd0/f0000.bin'], 1)\n"
        "        ctx.lib.mz_zip_cuda_reader_close(h)\n"
        "        print(f, err, n, r1, r2)\n"
        "    else:\n"
        "        print(f, err)\n"
        "    ctx.lib.mz_cuda_free(d_arc)\n") % str(tmp_path)
    r = _subprocess("libmz_strm_emu_san.so", body, dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0"))
    assert r.returncode == 0, r.stdout[-4000:]
    assert "ERROR: AddressSanitizer" not in r.stdout and "runtime error" not in r.stdout, r.stdout[-4000:]
    assert r.stdout.count(".zip ") == len(arcs)
