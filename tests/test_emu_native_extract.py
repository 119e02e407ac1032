"""mz_zip_cuda_extract_archive on the CPU: the real host C and kernel sources on the execution-model emulator
(tests/emu/libmz_strm_emu.so), archives held in memory streams (tests/support/libmztest.so). Every valid archive must deliver the
(name, bytes, crc) sequence CPython's zipfile reads; malformed ones must be refused with the reference's error codes."""
import ctypes as C
import io
import os
import struct
import subprocess
import sys
import zipfile
import zlib

import pytest

import datagen

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
MZ_DATA_ERROR, MZ_BUF_ERROR, MZ_FORMAT_ERROR, MZ_CRC_ERROR = -3, -5, -103, -105
MZ_PASSWORD_ERROR, MZ_SUPPORT_ERROR = -108, -109
HASH_SHA256, ALL_DEVICES, AES = 1, 2, 4


class Extractor:
    """ctypes driver of the native writer and extractor on one library (the emulator here, the product in the GPU twin)"""

    def __init__(self, lib):
        import cuharness
        self.pkg = cuharness.pkg()
        self.lib = lib
        self.t = cuharness.TestLib()

    def write(self, files, level=6, flags=0, password=None, strength=0):
        """the product's native writer into memory; files = [(name, bytes)]"""
        pkg = self.pkg
        items = (pkg.ZipItem * max(1, len(files)))()
        keep = []
        for i, (name, data) in enumerate(files):
            b = C.create_string_buffer(data, max(1, len(data)))
            keep.append(b)
            items[i] = pkg.ZipItem(name.encode(), C.cast(b, C.c_void_p), len(data), 1700000000, 0, 0)
        sink = self.t.sink()
        st = pkg.ZipStats()
        if flags & AES:
            err = self.lib.mz_zip_cuda_write_archive_aes(sink, items, len(files), level, flags, password.encode(), strength, C.byref(st))
        else:
            err = self.lib.mz_zip_cuda_write_archive(sink, items, len(files), level, flags, C.byref(st))
        assert err == 0, err
        out = self.t.sink_bytes(sink)
        self.t.delete(sink)
        return out

    def extract(self, archive, password=None, flags=0, stop_after=None, stop_code=7):
        """-> (err, [(name, bytes, crc)], stats)"""
        got = []

        def on_entry(_ud, name, data, size, crc):
            got.append((name.decode(), C.string_at(data, size) if size else b"", crc))
            if stop_after is not None and len(got) == stop_after:
                return stop_code
            return 0
        cb = self.pkg.ZIP_ENTRY_CB(on_entry)
        src, keep = self.t.source(archive)
        st = self.pkg.ZipStats()
        err = self.lib.mz_zip_cuda_extract_archive(src, password.encode() if password else None, flags, cb, None, C.byref(st))
        self.t.delete(src)
        del keep
        return err, got, st


def zipfile_view(archive, password=None):
    with zipfile.ZipFile(io.BytesIO(archive)) as z:
        return [(i.filename, z.read(i), i.CRC) for i in z.infolist()]


def corpus(n, size, seed=0):
    files = []
    for i in range(n):
        k = i % 5
        sz = [size, 0, 1, size // 3 + 7, size * 2 + 13][k]
        data = (datagen.text_like(sz, seed=seed + i) if k != 4 else datagen.random_bytes(sz, seed=seed + i))[:sz]
        files.append(("d%d/f%04d.bin" % (i % 3, i), data))
    return files


def py_zip(files, compression=zipfile.ZIP_DEFLATED, force_zip64=False, stream=False, dirs=()):
    bio = io.BytesIO()

    class Unseekable(io.RawIOBase):  # zipfile then writes data descriptors
        def writable(self):
            return True

        def write(self, b):
            return bio.write(b)
    target = Unseekable() if stream else bio
    with zipfile.ZipFile(target, "w", compression=compression) as z:
        for d in dirs:
            z.writestr(zipfile.ZipInfo(d), b"")
        for name, data in files:
            if force_zip64:
                zi = zipfile.ZipInfo(name)
                zi.compress_type = compression
                with z.open(zi, "w", force_zip64=True) as f:
                    f.write(data)
            else:
                z.writestr(name, data, compress_type=compression)
    return bio.getvalue()


def eocd_at(a):
    return a.rfind(b"PK\x05\x06")


def patch_zip64_end(a):
    """rewrite the end record as zip64: a zip64 end record and locator in front of a saturated classic one"""
    e = eocd_at(a)
    _, _, _, _, cnt, cd_size, cd_off, _ = struct.unpack("<IHHHHIIH", a[e:e + 22])
    body = a[:e]
    z64_off = len(body)
    z64 = struct.pack("<IQHHIIQQQQ", 0x06064b50, 44, 45, 45, 0, 0, cnt, cnt, cd_size, cd_off)
    loc = struct.pack("<IIQI", 0x07064b50, 0, z64_off, 1)
    end = struct.pack("<IHHHHIIH", 0x06054b50, 0, 0, 0xffff, 0xffff, 0xffffffff, 0xffffffff, 0)
    return body + z64 + loc + end


def reorder_directory(a):
    """the same archive with its central-directory records in reverse order"""
    e = eocd_at(a)
    cd_size, cd_off = struct.unpack("<II", a[e + 12:e + 20])
    recs, p, cd = [], 0, a[cd_off:cd_off + cd_size]
    while p < len(cd):
        nl, xl, cl = struct.unpack("<HHH", cd[p + 28:p + 34])
        recs.append(cd[p:p + 46 + nl + xl + cl])
        p += 46 + nl + xl + cl
    return a[:cd_off] + b"".join(reversed(recs)) + a[cd_off + cd_size:]


def edit_directory(a, fn):
    """the archive with central-directory record i replaced by fn(i, record); the end record's directory size follows"""
    e = eocd_at(a)
    cd_size, cd_off = struct.unpack("<II", a[e + 12:e + 20])
    recs, p, cd = [], 0, a[cd_off:cd_off + cd_size]
    while p < len(cd):
        nl, xl, cl = struct.unpack("<HHH", cd[p + 28:p + 34])
        recs.append(cd[p:p + 46 + nl + xl + cl])
        p += 46 + nl + xl + cl
    new = b"".join(fn(i, r) for i, r in enumerate(recs))
    end = bytearray(a[e:])
    end[12:16] = struct.pack("<I", len(new))
    return a[:cd_off] + new + bytes(end)


def append_extra(rec, field):
    """a directory record (without comment) with `field` appended to its extra field"""
    nl, xl, cl = struct.unpack("<HHH", rec[28:34])
    assert cl == 0
    return rec[:30] + struct.pack("<H", xl + len(field)) + rec[32:] + field


def zip64_directory(a):
    """every directory record with sizes and header offset saturated and a zip64 extra field holding them (mz_zip.c:325-343 order:
    uncompressed, compressed, offset)"""
    def fn(_i, rec):
        csize, usize = struct.unpack("<II", rec[20:28])
        off = struct.unpack("<I", rec[42:46])[0]
        r = bytearray(rec)
        r[20:28] = b"\xff" * 8
        r[42:46] = b"\xff" * 4
        return append_extra(bytes(r), struct.pack("<HHQQQ", 1, 24, usize, csize, off))
    return edit_directory(a, fn)


def first_data_offset(a):
    nl, xl = struct.unpack("<HH", a[26:30])
    return 30 + nl + xl


@pytest.fixture(scope="module")
def ex(built):
    r = subprocess.run(["make", "-s", "-C", EMU, "libmz_strm_emu.so"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    import cuharness
    return Extractor(cuharness.pkg().configure(C.CDLL(os.path.join(EMU, "libmz_strm_emu.so"))))


def check_same(ex, archive, password=None, flags=0):
    err, got, st = ex.extract(archive, password=password, flags=flags)
    assert err == 0, err
    assert got == zipfile_view(archive) if password is None else True
    assert st.entries == len(got)
    return got


@pytest.mark.parametrize("compression", [zipfile.ZIP_STORED, zipfile.ZIP_DEFLATED])
def test_zipfile_archives(ex, compression):
    files = corpus(12, 3000, seed=1)
    check_same(ex, py_zip(files, compression, dirs=("empty_dir/",)))


def test_data_descriptors_and_zip64_extra_fields(ex):
    files = corpus(7, 5000, seed=2)
    check_same(ex, py_zip(files, stream=True))
    check_same(ex, py_zip(files, force_zip64=True))  # zip64 extra fields in the local headers
    z = zip64_directory(py_zip(files))  # ... and in the central directory
    assert zipfile_view(z) == zipfile_view(py_zip(files))
    check_same(ex, z)


def test_refusal_ends_the_list_after_earlier_entries(ex):
    a = py_zip(corpus(6, 3000, seed=9))
    want = zipfile_view(a)

    def pkware_at(k):
        return lambda i, r: r[:8] + bytes([r[8] | 1]) + r[9:] if i == k else r
    err, got, _ = ex.extract(edit_directory(a, pkware_at(3)))
    assert err == MZ_SUPPORT_ERROR and got == want[:3]  # the entries in front of the refused one are delivered
    # an earlier entry's CRC error decides before a later refusal
    b = edit_directory(a, lambda i, r: r[:16] + struct.pack("<I", struct.unpack("<I", r[16:20])[0] ^ 1) + r[20:] if i == 1 else pkware_at(4)(i, r))
    err, got, _ = ex.extract(b)
    assert err == MZ_CRC_ERROR and got == []


@pytest.mark.parametrize("flags", [0, HASH_SHA256])
def test_native_writer_archives(ex, flags):
    files = corpus(9, 70000, seed=3)
    a = ex.write(files, flags=flags)
    got = check_same(ex, a)
    assert [(n, d) for n, d, _ in got] == files


@pytest.mark.parametrize("strength", [1, 2, 3])
def test_aes_archives(ex, strength):
    files = corpus(6, 4000, seed=4)
    a = ex.write(files, flags=AES | HASH_SHA256, password="pw-%d" % strength, strength=strength)
    err, got, _ = ex.extract(a, password="pw-%d" % strength)
    assert err == 0
    assert [(n, d, c) for n, d, c in got] == [(n, d, zlib.crc32(d)) for n, d in files]
    assert ex.extract(a, password="wrong")[0] == MZ_PASSWORD_ERROR
    assert ex.extract(a)[0] == MZ_PASSWORD_ERROR


def test_zip64_end_record_prepended_data_and_directory_order(ex):
    files = corpus(8, 2000, seed=5)
    a = py_zip(files)
    check_same(ex, patch_zip64_end(a))
    err, got, _ = ex.extract(b"\x7fSFX" * 250 + a)  # 1000 bytes in front: the offsets are corrected as the reference does
    assert err == 0 and got == zipfile_view(a)
    r = reorder_directory(a)
    err, got, _ = ex.extract(r)
    assert err == 0 and got == zipfile_view(r) and [g[0] for g in got] == [f[0] for f in reversed(files)]


def test_many_rounds_and_all_devices(ex, monkeypatch):
    files = corpus(60, 90000, seed=6)
    a = ex.write(files)
    one = check_same(ex, a)
    monkeypatch.setenv("MZ_CUDA_ZIP_ROUND_MB", "1")
    err, many, st = ex.extract(a)
    assert err == 0 and many == one and st.rounds >= 3
    err, alld, _ = ex.extract(a, flags=ALL_DEVICES)
    assert err == 0 and alld == one
    ex.lib.mz_zip_cuda_trim()


def test_callback_stops_delivery(ex):
    a = py_zip(corpus(10, 1000, seed=7))
    err, got, _ = ex.extract(a, stop_after=4)
    assert err == 7 and len(got) == 4


def malformed_cases(ex):
    files = corpus(6, 6000, seed=8)
    a = py_zip(files)
    cases = {}
    d0 = first_data_offset(a)
    b = bytearray(a)
    b[d0 + 40] ^= 0x55
    cases["flipped_compressed_byte"] = (bytes(b), (MZ_DATA_ERROR, MZ_BUF_ERROR, MZ_CRC_ERROR))
    b = bytearray(a)
    b[1] ^= 0xff
    cases["broken_local_signature"] = (bytes(b), (MZ_FORMAT_ERROR,))
    cases["truncated_no_end_record"] = (a[:len(a) * 2 // 3], (MZ_FORMAT_ERROR,))
    e = eocd_at(a)
    cd_off = struct.unpack("<I", a[e + 16:e + 20])[0]
    b = bytearray(a)
    b[cd_off + 42:cd_off + 46] = struct.pack("<I", cd_off + 10)  # first entry's header offset inside the directory
    cases["offset_past_directory"] = (bytes(b), (MZ_FORMAT_ERROR,))
    b = bytearray(a)
    b[e + 16:e + 20] = struct.pack("<I", e + 100)  # directory beyond the end record
    cases["directory_past_end"] = (bytes(b), (MZ_FORMAT_ERROR,))
    sha = ex.write(files[:3], flags=HASH_SHA256)
    e = eocd_at(sha)
    cd_off = struct.unpack("<I", sha[e + 16:e + 20])[0]
    b = bytearray(sha)
    b[b.index(b"\x51\x1a\x24\x00", cd_off) + 20] ^= 1
    cases["flipped_hash_byte"] = (bytes(b), (MZ_CRC_ERROR,))
    b = bytearray(a)
    cdh = cd_off = struct.unpack("<I", a[eocd_at(a) + 16:eocd_at(a) + 20])[0]
    b[cdh + 8] |= 1  # PKWARE-encrypted
    cases["pkware_entry"] = (bytes(b), (MZ_SUPPORT_ERROR,))
    b = bytearray(a)
    b[cdh + 10:cdh + 12] = struct.pack("<H", 12)  # bzip2
    cases["method_12"] = (bytes(b), (MZ_SUPPORT_ERROR,))
    b = bytearray(a)
    b[cdh + 16] ^= 1  # recorded CRC
    cases["wrong_crc"] = (bytes(b), (MZ_CRC_ERROR,))
    b = bytearray(a)
    b[cdh + 20:cdh + 24] = struct.pack("<I", 0x7ffff)  # compressed size past the extent
    cases["size_past_extent"] = (bytes(b), (MZ_FORMAT_ERROR,))
    b = bytearray(a)
    b[26:28] = struct.pack("<H", 0xffff)  # local name length past the extent
    cases["local_name_past_extent"] = (bytes(b), (MZ_FORMAT_ERROR,))
    last = len(files) - 1
    # extra fields cut short at the very end of the directory: a field's length is clamped to what is left, as the reference does,
    # so a truncated AES field is no AES field, and a truncated zip64 field leaves a saturated size saturated
    cases["truncated_aes_field"] = (edit_directory(a, lambda i, r: append_extra(r, b"\x01\x99\x07\x00") if i == last else r), (0,))
    cases["truncated_zip64_field"] = (edit_directory(a, lambda i, r: append_extra(r[:24] + b"\xff" * 4 + r[28:], b"\x01\x00\x08\x00")
                                                     if i == last else r), (MZ_SUPPORT_ERROR,))
    return cases


def test_malformed_archives_are_refused(ex):
    for name, (arc, codes) in malformed_cases(ex).items():
        err, got, _ = ex.extract(arc)
        assert err in codes, (name, err)
        assert not got or err != MZ_FORMAT_ERROR or name in ("broken_local_signature",), name


def test_malformed_archives_under_address_sanitizer(ex, tmp_path):
    """the same cases on the AddressSanitizer build: a hostile directory or header never reads outside the staging"""
    r = subprocess.run(["make", "-s", "-C", EMU, "libmz_strm_emu_san.so"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], stdout=subprocess.PIPE, text=True).stdout.strip()
    if not os.path.isabs(asan):
        pytest.skip("libasan not found")
    for name, (arc, codes) in malformed_cases(ex).items():
        (tmp_path / (name + ".zip")).write_bytes(arc)
    script = (
        "import ctypes as C, os, sys\n"
        "sys.path.insert(0, %r)\n"
        "import cuharness, test_emu_native_extract as t\n"
        "x = t.Extractor(cuharness.pkg().configure(C.CDLL(%r)))\n"
        "for f in sorted(os.listdir(%r)):\n"
        "    print(f, x.extract(open(os.path.join(%r, f), 'rb').read())[0])\n"
    ) % (HERE, os.path.join(EMU, "libmz_strm_emu_san.so"), str(tmp_path), str(tmp_path))
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([sys.executable, "-c", script], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:]
    assert "ERROR: AddressSanitizer" not in r.stdout and "runtime error" not in r.stdout, r.stdout[-4000:]
    cases = malformed_cases(ex)
    for line in r.stdout.splitlines():
        if line.endswith(".zip") is False and ".zip " in line:
            f, code = line.rsplit(" ", 1)
            assert int(code) in cases[f[:-4]][1], line


def pair_check(lib_path, tmp_path, archives):
    """extract_all (the reference's directory walk) and extract_archive on the same archives and base stream, in one process
    (tests/extract_pair.py): the same entries, byte for byte, and the same error"""
    if not os.path.exists(os.path.join(os.path.dirname(HERE), "oracle", "_ref", "libmzref.so")):
        pytest.skip("oracle/_ref/libmzref.so not built (needs the reference sources at build time)")
    import json
    for k, (arc, password) in enumerate(archives):
        path = tmp_path / ("pair%d.zip" % k)
        path.write_bytes(arc)
        r = subprocess.run([sys.executable, os.path.join(HERE, "extract_pair.py"), lib_path, str(path)] + ([password] if password else []),
                           stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=1800)
        assert r.returncode == 0, r.stderr[-2000:]
        out = json.loads(r.stdout.strip().splitlines()[-1])
        assert out["all"]["err"] == out["native"]["err"], (k, out["all"]["err"], out["native"]["err"])
        assert out["all"]["entries"] == out["native"]["entries"], k
    return out


def pair_archives(ex, n, size):
    """(libmzref.so is the reference without its WinZip AES stream, so its reader refuses AES entries: those are compared through
    oracle/_ref/zipbatch_cudae in the WinZip AES tests)"""
    files = corpus(n, size, seed=10)
    a = py_zip(files)
    cases = malformed_cases(ex)
    return [(a, None), (py_zip(files, zipfile.ZIP_STORED), None), (ex.write(files, flags=HASH_SHA256), None),
            (cases["wrong_crc"][0], None),
            (cases["flipped_hash_byte"][0], None)]


def test_same_output_as_extract_all(ex, tmp_path):
    pair_check(os.path.join(EMU, "libmz_strm_emu.so"), tmp_path, pair_archives(ex, 20, 20000))
