"""mz_zip_cuda_extract_device on the CPU: the real host C and kernel sources on the execution-model emulator
(tests/emu/libmz_strm_emu.so). Every archive is put in emulator device memory, in an allocation of exactly its length, and
extracted both by the device call and by mz_zip_cuda_extract_archive from a memory stream: the error codes must be equal, on
success the (name, bytes, crc) lists must be equal to each other and to zipfile's, and on an entry error every entry in front of
the first failing one must have status 0 and its right bytes."""
import ctypes as C
import os
import random
import struct
import subprocess
import sys
import zipfile
import zlib

import pytest

from test_emu_native_extract import (AES, EMU, HASH_SHA256, HERE, MZ_FORMAT_ERROR, MZ_PASSWORD_ERROR, MZ_SUPPORT_ERROR, Extractor, append_extra, corpus,
                                     edit_directory, eocd_at, malformed_cases, patch_zip64_end, py_zip, reorder_directory, zip64_directory, zipfile_view)

MZ_BUF_ERROR = -5


class DeviceExtractor:
    """ctypes driver of mz_zip_cuda_extract_device on one library (the emulator here, the product in the GPU twin)"""

    def __init__(self, lib):
        import cuharness
        self.pkg = cuharness.pkg()
        self.lib = lib

    def _dev(self, n):
        p = self.lib.mz_cuda_malloc(n)
        assert p, n
        return p

    def unchanged(self, d_arc, archive):
        """the call never writes the caller's archive (WinZip AES entries are decrypted in a copy)"""
        if archive:
            back = C.create_string_buffer(len(archive))
            assert self.lib.mz_cuda_memcpy_d2h(back, d_arc, len(archive), None) == 0
            assert back.raw == bytes(archive)

    def extract(self, archive, password=None, list_only=False):
        """-> (err, [(name, bytes, crc, status)], count, out_bytes); the archive sits in an allocation of exactly len(archive) bytes"""
        L = self.lib
        pw = password.encode() if password is not None else None
        d_arc = self._dev(len(archive))
        if archive:
            assert L.mz_cuda_memcpy_h2d(d_arc, archive, len(archive), None) == 0
        count, nbytes = C.c_uint32(0), C.c_uint64(0)
        st = self.pkg.ZipStats()
        d_ent = d_out = None
        try:
            err = L.mz_zip_cuda_extract_device(d_arc, len(archive), pw, None, 0, C.byref(count), None, 0, C.byref(nbytes), C.byref(st), None)
            if err not in (0, MZ_BUF_ERROR):  # the archive's error, or the first record refused: nothing accepted
                assert count.value == 0
                self.unchanged(d_arc, archive)
                return err, [], 0, nbytes.value
            assert (err == MZ_BUF_ERROR) == (count.value > 0)
            n, size = count.value, nbytes.value
            d_ent = self._dev(max(1, n) * C.sizeof(self.pkg.ZipDevEntry))
            d_out = None if list_only else self._dev(size)  # exactly out_bytes
            err = L.mz_zip_cuda_extract_device(d_arc, len(archive), pw, d_ent, n, C.byref(count), d_out, size, C.byref(nbytes), C.byref(st), None)
            assert count.value == n and nbytes.value == size  # MZ_BUF_ERROR now would be an entry's (a truncated stream)
            rows = (self.pkg.ZipDevEntry * max(1, n))()
            assert L.mz_cuda_memcpy_d2h(rows, d_ent, n * C.sizeof(self.pkg.ZipDevEntry), None) == 0
            out = C.create_string_buffer(max(1, size))
            if d_out and size:
                assert L.mz_cuda_memcpy_d2h(out, d_out, size, None) == 0
            raw = out.raw
            got = [(archive[r.name_off:r.name_off + r.name_len].decode("utf-8", "replace"),
                    b"" if list_only else raw[r.out_off:r.out_off + r.usize], r.crc, r.status) for r in rows[:n]]
            if not list_only and n:
                assert st.entries == n and st.bytes_out == sum(r.usize for r in rows[:n])
            self.unchanged(d_arc, archive)
            return err, got, n, size
        finally:
            for p in (d_arc, d_ent, d_out):
                if p:
                    L.mz_cuda_free(p)


@pytest.fixture(scope="module")
def pair(built):
    r = subprocess.run(["make", "-s", "-C", EMU, "libmz_strm_emu.so"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    import cuharness
    lib = cuharness.pkg().configure(C.CDLL(os.path.join(EMU, "libmz_strm_emu.so")))
    return Extractor(lib), DeviceExtractor(lib)


def archive_extract(ex, archive, password=None):
    """mz_zip_cuda_extract_archive from a memory stream -> (err, [(name, bytes, crc)]); names that are not UTF-8 are kept"""
    got = []

    def on_entry(_ud, name, data, size, crc):
        got.append((name.decode("utf-8", "replace"), C.string_at(data, size) if size else b"", crc))
        return 0
    cb = ex.pkg.ZIP_ENTRY_CB(on_entry)
    src, keep = ex.t.source(archive)
    err = ex.lib.mz_zip_cuda_extract_archive(src, password.encode() if password else None, 0, cb, None, None)
    ex.t.delete(src)
    del keep
    return err, got


def differential(pair, archive, password=None, want=None):
    """both extractors on the same bytes; returns (err, [(name, bytes, crc)] of the device call)"""
    ex, dx = pair
    err_a, got_a = archive_extract(ex, archive, password=password)
    err_d, got_d, n, size = dx.extract(archive, password=password)
    assert err_d == err_a, (err_d, err_a)
    plain = [(a.split("\0")[0], b, c) for a, b, c, _ in got_d]  # the callback of extract_archive takes names as C strings
    if err_a == 0:
        assert all(s == 0 for *_, s in got_d)
        assert plain == got_a
        if want is not None:
            assert plain == want
    else:
        first = next((i for i, g in enumerate(got_d) if g[3]), n)
        for name, data, crc in plain[:first]:
            assert zlib.crc32(data) == crc, name
        assert got_a == plain[:len(got_a)]  # extract_archive delivers whole verified rounds only
    # list only: the same table, nothing decoded
    err_l, got_l, n_l, size_l = dx.extract(archive, password=password, list_only=True)
    assert n_l == n and size_l == size and [g[:1] + g[2:] for g in got_l] == [(g[0], g[2], 0) for g in got_d]
    if any(g[3] for g in got_d):  # an entry error needs decoding: listing returns only what ended the list, if anything did
        assert err_l in (0, MZ_FORMAT_ERROR, MZ_SUPPORT_ERROR, MZ_PASSWORD_ERROR), err_l
    else:
        assert err_l == err_d, (err_l, err_d)
    return err_d, plain


def test_zipfile_archives(pair):
    files = corpus(12, 3000, seed=21)
    for comp in (zipfile.ZIP_STORED, zipfile.ZIP_DEFLATED):
        a = py_zip(files, comp, dirs=("empty_dir/",))
        assert differential(pair, a, want=zipfile_view(a))[0] == 0


def test_data_descriptors_and_zip64_fields(pair):
    files = corpus(7, 5000, seed=22)
    for a in (py_zip(files, stream=True), py_zip(files, force_zip64=True), zip64_directory(py_zip(files))):
        assert differential(pair, a, want=zipfile_view(a))[0] == 0


@pytest.mark.parametrize("flags", [0, HASH_SHA256])
def test_native_writer_archives(pair, flags):
    files = corpus(9, 70000, seed=23)
    a = pair[0].write(files, flags=flags)
    err, got = differential(pair, a, want=zipfile_view(a))
    assert err == 0 and [(n, d) for n, d, _ in got] == files


@pytest.mark.parametrize("strength", [1, 2, 3])
def test_aes_archives(pair, strength):
    files = corpus(6, 4000, seed=24)
    pw = "pw-%d" % strength
    a = pair[0].write(files, flags=AES | HASH_SHA256, password=pw, strength=strength)
    err, got = differential(pair, a, password=pw)  # the device archive is read back after every call: the copy was decrypted, not it
    assert err == 0 and got == [(n, d, zlib.crc32(d)) for n, d in files]
    assert differential(pair, a, password="wrong")[0] == -108
    assert differential(pair, a)[0] == -108


def test_zip64_end_prepended_data_and_reordered_directory(pair):
    files = corpus(8, 2000, seed=25)
    a = py_zip(files)
    want = zipfile_view(a)
    assert differential(pair, patch_zip64_end(a), want=want)[0] == 0
    assert differential(pair, b"\x7fSFX" * 250 + a, want=want)[0] == 0
    r = reorder_directory(a)  # local-header offsets out of order: the extents need the sort
    err, got = differential(pair, r, want=zipfile_view(r))
    assert err == 0 and [g[0] for g in got] == [f[0] for f in reversed(files)]


def test_malformed_archives(pair):
    for name, (arc, codes) in malformed_cases(pair[0]).items():
        assert differential(pair, arc)[0] in codes, name


def test_refusal_ends_the_list(pair):
    a = py_zip(corpus(6, 3000, seed=26))
    want = zipfile_view(a)
    b = edit_directory(a, lambda i, r: r[:8] + bytes([r[8] | 1]) + r[9:] if i == 3 else r)
    err, got = differential(pair, b)
    assert err == MZ_SUPPORT_ERROR and got == want[:3]


def test_buffers_too_small_write_nothing(pair):
    """MZ_BUF_ERROR: the counts are reported, and neither the table nor the output is touched"""
    dx = pair[1]
    L = dx.lib
    a = py_zip(corpus(5, 3000, seed=30))
    err, got, n, size = dx.extract(a)
    assert err == 0 and n == 5
    d_arc = dx._dev(len(a))
    assert L.mz_cuda_memcpy_h2d(d_arc, a, len(a), None) == 0
    row = C.sizeof(dx.pkg.ZipDevEntry)
    d_ent, d_out = dx._dev(n * row), dx._dev(size)
    for p, nb in ((d_ent, n * row), (d_out, size)):
        assert L.mz_cuda_memset(p, 0xab, nb, None) == 0
    count, nbytes = C.c_uint32(0), C.c_uint64(0)
    for max_entries, out_cap in ((n - 1, size), (n, size - 16), (n - 1, None)):
        err = L.mz_zip_cuda_extract_device(d_arc, len(a), None, d_ent, max_entries, C.byref(count), d_out if out_cap is not None else None,
                                           out_cap or 0, C.byref(nbytes), None, None)
        assert (err, count.value, nbytes.value) == (MZ_BUF_ERROR, n, size)
        for p, nb in ((d_ent, n * row), (d_out, size)):
            back = C.create_string_buffer(nb)
            assert L.mz_cuda_memcpy_d2h(back, p, nb, None) == 0
            assert back.raw == b"\xab" * nb
    for p in (d_arc, d_ent, d_out):
        L.mz_cuda_free(p)


def with_count(a, delta):
    e = eocd_at(a)
    b = bytearray(a)
    cnt = struct.unpack("<H", a[e + 10:e + 12])[0] + delta
    b[e + 8:e + 12] = struct.pack("<HH", cnt, cnt)
    return bytes(b)


def test_zero_entries_and_wrong_counts(pair):
    assert differential(pair, py_zip([]))[0] == 0
    a = py_zip(corpus(5, 1000, seed=27))
    assert differential(pair, with_count(a, -1))[0] == MZ_FORMAT_ERROR
    assert differential(pair, with_count(a, 1))[0] == MZ_FORMAT_ERROR
    assert differential(pair, b"")[0] == MZ_FORMAT_ERROR


def adversarial_cases(pair):
    """signatures the chain must never reach: PK\\1\\2 inside names, unknown extra fields and the archive comment, with lengths
    that chain into real records; a fake end record inside the comment"""
    files = corpus(6, 2000, seed=28)
    a = py_zip(files)
    e = eocd_at(a)
    cd_size, cd_off = struct.unpack("<II", a[e + 12:e + 20])
    cases = {}
    # a name that holds a whole fake record header whose lengths point at the next real record
    fake = b"PK\x01\x02" + b"\0" * 24 + struct.pack("<HHH", 0, 0, 0) + b"\0" * 12

    def long_name(i, r):
        if i != 1:
            return r
        nl, xl, cl = struct.unpack("<HHH", r[28:34])
        name = r[46:46 + nl] + fake
        return r[:28] + struct.pack("<H", len(name)) + r[30:46] + name + r[46 + nl:]
    b = edit_directory(a, long_name)
    # the names in the local headers differ now; the directory decides what the entry is called
    cases["signature_in_name"] = b
    cases["signature_in_extra_field"] = edit_directory(a, lambda i, r: append_extra(
        r, struct.pack("<HH", 0xcafe, len(fake)) + fake) if i in (0, 3) else r)
    # the archive comment: a fake record and a fake end record behind the real one
    comment = fake + b"PK\x05\x06" + b"\0" * 18
    c = bytearray(a)
    c[e + 20:e + 22] = struct.pack("<H", len(comment))
    cases["signatures_in_comment"] = bytes(c) + comment
    return cases


def test_adversarial_signatures(pair):
    for name, arc in adversarial_cases(pair).items():
        err, got = differential(pair, arc)
        if name == "signature_in_extra_field":
            assert err == 0 and len(got) == 6, name


def mutations(seed, rounds):
    rng = random.Random(seed)
    a = py_zip(corpus(5, 600, seed=29))
    e = eocd_at(a)
    cd_off = struct.unpack("<I", a[e + 16:e + 20])[0]
    out = []
    for _ in range(rounds):
        b = bytearray(a)
        for _k in range(rng.choice((1, 1, 2, 3))):
            pos = rng.randrange(cd_off, len(b))
            b[pos] = rng.choice((0, 0xff, rng.randrange(256), b[pos] ^ (1 << rng.randrange(8))))
        out.append(bytes(b))
    return out


def test_random_directory_mutations(pair):
    for k, arc in enumerate(mutations(1234, 300)):
        try:
            differential(pair, arc)
        except AssertionError as x:
            raise AssertionError("mutation %d: %s" % (k, x)) from None


def test_under_address_sanitizer(pair, tmp_path):
    """the malformed, adversarial and mutated archives on the AddressSanitizer build: every archive in an allocation of exactly its
    length, no report"""
    r = subprocess.run(["make", "-s", "-C", EMU, "libmz_strm_emu_san.so"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], stdout=subprocess.PIPE, text=True).stdout.strip()
    if not os.path.isabs(asan):
        pytest.skip("libasan not found")
    arcs = [arc for arc, _ in malformed_cases(pair[0]).values()] + list(adversarial_cases(pair).values()) + mutations(99, 40)
    for k, arc in enumerate(arcs):
        (tmp_path / ("%03d.zip" % k)).write_bytes(arc)
    script = (
        "import ctypes as C, os, sys\n"
        "sys.path.insert(0, %r)\n"
        "import cuharness, test_emu_device_extract as t\n"
        "x = t.DeviceExtractor(cuharness.pkg().configure(C.CDLL(%r)))\n"
        "for f in sorted(os.listdir(%r)):\n"
        "    print(f, x.extract(open(os.path.join(%r, f), 'rb').read())[0])\n"
    ) % (HERE, os.path.join(EMU, "libmz_strm_emu_san.so"), str(tmp_path), str(tmp_path))
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([sys.executable, "-c", script], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-4000:]
    assert "ERROR: AddressSanitizer" not in r.stdout and "runtime error" not in r.stdout, r.stdout[-4000:]
    assert r.stdout.count(".zip ") == len(arcs)
