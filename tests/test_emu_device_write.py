"""mz_zip_cuda_write_device on the CPU: the real host C and kernel sources on the execution-model emulator
(tests/emu/libmz_strm_emu.so). Every device buffer is an allocation of exactly its size. The device writer's archive must be byte for
byte what mz_zip_cuda_write_archive writes for the same entries (with AES: equal outside the salt, verifier, ciphertext and
authentication code), must read back through zipfile and mz_zip_cuda_extract_device, and must list the same table."""
import ctypes as C
import io
import os
import random
import struct
import subprocess
import sys
import threading
import zipfile

import pytest

from test_emu_native_extract import AES, EMU, HASH_SHA256, HERE, MZ_BUF_ERROR, MZ_PASSWORD_ERROR, MZ_SUPPORT_ERROR, corpus
from test_emu_device_extract import DeviceExtractor

MZ_PARAM_ERROR = -102
DATE = 1700000000


class DeviceWriter:
    """ctypes driver of mz_zip_cuda_write_device and mz_zip_cuda_write_archive[_aes] on one library (the emulator here, the product in
    the GPU twin)"""

    def __init__(self, lib):
        import cuharness
        self.pkg = cuharness.pkg()
        self.lib = lib
        self.t = cuharness.TestLib()

    def dev(self, data):
        """an allocation of exactly len(data) bytes holding data (None for no bytes)"""
        if not data:
            return None
        p = self.lib.mz_cuda_malloc(len(data))
        assert p
        assert self.lib.mz_cuda_memcpy_h2d(p, bytes(data), len(data), None) == 0
        return p

    def back(self, p, n):
        b = C.create_string_buffer(max(1, n))
        if n:
            assert self.lib.mz_cuda_memcpy_d2h(b, p, n, None) == 0
        return b.raw[:n]

    def host(self, files, level=6, flags=0, password=None, strength=0, date=DATE):
        """mz_zip_cuda_write_archive[_aes] into a memory sink -> (err, bytes)"""
        items = (self.pkg.ZipItem * max(1, len(files)))()
        keep = []
        for i, (name, data) in enumerate(files):
            b = C.create_string_buffer(data, max(1, len(data)))
            keep.append(b)
            items[i] = self.pkg.ZipItem(name if isinstance(name, bytes) else name.encode(), C.cast(b, C.c_void_p), len(data), date, 0, 0)
        sink = self.t.sink()
        if flags & AES:
            err = self.lib.mz_zip_cuda_write_archive_aes(sink, items, len(files), level, flags, password.encode(), strength, None)
        else:
            err = self.lib.mz_zip_cuda_write_archive(sink, items, len(files), level, flags, None)
        out = self.t.sink_bytes(sink)
        self.t.delete(sink)
        return err, out

    def layout(self, files, offsets=None, order=None):
        """-> (data, names, items): the entries' bytes at `offsets` (default: packed in order, 16-byte aligned) of one buffer"""
        n = len(files)
        if offsets is None:
            offsets, pos = [], 0
            for _, d in files:
                offsets.append(pos)
                pos += (len(d) + 15) & ~15
        end = max([o + len(d) for o, (_, d) in zip(offsets, files)] + [0])
        data = bytearray(end)
        for o, (_, d) in zip(offsets, files):
            data[o:o + len(d)] = d
        names, items = b"", (self.pkg.ZipDevItem * max(1, n))()
        for i, (name, d) in enumerate(files):
            nm = name if isinstance(name, bytes) else name.encode()
            items[i] = self.pkg.ZipDevItem(offsets[i], len(d), len(names), len(nm), self.pkg.dos_date(DATE), 0, 0)
            names += nm
        return bytes(data), names, bytes(items)[:n * 40]

    def device(self, files, level=6, flags=0, password=None, strength=0, offsets=None, cap=None, layout=None, entries=False, sizing=True, slack=0,
               null_data=False, null_names=False):
        """mz_zip_cuda_write_device -> (err, archive bytes, [entry rows], length, bound); inputs read back unchanged. slack: the archive
        buffer has that many bytes of 0xab behind cap, which must be left as they are; null_*: pass NULL for d_data / d_names"""
        L = self.lib
        data, names, items = layout or self.layout(files, offsets)
        d_data, d_names, d_items = self.dev(data), self.dev(names), self.dev(items)
        a_data, a_names = None if null_data else d_data, None if null_names else d_names
        pw = password.encode() if password is not None else None
        n = C.c_uint64(0)
        bound = None
        try:
            if sizing:
                err = L.mz_zip_cuda_write_device(a_data, a_names, d_items, len(files), level, flags, pw, strength, None, 0, C.byref(n), None, None, None)
                if err:
                    return err, b"", [], 0, None
                bound = n.value
            size = bound if cap is None else cap
            d_arc = L.mz_cuda_malloc(max(1, size + slack))
            if slack:
                assert L.mz_cuda_memset(d_arc, 0xab, size + slack, None) == 0
            d_ent = L.mz_cuda_malloc(max(1, len(files)) * 72) if entries else None
            st = self.pkg.ZipStats()
            err = L.mz_zip_cuda_write_device(a_data, a_names, d_items, len(files), level, flags, pw, strength, d_arc, size, C.byref(n), d_ent, C.byref(st), None)
            out = self.back(d_arc, min(n.value, size)) if err in (0, MZ_BUF_ERROR) else b""
            if slack:
                assert self.back(d_arc, size + slack)[size:] == b"\xab" * slack, "written at or beyond cap"
            rows = []
            if entries and err == 0:
                raw = self.back(d_ent, len(files) * 72)
                rows = list((self.pkg.ZipDevEntry * max(1, len(files))).from_buffer_copy(raw.ljust(72, b"\0")))[:len(files)]
            L.mz_cuda_free(d_arc)
            if d_ent:
                L.mz_cuda_free(d_ent)
            if err == 0:
                assert st.entries == len(files) and st.bytes_in == sum(len(d) for _, d in files)
            assert self.back(d_data, len(data)) == data and self.back(d_names, len(names)) == names and self.back(d_items, len(items)) == items
            return err, out, rows, n.value, bound
        finally:
            for p in (d_data, d_names, d_items):
                if p:
                    L.mz_cuda_free(p)


def aes_ranges(a):
    """the byte ranges of an AES archive that depend on the salts: salt, verifier, ciphertext and authentication code of every entry"""
    out, p = [], 0
    while a[p:p + 4] == b"PK\x03\x04":
        csize, _, nl, xl = struct.unpack("<IIHH", a[p + 18:p + 30])
        d = p + 30 + nl + xl
        out.append((d, d + csize))
        p = d + csize
    return out


def mask(a, ranges):
    b = bytearray(a)
    for lo, hi in ranges:
        b[lo:hi] = b"\0" * (hi - lo)
    return bytes(b)


def edge_corpus():
    return [("empty", b""), ("one", b"x"), ("a/65535", random.Random(7).randbytes(65535)), ("a/65536", bytes(range(256)) * 256),
            ("a/65537", (b"abcdefgh" * 9000)[:65537]), ("b/three", (b"0123456789" * 20000)[:3 * 65536 + 1]), ("n" * 65535, b"long name")]


@pytest.fixture(scope="module")
def dw(built):
    r = subprocess.run(["make", "-s", "-C", EMU, "libmz_strm_emu.so"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    import cuharness
    return DeviceWriter(cuharness.pkg().configure(C.CDLL(os.path.join(EMU, "libmz_strm_emu.so"))))


def same(dw, files, **kw):
    offsets = kw.pop("offsets", None)
    err_h, want = dw.host(files, **kw)
    err, got, rows, n, bound = dw.device(files, offsets=offsets, entries=True, **kw)
    assert (err, err_h) == (0, 0)
    assert got == want
    assert n == len(want) <= bound
    return got, rows


def check_reads(dw, archive, files, rows, password=None):
    """zipfile reads the entries back; extract_device decodes them and lists exactly the writer's table"""
    with zipfile.ZipFile(io.BytesIO(archive)) as z:
        if password is None:
            assert z.testzip() is None
            assert [(i.filename, z.read(i)) for i in z.infolist()] == [(n if isinstance(n, str) else n.decode(), d) for n, d in files]
    dx = DeviceExtractor(dw.lib)
    err, got, count, _ = dx.extract(archive, password=password)
    assert err == 0 and count == len(files)
    assert [g[1] for g in got] == [d for _, d in files]
    err_l, listed, _, _ = dx.extract(archive, password=password, list_only=True)
    assert err_l == 0
    d_arc = dw.dev(archive)
    d_ent = dw.lib.mz_cuda_malloc(max(1, len(files)) * 72)
    cnt, nb = C.c_uint32(0), C.c_uint64(0)
    pw = password.encode() if password else None
    assert dw.lib.mz_zip_cuda_extract_device(d_arc, len(archive), pw, d_ent, len(files), C.byref(cnt), None, 0, C.byref(nb), None, None) == 0
    table = dw.back(d_ent, len(files) * 72)
    dw.lib.mz_cuda_free(d_arc)
    dw.lib.mz_cuda_free(d_ent)
    assert table == b"".join(bytes(r) for r in rows)


def test_edges_byte_identical(dw):
    files = edge_corpus()
    for flags in (0, HASH_SHA256):
        got, rows = same(dw, files, flags=flags)
        check_reads(dw, got, files, rows)


@pytest.mark.parametrize("level", [0, 1, 2, 4, 6, 9])
def test_levels_byte_identical(dw, level):
    files = corpus(7, 70000, seed=40 + level)
    for flags in (0, HASH_SHA256):
        got, rows = same(dw, files, level=level, flags=flags)
    check_reads(dw, got, files, rows)


def test_offsets_sharing_and_order(dw):
    files = corpus(16, 9000, seed=50)
    # every residue mod 16, entries in reverse order of their bytes
    offs, pos = [0] * 16, 0
    for i in reversed(range(16)):
        offs[i] = pos + i
        pos += len(files[i][1]) + 32
    same(dw, files, offsets=offs, level=6, flags=HASH_SHA256)
    # items sharing bytes: every entry a slice of one buffer
    blob = corpus(1, 140000, seed=51)[0][1]
    shared = [("s%d" % i, blob[o:o + ln]) for i, (o, ln) in enumerate([(0, 140000), (3, 70000), (65536, 65536), (7, 0), (100, 40000)])]
    err_h, want = dw.host(shared)
    items = (dw.pkg.ZipDevItem * 5)()
    names = b""
    for i, (o, ln) in enumerate([(0, 140000), (3, 70000), (65536, 65536), (7, 0), (100, 40000)]):
        items[i] = dw.pkg.ZipDevItem(o, ln, len(names), len(shared[i][0]), dw.pkg.dos_date(DATE), 0, 0)
        names += shared[i][0].encode()
    err, got, _, _, _ = dw.device(shared, layout=(blob, names, bytes(items)))
    assert (err, err_h) == (0, 0) and got == want


def test_zero_entries(dw):
    got, rows = same(dw, [])
    assert got == b"PK\x05\x06" + b"\0" * 18 and rows == []


def test_rounds_cut_through_entries(dw, monkeypatch):
    files = corpus(6, 200000, seed=52)
    err, base, _, _, _ = dw.device(files, level=6, flags=HASH_SHA256)
    assert err == 0
    monkeypatch.setenv("MZ_CUDA_ZIP_ROUND_MB", "1")  # 16 chunks per round: rounds end inside entries
    err, small, _, _, _ = dw.device(files, level=6, flags=HASH_SHA256)
    assert err == 0 and small == base


@pytest.mark.parametrize("strength", [1, 2, 3])
def test_aes(dw, strength):
    files = corpus(6, 5000, seed=60 + strength)
    pw = "pw-%d" % strength
    err_h, want = dw.host(files, flags=AES | HASH_SHA256, password=pw, strength=strength)
    err, got, rows, _, _ = dw.device(files, flags=AES | HASH_SHA256, password=pw, strength=strength, entries=True)
    assert (err, err_h) == (0, 0) and len(got) == len(want)
    assert aes_ranges(got) == aes_ranges(want) and mask(got, aes_ranges(got)) == mask(want, aes_ranges(want))
    err2, again, _, _, _ = dw.device(files, flags=AES | HASH_SHA256, password=pw, strength=strength)
    assert err2 == 0 and again != got  # fresh salts
    check_reads(dw, got, files, rows, password=pw)
    dx = DeviceExtractor(dw.lib)
    assert dx.extract(got, password="wrong")[0] == MZ_PASSWORD_ERROR


def test_argument_and_item_errors(dw):
    files = corpus(4, 3000, seed=70)
    # arguments: the host writer's codes for the same input
    for kw in ({"level": 10}, {"level": -2}, {"flags": AES, "password": None}, {"flags": AES, "password": "p" * 129}, {"flags": AES, "password": "p", "strength": 4}):
        err_h = dw.host(files, **kw)[0] if kw.get("password") is not None or not (kw.get("flags", 0) & AES) else MZ_PARAM_ERROR
        assert dw.device(files, **kw)[0] == err_h == MZ_PARAM_ERROR, kw
    assert dw.device(files, flags=2)[0] == MZ_PARAM_ERROR  # MZ_ZIP_CUDA_ALL_DEVICES: the entries live on one device
    assert dw.device(files, password="ignored")[0] == 0
    # items: empty name, NUL in a name, oversized entry; the lower index decides
    data, names, items = dw.layout(files)

    def with_item(k, **f):
        arr = (dw.pkg.ZipDevItem * len(files)).from_buffer_copy(items)
        for name, v in f.items():
            setattr(arr[k], name, v)
        return data, names, bytes(arr)
    assert dw.host([("", b"x")] + files)[0] == MZ_PARAM_ERROR
    assert dw.device(files, layout=with_item(2, name_len=0))[0] == MZ_PARAM_ERROR
    assert dw.device(files, layout=with_item(1, name_len=65536))[0] == MZ_PARAM_ERROR
    nul = bytearray(names)
    nul[2] = 0
    assert dw.device(files, layout=(data, bytes(nul), items))[0] == MZ_PARAM_ERROR
    assert dw.device(files, layout=with_item(3, size=0xffff0000))[0] == MZ_SUPPORT_ERROR
    arr = (dw.pkg.ZipDevItem * len(files)).from_buffer_copy(items)
    arr[1].size, arr[3].name_len = 0xffff0000, 0
    assert dw.device(files, layout=(data, names, bytes(arr)))[0] == MZ_SUPPORT_ERROR
    arr[1].size, arr[1].name_len, arr[3].size = 5, 0, 0xffff0000
    assert dw.device(files, layout=(data, names, bytes(arr)))[0] == MZ_PARAM_ERROR
    # pointers: no names (the host writer's NULL filename), no data for a non-empty entry (its NULL data); with only empty entries
    # d_data may be NULL
    items_h = (dw.pkg.ZipItem * 2)()
    keep = C.create_string_buffer(b"abc", 3)
    items_h[0] = dw.pkg.ZipItem(b"a", C.cast(keep, C.c_void_p), 3, DATE, 0, 0)
    items_h[1] = dw.pkg.ZipItem(None, C.cast(keep, C.c_void_p), 3, DATE, 0, 0)
    sink = dw.t.sink()
    assert dw.lib.mz_zip_cuda_write_archive(sink, items_h, 2, 6, 0, None) == MZ_PARAM_ERROR
    items_h[1] = dw.pkg.ZipItem(b"b", None, 3, DATE, 0, 0)
    assert dw.lib.mz_zip_cuda_write_archive(sink, items_h, 2, 6, 0, None) == MZ_PARAM_ERROR
    dw.t.delete(sink)
    assert dw.device(files, null_names=True)[0] == MZ_PARAM_ERROR
    assert dw.device(files, null_data=True)[0] == MZ_PARAM_ERROR
    empties = [("e0", b""), ("e1", b"")]
    err, a, _, _, _ = dw.device(empties, null_data=True)
    assert err == 0 and a == dw.host(empties)[1]


def short_caps(full):
    """caps below the exact length: one byte short, half of it (chunks past it are not copied), and one ending 100 bytes into the
    largest entry's stream (the chunk across it is not copied)"""
    p, best = 0, (0, 0)
    while full[p:p + 4] == b"PK\x03\x04":
        csize, _, nl, xl = struct.unpack("<IIHH", full[p + 18:p + 30])
        best = max(best, (csize, p + 30 + nl + xl))
        p += 30 + nl + xl + csize
    return [len(full) - 1, len(full) // 2, best[1] + 100]


def test_cap_too_small(dw):
    files = corpus(5, 200000, seed=71)
    for fl, pw in ((HASH_SHA256, None), (AES, "pw")):
        err, full, _, n, bound = dw.device(files, level=6, flags=fl, password=pw)
        assert err == 0 and n == len(full) <= bound
        for cap in short_caps(full):
            err, part, _, n2, _ = dw.device(files, level=6, flags=fl, password=pw, cap=cap, sizing=False, slack=4096)
            assert (err, n2) == (MZ_BUF_ERROR, n), cap
            if cap == short_caps(full)[2]:  # the chunk across cap was not copied at all: its first 100 bytes are still the fill
                assert part[cap - 100:cap] == b"\xab" * 100
        err, again, _, _, _ = dw.device(files, level=6, flags=fl, password=pw, cap=n, sizing=False, slack=4096)
        assert err == 0 and (again == full if not pw else len(again) == len(full))


def test_two_threads(dw):
    sets = [corpus(5, 30000, seed=80), corpus(7, 20000, seed=81)]
    serial = [dw.device(f, level=6)[1] for f in sets]
    res = [None, None]

    def run(k):
        res[k] = dw.device(sets[k], level=6)[1]
    th = [threading.Thread(target=run, args=(k,)) for k in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert res == serial


def _subprocess(lib_name, body, env):
    script = ("import ctypes as C, os, sys\nsys.path.insert(0, %r)\nimport cuharness, test_emu_device_write as t\n"
              "w = t.DeviceWriter(cuharness.pkg().configure(C.CDLL(%r)))\n" % (HERE, os.path.join(EMU, lib_name))) + body
    return subprocess.run([sys.executable, "-c", script], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)


SCHED_BODY = (
    "import hashlib\n"
    "for lv, fl in ((1, 0), (6, t.HASH_SHA256), (9, 0)):\n"
    "    err, a, _, _, _ = w.device(t.edge_corpus()[:6], level=lv, flags=fl)\n"
    "    print('case', lv, fl, err, hashlib.sha256(a).hexdigest())\n")


def test_schedules_and_race_checker(dw):
    """the identity cases under three fixed thread / block schedules with the shared-memory race checker: the default schedule's bytes"""
    base = _subprocess("libmz_strm_emu.so", SCHED_BODY, dict(os.environ))
    assert base.returncode == 0, base.stdout[-3000:]
    want = [l for l in base.stdout.splitlines() if l.startswith("case")]
    assert len(want) == 3 and all(" 0 " in l for l in want)
    for seed in (3, 17, 101):
        r = _subprocess("libmz_strm_emu.so", SCHED_BODY, dict(os.environ, MZ_EMU_SCHED=str(seed), MZ_EMU_RACE="1"))
        assert r.returncode == 0, r.stdout[-3000:]
        assert [l for l in r.stdout.splitlines() if l.startswith("case")] == want, seed


def test_under_address_sanitizer(dw):
    """caps one byte short, half the archive and inside an entry's stream, each in an allocation of exactly cap bytes: nothing is written
    past it"""
    r = subprocess.run(["make", "-s", "-C", EMU, "libmz_strm_emu_san.so"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], stdout=subprocess.PIPE, text=True).stdout.strip()
    if not os.path.isabs(asan):
        pytest.skip("libasan not found")
    body = ("files = t.corpus(5, 20000, seed=72)\n"
            "for fl, pw in ((0, None), (t.HASH_SHA256, None), (t.AES, 'pw')):\n"
            "    err, full, _, n, _ = w.device(files, flags=fl, password=pw, strength=2)\n"
            "    assert err == 0\n"
            "    for cap in t.short_caps(full):\n"
            "        err, _, _, n2, _ = w.device(files, flags=fl, password=pw, strength=2, cap=cap, sizing=False)\n"
            "        print('cap', fl, err, n2 == n)\n")
    r = _subprocess("libmz_strm_emu_san.so", body, dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0"))
    assert r.returncode == 0, r.stdout[-4000:]
    assert "ERROR: AddressSanitizer" not in r.stdout and "runtime error" not in r.stdout, r.stdout[-4000:]
    assert r.stdout.count("cap ") == 9 and r.stdout.count(" -5 True") == 9, r.stdout[-2000:]


REFDIR = os.path.join(os.path.dirname(HERE), "oracle", "_ref")


@pytest.mark.parametrize("tool,flags", [("minizip_ref", 0), ("minizip_refc", HASH_SHA256), ("minizip_refe", AES | HASH_SHA256)])
def test_reference_extracts(dw, tmp_path, tool, flags):
    """the reference's own CLI extracts the device writer's archive: plain, with the hash field (built with a crypto provider, so it
    verifies the SHA-256), and WinZip AES with the password"""
    exe = os.path.join(REFDIR, tool)
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/%s not built (reference sources or OpenSSL headers absent at build time)" % tool)
    files = [(n, d) for n, d in corpus(8, 40000, seed=73) if d] + [("e/empty", b"")]
    pw = "secret" if flags & AES else None
    err, a, _, _, _ = dw.device(files, flags=flags, password=pw, strength=3)
    assert err == 0
    (tmp_path / "a.zip").write_bytes(a)
    cmd = [exe, "-x", "-o"] + (["-p", pw] if pw else []) + ["-d", "out", "a.zip"]
    r = subprocess.run(cmd, cwd=tmp_path, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=900)
    assert r.returncode == 0, (r.stdout[-600:], r.stderr[-600:])
    for name, data in files:
        assert (tmp_path / "out" / name).read_bytes() == data, name
