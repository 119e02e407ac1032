"""mz_zip_cuda_update_device on the CPU: the real host C and kernel sources on the execution-model emulator (tests/emu/libmz_strm_emu.so).
Every device buffer is an allocation of exactly its size. Updating an archive write_device wrote must give, byte for byte, what write_device
writes for the kept entries followed by the new ones (and the same table); foreign archives must keep their entries' bytes, names, extra
fields and comment and read back everywhere; errors must write nothing; in place, a failed call must leave the source as it was."""
import ctypes as C
import io
import os
import struct
import subprocess
import sys
import zipfile

import pytest

from test_emu_native_extract import AES, EMU, HASH_SHA256, HERE, MZ_BUF_ERROR, MZ_PASSWORD_ERROR, MZ_SUPPORT_ERROR, Extractor, corpus, malformed_cases, py_zip
from test_emu_device_extract import DeviceExtractor
from test_emu_device_write import MZ_PARAM_ERROR, DeviceWriter, edge_corpus

POISON = 0xab


class DeviceUpdater(DeviceWriter):
    """ctypes driver of mz_zip_cuda_update_device (and, inherited, write_device) on one library"""

    def keep_arr(self, keep):
        return None if keep is None else struct.pack("<%dI" % len(keep), *keep)

    def update(self, src, keep=None, files=(), level=6, flags=0, password=None, strength=0, cap=None, entries=False, sizing=True, slack=0,
               layout=None):
        """mz_zip_cuda_update_device of the archive bytes `src` -> (err, archive bytes, [rows], length, bound). The output buffer is
        poisoned (0xab) and has `slack` more poisoned bytes behind cap, which must be left as they are; the source and inputs are read back
        unchanged. On an error other than MZ_BUF_ERROR nothing may have been written."""
        L = self.lib
        files = list(files)
        data, names, items = layout or self.layout(files)
        d_src, d_data, d_names, d_items = self.dev(src), self.dev(data), self.dev(names), self.dev(items)
        kb = self.keep_arr(keep)
        d_keep = self.dev(kb) if kb else None
        nk = len(keep) if keep is not None else 0
        if keep is not None and not kb:  # an empty keep list: a valid pointer, no indices
            d_keep = L.mz_cuda_malloc(1)
        pw = password.encode() if password is not None else None
        n = C.c_uint64(0)
        bound = None
        args = (d_src, len(src), d_keep, nk, d_data, d_names, d_items, len(files), level, flags, pw, strength)
        try:
            if sizing:
                err = L.mz_zip_cuda_update_device(*args, None, 0, C.byref(n), None, None, None)
                if err:
                    return err, b"", [], 0, None
                bound = n.value
            size = bound if cap is None else cap
            d_arc = L.mz_cuda_malloc(max(1, size + slack))
            assert L.mz_cuda_memset(d_arc, POISON, max(1, size + slack), None) == 0
            nrows = (len(keep) if keep is not None else 1 << 16) + len(files)
            d_ent = None
            if entries:
                d_ent = L.mz_cuda_malloc(max(1, nrows) * 72)
            st = self.pkg.ZipStats()
            err = L.mz_zip_cuda_update_device(*args, d_arc, size, C.byref(n), d_ent, C.byref(st), None)
            whole = self.back(d_arc, size + slack)
            if slack:
                assert whole[size:] == bytes([POISON]) * slack, "written at or beyond cap"
            if err not in (0, MZ_BUF_ERROR):
                assert whole == bytes([POISON]) * (size + slack), "written on error %d" % err
            out = whole[:min(n.value, size)] if err in (0, MZ_BUF_ERROR) else b""
            rows = []
            if entries and err == 0:
                k = st.entries
                raw = self.back(d_ent, k * 72)
                rows = list((self.pkg.ZipDevEntry * max(1, k)).from_buffer_copy(raw.ljust(72, b"\0")))[:k]
            L.mz_cuda_free(d_arc)
            if d_ent:
                L.mz_cuda_free(d_ent)
            assert self.back(d_src, len(src)) == src
            assert self.back(d_data, len(data)) == data and self.back(d_names, len(names)) == names and self.back(d_items, len(items)) == items
            return err, out, rows, n.value, bound
        finally:
            for p in (d_src, d_data, d_names, d_items, d_keep):
                if p:
                    L.mz_cuda_free(p)

    def in_place(self, src, files=(), level=6, flags=0, cap=None, keep=None, arc_off=0, arc_cap=None):
        """update_device with d_archive == d_src (or, with arc_off, a buffer overlapping it): the source in an allocation of cap bytes
        (default: the sizing bound) -> (err, buffer bytes [0, cap), length)"""
        L = self.lib
        files = list(files)
        data, names, items = self.layout(files)
        d_data, d_names, d_items = self.dev(data), self.dev(names), self.dev(items)
        kb = self.keep_arr(keep)
        d_keep = self.dev(kb) if kb else None
        n = C.c_uint64(0)
        if cap is None:
            d_src = self.dev(src)
            assert L.mz_zip_cuda_update_device(d_src, len(src), None, 0, d_data, d_names, d_items, len(files), level, flags, None, 0, None, 0,
                                               C.byref(n), None, None, None) == 0
            L.mz_cuda_free(d_src)
            cap = max(n.value, len(src))
        buf = L.mz_cuda_malloc(cap)
        assert L.mz_cuda_memset(buf, POISON, cap, None) == 0
        assert L.mz_cuda_memcpy_h2d(buf, src, len(src), None) == 0
        try:
            err = L.mz_zip_cuda_update_device(buf, len(src), d_keep, len(keep) if keep else 0, d_data, d_names, d_items, len(files), level, flags,
                                              None, 0, buf + arc_off, (arc_cap if arc_cap is not None else cap - arc_off), C.byref(n), None, None, None)
            return err, self.back(buf, cap), n.value
        finally:
            L.mz_cuda_free(buf)
            for p in (d_data, d_names, d_items, d_keep):
                if p:
                    L.mz_cuda_free(p)


@pytest.fixture(scope="module")
def du(built):
    r = subprocess.run(["make", "-s", "-C", EMU, "libmz_strm_emu.so"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    import cuharness
    return DeviceUpdater(cuharness.pkg().configure(C.CDLL(os.path.join(EMU, "libmz_strm_emu.so"))))


def written(du, files, **kw):
    err, a, rows, n, _ = du.device(files, entries=True, **kw)
    assert err == 0
    return a, rows


def identical(du, A, S, B, **kw):
    """update(write_device(A), keep=S, files=B) == write_device(A[S] + B), archive and rows"""
    src, _ = written(du, A, **kw)
    kept = A if S is None else [A[i] for i in S]
    want, want_rows = written(du, kept + list(B), **kw)
    err, got, rows, n, bound = du.update(src, keep=S, files=B, entries=True, **kw)
    assert err == 0
    assert got == want
    assert n == len(want) <= bound
    assert [bytes(r) for r in rows] == [bytes(r) for r in want_rows]
    return got


def keep_sets(n):
    return [None, [], list(reversed(range(n))), [0, 0, n - 1, 1, n - 1], [n // 2]]


@pytest.mark.parametrize("level", [1, 6, 9])
@pytest.mark.parametrize("flags", [0, HASH_SHA256])
def test_identity_with_write_device(du, level, flags):
    A = corpus(6, 20000, seed=300 + level)
    B = corpus(3, 9000, seed=310 + level)
    B = [("new/" + n, d) for n, d in B]
    for S in keep_sets(len(A)):
        identical(du, A, S, B, level=level, flags=flags)
    identical(du, A, [2, 0], [], level=level, flags=flags)  # no new entries


def test_identity_edges(du):
    A = edge_corpus()
    identical(du, A, None, [("x", b"appended")])
    identical(du, A, [6, 0, 5], [])
    identical(du, [], None, [("only", b"one")])  # a source with zero entries
    identical(du, [], [], [])
    identical(du, A[:3], [], [])  # nothing kept, nothing new: an empty archive


def test_in_place_append(du):
    A = corpus(5, 30000, seed=320)
    B = [("in/" + n, d) for n, d in corpus(3, 7000, seed=321)]
    src, _ = written(du, A)
    err, want, _, n, _ = du.update(src, files=B)
    assert err == 0
    cd_off = struct.unpack("<I", src[-6:-2])[0]
    cap = n + 100
    err, buf, n2 = du.in_place(src, files=B, cap=cap)
    assert (err, n2) == (0, n)
    assert buf[:n] == want and buf[:cd_off] == src[:cd_off] and buf[n:] == bytes([POISON]) * 100
    # one byte short: MZ_BUF_ERROR with the exact length, and the source restored
    err, buf, n3 = du.in_place(src, files=B, cap=n - 1)
    assert (err, n3) == (MZ_BUF_ERROR, n)
    assert buf[:len(src)] == src
    with zipfile.ZipFile(io.BytesIO(buf[:len(src)])) as z:
        assert z.testzip() is None


def test_in_place_refused(du):
    A = corpus(4, 5000, seed=330)
    src, _ = written(du, A)
    # a keep list
    err, buf, _ = du.in_place(src, files=[("n", b"x")], keep=[0, 1, 2, 3], cap=len(src) + 4096)
    assert err == MZ_PARAM_ERROR and buf[:len(src)] == src
    # a prepended stub: the entries do not start at 0
    stub = b"#!stub\n" * 5
    bio = io.BytesIO()
    bio.write(stub)
    with zipfile.ZipFile(bio, "a") as z:
        for n, d in A:
            z.writestr(n, d)
    stubbed = bio.getvalue()
    err, buf, _ = du.in_place(stubbed, files=[("n", b"x")], cap=len(stubbed) + 4096)
    assert err == MZ_PARAM_ERROR and buf[:len(stubbed)] == stubbed
    # a gap between two entries
    gap = with_gap(src)
    err, buf, _ = du.in_place(gap, files=[("n", b"x")], cap=len(gap) + 4096)
    assert err == MZ_PARAM_ERROR and buf[:len(gap)] == gap
    # partly overlapping buffers
    for off in (1, 16, len(src) // 2):
        err, buf, _ = du.in_place(src, files=[("n", b"x")], cap=len(src) * 3, arc_off=off, arc_cap=len(src) * 2)
        assert err == MZ_PARAM_ERROR and buf[:len(src)] == src


def with_gap(a):
    """a with 37 zero bytes inserted behind the first entry (offsets of the later entries and the directory moved)"""
    with zipfile.ZipFile(io.BytesIO(a)) as z:
        infos = z.infolist()
    cut = infos[1].header_offset
    out = bytearray(a[:cut] + b"\0" * 37 + a[cut:])
    e = len(out) - 22
    cd_off, = struct.unpack("<I", out[e + 16:e + 20])
    cd_off += 37
    out[e + 16:e + 20] = struct.pack("<I", cd_off)
    p = cd_off
    while out[p:p + 4] == b"PK\x01\x02":
        nl, xl, cl = struct.unpack("<HHH", out[p + 28:p + 34])
        off, = struct.unpack("<I", out[p + 42:p + 46])
        if off >= cut:
            out[p + 42:p + 46] = struct.pack("<I", off + 37)
        p += 46 + nl + xl + cl
    return bytes(out)


def foreign_sources():
    files = corpus(6, 12000, seed=340)
    out = {}
    out["deflate"] = py_zip(files)
    out["store"] = py_zip(files, compression=zipfile.ZIP_STORED)
    out["descriptors"] = py_zip(files, stream=True)
    out["forced_zip64"] = py_zip(files, force_zip64=True)
    bio = io.BytesIO()
    with zipfile.ZipFile(bio, "w", zipfile.ZIP_DEFLATED) as z:
        z.comment = b"an archive comment"
        for i, (n, d) in enumerate(files):
            zi = zipfile.ZipInfo(n, date_time=(2020, 1, 2, 3, 4, 6))
            zi.compress_type = zipfile.ZIP_DEFLATED
            zi.extra = struct.pack("<HH", 0xcafe, 5) + bytes([i, 1, 2, 3, 4]) + struct.pack("<HHBI", 0x5455, 5, 1, 1600000000)
            zi.comment = b"file comment %d" % i
            z.writestr(zi, d)
    out["comment_and_extras"] = bio.getvalue()
    bio = io.BytesIO()
    bio.write(b"MZ-stub" * 9)
    with zipfile.ZipFile(bio, "a", zipfile.ZIP_DEFLATED) as z:
        for n, d in files:
            z.writestr(n, d)
    out["prepended_stub"] = bio.getvalue()
    return files, out


def extras_of(a):
    """[(name, [non-zip64 extra fields as (id, bytes)], file comment)] of the directory, and the archive comment"""
    with zipfile.ZipFile(io.BytesIO(a)) as z:
        infos = z.infolist()
        comment = z.comment
    res = []
    for i in infos:
        x, fields = i.extra, []
        p = 0
        while p + 4 <= len(x):
            fid, fs = struct.unpack("<HH", x[p:p + 4])
            if fid != 1:
                fields.append((fid, x[p:p + 4 + fs]))
            p += 4 + fs
        res.append((i.filename, fields, i.comment))
    return res, comment


def ref_extracts(tmp_path, a, files, password=None):
    exe = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "minizip_ref" if password is None else "minizip_refe")
    if not os.path.exists(exe):
        return False
    d = tmp_path / ("x%d" % len(os.listdir(tmp_path)))
    d.mkdir()
    (d / "a.zip").write_bytes(a)
    cmd = [exe, "-x", "-o"] + (["-p", password] if password else []) + ["-d", "out", "a.zip"]
    r = subprocess.run(cmd, cwd=d, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=900)
    assert r.returncode == 0, (r.stdout[-600:], r.stderr[-600:])
    for name, data in files:
        assert (d / "out" / name).read_bytes() == data, name
    return True


@pytest.mark.parametrize("kind", ["deflate", "store", "descriptors", "forced_zip64", "comment_and_extras", "prepended_stub"])
def test_foreign_sources(du, tmp_path, kind):
    files, srcs = foreign_sources()
    src = srcs[kind]
    B = [("new/a.txt", b"appended " * 500), ("new/b.bin", bytes(range(256)) * 40)]
    n = len(files)
    src_meta, src_comment = extras_of(src)
    for S in (None, [n - 1, 0, 2, 2]):
        err, out, rows, _, _ = du.update(src, keep=S, files=B, entries=True)
        assert err == 0, (kind, err)
        kept = files if S is None else [files[i] for i in S]
        want = kept + B
        with zipfile.ZipFile(io.BytesIO(out)) as z:
            assert z.testzip() is None
            assert [(i.filename, z.read(i)) for i in z.infolist()] == want
            assert z.comment == src_comment
        meta, _ = extras_of(out)
        idx = list(range(n)) if S is None else S
        assert meta[:len(idx)] == [src_meta[i] for i in idx]
        dx = DeviceExtractor(du.lib)
        err, got, count, _ = dx.extract(out)
        assert err == 0 and count == len(want)
        assert [(g[0], g[1], g[3]) for g in got] == [(nm, d, 0) for nm, d in want]
        _, src_got, _, _ = dx.extract(src)
        assert [g[2] for g in got[:len(idx)]] == [src_got[i][2] for i in idx]  # CRCs carried over
        err_l, listed, _, _ = dx.extract(out, list_only=True)
        assert err_l == 0
        ref_extracts(tmp_path, out, want)  # a repeated entry extracts to the same file twice, with the same bytes


def test_reference_written_source(du, tmp_path):
    """an archive the reference CLI wrote (where oracle/_ref was built) is updated and still extracts with it"""
    exe = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "minizip_ref")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/minizip_ref not built")
    files = [(n.split("/")[-1], d) for n, d in corpus(5, 20000, seed=350) if d]  # the CLI stores the names without directories
    for n, d in files:
        p = tmp_path / "in" / n
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_bytes(d)
    r = subprocess.run([exe, "-o", "-9", os.path.join(str(tmp_path), "src.zip")] + [n for n, _ in files], cwd=tmp_path / "in",
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=900)
    assert r.returncode == 0, r.stderr[-600:]
    src = (tmp_path / "src.zip").read_bytes()
    with zipfile.ZipFile(io.BytesIO(src)) as z:
        order = [i.filename for i in z.infolist()]
    byname = dict(files)
    err, out, _, _, _ = du.update(src, keep=[1, 0], files=[("added", b"more " * 999)])
    assert err == 0
    want = [(order[1], byname[order[1]]), (order[0], byname[order[0]]), ("added", b"more " * 999)]
    with zipfile.ZipFile(io.BytesIO(out)) as z:
        assert z.testzip() is None and [(i.filename, z.read(i)) for i in z.infolist()] == want
    assert ref_extracts(tmp_path, out, want)


def test_aes_kept_without_password(du, tmp_path):
    A = corpus(4, 6000, seed=360)
    err, src, _, _, _ = du.device(A, flags=AES | HASH_SHA256, password="old", strength=3)
    assert err == 0
    B = [("plain/new", b"no password " * 100)]
    err, out, rows, _, _ = du.update(src, keep=[3, 1], files=B, entries=True)
    assert err == 0
    dx = DeviceExtractor(du.lib)
    # the kept entries still need (and open with) the old password; the new plain one needs none
    err, got, count, _ = dx.extract(out, password="old")
    assert err == 0 and [g[1] for g in got] == [A[3][1], A[1][1], B[0][1]]
    # new AES entries under the same password
    B2 = [("enc/new", b"secret " * 700)]
    err, out2, _, _, _ = du.update(src, files=B2, flags=AES, password="old", strength=2)
    assert err == 0
    err, got, _, _ = dx.extract(out2, password="old")
    assert err == 0 and [g[1] for g in got] == [d for _, d in A] + [B2[0][1]]
    assert dx.extract(out2, password="wrong")[0] == MZ_PASSWORD_ERROR
    ref_extracts(tmp_path, out2, A + B2, password="old")


def test_errors_write_nothing(du):
    dx = DeviceExtractor(du.lib)
    for name, (arc, _) in malformed_cases(Extractor(du.lib)).items():
        want = dx.extract(arc, password="pw", list_only=True)[0]
        err, _, _, _, _ = du.update(arc, files=[("n", b"x")], sizing=False, cap=4096)
        if want in (0, MZ_BUF_ERROR):
            continue  # the archive lists: its damage is in the entries' bytes, which update copies as they are
        assert err == want, (name, err, want)
    A = corpus(4, 3000, seed=370)
    src, _ = written(du, A)
    # a refused record: PKWARE encryption bit set on the second record
    b = bytearray(src)
    cd_off = struct.unpack("<I", src[-6:-2])[0]
    p, k = cd_off, 0
    while b[p:p + 4] == b"PK\x01\x02":
        nl, xl, cl = struct.unpack("<HHH", b[p + 28:p + 34])
        if k == 1:
            b[p + 8] |= 1
        p += 46 + nl + xl + cl
        k += 1
    err, _, _, _, _ = du.update(bytes(b), files=[("n", b"x")], sizing=False, cap=1 << 16)
    assert err == MZ_SUPPORT_ERROR
    # a keep index out of range
    for keep in ([4], [0, 1, 99], [0xffffffff]):
        err, _, _, _, _ = du.update(src, keep=keep, sizing=False, cap=1 << 16)
        assert err == MZ_PARAM_ERROR, keep
    # arguments and items, as write_device reports them (and in front of nothing else)
    assert du.update(src, files=A, level=10)[0] == MZ_PARAM_ERROR
    assert du.update(src, files=A, flags=2)[0] == MZ_PARAM_ERROR
    assert du.update(src, files=A, flags=AES, password=None)[0] == MZ_PARAM_ERROR
    data, names, items = du.layout(A)
    arr = (du.pkg.ZipDevItem * len(A)).from_buffer_copy(items)
    arr[2].name_len = 0
    assert du.update(src, files=A, layout=(data, names, bytes(arr)), sizing=False, cap=1 << 16)[0] == MZ_PARAM_ERROR
    arr[2].name_len, arr[1].size = 3, 0xffff0000
    assert du.update(src, files=A, layout=(data, names, bytes(arr)), sizing=False, cap=1 << 16)[0] == MZ_SUPPORT_ERROR
    # the source's error comes before the keep index, the keep index before the items
    assert du.update(src[:len(src) // 2], keep=[99], files=A, layout=(data, names, bytes(arr)), sizing=False, cap=1 << 16)[0] == -103
    assert du.update(src, keep=[99], files=A, layout=(data, names, bytes(arr)), sizing=False, cap=1 << 16)[0] == MZ_PARAM_ERROR


def with_zip64_fields(a):
    """a (an archive write_device wrote, no zip64 end records) with a zip64 field (the plain size, 8 bytes) in front of every directory
    record's other extra fields, and version needed 45 where it was lower: the fields K10 reads past (the fixed sizes are not
    saturated) and an update drops"""
    e = len(a) - 22
    cd_off, = struct.unpack("<I", a[e + 16:e + 20])
    recs, p = b"", cd_off
    while a[p:p + 4] == b"PK\x01\x02":
        h = bytearray(a[p:p + 46])
        nl, xl, cl = struct.unpack("<HHH", h[28:34])
        usize, = struct.unpack("<I", h[24:28])
        ver, = struct.unpack("<H", h[6:8])
        h[6:8] = struct.pack("<H", max(ver, 45))
        h[30:32] = struct.pack("<H", xl + 12)
        recs += bytes(h) + a[p + 46:p + 46 + nl] + struct.pack("<HHQ", 1, 8, usize) + a[p + 46 + nl:p + 46 + nl + xl + cl]
        p += 46 + nl + xl + cl
    end = bytearray(a[e:])
    end[12:16] = struct.pack("<I", len(recs))
    return a[:cd_off] + recs + bytes(end)


def test_source_zip64_fields_dropped(du):
    """records with a zip64 field in front of the hash (and AES) fields: the field is dropped, version needed goes back to 20 (non-AES),
    the digest moves with its field, and the records come out as write_device writes them"""
    A = corpus(6, 9000, seed=395)
    B = [("new/z", b"zip64 " * 900)]
    src, _ = written(du, A, flags=HASH_SHA256)
    patched = with_zip64_fields(src)
    with zipfile.ZipFile(io.BytesIO(patched)) as z:
        assert z.testzip() is None and all(i.extra[:4] == b"\x01\x00\x08\x00" for i in z.infolist())
    for S in (None, [5, 0, 0, 3]):
        kept = A if S is None else [A[i] for i in S]
        want, want_rows = written(du, kept + B, flags=HASH_SHA256)
        err, got, rows, _, _ = du.update(patched, keep=S, files=B, flags=HASH_SHA256, entries=True)
        assert err == 0 and got == want
        assert [bytes(r) for r in rows] == [bytes(r) for r in want_rows]  # sha_off included
    # WinZip AES records (version 51, the 0x9901 and hash fields behind the zip64 field): the same output as from the unpatched source
    err, aes_src, _, _, _ = du.device(A, flags=AES | HASH_SHA256, password="pw", strength=1)
    assert err == 0
    for S in (None, [2, 1]):
        a1 = du.update(aes_src, keep=S, files=B, entries=True)
        a2 = du.update(with_zip64_fields(aes_src), keep=S, files=B, entries=True)
        assert a1[0] == a2[0] == 0 and a1[1] == a2[1] and [bytes(r) for r in a1[2]] == [bytes(r) for r in a2[2]]
    dx = DeviceExtractor(du.lib)
    err, got, _, _ = dx.extract(a2[1], password="pw")
    assert err == 0 and [g[1] for g in got] == [A[2][1], A[1][1], B[0][1]]


def test_longest_archive_comment(du):
    """a 65535-byte archive comment is carried over whole, out of place and in place"""
    files = corpus(4, 7000, seed=396)
    bio = io.BytesIO()
    with zipfile.ZipFile(bio, "w", zipfile.ZIP_DEFLATED) as z:
        z.comment = bytes((i * 7 + 3) % 251 + 1 for i in range(65535))
        for n, d in files:
            z.writestr(n, d)
    src = bio.getvalue()
    B = [("new/c", b"comment " * 100)]
    err, out, _, _, _ = du.update(src, keep=[3, 1], files=B)
    assert err == 0
    with zipfile.ZipFile(io.BytesIO(out)) as z:
        assert z.testzip() is None and z.comment == bytes((i * 7 + 3) % 251 + 1 for i in range(65535))
        assert [(i.filename, z.read(i)) for i in z.infolist()] == [files[3], files[1]] + B
    err, buf, n = du.in_place(src, files=B)
    assert err == 0
    with zipfile.ZipFile(io.BytesIO(buf[:n])) as z:
        assert z.testzip() is None and z.comment == bytes((i * 7 + 3) % 251 + 1 for i in range(65535))
        assert [(i.filename, z.read(i)) for i in z.infolist()] == files + B


class ZipUp(C.Structure):
    """mz_cuda_zip_up (include/mz_cuda_batch.h): the call state of the K13 launchers"""
    _fields_ = [("src", C.c_void_p), ("ent", C.c_void_p), ("count", C.c_uint32), ("n", C.c_uint32), ("keep", C.c_void_p), ("dir", C.c_void_p),
                ("dir_off", C.c_uint64), ("src_len", C.c_uint64), ("cnt", C.c_void_p), ("pre", C.c_void_p), ("part", C.c_void_p), ("info", C.c_void_p),
                ("archive", C.c_void_p), ("cap", C.c_uint64), ("cd_off", C.c_uint64), ("entries", C.c_void_p)]


COPY_LENGTHS = (0, 1, 5, 15, 16, 17, 31, 32, 33, 100, 16 * 31 + 3, 16 * 32, 16 * 33 + 9, 2000)


def copy_pairs(lib, lengths=COPY_LENGTHS, seed=7):
    """K13's copy kernel (mz_cuda_zip_up_copy) on every pair (source address mod 16, destination address mod 16) and each length:
    extents of random bytes, the destination poisoned with 16 poisoned bytes between slots. With cap = all, every slot's bytes arrive
    and nothing else changes; with cap inside a slot, nothing at or past cap is written. Returns the number of slots checked."""
    import random
    import cuharness
    pkg = cuharness.pkg()
    slots = [(s, d, ln) for s in range(16) for d in range(16) for ln in lengths]
    size = sum(ln + 32 for _, _, ln in slots) + 128
    src, dst = lib.mz_cuda_malloc(size), lib.mz_cuda_malloc(size)
    assert src and dst
    rng = random.Random(seed)
    data = rng.randbytes(size)
    lay, ps, pd = [], 64, 64
    for s, d, ln in slots:
        ps += (s - (src + ps)) % 16
        pd += (d - (dst + pd)) % 16
        lay.append((ps, pd, ln))
        ps += ln + 16
        pd += ln + 16
    n = len(slots)
    ents = (pkg.ZipDevEntry * n)()
    pre = (C.c_uint64 * (5 * (n + 1)))()
    for i, (o_s, o_d, ln) in enumerate(lay):
        ents[i].local_off, ents[i].extent = o_s, ln
        pre[5 * i] = o_d
    d_ent, d_pre = lib.mz_cuda_malloc(C.sizeof(ents)), lib.mz_cuda_malloc(C.sizeof(pre))
    try:
        assert lib.mz_cuda_memcpy_h2d(src, data, size, None) == 0
        assert lib.mz_cuda_memcpy_h2d(d_ent, C.cast(ents, C.c_void_p), C.sizeof(ents), None) == 0
        assert lib.mz_cuda_memcpy_h2d(d_pre, C.cast(pre, C.c_void_p), C.sizeof(pre), None) == 0
        mid = lay[n // 2][1] + 7
        for cap in (size, mid):
            assert lib.mz_cuda_memset(dst, POISON, size, None) == 0
            u = ZipUp(src=src, ent=d_ent, count=n, n=n, src_len=size, pre=d_pre, archive=dst, cap=cap)
            assert lib.mz_cuda_zip_up_copy(C.byref(u), None) == 0
            assert lib.mz_cuda_stream_sync(None) == 0
            out = C.create_string_buffer(size)
            assert lib.mz_cuda_memcpy_d2h(out, dst, size, None) == 0
            want = bytearray([POISON]) * size
            for o_s, o_d, ln in lay:
                want[o_d:o_d + ln] = data[o_s:o_s + ln]
            want[cap:] = bytes([POISON]) * (size - cap)
            got = out.raw
            if got != bytes(want):
                k = next(k for k in range(size) if got[k] != want[k])
                slot = max(i for i, (_, o_d, _) in enumerate(lay) if o_d <= k)
                raise AssertionError("cap %d: first wrong byte %d in slot %s" % (cap, k, slots[slot]))
        return n
    finally:
        for p in (src, dst, d_ent, d_pre):
            lib.mz_cuda_free(p)


def test_copy_kernel_every_alignment_pair(du):
    assert copy_pairs(du.lib) == 16 * 16 * len(COPY_LENGTHS)


def test_cap_too_small(du):
    A = corpus(5, 40000, seed=380)
    src, _ = written(du, A, flags=HASH_SHA256)
    B = corpus(3, 30000, seed=381)
    B = [("b/" + n, d) for n, d in B]
    err, full, _, n, _ = du.update(src, keep=[4, 0, 1], files=B, flags=HASH_SHA256)
    assert err == 0
    for cap in (n - 1, n // 2, 100):
        err, part, _, n2, _ = du.update(src, keep=[4, 0, 1], files=B, flags=HASH_SHA256, cap=cap, sizing=False, slack=4096)
        assert (err, n2) == (MZ_BUF_ERROR, n), cap


def _subprocess(lib_name, body, env):
    script = ("import ctypes as C, os, sys\nsys.path.insert(0, %r)\nimport cuharness, test_emu_device_update as t\n"
              "u = t.DeviceUpdater(cuharness.pkg().configure(C.CDLL(%r)))\n" % (HERE, os.path.join(EMU, lib_name))) + body
    return subprocess.run([sys.executable, "-c", script], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)


SCHED_BODY = (
    "import hashlib\n"
    "A = t.edge_corpus()[:5]\n"
    "src = u.device(A, level=6)[1]\n"
    "for lv, fl, keep in ((1, 0, None), (6, t.HASH_SHA256, [4, 0, 0]), (9, 0, [])):\n"
    "    err, a, _, _, _ = u.update(src, keep=keep, files=[('n/1', b'new' * 3000), ('n/2', b'')], level=lv, flags=fl)\n"
    "    print('case', lv, fl, err, hashlib.sha256(a).hexdigest())\n")


def test_schedules_and_race_checker(du):
    """the identity cases under three fixed thread / block schedules with the shared-memory race checker: the default schedule's bytes"""
    base = _subprocess("libmz_strm_emu.so", SCHED_BODY, dict(os.environ))
    assert base.returncode == 0, base.stdout[-3000:]
    want = [l for l in base.stdout.splitlines() if l.startswith("case")]
    assert len(want) == 3 and all(" 0 " in l for l in want)
    for seed in (3, 17, 101):
        r = _subprocess("libmz_strm_emu.so", SCHED_BODY, dict(os.environ, MZ_EMU_SCHED=str(seed), MZ_EMU_RACE="1"))
        assert r.returncode == 0, r.stdout[-3000:]
        assert [l for l in r.stdout.splitlines() if l.startswith("case")] == want, seed


def test_under_address_sanitizer(du):
    """caps one byte short and half the archive, each in an allocation of exactly cap bytes: nothing is written past it; a full run reads
    nothing outside the source"""
    r = subprocess.run(["make", "-s", "-C", EMU, "libmz_strm_emu_san.so"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], stdout=subprocess.PIPE, text=True).stdout.strip()
    if not os.path.isabs(asan):
        pytest.skip("libasan not found")
    body = ("A = t.corpus(5, 20000, seed=390)\n"
            "src = u.device(A, flags=t.HASH_SHA256)[1]\n"
            "B = [('b/x', b'xyz' * 5000)]\n"
            "for keep in (None, [3, 0, 4]):\n"
            "    err, full, _, n, _ = u.update(src, keep=keep, files=B)\n"
            "    assert err == 0\n"
            "    for cap in (n - 1, n // 2):\n"
            "        err, _, _, n2, _ = u.update(src, keep=keep, files=B, cap=cap, sizing=False)\n"
            "        print('cap', err, n2 == n)\n")
    r = _subprocess("libmz_strm_emu_san.so", body, dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0"))
    assert r.returncode == 0, r.stdout[-4000:]
    assert "ERROR: AddressSanitizer" not in r.stdout and "runtime error" not in r.stdout, r.stdout[-4000:]
    assert r.stdout.count("cap ") == 4 and r.stdout.count(" -5 True") == 4, r.stdout[-2000:]
