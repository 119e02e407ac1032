"""mz_zip_cuda_extract_device on the H100: the differential of tests/test_emu_device_extract.py against mz_zip_cuda_extract_archive
at larger sizes, a 70 000-entry native archive (zip64 end records), 10^6 empty entries (the directory parse at scale) and the
Python extract_device on a tensor."""
import hashlib
import struct
import zlib

import pytest

import datagen
from test_emu_device_extract import DeviceExtractor, adversarial_cases, differential, mutations, with_count
from test_emu_native_extract import (AES, HASH_SHA256, MZ_FORMAT_ERROR, Extractor, corpus, malformed_cases, patch_zip64_end, py_zip,
                                     reorder_directory, zip64_directory, zipfile_view)

pytestmark = pytest.mark.gpu


def empty_entries_archive(n):
    """n empty STORE entries named e/0000000.., with zip64 end records: a directory-heavy archive built directly"""
    loc, cd, off = [], [], 0
    for i in range(n):
        name = b"e/%07d" % i
        loc.append(struct.pack("<IHHHHHIIIHH", 0x04034b50, 10, 0, 0, 0, 0, 0, 0, 0, len(name), 0) + name)
        cd.append(struct.pack("<IHHHHHHIIIHHHHHII", 0x02014b50, 20, 10, 0, 0, 0, 0, 0, 0, 0, len(name), 0, 0, 0, 0, 0, off) + name)
        off += 30 + len(name)
    body, cdb = b"".join(loc), b"".join(cd)
    z64 = struct.pack("<IQHHIIQQQQ", 0x06064b50, 44, 45, 45, 0, 0, n, n, len(cdb), len(body))
    end = struct.pack("<IIQI", 0x07064b50, 0, len(body) + len(cdb), 1) + struct.pack("<IHHHHIIH", 0x06054b50, 0, 0, 0xffff, 0xffff, 0xffffffff,
                                                                                      0xffffffff, 0)
    return body + cdb + z64 + end


@pytest.fixture(scope="module")
def pair(built):
    import cuharness
    lib = cuharness.pkg().load()
    assert lib.mz_cuda_init() == 0
    return Extractor(lib), DeviceExtractor(lib)


def test_archives_and_layouts(pair):
    files = corpus(200, 200_000, seed=31)
    a = py_zip(files)
    want = zipfile_view(a)
    for arc in (a, py_zip(files, stream=True), py_zip(files[:40], force_zip64=True), pair[0].write(files), pair[0].write(files, flags=HASH_SHA256)):
        assert differential(pair, arc, want=zipfile_view(arc))[0] == 0
    for arc in (patch_zip64_end(a), zip64_directory(a), b"\0" * 1000 + a):
        assert differential(pair, arc, want=want)[0] == 0
    r = reorder_directory(a)
    assert differential(pair, r, want=zipfile_view(r))[0] == 0
    assert differential(pair, with_count(a, 1))[0] == MZ_FORMAT_ERROR
    assert differential(pair, py_zip([]))[0] == 0


@pytest.mark.parametrize("strength", [1, 2, 3])
def test_aes(pair, strength):
    files = corpus(100, 100_000, seed=32)
    a = pair[0].write(files, flags=AES | HASH_SHA256, password="secret", strength=strength)
    err, got = differential(pair, a, password="secret")
    assert err == 0 and got == [(n, d, zlib.crc32(d)) for n, d in files]
    assert differential(pair, a, password="nope")[0] == -108


def test_malformed_adversarial_and_mutated(pair):
    for name, (arc, codes) in malformed_cases(pair[0]).items():
        assert differential(pair, arc)[0] in codes, name
    for arc in adversarial_cases(pair).values():
        differential(pair, arc)
    for arc in mutations(4321, 200):
        differential(pair, arc)


def test_70000_entries_with_zip64_end_records(pair):
    texts = [datagen.text_like(3000, seed=s) for s in range(97)]
    files = [("n/%06d" % i, texts[i % 97][:1 + (i * 7919) % 3000]) for i in range(70_000)]
    a = pair[0].write(files, level=1)
    assert b"PK\x06\x06" in a[-200:]
    err, got = differential(pair, a)
    assert err == 0 and len(got) == 70_000
    assert all(g[0] == f[0] and g[1] == f[1] and g[2] == zlib.crc32(f[1]) for g, f in zip(got, files))
    pair[0].lib.mz_zip_cuda_trim()


def test_million_empty_entries(pair):
    a = empty_entries_archive(1_000_000)
    assert zipfile_view(empty_entries_archive(70_000))[-1] == ("e/0069999", b"", 0)
    err, got, n, size = pair[1].extract(a)
    assert err == 0 and n == 1_000_000 and size == 0
    assert [g[0] for g in got[:3]] == ["e/0000000", "e/0000001", "e/0000002"] and got[-1][0] == "e/0999999"
    assert all(g[1] == b"" and g[2] == 0 and g[3] == 0 for g in got)


def test_python_extract_device(pair):
    import torch
    import cuharness
    pkg = cuharness.pkg()
    files = corpus(50, 50_000, seed=33)
    a = pair[0].write(files, flags=HASH_SHA256)
    t = torch.frombuffer(bytearray(a), dtype=torch.uint8).cuda()
    entries, out = pkg.extract_device(t)
    host = out.cpu().numpy().tobytes()
    assert [(n, host[o:o + s], c) for n, o, s, c in entries] == [(n, d, zlib.crc32(d)) for n, d in files]
    assert all(o % 16 == 0 for _, o, _, _ in entries)
    with pytest.raises(RuntimeError):
        pkg.extract_device(t[:len(a) // 2])
    enc = pair[0].write(files[:5], flags=AES, password="pw", strength=3)
    te = torch.frombuffer(bytearray(enc), dtype=torch.uint8).cuda()
    entries, out = pkg.extract_device(te, password="pw")
    host = out.cpu().numpy().tobytes()
    assert hashlib.sha256(b"".join(host[o:o + s] for _, o, s, _ in entries)).digest() == hashlib.sha256(b"".join(d for _, d in files[:5])).digest()
    assert bytes(te.cpu().numpy().tobytes()) == enc  # the archive is left as it was
