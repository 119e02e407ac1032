"""The device reader (mz_zip_cuda_reader_*) on the H100: the differential of tests/test_emu_device_reader.py against
mz_zip_cuda_extract_device at larger sizes, a 70 000-entry archive with random selections and locate of every name, locate over the
10^6-empty-entry archive, and the Python ZipDeviceReader."""
import hashlib
import random

import pytest

import datagen
from test_emu_device_reader import MISS, Case, Ctx, identity, merge_archives
from test_emu_native_extract import AES, HASH_SHA256, corpus, py_zip
from test_gpu_device_extract import empty_entries_archive

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(built):
    import cuharness
    lib = cuharness.pkg().load()
    assert lib.mz_cuda_init() == 0
    return Ctx(lib)


def test_archives_and_aes(ctx):
    files = corpus(200, 200_000, seed=41)
    for arc in (py_zip(files), ctx.ex.write(files), ctx.ex.write(files, flags=HASH_SHA256)):
        assert identity(ctx, arc, seed=1, selections=6) == 0
    enc = corpus(60, 100_000, seed=42)
    parts = [ctx.ex.write([("s%d/%s" % (s, n), d) for n, d in enc], flags=AES | HASH_SHA256, password="secret", strength=s) for s in (1, 2, 3)]
    mixed = merge_archives(parts)
    assert identity(ctx, mixed, password="secret", seed=2, selections=6) == 0
    assert identity(ctx, mixed, password="nope", seed=3, selections=2) == -108


def test_70000_entries(ctx):
    texts = [datagen.text_like(3000, seed=s) for s in range(97)]
    files = [("n/%06d" % i, texts[i % 97][:1 + (i * 7919) % 3000]) for i in range(70_000)]
    a = ctx.ex.write(files, level=1)
    c = Case(ctx, a)
    try:
        assert c.check_open() and c.count == 70_000
        rng = random.Random(9)
        for _ in range(20):
            c.check_selection([rng.randrange(70_000) for _ in range(rng.randint(1, 5000))])
        names = [n.encode() for n, _ in files]
        misses = [b"n/%06d" % (70_000 + i) for i in range(70_000)]
        got = ctx.rd.locate(c.h, names + misses, 0)
        first = {}
        for i, n in enumerate(names):
            first.setdefault(n, i)
        assert got == [first[n] for n in names] + [MISS] * 70_000
        assert ctx.rd.locate(c.h, [n.upper() for n in names[:1000]], 1) == list(range(1000))
    finally:
        c.close()
    ctx.lib.mz_zip_cuda_trim()


def test_million_empty_entries(ctx):
    a = empty_entries_archive(1_000_000)
    d_arc = ctx.rd.put(a)
    err, h, n, refuse = ctx.rd.open(d_arc, len(a))
    try:
        assert (err, n, refuse) == (0, 1_000_000, 0)
        names = [b"e/%07d" % i for i in range(1_000_000)]
        assert ctx.rd.locate(h, names, 0) == list(range(1_000_000))
        assert ctx.rd.locate(h, [b"E/0000007", b"e\\0999999", b"e/1000000"], 1) == [7, 999_999, MISS]
        err, size, _, offs, sts = ctx.rd.decode(h, [5, 999_999, 1_000_000])
        assert (err, size, offs, sts) == (-100, 0, [0, 0, 0, 0], [0, 0, -100])
    finally:
        ctx.lib.mz_zip_cuda_reader_close(h)
        ctx.lib.mz_cuda_free(d_arc)


def test_python_reader(ctx):
    import torch
    import cuharness
    pkg = cuharness.pkg()
    files = corpus(50, 50_000, seed=43)
    a = ctx.ex.write(files, flags=HASH_SHA256)
    t = torch.frombuffer(bytearray(a), dtype=torch.uint8).cuda()
    with pkg.ZipDeviceReader(t) as r:
        assert r.entries == [(n, len(d), __import__("zlib").crc32(d)) for n, d in files] and r.refuse == 0
        for sel in ([3, 3, 0, 49], torch.tensor([7, 1], device="cuda"), torch.tensor([], dtype=torch.int64), list(range(50))):
            offs, out = r.read(sel)
            idx = [int(x) for x in (sel.tolist() if torch.is_tensor(sel) else sel)]
            host, o = out.cpu().numpy().tobytes(), offs.cpu().tolist()
            assert offs.is_cuda and out.is_cuda and len(o) == len(idx) + 1 and all(x % 16 == 0 for x in o)
            assert [host[o[k]:o[k] + len(files[i][1])] for k, i in enumerate(idx)] == [files[i][1] for i in idx]
        found = r.locate([files[9][0], files[9][0].upper(), "missing", ""], ignore_case=True)
        assert found.is_cuda and found.dtype == torch.int64 and found.tolist() == [9, 9, -1, -1]
        with pytest.raises(RuntimeError):
            r.read(found)  # a miss: MZ_END_OF_LIST
        offs, out = r.read(found[:2])
        assert out.cpu().numpy().tobytes()[:len(files[9][1])] == files[9][1]
    with pytest.raises(RuntimeError):
        r.read([0])  # closed
    with pytest.raises(RuntimeError):
        pkg.ZipDeviceReader(t[:len(a) // 2])
    enc = ctx.ex.write(files[:5], flags=AES, password="pw", strength=3)
    te = torch.frombuffer(bytearray(enc), dtype=torch.uint8).cuda()
    with pkg.ZipDeviceReader(te, password="pw") as r:
        offs, out = r.read([4, 0, 4])
        host, o = out.cpu().numpy().tobytes(), offs.cpu().tolist()
        got = b"".join(host[o[k]:o[k] + len(files[i][1])] for k, i in enumerate([4, 0, 4]))
        assert hashlib.sha256(got).digest() == hashlib.sha256(files[4][1] + files[0][1] + files[4][1]).digest()
    with pkg.ZipDeviceReader(te, password="wrong") as r:
        with pytest.raises(RuntimeError):
            r.read([0])
    assert bytes(te.cpu().numpy().tobytes()) == enc  # the archive is left as it was
    assert bytes(t.cpu().numpy().tobytes()) == a
