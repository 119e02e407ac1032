"""mz_zip_cuda_write_device on the H100: byte identity with mz_zip_cuda_write_archive at larger sizes and every source alignment (the
deflate kernel's bulk-load path for 16-byte aligned units, its byte path otherwise), the C4 shape, an archive past 4 GiB with more than
65535 entries (zip64 directory fields and end records), AES round trips and the Python write_device."""
import ctypes as C
import hashlib
import zlib

import pytest

import datagen
from test_emu_device_extract import DeviceExtractor
from test_emu_device_write import DATE, DeviceWriter, aes_ranges, check_reads, mask
from test_emu_native_extract import AES, HASH_SHA256, corpus

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dw(built):
    import cuharness
    lib = cuharness.pkg().load()
    assert lib.mz_cuda_init() == 0
    w = DeviceWriter(lib)

    def sink_bytes(m):  # archives past 2 GiB
        p = C.c_void_p()
        n = w.t.lib.mz_stream_mem64_get_buffer(m, C.byref(p))
        return bytes((C.c_char * n).from_address(p.value)) if n else b""
    w.t.sink_bytes = sink_bytes
    return w


def mib_entries(count, seed=90):
    """count entries cycling over five kinds (text of ~1 MiB, empty, one byte, text of ~0.35 MiB, incompressible ~2.1 MiB), each a
    distinct slice of a generated pool: with offsets i mod 16, every residue meets every kind"""
    import random
    text = datagen.text_like(12 << 20, seed=seed)
    noise = datagen.random_bytes(12 << 20, seed=seed + 1)
    rng = random.Random(seed)
    sizes = [1_100_000, 0, 1, 366_673, 2_200_013]
    out = []
    for i in range(count):
        k, n = i % 5, sizes[i % 5]
        pool = noise if k == 4 else text
        o = rng.randrange(len(pool) - n + 1)
        out.append(("m%d/f%04d.bin" % (i % 3, i), pool[o:o + n]))
    return out


def test_identity_levels_and_alignments(dw):
    files = mib_entries(320)
    offs, pos = [], 0
    for i, (_, d) in enumerate(files):
        offs.append(pos + i % 16)
        pos += (len(d) + 47) & ~15
    for level in (1, 6, 9):
        for flags in (0, HASH_SHA256):
            err_h, want = dw.host(files, level=level, flags=flags)
            err, got, rows, n, bound = dw.device(files, level=level, flags=flags, offsets=offs, entries=True)
            assert (err, err_h) == (0, 0) and got == want and n <= bound, (level, flags)
    check_reads(dw, got, files, rows)


def c4_blobs(entry_bytes=65536):
    gens = [datagen.text_like] * 7 + [datagen.binary_records] * 2 + [datagen.random_bytes]
    return [gens[k % 10](entry_bytes, seed=k)[:entry_bytes] for k in range(100)]


def repeated(dw, blobs, count, level, prefix):
    """count entries cycling over 100 blobs: device items share the blobs' bytes, the host writer gets the same bytes"""
    files = [("%s/%06d" % (prefix, i), blobs[i % 100]) for i in range(count)]
    data = b"".join(blobs)
    names = b"".join(n.encode() for n, _ in files)
    items = (dw.pkg.ZipDevItem * count)()
    pos = 0
    for i, (n, d) in enumerate(files):
        items[i] = dw.pkg.ZipDevItem((i % 100) * len(blobs[0]), len(d), pos, len(n), dw.pkg.dos_date(DATE), 0, 0)
        pos += len(n)
    err_h, want = dw.host(files, level=level)
    assert err_h == 0
    err, got, rows, n, _ = dw.device(files, level=level, layout=(data, names, bytes(items)), entries=True)
    assert err == 0 and n == len(want)
    assert hashlib.sha256(got).digest() == hashlib.sha256(want).digest()
    del want
    dx = DeviceExtractor(dw.lib)
    err, out, count_x, _ = dx.extract(got)
    assert err == 0 and count_x == count
    assert all(o[0] == f[0] and o[1] == f[1] and o[2] == zlib.crc32(f[1]) for o, f in zip(out, files))
    assert [(r.crc, r.usize) for r in rows] == [(o[2], len(o[1])) for o in out]
    return got


def test_c4_shape(dw):
    repeated(dw, c4_blobs(), 100_000, 6, "e")
    dw.lib.mz_zip_cuda_trim()


def test_zip64_past_4_gib(dw):
    a = repeated(dw, c4_blobs(), 70_000, 0, "z")
    assert len(a) > 1 << 32 and b"PK\x06\x06" in a[-200:] and b"PK\x06\x07" in a[-200:]
    dw.lib.mz_zip_cuda_trim()


def test_stored_size_past_32_bits_is_refused(dw):
    """one incompressible entry of 0xfff80000 bytes: at level 0 its stream carries ten or more bytes of stored-block headers and sync
    marker per 64 KiB chunk, so the stored size passes 0xffffffff and the local header cannot hold it. The host writer returns
    MZ_INTERNAL_ERROR for such an entry (za_prepare); the device writer must too, not an archive with truncated sizes."""
    import torch
    size = 0xfff80000
    data = torch.randint(0, 256, (size,), dtype=torch.uint8, device="cuda")
    names = torch.frombuffer(bytearray(b"big.bin"), dtype=torch.uint8).cuda()
    item = dw.pkg.ZipDevItem(0, size, 0, 7, dw.pkg.dos_date(DATE), 0, 0)
    items = torch.frombuffer(bytearray(bytes(item)), dtype=torch.uint8).cuda()
    n = C.c_uint64(0)
    args = (data.data_ptr(), names.data_ptr(), items.data_ptr(), 1, 0, 0, None, 0)
    assert dw.lib.mz_zip_cuda_write_device(*args, None, 0, C.byref(n), None, None, None) == 0
    arc = torch.empty(n.value, dtype=torch.uint8, device="cuda")
    assert dw.lib.mz_zip_cuda_write_device(*args, arc.data_ptr(), arc.numel(), C.byref(n), None, None, None) == -104  # MZ_INTERNAL_ERROR
    del arc, data
    torch.cuda.empty_cache()


@pytest.mark.parametrize("strength", [1, 2, 3])
def test_aes_round_trip(dw, strength):
    files = corpus(60, 300_000, seed=91 + strength)
    err_h, want = dw.host(files, flags=AES | HASH_SHA256, password="secret", strength=strength)
    err, got, rows, _, _ = dw.device(files, flags=AES | HASH_SHA256, password="secret", strength=strength, entries=True)
    assert (err, err_h) == (0, 0)
    assert mask(got, aes_ranges(got)) == mask(want, aes_ranges(want))
    check_reads(dw, got, files, rows, password="secret")
    assert DeviceExtractor(dw.lib).extract(got, password="nope")[0] == -108


def test_python_write_device(dw):
    import torch
    import cuharness
    pkg = cuharness.pkg()
    files = corpus(30, 200_000, seed=95)
    tensors = [("t/%02d" % i, torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda() if d else torch.empty(0, dtype=torch.uint8, device="cuda"))
               for i, (_, d) in enumerate(files)]
    for kw in ({}, {"sha256": True, "level": 9}, {"password": "pw", "aes_strength": 2}):
        arc = pkg.write_device(tensors, mtime=DATE, **kw)
        entries, out = pkg.extract_device(arc, password=kw.get("password"))
        host = out.cpu().numpy().tobytes()
        assert [(n, host[o:o + s]) for n, o, s, _ in entries] == [(n, d) for (n, _), (_, d) in zip(tensors, files)]
    err_h, want = dw.host([(n, d) for (n, _), (_, d) in zip(tensors, files)])
    arc = pkg.write_device(tensors, mtime=DATE)
    assert arc.cpu().numpy().tobytes() == want
    assert arc.untyped_storage().nbytes() == len(want)  # the archive's storage is exactly its length, not the sizing bound
