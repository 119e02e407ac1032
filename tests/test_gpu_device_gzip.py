"""mz_cuda_gzip_compress_device / mz_cuda_gzip_decompress_device on the H100: the emulator suite's identity and parity matrix at small
sizes on the product library, then C2's shape (256 MiB of bench text at level 6, read back by the reference's minigzip and by zlib),
a member of more than 1 GiB written by the reference's minigzip and decoded on the device (K6 rounds), an input of 4 GiB + 1 MiB whose
ISIZE wraps, and the Python wrappers."""
import ctypes as C
import gzip
import hashlib
import os
import subprocess
import zlib

import pytest

import datagen
import test_emu_device_gzip as emu
from test_emu_device_gzip import GzipDevice, check_member, compress_inputs, decode_inputs, same_as_vtbl

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
REFDIR = os.path.join(os.path.dirname(HERE), "oracle", "_ref")


@pytest.fixture(scope="module")
def gz(built):
    import cuharness
    lib = cuharness.pkg().load()
    assert lib.mz_cuda_init() == 0
    return GzipDevice(lib)


@pytest.mark.parametrize("level", [0, 1, 2, 4, 6, 9, -1])
def test_compress_matches_vtbl(gz, level):
    for name, data in compress_inputs():
        err, member, n, bound, _ = gz.compress(data, level)
        assert err == 0, name
        check_member(gz, data, level, member, n, bound)


def test_compress_rounds_and_cap(gz, monkeypatch):
    data = datagen.text_like(5 << 20, seed=61)
    err, one, n, _, _ = gz.compress(data, 6)
    monkeypatch.setenv("MZ_CUDA_ZIP_ROUND_MB", "1")
    err2, many, _, _, st = gz.compress(data, 6)
    assert (err, err2) == (0, 0) and st.rounds == 5 and many == one and one == gz.vtbl_compress(data, 6)
    for cap in (n - 1, n // 2):
        err, _, n2, _, _ = gz.compress(data, 6, cap=cap, slack=4096)
        assert (err, n2) == (emu.MZ_BUF_ERROR, n)


def test_decode_matrix(gz):
    for name, member, want in decode_inputs():
        err, _, res, _ = same_as_vtbl(gz, member, want=want)
        assert err == 0 and res.in_used == len(member), name
        for shift in (1, 3):
            assert same_as_vtbl(gz, member, shift=shift, want=want)[0] == 0, (name, shift)


def test_decode_errors_and_output_full(gz):
    emu.test_decode_header_errors(gz)
    emu.test_decode_trailer_and_stream_errors(gz)
    emu.test_decode_output_full(gz)
    emu.test_decode_ignores_what_follows(gz)


def test_decode_speculative_rounds_and_spec_off(gz, monkeypatch):
    text = datagen.text_like(24 << 20, seed=62)
    member = emu.wbits31(text, 6)
    err, out, res, st = same_as_vtbl(gz, member, want=text)
    assert err == 0 and st.k6_rounds > 0
    monkeypatch.setenv("MZ_CUDA_SPEC", "0")
    err, out0, res0, st0 = gz.decompress(member, len(text))
    assert err == 0 and out0 == text and st0.k6_rounds == 0 and res0.in_used == res.in_used


def _ref(name):
    p = os.path.join(REFDIR, name)
    if not os.path.exists(p):
        pytest.skip("oracle/_ref/%s not built (reference sources absent at build time)" % name)
    return p


def test_c2_shape_read_by_reference_and_zlib(built, tmp_path):
    """256 MiB of bench text at level 6, compressed on the device: zlib and the reference's minigzip -x both give the input back"""
    import torch
    import textgen
    pkg = __import__("cuharness").pkg()
    n = 256 << 20
    src = textgen.device(n, seed=1234)
    member = pkg.gzip_compress_device(src, level=6)
    host = bytes(src.cpu().numpy().tobytes())
    m = bytes(member.cpu().numpy().tobytes())
    assert m[:10] == bytes([0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 0, 3])
    assert zlib.decompress(m, 31) == host
    out, used = pkg.gzip_decompress_device(member)
    assert used == len(m) and torch.equal(out, src)
    (tmp_path / "c2.txt.gz").write_bytes(m)
    ref = _ref("minigzip_ref")
    r = subprocess.run([ref, "-x", "-d", "x", "c2.txt.gz"], cwd=tmp_path, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=900)
    assert r.returncode == 0, r.stdout[-600:]
    assert hashlib.sha256((tmp_path / "x" / "c2.txt").read_bytes()).digest() == hashlib.sha256(host).digest()


def test_reference_member_over_1gib(built, tmp_path):
    """a member of more than 1 GiB of text written by the reference's minigzip -6, decoded on the device with K6 rounds"""
    import torch
    import textgen
    ref = _ref("minigzip_ref")
    pkg = __import__("cuharness").pkg()
    n = (1 << 30) + 12345
    (tmp_path / "big.txt").write_bytes(textgen.host_buffer(n, seed=77))
    want = hashlib.sha256((tmp_path / "big.txt").read_bytes()).digest()
    r = subprocess.run([ref, "-6", "big.txt"], cwd=tmp_path, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=1800)
    assert r.returncode == 0, r.stdout[-600:]
    (tmp_path / "big.txt").unlink()
    m = (tmp_path / "big.txt.gz").read_bytes()
    d_in = torch.frombuffer(bytearray(m), dtype=torch.uint8).cuda()
    lib = pkg.load()
    out = torch.empty(n, dtype=torch.uint8, device="cuda")
    res, st = pkg.GzipResult(), pkg.GzipStats()
    assert lib.mz_cuda_gzip_decompress_device(d_in.data_ptr(), len(m), out.data_ptr(), n, C.byref(res), C.byref(st), None) == 0
    assert res.in_used == len(m) and res.out_len == n and st.k6_rounds > 0
    assert hashlib.sha256(out.cpu().numpy().tobytes()).digest() == want


def test_past_4gib_isize_wraps(built):
    """4 GiB + 1 MiB compressed and decoded on the device: ISIZE is the length mod 2^32, length and CRC-32 come back right"""
    import torch
    import textgen
    pkg = __import__("cuharness").pkg()
    n = (4 << 30) + (1 << 20)
    src = textgen.device(n, seed=4321)
    crc = pkg.crc32_device(src)
    member = pkg.gzip_compress_device(src, level=1)
    tail = bytes(member[-8:].cpu().numpy().tobytes())
    assert int.from_bytes(tail[:4], "little") == crc and int.from_bytes(tail[4:], "little") == n & 0xffffffff == 1 << 20
    out, used = pkg.gzip_decompress_device(member)  # the ISIZE hint is 1 MiB: the retry takes 2^32 more
    assert used == member.numel() and out.numel() == n and pkg.crc32_device(out) == crc
    assert torch.equal(out, src)


def test_python_wrappers(built):
    import torch
    pkg = __import__("cuharness").pkg()
    data = datagen.text_like(300000, seed=63)
    t = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    for level in (0, 1, 6, 9, -1):
        m = pkg.gzip_compress_device(t, level)
        assert gzip.decompress(bytes(m.cpu().numpy().tobytes())) == data
        out, used = pkg.gzip_decompress_device(m)
        assert used == m.numel() and bytes(out.cpu().numpy().tobytes()) == data
    m = gzip.compress(data) + b"pad\0\0\0\0"
    out, used = pkg.gzip_decompress_device(torch.frombuffer(bytearray(m), dtype=torch.uint8).cuda())  # the hint is 0: one retry
    assert used == len(m) - 7 and bytes(out.cpu().numpy().tobytes()) == data
    with pytest.raises(RuntimeError):
        pkg.gzip_decompress_device(torch.frombuffer(bytearray(b"not a gzip member"), dtype=torch.uint8).cuda())
    with pytest.raises(RuntimeError):
        pkg.gzip_compress_device(t, 10)
    e = pkg.gzip_compress_device(torch.empty(0, dtype=torch.uint8, device="cuda"))
    assert gzip.decompress(bytes(e.cpu().numpy().tobytes())) == b""
    assert pkg.gzip_decompress_device(e)[0].numel() == 0
