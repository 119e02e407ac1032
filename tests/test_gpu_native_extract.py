"""mz_zip_cuda_extract_archive on the H100: the scenarios of tests/test_emu_native_extract.py at larger sizes, a 70 000-entry
native archive (zip64 end records), a reference-written archive next to extract_all, and ALL_DEVICES."""
import os
import subprocess
import zlib

import pytest

import datagen
from test_emu_native_extract import (ALL_DEVICES, AES, HASH_SHA256, MZ_PASSWORD_ERROR, Extractor, corpus, malformed_cases, pair_archives, pair_check,
                                     patch_zip64_end, py_zip, reorder_directory, zip64_directory, zipfile_view)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFDIR = os.path.join(ROOT, "oracle", "_ref")


@pytest.fixture(scope="module")
def ex(built):
    import cuharness
    lib = cuharness.pkg().load()
    assert lib.mz_cuda_init() == 0
    return Extractor(lib)


def test_zipfile_and_native_archives(ex):
    files = corpus(200, 200_000, seed=11)
    for a in (py_zip(files), py_zip(files, stream=True), py_zip(files[:40], force_zip64=True), ex.write(files), ex.write(files, flags=HASH_SHA256)):
        err, got, st = ex.extract(a)
        assert err == 0 and got == zipfile_view(a) and st.entries == len(got)


@pytest.mark.parametrize("strength", [1, 2, 3])
def test_aes(ex, strength):
    files = corpus(100, 100_000, seed=12)
    a = ex.write(files, flags=AES | HASH_SHA256, password="secret", strength=strength)
    err, got, _ = ex.extract(a, password="secret")
    assert err == 0 and got == [(n, d, zlib.crc32(d)) for n, d in files]
    assert ex.extract(a, password="nope")[0] == MZ_PASSWORD_ERROR


def test_layouts_rounds_and_refusals(ex, monkeypatch):
    files = corpus(120, 150_000, seed=13)
    a = py_zip(files)
    want = zipfile_view(a)
    assert ex.extract(patch_zip64_end(a))[1] == want
    assert ex.extract(zip64_directory(a))[1] == want
    assert ex.extract(b"\0" * 1000 + a)[1] == want
    r = reorder_directory(a)
    assert ex.extract(r)[1] == zipfile_view(r)
    monkeypatch.setenv("MZ_CUDA_ZIP_ROUND_MB", "1")
    err, got, st = ex.extract(a)
    assert err == 0 and got == want and st.rounds > 4
    monkeypatch.delenv("MZ_CUDA_ZIP_ROUND_MB")
    for name, (arc, codes) in malformed_cases(ex).items():
        assert ex.extract(arc)[0] in codes, name


def test_70000_entries_with_zip64_end_records(ex):
    texts = [datagen.text_like(3000, seed=s) for s in range(97)]
    files = [("n/%06d" % i, texts[i % 97][:1 + (i * 7919) % 3000]) for i in range(70_000)]
    a = ex.write(files, level=1)
    assert b"PK\x06\x06" in a[-200:]
    err, got, st = ex.extract(a)
    assert err == 0 and len(got) == 70_000
    assert all(g[0] == f[0] and g[1] == f[1] and g[2] == zlib.crc32(f[1]) for g, f in zip(got, files))
    ex.lib.mz_zip_cuda_trim()


def test_all_devices(ex):
    import torch
    files = corpus(300, 100_000, seed=14)
    a = ex.write(files)
    one = ex.extract(a)[1]
    err, got, _ = ex.extract(a, flags=ALL_DEVICES)
    assert err == 0 and got == one
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: ALL_DEVICES ran on it; the two-GPU split needs two")


def test_reference_written_archive_against_extract_all(ex, tmp_path):
    """extract_all and extract_archive in one process on the same base stream, entry by entry: a 2500 x 64 KiB reference-written
    archive and the emulator test's archives at larger sizes"""
    exe = os.path.join(REFDIR, "zipbatch_cuda")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/zipbatch_cuda not built (needs the reference sources at build time)")
    path = tmp_path / "c4.zip"
    r = subprocess.run([exe, str(path), "2500", "65536", "6", "ref"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=900)
    assert r.returncode == 0, r.stderr[-500:]
    a = path.read_bytes()
    err, got, _ = ex.extract(a)
    assert err == 0 and got == zipfile_view(a) and len(got) == 2500
    out = pair_check(ex.pkg.LIB_PATH, tmp_path, [(a, None)] + pair_archives(ex, 300, 100_000))
    assert out is not None
