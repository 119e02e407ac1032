"""Inflate conformance on the H100: the emulator suite's hand-built DEFLATE streams and their prefixes through the real kernels -- one
mz_cuda_inflate_streams launch over every prefix of every case, mz_cuda_gzip_decompress_device on each case and its cuts, and
extract_device on the two zip archives -- each compared with CPython's zlib as on the emulator."""
import pytest

import test_emu_inflate_conformance as emu

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib(built):
    import cuharness
    L = cuharness.pkg().load()
    assert L.mz_cuda_init() == 0
    return L


def test_batch_launch_every_prefix(lib):
    jobs = emu.prefix_jobs(sample=emu.BATCH_SAMPLE)
    assert len(jobs) > 4000
    emu.batch_check(lib, jobs)


def test_gzip_device(lib):
    from test_emu_device_gzip import GzipDevice
    gz = GzipDevice(lib)
    jobs = [(i, len(s)) for i, (_, s, _) in enumerate(emu.CASES)] + emu.header_prefixes()
    for i, k in jobs:
        zs, zout, _ = emu.CASES[i][2].at(k)
        want = emu.MZ_OK if zs == emu.D.END else zs
        member = emu.gzip_member(i, k)
        err, out, res, _ = gz.decompress(member, len(emu.CASES[i][2].out) + 1024)
        assert err == want, (emu.CASES[i][0], k, err, want)
        if want == emu.MZ_OK:
            assert out == zout and res.in_used == len(member), (emu.CASES[i][0], k)
        else:
            assert zout[:len(out)] == out and res.in_used <= len(member), (emu.CASES[i][0], k)


def test_extract_device(lib):
    from test_emu_device_extract import DeviceExtractor
    emu.zip_check(DeviceExtractor(lib), *emu.zip_archives())
