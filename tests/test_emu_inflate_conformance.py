"""Inflate conformance on the CPU emulator: hand-built DEFLATE streams (tests/deflate_craft.py) and every prefix of each, decoded by
K5 (whole input and through small input / output windows), by K6 with its serial fallback, by one mz_cuda_inflate_streams launch over
all of them, by mz_cuda_gzip_decompress_device and the vtbl read of each wrapped as a gzip member, and by extract_device on zip
archives of them. CPython's zlib, fed one byte at a time, is the reference: the status (end, data error, truncated) must be zlib's;
on success the bytes and the bytes consumed are zlib's; on an error the output is a prefix of what zlib delivered and no more than
the input is consumed."""
import ctypes as C
import hashlib
import io
import os
import random
import struct
import subprocess
import sys
import zipfile
import zlib

import pytest

import deflate_craft as D

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
MZ_OK = 0


def corpus():
    """[(name, stream, ZlibTrace)]: the valid cases, then the invalid ones"""
    cases = [(n, s) for n, s, _ in D.valid_cases()] + D.invalid_cases()
    return [(n, s, D.ZlibTrace(s)) for n, s in cases]


CASES = corpus()


def prefix_jobs(sample=None):
    """[(case index, k)]: every prefix of every case (sampled for the long stored cases, or all of them when `sample` is given)"""
    return [(i, k) for i, (_, s, _) in enumerate(CASES) for k in D.prefixes(len(s), sample=sample, seed=i)] + \
           [(i, len(s)) for i, (_, s, _) in enumerate(CASES)]


def out_cap(i):
    return len(CASES[i][2].out) + 1024


def agree(i, k, status, out, consumed, what=""):
    """one decode of the first k bytes of case i against zlib"""
    name, _, ref = CASES[i]
    zs, zout, zcons = ref.at(k)
    where = (name, k, what)
    assert status == zs, (where, status, zs)
    if zs == D.END:
        assert out == zout and consumed == zcons, (where, len(out), len(zout), consumed, zcons)
    else:
        assert zout[:len(out)] == out, (where, len(out), len(zout))
        assert consumed <= k, (where, consumed)


# ---- the reference ------------------------------------------------------------------------------------------------------------
def test_builder_and_oracle_agree_with_zlib(orc):
    """every valid stream decodes in zlib to the bytes the builder recorded; zlib rejects every invalid one with a data error; the
    oracle's status agrees with zlib on every prefix (a guard on the reference, not on the product)"""
    valid = {n: out for n, _, out in D.valid_cases()}
    for i, (name, s, ref) in enumerate(CASES):
        if name in valid:
            assert ref.status == D.END and ref.out == valid[name] and ref.stop == len(s), name
        else:
            assert ref.status == D.DATA_ERROR, name
    for i, k in prefix_jobs():
        err, out, cons = orc.inflate(CASES[i][1][:k], out_cap(i))
        zs = CASES[i][2].at(k)[0]
        assert err == (MZ_OK if zs == D.END else zs), (CASES[i][0], k, err)


# ---- K5 and K6 on the kernel emulator -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(built):
    r = subprocess.run(["make", "-s", "-C", EMU, "libmzemu.so"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    import emushim
    return emushim.EmuLib()


def test_k5_every_prefix(emu):
    for i, k in prefix_jobs():
        st, out, cons, _ = emu.inflate(CASES[i][1][:k], out_cap(i))
        agree(i, k, st, out, cons, "k5")


@pytest.mark.parametrize("window", [(33, 0), (0, 258), (7, 300)])
def test_k5_windows(emu, window):
    """the decoder resumed across input refills and output drains: every whole case and a sample of prefixes"""
    jobs = [(i, len(s)) for i, (_, s, _) in enumerate(CASES)] + prefix_jobs(sample=8)
    for i, k in random.Random(window[0] * 1000 + window[1]).sample(jobs, 600) + jobs[:len(CASES)]:
        st, out, cons, _ = emu.inflate(CASES[i][1][:k], out_cap(i), in_window=window[0], out_window=window[1])
        agree(i, k, st, out, cons, window)


def header_prefixes():
    """[(case index, k)]: the cuts inside the first dynamic header of each case that has one (and inside its first bytes otherwise)"""
    return [(i, k) for i, (_, s, _) in enumerate(CASES) for k in range(min(len(s), 24))]


@pytest.mark.parametrize("seg", [1024, 4096])
def test_k6_with_serial_fallback(emu, seg):
    """every whole case, the cuts in the first header and a sample of the other prefixes (each call sets up 64 segments)"""
    jobs = [(i, len(s)) for i, (_, s, _) in enumerate(CASES)] + header_prefixes()
    for i, k in jobs + random.Random(seg).sample(prefix_jobs(sample=8), 100):
        st, out, cons, _ = emu.inflate_spec(CASES[i][1][:k], out_cap(i), seg_bytes=seg)
        agree(i, k, st, out, cons, ("k6", seg))


# ---- the product library on the emulator: one batch launch, the gzip call and the vtbl, zip extraction ---------------------------
class BatchInflate:
    """one mz_cuda_inflate_streams launch over many streams, each a job with in_final = 1; input j starts at an offset = j mod 4 and
    is followed by 16 bytes of 0xa5 (the kernel may read that far)"""

    def __init__(self, lib):
        import cuharness
        self.pkg = cuharness.pkg()
        self.lib = lib

    def run(self, inputs, caps):
        L, pkg = self.lib, self.pkg
        src, offs = bytearray(), []
        for j, s in enumerate(inputs):
            src += b"\xa5" * ((j - len(src)) % 4)
            offs.append(len(src))
            src += s + b"\xa5" * 16
        oofs, total = [], 0
        for c in caps:
            oofs.append(total)
            total += (c + 15) // 16 * 16
        n = len(inputs)
        d_in, d_out = L.mz_cuda_malloc(len(src)), L.mz_cuda_malloc(max(total, 1))
        d_jobs = L.mz_cuda_malloc(n * C.sizeof(pkg.InflateJob))
        d_st = L.mz_cuda_malloc(n * C.sizeof(pkg.InflateState))
        try:
            assert L.mz_cuda_memcpy_h2d(d_in, bytes(src), len(src), None) == 0
            jobs = (pkg.InflateJob * n)(*[pkg.InflateJob(d_in + o, 0, len(s), d_out + oo, 0, c, 1, 0)
                                          for o, s, oo, c in zip(offs, inputs, oofs, caps)])
            assert L.mz_cuda_memcpy_h2d(d_jobs, jobs, C.sizeof(jobs), None) == 0
            zero = bytes(n * C.sizeof(pkg.InflateState))
            assert L.mz_cuda_memcpy_h2d(d_st, zero, len(zero), None) == 0
            assert L.mz_cuda_inflate_streams(d_jobs, d_st, n, None) == 0
            assert L.mz_cuda_stream_sync(None) == 0
            states = (pkg.InflateState * n)()
            assert L.mz_cuda_memcpy_d2h(states, d_st, C.sizeof(states), None) == 0
            out = C.create_string_buffer(max(total, 1))
            assert L.mz_cuda_memcpy_d2h(out, d_out, total, None) == 0
            raw = out.raw
            return [(s.status, raw[oo:oo + s.out_pos], (s.in_bitpos + 7) // 8, s) for s, oo in zip(states, oofs)]
        finally:
            for p in (d_in, d_out, d_jobs, d_st):
                L.mz_cuda_free(p)


def batch_check(lib, jobs):
    """decode the jobs in one launch; returns a digest of the results (to compare schedules)"""
    res = BatchInflate(lib).run([CASES[i][1][:k] for i, k in jobs], [out_cap(i) for i, _ in jobs])
    h = hashlib.sha256()
    for (i, k), (st, out, cons, s) in zip(jobs, res):
        assert s.status != 0 and s.why == 0, (CASES[i][0], k, s.status, s.why)
        agree(i, k, st, out, cons, "batch")
        h.update(struct.pack("<iQQ", st, len(out), cons) + out)
    return h.hexdigest()


@pytest.fixture(scope="module")
def prod(built):
    r = subprocess.run(["make", "-s", "-C", EMU, "libmz_strm_emu.so"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    import cuharness
    return cuharness.pkg().configure(C.CDLL(os.path.join(EMU, "libmz_strm_emu.so")))


BATCH_SAMPLE = 40  # prefixes of each long stored case in the batch (each takes a 65 KiB output buffer)


def test_batch_launch_every_prefix(prod):
    batch_check(prod, prefix_jobs(sample=BATCH_SAMPLE))


def gzip_member(i, k):
    """case i as a gzip member with zlib's CRC-32 and ISIZE, or its first k stream bytes alone after the header (a member cut short in
    its stream)"""
    s, out = CASES[i][1], CASES[i][2].out
    trailer = struct.pack("<II", zlib.crc32(out), len(out) & 0xffffffff) if k == len(s) else b""
    return b"\x1f\x8b\x08\x00\x00\x00\x00\x00\x00\x03" + s[:k] + trailer


def gzip_check(gz, ref, jobs):
    """mz_cuda_gzip_decompress_device and the vtbl read on each member: zlib's status, the reference reader's return code and
    TOTAL_IN (when the reference library is built)"""
    for i, k in jobs:
        member = gzip_member(i, k)
        zs, zout, _ = CASES[i][2].at(k)
        want = MZ_OK if zs == D.END else zs
        err, out, res, _ = gz.decompress(member, len(CASES[i][2].out) + 1024)
        code, vout, total_in = gz.vtbl_decompress(member, len(CASES[i][2].out) + 1024)
        where = (CASES[i][0], k)
        assert err == want and code == want, (where, err, code, want)
        if want == MZ_OK:
            assert out == zout and vout == zout and res.in_used == total_in == len(member), where
        else:
            assert zout[:len(out)] == out and res.in_used <= len(member) and total_in <= len(member), (where, res.in_used, total_in)
        if ref is not None:
            rout, info = ref.decompress_with(ref.lib.mz_stream_zlib_create, member, window_bits=31)
            assert info["read_err"] == want, (where, info["read_err"])
            if want == MZ_OK:
                assert info["total_in"] == total_in, (where, info["total_in"], total_in)


@pytest.fixture(scope="module")
def gz(prod):
    from test_emu_device_gzip import GzipDevice
    return GzipDevice(prod)


@pytest.fixture(scope="module")
def refmaybe(built):
    import refshim
    return refshim.RefLib() if refshim.ref_available() else None


def test_gzip_device_and_vtbl(gz, refmaybe):
    gzip_check(gz, refmaybe, prefix_jobs(sample=3)[::3] + [(i, len(s)) for i, (_, s, _) in enumerate(CASES)] +
               [(i, k) for i, (n, s, _) in enumerate(CASES) if n.startswith(("long", "repeat", "hlit257")) for k in range(min(len(s), 40))])


def zip_of(entries):
    """a zip archive of raw DEFLATE entries: [(name, stream, crc, size)]"""
    body, cd = bytearray(), bytearray()
    for name, s, crc, size in entries:
        nm = name.encode()
        fields = struct.pack("<HHHHHIII", 20, 0, 8, 0, 0x21, crc, len(s), size)
        cd += b"PK\x01\x02" + struct.pack("<H", 20) + fields + struct.pack("<HHHHHII", len(nm), 0, 0, 0, 0, 0, len(body)) + nm
        body += b"PK\x03\x04" + fields + struct.pack("<HH", len(nm), 0) + nm + s
    n = len(entries)
    return bytes(body + cd + b"PK\x05\x06" + struct.pack("<HHHHIIH", 0, 0, n, n, len(cd), len(body), 0))


def zip_archives():
    """(an archive of every valid case, [an archive of each invalid case])"""
    valid = [(n, s, zlib.crc32(t.out), len(t.out)) for n, s, t in CASES if t.status == D.END]
    bad = [zip_of([(n, s, 0, 65536)]) for n, s, t in CASES if t.status != D.END]
    return zip_of(valid), bad


def zip_check(dx, good, bad):
    err, got, n, _ = dx.extract(good)
    with zipfile.ZipFile(io.BytesIO(good)) as z:
        want = [(info.filename, z.read(info)) for info in z.infolist()]
    assert err == 0 and n == len(want) and [(g[0], g[1]) for g in got] == want
    for a in bad:
        err, got, _, _ = dx.extract(a)
        assert err != 0 and all(g[3] != 0 for g in got), (err, [g[3] for g in got])


def test_extract_device(prod):
    from test_emu_device_extract import DeviceExtractor
    zip_check(DeviceExtractor(prod), *zip_archives())


# ---- the batch launch under seeded schedules with the shared-memory race checker ---------------------------------------------------
def test_batch_launch_schedules_and_race_checker(prod):
    jobs = prefix_jobs(sample=4)[::2]
    want = batch_check(prod, jobs)
    for seed in (5, 23):
        script = ("import ctypes as C, sys\nsys.path.insert(0, %r)\nimport cuharness, test_emu_inflate_conformance as t\n"
                  "lib = cuharness.pkg().configure(C.CDLL(%r))\nprint('digest', t.batch_check(lib, t.prefix_jobs(sample=4)[::2]))\n"
                  % (HERE, os.path.join(EMU, "libmz_strm_emu.so")))
        r = subprocess.run([sys.executable, "-c", script], env=dict(os.environ, MZ_EMU_SCHED=str(seed), MZ_EMU_RACE="1"),
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
        assert r.returncode == 0, r.stdout[-3000:]
        assert ("digest " + want) in r.stdout.splitlines(), (seed, r.stdout[-2000:])
