"""Round placement of the device-memory writers on the CPU emulator (tests/emu/libmz_strm_emu.so): mz_cuda_zip_wr_place (K11) and
mz_cuda_gzip_place (K14) called directly, S, dst and glen compared with a numpy reference. A round of more than 2048 chunks spans
several scan tiles, which the writer tests only reach with more than 128 MiB per round. Also pins the K6 / K5 schedule of
mz_cuda_gzip_decompress_device on two foreign members."""
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pytest

import datagen

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
MZ_OK, MZ_PARAM_ERROR = 0, -102
TILE = 2048            # MZ_CUDA_ZIP_WR_TILE
SLOT = 65536 + 5 + 64  # at least mz_cuda_deflate_slot_bound(65536): the most one chunk's stream can take


class ZipWr(C.Structure):
    """mz_cuda_zip_wr (include/mz_cuda_batch.h)"""
    vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
    _fields_ = [("data", vp), ("names", vp), ("items", vp), ("n", u32), ("aes", u32), ("sha", u32), ("dos_now", u32), ("archive", vp),
                ("cap", u64), ("bad", vp), ("cnt", vp), ("pre", vp), ("part", vp), ("nch", u64), ("c_off", vp), ("c_len", vp),
                ("c_flags", vp), ("c_item", vp), ("out_len", vp), ("residue", vp), ("glen", vp), ("S", vp), ("dst", vp), ("e_lh", vp),
                ("e_csize", vp), ("e_cd", vp), ("e_cdpre", vp), ("e_coff", vp), ("e_off", vp), ("e_len", vp), ("e_crc", vp),
                ("max_csize", vp), ("digest", vp), ("salt", vp), ("keys", vp), ("mac", vp), ("entries", vp), ("lh_base", u64),
                ("cd_base", u64), ("out_base", u64), ("n_base", u32), ("comment_len", u32), ("comment", vp)]


@pytest.fixture(scope="module")
def lib(built):
    import cuharness
    r = subprocess.run(["make", "-s", "-C", EMU, "libmz_strm_emu.so"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    L = cuharness.pkg().configure(C.CDLL(os.path.join(EMU, "libmz_strm_emu.so")))
    L.mz_cuda_zip_wr_place.argtypes = [C.POINTER(ZipWr), C.c_uint64, C.c_uint32, C.c_void_p]
    L.mz_cuda_zip_wr_place.restype = C.c_int32
    assert L.mz_cuda_init() == MZ_OK
    return L


class Dev:
    """device arrays of one test, freed at the end"""

    def __init__(self, L):
        self.L, self.ptrs = L, []

    def put(self, a):
        a = np.ascontiguousarray(a)
        p = self.L.mz_cuda_malloc(max(1, a.nbytes))
        assert p
        self.ptrs.append(p)
        if a.nbytes:
            assert self.L.mz_cuda_memcpy_h2d(p, a.ctypes.data, a.nbytes, None) == 0
        return p

    def get(self, p, n, dtype):
        a = np.empty(n, dtype=dtype)
        if a.nbytes:
            assert self.L.mz_cuda_memcpy_d2h(a.ctypes.data, p, a.nbytes, None) == 0
        return a

    def free(self):
        for p in self.ptrs:
            self.L.mz_cuda_free(p)


GUARD64, GUARD32 = np.uint64(0xabababababababab), np.uint32(0xabababab)


def reference(out_len, rounds, base, cap, s0):
    """S, dst, glen after the rounds [(c0, m)]: S(c) = s0 + the stream bytes in front of c; chunk c goes to base[c] + S(c) with copy
    length 0 when its bytes would pass cap. Arrays start as the guard pattern; S[0] = s0."""
    nch = len(out_len)
    S = np.full(nch + 1, GUARD64, dtype=np.uint64)
    dst = np.full(nch, GUARD64, dtype=np.uint64)
    glen = np.full(nch, GUARD32, dtype=np.uint32)
    S[0] = s0
    for c0, m in rounds:
        if m == 0:
            continue
        run = int(S[c0])
        for c in range(c0, c0 + m):
            S[c] = run
            d = int(base[c]) + run
            dst[c] = d
            glen[c] = out_len[c] if d + int(out_len[c]) <= cap else 0
            run += int(out_len[c])
        S[c0 + m] = run
    return S, dst, glen


class Round:
    """the S / dst / glen / part arrays of one stream of nch chunks, as the writers carve them"""

    def __init__(self, dev, out_len, s0, rmax):
        nch = len(out_len)
        self.nch = nch
        self.out_len = dev.put(out_len.astype(np.uint32))
        S = np.full(nch + 1, GUARD64, dtype=np.uint64)
        S[0] = s0
        self.S = dev.put(S)
        self.dst = dev.put(np.full(nch, GUARD64, dtype=np.uint64))
        self.glen = dev.put(np.full(nch, GUARD32, dtype=np.uint32))
        self.part = dev.put(np.zeros(rmax // TILE + 1, dtype=np.uint32))

    def result(self, dev):
        return dev.get(self.S, self.nch + 1, np.uint64), dev.get(self.dst, self.nch, np.uint64), dev.get(self.glen, self.nch, np.uint32)


def zip_case(dev, out_len, s0, rmax, cap, aes, sha, seed):
    """an mz_cuda_zip_wr over nch chunks of random entries; -> (w, base[c])"""
    rng = np.random.default_rng(seed)
    nch = len(out_len)
    n = max(1, nch // 3)
    c_item = np.sort(rng.integers(0, n, nch)).astype(np.uint32)
    name_len = rng.integers(1, 300, n).astype(np.uint32)
    overhead = rng.integers(0, 1 << 20, n + 1).astype(np.uint64)
    items = np.zeros((n, 10), dtype=np.uint32)  # mz_cuda_zip_dev_item: 40 bytes, name_len at byte 24
    items[:, 6] = name_len
    pre = np.zeros((n + 1, 6), dtype=np.uint64)  # mz_cuda_zip_wr_count: 48 bytes, overhead second
    pre[:, 1] = overhead
    r = Round(dev, out_len, s0, rmax)
    w = ZipWr()
    w.items, w.n, w.aes, w.sha, w.cap, w.pre, w.part, w.nch = dev.put(items), n, aes, sha, cap, dev.put(pre), r.part, nch
    w.c_item, w.out_len, w.glen, w.S, w.dst, w.lh_base = dev.put(c_item), r.out_len, r.glen, r.S, r.dst, 7777
    # local header, name, extra fields (AES 11, hash 40), salt and verifier: zw_head
    head = 30 + name_len.astype(np.uint64) + (11 if aes else 0) + (40 if sha else 0) + ((4 * aes + 4 + 2) if aes else 0)
    base = 7777 + overhead[c_item] + head[c_item]
    return w, r, base


def lengths(m, seed):
    return np.random.default_rng(seed).integers(0, SLOT + 1, m).astype(np.uint32)


@pytest.mark.parametrize("m", [1, 2047, 2048, 2049, 5000])
def test_gzip_place_one_round(lib, m):
    dev = Dev(lib)
    try:
        out_len = lengths(m, m)
        r = Round(dev, out_len, 0, m)
        cap = 1 << 62
        assert lib.mz_cuda_gzip_place(r.out_len, 0, m, r.S, r.dst, r.glen, 10, cap, r.part, None) == MZ_OK
        want = reference(out_len, [(0, m)], np.full(m, 10, dtype=np.uint64), cap, 0)
        for got, exp in zip(r.result(dev), want):
            assert np.array_equal(got, exp)
    finally:
        dev.free()


@pytest.mark.parametrize("aes,sha", [(0, 0), (3, 1)])
@pytest.mark.parametrize("m", [1, 2047, 2048, 2049, 5000])
def test_zip_place_one_round(lib, m, aes, sha):
    dev = Dev(lib)
    try:
        out_len = lengths(m, 100 + m)
        cap = 1 << 62
        w, r, base = zip_case(dev, out_len, 0, m, cap, aes, sha, seed=m)
        assert lib.mz_cuda_zip_wr_place(C.byref(w), 0, m, None) == MZ_OK
        want = reference(out_len, [(0, m)], base, cap, 0)
        for got, exp in zip(r.result(dev), want):
            assert np.array_equal(got, exp)
    finally:
        dev.free()


@pytest.mark.parametrize("which", ["zip", "gzip"])
def test_place_two_rounds_and_cap(lib, which):
    """two rounds carried by S[c0] (c0 > 0, from a nonzero S[0]), and a cap inside a chunk of the second round"""
    dev = Dev(lib)
    try:
        rounds = [(0, 2100), (2100, 3000)]
        nch = 5100
        out_len = lengths(nch, 7)
        s0 = 123457
        if which == "zip":
            w, r, base = zip_case(dev, out_len, s0, 3000, 0, 0, 1, seed=8)
        else:
            r, base = Round(dev, out_len, s0, 3000), np.full(nch, 10, dtype=np.uint64)
        cut = 3500  # the cap falls strictly inside chunk `cut`
        assert out_len[cut] > 2
        cap = int(base[cut]) + s0 + int(out_len[:cut].sum(dtype=np.uint64)) + int(out_len[cut]) // 2
        for c0, m in rounds:
            if which == "zip":
                w.cap = cap
                assert lib.mz_cuda_zip_wr_place(C.byref(w), c0, m, None) == MZ_OK
            else:
                assert lib.mz_cuda_gzip_place(r.out_len, c0, m, r.S, r.dst, r.glen, 10, cap, r.part, None) == MZ_OK
        S, dst, glen = r.result(dev)
        wS, wdst, wglen = reference(out_len, rounds, base, cap, s0)
        assert np.array_equal(S, wS) and np.array_equal(dst, wdst) and np.array_equal(glen, wglen)
        assert glen[cut] == 0 and (which == "zip" or glen[cut - 1] == out_len[cut - 1])
    finally:
        dev.free()


@pytest.mark.parametrize("which", ["zip", "gzip"])
def test_place_empty_and_oversized_rounds(lib, which):
    """m = 0 writes nothing; a round of more than 32768 chunks is refused before anything is launched"""
    dev = Dev(lib)
    try:
        nch = 40000
        out_len = lengths(nch, 9)
        if which == "zip":
            w, r, _ = zip_case(dev, out_len, 0, 32769, 1 << 62, 0, 0, seed=10)
            place = lambda c0, m: lib.mz_cuda_zip_wr_place(C.byref(w), c0, m, None)
        else:
            r = Round(dev, out_len, 0, 32769)
            place = lambda c0, m: lib.mz_cuda_gzip_place(r.out_len, c0, m, r.S, r.dst, r.glen, 10, 1 << 62, r.part, None)
        untouched = reference(out_len, [], np.zeros(nch, dtype=np.uint64), 0, 0)
        assert place(0, 0) == MZ_OK
        assert place(5, 0) == MZ_OK
        assert place(0, 32769) == MZ_PARAM_ERROR
        for got, exp in zip(r.result(dev), untouched):
            assert np.array_equal(got, exp)
    finally:
        dev.free()


# k6_rounds and k5_launches of mz_cuda_gzip_decompress_device with 4 KiB segments, recorded at commit 9a7555e (before the K6 schedule
# was shared between the vtbl and this call): the round sizes, the running ratio and the resume bit decide both counts.
K6_PINNED = {"text": (3, 0), "mixed": (3, 1)}


def member_data(kind):
    """text, or records, seeded random bytes (stored blocks: a round there finds no block start) and text"""
    if kind == "text":
        return datagen.text_like(1 << 20, seed=61)
    noise = np.random.default_rng(63).integers(0, 256, 256 << 10, dtype=np.uint8).tobytes()
    return datagen.binary_records(512 << 10, seed=62) + noise + datagen.text_like(512 << 10, seed=64)


@pytest.mark.parametrize("kind", ["text", "mixed"])
def test_gzip_decompress_schedule_pinned(lib, monkeypatch, kind):
    import cuharness
    pkg = cuharness.pkg()
    data = member_data(kind)
    c = zlib.compressobj(6, zlib.DEFLATED, 31)
    member = c.compress(data) + c.flush()
    monkeypatch.setenv("MZ_CUDA_SPEC_SEG_KB", "4")
    dev = Dev(lib)
    try:
        d_in = dev.put(np.frombuffer(member, dtype=np.uint8))
        d_out = dev.put(np.zeros(len(data), dtype=np.uint8))
        res, st = pkg.GzipResult(), pkg.GzipStats()
        err = lib.mz_cuda_gzip_decompress_device(d_in, len(member), d_out, len(data), C.byref(res), C.byref(st), None)
        assert err == MZ_OK and res.out_len == len(data) and res.in_used == len(member)
        assert dev.get(d_out, len(data), np.uint8).tobytes() == data
        assert (st.k6_rounds, st.k5_launches) == K6_PINNED[kind]
    finally:
        dev.free()
