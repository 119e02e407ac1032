"""The join copy (gather_slots_kernel) and the CRC segments kernel on the CPU emulator, at every alignment that matters to them:
destination offsets 0..15 mod 16 against lengths around 16-byte and 512-byte boundaries, many tiny slots sharing one 16-byte
word, explicit destinations with guard bytes around every range, and CRC segments at every start misalignment, ragged and
uniform. Checked against plain Python slicing and zlib.crc32. The harness is tests/emu/emu_join_crc.cc, built here with the
emulator runtime, plain and with AddressSanitizer + UBSan."""
import ctypes as C
import os
import random
import subprocess
import sys
import zlib

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
SRC = os.path.join(os.path.dirname(HERE), "minizip-ng_b200", "csrc")
SAN_FLAGS = ["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-fno-omit-frame-pointer"]
STRIDE = 8 * 1024 + 16  # slot stride of these tests (16-byte multiple); a slot of exactly STRIDE bytes ends its allocation
LENGTHS = [0, 1, 2, 3, 15, 16, 17, 31, 32, 33, 511, 512, 513, 7937, STRIDE]
CRC_LENGTHS = [0, 1, 15, 16, 17, 31, 32, 33, 511, 512, 513, 1023, 1024, 1025, 2047, 2048, 2049, 2063]


def build(out_dir, sanitize=False):
    """compile the harness with the emulator runtime into out_dir; returns the library's path and the compiler's output"""
    out = os.path.join(str(out_dir), "libemu_join_crc%s.so" % ("_san" if sanitize else ""))
    cxx = "/usr/bin/g++" if sanitize else os.environ.get("CXX", "g++")
    cmd = [cxx, "-O1", "-g", "-fPIC", "-std=c++17", "-Wno-unused-function", "-Wno-unknown-pragmas", "-Wno-unused-variable"] + \
        (SAN_FLAGS if sanitize else []) + ["-I" + EMU, "-I" + SRC, "-shared", "-o", out, os.path.join(EMU, "emu_join_crc.cc"),
                                           os.path.join(EMU, "cuda_emu.cc")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return (out if r.returncode == 0 else None), r.stdout


def load(path):
    L = C.CDLL(path)
    vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32
    L.emu_join.restype = None
    L.emu_join.argtypes = [vp, u64, vp, u32, vp, vp, u64, u32, vp]
    L.emu_crc32_segments.restype = None
    L.emu_crc32_segments.argtypes = [vp, u64, vp, vp, u32, u32, vp, vp]
    L.emu_crc32_uniform.restype = None
    L.emu_crc32_uniform.argtypes = [vp, u64, u64, u32, vp]
    return L


def join(L, slots, lens, dst, offsets=None, misalign=0):
    """run the join; returns (dst bytes after it, offsets used)"""
    n = len(lens)
    ln = (C.c_uint32 * max(n, 1))(*lens)
    off = (C.c_uint64 * max(n, 1))(*offsets) if offsets is not None else None
    buf = C.create_string_buffer(bytes(dst), max(len(dst), 1))
    out_off = (C.c_uint64 * (n + 1))()
    L.emu_join(bytes(slots), STRIDE, ln, n, off, buf, len(dst), misalign, out_off)
    return buf.raw[:len(dst)], list(out_off)


def crc_segments(L, data, segs, misalign):
    n = len(segs)
    off = (C.c_uint64 * max(n, 1))(*[o for o, _ in segs])
    ln = (C.c_uint32 * max(n, 1))(*[k for _, k in segs])
    res, crc = (C.c_uint32 * max(n, 1))(), (C.c_uint32 * max(n, 1))()
    L.emu_crc32_segments(bytes(data), len(data), off, ln, n, misalign, res, crc)
    return list(crc)[:n]


def make_slots(rng, n):
    return rng.randbytes(n * STRIDE)  # bytes past each slot's length are random too, so copying one too many shows


def aligned_case(rng):
    """one slot per (destination offset mod 16, length), placed with 16..47 random guard bytes between the ranges"""
    cases = [(o, k) for o in range(16) for k in LENGTHS]
    offs, pos = [], 0
    for o, k in cases:
        pos += 16 + rng.randrange(32)
        pos += (o - pos) % 16
        offs.append(pos)
        pos += k
    return cases, offs, pos + 48


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    path, log = build(tmp_path_factory.mktemp("emu_join_crc"))
    assert path, log
    return load(path)


@pytest.mark.parametrize("misalign", [0, 9])
def test_join_explicit_destinations_every_alignment_keeps_guards(emu, misalign):
    rng = random.Random(1 + misalign)
    cases, offs, size = aligned_case(rng)
    lens = [k for _, k in cases]
    slots = make_slots(rng, len(cases))
    dst = rng.randbytes(size)
    got, _ = join(emu, slots, lens, dst, offs, misalign)
    want = bytearray(dst)
    for i, (o, k) in enumerate(zip(offs, lens)):
        want[o:o + k] = slots[i * STRIDE:i * STRIDE + k]
    assert got == bytes(want)


@pytest.mark.parametrize("misalign", [0, 1, 7, 15])
def test_join_packed_matches_slicing(emu, misalign):
    rng = random.Random(100 + misalign)
    lens = LENGTHS + [rng.randrange(STRIDE + 1) for _ in range(9)]
    rng.shuffle(lens)
    lens.append(STRIDE)  # the last slot is full: reading past its last word leaves the allocation
    slots = make_slots(rng, len(lens))
    total = sum(lens)
    dst = rng.randbytes(total + 16)
    got, offs = join(emu, slots, lens, dst, None, misalign)
    want = b"".join(slots[i * STRIDE:i * STRIDE + k] for i, k in enumerate(lens))
    assert offs[-1] == total and offs[:-1] == [sum(lens[:i]) for i in range(len(lens))]
    assert got[:total] == want and got[total:] == dst[total:]


def test_join_many_tiny_slots_share_words(emu):
    rng = random.Random(7)
    lens = [rng.choice([0, 1, 1, 2, 3]) for _ in range(300)]
    slots = make_slots(rng, len(lens))
    total = sum(lens)
    for misalign in (0, 5, 13):
        dst = rng.randbytes(total + 32)
        got, _ = join(emu, slots, lens, dst, None, misalign)
        want = b"".join(slots[i * STRIDE:i * STRIDE + k] for i, k in enumerate(lens))
        assert got[:total] == want and got[total:] == dst[total:]


@pytest.mark.parametrize("misalign", range(16))
def test_crc_ragged_segments_every_start_alignment(emu, misalign):
    rng = random.Random(misalign)
    segs, pos = [], 0
    for k in CRC_LENGTHS:  # back to back: each start sits at a different alignment too
        segs.append((pos, k))
        pos += k + rng.randrange(3)
    data = rng.randbytes(pos + 5)
    got = crc_segments(emu, data, segs, misalign)
    assert got == [zlib.crc32(data[o:o + k]) for o, k in segs]


@pytest.mark.parametrize("seg", [512, 700, 1000, 4100])
def test_crc_uniform_segments_not_multiple_of_512(emu, seg):
    rng = random.Random(seg)
    data = rng.randbytes(5 * seg + 77)
    for misalign in (0, 3, 8, 15):
        crc = (C.c_uint32 * 6)()
        emu.emu_crc32_uniform(data, len(data), seg, misalign, crc)
        assert list(crc) == [zlib.crc32(data[i:i + seg]) for i in range(0, len(data), seg)]


SAN_SCRIPT = r"""
import random, sys, zlib
sys.path.insert(0, sys.argv[1])
import test_emu_join_crc_alignment as t
L = t.load(sys.argv[2])
rng = random.Random(3)
lens = t.LENGTHS + [t.STRIDE]
slots = t.make_slots(rng, len(lens))
for m in (0, 11):
    got, _ = t.join(L, slots, lens, bytes(sum(lens)), None, m)
    assert got == b"".join(slots[i * t.STRIDE:i * t.STRIDE + k] for i, k in enumerate(lens))
cases, offs, size = t.aligned_case(rng)
sl = t.make_slots(rng, len(cases))
got, _ = t.join(L, sl, [k for _, k in cases], bytes(size), offs, 0)
data = rng.randbytes(3000)
segs = [(0, 0), (1, 17), (20, 513), (533, 1025), (1558, 1442)]
assert t.crc_segments(L, data, segs, 5) == [zlib.crc32(data[o:o + k]) for o, k in segs]
print("sanitized join/crc ok")
"""


def test_join_and_crc_under_sanitizers(tmp_path):
    """The same kernels under AddressSanitizer: the slots end exactly at the last one, so an over-read past a slot's last
    16-byte word is reported."""
    path, _ = build(tmp_path, sanitize=True)
    asan = subprocess.run(["/usr/bin/gcc", "-print-file-name=libasan.so"], stdout=subprocess.PIPE).stdout.decode().strip()
    if not path or not os.path.isabs(asan) or not os.path.exists(asan):
        pytest.skip("no sanitizer runtime in this toolchain")
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:detect_stack_use_after_return=0:halt_on_error=1")
    r = subprocess.run([sys.executable, "-c", SAN_SCRIPT, HERE, path], env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, timeout=900)
    assert r.returncode == 0 and b"sanitized join/crc ok" in r.stdout, r.stdout[-3000:]
