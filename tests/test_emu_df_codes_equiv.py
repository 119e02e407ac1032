"""The deflate kernel's code builder (block_build_codes) against its frozen v3.4 form (tests/emu/df_codes_v34.cuh) on the CPU
emulator: both run on the same histograms and must agree on every code length, code word, bits-per-symbol entry, header bit and
header size. The corpus: the real per-unit histograms of the bench text at levels 1, 2, 4 and 6 (captured from the kernel on the
emulator), 0, 1 and 2 used symbols in either alphabet, all symbols equal, one dominant symbol, Fibonacci counts that reach the
15-bit limit, the largest counts a unit can produce, and 10^5 random Zipf-shaped histograms, each at a random header bit position
and BFINAL. tests/test_gpu_df_codes_equiv.py runs the same corpus on the GPU, where __log2f is the hardware's approximation."""
import ctypes as C
import multiprocessing
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
SRC = os.path.join(os.path.dirname(HERE), "minizip-ng_b200", "csrc")
HIST_WORDS = 288 + 32 + 256  # literal/length counts | distance counts | second copy of the literal counts
CAPTURE_LEVELS = (1, 2, 4, 6)
CAPTURE_BYTES = 16 * 65536 + 12345
N_ZIPF = 100000
UNIT_MAX = 32768  # positions in a unit: no count, and no literal total, exceeds it (+ 1 for the end of block)
FIELDS = (("code words", 0, 320), ("code lengths", 320, 400), ("bits per symbol", 400, 480), ("header staging", 480, 576),
          ("header size", 576, 577))


def build(out_dir):
    """compile the emulator harness into out_dir; returns the library's path and the compiler's output"""
    out = os.path.join(str(out_dir), "libemu_df_codes.so")
    cmd = [os.environ.get("CXX", "g++"), "-O1", "-g", "-fPIC", "-std=c++17", "-Wno-unused-function", "-Wno-unknown-pragmas",
           "-Wno-unused-variable", "-Wno-stringop-overflow", "-I" + EMU, "-I" + SRC, "-shared", "-o", out,
           os.path.join(EMU, "emu_df_codes.cc"), os.path.join(EMU, "cuda_emu.cc")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return (out if r.returncode == 0 else None), r.stdout


def load(path):
    L = C.CDLL(path)
    vp, u32 = C.c_void_p, C.c_uint32
    L.emu_df_hist_words.restype = u32
    L.emu_df_out_words.restype = u32
    L.emu_df_capture.restype = u32
    L.emu_df_capture.argtypes = [vp, C.c_uint64, C.c_int, vp, u32]
    L.emu_df_codes_pair.restype = None
    L.emu_df_codes_pair.argtypes = [vp, vp, u32, vp, vp]
    assert L.emu_df_hist_words() == HIST_WORDS and L.emu_df_out_words() >= FIELDS[-1][2]
    return L


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def captured(L):
    """the per-unit histograms of the bench text (host generator, seed 1000) at each capture level, on the emulator"""
    import textgen
    text = textgen.host(CAPTURE_BYTES, seed=1000)
    out = []
    for level in CAPTURE_LEVELS:
        cap = 4 * (CAPTURE_BYTES // 32768 + 2)
        buf = np.zeros((cap, HIST_WORDS), dtype=np.uint32)
        n = L.emu_df_capture(text, len(text), level, ptr(buf), cap)
        assert 0 < n <= cap
        out.append(buf[:n])
    return np.concatenate(out)


def hist(ll=None, d=None, lit2=None):
    h = np.zeros(HIST_WORDS, dtype=np.uint32)
    for part, off, n in ((ll, 0, 286), (d, 288, 30), (lit2, 320, 256)):
        if part is not None:
            part = np.asarray(part, dtype=np.uint64)
            assert len(part) <= n
            h[off:off + len(part)] = part
    return h


def edge_cases():
    """the hand-made shapes: few symbols, all equal, one dominant, Fibonacci, the largest totals"""
    hs = []
    eob = np.zeros(286, dtype=np.uint64)
    eob[256] = 1
    few = {0: [], 1: [[0], [5], [256], [285]], 2: [[0, 1], [0, 7], [3, 256], [256, 285], [284, 285]]}
    dfew = {0: [], 1: [[0], [1], [29]], 2: [[0, 1], [0, 29], [1, 2], [28, 29]]}
    for nl, lsets in few.items():
        for ls in (lsets or [[]]):
            for nd, dsets in dfew.items():
                for ds in (dsets or [[]]):
                    for cnt in (1, 1000, UNIT_MAX):
                        ll = np.zeros(286, dtype=np.uint64)
                        ll[ls] = cnt
                        d = np.zeros(30, dtype=np.uint64)
                        d[ds] = cnt
                        hs.append(hist(ll, d))
                        hs.append(hist(ll + eob, d))
    for v in (1, 2, 3, 100, UNIT_MAX // 286):  # all symbols equal
        hs.append(hist(np.full(286, v), np.full(30, v)))
        hs.append(hist(np.full(286, v), None))
    for v in (1, 7):  # all literals equal, split between the two copies
        hs.append(hist(np.concatenate([np.full(256, v), [1], np.zeros(29)]), np.full(30, v), np.full(256, v)))
    for sym in (0, 97, 256, 257, 285):  # one dominant symbol
        for big in (1000, UNIT_MAX - 285, UNIT_MAX):
            ll = np.ones(286, dtype=np.uint64)
            ll[sym] = big
            d = np.ones(30, dtype=np.uint64)
            d[sym % 30] = big
            hs.append(hist(ll, d))
    fib = [1, 1]
    while len(fib) < 30:
        fib.append(fib[-1] + fib[-2])
    for n in (15, 18, 20, 21, 22, 24, 27, 30):  # Fibonacci counts: the ideal lengths pass 15 bits
        f = np.array(fib[:n], dtype=np.uint64)
        ll = np.zeros(286, dtype=np.uint64)
        ll[np.arange(n) * 9 % 286] = f
        hs.append(hist(ll, f))
        hs.append(hist(ll[::-1].copy(), f[::-1].copy()))
    ll = np.zeros(286, dtype=np.uint64)  # the largest totals: every position a literal, split over the two copies
    ll[:256] = UNIT_MAX // 256
    ll[256] = 1
    hs.append(hist(ll, None, np.full(256, UNIT_MAX // 256)))
    ll = np.zeros(286, dtype=np.uint64)
    ll[65] = UNIT_MAX
    ll[256] = 1
    hs.append(hist(ll, None, np.full(256, 0)))
    ll[65] = UNIT_MAX // 2
    hs.append(hist(ll, np.array([UNIT_MAX // 4]), np.eye(1, 256, 65, dtype=np.uint64)[0] * (UNIT_MAX // 2)))
    ll = np.zeros(286, dtype=np.uint64)  # the most matches: every 4 bytes a length-4 match, every one at its own distance code
    ll[256] = 1
    ll[258] = UNIT_MAX // 4
    hs.append(hist(ll, np.full(30, UNIT_MAX // 4 // 30)))
    return np.stack(hs)


def zipf(n, seed):
    """n random Zipf-shaped histograms: a random set of used symbols, exponent 0.3..2.5, totals up to a unit's"""
    rng = np.random.default_rng(seed)
    out = np.zeros((n, HIST_WORDS), dtype=np.uint32)
    for i in range(n):
        for off, nsym, cap in ((0, 286, UNIT_MAX), (288, 30, UNIT_MAX // 3)):
            used = int(rng.integers(1, nsym + 1)) if rng.random() < 0.9 else int(rng.integers(0, 4))
            if used == 0:
                continue
            total = int(rng.integers(used, cap + 1)) if rng.random() < 0.7 else int(rng.integers(used, 4 * used + 2))
            w = 1.0 / np.arange(1, used + 1) ** rng.uniform(0.3, 2.5)
            c = rng.multinomial(total - used, w / w.sum()) + 1
            syms = rng.choice(nsym, used, replace=False)
            out[i, off + syms] = c
        if rng.random() < 0.5:  # the kernel counts odd lanes' literals in the second copy
            lit = out[i, :256].astype(np.int64)
            half = rng.binomial(lit, 0.5)
            out[i, :256] = lit - half
            out[i, 320:576] = half
        if rng.random() < 0.9:
            out[i, 256] = max(out[i, 256], 1)  # the end of block, as the kernel always has it
    return out


def corpus(L):
    """(histograms, posfin): every histogram with a random header bit position (0..127) and BFINAL"""
    h = np.concatenate([captured(L), edge_cases(), zipf(N_ZIPF, 20261016)])
    rng = np.random.default_rng(7)
    posfin = rng.integers(0, 128, len(h), dtype=np.uint32) | (rng.integers(0, 2, len(h), dtype=np.uint32) << 31)
    return np.ascontiguousarray(h), posfin.astype(np.uint32)


def mismatches(h, old, new, base=0):
    """how many histograms' outputs differ, and a readable line for each of the first few (base = index of h[0] in the corpus)"""
    bad = np.nonzero((old != new).any(axis=1))[0]
    msgs = []
    for i in bad[:5]:
        fields = [name for name, a, b in FIELDS if (old[i, a:b] != new[i, a:b]).any()]
        msgs.append("histogram %d (ll used %d, d used %d): %s differ" % (base + i, int((h[i, :286] + np.pad(h[i, 320:], (0, 30)) > 0).sum()),
                                                                   int((h[i, 288:318] > 0).sum()), ", ".join(fields)))
    return len(bad), msgs


def compare(L, h, posfin, base=0):
    """both builders on h; returns (number of histograms whose outputs differ, messages for the first few, headers all written)"""
    words = L.emu_df_out_words()
    old, new = np.zeros((len(h), words), dtype=np.uint32), np.zeros((len(h), words), dtype=np.uint32)
    h, posfin = np.ascontiguousarray(h), np.ascontiguousarray(posfin)
    L.emu_df_codes_pair(ptr(h), ptr(posfin), len(h), ptr(old), ptr(new))
    nbad, msgs = mismatches(h, old, new, base)
    return nbad, msgs, bool((old[:, 576] > 0).all())


_JOB = {}  # what the forked workers see: the library's path and the corpus


def _slice(ab):
    a, b = ab
    return compare(load(_JOB["path"]), _JOB["h"][a:b], _JOB["posfin"][a:b], a)


def run_corpus(path, h, posfin, step=2048):
    """compare() over the corpus in slices, one emulator process per CPU (the emulator runs one CTA at a time per process)"""
    _JOB.update(path=path, h=h, posfin=posfin)
    slices = [(a, min(a + step, len(h))) for a in range(0, len(h), step)]
    with multiprocessing.get_context("fork").Pool(min(len(slices), os.cpu_count() or 1)) as pool:
        res = pool.map(_slice, slices)
    return sum(r[0] for r in res), [m for r in res for m in r[1]][:5], all(r[2] for r in res)


@pytest.fixture(scope="module")
def emu_path(tmp_path_factory):
    path, log = build(tmp_path_factory.mktemp("emu_df_codes"))
    assert path, log
    return path


@pytest.fixture(scope="module")
def emu(emu_path):
    return load(emu_path)


def test_capture_sees_every_unit(emu):
    import textgen
    text = textgen.host(3 * 65536 + 12345, seed=1000)
    buf = np.zeros((16, HIST_WORDS), dtype=np.uint32)
    assert emu.emu_df_capture(text, len(text), 1, ptr(buf), 16) == 7  # 4 chunks: 2 + 2 + 2 + 1 units
    assert (buf[:7, 256] == 1).all()  # one end of block per unit


def test_code_builder_matches_v34_on_the_whole_corpus(emu, emu_path):
    h, posfin = corpus(emu)
    assert len(h) > N_ZIPF
    nbad, msgs, headers = run_corpus(emu_path, h, posfin)
    assert headers  # every run wrote a header
    assert nbad == 0, "%d of %d histograms differ:\n%s" % (nbad, len(h), "\n".join(msgs))
