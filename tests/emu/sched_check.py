"""Every emulated kernel family against its plain reference, under the schedule the environment selects (MZ_EMU_SCHED=<seed>,
MZ_EMU_RACE=1; see cuda_emu.h). Prints one JSON line {case: digest} for comparison with the default schedule's run; any
mismatch with a reference raises, and a race report aborts the process.
  python tests/emu/sched_check.py <part> [--full]        part: deflate | kernels | df_codes | join_crc | product
  python tests/emu/sched_check.py --seeds N [--full]     every part under seeds 1..N with the race checker, against seed 0
TEST INFRASTRUCTURE ONLY. Needs tests/emu/libmzemu.so and libmz_strm_emu.so (make -C tests/emu libmzemu.so libmz_strm_emu.so)."""
import contextlib
import ctypes as C
import hashlib
import json
import os
import random
import subprocess
import sys
import tempfile
import zlib

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
sys.path.insert(0, TESTS)
sys.path.insert(0, os.path.dirname(TESTS))
PARTS = ("deflate", "kernels", "df_codes", "join_crc", "product")
DEFLATE_LEVELS = (0, 1, 2, 4, 6, 9)
DEFLATE_FLAGS = (1, 3)  # FINAL; FINAL | DICT (one stream: chunks refer back)


def h(b):
    return hashlib.sha256(bytes(b)).hexdigest()[:16]


def deflate_sizes(full):
    edges = list(range(0, 41)) + list(range(254, 262)) + list(range(32760, 32776)) + list(range(65529, 65537))
    multi = [65537, 131072 + 4099, 200000]
    return edges + multi if full else edges[::3] + [32767, 32768, 65535, 65536] + multi[:1]


def part_deflate(full):
    import datagen
    import emushim
    from test_emu_deflate_digests import inputs
    emu = emushim.EmuLib()
    out = {}
    base = datagen.text_like(200000, seed=3) + datagen.random_bytes(1000, seed=4)
    for n in deflate_sizes(full):
        data = base[:n]
        for level in DEFLATE_LEVELS:
            for flags in DEFLATE_FLAGS:
                comp, _ = emu.deflate(data, level=level, final=flags)
                assert zlib.decompress(comp, -15) == data, (n, level, flags)
                out["size/%d/%d/%d" % (n, level, flags)] = h(comp)
    # the committed digests, on the inputs they list
    want = json.load(open(os.path.join(TESTS, "golden", "deflate_digests.json")))
    names = ("text", "runs", "periods", "traps") if full else ("traps",)
    for name, data in inputs().items():
        if name not in names:
            continue
        for level in DEFLATE_LEVELS:
            for mode, flags in (("chunks", 1), ("stream", 3)):
                comp, _ = emu.deflate(data, level=level, final=flags)
                key = "%s/%d/%s" % (name, level, mode)
                assert [len(comp), hashlib.sha256(comp).hexdigest()] == want[key], key
                out[key] = h(comp)
    return out


def raw_deflate(data, level, flush_every=0):
    co = zlib.compressobj(level, zlib.DEFLATED, -15)
    if not flush_every:
        return co.compress(data) + co.flush()
    parts = []
    for o in range(0, len(data), flush_every):
        parts.append(co.compress(data[o:o + flush_every]) + co.flush(zlib.Z_SYNC_FLUSH))
    return b"".join(parts) + co.flush()


def part_kernels(full):
    import datagen
    import emushim
    emu = emushim.EmuLib()
    out = {}
    data = datagen.text_like(90000 if full else 40000, seed=11) + datagen.binary_records(20000, seed=12)
    # K5 through small windows
    for level, iw, ow in ((1, 100, 300), (6, 3000, 5000), (9, 0, 0)):
        comp = raw_deflate(data, level, flush_every=7000 if level == 6 else 0)
        st, got, cons, _ = emu.inflate(comp + b"\x55" * 5, len(data), iw, ow)
        assert st == 1 and got == data and cons == len(comp), (level, iw, ow, st)
        out["inflate/%d/%d/%d" % (level, iw, ow)] = h(got)
    # K6 on small segments, then corrupted members: never more than zlib gives
    comp = raw_deflate(data, 6, flush_every=2500)
    for seg, max_seg, win in ((512, 256, 0), (1024, 64, 16384)):
        st, got, cons, stats = emu.inflate_spec(comp, len(data), seg_bytes=seg, max_seg=max_seg, window=win)
        assert st == 1 and got == data and cons == len(comp), (seg, stats)
        out["spec/%d/%d" % (seg, win)] = h(got)
    rng = random.Random(5)
    for trial in range(6 if full else 3):
        bad = bytearray(comp)
        pos = rng.randrange(len(bad) // 8, len(bad) - 64)
        if trial % 2:
            bad[pos] ^= 1 << rng.randrange(8)
        else:
            for k in range(rng.randrange(2, 40)):
                bad[pos + k] = rng.randrange(256)
        ref, good, ok = zlib.decompressobj(-15), b"", False
        try:
            for o in range(0, len(bad), 4096):
                good += ref.decompress(bytes(bad[o:o + 4096]))
            ok = ref.eof
        except zlib.error:
            pass
        st, got, _, stats = emu.inflate_spec(bytes(bad), len(data) + 50000, seg_bytes=1024, max_seg=128)
        if ok:
            assert st == 1 and got == good, (trial, st, stats)
        else:
            n = min(len(got), len(good))
            assert st < 0 and got[:n] == good[:n], (trial, st, stats)
        out["spec_bad/%d" % trial] = "%d:%s" % (st, h(got))
    # CRC-32 at every start misalignment, segment sizes around the kernel's rows
    for n, seg, mis in ((0, 4096, 0), (1, 4096, 3), (33, 512, 7), (70001, 65536, 1), (200003, 16384, 15), (5000, 700, 9)):
        ref = (data * 4)[:n]
        crc, segs = emu.crc32(ref, seg, mis)
        assert crc == zlib.crc32(ref) and segs == [zlib.crc32(ref[o:o + seg]) for o in range(0, n, seg)], (n, seg, mis)
        out["crc/%d/%d/%d" % (n, seg, mis)] = crc
    # SHA-256 on every padding case and unaligned packing
    msgs = [data[:k] for k in list(range(0, 130)) + [1000, 4097, 65536 + 7]]
    for align, shift in ((16, 0), (1, 3)):
        got = emu.sha256(msgs, align=align, shift=shift)
        assert got == [hashlib.sha256(m).digest() for m in msgs], (align, shift)
        out["sha/%d/%d" % (align, shift)] = h(b"".join(got))
    return out


@contextlib.contextmanager
def harness_dir():
    """where the df_codes and join_crc harnesses are built: SCHED_CHECK_BUILD_DIR (kept, so that runs under several seeds compile
    them once), or a fresh temporary directory"""
    keep = os.environ.get("SCHED_CHECK_BUILD_DIR")
    if keep:
        yield keep
    else:
        with tempfile.TemporaryDirectory() as d:
            yield d


def harness(t, d):
    """the harness library of test module t in directory d, built unless it is there"""
    path = os.path.join(d, "lib" + t.__name__ + ".so")
    if not os.path.exists(path):
        built, log = t.build(d)
        assert built, log
        os.replace(built, path)
    return path


def part_df_codes(full):
    import numpy as np
    import test_emu_df_codes_equiv as t
    with harness_dir() as d:
        L = t.load(harness(t, d))
        out = {}
        for k, hist in enumerate([t.edge_cases()] + [t.zipf(200 if full else 60, seed) for seed in (1, 2)]):
            posfin = np.array([(i * 7) % 128 | ((i & 1) << 31) for i in range(len(hist))], dtype=np.uint32)
            nbad, msgs, headers = t.compare(L, hist, posfin)  # against the frozen previous builder
            assert nbad == 0 and headers, (k, msgs)
            out["df_codes/%d" % k] = nbad
        return out


def part_join_crc(full):
    import test_emu_join_crc_alignment as t
    with harness_dir() as d:
        L = t.load(harness(t, d))
        out = {}
        rng = random.Random(8)
        for misalign in ((0, 9) if full else (0,)):  # every destination offset mod 16 against lengths around 16 and 512
            cases, offs, size = t.aligned_case(rng)
            lens = [k for _, k in cases]
            slots = t.make_slots(rng, len(cases))
            dst = rng.randbytes(size)
            got, _ = t.join(L, slots, lens, dst, offs, misalign)
            want = bytearray(dst)
            for i, (o, k) in enumerate(zip(offs, lens)):
                want[o:o + k] = slots[i * t.STRIDE:i * t.STRIDE + k]
            assert got == bytes(want), misalign
            out["join/%d" % misalign] = h(got)
        lens = [rng.choice([0, 1, 1, 2, 3]) for _ in range(200)]  # tiny slots sharing one 16-byte word
        slots = t.make_slots(rng, len(lens))
        total = sum(lens)
        for misalign in (0, 5, 13):
            dst = rng.randbytes(total + 32)
            got, _ = t.join(L, slots, lens, dst, None, misalign)
            assert got[:total] == b"".join(slots[i * t.STRIDE:i * t.STRIDE + k] for i, k in enumerate(lens)) and got[total:] == dst[total:]
            out["tiny/%d" % misalign] = h(got)
        for misalign in (range(16) if full else (0, 1, 7, 15)):
            segs, pos = [], 0
            for k in t.CRC_LENGTHS:
                segs.append((pos, k))
                pos += k + rng.randrange(3)
            data = rng.randbytes(pos + 5)
            got = t.crc_segments(L, data, segs, misalign)
            assert got == [zlib.crc32(data[o:o + k]) for o, k in segs], misalign
            out["crc/%d" % misalign] = h(repr(got).encode())
        return out


def part_product(full):
    import cuharness
    import test_emu_device_extract as d
    import test_emu_native_extract as n
    import wzaes_checks
    lib = cuharness.pkg().configure(C.CDLL(os.path.join(HERE, "libmz_strm_emu.so")))
    out = {}
    try:
        import cryptography  # noqa: F401
        have_crypto = True
    except ImportError:
        have_crypto = False
    if have_crypto:  # K8 against hashlib and the cryptography package
        def buf(b):
            m = C.create_string_buffer(bytes(b), max(len(b), 1))
            return C.cast(m, C.c_void_p), m
        wzaes_checks.run(lambda name, *a: getattr(lib, name)(*a), buf, lambda p, k: C.string_at(p, k), lens=(0, 1, 17, 4097))
        out["k8"] = "ok"
    pair = (n.Extractor(lib), d.DeviceExtractor(lib))
    files = n.corpus(6, 3000, seed=21)
    arcs = {"stored": n.py_zip(files, d.zipfile.ZIP_STORED, dirs=("empty_dir/",)), "deflated": n.py_zip(files),
            "zip64": n.zip64_directory(n.py_zip(files)), "reordered": n.reorder_directory(n.py_zip(files))}
    for name, a in arcs.items():  # K9 and K10 against each other and zipfile
        err, got = d.differential(pair, a, want=n.zipfile_view(a))
        assert err == 0, name
        out["zip/" + name] = h(repr(got).encode())
    pw = "pw-2"
    a = pair[0].write(files, flags=n.AES | n.HASH_SHA256, password=pw, strength=2)
    err, got = d.differential(pair, a, password=pw)
    assert err == 0 and got == [(k, v, zlib.crc32(v)) for k, v in files]
    out["zip/aes"] = h(repr(got).encode())
    name, (arc, codes) = sorted(n.malformed_cases(pair[0]).items())[0]
    err, _ = d.differential(pair, arc)
    assert err in codes, name
    out["zip/malformed"] = err
    for k, arc in enumerate(d.mutations(1234, 60 if full else 20)):
        # differential() checks every entry in front of the first failing one; that entry's output bytes are unspecified
        out["zip/mutation/%d" % k] = d.differential(pair, arc)[0]
    return out


def run_part(part, seed, full, race=True):
    """the part in a subprocess under the given seed (0 = the default schedule) -> (returncode, output)"""
    env = dict(os.environ)
    env.pop("MZ_EMU_SCHED", None)
    env.pop("MZ_EMU_RACE", None)
    if seed:
        env["MZ_EMU_SCHED"] = str(seed)
    if race:
        env["MZ_EMU_RACE"] = "1"
    r = subprocess.run([sys.executable, os.path.abspath(__file__), part] + (["--full"] if full else []), env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=3600)
    return r.returncode, r.stdout


def main():
    args = sys.argv[1:]
    full = "--full" in args
    args = [a for a in args if a != "--full"]
    if args and args[0] == "--seeds":
        fails = 0
        build_dir = tempfile.TemporaryDirectory()
        os.environ.setdefault("SCHED_CHECK_BUILD_DIR", build_dir.name)
        for part in PARTS:
            rc, base = run_part(part, 0, full, race=False)
            assert rc == 0, base[-3000:]
            for seed in range(1, int(args[1]) + 1):
                rc, got = run_part(part, seed, full)
                ok = rc == 0 and got.splitlines()[-1] == base.splitlines()[-1]
                fails += not ok
                print(part, "seed", seed, "ok" if ok else "FAIL\n" + got[-3000:], flush=True)
        print("fails", fails)
        sys.exit(1 if fails else 0)
    part = args[0]
    assert part in PARTS, part
    print(json.dumps(globals()["part_" + part](full), sort_keys=True))


if __name__ == "__main__":
    main()
