"""The staging pools on the CPU emulator (tests/emu/libmz_strm_emu.so): which calls of the native writer, the extractors and the
mz_stream_cuda vtbl make new staging and which reuse pooled staging.

Each scenario runs in its own process with an LD_PRELOAD interposer that counts posix_memalign(..., 4096, ...) calls: on the
emulator those are exactly cudaMalloc and cudaHostAlloc (tests/emu/shim/cuda_runtime.h). The child prints the allocations of every
call, and checks every call's output against zlib or zipfile."""
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EMU = os.path.join(HERE, "emu", "libmz_strm_emu.so")
AES = 4

INTERPOSER = r"""
#define _GNU_SOURCE
#include <dlfcn.h>
#include <stddef.h>
long mzp_allocs;
int posix_memalign(void **p, size_t align, size_t n) {
    static int (*real)(void **, size_t, size_t);
    if (!real)
        real = (int (*)(void **, size_t, size_t))dlsym(RTLD_NEXT, "posix_memalign");
    if (align == 4096)
        __atomic_add_fetch(&mzp_allocs, 1, __ATOMIC_RELAXED);
    return real(p, align, n);
}
"""


@pytest.fixture(scope="module")
def interposer(built, tmp_path_factory):
    d = tmp_path_factory.mktemp("interposer")
    (d / "count.c").write_text(INTERPOSER)
    so = str(d / "libcount.so")
    subprocess.run(["gcc", "-O1", "-shared", "-fPIC", "-o", so, str(d / "count.c"), "-ldl"], check=True)
    return so


def run(interposer, scenario, **env):
    """-> the allocations of each call of `scenario` (see child())"""
    e = dict(os.environ)
    e.pop("MZ_CUDA_ZIP_POOL", None)
    e.update(LD_PRELOAD=interposer, MZ_CUDA_ZIP_ROUND_MB="1", MZ_CUDA_BATCH_KB="1024", **env)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), scenario], env=e, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_writer_second_identical_call_allocates_nothing(interposer):
    first, second = run(interposer, "write_twice")
    assert first > 0 and second == 0


def test_writer_larger_round_allocates(interposer):
    small, larger = run(interposer, "write_then_larger_round")
    assert small > 0 and larger > 0


def test_writer_aes_not_served_by_plain_but_plain_served_by_aes(interposer):
    plain, aes_after_plain, aes, plain_after_aes = run(interposer, "write_aes_rules")
    assert plain > 0 and aes > 0
    assert aes_after_plain > 0     # a pooled plain slot has no WinZip AES buffers
    assert plain_after_aes == 0    # a pooled AES slot serves a plain request


def test_writer_pool_off_allocates_every_call(interposer):
    first, second = run(interposer, "write_twice", MZ_CUDA_ZIP_POOL="0")
    assert first > 0 and second > 0


def test_writer_trim_empties_the_pool(interposer):
    first, after_trim = run(interposer, "write_trim")
    assert first > 0 and after_trim > 0


def test_extractor_second_identical_call_allocates_nothing(interposer):
    first, second = run(interposer, "extract_twice")
    assert first > 0 and second == 0


def test_extractor_larger_round_allocates(interposer):
    small, larger = run(interposer, "extract_then_larger_round")
    assert small > 0 and larger > 0


def test_extractor_pool_off_allocates_every_call(interposer):
    first, second = run(interposer, "extract_twice", MZ_CUDA_ZIP_POOL="0")
    assert first > 0 and second > 0


def test_extractor_trim_empties_the_pool(interposer):
    first, after_trim = run(interposer, "extract_trim")
    assert first > 0 and after_trim > 0


def test_oversized_extract_is_not_pooled(interposer):
    first, second = run(interposer, "extract_oversized")
    assert first > 0 and second > 0


def test_extract_all_is_not_pooled(interposer):
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libmzref.so")):
        pytest.skip("oracle/_ref/libmzref.so not built (needs the reference sources at build time)")
    first, second = run(interposer, "extract_all_twice")
    assert first > 0 and second > 0


def test_stream_workspaces_are_reused(interposer):
    w1, w2, r1, r2 = run(interposer, "stream_twice")
    assert w1 > 0 and w2 == 0
    assert r1 > 0 and r2 == 0


# ---- the child: one scenario, every call's allocations as one JSON line --------------------------------------------------------
def files_of(n, size, seed):
    import datagen
    return [("d%d/f%03d.txt" % (i % 3, i), datagen.text_like(size + 97 * i, seed=seed + i)[:size + 97 * i]) for i in range(n)]


def child(scenario):
    import ctypes as C
    import zlib
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    counter = C.c_long.in_dll(C.CDLL(os.environ["LD_PRELOAD"]), "mzp_allocs")
    if scenario == "extract_all_twice":  # the reference's zip reader first and global, so that extract_all finds it
        import extract_pair
        files = files_of(12, 40000, 5)
        pair = extract_pair.Pair(EMU, py_zip(files))
        out = []
        for _ in range(2):
            got = []
            n0 = counter.value
            err, _st = pair.run("all", on_entry=lambda _u, name, data, size, crc: got.append((name.decode(), C.string_at(data, size))) or 0)
            out.append(counter.value - n0)
            assert err == 0 and got == files, err
        pair.close()
        print(json.dumps(out))
        return
    import cuharness
    import test_emu_native_extract as ne
    ex = ne.Extractor(cuharness.pkg().configure(C.CDLL(EMU)))
    lib = ex.lib
    out = []

    def count(fn, *a, **k):
        n0 = counter.value
        r = fn(*a, **k)
        out.append(counter.value - n0)
        return r

    def write(files, **k):
        a = count(ex.write, files, **k)
        if k.get("flags", 0) & AES:
            err, got, _ = ex.extract(a, password=k["password"])
            assert err == 0 and [(n, d) for n, d, _c in got] == files, err
        else:
            assert [(n, d) for n, d, _c in ne.zipfile_view(a)] == files
        return a

    def extract(archive, files):
        err, got, _ = count(ex.extract, archive)
        assert err == 0 and [(n, d) for n, d, _c in got] == files, err

    files = files_of(12, 40000, 1)
    lib.mz_zip_cuda_trim()
    if scenario == "write_twice":
        write(files)
        write(files)
    elif scenario == "write_then_larger_round":
        write(files)
        os.environ["MZ_CUDA_ZIP_ROUND_MB"] = "3"
        write(files)
    elif scenario == "write_aes_rules":
        write(files)
        write(files, flags=AES, password="pool", strength=3)
        lib.mz_zip_cuda_trim()
        write(files, flags=AES, password="pool", strength=3)
        write(files)
    elif scenario == "write_trim":
        write(files)
        lib.mz_zip_cuda_trim()
        write(files)
    elif scenario in ("extract_twice", "extract_then_larger_round", "extract_trim"):
        archive = py_zip(files)
        extract(archive, files)
        if scenario == "extract_then_larger_round":
            os.environ["MZ_CUDA_ZIP_ROUND_MB"] = "3"
        if scenario == "extract_trim":
            lib.mz_zip_cuda_trim()
        extract(archive, files)
    elif scenario == "extract_oversized":  # one entry larger than a 1 MiB round
        big = files + [("big.bin", os.urandom(1536 * 1024))]
        archive = py_zip(big)
        extract(archive, big)
        extract(archive, big)
    elif scenario == "stream_twice":
        t = ex.t
        data = b"".join(d for _n, d in files)
        for _ in range(2):
            comp, info = count(t.compress, lib.mz_stream_cuda_create, data, level=6, window_bits=31)
            assert info["close"] == 0 and zlib.decompress(comp, 31) == data
        comp = zlib.compressobj(6, zlib.DEFLATED, 31)
        gz = comp.compress(data) + comp.flush()
        for _ in range(2):
            got, info = count(t.decompress, lib.mz_stream_cuda_create, gz, len(data), window_bits=31)
            assert got == data, info
    else:
        raise SystemExit("unknown scenario " + scenario)
    lib.mz_zip_cuda_trim()
    print(json.dumps(out))


def py_zip(files):
    import io
    import zipfile
    bio = io.BytesIO()
    with zipfile.ZipFile(bio, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for name, data in files:
            z.writestr(name, data)
    return bio.getvalue()


if __name__ == "__main__":
    child(sys.argv[1])
