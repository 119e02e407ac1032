"""Times zip extraction on one archive held in host memory, in one process: mz_zip_cuda_extract_all (the reference's own
directory walk and raw-seam reads: oracle/_ref/libmzref.so, when it was built) against mz_zip_cuda_extract_archive (directory
parsed natively), and extract_archive with MZ_ZIP_CUDA_ALL_DEVICES when more than one GPU is visible. Every call reads the same
bytes from the same 64-bit memory base stream (tests/support/libmztest.so), so disk is not measured; the calls alternate
`--pairs` times after one warm-up of each. extract_all makes its page-locked and device staging on every call, so its times
include that; extract_archive's staging is pooled between calls (setup_ms). The archive is the C4 shape (entries x 64 KiB, 70 %
text-like / 20 % records / 10 % incompressible, level 6), written by the product's native writer.

    python tools/bench_extract.py [--entries 100000] [--entry-bytes 65536] [--pairs 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    q = "name,power.limit,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--entries", type=int, default=100_000)
    ap.add_argument("--entry-bytes", type=int, default=65536)
    ap.add_argument("--pairs", type=int, default=3)
    args = ap.parse_args()
    import cuharness
    import extract_pair
    pkg = cuharness.pkg()
    have_ref = os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libmzref.so"))
    if have_ref:  # the reference's reader must be loaded (globally) before the product
        extract_pair.load(pkg.LIB_PATH)
    lib = pkg.load()
    pkg.check(lib.mz_cuda_init(), "mz_cuda_init")
    gen = os.path.join(ROOT, "oracle", "_ref", "zipbatch_cuda")
    tmpdir = tempfile.mkdtemp(dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    path = os.path.join(tmpdir, "c4.zip")
    if os.path.exists(gen):  # the archive exactly as zipbatch's C4 generator makes it, written natively
        r = subprocess.run([gen, path, str(args.entries), str(args.entry_bytes), "6", "native"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
        assert r.returncode == 0, r.stderr[-500:]
        archive = open(path, "rb").read()
    else:
        import datagen
        from test_emu_native_extract import Extractor
        gens = [datagen.text_like] * 7 + [datagen.binary_records] * 2 + [datagen.random_bytes]
        blobs = [gens[k % 10](args.entry_bytes, seed=k) for k in range(100)]  # a hundred distinct entries, repeated
        archive = Extractor(lib).write([("e/%06d" % i, blobs[i % 100]) for i in range(args.entries)], level=6)
    if os.path.exists(path):
        os.remove(path)
    os.rmdir(tmpdir)
    print("# archive: %d entries, %.1f MiB stored; GPU: %s; host cores: %d; one memory base stream for every call (disk not measured)"
          % (args.entries, len(archive) / 2**20, gpu_info(), os.cpu_count()), flush=True)
    pair = extract_pair.Pair(pkg.LIB_PATH, archive)
    count = [0, 0]

    def on_entry(_ud, _name, _data, size, _crc):
        count[0] += 1
        count[1] += size
        return 0

    def timed(which, flags=0):
        count[0] = count[1] = 0
        t0 = time.perf_counter()
        err, st = pair.run(which, None, flags, on_entry)
        dt = time.perf_counter() - t0
        assert err == 0 and count[0] == args.entries, (which, err, count[0])
        mode = "extract_all" if which == "all" else "extract_archive" + ("_all_devices" if flags else "")
        return {"mode": mode, "err": err, "entries": count[0], "s": round(dt, 4), "entries_per_s": round(count[0] / dt),
                "GiB_per_s": round(count[1] / 2**30 / dt, 3), "pack_ms": round(st.pack_ms, 1), "gpu_ms": round(st.gpu_ms, 1),
                "container_ms": round(st.container_ms, 1), "setup_ms": round(st.setup_ms, 1), "rounds": st.rounds}
    import torch
    multi = torch.cuda.device_count() > 1
    modes = (["all"] if have_ref else []) + ["native"]
    for m in modes:  # warm-up
        timed(m)
    for p in range(args.pairs):
        for m in modes:
            print(json.dumps(dict(timed(m), pair=p)), flush=True)
        if multi:
            print(json.dumps(dict(timed("native", pkg.MZ_ZIP_CUDA_ALL_DEVICES), pair=p)), flush=True)
    pair.close()
    lib.mz_zip_cuda_trim()


if __name__ == "__main__":
    main()
