"""Times mz_zip_cuda_extract_device (archive and output in device memory, directory parsed on the device) against
mz_zip_cuda_extract_archive (the same bytes in a 64-bit memory base stream, directory parsed on the caller's thread), in one
process. The archive is the C4 shape of tools/bench_extract.py (entries x 64 KiB, 70 % text-like / 20 % records / 10 %
incompressible, level 6, written by the product's native writer); it is uploaded once. Before anything is printed, both extractors must
have produced the same CRC list and the same SHA-256 over the concatenated plain bytes (that pass hashes in the callback). Then,
after one warm-up of each, `--pairs` rounds alternate: the device call list-only, the device call with full decode,
extract_archive with a callback that only counts the entries (as tools/bench_extract.py's does). Each time is a host clock around
work that ends in a synchronise (both calls synchronise before they return). A second archive of --empty empty STORE entries (zip64 end records) times the
directory parse alone (CUDA events around list-only calls: K10 and its few readbacks).

    python tools/bench_extract_device.py [--entries 100000] [--entry-bytes 65536] [--pairs 3] [--empty 1000000]
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
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
    ap.add_argument("--empty", type=int, default=1_000_000)
    args = ap.parse_args()
    import torch
    import cuharness
    import datagen
    from test_emu_native_extract import Extractor
    pkg = cuharness.pkg()
    lib = pkg.load()
    pkg.check(lib.mz_cuda_init(), "mz_cuda_init")
    ex = Extractor(lib)

    def sink_bytes(m):  # archives past 2 GiB
        p = C.c_void_p()
        n = ex.t.lib.mz_stream_mem64_get_buffer(m, C.byref(p))
        return bytes((C.c_char * n).from_address(p.value)) if n else b""
    ex.t.sink_bytes = sink_bytes
    gens = [datagen.text_like] * 7 + [datagen.binary_records] * 2 + [datagen.random_bytes]
    blobs = [gens[k % 10](args.entry_bytes, seed=k) for k in range(100)]  # a hundred distinct entries, repeated
    archive = ex.write([("e/%06d" % i, blobs[i % 100]) for i in range(args.entries)], level=6)
    dev = torch.frombuffer(bytearray(archive), dtype=torch.uint8).cuda()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    count, nbytes = C.c_uint32(0), C.c_uint64(0)
    err = lib.mz_zip_cuda_extract_device(dev.data_ptr(), len(archive), None, None, 0, C.byref(count), None, 0, C.byref(nbytes), None, stream)
    assert err == pkg.MZ_BUF_ERROR and count.value == args.entries, err
    table = torch.empty(count.value * C.sizeof(pkg.ZipDevEntry), dtype=torch.uint8, device="cuda")
    out = torch.empty(nbytes.value, dtype=torch.uint8, device="cuda")

    def device_call(decode):
        st = pkg.ZipStats()
        t0 = time.perf_counter()
        err = lib.mz_zip_cuda_extract_device(dev.data_ptr(), len(archive), None, table.data_ptr(), count.value, C.byref(count),
                                             out.data_ptr() if decode else None, nbytes.value, C.byref(nbytes), C.byref(st), stream)
        dt = time.perf_counter() - t0
        assert err == 0, err
        return dt, st

    crcs, h, delivered = [], hashlib.sha256(), [0]

    def on_entry_verify(_ud, _name, data, size, crc):  # the verification pass: every CRC and every plain byte
        crcs.append(crc)
        h.update(C.string_at(data, size) if size else b"")
        return 0

    def on_entry_count(_ud, _name, _data, _size, _crc):  # the timed rounds: the bytes are dropped, as bench_extract.py does
        delivered[0] += 1
        return 0
    cb_verify, cb_count = pkg.ZIP_ENTRY_CB(on_entry_verify), pkg.ZIP_ENTRY_CB(on_entry_count)
    src, keep = ex.t.source(archive)

    def archive_call(cb):
        st = pkg.ZipStats()
        delivered[0] = 0
        t0 = time.perf_counter()
        err = lib.mz_zip_cuda_extract_archive(src, None, 0, cb, None, C.byref(st))
        dt = time.perf_counter() - t0
        assert err == 0, err
        return dt, st
    # equality of the two extractors' results (and warm-up of both)
    archive_call(cb_verify)
    want_crc, want_sha = crcs, h.digest()
    device_call(True)
    rows = (pkg.ZipDevEntry * count.value).from_buffer_copy(table.cpu().numpy().tobytes())
    host = out.cpu().numpy().tobytes()
    assert [r.crc for r in rows] == want_crc and all(r.status == 0 for r in rows)
    assert hashlib.sha256(b"".join(host[r.out_off:r.out_off + r.usize] for r in rows)).digest() == want_sha
    plain = sum(r.usize for r in rows)
    print("# archive: %d entries, %.1f MiB stored, %.1f MiB plain; GPU: %s (name, power limit, SM clock, max SM clock); host cores: %d"
          % (args.entries, len(archive) / 2**20, plain / 2**20, gpu_info(), os.cpu_count()), flush=True)
    print("# both extractors: the same %d CRCs and SHA-256 %s over the plain bytes" % (len(want_crc), want_sha.hex()[:16]), flush=True)
    device_call(False)
    archive_call(cb_count)
    for p in range(args.pairs):
        for mode in ("device_list", "device_decode", "extract_archive"):
            if mode == "extract_archive":
                dt, st = archive_call(cb_count)
                assert delivered[0] == args.entries
            else:
                dt, st = device_call(mode == "device_decode")
            print(json.dumps({"pair": p, "mode": mode, "s": round(dt, 4), "entries_per_s": round(args.entries / dt),
                              "GiB_per_s": round(plain / 2**30 / dt, 3) if mode != "device_list" else None, "pack_ms": round(st.pack_ms, 2), "container_ms": round(st.container_ms, 2),
                              "gpu_ms": round(st.gpu_ms, 2), "setup_ms": round(st.setup_ms, 2)}), flush=True)
    ex.t.delete(src)
    del keep
    lib.mz_zip_cuda_trim()
    # the directory parse at scale: list-only calls on a directory of empty STORE entries, timed with CUDA events
    if args.empty:
        from test_gpu_device_extract import empty_entries_archive
        big = empty_entries_archive(args.empty)
        dbig = torch.frombuffer(bytearray(big), dtype=torch.uint8).cuda()
        n2, b2 = C.c_uint32(0), C.c_uint64(0)
        lib.mz_zip_cuda_extract_device(dbig.data_ptr(), len(big), None, None, 0, C.byref(n2), None, 0, C.byref(b2), None, stream)
        t2 = torch.empty(n2.value * C.sizeof(pkg.ZipDevEntry), dtype=torch.uint8, device="cuda")
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        times = []
        for k in range(6):
            ev[0].record()
            err = lib.mz_zip_cuda_extract_device(dbig.data_ptr(), len(big), None, t2.data_ptr(), n2.value, C.byref(n2), None, 0, C.byref(b2), None, stream)
            ev[1].record()
            torch.cuda.synchronize()
            assert err == 0 and n2.value == args.empty, err
            if k:
                times.append(ev[0].elapsed_time(ev[1]))
        print(json.dumps({"mode": "parse_only_empty_entries", "entries": args.empty, "archive_MiB": round(len(big) / 2**20, 1),
                          "ms": [round(t, 3) for t in times], "entries_per_s": round(args.empty / (min(times) / 1e3))}), flush=True)


if __name__ == "__main__":
    main()
