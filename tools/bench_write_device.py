"""Times mz_zip_cuda_write_device (entries and archive in device memory, headers and directory built on the device) against
mz_zip_cuda_write_archive (the same entries from host memory into a 64-bit memory base stream), in one process. The entries are the C4
shape of tools/bench_extract.py: `--entries` x `--entry-bytes`, 70 % text-like / 20 % records / 10 % incompressible, level 6. On the
device every entry is a distinct copy in HBM (100 000 x 64 KiB = 6.1 GiB: a hundred repeated blobs would sit in L2); the host writer
reads the hundred host blobs the copies were made from. Before anything is timed both writers must produce identical bytes. Then,
after one warm-up of each, `--pairs` rounds alternate the two calls. Each time is a host clock around a call that synchronises before
it returns; stats are the calls' own.

    python tools/bench_write_device.py [--entries 100000] [--entry-bytes 65536] [--level 6] [--pairs 3]
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--entries", type=int, default=100_000)
    ap.add_argument("--entry-bytes", type=int, default=65536)
    ap.add_argument("--level", type=int, default=6)
    ap.add_argument("--pairs", type=int, default=3)
    args = ap.parse_args()
    import torch
    import cuharness
    import datagen
    from bench_extract_device import gpu_info
    pkg = cuharness.pkg()
    lib = pkg.load()
    pkg.check(lib.mz_cuda_init(), "mz_cuda_init")
    t = cuharness.TestLib()
    n, eb = args.entries, args.entry_bytes
    gens = [datagen.text_like] * 7 + [datagen.binary_records] * 2 + [datagen.random_bytes]
    blobs = [gens[k % 10](eb, seed=k)[:eb] for k in range(100)]
    names = [("e/%06d" % i).encode() for i in range(n)]
    date = 1700000000
    # host items: the hundred blobs
    keep = [C.create_string_buffer(b, len(b)) for b in blobs]
    hitems = (pkg.ZipItem * n)()
    for i in range(n):
        hitems[i] = pkg.ZipItem(names[i], C.cast(keep[i % 100], C.c_void_p), eb, date, 0, 0)
    # device entries: distinct copies, packed
    src = torch.frombuffer(bytearray(b"".join(blobs)), dtype=torch.uint8).cuda().view(100, eb)
    data = src.repeat((n + 99) // 100, 1)[:n].contiguous().view(-1)
    blob = b"".join(names)
    d_names = torch.frombuffer(bytearray(blob), dtype=torch.uint8).cuda()
    ditems = (pkg.ZipDevItem * n)()
    pos = 0
    for i in range(n):
        ditems[i] = pkg.ZipDevItem(i * eb, eb, pos, len(names[i]), pkg.dos_date(date), 0, 0)
        pos += len(names[i])
    d_items = torch.frombuffer(bytearray(bytes(ditems)), dtype=torch.uint8).cuda()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    alen = C.c_uint64(0)
    dargs = (data.data_ptr(), d_names.data_ptr(), d_items.data_ptr(), n, args.level, 0, None, 0)
    pkg.check(lib.mz_zip_cuda_write_device(*dargs, None, 0, C.byref(alen), None, None, stream), "sizing")
    arc = torch.empty(alen.value, dtype=torch.uint8, device="cuda")

    def device_call():
        st = pkg.ZipStats()
        t0 = time.perf_counter()
        err = lib.mz_zip_cuda_write_device(*dargs, arc.data_ptr(), arc.numel(), C.byref(alen), None, C.byref(st), stream)
        dt = time.perf_counter() - t0
        assert err == 0, err
        return dt, st

    def host_call(keep_bytes=False):
        sink = t.sink()
        st = pkg.ZipStats()
        t0 = time.perf_counter()
        err = lib.mz_zip_cuda_write_archive(sink, hitems, n, args.level, 0, C.byref(st))
        dt = time.perf_counter() - t0
        assert err == 0, err
        out = None
        if keep_bytes:
            p = C.c_void_p()
            k = t.lib.mz_stream_mem64_get_buffer(sink, C.byref(p))
            out = hashlib.sha256((C.c_char * k).from_address(p.value)).hexdigest(), k
        t.delete(sink)
        return dt, st, out
    # identical bytes (and the warm-up of both)
    _, _, (want_sha, want_len) = host_call(True)
    device_call()
    got = arc[:alen.value].cpu().numpy().tobytes()
    assert len(got) == want_len and hashlib.sha256(got).hexdigest() == want_sha, "the two writers differ"
    del got
    plain = n * eb
    print("# %d entries x %d bytes, level %d: %.1f MiB plain, archive %.1f MiB; GPU: %s (name, power limit, SM clock, max SM clock); host cores: %d"
          % (n, eb, args.level, plain / 2**20, want_len / 2**20, gpu_info(), os.cpu_count()), flush=True)
    print("# both writers: identical %d bytes, SHA-256 %s" % (want_len, want_sha[:16]), flush=True)
    for p in range(args.pairs):
        for mode in ("write_device", "write_archive"):
            if mode == "write_device":
                dt, st = device_call()
            else:
                dt, st, _ = host_call()
            print(json.dumps({"pair": p, "mode": mode, "s": round(dt, 4), "GiB_per_s": round(plain / 2**30 / dt, 3), "rounds": st.rounds,
                              "pack_ms": round(st.pack_ms, 2), "gpu_ms": round(st.gpu_ms, 2), "container_ms": round(st.container_ms, 2),
                              "setup_ms": round(st.setup_ms, 2)}), flush=True)
    # where the device call's time goes: the deflate kernel alone over the same chunks, CUDA events
    slots = torch.empty(16384 * int(lib.mz_cuda_deflate_slot_bound(65536)), dtype=torch.uint8, device="cuda")
    out_len = torch.empty(16384, dtype=torch.int32, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ms = 0.0
    ev[0].record()
    for c0 in range(0, n * eb // 65536, 16384):
        k = min(16384, n * eb // 65536 - c0)
        pkg.check(lib.mz_cuda_deflate_chunks(data.data_ptr() + c0 * 65536, k * 65536, 65536, None, None, None, k, 1, args.level, slots.data_ptr(),
                                             int(lib.mz_cuda_deflate_slot_bound(65536)), out_len.data_ptr(), stream), "deflate")
    ev[1].record()
    torch.cuda.synchronize()
    ms = ev[0].elapsed_time(ev[1])
    print(json.dumps({"mode": "deflate_only_same_chunks", "ms": round(ms, 2), "GiB_per_s": round(plain / 2**30 / (ms / 1e3), 3)}), flush=True)
    lib.mz_zip_cuda_trim()


if __name__ == "__main__":
    main()
