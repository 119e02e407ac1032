"""Times the device reader (mz_zip_cuda_reader_*: open once, locate by name, decode chosen entries) on the C4 archive of
tools/bench_extract_device.py (entries x 64 KiB, 70 % text-like / 20 % records / 10 % incompressible, level 6, written by the
product's native writer), held in HBM, in one process, against mz_zip_cuda_extract_device's full decode.

Before anything is timed, every batch's bytes are checked against extract_device's slices of the same entries by SHA-256, and
locate of every name must return its index. Then:
  - open: host clock around mz_zip_cuda_reader_open (directory parse and name index; synchronous), then close;
  - locate: CUDA events around one locate of `--names` names (enqueued only, no host synchronisation inside);
  - decode: random selections of each batch size (seeded, repeats allowed), host clock around the synchronous call, with the
    call's own split (to the first readback, device work);
  - extract_device full decode, alternating with the reader's rounds.
Each round runs every batch size once and extract_device once; medians and the spread over `--rounds` rounds are printed.

    python tools/bench_read_device.py [--entries 100000] [--entry-bytes 65536] [--rounds 5] [--names 100000]
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import random
import statistics
import struct
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
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--names", type=int, default=100_000)
    ap.add_argument("--sizes", default="1,64,256,1024,4096,16384,100000")
    args = ap.parse_args()
    import torch
    import cuharness
    import datagen
    from bench_extract_device import gpu_info
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
    blobs = [gens[k % 10](args.entry_bytes, seed=k) for k in range(100)]
    names = ["e/%06d" % i for i in range(args.entries)]
    archive = ex.write([(names[i], blobs[i % 100]) for i in range(args.entries)], level=6)
    dev = torch.frombuffer(bytearray(archive), dtype=torch.uint8).cuda()
    del archive
    alen = dev.numel()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    # extract_device: the reference slices
    count, nbytes = C.c_uint32(0), C.c_uint64(0)
    err = lib.mz_zip_cuda_extract_device(dev.data_ptr(), alen, None, None, 0, C.byref(count), None, 0, C.byref(nbytes), None, stream)
    assert err == pkg.MZ_BUF_ERROR and count.value == args.entries, err
    n = count.value
    table = torch.empty(n * C.sizeof(pkg.ZipDevEntry), dtype=torch.uint8, device="cuda")
    full = torch.empty(nbytes.value, dtype=torch.uint8, device="cuda")

    def extract_call():
        st = pkg.ZipStats()
        t0 = time.perf_counter()
        e = lib.mz_zip_cuda_extract_device(dev.data_ptr(), alen, None, table.data_ptr(), n, C.byref(count), full.data_ptr(), nbytes.value,
                                           C.byref(nbytes), C.byref(st), stream)
        dt = time.perf_counter() - t0
        assert e == 0, e
        return dt, st
    extract_call()
    rows = (pkg.ZipDevEntry * n).from_buffer_copy(table.cpu().numpy().tobytes())
    usize = [r.usize for r in rows]
    full_host = full.cpu().numpy()

    # the reader
    def open_reader():
        h, cnt, ref = C.c_void_p(), C.c_uint32(0), C.c_int32(0)
        st = pkg.ZipStats()
        t0 = time.perf_counter()
        e = lib.mz_zip_cuda_reader_open(dev.data_ptr(), alen, None, C.byref(h), C.byref(cnt), C.byref(ref), C.byref(st), stream)
        dt = time.perf_counter() - t0
        assert e == 0 and cnt.value == n and ref.value == 0, e
        return h, dt, st
    h, _, _ = open_reader()
    lib.mz_zip_cuda_reader_close(h)
    sizes = [int(s) for s in args.sizes.split(",") if int(s) <= n]
    rng = random.Random(12345)
    sels = {k: [rng.randrange(n) for _ in range(k)] if k < n else rng.sample(range(n), n) for k in sizes}
    d_sel = {k: torch.tensor(v, dtype=torch.int32, device="cuda") for k, v in sels.items()}
    out = torch.empty(nbytes.value + 16 * max(sizes), dtype=torch.uint8, device="cuda")
    offs = torch.empty(max(sizes) + 1, dtype=torch.int64, device="cuda")
    h, _, _ = open_reader()

    def decode_call(k):
        st = pkg.ZipStats()
        size = C.c_uint64(0)
        t0 = time.perf_counter()
        e = lib.mz_zip_cuda_reader_decode(h, d_sel[k].data_ptr(), k, out.data_ptr(), out.numel(), C.byref(size), offs.data_ptr(), None, C.byref(st), stream)
        dt = time.perf_counter() - t0
        assert e == 0, e
        return dt, st, size.value

    # correctness first: every batch against extract_device's slices, and locate of every name
    for k in sizes:
        _, _, total = decode_call(k)
        o = offs[:k + 1].cpu().tolist()
        got_host = out[:total].cpu().numpy()
        ha, hb = hashlib.sha256(), hashlib.sha256()
        for s, i in enumerate(sels[k]):
            ha.update(got_host[o[s]:o[s] + usize[i]])
            hb.update(full_host[rows[i].out_off:rows[i].out_off + usize[i]])
        assert ha.digest() == hb.digest(), k
    del full_host
    qn = min(args.names, n)
    qnames = [names[i].encode() for i in rng.sample(range(n), qn)]
    want_idx = [int(q[2:]) for q in qnames]
    blob = b"".join(qnames)
    d_names = torch.frombuffer(bytearray(blob), dtype=torch.uint8).cuda()
    d_off = torch.tensor([8 * i for i in range(qn)], dtype=torch.int64, device="cuda")
    assert all(len(q) == 8 for q in qnames)
    d_len = torch.full((qn,), 8, dtype=torch.int32, device="cuda")
    d_idx = torch.empty(qn, dtype=torch.int32, device="cuda")

    def locate_call():
        e = lib.mz_zip_cuda_reader_locate(h, d_names.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), qn, 0, d_idx.data_ptr(), stream)
        assert e == 0, e
    locate_call()
    assert d_idx.cpu().tolist() == want_idx
    plain = {k: sum(usize[i] for i in sels[k]) for k in sizes}
    print("# archive: %d entries, %.1f MiB stored, %.1f MiB plain; GPU: %s (name, power limit, SM clock, max SM clock)"
          % (n, alen / 2**20, sum(usize) / 2**20, gpu_info()), flush=True)
    print("# every batch equals extract_device's slices by SHA-256; locate of %d names returned their indices" % qn, flush=True)

    # timed
    lib.mz_zip_cuda_reader_close(h)
    opens = []
    for _ in range(args.rounds):
        h, dt, st = open_reader()
        opens.append((dt, st.pack_ms, st.gpu_ms))
        lib.mz_zip_cuda_reader_close(h)
    h, _, _ = open_reader()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    loc = []
    for _ in range(args.rounds):
        torch.cuda.synchronize()
        ev[0].record()
        locate_call()
        ev[1].record()
        torch.cuda.synchronize()
        loc.append(ev[0].elapsed_time(ev[1]))
    res = {k: [] for k in sizes}
    ext = []
    for k in sizes:  # warm-up of every shape
        decode_call(k)
    extract_call()
    for _ in range(args.rounds):
        for k in sizes:
            res[k].append(decode_call(k))
        ext.append(extract_call())
    print(json.dumps({"mode": "open", "s": [round(o[0], 4) for o in opens], "median_s": round(statistics.median(o[0] for o in opens), 4),
                      "parse_ms": [round(o[1], 2) for o in opens], "index_ms": [round(o[2], 2) for o in opens]}), flush=True)
    print(json.dumps({"mode": "locate", "names": qn, "ms": [round(t, 3) for t in loc], "median_ms": round(statistics.median(loc), 3),
                      "names_per_s": round(qn / (statistics.median(loc) / 1e3))}), flush=True)
    for k in sizes:
        ts = [r[0] for r in res[k]]
        med = statistics.median(ts)
        print(json.dumps({"mode": "decode", "entries": k, "s": [round(t, 4) for t in ts], "median_s": round(med, 4), "entries_per_s": round(k / med),
                          "GiB_per_s": round(plain[k] / 2**30 / med, 3), "to_readback_ms": round(statistics.median(r[1].pack_ms for r in res[k]), 3),
                          "device_ms": round(statistics.median(r[1].gpu_ms for r in res[k]), 3), "alloc_ms": round(max(r[1].setup_ms for r in res[k]), 3)}),
              flush=True)
    ts = [e[0] for e in ext]
    med = statistics.median(ts)
    print(json.dumps({"mode": "extract_device", "entries": n, "s": [round(t, 4) for t in ts], "median_s": round(med, 4), "entries_per_s": round(n / med),
                      "GiB_per_s": round(sum(usize) / 2**30 / med, 3), "decode_ms": [round(e[1].gpu_ms, 2) for e in ext],
                      "parse_ms": [round(e[1].pack_ms, 2) for e in ext]}), flush=True)
    lib.mz_zip_cuda_reader_close(h)
    lib.mz_zip_cuda_trim()


if __name__ == "__main__":
    main()
