"""Times mz_cuda_gzip_compress_device / mz_cuda_gzip_decompress_device (member and plain bytes in device memory) against the vtbl stream
with window bits 31 (mz_stream_cuda_write / _read from and to host memory through a 64-bit memory base stream) on the same bytes, in
one process:
  - compress of --c2-mib MiB of bench text at level 6 (C2's shape) and of --big-gib GiB at level 1;
  - decode of a foreign level-6 member of --c3-gib GiB of output (C3's shape; zlib-made, bench.make_gzip_member), with the device
    call's split: header readback, staging copy (scratch allocation included), K5 / K6 decode, CRC-32 and trailer.
Each shape first checks that the device call's output decodes (compress: its length and trailer; decode: CRC-32 and length against
the source), warms both arms up once, then alternates them for `--pairs` pairs. Times are host clocks around calls that synchronise
before they return. The GPU's name, power limit and SM clocks are printed with the results.

    python tools/bench_gzip_device.py [--c2-mib 256] [--big-gib 4] [--c3-gib 4] [--pairs 3]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

MZ_OPEN_MODE_READ, MZ_OPEN_MODE_WRITE = 1, 2
PROP_TOTAL_IN, PROP_COMPRESS_LEVEL, PROP_COMPRESS_WINDOW = 1, 9, 11


class Vtbl:
    """the vtbl stream with window bits 31 over a memory base, driven through tests/support/libmztest.so"""

    def __init__(self, lib):
        import cuharness
        self.lib = lib
        self.t = cuharness.TestLib()

    def compress(self, hbuf, n, level, piece=16384):  # hbuf: the input's host address
        T = self.t.lib
        sink = self.t.sink()
        s = self.lib.mz_stream_cuda_create()
        T.mzt_set_prop(s, PROP_COMPRESS_LEVEL, level)
        T.mzt_set_prop(s, PROP_COMPRESS_WINDOW, 31)
        T.mzt_set_base(s, sink)
        assert T.mzt_open(s, None, MZ_OPEN_MODE_WRITE) == 0
        t0 = time.perf_counter()
        wrote = T.mzt_write_all(s, hbuf, n, piece)
        err = T.mzt_close(s)
        dt = time.perf_counter() - t0
        assert wrote == n and err == 0, (wrote, err)
        p = C.c_void_p()
        k = T.mz_stream_mem64_get_buffer(sink, C.byref(p))
        self.t.delete(s)
        self.t.delete(sink)
        return dt, k

    def decompress(self, member, out, cap, piece=1 << 20):  # member, out: numpy uint8 arrays
        T = self.t.lib
        src = T.mz_stream_mem64_create()
        T.mz_stream_mem64_set_buffer(src, member.ctypes.data, member.size)
        s = self.lib.mz_stream_cuda_create()
        T.mzt_set_prop(s, PROP_COMPRESS_WINDOW, 31)
        T.mzt_set_base(s, src)
        assert T.mzt_open(s, None, MZ_OPEN_MODE_READ) == 0
        t0 = time.perf_counter()
        got = T.mzt_read_all(s, out.ctypes.data, cap, piece)
        dt = time.perf_counter() - t0
        _, total_in = self.t.get_prop(s, PROP_TOTAL_IN)
        T.mzt_close(s)
        self.t.delete(s)
        self.t.delete(src)
        return dt, got, total_in


def summary(xs):
    return {"median": round(statistics.median(xs), 4), "min": round(min(xs), 4), "max": round(max(xs), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--c2-mib", type=int, default=256)
    ap.add_argument("--big-gib", type=float, default=4)
    ap.add_argument("--c3-gib", type=float, default=4)
    ap.add_argument("--pairs", type=int, default=3)
    args = ap.parse_args()
    import torch
    import cuharness
    import textgen
    from bench import make_gzip_member
    from bench_extract_device import gpu_info
    pkg = cuharness.pkg()
    lib = pkg.load()
    pkg.check(lib.mz_cuda_init(), "mz_cuda_init")
    vt = Vtbl(lib)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    print("# GPU: %s (name, power limit, SM clock, max SM clock); host cores: %d" % (gpu_info(), os.cpu_count()), flush=True)
    results = []

    # ---- compress: C2's shape at level 6, a large buffer at level 1 ----
    for label, n, level in (("compress_c2", args.c2_mib << 20, 6), ("compress_big", int(args.big_gib * (1 << 30)), 1)):
        src = textgen.device(n, seed=1000 + level)
        host = src.cpu().numpy()  # the vtbl's input: the same bytes in (pageable) host memory
        hbuf = host.ctypes.data
        size = C.c_uint64(0)
        pkg.check(lib.mz_cuda_gzip_compress_device(src.data_ptr(), n, level, None, 0, C.byref(size), None, stream), "sizing")
        out = torch.empty(size.value, dtype=torch.uint8, device="cuda")

        def device_call():
            st = pkg.GzipStats()
            t0 = time.perf_counter()
            err = lib.mz_cuda_gzip_compress_device(src.data_ptr(), n, level, out.data_ptr(), out.numel(), C.byref(size), C.byref(st), stream)
            dt = time.perf_counter() - t0
            assert err == 0, err
            return dt, st
        device_call()
        tail = bytes(out[size.value - 8:size.value].cpu().numpy().tobytes())
        assert int.from_bytes(tail[:4], "little") == pkg.crc32_device(src) and int.from_bytes(tail[4:], "little") == n & 0xffffffff
        _, vlen = vt.compress(hbuf, n, level)
        print("# %s: %d bytes at level %d -> device member %d bytes, vtbl member %d bytes" % (label, n, level, size.value, vlen), flush=True)
        dev_s, vt_s = [], []
        for p in range(args.pairs):
            dt, st = device_call()
            dev_s.append(dt)
            print(json.dumps({"shape": label, "pair": p, "mode": "device", "s": round(dt, 4), "GiB_per_s": round(n / 2**30 / dt, 2), "rounds": st.rounds,
                              "header_ms": round(st.header_ms, 3), "work_ms": round(st.work_ms, 2), "crc_ms": round(st.crc_ms, 2),
                              "setup_ms": round(st.setup_ms, 2)}), flush=True)
            dt, _ = vt.compress(hbuf, n, level)
            vt_s.append(dt)
            print(json.dumps({"shape": label, "pair": p, "mode": "vtbl", "s": round(dt, 4), "GiB_per_s": round(n / 2**30 / dt, 2)}), flush=True)
        results.append({"shape": label, "bytes": n, "level": level, "device_s": summary(dev_s), "vtbl_s": summary(vt_s)})
        del src, out, host
        torch.cuda.empty_cache()

    # ---- decode: C3's shape, a foreign level-6 member ----
    n = int(args.c3_gib * (1 << 30))
    src = textgen.device(n, seed=3)
    crc = pkg.crc32_device(src)
    hsrc = src.cpu().numpy()
    member, mcrc = make_gzip_member(hsrc, n, level=6)
    assert mcrc == crc
    del hsrc
    hmember = np.frombuffer(member, dtype=np.uint8)
    d_member = torch.from_numpy(hmember.copy()).cuda()
    out = torch.empty(n, dtype=torch.uint8, device="cuda")
    hout = np.empty(n + 1, dtype=np.uint8)

    def device_decode():
        res, st = pkg.GzipResult(), pkg.GzipStats()
        t0 = time.perf_counter()
        err = lib.mz_cuda_gzip_decompress_device(d_member.data_ptr(), len(member), out.data_ptr(), n, C.byref(res), C.byref(st), stream)
        dt = time.perf_counter() - t0
        assert err == 0 and res.out_len == n and res.in_used == len(member) and res.crc == crc, (err, res.out_len, res.in_used)
        return dt, st
    device_decode()
    assert torch.equal(out, src)
    dt, got, total_in = vt.decompress(hmember, hout, n + 1)
    assert got == n and total_in == len(member), (got, total_in)
    print("# decode_c3: member %d bytes -> %d bytes (level 6, zlib)" % (len(member), n), flush=True)
    dev_s, vt_s, split = [], [], []
    for p in range(args.pairs):
        dt, st = device_decode()
        dev_s.append(dt)
        split.append(st)
        print(json.dumps({"shape": "decode_c3", "pair": p, "mode": "device", "s": round(dt, 4), "GiB_per_s": round(n / 2**30 / dt, 2),
                          "header_ms": round(st.header_ms, 3), "staging_ms": round(st.setup_ms, 2), "decode_ms": round(st.work_ms, 2),
                          "crc_ms": round(st.crc_ms, 2), "k5_launches": st.k5_launches, "k6_rounds": st.k6_rounds}), flush=True)
        dt, got, _ = vt.decompress(hmember, hout, n + 1)
        assert got == n
        vt_s.append(dt)
        print(json.dumps({"shape": "decode_c3", "pair": p, "mode": "vtbl", "s": round(dt, 4), "GiB_per_s": round(n / 2**30 / dt, 2)}), flush=True)
    results.append({"shape": "decode_c3", "bytes": n, "member": len(member), "device_s": summary(dev_s), "vtbl_s": summary(vt_s),
                    "header_ms": summary([s.header_ms for s in split]), "staging_ms": summary([s.setup_ms for s in split]),
                    "decode_ms": summary([s.work_ms for s in split]), "crc_ms": summary([s.crc_ms for s in split])})
    print(json.dumps({"gpu": gpu_info(), "results": results}), flush=True)


if __name__ == "__main__":
    main()
