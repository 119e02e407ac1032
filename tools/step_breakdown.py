#!/usr/bin/env python3
"""Where the time of one C5 step goes, per launch, on the GPU, set against the memory's measured floors.

Generates the bench's C5 input on one GPU (the bench text, one seed per 64 MiB segment, 16 GiB by default, 64 KiB chunks) and
issues the same launches as one bench step, with CUDA events between them:
    deflate | CRC segments | CRC fold | concat (exclusive scan of the lengths + join copy)
After the steps it times the join copy alone (mz_cuda_gather with the offsets concat produced), so scan = concat - gather.
In the same run it measures two practical floors: a device-to-device copy of the compressed size (cudaMemcpyAsync) and a
read-only pass over the input (a torch sum). Every launch is printed with its time, the bytes it must move, GB/s and, for
the two that only move bytes, its share of the matching floor (floor time over launch time). The GPU's name, power limit and
SM clock are printed with the numbers.

--lib PATH runs the same launches through another build of libmz_strm_cuda.so (e.g. an older commit's), so two builds can be
compared on the same GPU.
  python tools/step_breakdown.py [--gib 16] [--steps 5] [--warmup 2] [--lib PATH] [--json OUT]"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
CHUNK = 65536
LAUNCHES = ["deflate", "crc segments", "crc fold", "concat"]


def stats(v):
    return {"mean": round(sum(v) / len(v), 4), "min": round(min(v), 4), "max": round(max(v), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=16.0)
    ap.add_argument("--level", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--lib", default=None, help="another build of libmz_strm_cuda.so to run the launches through")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import torch
    import __graft_entry__ as ge
    import textgen
    from deflate_phases import gpu_info
    pkg = ge._load_pkg()
    if args.lib:  # every call below, DeflateBatch's and pkg.check's included, goes through this build
        pkg._lib = pkg.configure(C.CDLL(os.path.abspath(args.lib)))
    lib = pkg.load()
    torch.cuda.set_device(0)
    pkg.check(lib.mz_cuda_init(), "mz_cuda_init")

    n = int(args.gib * (1 << 30)) // CHUNK * CHUNK
    nch = n // CHUNK
    src = torch.empty(n, dtype=torch.uint8, device="cuda")
    seg = 64 << 20
    for o in range(0, n, seg):  # the bench's text: one seed per 64 MiB segment
        textgen.device_into(src.data_ptr() + o, min(seg, n - o), 1000 + o // seg)
    b = pkg.DeflateBatch(n)
    s = pkg._stream_ptr()
    stream = torch.cuda.current_stream()

    def step(ev=None):
        rec = (lambda i: ev[i].record(stream)) if ev else (lambda i: None)
        rec(0)
        pkg.check(lib.mz_cuda_deflate_chunks(src.data_ptr(), n, CHUNK, None, None, None, nch, pkg.FLAG_FINAL, args.level, b.slots.data_ptr(),
                                             b.stride, b.out_len.data_ptr(), s), "deflate")
        rec(1)
        pkg.check(lib.mz_cuda_crc32_segments(src.data_ptr(), n, CHUNK, None, None, nch, b.residue.data_ptr(), b.chunk_crc.data_ptr(), s), "crc")
        rec(2)
        pkg.check(lib.mz_cuda_crc32_fold(b.residue.data_ptr(), nch, CHUNK, n, b.crc_out.data_ptr(), s), "fold")
        rec(3)
        pkg.check(lib.mz_cuda_concat(b.slots.data_ptr(), b.stride, b.out_len.data_ptr(), nch, b.offsets.data_ptr(), b.joined.data_ptr(), s), "concat")
        rec(4)

    def timed(fn, reps):
        """ms per call of fn over `reps` calls, one event pair per call"""
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
        for a, z in evs:
            a.record(stream)
            fn()
            z.record(stream)
        torch.cuda.synchronize()
        return [a.elapsed_time(z) for a, z in evs]

    for _ in range(max(1, args.warmup)):
        step()
    torch.cuda.synchronize()
    evs = [[torch.cuda.Event(enable_timing=True) for _ in range(5)] for _ in range(args.steps)]
    for e in evs:
        step(e)
    torch.cuda.synchronize()
    info = gpu_info()  # right after the timed steps (the clock it reports is the current one)
    per = {name: [e[i].elapsed_time(e[i + 1]) for e in evs] for i, name in enumerate(LAUNCHES)}
    per["step"] = [e[0].elapsed_time(e[4]) for e in evs]
    comp = int(b.offsets[nch].item())
    reps = max(3, args.steps)
    per["gather"] = timed(lambda: pkg.check(lib.mz_cuda_gather(b.slots.data_ptr(), b.stride, b.out_len.data_ptr(), nch, b.offsets.data_ptr(),
                                                               b.joined.data_ptr(), s), "gather"), reps)
    per["scan"] = [c - g for c, g in zip(per["concat"], per["gather"])]
    # floors: what the memory does for a plain copy of the compressed size and a plain read of the input
    wide = src.view(torch.int64)
    timed(lambda: wide.sum(), 1)
    floor_read = timed(lambda: wide.sum(), reps)
    floor_copy = timed(lambda: pkg.check(lib.mz_cuda_memcpy_d2d(b.joined.data_ptr(), b.slots.data_ptr(), comp, s), "d2d"), reps)
    step()  # leave the joined stream as concat wrote it
    torch.cuda.synchronize()

    fr, fc = sum(floor_read) / reps, sum(floor_copy) / reps
    moved = {"deflate": n + comp, "crc segments": n, "crc fold": 4 * nch, "scan": 4 * nch + 8 * (nch + 1), "gather": 2 * comp,
             "concat": 4 * nch + 8 * (nch + 1) + 2 * comp}
    floor = {"crc segments": ("read", fr), "gather": ("copy", fc)}
    rows = {}
    for name in ["deflate", "crc segments", "crc fold", "scan", "gather", "concat"]:
        ms = sum(per[name]) / len(per[name])
        r = {"ms": stats(per[name]), "bytes": moved[name], "GBps": round(moved[name] / ms / 1e6, 1) if ms > 0 else None}
        if name in floor:
            r["floor"] = floor[name][0]
            r["share_of_floor"] = round(floor[name][1] / ms, 3)
        rows[name] = r
    after_deflate = [st - d for st, d in zip(per["step"], per["deflate"])]
    res = {"gpu": info.get("name"), "power_limit": info.get("power.limit"), "sm_clock_after": info.get("clocks.sm"),
           "sm_clock_max": info.get("clocks.max.sm"), "lib": os.path.abspath(args.lib) if args.lib else pkg.LIB_PATH, "level": args.level,
           "bytes": n, "chunks": nch, "compressed": comp, "ratio": round(comp / n, 4), "steps": args.steps, "step_ms": stats(per["step"]),
           "launches_2_5_ms": stats(after_deflate), "launches": rows,
           "floor_read": {"ms": round(fr, 4), "GBps": round(n / fr / 1e6, 1)}, "floor_copy": {"ms": round(fc, 4), "GBps": round(2 * comp / fc / 1e6, 1)}}
    print("%s, power limit %s, SM clock %s (max %s); %s" % (res["gpu"], res["power_limit"], res["sm_clock_after"], res["sm_clock_max"], res["lib"]))
    print("C5 step: %.2f GiB of bench text, level %d, %d chunks of 64 KiB, ratio %.4f; %d steps after %d warm-up" % (
        n / (1 << 30), args.level, nch, res["ratio"], args.steps, max(1, args.warmup)))
    print("floors: read %.3f ms (%.1f GB/s), copy of %d B %.3f ms (%.1f GB/s read + written)" % (
        fr, res["floor_read"]["GBps"], comp, fc, res["floor_copy"]["GBps"]))
    print("%-14s %10s %18s %14s %9s %9s" % ("launch", "ms", "min-max", "bytes", "GB/s", "of floor"))
    for name, r in rows.items():
        share = "%5.1f%% %s" % (100 * r["share_of_floor"], r["floor"]) if "floor" in r else ""
        print("%-14s %10.3f %8.3f-%-9.3f %14d %9s %s" % (name, r["ms"]["mean"], r["ms"]["min"], r["ms"]["max"], r["bytes"],
                                                        "%.1f" % r["GBps"] if r["GBps"] else "-", share))
    print("%-14s %10.3f %8.3f-%-9.3f" % ("step", res["step_ms"]["mean"], res["step_ms"]["min"], res["step_ms"]["max"]))
    print("%-14s %10.3f %8.3f-%-9.3f" % ("launches 2-5", res["launches_2_5_ms"]["mean"], res["launches_2_5_ms"]["min"], res["launches_2_5_ms"]["max"]))
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
