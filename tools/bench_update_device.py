"""Times mz_zip_cuda_update_device against mz_zip_cuda_write_device of the same final entry set, in one process. The source is the C4
archive (`--entries` x `--entry-bytes`, 70 % text-like / 20 % records / 10 % incompressible, level 6) written by write_device into HBM,
every entry a distinct copy of one of a hundred blobs. Three workloads:
  (a) append `--append` new entries in place (the source buffer has room behind it; each timed call starts from a fresh copy of the
      source, restored outside the timed window);
  (b) the same append into a separate buffer;
  (c) drop every 100th entry and append `--append`, into a separate buffer.
Before anything is timed, (b) and (c) must be byte-identical to write_device's archive of the same entries, and (a) to (b). Then, after
one warm-up of each, `--pairs` rounds alternate each workload with write_device of its final set. Each time is a host clock around a
call that synchronises before it returns; stats are the calls' own. The kept-entry copy of (c) is also timed alone with CUDA events.

    python tools/bench_update_device.py [--entries 100000] [--entry-bytes 65536] [--append 1000] [--level 6] [--pairs 3]
"""
import argparse
import ctypes as C
import json
import os
import statistics
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
    ap.add_argument("--append", type=int, default=1000)
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
    n, eb, na, lv = args.entries, args.entry_bytes, args.append, args.level
    gens = [datagen.text_like] * 7 + [datagen.binary_records] * 2 + [datagen.random_bytes]
    blobs = [gens[k % 10](eb, seed=k)[:eb] for k in range(100)]
    pool = torch.frombuffer(bytearray(b"".join(blobs)), dtype=torch.uint8).cuda().view(100, eb)
    # entries 0..n-1 are the source's, n..n+na-1 the new ones: distinct copies in HBM
    data = pool.repeat((n + na + 99) // 100, 1)[:n + na].contiguous().view(-1)
    date = pkg.dos_date(1700000000)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def table(ids):
        names = [("e/%06d" % i).encode() for i in ids]
        items = (pkg.ZipDevItem * max(1, len(ids)))()
        pos = 0
        for k, i in enumerate(ids):
            items[k] = pkg.ZipDevItem(i * eb, eb, pos, len(names[k]), date, 0, 0)
            pos += len(names[k])
        return (torch.frombuffer(bytearray(b"".join(names) or b"\0"), dtype=torch.uint8).cuda(),
                torch.frombuffer(bytearray(bytes(items)), dtype=torch.uint8).cuda(), len(ids))

    def write(tab, out=None):
        d_names, d_items, k = tab
        alen = C.c_uint64(0)
        a = (data.data_ptr(), d_names.data_ptr(), d_items.data_ptr(), k, lv, 0, None, 0)
        if out is None:
            pkg.check(lib.mz_zip_cuda_write_device(*a, None, 0, C.byref(alen), None, None, stream), "sizing")
            out = torch.empty(alen.value, dtype=torch.uint8, device="cuda")
        st = pkg.ZipStats()
        t0 = time.perf_counter()
        err = lib.mz_zip_cuda_write_device(*a, out.data_ptr(), out.numel(), C.byref(alen), None, C.byref(st), stream)
        dt = time.perf_counter() - t0
        assert err == 0, err
        return out, alen.value, dt, st

    def update(src, src_len, keep, tab, out):
        d_names, d_items, k = tab
        alen = C.c_uint64(0)
        st = pkg.ZipStats()
        t0 = time.perf_counter()
        err = lib.mz_zip_cuda_update_device(src.data_ptr(), src_len, keep.data_ptr() if keep is not None else None, keep.numel() if keep is not None else 0,
                                            data.data_ptr(), d_names.data_ptr(), d_items.data_ptr(), k, lv, 0, None, 0, out.data_ptr(), out.numel(),
                                            C.byref(alen), None, C.byref(st), stream)
        dt = time.perf_counter() - t0
        assert err == 0, err
        return alen.value, dt, st

    new = table(range(n, n + na))
    src, src_len, _, _ = write(table(range(n)))
    kept_ids = [i for i in range(n) if i % 100 != 99]
    keep_c = torch.tensor(kept_ids, dtype=torch.int32, device="cuda")
    ref_ab, len_ab, _, _ = write(table(list(range(n)) + list(range(n, n + na))))
    ref_c, len_c, _, _ = write(table(kept_ids + list(range(n, n + na))))
    out_b = torch.empty(len_ab + (1 << 20), dtype=torch.uint8, device="cuda")
    out_c = torch.empty(len_c + (1 << 20), dtype=torch.uint8, device="cuda")
    inplace = torch.empty(len_ab + (1 << 20), dtype=torch.uint8, device="cuda")

    def reset_inplace():
        inplace[:src_len].copy_(src[:src_len])
        torch.cuda.synchronize()

    # byte identity before timing (and the warm-up of every call)
    lb, _, _ = update(src, src_len, None, new, out_b)
    lc, _, _ = update(src, src_len, keep_c, new, out_c)
    reset_inplace()
    la, _, _ = update(inplace, src_len, None, new, inplace)
    assert lb == len_ab and torch.equal(out_b[:lb], ref_ab[:len_ab]), "(b) differs from write_device"
    assert lc == len_c and torch.equal(out_c[:lc], ref_c[:len_c]), "(c) differs from write_device"
    assert la == len_ab and torch.equal(inplace[:la], ref_ab[:len_ab]), "(a) differs from write_device"
    print("# source: %d entries x %d bytes, level %d, archive %.1f MiB; append %d entries; GPU: %s (name, power limit, SM clock, max SM clock)"
          % (n, eb, lv, src_len / 2**20, na, gpu_info()), flush=True)
    print("# identical to write_device: (a) %d bytes, (b) %d bytes, (c) %d bytes" % (la, lb, lc), flush=True)
    full_ab, full_c = table(list(range(n)) + list(range(n, n + na))), table(kept_ids + list(range(n, n + na)))
    times = {}

    def rec(mode, dt, st):
        times.setdefault(mode, []).append(dt)
        print(json.dumps({"mode": mode, "ms": round(dt * 1e3, 2), "pack_ms": round(st.pack_ms, 2), "gpu_ms": round(st.gpu_ms, 2),
                          "setup_ms": round(st.setup_ms, 2), "rounds": st.rounds}), flush=True)
    for p in range(args.pairs):
        reset_inplace()
        _, dt, st = update(inplace, src_len, None, new, inplace)
        rec("a_append_in_place", dt, st)
        _, _, dt, st = write(full_ab, ref_ab)
        rec("write_device_ab", dt, st)
        _, dt, st = update(src, src_len, None, new, out_b)
        rec("b_append", dt, st)
        _, _, dt, st = write(full_ab, ref_ab)
        rec("write_device_ab", dt, st)
        _, dt, st = update(src, src_len, keep_c, new, out_c)
        rec("c_drop_and_append", dt, st)
        _, _, dt, st = write(full_c, ref_c)
        rec("write_device_c", dt, st)
    for mode, v in times.items():
        print(json.dumps({"summary": mode, "median_ms": round(statistics.median(v) * 1e3, 2), "min_ms": round(min(v) * 1e3, 2),
                          "max_ms": round(max(v) * 1e3, 2), "n": len(v)}), flush=True)
    # the kept-entry copy of (c) alone (K13 counts, then the copy kernel timed by CUDA events): bytes read + written over its time
    ent = torch.empty(n * 72, dtype=torch.uint8, device="cuda")
    cnt = C.c_uint32(0)
    nb = C.c_uint64(0)
    pkg.check(lib.mz_zip_cuda_extract_device(src.data_ptr(), src_len, None, ent.data_ptr(), n, C.byref(cnt), None, 0, C.byref(nb), None, stream), "list")
    rows = (pkg.ZipDevEntry * n).from_buffer_copy(ent.cpu().numpy().tobytes())
    moved = sum(rows[i].extent for i in kept_ids)
    m = len(kept_ids)
    tiles = m // 2048 + 1
    scratch = torch.empty((2 * (m + 1) + tiles) * 40 + 64, dtype=torch.uint8, device="cuda")
    from test_emu_device_update import ZipUp
    u = ZipUp()
    u.src, u.ent, u.count, u.n, u.keep = src.data_ptr(), ent.data_ptr(), n, m, keep_c.data_ptr()
    u.dir, u.dir_off, u.src_len = src.data_ptr(), 0, src_len
    base = scratch.data_ptr()
    u.cnt, u.pre, u.part, u.info = base, base + (m + 1) * 40, base + 2 * (m + 1) * 40, base + (2 * (m + 1) + tiles) * 40
    u.archive, u.cap, u.cd_off, u.entries = out_c.data_ptr(), out_c.numel(), 0, None
    # the records' directory reads need dir = the source's directory: take it from the first row's record
    cd_off = min(r.name_off for r in rows) - 46
    u.dir, u.dir_off = src.data_ptr() + cd_off, cd_off
    lib.mz_cuda_memset(u.info, 0xff, 48, stream)
    pkg.check(lib.mz_cuda_zip_up_counts(C.byref(u), stream), "counts")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ms = []
    for _ in range(5):
        ev[0].record()
        pkg.check(lib.mz_cuda_zip_up_copy(C.byref(u), stream), "copy")
        ev[1].record()
        torch.cuda.synchronize()
        ms.append(ev[0].elapsed_time(ev[1]))
    assert torch.equal(out_c[:moved], ref_c[:moved]), "copy kernel output differs"
    print(json.dumps({"mode": "c_copy_kernel_only", "bytes_moved": moved, "median_ms": round(statistics.median(ms), 3),
                      "GB_per_s_read_plus_write": round(2 * moved / 1e9 / (statistics.median(ms) / 1e3), 1)}), flush=True)
    lib.mz_zip_cuda_trim()


if __name__ == "__main__":
    main()
