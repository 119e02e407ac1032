#!/usr/bin/env python3
"""Where the deflate kernel's cycles go, per phase, on the GPU: runs the instrumented library (minizip-ng_b200/
libmz_strm_cuda_phases.so, built by `make -C minizip-ng_b200/csrc phases`: deflate_kernel.cuh with -DMZ_DF_PHASES) on the bench
text with the C5 launch (64 KiB chunks, one launch over the whole buffer, 2 CTAs per SM) and prints SM cycles per 32 KiB unit
and each phase's share, with the GPU's name, power limit and SM clock. D (the code construction) is split further at its named
barriers: stats, the two sweeps, Kraft completion (with the number of units per pass count), canonical codes, and the header. The
parse is split at the two barriers of each batch: (a) loads, hashes and the reads of the table before the batch's inserts, (b) the
inserts, (c) thread 0's reads after the inserts, verification, walk and record stores. M0 is split into thread 0's time in the
capped-span index, the near-source test and the extension; the rest of M0 is the wait for the other warps. The count-and-emit
pass is split at its barrier per pair of batches: (i) code words, span sizes and the warp scan up to the barrier, (ii) thread
0's emit of the pair, (iii) M3; the rest is the stored decision, the end-of-block code and the wait at the pass's closing barrier.

The counters are thread 0's clock64() readings at the kernel's barriers, summed per CTA; cycles per unit = all CTAs' cycles over
all units. The counting itself costs a few atomics per unit, so the kernel time printed here is not the product's.
  python tools/deflate_phases.py [--gib 2] [--level 1] [--reps 3] [--json OUT]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
PHASES = ["load + hash reset", "parse batches", "M0", "cover", "T + M1", "D (codes + header)", "E + F + M3 (count, emit)", "flush"]
UNITS = len(PHASES)  # column layout of g_df_phases (deflate_kernel.cuh): the phases, the unit count, D's sub-phases, the pass counts
D_SUB = ["stats", "sweep 1", "sweep 2", "Kraft completion", "canonical codes"]  # + "header": the rest of D
D_COL = PHASES.index("D (codes + header)")
NPASS = 8  # units whose Kraft completion ran 0, 1, .. 6, 7 or more passes
P_SUB = ["(a) loads, hashes, old keys", "(b) inserts", "(c) verify, walk, stores"]  # + "rest": the end of the last batch
P_COL = PHASES.index("parse batches")
M_SUB = ["index", "near-source test", "extension"]  # + "wait": the closing barrier
M_COL = PHASES.index("M0")
X_SUB = ["(i) code words, sizes, scan", "(ii) emit", "(iii) M3"]  # + "rest": the stored decision, the end of block, the last barrier
X_COL = PHASES.index("E + F + M3 (count, emit)")
SUB0 = UNITS + 1 + len(D_SUB) + NPASS
COLS = SUB0 + len(P_SUB) + len(M_SUB) + len(X_SUB)
ROWS = 1024


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], stdout=subprocess.PIPE, text=True, timeout=30)
        return dict(zip(q.split(","), [s.strip() for s in r.stdout.strip().split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=2.0)
    ap.add_argument("--level", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    import torch
    import __graft_entry__ as ge
    import textgen
    path = os.path.join(ROOT, "minizip-ng_b200", "libmz_strm_cuda_phases.so")
    if not os.path.exists(path):
        sys.exit("%s is missing: make -C minizip-ng_b200/csrc phases" % path)
    pkg = ge._load_pkg()
    lib = pkg.configure(C.CDLL(path))
    lib.mz_cuda_deflate_phases.restype = C.c_int32
    lib.mz_cuda_deflate_phases.argtypes = [C.c_void_p, C.c_uint32]
    torch.cuda.set_device(0)
    pkg.check(lib.mz_cuda_init(), "mz_cuda_init")

    chunk = 65536
    n = int(args.gib * (1 << 30)) // chunk * chunk
    nch = n // chunk
    src = torch.empty(n, dtype=torch.uint8, device="cuda")
    seg = 64 << 20
    for o in range(0, n, seg):  # the bench's text: one seed per 64 MiB segment
        textgen.device_into(src.data_ptr() + o, min(seg, n - o), 1000 + o // seg)
    stride = int(lib.mz_cuda_deflate_slot_bound(chunk))
    slots = torch.empty(nch * stride, dtype=torch.uint8, device="cuda")
    out_len = torch.empty(nch, dtype=torch.int32, device="cuda")
    rows = (C.c_uint64 * (ROWS * COLS))()

    def launch():
        pkg.check(lib.mz_cuda_deflate_chunks(src.data_ptr(), n, chunk, None, None, None, nch, pkg.FLAG_FINAL, args.level, slots.data_ptr(),
                                             stride, out_len.data_ptr(), pkg._stream_ptr()), "deflate")

    launch()  # warm-up
    pkg.check(lib.mz_cuda_deflate_phases(rows, ROWS), "phases")
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(args.reps):
        launch()
    ev1.record()
    torch.cuda.synchronize()
    info = gpu_info()  # right after the timed launches (the clock it reports is the current one)
    kms = ev0.elapsed_time(ev1) / args.reps
    pkg.check(lib.mz_cuda_deflate_phases(rows, ROWS), "phases")
    tab = [[rows[r * COLS + c] for c in range(COLS)] for r in range(ROWS)]
    tab = [r for r in tab if r[UNITS]]
    units = sum(r[UNITS] for r in tab)
    per = [sum(r[c] for r in tab) for c in range(len(PHASES))]
    total = sum(per)
    busiest = max(sum(r[:UNITS]) for r in tab) / args.reps
    dsub = [sum(r[UNITS + 1 + i] for r in tab) for i in range(len(D_SUB))]
    dsub.append(per[D_COL] - sum(dsub))
    psub = [sum(r[SUB0 + i] for r in tab) for i in range(len(P_SUB))]
    psub.append(per[P_COL] - sum(psub))
    msub = [sum(r[SUB0 + len(P_SUB) + i] for r in tab) for i in range(len(M_SUB))]
    msub.append(per[M_COL] - sum(msub))
    xsub = [sum(r[SUB0 + len(P_SUB) + len(M_SUB) + i] for r in tab) for i in range(len(X_SUB))]
    xsub.append(per[X_COL] - sum(xsub))
    passes = [sum(r[UNITS + 1 + len(D_SUB) + i] for r in tab) // args.reps for i in range(NPASS)]  # a CTA's cycles over the launch ~ kernel time x SM clock
    res = {"gpu": info.get("name"), "power_limit": info.get("power.limit"), "sm_clock_after": info.get("clocks.sm"),
           "sm_clock_max": info.get("clocks.max.sm"), "level": args.level, "bytes": n, "ctas": len(tab), "units": units // args.reps,
           "kernel_ms": round(kms, 3), "input_GBps": round(n / kms / 1e6, 1), "effective_sm_MHz": round(busiest / (kms * 1e3), 0),
           "ratio": round(int(out_len.sum().item()) / n, 4), "cycles_per_unit": round(total / units, 0),
           "phases": {p: {"cycles_per_unit": round(c / units, 0), "share": round(c / total, 4)} for p, c in zip(PHASES, per)},
           "d_subphases": {p: {"cycles_per_unit": round(c / units, 0), "share_of_d": round(c / max(per[D_COL], 1), 4)}
                           for p, c in zip(D_SUB + ["header"], dsub)},
           "parse_subphases": {p: {"cycles_per_unit": round(c / units, 0), "share_of_parse": round(c / max(per[P_COL], 1), 4)}
                               for p, c in zip(P_SUB + ["rest"], psub)},
           "m0_subphases": {p: {"cycles_per_unit": round(c / units, 0), "share_of_m0": round(c / max(per[M_COL], 1), 4)}
                            for p, c in zip(M_SUB + ["wait"], msub)},
           "emit_subphases": {p: {"cycles_per_unit": round(c / units, 0), "share_of_emit": round(c / max(per[X_COL], 1), 4)}
                              for p, c in zip(X_SUB + ["rest"], xsub)},
           "kraft_passes": {("%d+" % i if i == NPASS - 1 else str(i)): n for i, n in enumerate(passes)}}
    print("%s, power limit %s, SM clock %s (max %s); effective clock during the launches %d MHz" % (
        res["gpu"], res["power_limit"], res["sm_clock_after"], res["sm_clock_max"], res["effective_sm_MHz"]))
    print("level %d, %.2f GiB of bench text, 64 KiB chunks, %d CTAs, %d units: %.3f ms per launch (instrumented), ratio %.4f" % (
        args.level, n / (1 << 30), res["ctas"], res["units"], kms, res["ratio"]))
    print("%-30s %12s %7s" % ("phase", "cycles/unit", "share"))
    for p, c in zip(PHASES, per):
        print("%-30s %12.0f %6.1f%%" % (p, c / units, 100.0 * c / total))
        for col, names, sub, tag in ((D_COL, D_SUB + ["header"], dsub, "D"), (P_COL, P_SUB + ["rest"], psub, "parse"),
                                     (M_COL, M_SUB + ["wait"], msub, "M0"), (X_COL, X_SUB + ["rest"], xsub, "emit")):
            if p == PHASES[col]:
                for q, d in zip(names, sub):
                    print("  %-28s %12.0f %6.1f%% of %s" % (q, d / units, 100.0 * d / max(per[col], 1), tag))
    print("%-30s %12.0f" % ("total", total / units))
    print("units by Kraft completion passes: " + ", ".join("%s: %d" % kv for kv in res["kraft_passes"].items()))
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
