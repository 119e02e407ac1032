"""The emulated kernels under seeded schedules with the shared-memory race checker (tests/emu/cuda_emu.h: MZ_EMU_SCHED, MZ_EMU_RACE).

The default emulator schedule runs one interleaving: fibers in tid order, each to its next barrier, CTAs in blockIdx order,
shared memory filled with one constant. A missing barrier, a dependence on CTA order or a read of shared memory nobody wrote
gives the same answer under it every time. Here:
- toy kernels with one planted defect each (tests/emu/emu_sched_selftest.cc) must be reported by the race checker or give
  output that differs between seeds, and their corrected twins must run clean with one output under every seed;
- every kernel family (tests/emu/sched_check.py: deflate, inflate / K6 / CRC-32 / SHA-256, the phase-D code builder, the join
  and CRC segments, and K8 / K9 / K10 through the product library) runs under a few fixed seeds, each in its own process with
  the race checker on, and must match its references and the default schedule's output exactly.
More seeds by hand: python tests/emu/sched_check.py --seeds N [--full].

The race checker sees shared memory only through the Smem accessors and the emulated atomics, so it covers mainly the deflate
kernel (and the shared atomics of phase D and of the K6 candidate count). Kernels whose shared state goes mainly through raw
pointers or static __shared__ arrays are covered by the poisoning and the schedules alone: inflate (K5 tables and windows), the
K6 kernels, the CRC-32 segments and fold, the length scan, SHA-256, K8 (AES tables) and K10 (block reductions)."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
EMU = os.path.join(HERE, "emu")
SRC = os.path.join(os.path.dirname(HERE), "minizip-ng_b200", "csrc")
sys.path.insert(0, EMU)
import sched_check  # noqa: E402

SEEDS = (1, 2, 3)  # the default suite's fixed seeds; more by hand through sched_check.py --seeds
SELFTEST_SEEDS = range(1, 9)
TOYS = ("no_sync", "plain_counter", "named_barrier_short", "syncwarp_mask", "unwritten_dynamic", "unwritten_static", "cta_order")
RACE = b"shared-memory race"

SELFTEST_SCRIPT = r"""
import ctypes as C, sys
L = C.CDLL(sys.argv[1])
out = (C.c_uint32 * 64)()
assert L.emu_selftest(sys.argv[2].encode(), int(sys.argv[3]), out) == 0
print(" ".join(str(v) for v in out))
"""


def env_for(seed, race):
    env = dict(os.environ)
    env.pop("MZ_EMU_SCHED", None)
    env.pop("MZ_EMU_RACE", None)
    if seed:
        env["MZ_EMU_SCHED"] = str(seed)
    if race:
        env["MZ_EMU_RACE"] = "1"
    return env


@pytest.fixture(scope="module")
def selftest_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu_sched") / "libemu_sched_selftest.so")
    cmd = [os.environ.get("CXX", "g++"), "-O1", "-g", "-fPIC", "-std=c++17", "-Wall", "-Wno-unused-function", "-Wno-unknown-pragmas",
           "-Wno-unused-variable", "-I" + EMU, "-I" + SRC, "-shared", "-o", out, os.path.join(EMU, "emu_sched_selftest.cc"),
           os.path.join(EMU, "cuda_emu.cc")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return out


def toy_runs(lib, toy, fixed):
    """(returncode, stdout, stderr) of the toy under the default schedule and under every self-test seed with the race checker"""
    def one(seed):
        r = subprocess.run([sys.executable, "-c", SELFTEST_SCRIPT, lib, toy, str(fixed)], env=env_for(seed, seed != 0),
                           stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=120)
        return r.returncode, r.stdout, r.stderr
    with ThreadPoolExecutor(os.cpu_count() or 1) as pool:
        return list(pool.map(one, [0] + list(SELFTEST_SEEDS)))


@pytest.mark.parametrize("toy", TOYS)
def test_planted_defect_is_reported_or_diverges(selftest_lib, toy):
    runs = toy_runs(selftest_lib, toy, 0)[1:]
    reported = [rc != 0 and RACE in err for rc, _, err in runs]
    outputs = {out for rc, out, _ in runs if rc == 0}
    assert all(rc == 0 or RACE in err for rc, _, err in runs), [err[-500:] for rc, _, err in runs if rc]
    assert any(reported) or len(outputs) > 1, "the planted defect went unnoticed under every seed"


@pytest.mark.parametrize("toy", TOYS)
def test_corrected_twin_is_silent(selftest_lib, toy):
    runs = toy_runs(selftest_lib, toy, 1)
    assert all(rc == 0 and not err for rc, _, err in runs), [err[-500:] for _, _, err in runs]
    assert len({out for _, out, _ in runs}) == 1


def test_race_report_names_launch_block_word_and_threads(selftest_lib):
    r = subprocess.run([sys.executable, "-c", SELFTEST_SCRIPT, selftest_lib, "syncwarp_mask", "0"], env=env_for(0, True),
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=120)
    assert r.returncode != 0 and RACE in r.stderr, r.stderr  # the default schedule runs into it too
    line = r.stderr.decode().splitlines()[0]
    for part in ("read then write", "launch 1", "block (0,0,0)", "dynamic shared word at byte offset 0x7c", "thread 30 (read)",
                 "thread 31 (plain write)"):
        assert part in line, line


@pytest.fixture(scope="module")
def emu_libs(built, tmp_path_factory):
    r = subprocess.run(["make", "-s", "-C", EMU, "libmzemu.so", "libmz_strm_emu.so"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    return str(tmp_path_factory.mktemp("sched_check_build"))


@pytest.mark.parametrize("part", sched_check.PARTS)
def test_kernels_under_seeded_schedules_with_race_checker(emu_libs, part, monkeypatch):
    monkeypatch.setenv("SCHED_CHECK_BUILD_DIR", emu_libs)
    rc, base = sched_check.run_part(part, 0, False, race=False)
    assert rc == 0, base[-3000:]
    with ThreadPoolExecutor(len(SEEDS)) as pool:
        runs = list(pool.map(lambda s: sched_check.run_part(part, s, False), SEEDS))
    for seed, (rc, out) in zip(SEEDS, runs):
        assert rc == 0, (seed, out[-3000:])
        assert out.splitlines()[-1] == base.splitlines()[-1], "seed %d: output differs from the default schedule's" % seed
