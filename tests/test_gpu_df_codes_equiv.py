"""GPU twin of test_emu_df_codes_equiv.py (pytest -m gpu): the deflate kernel's code builder against its frozen v3.4 form on the
same corpus, compiled for sm_90a (tests/emu/gpu_df_codes.cu). On the GPU __log2f is the approximate hardware log2 where the
emulator uses log2f, so this run is the one that sees a change in the floating-point path that decides the code lengths."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import test_emu_df_codes_equiv as m

pytestmark = pytest.mark.gpu


def nvcc():
    cand = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
    return cand if os.path.exists(cand) else shutil.which("nvcc")


@pytest.fixture(scope="module")
def gpu_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("gpu_df_codes") / "libgpu_df_codes.so")
    cmd = [nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
           "-I" + m.EMU, "-I" + m.SRC, "-o", out, os.path.join(m.EMU, "gpu_df_codes.cu")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    L = C.CDLL(out)
    L.gpu_df_out_words.restype = C.c_uint32
    L.gpu_df_codes_pair.restype = C.c_int
    L.gpu_df_codes_pair.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    return L


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    path, log = m.build(tmp_path_factory.mktemp("emu_df_codes"))
    assert path, log
    return m.load(path)


def test_gpu_code_builder_matches_v34_on_the_whole_corpus(gpu_lib, emu):
    h, posfin = m.corpus(emu)  # the captured histograms come from the kernel source on the emulator
    words = gpu_lib.gpu_df_out_words()
    old = np.zeros((len(h), words), dtype=np.uint32)
    new = np.zeros_like(old)
    assert gpu_lib.gpu_df_codes_pair(m.ptr(h), m.ptr(posfin), len(h), m.ptr(old), m.ptr(new)) == 0
    assert (old[:, 576] > 0).all()
    nbad, msgs = m.mismatches(h, old, new)
    assert nbad == 0, "%d of %d histograms differ on the GPU:\n%s" % (nbad, len(h), "\n".join(msgs))
