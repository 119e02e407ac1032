"""The deflate kernel's exact output, pinned: SHA-256 of the streams the kernel SOURCES write on the CPU emulator for fixed
seeded inputs, at every level, as independent chunks and as one stream (MZ_CUDA_FLAG_DICT), against digests committed in
tests/golden/deflate_digests.json.

Changes that only make the kernel faster must leave every digest as it is. A change that is meant to alter the encoder's
output regenerates the file (python tests/test_emu_deflate_digests.py --write) and says why.
"""
import hashlib
import json
import os
import subprocess
import sys
import zlib

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import datagen  # noqa: E402

DIGESTS = os.path.join(HERE, "golden", "deflate_digests.json")
LEVELS = range(10)
FLAGS = {"chunks": 1, "stream": 3}  # FINAL, FINAL | DICT


def inputs():
    """name -> bytes. The bench text comes from the host generator (the same bytes as the bench's device generator, seed 1000)."""
    import textgen
    text = textgen.host(3 * 65536 + 12345, seed=1000)
    runs = b"".join(bytes([c]) * n for c, n in ((0, 40000), (0x41, 3), (0x20, 70001), (0, 258), (7, 259), (0, 33000)))
    periods = b"".join((p * (n // len(p) + 1))[:n] for p, n in ((b"ab", 20001), (b"abc", 30000), (b"\x00\x00\x01\x00", 25000),
                                                                 (b"0123456", 9000), (datagen.random_bytes(30000, 41), 95000)))
    return {"text": text, "runs": runs, "periods": periods, "traps": datagen.near_period_traps()}


def digests(emu):
    out = {}
    for name, data in inputs().items():
        for level in LEVELS:
            for mode, flags in FLAGS.items():
                comp, _ = emu.deflate(data, level=level, final=flags)
                assert zlib.decompress(comp, -15) == data, (name, level, mode)
                out["%s/%d/%s" % (name, level, mode)] = [len(comp), hashlib.sha256(comp).hexdigest()]
    return out


def _emu():
    r = subprocess.run(["make", "-s"], cwd=os.path.join(HERE, "emu"), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    import emushim
    return emushim.EmuLib()


def test_emu_deflate_digests(built):
    want = json.load(open(DIGESTS))
    got = digests(_emu())
    assert sorted(got) == sorted(want)
    diff = {k: (want[k], got[k]) for k in want if want[k] != got[k]}
    assert not diff, diff


if __name__ == "__main__":
    if sys.argv[1:] != ["--write"]:
        sys.exit("usage: test_emu_deflate_digests.py --write   (after __graft_entry__.build())")
    sys.path.insert(0, os.path.dirname(HERE))
    d = digests(_emu())
    with open(DIGESTS, "w") as f:
        f.write("{\n" + ",\n".join('"%s": %s' % (k, json.dumps(d[k])) for k in sorted(d)) + "\n}\n")
    print("wrote %d digests to %s" % (len(d), DIGESTS))
