"""GPU twin of test_emu_deflate_audit.py (pytest -m gpu): what the sm_90a deflate kernel writes, block by block.

a. Every rule of tests/deflate_audit.py on the device's slots, for the emulator test's corpus, with chunk starts 16-byte aligned
   (the TMA bulk load) and unaligned (the plain load; both must give the same bytes). The code builder is the sm_90a one
   (tests/emu/gpu_df_codes.cu), where __log2f is the hardware approximation.
b. The same parse as the emulator, unit by unit: equal token lists where both code a unit, equal stored blocks where both store
   it, and where one side stores what the other codes, each side's choice follows the stored rule under its own builder (the
   histogram the emulator's builder was given judges the stored side). Blocks whose code lengths differ between the two
   builders (the effect of __log2f) are counted and printed, not asserted.
c. Under load: 256 MiB of the bench text and 64 MiB of mixed data at levels 1, 4, 6 and 6 as one stream. Two runs give the same
   lengths and bytes (the work counter hands chunks to other CTAs each time); 64 sampled chunks recompressed alone give the same
   bytes as in the big run and pass every rule. Each configuration runs twice, no more.
"""
import random

import numpy as np
import pytest

import deflate_audit as A
import test_emu_deflate_audit as E
import test_emu_df_codes_equiv as codes_equiv
from test_gpu_df_codes_equiv import emu, gpu_lib  # noqa: F401 (fixtures: the builders on the emulator and on sm_90a)

pytestmark = pytest.mark.gpu

LOAD_SAMPLE = 64


@pytest.fixture(scope="module")
def cu(built):
    import torch
    import cuharness
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    p = cuharness.pkg()
    lib = p.load()
    p.check(lib.mz_cuda_init(), "mz_cuda_init")
    return p, lib, torch


@pytest.fixture(scope="module")
def codes(emu):  # noqa: F811
    return E.with_capture(emu)


@pytest.fixture(scope="module")
def emushim_lib(built):
    return E.digests._emu()


@pytest.fixture(scope="module")
def corpus(codes):
    return E.corpus(codes)


def gpu_builder(L):
    def run(h, pf):
        h, pf = np.ascontiguousarray(h, dtype=np.uint32), np.ascontiguousarray(pf, dtype=np.uint32)
        old = np.zeros((len(h), L.gpu_df_out_words()), dtype=np.uint32)
        new = np.zeros_like(old)
        assert L.gpu_df_codes_pair(codes_equiv.ptr(h), codes_equiv.ptr(pf), len(h), codes_equiv.ptr(old), codes_equiv.ptr(new)) == 0
        return new
    return run


def to_device(torch, data, misalign=0):
    t = torch.zeros(len(data) + 16 + misalign, dtype=torch.uint8, device="cuda")
    if data:
        t[misalign:misalign + len(data)] = torch.from_numpy(np.frombuffer(bytes(data), dtype=np.uint8).copy()).cuda()
    return t[misalign:]


def gpu_slots(cu, data, chunk, level, flags, misalign):
    """the device's slots for the uniform partition of data (base address misaligned by `misalign` bytes)"""
    p, lib, torch = cu
    n = len(data)
    src = to_device(torch, data, misalign)
    assert (src.data_ptr() % 16 == 0) == (misalign == 0)
    b = p.DeflateBatch(max(n, 1), chunk=chunk, with_crc=False)
    k = b.compress(src, n, level=level, final=bool(flags & A.FLAG_FINAL), join=False, one_stream=bool(flags & A.FLAG_DICT))
    torch.cuda.synchronize()
    lens = b.out_len[:k].cpu().tolist()
    raw = b.slots[:k * b.stride].cpu().numpy()
    return [raw[i * b.stride:i * b.stride + lens[i]].tobytes() for i in range(k)]


def same_parse(es, gs, stats):
    """3b, for one chunk: the emulator's and the device's blocks unit by unit"""
    for u, (eb, gb) in enumerate(zip(es.units, gs.units)):
        if eb.btype != gb.btype:
            stats["stored on one side"] += 1  # judged by check_codes on each side, under its own builder
        elif eb.btype == 0:
            assert (eb.stored_len, eb.pad_bits) == (gb.stored_len, gb.pad_bits), "unit %d: stored blocks differ" % u
        else:
            assert eb.tokens == gb.tokens, "unit %d: the device's parse differs from the emulator's" % u
            stats["differing lengths"] += (eb.ll_lens, eb.d_lens) != (gb.ll_lens, gb.d_lens)
    assert len(es.units) == len(gs.units)


@pytest.mark.parametrize("level", E.LEVELS)
def test_device_blocks_follow_the_rules_and_the_emulator_parse(cu, emushim_lib, codes, gpu_lib, corpus, level):  # noqa: F811
    stats = {"blocks": 0, "differing lengths": 0, "stored on one side": 0}
    for name, data, chunk in corpus:
        for mode, flags in E.MODES.items():
            try:
                eslots, _ = E.run_config(emushim_lib, codes, data, chunk, level, flags)
                offs, lens, fl = E.chunk_table(len(data), chunk, flags)
                hists = E.capture(codes, data, offs, lens, fl, level) if level else None
                aligned = gpu_slots(cu, data, chunk, level, flags, 0)
                assert gpu_slots(cu, data, chunk, level, flags, 3) == aligned, "the TMA and the plain load give different bytes"
                gslots = E.slots_of(data, b"".join(aligned), [len(x) for x in aligned], offs, lens, fl, level)
                for s in gslots:
                    A.check_slot(s)
                A.check_codes(gslots, gpu_builder(gpu_lib), hists)
                for es, gs in zip(eslots, gslots):
                    same_parse(es, gs, stats)
                stats["blocks"] += sum(len(s.units) for s in gslots)
            except AssertionError as e:
                raise AssertionError("%s, chunk %d, level %d, %s: %s" % (name, chunk, level, mode, e)) from e
    print("level %d: %d blocks; %d with code lengths that differ from the emulator's (__log2f); %d stored on one side only" % (
        level, stats["blocks"], stats["differing lengths"], stats["stored on one side"]))


# ---- c. under load ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def load_inputs(cu):
    import datagen
    import textgen
    p, lib, torch = cu
    text = textgen.device(256 << 20, seed=1000)
    mixed = datagen.mixed(4 << 20, 3)  # (the Python generator is slow: 4 MiB of it, repeated)
    return {"text": text, "mixed": to_device(torch, mixed * 16)[:64 << 20]}


@pytest.mark.parametrize("source", ["text", "mixed"])
@pytest.mark.parametrize("level,one", [(1, False), (4, False), (6, False), (6, True)])
def test_device_output_under_load(cu, codes, gpu_lib, load_inputs, source, level, one):  # noqa: F811
    p, lib, torch = cu
    src = load_inputs[source]
    n = src.numel()
    flags = A.FLAG_FINAL | (A.FLAG_DICT if one else 0)
    b = p.DeflateBatch(n, with_crc=False)
    runs = []
    for _ in range(2):
        k = b.compress(src, n, level=level, final=True, join=False, one_stream=one)
        torch.cuda.synchronize()
        runs.append((b.out_len[:k].clone(), b.slots[:k * b.stride].clone()))
    (len0, slots0), (len1, slots1) = runs
    assert torch.equal(len0, len1), "two runs give different lengths"
    used = torch.arange(b.stride, device="cuda")[None, :] < len0.to(torch.int64)[:, None]
    assert torch.equal(slots0.view(k, b.stride)[used], slots1.view(k, b.stride)[used]), "two runs give different bytes"
    del runs, slots1, used

    # 64 chunks recompressed alone (explicit offsets; one-stream chunks with DICT read the 32 KiB in front of them)
    idx = sorted(random.Random(level * 2 + one + (source == "mixed") * 100).sample(range(k), LOAD_SAMPLE))
    offs, lens, fl = E.chunk_table(n, b.chunk, flags)
    offs, lens, fl = [offs[i] for i in idx], [lens[i] for i in idx], [fl[i] for i in idx]
    d_off = torch.tensor(offs, dtype=torch.int64, device="cuda")
    d_len = torch.tensor(lens, dtype=torch.int32, device="cuda")
    d_fl = torch.tensor(fl, dtype=torch.uint8, device="cuda")
    alone = torch.empty(LOAD_SAMPLE * b.stride, dtype=torch.uint8, device="cuda")
    alone_len = torch.empty(LOAD_SAMPLE, dtype=torch.int32, device="cuda")
    p.check(lib.mz_cuda_deflate_chunks(src.data_ptr(), 0, 0, d_off.data_ptr(), d_len.data_ptr(), d_fl.data_ptr(), LOAD_SAMPLE, 0, level,
                                       alone.data_ptr(), b.stride, alone_len.data_ptr(), None), "deflate")
    torch.cuda.synchronize()
    big_len = len0.cpu().tolist()
    alone_len = alone_len.cpu().tolist()
    assert alone_len == [big_len[i] for i in idx], "a chunk compressed alone has another length"
    big = slots0.view(k, b.stride)[torch.tensor(idx, device="cuda")].cpu().numpy()
    alone = alone.view(LOAD_SAMPLE, b.stride).cpu().numpy()

    # the sampled chunks (+ the 32 KiB in front where DICT lets them reach back) on the host, and every rule
    host = src.cpu().numpy()
    slots, segs, seg_offs, pos = [], [], [], 0
    for j, (o, ln, f) in enumerate(zip(offs, lens, fl)):
        assert alone[j, :alone_len[j]].tobytes() == big[j, :alone_len[j]].tobytes(), "chunk %d: alone != in the big run" % idx[j]
        win = host[o - A.DF_UNIT:o].tobytes() if (level >= 6 and one and o >= A.DF_UNIT) else b""
        chunk = host[o:o + ln].tobytes()
        slots.append(A.Slot(alone[j, :alone_len[j]].tobytes(), chunk, level, f, win))
        A.check_slot(slots[-1])
        segs.append(win + chunk)
        seg_offs.append(pos + len(win))
        pos += len(win) + ln
    hists = E.capture(codes, b"".join(segs), seg_offs, lens, fl, level)
    A.check_codes(slots, gpu_builder(gpu_lib), hists)
