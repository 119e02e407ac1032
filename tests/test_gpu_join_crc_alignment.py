"""GPU twin of test_emu_join_crc_alignment.py (pytest -m gpu): the product library's mz_cuda_gather, mz_cuda_concat and
mz_cuda_crc32_segments at every alignment that matters to the join copy and the CRC kernel, against plain slicing and
zlib.crc32, plus one 1 GiB pass shaped like the bench's C5 step."""
import random
import zlib

import numpy as np
import pytest

import test_emu_join_crc_alignment as m

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu(built):
    import torch
    import cuharness
    p = cuharness.pkg()
    lib = p.load()
    assert lib.mz_cuda_init() == 0, lib.mz_cuda_last_error()
    torch.cuda.set_device(0)
    return torch, p, lib


def dev(torch, b):
    return torch.from_numpy(np.frombuffer(bytes(b), dtype=np.uint8).copy()).cuda()


def host(t):
    return bytes(t.cpu().numpy().tobytes())


def run_join(gpu, slots, lens, dst, offsets=None, misalign=0):
    torch, p, lib = gpu
    n = len(lens)
    d_slots = dev(torch, slots)  # a tensor of exactly n * STRIDE bytes
    d_len = torch.tensor(lens, dtype=torch.int32, device="cuda")
    d_dst = dev(torch, bytes(misalign) + bytes(dst) + bytes(16))  # the allocation is 16-byte aligned, so dst sits at misalign mod 16
    assert d_dst.data_ptr() % 16 == 0
    if offsets is None:
        d_off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
        p.check(lib.mz_cuda_concat(d_slots.data_ptr(), m.STRIDE, d_len.data_ptr(), n, d_off.data_ptr(), d_dst.data_ptr() + misalign, None), "concat")
    else:
        d_off = torch.tensor(offsets, dtype=torch.int64, device="cuda")
        p.check(lib.mz_cuda_gather(d_slots.data_ptr(), m.STRIDE, d_len.data_ptr(), n, d_off.data_ptr(), d_dst.data_ptr() + misalign, None), "gather")
    torch.cuda.synchronize()
    return host(d_dst[misalign:misalign + len(dst)]), d_off.cpu().tolist()


@pytest.mark.parametrize("misalign", [0, 9])
def test_gpu_gather_every_alignment_keeps_guards(gpu, misalign):
    rng = random.Random(1 + misalign)
    cases, offs, size = m.aligned_case(rng)
    lens = [k for _, k in cases]
    slots = m.make_slots(rng, len(cases))
    dst = rng.randbytes(size)
    got, _ = run_join(gpu, slots, lens, dst, offs, misalign)
    want = bytearray(dst)
    for i, (o, k) in enumerate(zip(offs, lens)):
        want[o:o + k] = slots[i * m.STRIDE:i * m.STRIDE + k]
    assert got == bytes(want)


@pytest.mark.parametrize("misalign", [0, 1, 7, 15])
def test_gpu_concat_matches_slicing(gpu, misalign):
    rng = random.Random(100 + misalign)
    lens = m.LENGTHS + [rng.randrange(m.STRIDE + 1) for _ in range(200)]
    rng.shuffle(lens)
    lens.append(m.STRIDE)
    slots = m.make_slots(rng, len(lens))
    total = sum(lens)
    dst = rng.randbytes(total + 16)
    got, offs = run_join(gpu, slots, lens, dst, None, misalign)
    assert offs[-1] == total and offs[:-1] == [sum(lens[:i]) for i in range(len(lens))]
    assert got[:total] == b"".join(slots[i * m.STRIDE:i * m.STRIDE + k] for i, k in enumerate(lens)) and got[total:] == dst[total:]


def test_gpu_concat_many_tiny_slots_share_words(gpu):
    rng = random.Random(7)
    lens = [rng.choice([0, 1, 1, 2, 3]) for _ in range(5000)]
    slots = m.make_slots(rng, len(lens))
    total = sum(lens)
    for misalign in (0, 5, 13):
        dst = rng.randbytes(total + 32)
        got, _ = run_join(gpu, slots, lens, dst, None, misalign)
        assert got[:total] == b"".join(slots[i * m.STRIDE:i * m.STRIDE + k] for i, k in enumerate(lens)) and got[total:] == dst[total:]


@pytest.mark.parametrize("misalign", range(16))
def test_gpu_crc_ragged_segments_every_start_alignment(gpu, misalign):
    torch, p, lib = gpu
    rng = random.Random(misalign)
    segs, pos = [], 0
    for k in m.CRC_LENGTHS:
        segs.append((pos, k))
        pos += k + rng.randrange(3)
    data = rng.randbytes(pos + 5)
    d = dev(torch, bytes(misalign) + data)
    n = len(segs)
    d_off = torch.tensor([misalign + o for o, _ in segs], dtype=torch.int64, device="cuda")
    d_len = torch.tensor([k for _, k in segs], dtype=torch.int32, device="cuda")
    res = torch.empty(n, dtype=torch.int32, device="cuda")
    crc = torch.empty(n, dtype=torch.int32, device="cuda")
    p.check(lib.mz_cuda_crc32_segments(d.data_ptr(), 0, 0, d_off.data_ptr(), d_len.data_ptr(), n, res.data_ptr(), crc.data_ptr(), None))
    got = [v & 0xFFFFFFFF for v in crc.cpu().tolist()]
    assert got == [zlib.crc32(data[o:o + k]) for o, k in segs]


@pytest.mark.parametrize("seg", [512, 700, 1000, 4100, 65536])
def test_gpu_crc_uniform_segments(gpu, seg):
    torch, p, lib = gpu
    rng = random.Random(seg)
    data = rng.randbytes(37 * seg + 77)
    nseg = (len(data) + seg - 1) // seg
    for misalign in (0, 3, 8, 15):
        d = dev(torch, bytes(misalign) + data)
        res = torch.empty(nseg, dtype=torch.int32, device="cuda")
        crc = torch.empty(nseg, dtype=torch.int32, device="cuda")
        out2 = torch.empty(2, dtype=torch.int32, device="cuda")
        p.check(lib.mz_cuda_crc32_segments(d.data_ptr() + misalign, len(data), seg, None, None, nseg, res.data_ptr(), crc.data_ptr(), None))
        p.check(lib.mz_cuda_crc32_fold(res.data_ptr(), nseg, seg, len(data), out2.data_ptr(), None))
        assert [v & 0xFFFFFFFF for v in crc.cpu().tolist()] == [zlib.crc32(data[i:i + seg]) for i in range(0, len(data), seg)]
        assert int(out2[1].item()) & 0xFFFFFFFF == zlib.crc32(data)


def test_gpu_c5_shaped_pass_1gib(gpu):
    """One C5-shaped step over 1 GiB of the bench text: the joined stream is the concatenation of the slots, and the per-chunk
    CRCs of a sample of chunks are zlib's."""
    torch, p, lib = gpu
    import textgen
    n = 1 << 30
    nch = n // 65536
    src = torch.empty(n, dtype=torch.uint8, device="cuda")
    for o in range(0, n, 64 << 20):
        textgen.device_into(src.data_ptr() + o, 64 << 20, 1000 + o // (64 << 20))
    b = p.DeflateBatch(n)
    assert b.compress(src, n, level=1, final=True) == nch
    joined, crc = b.result(nch)
    lens = b.out_len[:nch].to(torch.int64)
    offs = b.offsets[:nch + 1]
    assert int(offs[0].item()) == 0 and torch.equal(offs[1:], torch.cumsum(lens, 0))
    stride = b.stride
    slots = b.slots[:nch * stride].view(nch, stride)
    idx = torch.arange(stride, device="cuda").unsqueeze(0) < lens.unsqueeze(1)
    assert torch.equal(joined, slots[idx])  # row-major masked select = the slots' bytes concatenated in order
    sample = random.Random(5).sample(range(nch), 64) + [0, nch - 1]
    chunk_crc = b.chunk_crc[:nch].cpu().numpy().view(np.uint32)
    for c in sample:
        assert int(chunk_crc[c]) == zlib.crc32(host(src[c * 65536:(c + 1) * 65536]))
    del slots, idx
