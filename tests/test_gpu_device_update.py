"""mz_zip_cuda_update_device on the H100: byte identity with mz_zip_cuda_write_device of the kept entries followed by the new ones at MiB
sizes with the new items at every alignment mod 16, the copy kernel on every pair of source and destination alignment mod 16, the C4 shape with every 100th entry dropped, an archive past 4 GiB with more than 65535 entries
(new local headers past 4 GiB on append; kept records moved below 4 GiB when early entries are dropped) and the Python update_device
round trip through ZipDeviceReader, with empty keep lists and boolean masks. Large archives stay in device memory and are compared there."""
import ctypes as C

import pytest

from test_emu_device_update import COPY_LENGTHS, DeviceUpdater, copy_pairs, identical
from test_emu_device_write import DATE
from test_gpu_device_write import c4_blobs, mib_entries
from test_emu_native_extract import HASH_SHA256, corpus

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def du(built):
    import cuharness
    lib = cuharness.pkg().load()
    assert lib.mz_cuda_init() == 0
    return DeviceUpdater(lib)


def test_identity_mib_entries_every_alignment(du):
    A = mib_entries(40, seed=400)
    B = [("new/" + n, d) for n, d in mib_entries(16, seed=401)]
    # the new items at every offset mod 16 in their buffer
    offs, pos = [], 0
    for i, (_, d) in enumerate(B):
        offs.append(pos + i % 16)
        pos += (len(d) + 47) & ~15
    layout = du.layout(B, offs)
    for level, flags in ((1, 0), (6, HASH_SHA256), (9, 0)):
        src = du.device(A, level=level, flags=flags)[1]
        for S in (None, list(range(39, -1, -3)), [5, 5, 0]):
            kept = A if S is None else [A[i] for i in S]
            want = du.device(kept + B, level=level, flags=flags, layout=_join_layout(du, kept, layout))[1]
            err, got, _, n, bound = du.update(src, keep=S, files=B, level=level, flags=flags, layout=layout)
            assert err == 0 and got == want and n <= bound, (level, flags, S)
    identical(du, A[:10], [9, 1], B[:3], level=6)


def test_copy_kernel_every_alignment_pair(du):
    """the copy kernel on every (source mod 16, destination mod 16) pair, short and long extents, and a cap inside a slot"""
    assert copy_pairs(du.lib) == 16 * 16 * len(COPY_LENGTHS)


def _join_layout(du, kept, layout_b):
    """the layout of kept + B for write_device: kept entries packed in front of B's buffer, B's items at their offsets behind them"""
    data_k, names_k, items_k = du.layout(kept)
    data_b, names_b, items_b = layout_b
    shift = (len(data_k) + 15) & ~15
    arr = (du.pkg.ZipDevItem * max(1, len(items_b) // 40)).from_buffer_copy(items_b or bytes(40))
    for it in arr[:len(items_b) // 40]:
        it.data_off += shift
        it.name_off += len(names_k)
    return data_k.ljust(shift, b"\0") + data_b, names_k + names_b, items_k + bytes(arr)[:len(items_b)]


class Dev:
    """entries as rows of a device pool of 100 blobs; archives in torch tensors"""

    def __init__(self, lib, pkg, blobs):
        import torch
        self.lib, self.pkg, self.eb = lib, pkg, len(blobs[0])
        self.pool = torch.frombuffer(bytearray(b"".join(blobs)), dtype=torch.uint8).cuda()

    def items(self, ids, prefix):
        """[(name, blob index)] -> (d_names, d_items)"""
        import torch
        names = [("%s/%06d" % (prefix, i)).encode() for i in ids]
        its = (self.pkg.ZipDevItem * max(1, len(ids)))()
        pos = 0
        for k, i in enumerate(ids):
            its[k] = self.pkg.ZipDevItem((i % 100) * self.eb, self.eb, pos, len(names[k]), self.pkg.dos_date(DATE), 0, 0)
            pos += len(names[k])
        return (torch.frombuffer(bytearray(b"".join(names) or b"\0"), dtype=torch.uint8).cuda(),
                torch.frombuffer(bytearray(bytes(its)), dtype=torch.uint8).cuda())

    def write(self, parts, level):
        """write_device of the concatenated [(ids, prefix)] -> tensor"""
        import torch
        names, its = [], (self.pkg.ZipDevItem * max(1, sum(len(i) for i, _ in parts)))()
        k, pos = 0, 0
        for ids, prefix in parts:
            for i in ids:
                nm = ("%s/%06d" % (prefix, i)).encode()
                its[k] = self.pkg.ZipDevItem((i % 100) * self.eb, self.eb, pos, len(nm), self.pkg.dos_date(DATE), 0, 0)
                names.append(nm)
                pos += len(nm)
                k += 1
        nb = torch.frombuffer(bytearray(b"".join(names) or b"\0"), dtype=torch.uint8).cuda()
        d_items = torch.frombuffer(bytearray(bytes(its)), dtype=torch.uint8).cuda()
        n = C.c_uint64(0)
        args = (self.pool.data_ptr(), nb.data_ptr(), d_items.data_ptr(), k, level, 0, None, 0)
        assert self.lib.mz_zip_cuda_write_device(*args, None, 0, C.byref(n), None, None, None) == 0
        out = torch.empty(n.value, dtype=torch.uint8, device="cuda")
        assert self.lib.mz_zip_cuda_write_device(*args, out.data_ptr(), out.numel(), C.byref(n), None, None, None) == 0
        return out[:n.value]

    def update(self, src, keep, ids, prefix, level):
        import torch
        d_names, d_items = self.items(ids, prefix)
        d_keep = torch.tensor(keep, dtype=torch.int32, device="cuda") if keep is not None else None
        n = C.c_uint64(0)
        args = (src.data_ptr(), src.numel(), d_keep.data_ptr() if keep is not None else None, len(keep) if keep is not None else 0,
                self.pool.data_ptr(), d_names.data_ptr(), d_items.data_ptr(), len(ids), level, 0, None, 0)
        assert self.lib.mz_zip_cuda_update_device(*args, None, 0, C.byref(n), None, None, None) == 0
        out = torch.empty(n.value, dtype=torch.uint8, device="cuda")
        err = self.lib.mz_zip_cuda_update_device(*args, out.data_ptr(), out.numel(), C.byref(n), None, None, None)
        assert err == 0, err
        return out[:n.value]


def _same(a, b):
    import torch
    return a.numel() == b.numel() and bool(torch.equal(a, b))


def test_c4_drop_every_100th_and_append(du):
    import cuharness
    d = Dev(du.lib, cuharness.pkg(), c4_blobs())
    n = 100_000
    src = d.write([(range(n), "e")], 6)
    keep = [i for i in range(n) if i % 100 != 99]
    got = d.update(src, keep, range(1000), "new", 6)
    want = d.write([(keep, "e"), (range(1000), "new")], 6)
    assert _same(got, want)
    del src, got, want
    du.lib.mz_zip_cuda_trim()


def test_zip64_past_4_gib(du):
    import torch
    import cuharness
    d = Dev(du.lib, cuharness.pkg(), c4_blobs())
    n = 70_000
    src = d.write([(range(n), "z")], 0)
    assert src.numel() > 1 << 32
    # append: the new local headers lie past 4 GiB
    got = d.update(src, None, range(100), "new", 0)
    want = d.write([(range(n), "z"), (range(100), "new")], 0)
    assert _same(got, want)
    del got, want
    torch.cuda.empty_cache()
    # drop the first 3000 entries: kept entries past 4 GiB move below it and lose their zip64 fields, the last ones keep them
    keep = list(range(3000, n))
    got = d.update(src, keep, range(10), "new", 0)
    want = d.write([(keep, "z"), (range(10), "new")], 0)
    assert _same(got, want)
    del src, got, want
    torch.cuda.empty_cache()
    du.lib.mz_zip_cuda_trim()


def test_python_update_device_round_trip(du):
    import torch
    import cuharness
    pkg = cuharness.pkg()
    files = corpus(12, 150_000, seed=410)
    t = lambda d: torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda() if d else torch.empty(0, dtype=torch.uint8, device="cuda")
    arc = pkg.write_device([(n, t(d)) for n, d in files], mtime=DATE)
    with pkg.ZipDeviceReader(arc) as r:
        drop = r.locate([files[3][0], files[7][0]])
        keep = torch.arange(r.count, device="cuda")
        keep = keep[~torch.isin(keep, drop)]
    new = [("added/one", t(b"one " * 5000)), ("added/two", t(b""))]
    out = pkg.update_device(arc, keep=keep, files=new, mtime=DATE)
    want = [f for i, f in enumerate(files) if i not in (3, 7)] + [("added/one", b"one " * 5000), ("added/two", b"")]
    assert out.untyped_storage().nbytes() == out.numel()
    with pkg.ZipDeviceReader(out) as r:
        assert [e[0] for e in r.entries] == [n for n, _ in want]
        offs, data = r.read(list(range(r.count)))
        host, o = data.cpu().numpy().tobytes(), offs.cpu().tolist()
        assert [host[o[k]:o[k] + len(want[k][1])] for k in range(len(want))] == [d for _, d in want]
    direct = pkg.write_device([(n, t(d)) for n, d in want], mtime=DATE)
    assert _same(out, direct)
    assert _same(pkg.update_device(arc, mtime=DATE), arc)  # keep everything, append nothing: the same archive


def test_python_update_device_keep_none_and_masks(du):
    """keep=[] (or an all-False mask) keeps no entry: the output is write_device of the new files alone; a boolean mask keeps the
    entries where it is True"""
    import torch
    import cuharness
    pkg = cuharness.pkg()
    files = corpus(6, 40_000, seed=420)
    t = lambda d: torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda() if d else torch.empty(0, dtype=torch.uint8, device="cuda")
    arc = pkg.write_device([(n, t(d)) for n, d in files], mtime=DATE)
    new = [("only/new", t(b"new " * 3000))]
    alone = pkg.write_device(new, mtime=DATE)
    for keep in ([], torch.empty(0, dtype=torch.int64, device="cuda"), torch.zeros(len(files), dtype=torch.bool)):
        assert _same(pkg.update_device(arc, keep=keep, files=new, mtime=DATE), alone)
    mask = torch.tensor([i % 2 == 0 for i in range(len(files))], device="cuda")
    want = pkg.write_device([(n, t(d)) for i, (n, d) in enumerate(files) if i % 2 == 0] + new, mtime=DATE)
    assert _same(pkg.update_device(arc, keep=mask, files=new, mtime=DATE), want)
