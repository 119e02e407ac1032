"""minizip-ng_b200 -- host-side Python mirror of the H100 DEFLATE + CRC-32 backend.

The product is the C-ABI shared library ``libmz_strm_cuda.so`` (include/mz_strm_cuda.h,
include/mz_cuda_batch.h).  This package only (a) loads it with ctypes, (b) wraps device buffers in
torch tensors for the bench / multi-GPU plumbing, (c) mirrors the reference's stream interface names so
tests read like test/test_stream_compress.cc.  There is no Python or CPU codec here: if the library is
missing or no sm_90 GPU is usable, calls raise.

Import note: the directory name contains a hyphen (the project name); load it with
``importlib`` (see __graft_entry__._load_pkg) -- it registers itself as ``minizip_ng_b200``.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmz_strm_cuda.so")

MZ_OK = 0
MZ_DATA_ERROR, MZ_MEM_ERROR, MZ_BUF_ERROR = -3, -4, -5
MZ_SUPPORT_ERROR, MZ_OPEN_ERROR, MZ_CLOSE_ERROR = -109, -111, -112
MZ_OPEN_MODE_READ, MZ_OPEN_MODE_WRITE = 0x01, 0x02
MZ_STREAM_PROP_TOTAL_IN, MZ_STREAM_PROP_TOTAL_IN_MAX, MZ_STREAM_PROP_TOTAL_OUT = 1, 2, 3
MZ_STREAM_PROP_COMPRESS_LEVEL, MZ_STREAM_PROP_COMPRESS_WINDOW = 9, 11
CHUNK_MAX = 65536
FLAG_FINAL = 1
FLAG_DICT = 2  # the buffer is ONE stream: at levels 6-9 a chunk may refer back into the 32 KiB before it

_lib = None


class InflateJob(C.Structure):
    _fields_ = [("d_in", C.c_void_p), ("in_base", C.c_uint64), ("in_avail", C.c_uint64), ("d_out", C.c_void_p),
                ("out_base", C.c_uint64), ("out_cap", C.c_uint64), ("in_final", C.c_uint32), ("flags", C.c_uint32)]


class InflateState(C.Structure):
    _fields_ = [("in_bitpos", C.c_uint64), ("out_pos", C.c_uint64), ("status", C.c_int32), ("why", C.c_int32),
                ("phase", C.c_uint32), ("last_block", C.c_uint32), ("stored_remaining", C.c_uint32), ("nlit", C.c_uint32),
                ("ndist", C.c_uint32), ("blocks", C.c_uint32), ("lens", C.c_uint8 * 320)]


EXPORTS = [
    # include/mz_strm_cuda.h
    "mz_stream_cuda_open", "mz_stream_cuda_is_open", "mz_stream_cuda_read", "mz_stream_cuda_write", "mz_stream_cuda_tell",
    "mz_stream_cuda_seek", "mz_stream_cuda_close", "mz_stream_cuda_error", "mz_stream_cuda_get_prop_int64",
    "mz_stream_cuda_set_prop_int64", "mz_stream_cuda_create", "mz_stream_cuda_delete", "mz_stream_cuda_get_interface",
    "mz_crypt_crc32_update",
    # include/mz_cuda_batch.h
    "mz_cuda_init", "mz_cuda_device_count", "mz_cuda_set_device", "mz_cuda_get_device", "mz_cuda_last_error", "mz_cuda_sm_count", "mz_cuda_malloc",
    "mz_cuda_free", "mz_cuda_host_alloc", "mz_cuda_host_free", "mz_cuda_memcpy_h2d", "mz_cuda_memcpy_d2h", "mz_cuda_memcpy_d2d",
    "mz_cuda_memset", "mz_cuda_host_is_pinned", "mz_cuda_stream_sync", "mz_cuda_stream_create", "mz_cuda_stream_destroy",
    "mz_cuda_event_create", "mz_cuda_event_destroy", "mz_cuda_event_record", "mz_cuda_event_sync", "mz_cuda_event_query", "mz_cuda_event_elapsed_ms",
    "mz_cuda_crc32_segments", "mz_cuda_crc32_fold", "mz_cuda_crc32_device", "mz_cuda_crc32_device_stream", "mz_cuda_crc32_combine",
    "mz_cuda_deflate_slot_bound", "mz_cuda_deflate_chunks", "mz_cuda_concat", "mz_cuda_inflate_streams",
    "mz_cuda_inflate_spec_workspace_bytes", "mz_cuda_inflate_spec_round", "mz_cuda_sha256_batch",
    "mz_cuda_wzaes_derive", "mz_cuda_wzaes_ctr", "mz_cuda_wzaes_hmac",
    "mz_cuda_gather_region_bound", "mz_cuda_deflate_sharded", "mz_cuda_ipc_export", "mz_cuda_ipc_open", "mz_cuda_ipc_close", "mz_cuda_memcpy_peer",
    "mz_cuda_stream_wait_event", "mz_cuda_gather", "mz_cuda_scatter_blobs",
    # include/mz_zip_cuda.h
    "mz_zip_cuda_add_buffers", "mz_zip_cuda_add_buffers_ex", "mz_zip_cuda_write_archive", "mz_zip_cuda_trim", "mz_zip_cuda_write_archive_aes", "mz_zip_cuda_extract_all",
    "mz_zip_cuda_extract_all_aes", "mz_zip_cuda_extract_archive", "mz_zip_cuda_extract_device", "mz_zip_cuda_write_device", "mz_zip_cuda_abi_file_info_size",
    "mz_zip_cuda_reader_open", "mz_zip_cuda_reader_entries", "mz_zip_cuda_reader_locate", "mz_zip_cuda_reader_decode", "mz_zip_cuda_reader_close",
    "mz_zip_cuda_update_device",
    # include/mz_cuda_batch.h, K9 and K10
    "mz_cuda_zip_locate", "mz_cuda_zip_copy_stored", "mz_cuda_zip_verify", "mz_cuda_zip_parse_directory", "mz_cuda_zip_statuses",
    # include/mz_cuda_batch.h, K11
    "mz_cuda_zip_wr_items", "mz_cuda_zip_wr_chunks", "mz_cuda_zip_wr_place", "mz_cuda_zip_wr_entries", "mz_cuda_zip_wr_emit",
    # include/mz_cuda_batch.h, K12
    "mz_cuda_zip_name_index", "mz_cuda_zip_name_lookup", "mz_cuda_zip_sel_counts", "mz_cuda_zip_sel_fill", "mz_cuda_zip_sel_gather",
    "mz_cuda_zip_sel_status",
    # include/mz_cuda_batch.h, K13
    "mz_cuda_zip_up_counts", "mz_cuda_zip_up_copy", "mz_cuda_zip_up_records",
]

# mz_cuda_zip_entry_cb (include/mz_zip_cuda.h): (userdata, filename, data, size, crc32) -> 0 or an error that stops the extraction
ZIP_ENTRY_CB = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.c_uint32)
MZ_ZIP_CUDA_HASH_SHA256, MZ_ZIP_CUDA_ALL_DEVICES, MZ_ZIP_CUDA_AES = 1, 2, 4


class ZipStats(C.Structure):
    """mz_cuda_zip_stats (include/mz_zip_cuda.h)"""
    _fields_ = [("bytes_in", C.c_uint64), ("bytes_out", C.c_uint64), ("entries", C.c_uint32), ("rounds", C.c_uint32),
                ("pack_ms", C.c_double), ("gpu_ms", C.c_double), ("container_ms", C.c_double), ("setup_ms", C.c_double)]


class ZipDevEntry(C.Structure):
    """mz_cuda_zip_dev_entry (include/mz_zip_cuda.h)"""
    _fields_ = [("local_off", C.c_uint64), ("csize", C.c_uint64), ("usize", C.c_uint64), ("out_off", C.c_uint64), ("name_off", C.c_uint64),
                ("extent", C.c_uint64), ("sha_off", C.c_uint64), ("crc", C.c_uint32), ("name_len", C.c_uint32), ("method", C.c_uint16),
                ("aes", C.c_uint8), ("has_sha", C.c_uint8), ("status", C.c_int32)]


class ZipItem(C.Structure):
    """mz_cuda_zip_item (include/mz_zip_cuda.h)"""
    _fields_ = [("filename", C.c_char_p), ("data", C.c_void_p), ("size", C.c_int64), ("modified_date", C.c_int64),
                ("external_fa", C.c_uint32), ("reserved", C.c_uint32)]


class ZipDevItem(C.Structure):
    """mz_cuda_zip_dev_item (include/mz_zip_cuda.h)"""
    _fields_ = [("data_off", C.c_uint64), ("size", C.c_uint64), ("name_off", C.c_uint64), ("name_len", C.c_uint32), ("dos_date", C.c_uint32),
                ("external_fa", C.c_uint32), ("reserved", C.c_uint32)]


def dos_date(t):
    """the MS-DOS date/time the zip headers store for unix time t, in local time (the native writer's za_dos_date)"""
    import time
    tm = time.localtime(t)
    year = tm.tm_year - 1980 if tm.tm_year >= 1980 else 0
    return ((tm.tm_mday + 32 * tm.tm_mon + 512 * year) << 16) | (tm.tm_sec // 2 + 32 * tm.tm_min + 2048 * tm.tm_hour)


def load():
    """Load the product library; fail loudly if it has not been built (no fallback of any kind)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("libmz_strm_cuda.so is missing: run __graft_entry__.build() (nvcc, sm_90a). "
                           "There is no CPU fallback.")
    _lib = configure(C.CDLL(LIB_PATH))
    return _lib


def configure(L):
    """ctypes prototypes of the C-ABI on an already loaded library (the product .so, or -- in the CPU test suite -- the same
    sources built against the execution-model emulator, tests/emu/libmz_strm_emu.so)."""
    vp, i32, i64, u32, u64, sz = C.c_void_p, C.c_int32, C.c_int64, C.c_uint32, C.c_uint64, C.c_size_t

    def sig(name, res, args):
        f = getattr(L, name)
        f.restype = res
        f.argtypes = args

    sig("mz_stream_cuda_open", i32, [vp, C.c_char_p, i32])
    sig("mz_stream_cuda_is_open", i32, [vp])
    sig("mz_stream_cuda_read", i32, [vp, vp, i32])
    sig("mz_stream_cuda_write", i32, [vp, vp, i32])
    sig("mz_stream_cuda_tell", i64, [vp])
    sig("mz_stream_cuda_seek", i32, [vp, i64, i32])
    sig("mz_stream_cuda_close", i32, [vp])
    sig("mz_stream_cuda_error", i32, [vp])
    sig("mz_stream_cuda_get_prop_int64", i32, [vp, i32, C.POINTER(i64)])
    sig("mz_stream_cuda_set_prop_int64", i32, [vp, i32, i64])
    sig("mz_stream_cuda_create", vp, [])
    sig("mz_stream_cuda_delete", None, [C.POINTER(vp)])
    sig("mz_stream_cuda_get_interface", vp, [])
    sig("mz_crypt_crc32_update", u32, [u32, vp, i32])
    sig("mz_cuda_init", i32, [])
    sig("mz_cuda_device_count", i32, [])
    sig("mz_cuda_set_device", i32, [i32])
    sig("mz_cuda_last_error", C.c_char_p, [])
    sig("mz_cuda_sm_count", i32, [])
    sig("mz_cuda_malloc", vp, [sz])
    sig("mz_cuda_free", None, [vp])
    sig("mz_cuda_host_alloc", vp, [sz])
    sig("mz_cuda_host_free", None, [vp])
    sig("mz_cuda_memcpy_h2d", i32, [vp, vp, sz, vp])
    sig("mz_cuda_memcpy_d2h", i32, [vp, vp, sz, vp])
    sig("mz_cuda_memcpy_d2d", i32, [vp, vp, sz, vp])
    sig("mz_cuda_memset", i32, [vp, C.c_int, sz, vp])
    sig("mz_cuda_host_is_pinned", i32, [vp])
    sig("mz_cuda_stream_sync", i32, [vp])
    sig("mz_cuda_stream_create", vp, [])
    sig("mz_cuda_stream_destroy", None, [vp])
    sig("mz_cuda_event_create", vp, [])
    sig("mz_cuda_event_destroy", None, [vp])
    sig("mz_cuda_event_record", i32, [vp, vp])
    sig("mz_cuda_event_sync", i32, [vp])
    sig("mz_cuda_event_elapsed_ms", C.c_float, [vp, vp])
    sig("mz_cuda_crc32_segments", i32, [vp, u64, u64, vp, vp, u32, vp, vp, vp])
    sig("mz_cuda_crc32_fold", i32, [vp, u32, u64, u64, vp, vp])
    sig("mz_cuda_crc32_device", i32, [vp, u64, u32, C.POINTER(u32)])
    sig("mz_cuda_crc32_combine", u32, [u32, u32, u64])
    sig("mz_cuda_deflate_slot_bound", u64, [u32])
    sig("mz_cuda_deflate_chunks", i32, [vp, u64, u32, vp, vp, vp, u32, u32, i32, vp, u64, vp, vp])
    sig("mz_cuda_concat", i32, [vp, u64, vp, u32, vp, vp, vp])
    sig("mz_cuda_inflate_streams", i32, [vp, vp, u32, vp])
    sig("mz_cuda_sha256_batch", i32, [vp, vp, vp, u32, vp, vp])
    sig("mz_cuda_wzaes_derive", i32, [vp, u32, vp, u32, u32, vp, vp])
    sig("mz_cuda_wzaes_ctr", i32, [vp, vp, vp, u32, u64, vp, u32, vp])
    sig("mz_cuda_wzaes_hmac", i32, [vp, vp, vp, u32, vp, u32, vp, vp])
    sig("mz_cuda_gather_region_bound", u64, [u64])
    sig("mz_cuda_deflate_sharded", i32, [vp, i32, i32, i32, C.POINTER(u64), C.POINTER(u64), C.POINTER(u32)])
    sig("mz_cuda_ipc_export", i32, [vp, vp])
    sig("mz_cuda_ipc_open", i32, [vp, C.POINTER(vp)])
    sig("mz_cuda_ipc_close", i32, [vp])
    sig("mz_cuda_memcpy_peer", i32, [vp, vp, sz, vp])
    sig("mz_cuda_stream_wait_event", i32, [vp, vp])
    sig("mz_cuda_gather", i32, [vp, u64, vp, u32, vp, vp, vp])
    sig("mz_cuda_scatter_blobs", i32, [vp, vp, vp, u32, vp, vp])
    sig("mz_cuda_zip_locate", i32, [vp, vp])
    sig("mz_cuda_zip_copy_stored", i32, [vp, vp])
    sig("mz_cuda_zip_verify", i32, [vp, vp])
    sig("mz_zip_cuda_write_archive", i32, [vp, vp, u32, C.c_int16, u32, vp])
    sig("mz_zip_cuda_write_archive_aes", i32, [vp, vp, u32, C.c_int16, u32, C.c_char_p, C.c_uint8, vp])
    sig("mz_zip_cuda_extract_archive", i32, [vp, C.c_char_p, u32, ZIP_ENTRY_CB, vp, vp])
    sig("mz_zip_cuda_trim", None, [])
    sig("mz_zip_cuda_extract_device", i32, [vp, u64, C.c_char_p, vp, u32, C.POINTER(u32), vp, u64, C.POINTER(u64), vp, vp])
    sig("mz_zip_cuda_write_device", i32, [vp, vp, vp, u32, C.c_int16, u32, C.c_char_p, C.c_uint8, vp, u64, C.POINTER(u64), vp, vp, vp])
    sig("mz_zip_cuda_update_device", i32, [vp, u64, vp, u32, vp, vp, vp, u32, C.c_int16, u32, C.c_char_p, C.c_uint8, vp, u64, C.POINTER(u64), vp, vp,
                                           vp])
    sig("mz_cuda_zip_parse_directory", i32, [vp, u64, vp, vp])
    sig("mz_cuda_zip_statuses", i32, [vp, u32, vp, vp, vp])
    sig("mz_zip_cuda_reader_open", i32, [vp, u64, C.c_char_p, C.POINTER(vp), C.POINTER(u32), C.POINTER(i32), vp, vp])
    sig("mz_zip_cuda_reader_entries", vp, [vp])
    sig("mz_zip_cuda_reader_locate", i32, [vp, vp, vp, vp, u32, C.c_uint8, vp, vp])
    sig("mz_zip_cuda_reader_decode", i32, [vp, vp, u32, vp, u64, C.POINTER(u64), vp, vp, vp, vp])
    sig("mz_zip_cuda_reader_close", None, [vp])
    sig("mz_cuda_zip_name_index", i32, [vp, vp, u32, vp, u32, vp])
    sig("mz_cuda_zip_name_lookup", i32, [vp, vp, vp, u32, vp, vp, vp, u32, C.c_uint8, vp, vp])
    sig("mz_cuda_zip_sel_counts", i32, [vp, vp])
    sig("mz_cuda_zip_sel_fill", i32, [vp, vp])
    sig("mz_cuda_zip_sel_gather", i32, [vp, vp])
    sig("mz_cuda_zip_sel_status", i32, [vp, vp, u32, u32, vp, vp, vp])
    return L


class Shard(C.Structure):
    """mz_cuda_shard (include/mz_cuda_batch.h)"""
    _fields_ = [("device", C.c_int32), ("d_in", C.c_void_p), ("len", C.c_uint64), ("d_gathered", C.c_void_p), ("gathered_cap", C.c_uint64),
                ("d_rows", C.c_void_p)]


def check(err, what="call"):
    if err != MZ_OK:
        msg = load().mz_cuda_last_error()
        raise RuntimeError("%s failed: %d (%s)" % (what, err, msg.decode() if msg else ""))


def _stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class DeflateBatch:
    """Device-resident compression of one buffer cut into independent <=64 KiB chunks (K2+K3, K4, K1).

    Buffers are torch uint8 CUDA tensors; all work is enqueued on torch's current stream.
    """

    def __init__(self, max_bytes, chunk=CHUNK_MAX, with_crc=True):
        import torch
        self.lib = load()
        check(self.lib.mz_cuda_init(), "mz_cuda_init")
        self.chunk = chunk
        self.max_chunks = max(1, (max_bytes + chunk - 1) // chunk)
        self.stride = int(self.lib.mz_cuda_deflate_slot_bound(chunk))
        dev = torch.device("cuda", torch.cuda.current_device())
        self.slots = torch.empty(self.max_chunks * self.stride, dtype=torch.uint8, device=dev)
        self.out_len = torch.empty(self.max_chunks, dtype=torch.int32, device=dev)
        self.offsets = torch.empty(self.max_chunks + 1, dtype=torch.int64, device=dev)
        self.joined = torch.empty(self.max_chunks * self.stride, dtype=torch.uint8, device=dev)
        self.with_crc = with_crc
        if with_crc:
            self.residue = torch.empty(self.max_chunks, dtype=torch.int32, device=dev)
            self.chunk_crc = torch.empty(self.max_chunks, dtype=torch.int32, device=dev)
            self.crc_out = torch.empty(2, dtype=torch.int32, device=dev)

    def nchunks(self, nbytes):
        return max(1, (nbytes + self.chunk - 1) // self.chunk)

    def compress(self, src, nbytes, level=1, final=True, join=True, one_stream=False):
        """Enqueue K2+K3 (+K1 per-chunk CRC and fold) (+K4 join). Returns number of chunks."""
        n = self.nchunks(nbytes)
        assert n <= self.max_chunks and src.is_cuda and src.dtype.itemsize == 1
        s = _stream_ptr()
        check(self.lib.mz_cuda_deflate_chunks(src.data_ptr(), nbytes, self.chunk, None, None, None, n, (FLAG_FINAL if final else 0) | (FLAG_DICT if one_stream else 0),
                                              level, self.slots.data_ptr(), self.stride, self.out_len.data_ptr(), s), "deflate")
        if self.with_crc and nbytes > 0:
            check(self.lib.mz_cuda_crc32_segments(src.data_ptr(), nbytes, self.chunk, None, None, n, self.residue.data_ptr(),
                                                  self.chunk_crc.data_ptr(), s), "crc32")
            check(self.lib.mz_cuda_crc32_fold(self.residue.data_ptr(), n, self.chunk, nbytes, self.crc_out.data_ptr(), s), "crc fold")
        if join:
            check(self.lib.mz_cuda_concat(self.slots.data_ptr(), self.stride, self.out_len.data_ptr(), n, self.offsets.data_ptr(),
                                          self.joined.data_ptr(), s), "concat")
        return n

    def result(self, nchunks):
        """Synchronise and return (joined bytes as a CUDA tensor view, crc32 or None)."""
        import torch
        torch.cuda.current_stream().synchronize()
        total = int(self.offsets[nchunks].item())
        crc = (int(self.crc_out[1].item()) & 0xFFFFFFFF) if self.with_crc else None
        return self.joined[:total], crc


def crc32_device(tensor, nbytes=None, value=0):
    """mz_crypt_crc32_update over a CUDA tensor (K1)."""
    lib = load()
    out = C.c_uint32(0)
    n = tensor.numel() * tensor.element_size() if nbytes is None else nbytes
    check(lib.mz_cuda_crc32_device(tensor.data_ptr(), n, value, C.byref(out)), "crc32_device")
    return out.value


def extract_device(archive, password=None):
    """Extract every entry of a zip archive held in a CUDA uint8 tensor (mz_zip_cuda_extract_device): the directory is parsed and
    the entries decoded on the device. Returns (entries, out): entries = [(name, offset, size, crc)] in directory order, the plain
    bytes of each at out[offset:offset + size] in the CUDA tensor `out`. Raises on any error, as check() does."""
    import torch
    lib = load()
    check(lib.mz_cuda_init(), "mz_cuda_init")
    assert archive.is_cuda and archive.dtype == torch.uint8, "archive: a CUDA uint8 tensor"
    archive = archive.contiguous()
    pw = password.encode() if password is not None else None
    count, nbytes = C.c_uint32(0), C.c_uint64(0)
    s = _stream_ptr()
    n = archive.numel()
    ptr = archive.data_ptr() if n else None
    err = lib.mz_zip_cuda_extract_device(ptr, n, pw, None, 0, C.byref(count), None, 0, C.byref(nbytes), None, s)  # sizes only
    if err not in (MZ_OK, MZ_BUF_ERROR):
        check(err, "extract_device")
    table = torch.empty(max(1, count.value) * C.sizeof(ZipDevEntry), dtype=torch.uint8, device=archive.device)
    out = torch.empty(max(16, nbytes.value), dtype=torch.uint8, device=archive.device)
    check(lib.mz_zip_cuda_extract_device(ptr, n, pw, table.data_ptr(), count.value, C.byref(count), out.data_ptr(), nbytes.value,
                                         C.byref(nbytes), None, s), "extract_device")
    rows = (ZipDevEntry * max(1, count.value)).from_buffer_copy(table.cpu().numpy().tobytes())[:count.value]
    entries = []
    if rows:
        lo = min(r.name_off for r in rows)
        names = archive[lo:max(r.name_off + r.name_len for r in rows)].cpu().numpy().tobytes()
        entries = [(names[r.name_off - lo:r.name_off - lo + r.name_len].decode("utf-8", "replace"), r.out_off, r.usize, r.crc) for r in rows]
    return entries, out[:nbytes.value]


class ZipDeviceReader:
    """Random access to a zip archive held in a CUDA uint8 tensor (mz_zip_cuda_reader_*): the directory is parsed once on the device,
    entries are looked up by name and any subset of them decoded on the device, as often as needed. The tensor must stay unchanged
    while the reader is open; the reader never writes it.

    .entries: [(name, size, crc)] of the accepted entries in directory order (read once at open); .refuse: the error that ended the
    list, or MZ_OK. .locate(names, ignore_case=False): a CUDA int64 tensor of entry indices, -1 for a miss. .read(indices): decodes
    the entries (a CUDA or CPU integer tensor, or a list; repeats and any order allowed) and returns (offsets, out) as CUDA tensors:
    entry k of the selection is out[offsets[k]:offsets[k] + size]. Errors raise, as extract_device's do. .close() or `with`."""

    def __init__(self, archive, password=None):
        import torch
        self.lib = load()
        check(self.lib.mz_cuda_init(), "mz_cuda_init")
        assert archive.is_cuda and archive.dtype == torch.uint8, "archive: a CUDA uint8 tensor"
        self.archive = archive.contiguous()  # kept: the reader reads it until close
        self.device = self.archive.device
        self._r = C.c_void_p()
        n = self.archive.numel()
        count, refuse = C.c_uint32(0), C.c_int32(0)
        with torch.cuda.device(self.device):
            check(self.lib.mz_zip_cuda_reader_open(self.archive.data_ptr() if n else None, n, password.encode() if password is not None else None,
                                                   C.byref(self._r), C.byref(count), C.byref(refuse), None, _stream_ptr()), "reader_open")
        self.count, self.refuse = count.value, refuse.value
        self._rows = []
        self.entries = []
        if self.count:
            table = torch.empty(self.count * C.sizeof(ZipDevEntry), dtype=torch.uint8, device=self.device)
            check(self.lib.mz_cuda_memcpy_d2d(table.data_ptr(), self.lib.mz_zip_cuda_reader_entries(self._r), table.numel(), _stream_ptr()), "entries")
            self._rows = (ZipDevEntry * self.count).from_buffer_copy(table.cpu().numpy().tobytes())
            lo = min(r.name_off for r in self._rows)
            names = self.archive[lo:max(r.name_off + r.name_len for r in self._rows)].cpu().numpy().tobytes()
            self.entries = [(names[r.name_off - lo:r.name_off - lo + r.name_len].decode("utf-8", "replace"), r.usize, r.crc) for r in self._rows]

    def _live(self):
        if not self._r:
            raise RuntimeError("ZipDeviceReader is closed")

    def locate(self, names, ignore_case=False):
        import torch
        self._live()
        raw = [n.encode() if isinstance(n, str) else bytes(n) for n in names]
        out = torch.empty(max(1, len(raw)), dtype=torch.int32, device=self.device)
        if raw:
            blob = b"".join(raw) or b"\0"
            offs, pos = [], 0
            for r in raw:
                offs.append(pos)
                pos += len(r)
            d_names = torch.frombuffer(bytearray(blob), dtype=torch.uint8).to(self.device)
            d_off = torch.tensor(offs, dtype=torch.int64, device=self.device)
            d_len = torch.tensor([len(r) for r in raw], dtype=torch.int32, device=self.device)
            with torch.cuda.device(self.device):
                check(self.lib.mz_zip_cuda_reader_locate(self._r, d_names.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), len(raw), 1 if ignore_case else 0,
                                                         out.data_ptr(), _stream_ptr()), "reader_locate")
        return out[:len(raw)].to(torch.int64)  # a miss, 0xffffffff, reads as -1

    def read(self, indices):
        import torch
        self._live()
        sel = torch.as_tensor(indices, dtype=torch.int64).to(self.device).reshape(-1)
        # an index outside the entries (a miss from locate included) becomes 0xffffffff: the decode reports MZ_END_OF_LIST for it
        d_sel = torch.where((sel < 0) | (sel >= self.count), torch.full_like(sel, -1), sel).to(torch.int32)
        n = d_sel.numel()
        offs = torch.empty(n + 1, dtype=torch.int64, device=self.device)
        size = C.c_uint64(0)
        s = _stream_ptr()
        with torch.cuda.device(self.device):
            check(self.lib.mz_zip_cuda_reader_decode(self._r, d_sel.data_ptr() if n else None, n, None, 0, C.byref(size), None, None, None, s), "reader_decode")
            out = torch.empty(max(16, size.value), dtype=torch.uint8, device=self.device)
            check(self.lib.mz_zip_cuda_reader_decode(self._r, d_sel.data_ptr() if n else None, n, out.data_ptr(), size.value, C.byref(size),
                                                     offs.data_ptr(), None, None, s), "reader_decode")
        return offs, out[:size.value]

    def close(self):
        if self._r:
            self.lib.mz_zip_cuda_reader_close(self._r)
            self._r = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001 -- interpreter shutdown
            pass


def write_device(files, level=6, sha256=False, password=None, aes_strength=3, mtime=None):
    """Write a zip archive into device memory from entries in device memory (mz_zip_cuda_write_device): files = [(name, CUDA uint8
    tensor)], all on the current device; the tensors may be separate allocations. The archive is what write_archive writes for the same
    bytes (with a password: WinZip AES of aes_strength). mtime: unix time of every entry (None = now). Returns a CUDA uint8 tensor of
    exactly the archive's length. Raises on any error, as check() does."""
    import torch
    lib = load()
    check(lib.mz_cuda_init(), "mz_cuda_init")
    dev = torch.device("cuda", torch.cuda.current_device())
    flags = (MZ_ZIP_CUDA_HASH_SHA256 if sha256 else 0) | (MZ_ZIP_CUDA_AES if password is not None else 0)
    base, d_names, d_items = _dev_items(files, dev, mtime)
    pw = password.encode() if password is not None else None
    s = _stream_ptr()
    n = C.c_uint64(0)
    args = (base or None, d_names.data_ptr(), d_items.data_ptr(), len(files), level, flags, pw, aes_strength)
    check(lib.mz_zip_cuda_write_device(*args, None, 0, C.byref(n), None, None, s), "write_device")  # sizing: an upper bound
    out = torch.empty(max(1, n.value), dtype=torch.uint8, device=dev)
    check(lib.mz_zip_cuda_write_device(*args, out.data_ptr(), n.value, C.byref(n), None, None, s), "write_device")
    return out[:n.value].clone()  # the bound-sized buffer is released: the archive's own storage is exactly its length


def _dev_items(files, dev, mtime):
    """-> (base, d_names, d_items): the mz_cuda_zip_dev_item table of files = [(name, CUDA uint8 tensor)] on dev, data offsets from
    base (the lowest data pointer, 0 without data); the tensors in `files` must stay alive while the table is used"""
    import time
    import torch
    date = dos_date(int(time.time() if mtime is None else mtime))
    tensors = []
    for name, t in files:
        assert t.is_cuda and t.dtype == torch.uint8 and t.device == dev, "%s: a CUDA uint8 tensor on the current device" % name
        tensors.append(t.contiguous())
    ptrs = [t.data_ptr() for t in tensors if t.numel()]
    base = min(ptrs) if ptrs else 0
    names = [n.encode() for n, _ in files]
    blob = b"".join(names)
    d_names = torch.frombuffer(bytearray(blob or b"\0"), dtype=torch.uint8).to(dev)
    items = (ZipDevItem * max(1, len(files)))()
    pos = 0
    for i, (nm, t) in enumerate(zip(names, tensors)):
        items[i] = ZipDevItem(t.data_ptr() - base if t.numel() else 0, t.numel(), pos, len(nm), date, 0, 0)
        pos += len(nm)
    d_items = torch.frombuffer(bytearray(bytes(items)), dtype=torch.uint8).to(dev)
    return base, d_names, d_items


def update_device(archive, keep=None, files=(), level=6, sha256=False, password=None, aes_strength=3, mtime=None):
    """Update a zip archive held in a CUDA uint8 tensor without recompressing the entries it keeps (mz_zip_cuda_update_device): the
    kept entries are copied as raw bytes and their directory records rewritten, then `files` (as write_device takes them) are appended.
    keep: None keeps every entry (append); otherwise entry indices as ZipDeviceReader.entries and .locate give them (a list, or a CPU
    or CUDA integer tensor; any order, repeats allowed; empty keeps none), or a boolean mask over the entries (the entries where it is
    True, in order), e.g. a locate followed by a mask to drop files by name. Kept WinZip AES entries
    stay encrypted under their own password; `password` applies to the new entries. The archive's comment is kept. Returns a new CUDA
    uint8 tensor of exactly the archive's length; `archive` is not changed. Raises on any error, as check() does."""
    import torch
    lib = load()
    check(lib.mz_cuda_init(), "mz_cuda_init")
    dev = torch.device("cuda", torch.cuda.current_device())
    assert archive.is_cuda and archive.dtype == torch.uint8 and archive.device == dev, "archive: a CUDA uint8 tensor on the current device"
    src = archive.contiguous()
    d_keep, nkeep = None, 0
    if keep is not None:
        k = torch.as_tensor(keep)
        if k.numel() == 0:  # [] comes as float32: an empty list of indices
            k = torch.empty(0, dtype=torch.int64)
        if k.dtype == torch.bool:  # a mask over the entries: keep the entries it selects
            k = k.reshape(-1).nonzero().reshape(-1)
        if k.is_floating_point() or k.is_complex():
            raise TypeError("update_device: keep holds entry indices or a boolean mask")
        k = k.to(torch.int64).reshape(-1)
        if k.numel() and bool((k < 0).any()):
            raise ValueError("update_device: negative entry index")
        # never NULL: the C call reads a NULL d_keep as "keep every entry", an empty list keeps none
        d_keep = torch.zeros(max(1, k.numel()), dtype=torch.int32, device=dev)
        d_keep[:k.numel()] = k.to(torch.int32).to(dev)
        nkeep = k.numel()
    flags = (MZ_ZIP_CUDA_HASH_SHA256 if sha256 else 0) | (MZ_ZIP_CUDA_AES if password is not None else 0)
    base, d_names, d_items = _dev_items(files, dev, mtime)
    pw = password.encode() if password is not None else None
    s = _stream_ptr()
    n = C.c_uint64(0)
    args = (src.data_ptr() if src.numel() else None, src.numel(), d_keep.data_ptr() if d_keep is not None else None, nkeep,
            base or None, d_names.data_ptr(), d_items.data_ptr(), len(files), level, flags, pw, aes_strength)
    check(lib.mz_zip_cuda_update_device(*args, None, 0, C.byref(n), None, None, s), "update_device")  # sizing: an upper bound
    out = torch.empty(max(1, n.value), dtype=torch.uint8, device=dev)
    check(lib.mz_zip_cuda_update_device(*args, out.data_ptr(), n.value, C.byref(n), None, None, s), "update_device")
    return out[:n.value].clone()


def inflate_device(comp, out_cap):
    """Decode ONE raw deflate stream held in a CUDA uint8 tensor (padded >=16 bytes). Returns (status, out tensor, consumed)."""
    import torch
    lib = load()
    dev = comp.device
    n = comp.numel()
    padded = torch.zeros(n + 64, dtype=torch.uint8, device=dev)
    padded[:n] = comp
    out = torch.empty(out_cap + 512, dtype=torch.uint8, device=dev)
    job = InflateJob(padded.data_ptr(), 0, n, out.data_ptr(), 0, out_cap, 1, 0)
    st = InflateState()
    d_job = torch.frombuffer(bytearray(bytes(job)), dtype=torch.uint8).to(dev)
    d_st = torch.zeros(C.sizeof(InflateState), dtype=torch.uint8, device=dev)
    check(lib.mz_cuda_inflate_streams(d_job.data_ptr(), d_st.data_ptr(), 1, _stream_ptr()), "inflate")
    torch.cuda.current_stream().synchronize()
    raw = bytes(d_st.cpu().numpy().tobytes())
    C.memmove(C.byref(st), raw, C.sizeof(InflateState))
    return st.status, out[:st.out_pos], (st.in_bitpos + 7) // 8, st
