"""Runs both batch extractors on one archive in one process and prints what each delivered, entry by entry, as one JSON line:
mz_zip_cuda_extract_all over the reference's own zip reader (oracle/_ref/libmzref.so, loaded first and globally, so that the
product's weak mz_zip_* references resolve to it), and mz_zip_cuda_extract_archive, both from the same 64-bit memory base stream
(tests/support/libmztest.so).

    python tests/extract_pair.py <product library> <archive> [password]

It runs in its own process because a product library loaded earlier without the reference has its weak references bound to NULL.
"""
import ctypes as C
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

MZ_OPEN_MODE_READ = 1


def load(product):
    """the reference's zip reader (global), the memory stream, then the product; returns (reference, product, TestLib)"""
    ref = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libmzref.so"), mode=C.RTLD_GLOBAL)
    ref.mz_zip_create.restype = C.c_void_p
    ref.mz_zip_open.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
    ref.mz_zip_close.argtypes = [C.c_void_p]
    ref.mz_zip_delete.argtypes = [C.POINTER(C.c_void_p)]
    import cuharness
    lib = cuharness.pkg().configure(C.CDLL(product))
    lib.mz_zip_cuda_extract_all_aes.restype = C.c_int32
    lib.mz_zip_cuda_extract_all_aes.argtypes = [C.c_void_p, C.c_char_p, lib.mz_zip_cuda_extract_archive.argtypes[3], C.c_void_p, C.c_void_p]
    return ref, lib, cuharness.TestLib()


class Pair:
    """both extractors over one memory base stream holding `archive`"""

    def __init__(self, product, archive):
        self.ref, self.lib, self.t = load(product)
        import cuharness
        self.pkg = cuharness.pkg()
        self.src, self._keep = self.t.source(archive)

    def run(self, which, password=None, flags=0, on_entry=None):
        """-> (err, stats); which = 'all' (reference directory walk) or 'native'"""
        cb = self.pkg.ZIP_ENTRY_CB(on_entry or (lambda *a: 0))
        st = self.pkg.ZipStats()
        pw = password.encode() if password else None
        if which == "native":
            return self.lib.mz_zip_cuda_extract_archive(self.src, pw, flags, cb, None, C.byref(st)), st
        zip_ = self.ref.mz_zip_create()
        err = self.ref.mz_zip_open(zip_, self.src, MZ_OPEN_MODE_READ)
        if err == 0:
            err = self.lib.mz_zip_cuda_extract_all_aes(zip_, pw, cb, None, C.byref(st))
            self.ref.mz_zip_close(zip_)
        z = C.c_void_p(zip_)
        self.ref.mz_zip_delete(C.byref(z))
        return err, st

    def close(self):
        self.t.delete(self.src)


def main():
    product, path = sys.argv[1], sys.argv[2]
    password = sys.argv[3] if len(sys.argv) > 3 else None
    pair = Pair(product, open(path, "rb").read())
    out = {}
    for which in ("all", "native"):
        got = []

        def on_entry(_ud, name, data, size, crc):
            got.append([name.decode(), hashlib.sha256(C.string_at(data, size) if size else b"").hexdigest(), size, crc])
            return 0
        err, _ = pair.run(which, password, 0, on_entry)
        out[which] = {"err": err, "entries": got}
    pair.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
