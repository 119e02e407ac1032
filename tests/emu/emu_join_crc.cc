/* emu_join_crc.cc -- the join copy (gather_slots_kernel, with scan_lengths_kernel) and the CRC segments kernel on the CPU
 * emulator, with buffers sized to the byte so that AddressSanitizer sees a read past them (TEST INFRASTRUCTURE ONLY).
 * Built together with cuda_emu.cc by tests/test_emu_join_crc_alignment.py, plain and with sanitizers; never part of the
 * product library. */
#define MZ_EMU 1
#include "../../minizip-ng_b200/csrc/concat_kernel.cuh"
#include "../../minizip-ng_b200/csrc/crc32_kernel.cuh"

#include <memory>

using namespace mzc;

static CrcConsts g_consts;
static bool g_ready;
static void ensure() {
    if (!g_ready) {
        crc_consts_init(g_consts);
        g_ready = true;
    }
}

extern "C" {

/* The join on its own: n slots of `stride` bytes (copied into an allocation of exactly n * stride bytes) go to dst + offsets[i].
 * With offsets == NULL they are packed (the exclusive scan of len, as mz_cuda_concat does) and the n + 1 offsets are written to
 * offs_out; otherwise they are explicit destinations (mz_cuda_gather). dst holds dst_len bytes; the kernel sees it at an address
 * that is `misalign` (0..15) past a 16-byte boundary, in an allocation that ends at the first 16-byte boundary at or after its
 * last byte. */
void emu_join(const uint8_t *slots_in, uint64_t stride, const uint32_t *len, uint32_t n, const uint64_t *offsets, uint8_t *dst_io,
              uint64_t dst_len, uint32_t misalign, uint64_t *offs_out) {
    std::unique_ptr<uint8_t, decltype(&free)> sl((uint8_t *)aligned_alloc(16, (size_t)(stride * n + (n ? 0 : 16))), &free);
    memcpy(sl.get(), slots_in, (size_t)(stride * n));
    misalign &= 15;
    const size_t dcap = ((size_t)misalign + (size_t)dst_len + 15) & ~(size_t)15;
    std::unique_ptr<uint8_t, decltype(&free)> db((uint8_t *)aligned_alloc(16, dcap ? dcap : 16), &free);
    uint8_t *d = db.get() + misalign;
    memcpy(d, dst_io, (size_t)dst_len);
    std::vector<uint64_t> offs(n + 1);
    if (offsets)
        memcpy(offs.data(), offsets, (size_t)n * 8);
    else
        MZ_LAUNCH(scan_lengths_kernel, dim3(1), dim3(SCAN_THREADS), 0, 0, len, n, (uint64_t)0, offs.data());
    if (n) MZ_LAUNCH(gather_slots_kernel, dim3(n < 24 ? (n + 7) / 8 : 3), dim3(GATHER_THREADS), 0, 0, (const uint8_t *)sl.get(), stride, len,
                     (const uint64_t *)offs.data(), n, d);
    memcpy(dst_io, d, (size_t)dst_len);
    if (offs_out) memcpy(offs_out, offs.data(), (size_t)(n + 1) * 8);
}

/* crc32_segments_kernel over explicit (ragged) segments: off[i], len[i] into `in`, which is placed `misalign` bytes past a
 * 16-byte boundary; residues and finalized CRCs per segment */
void emu_crc32_segments(const uint8_t *in, uint64_t total, const uint64_t *off, const uint32_t *len, uint32_t nseg, uint32_t misalign,
                        uint32_t *res_out, uint32_t *crc_out) {
    ensure();
    misalign &= 15;
    std::unique_ptr<uint8_t, decltype(&free)> buf((uint8_t *)aligned_alloc(16, (misalign + total + 15) & ~15ull), &free);
    uint8_t *a = buf.get() + misalign;
    memcpy(a, in, (size_t)total);
    CrcParams P;
    memset(&P, 0, sizeof(P));
    P.in = a;
    P.in_off = off;
    P.in_len = len;
    P.nseg = nseg;
    P.consts = &g_consts;
    P.out_residue = res_out;
    P.out_crc = crc_out;
    if (nseg) MZ_LAUNCH(crc32_segments_kernel, dim3(2), dim3(CRC_THREADS), CRC_SMEM_BYTES, 0, P);
}


/* crc32_segments_kernel over a uniform partition of `in` into seg_size-byte segments (the last may be shorter), `in` placed
 * `misalign` bytes past a 16-byte boundary; finalized CRCs per segment */
void emu_crc32_uniform(const uint8_t *in, uint64_t total, uint64_t seg_size, uint32_t misalign, uint32_t *crc_out) {
    ensure();
    misalign &= 15;
    std::unique_ptr<uint8_t, decltype(&free)> buf((uint8_t *)aligned_alloc(16, (misalign + total + 15) & ~15ull), &free);
    uint8_t *a = buf.get() + misalign;
    memcpy(a, in, (size_t)total);
    const uint32_t nseg = (uint32_t)((total + seg_size - 1) / seg_size);
    std::vector<uint32_t> res(nseg + 1);
    CrcParams P;
    memset(&P, 0, sizeof(P));
    P.in = a;
    P.total_len = total;
    P.seg_size = seg_size;
    P.nseg = nseg;
    P.consts = &g_consts;
    P.out_residue = res.data();
    P.out_crc = crc_out;
    P.init_len = seg_size;
    P.init = crc_init_term(g_consts, seg_size);
    if (nseg) MZ_LAUNCH(crc32_segments_kernel, dim3(2), dim3(CRC_THREADS), CRC_SMEM_BYTES, 0, P);
}
}
