/* gzip_kernel.cuh -- K14: one gzip member (RFC 1952) written into device memory from a buffer in device memory
 * (mz_cuda_gzip_compress_device, include/mz_cuda_batch.h; launches: mz_cuda_gzip_place / mz_cuda_gzip_trailer in mz_cuda_api.cu).
 *
 * The member is   10-byte header | one raw DEFLATE stream of the whole buffer | CRC-32 | ISIZE.
 * The buffer is compressed in rounds of 64 KiB chunks (K2+K3 into slots); per round
 *   place    an exclusive scan of the round's stream lengths (the K10 scan kernels for the tiles' sums, then this kernel), carried in
 *            from the previous round by S[c0] in device memory: S(c) = the stream bytes in front of chunk c, its destination head + S(c),
 *            and copy length 0 for a chunk whose bytes would pass `cap`. K4 mz_cuda_gather copies the slots straight into the member.
 *            This is K11's place (zipwr_kernel.cuh) for a single entry whose stream starts `head` bytes into the output.
 *   trailer  after the last round and the CRC fold (K1): the 8 trailer bytes behind the stream when all of them fit below `cap`, and
 *            the member's exact length for the host.
 * No CTA waits on another, so the kernels also run on the CPU emulator.
 */
#ifndef MZ_GZIP_KERNEL_CUH
#define MZ_GZIP_KERNEL_CUH

#include "mzcuda_common.cuh"
#include "zipcd_kernel.cuh"

namespace mzc {

/* chunks [c0, c0 + m), per tile of ZC_TILE chunks, with part[] the exclusive prefix of the tiles' stream bytes (zc_scan_reduce /
 * zc_scan_parts over out_len + c0); S[c0 + m] carries the total into the next round */
__global__ void __launch_bounds__(ZC_THREADS) gz_place_kernel(const uint32_t *out_len, uint64_t c0, uint32_t m, const uint32_t *part, uint64_t *S,
                                                              uint64_t *dst, uint32_t *glen, uint64_t head, uint64_t cap) {
    __shared__ uint64_t s[ZC_THREADS];
    const uint64_t base = S[c0];
    const uint32_t b0 = blockIdx.x * ZC_TILE + threadIdx.x * ZC_ITEMS;
    uint64_t v = 0;
    for (uint32_t k = 0; k < ZC_ITEMS; k++)
        if (b0 + k < m) v += out_len[c0 + b0 + k];
    uint64_t tot;
    uint64_t run = base + part[blockIdx.x] + zc_block_scan<uint64_t>(v, s, &tot);
    for (uint32_t k = 0; k < ZC_ITEMS; k++) {
        const uint32_t j = b0 + k;
        if (j > m) break;
        const uint64_t c = c0 + j;
        if (j) S[c] = run; /* S[c0] is the previous round's: read above by every thread, not written again */
        if (j == m) break;
        const uint32_t len = out_len[c];
        const uint64_t d = head + run;
        dst[c] = d;
        glen[c] = d + len <= cap ? len : 0u;
        run += len;
    }
}

/* one warp: lanes 0..7 write CRC-32 and ISIZE (len mod 2^32) little-endian behind the stream (S_end bytes from head) when the whole
 * trailer lies below cap; lane 0 stores the member's length */
__global__ void __launch_bounds__(32) gz_trailer_kernel(const uint64_t *S_end, const uint32_t *crc, uint64_t len, uint64_t head, uint8_t *out,
                                                        uint64_t cap, uint64_t *total) {
    const uint32_t lane = threadIdx.x;
    const uint64_t p = head + *S_end;
    if (lane < 8 && p + 8 <= cap) out[p + lane] = (uint8_t)((lane < 4 ? *crc : (uint32_t)len) >> (8 * (lane & 3)));
    if (lane == 0) *total = p + 8;
}

} // namespace mzc
#endif
