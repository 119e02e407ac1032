/* concat_kernel.cuh -- K4: join per-chunk bitstreams (byte-aligned by construction) into one stream.
 *
 * Every chunk slot ends on a byte boundary (sync-flush marker or final padding, see deflate_kernel.cuh),
 * so concatenation is an exclusive scan over out_len[] followed by a gather-copy. The result is one
 * valid RFC1951 stream: what mz_stream_zlib_write + close hand to the base stream (mz_strm_zlib.c:196-201).
 */
#ifndef MZ_CONCAT_KERNEL_CUH
#define MZ_CONCAT_KERNEL_CUH

#include "mzcuda_common.cuh"

namespace mzc {

constexpr int SCAN_THREADS = 1024;

/* exclusive scan of n 32-bit lengths into 64-bit offsets; offsets[n] = total. Single CTA. */
__global__ void __launch_bounds__(SCAN_THREADS, 1) scan_lengths_kernel(const uint32_t *len, uint32_t n, uint64_t base, uint64_t *offsets) {
    __shared__ uint64_t s_part[SCAN_THREADS];
    const uint32_t tid = threadIdx.x;
    const uint32_t per = (n + SCAN_THREADS - 1) / SCAN_THREADS;
    const uint64_t lo = (uint64_t)tid * per;
    uint64_t sum = 0;
    for (uint32_t k = 0; k < per; k++)
        if (lo + k < n) sum += len[lo + k];
    s_part[tid] = sum;
    __syncthreads();
    /* Hillis-Steele inclusive scan over the 1024 partial sums */
    for (uint32_t d = 1; d < SCAN_THREADS; d <<= 1) {
        uint64_t v = tid >= d ? s_part[tid - d] : 0;
        __syncthreads();
        s_part[tid] += v;
        __syncthreads();
    }
    uint64_t run = base + s_part[tid] - sum;
    for (uint32_t k = 0; k < per; k++)
        if (lo + k < n) {
            offsets[lo + k] = run;
            run += len[lo + k];
        }
    if (tid == SCAN_THREADS - 1) offsets[n] = base + s_part[tid];
}

constexpr int GATHER_THREADS = 256;
constexpr int GATHER_CTAS_PER_SM = 4;  /* 32 warps per SM */
constexpr int GATHER_UNROLL = 4;       /* 16-byte loads in flight per lane: 2 KiB per warp, 64 KiB per SM */

/* the 16 bytes that start at byte sh (0..15) of the 32-byte string lo || hi (little-endian words) */
__device__ __forceinline__ uint4 bytes_at(uint4 lo, uint4 hi, uint32_t sh) {
    const bool s8 = (sh & 8) != 0, s4 = (sh & 4) != 0;
    /* whole-word part of the shift: by two words, then by one */
    const uint32_t b0 = s8 ? lo.z : lo.x, b1 = s8 ? lo.w : lo.y, b2 = s8 ? hi.x : lo.z, b3 = s8 ? hi.y : lo.w, b4 = s8 ? hi.z : hi.x,
                   b5 = s8 ? hi.w : hi.y;
    const uint32_t c0 = s4 ? b1 : b0, c1 = s4 ? b2 : b1, c2 = s4 ? b3 : b2, c3 = s4 ? b4 : b3, c4 = s4 ? b5 : b4;
    const uint32_t f = (sh & 3) * 8; /* byte part; a funnel shift by 0 returns the low word */
    return make_uint4(__funnelshift_r(c0, c1, f), __funnelshift_r(c1, c2, f), __funnelshift_r(c2, c3, f), __funnelshift_r(c3, c4, f));
}

__device__ __forceinline__ uint4 shfl_uint4(uint4 v, int src) {
    return make_uint4(__shfl_sync(MZ_FULL_MASK, v.x, src), __shfl_sync(MZ_FULL_MASK, v.y, src), __shfl_sync(MZ_FULL_MASK, v.z, src),
                      __shfl_sync(MZ_FULL_MASK, v.w, src));
}

/* Copy slot c (16-byte aligned, slot_stride apart) to dst + offsets[c] (any alignment), one warp per slot, warps striding over
 * the slots. Destination bytes fall into three parts:
 *   - interior: the 16-byte aligned words that lie wholly inside the slot's range. Each is one 16-byte store, built from the two
 *     source words that cover it, shifted by head = (-(dst + offsets[c])) mod 16 bytes. Lane l holds source words i0 + l + 32u
 *     (u < GATHER_UNROLL, all loaded before the first store); the next word comes from lane l + 1, or for lane 31 from lane 0 of
 *     the next u, or from one more load after the last u.
 *   - head and tail: the bytes before the first and after the last interior word (fewer than 16 each). They are byte stores:
 *     the word they sit in may also hold bytes of the neighbouring slots (many tiny slots can share one word), whose warps
 *     write their own bytes of it.
 * A source word is read only if it holds at least one of the slot's bytes, so a slot is never read past the 16-byte word
 * that holds its last byte. */
__global__ void __launch_bounds__(GATHER_THREADS, GATHER_CTAS_PER_SM)
    gather_slots_kernel(const uint8_t *__restrict__ slots, uint64_t slot_stride, const uint32_t *__restrict__ len, const uint64_t *__restrict__ offsets,
                        uint32_t n, uint8_t *__restrict__ dst) {
    const unsigned lane = lane_id();
    const int next_lane = (int)((lane + 1) & 31);
    const uint32_t nwarps = gridDim.x * (GATHER_THREADS / 32);
    uint32_t c = blockIdx.x * (GATHER_THREADS / 32) + warp_id();
    uint64_t off = 0;
    uint32_t nbytes = 0;
    if (c < n) {
        off = offsets[c];
        nbytes = len[c];
    }
    for (; c < n; c += nwarps) {
        /* the next slot's place and length are loaded while this one is copied */
        const uint32_t cn = c + nwarps;
        uint64_t off_next = 0;
        uint32_t nbytes_next = 0;
        if (cn < n) {
            off_next = offsets[cn];
            nbytes_next = len[cn];
        }
        const uint8_t *src = slots + (uint64_t)c * slot_stride;
        uint8_t *d = dst + off;
        const uint32_t head = (uint32_t)(0 - (uintptr_t)d) & 15u;
        const uint32_t nh = head < nbytes ? head : nbytes;
        const uint32_t nw = (nbytes - nh) >> 4; /* interior words */
        const uint32_t tail = nh + (nw << 4);   /* first tail byte; nbytes - tail < 16 */
        if (lane < nh)
            d[lane] = src[lane];
        else if (lane >= 16 && lane - 16 < nbytes - tail)
            d[tail + lane - 16] = src[tail + lane - 16];
        /* interior word i is bytes head .. head + 15 of source words i, i + 1; word nw is needed (and holds slot bytes) iff head != 0 */
        const uint32_t nread = nw + (nw != 0 && head != 0 ? 1u : 0u);
        const uint4 *sw = (const uint4 *)src;
        uint4 *dw = (uint4 *)(d + nh);
        const uint4 zero = make_uint4(0, 0, 0, 0);
        for (uint32_t i0 = 0; i0 < nw; i0 += 32 * GATHER_UNROLL) {
            uint4 w[GATHER_UNROLL];
#pragma unroll
            for (int u = 0; u < GATHER_UNROLL; u++) {
                const uint32_t x = i0 + 32 * u + lane;
                w[u] = x < nread ? ldg_stream(sw + x) : zero;
            }
            const uint32_t xe = i0 + 32 * GATHER_UNROLL;
            const uint4 extra = lane == 31 && xe < nread ? ldg_stream(sw + xe) : zero;
            uint4 r = shfl_uint4(w[0], next_lane);
#pragma unroll
            for (int u = 0; u < GATHER_UNROLL; u++) {
                const uint4 rn = u + 1 < GATHER_UNROLL ? shfl_uint4(w[u + 1 < GATHER_UNROLL ? u + 1 : u], next_lane) : extra;
                const uint32_t x = i0 + 32 * u + lane;
                if (x < nw) dw[x] = bytes_at(w[u], lane == 31 ? rn : r, head);
                r = rn;
            }
        }
        off = off_next;
        nbytes = nbytes_next;
    }
}

/* copy n small blobs (zip local headers) from a packed source to dst + dst_off[i]: one warp per blob, byte copies */
__global__ void __launch_bounds__(256) scatter_blobs_kernel(const uint8_t *blob, const uint32_t *blob_off, const uint64_t *dst_off, uint32_t n, uint8_t *dst) {
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i = warp; i < n; i += nwarps) {
        const uint32_t a = blob_off[i], b = blob_off[i + 1];
        uint8_t *d = dst + dst_off[i];
        for (uint32_t k = a + lane; k < b; k += 32) d[k - a] = blob[k];
    }
}

/* per-chunk rows {crc32, in_len, out_len} for the multi-GPU table (one thread per chunk) */
__global__ void __launch_bounds__(256) pack_rows_kernel(const uint32_t *chunk_crc, const uint32_t *out_len, uint32_t nchunks, uint64_t total_len,
                                                        uint32_t chunk_size, uint32_t *rows) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= nchunks) return;
    const uint64_t off = (uint64_t)c * chunk_size;
    const uint64_t rem = total_len - off;
    rows[3 * c] = chunk_crc[c];
    rows[3 * c + 1] = rem < chunk_size ? (uint32_t)rem : chunk_size;
    rows[3 * c + 2] = out_len[c];
}

} // namespace mzc
#endif
