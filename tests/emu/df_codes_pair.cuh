/* df_codes_pair.cuh -- runs the deflate kernel's code builder (block_build_codes) and its frozen v3.4 form (df_codes_v34.cuh) on
 * the same histograms and writes what each produced (TEST INFRASTRUCTURE ONLY). Compiled by g++ on the CPU emulator
 * (emu_df_codes.cc) and by nvcc for sm_90a (gpu_df_codes.cu); the tests compare the two outputs byte for byte.
 *
 * One histogram = DFC_HIST_WORDS words: literal/length counts [0, 288), distance counts [288, 320), the second copy of the literal
 * counts [320, 576) -- the kernel's DF_OFF_HIST + DF_OFF_HIST2 layout. posfin[h] = header bit position (bits 0-6) | BFINAL << 31.
 * One result = DFC_OUT_WORDS words: code words [0, 320), code lengths as bytes [320, 400), bits per symbol as bytes [400, 480),
 * the staging words the header went into [480, 480 + DF_HDR_WORDS), the header size in bits (bb[BB_HDRBITS]) at DFC_OUT_HDRBITS. */
#ifndef MZ_DF_CODES_PAIR_CUH
#define MZ_DF_CODES_PAIR_CUH

#include "df_codes_v34.cuh"

namespace mzc {

constexpr int DFC_HIST_WORDS = 288 + 32 + 256;
constexpr int DFC_OUT_STAGE = 480;
constexpr int DFC_OUT_HDRBITS = DFC_OUT_STAGE + DF_HDR_WORDS;
constexpr int DFC_OUT_WORDS = DFC_OUT_HDRBITS + 8;

template <bool OLD>
__global__ void __launch_bounds__(DF_BB_THREADS) df_codes_pair_kernel(const uint32_t *hists, const uint32_t *posfin, uint32_t n, uint32_t *out) {
    __shared__ uint32_t s_hist[DFC_HIST_WORDS];
    __shared__ uint32_t s_code[320];
    __shared__ uint32_t s_lb[160]; /* lens (320 bytes), then bits (320 bytes) */
    __shared__ uint32_t s_bb[512];
    __shared__ uint32_t s_stage[DF_HDR_WORDS];
    const uint32_t tid = threadIdx.x;
    uint8_t *lens = (uint8_t *)s_lb, *bits = lens + 320;
    for (uint32_t h = blockIdx.x; h < n; h += gridDim.x) {
        for (uint32_t i = tid; i < (uint32_t)DFC_HIST_WORDS; i += DF_BB_THREADS) s_hist[i] = hists[(size_t)h * DFC_HIST_WORDS + i];
        /* what the builder must overwrite starts as garbage, the scratch too (the kernel leaves it dirty from the unit before);
         * the staging words start clean, as in the kernel */
        for (uint32_t i = tid; i < 512; i += DF_BB_THREADS) s_bb[i] = 0xa5a5a5a5u ^ (i * 2654435761u) ^ h;
        for (uint32_t i = tid; i < 320; i += DF_BB_THREADS) s_code[i] = 0xdeadbeefu;
        for (uint32_t i = tid; i < 160; i += DF_BB_THREADS) s_lb[i] = 0x5a5a5a5au;
        for (uint32_t i = tid; i < (uint32_t)DF_HDR_WORDS; i += DF_BB_THREADS) s_stage[i] = 0;
        __syncthreads();
        const uint32_t pos = posfin[h] & 127u, fin = posfin[h] >> 31;
        if (OLD)
            v34::block_build_codes_v34(s_hist, s_hist + 320, s_hist + 288, lens, lens + 288, s_code, s_code + 288, bits, bits + 288, s_bb,
                                       s_stage, pos, fin);
        else
            block_build_codes(s_hist, s_hist + 320, s_hist + 288, lens, lens + 288, s_code, s_code + 288, bits, bits + 288, s_bb, s_stage,
                              pos, fin);
        __syncthreads();
        uint32_t *o = out + (size_t)h * DFC_OUT_WORDS;
        for (uint32_t i = tid; i < 320; i += DF_BB_THREADS) o[i] = s_code[i];
        for (uint32_t i = tid; i < 160; i += DF_BB_THREADS) o[320 + i] = s_lb[i];
        for (uint32_t i = tid; i < (uint32_t)DF_HDR_WORDS; i += DF_BB_THREADS) o[DFC_OUT_STAGE + i] = s_stage[i];
        if (tid < 8) o[DFC_OUT_HDRBITS + tid] = tid == 0 ? s_bb[OLD ? (int)v34::BB_HDRBITS : (int)BB_HDRBITS] : 0u;
        __syncthreads();
    }
}

} /* namespace mzc */

#endif
