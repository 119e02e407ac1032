/* emu_df_codes.cc -- the code-builder equivalence harness on the CPU emulator (TEST INFRASTRUCTURE ONLY): captures the per-unit
 * histograms the deflate kernel hands its code builder, and runs today's and the frozen v3.4 builder on given histograms
 * (df_codes_pair.cuh). Built together with cuda_emu.cc by tests/test_emu_df_codes_equiv.py; never part of the product library. */
#define MZ_EMU 1
#include <stdint.h>
#include <vector>

static std::vector<uint32_t> g_captured; /* DFC_HIST_WORDS words per histogram */
static void df_capture(const uint32_t *ll, const uint32_t *lit2, const uint32_t *d) {
    g_captured.insert(g_captured.end(), ll, ll + 288);
    g_captured.insert(g_captured.end(), d, d + 32);
    g_captured.insert(g_captured.end(), lit2, lit2 + 256);
}
#define MZ_DF_CODES_HOOK(ll, lit2, d) df_capture(ll, lit2, d)

#include "../../minizip-ng_b200/csrc/deflate_kernel.cuh"
#include "df_codes_pair.cuh"

using namespace mzc;

extern "C" {

uint32_t emu_df_hist_words(void) { return DFC_HIST_WORDS; }
uint32_t emu_df_out_words(void) { return DFC_OUT_WORDS; }

/* Deflate `in` as one buffer of 64 KiB chunks (the last one FINAL) at `level` and return how many histograms the code builder
 * was given; up to `cap` of them are copied to out (DFC_HIST_WORDS words each). */
uint32_t emu_df_capture(const uint8_t *in, uint64_t len, int level, uint32_t *out, uint32_t cap) {
    const uint32_t chunk = 65536, nchunks = (uint32_t)((len + chunk - 1) / chunk);
    const uint64_t stride = deflate_slot_bound(chunk);
    std::vector<uint8_t> slots((size_t)(stride * nchunks + 64));
    std::vector<uint8_t> inbuf((size_t)len + 64);
    uint8_t *ia = (uint8_t *)(((uintptr_t)inbuf.data() + 15) & ~(uintptr_t)15);
    memcpy(ia, in, (size_t)len);
    std::vector<uint32_t> out_len(nchunks);
    DeflateParams P;
    memset(&P, 0, sizeof(P));
    P.in = ia;
    P.total_len = len;
    P.chunk_size = chunk;
    P.nchunks = nchunks;
    P.last_flags = DF_FLAG_FINAL;
    P.level = level;
    P.out = (uint8_t *)(((uintptr_t)slots.data() + 15) & ~(uintptr_t)15);
    P.slot_stride = stride;
    P.out_len = out_len.data();
    g_captured.clear();
    if (deflate_stride_for_level(level) == 2) MZ_LAUNCH((deflate_chunks_kernel<2, false>), dim3(nchunks), dim3(DF_THREADS), DF_SMEM_BYTES, 0, P);
    else if (!deflate_lazy_for_level(level)) MZ_LAUNCH((deflate_chunks_kernel<1, false>), dim3(nchunks), dim3(DF_THREADS), DF_SMEM_BYTES, 0, P);
    else if (!deflate_hist_for_level(level)) MZ_LAUNCH((deflate_chunks_kernel<1, true>), dim3(nchunks), dim3(DF_THREADS), DF_SMEM_BYTES, 0, P);
    else MZ_LAUNCH((deflate_chunks_kernel<1, true, true>), dim3(nchunks), dim3(DF_THREADS), DFH_SMEM_BYTES, 0, P);
    const uint32_t n = (uint32_t)(g_captured.size() / DFC_HIST_WORDS);
    memcpy(out, g_captured.data(), (size_t)(n < cap ? n : cap) * DFC_HIST_WORDS * 4);
    return n;
}

/* Both builders on n histograms; DFC_OUT_WORDS words per histogram into out_old and out_new. */
void emu_df_codes_pair(const uint32_t *hists, const uint32_t *posfin, uint32_t n, uint32_t *out_old, uint32_t *out_new) {
    MZ_LAUNCH(df_codes_pair_kernel<true>, dim3(1), dim3(DF_BB_THREADS), 0, 0, hists, posfin, n, out_old);
    MZ_LAUNCH(df_codes_pair_kernel<false>, dim3(1), dim3(DF_BB_THREADS), 0, 0, hists, posfin, n, out_new);
}
}
