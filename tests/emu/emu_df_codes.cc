/* emu_df_codes.cc -- the code-builder equivalence harness on the CPU emulator (TEST INFRASTRUCTURE ONLY): captures the per-unit
 * histograms the deflate kernel hands its code builder, and runs today's and the frozen v3.4 builder on given histograms
 * (df_codes_pair.cuh). Built together with cuda_emu.cc by tests/test_emu_df_codes_equiv.py; never part of the product library. */
#define MZ_EMU 1
#include <stdint.h>
#include <vector>

static std::vector<uint32_t> g_captured; /* DFC_HIST_WORDS words per histogram */
static std::vector<uint32_t> g_tags;     /* per histogram: chunk << 8 | unit */
static void df_capture(const uint32_t *ll, const uint32_t *lit2, const uint32_t *d) {
    g_captured.insert(g_captured.end(), ll, ll + 288);
    g_captured.insert(g_captured.end(), d, d + 32);
    g_captured.insert(g_captured.end(), lit2, lit2 + 256);
}
#define MZ_DF_CODES_HOOK(ll, lit2, d) df_capture(ll, lit2, d)
#define MZ_DF_UNIT_HOOK(chunk, unit) g_tags.push_back((chunk) << 8 | (unit))

#include "../../minizip-ng_b200/csrc/deflate_kernel.cuh"
#include "df_codes_pair.cuh"

using namespace mzc;

extern "C" {

uint32_t emu_df_hist_words(void) { return DFC_HIST_WORDS; }
uint32_t emu_df_out_words(void) { return DFC_OUT_WORDS; }

/* Deflate the n chunks in[offs[i], offs[i] + lens[i]) with flags[i] (DF_FLAG_*) at `level`, as mz_cuda_deflate_chunks does with
 * explicit chunks, and return how many histograms the code builder was given; up to `cap` of them are copied to out
 * (DFC_HIST_WORDS words each) and their tags (chunk << 8 | unit) to tags (may be NULL). Stored or not, every unit of a level
 * above 0 hands its histogram to the builder. */
uint32_t emu_df_capture_chunks(const uint8_t *in, uint64_t len, const uint64_t *offs, const uint32_t *lens, const uint8_t *flags, uint32_t n,
                               int level, uint32_t *out, uint32_t *tags, uint32_t cap) {
    const uint64_t stride = deflate_slot_bound(DF_CHUNK_MAX);
    std::vector<uint8_t> slots((size_t)(stride * n + 64));
    std::vector<uint8_t> inbuf((size_t)len + 64);
    uint8_t *ia = (uint8_t *)(((uintptr_t)inbuf.data() + 15) & ~(uintptr_t)15);
    memcpy(ia, in, (size_t)len);
    std::vector<uint32_t> out_len(n);
    DeflateParams P;
    memset(&P, 0, sizeof(P));
    P.in = ia;
    P.in_off = offs;
    P.in_len = lens;
    P.flags = flags;
    P.nchunks = n;
    P.level = level;
    P.out = (uint8_t *)(((uintptr_t)slots.data() + 15) & ~(uintptr_t)15);
    P.slot_stride = stride;
    P.out_len = out_len.data();
    g_captured.clear();
    g_tags.clear();
    if (deflate_stride_for_level(level) == 2) MZ_LAUNCH((deflate_chunks_kernel<2, false>), dim3(n), dim3(DF_THREADS), DF_SMEM_BYTES, 0, P);
    else if (!deflate_lazy_for_level(level)) MZ_LAUNCH((deflate_chunks_kernel<1, false>), dim3(n), dim3(DF_THREADS), DF_SMEM_BYTES, 0, P);
    else if (!deflate_hist_for_level(level)) MZ_LAUNCH((deflate_chunks_kernel<1, true>), dim3(n), dim3(DF_THREADS), DF_SMEM_BYTES, 0, P);
    else MZ_LAUNCH((deflate_chunks_kernel<1, true, true>), dim3(n), dim3(DF_THREADS), DFH_SMEM_BYTES, 0, P);
    const uint32_t k = (uint32_t)(g_captured.size() / DFC_HIST_WORDS), m = k < cap ? k : cap;
    memcpy(out, g_captured.data(), (size_t)m * DFC_HIST_WORDS * 4);
    if (tags) memcpy(tags, g_tags.data(), (size_t)m * 4);
    return k;
}

/* Deflate `in` as one buffer of 64 KiB chunks (the last one FINAL) at `level` and return how many histograms the code builder
 * was given; up to `cap` of them are copied to out (DFC_HIST_WORDS words each). */
uint32_t emu_df_capture(const uint8_t *in, uint64_t len, int level, uint32_t *out, uint32_t cap) {
    const uint32_t chunk = DF_CHUNK_MAX, nchunks = (uint32_t)((len + chunk - 1) / chunk);
    std::vector<uint64_t> offs(nchunks);
    std::vector<uint32_t> lens(nchunks);
    std::vector<uint8_t> flags(nchunks);
    for (uint32_t i = 0; i < nchunks; i++) {
        offs[i] = (uint64_t)i * chunk;
        lens[i] = (uint32_t)(len - offs[i] < chunk ? len - offs[i] : chunk);
        flags[i] = i == nchunks - 1 ? DF_FLAG_FINAL : 0;
    }
    return emu_df_capture_chunks(in, len, offs.data(), lens.data(), flags.data(), nchunks, level, out, nullptr, cap);
}

/* Both builders on n histograms; DFC_OUT_WORDS words per histogram into out_old and out_new. */
void emu_df_codes_pair(const uint32_t *hists, const uint32_t *posfin, uint32_t n, uint32_t *out_old, uint32_t *out_new) {
    MZ_LAUNCH(df_codes_pair_kernel<true>, dim3(1), dim3(DF_BB_THREADS), 0, 0, hists, posfin, n, out_old);
    MZ_LAUNCH(df_codes_pair_kernel<false>, dim3(1), dim3(DF_BB_THREADS), 0, 0, hists, posfin, n, out_new);
}
}
