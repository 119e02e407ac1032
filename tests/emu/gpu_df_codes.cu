/* gpu_df_codes.cu -- the code-builder equivalence harness on the GPU (TEST INFRASTRUCTURE ONLY): today's and the frozen v3.4
 * builder (df_codes_pair.cuh) on the same histograms, compiled for sm_90a by tests/test_gpu_df_codes_equiv.py. The GPU is where
 * __log2f is the hardware's approximate log2, so this is the run that would see a float path that differs from the emulator's. */
#include <cuda_runtime.h>

#include "df_codes_pair.cuh"

using namespace mzc;

extern "C" {

uint32_t gpu_df_out_words(void) { return DFC_OUT_WORDS; }

/* returns 0, or the CUDA error code */
int gpu_df_codes_pair(const uint32_t *hists, const uint32_t *posfin, uint32_t n, uint32_t *out_old, uint32_t *out_new) {
    uint32_t *d_h = nullptr, *d_p = nullptr, *d_o = nullptr, *d_n = nullptr;
    const size_t hb = (size_t)n * DFC_HIST_WORDS * 4, ob = (size_t)n * DFC_OUT_WORDS * 4;
    cudaError_t e = cudaMalloc(&d_h, hb);
    if (!e) e = cudaMalloc(&d_p, (size_t)n * 4);
    if (!e) e = cudaMalloc(&d_o, ob);
    if (!e) e = cudaMalloc(&d_n, ob);
    if (!e) e = cudaMemcpy(d_h, hists, hb, cudaMemcpyHostToDevice);
    if (!e) e = cudaMemcpy(d_p, posfin, (size_t)n * 4, cudaMemcpyHostToDevice);
    if (!e) {
        const uint32_t grid = n < 1056u ? (n ? n : 1u) : 1056u;
        df_codes_pair_kernel<true><<<grid, DF_BB_THREADS>>>(d_h, d_p, n, d_o);
        df_codes_pair_kernel<false><<<grid, DF_BB_THREADS>>>(d_h, d_p, n, d_n);
        e = cudaGetLastError();
    }
    if (!e) e = cudaDeviceSynchronize();
    if (!e) e = cudaMemcpy(out_old, d_o, ob, cudaMemcpyDeviceToHost);
    if (!e) e = cudaMemcpy(out_new, d_n, ob, cudaMemcpyDeviceToHost);
    cudaFree(d_h);
    cudaFree(d_p);
    cudaFree(d_o);
    cudaFree(d_n);
    return (int)e;
}
}
