// Standalone check of k_panmix_tc (csrc/panmix_tc.cuh) against a double-precision CPU sum.
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++20 -o panmix_tc_test panmix_tc_test.cu
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "../../openal-soft_b200/csrc/panmix_tc.cuh"

using namespace b200mix;

#define CK(x) do { cudaError_t e = (x); if(e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); return 1; } } while(0)

int main(int argc, char **argv)
{
    const uint32_t V = argc > 1 ? atoi(argv[1]) : 1000, cw = argc > 2 ? atoi(argv[2]) : 16;
    const uint32_t chunks = std::max(1u, std::min(128u, (V + 63u)/64u));
    std::mt19937 rng(5);
    std::uniform_real_distribution<float> U(-1.f, 1.f);
    std::vector<float> lines(size_t(V)*kLine), geff(size_t(V)*cw);
    for(auto &x : lines) x = U(rng)*0.25f;
    for(auto &x : geff) x = U(rng)*0.05f;
    std::vector<SendEntry> entries(V);
    for(uint32_t i = 0;i < V;++i) entries[i] = SendEntry{(i*7919u) % V, 0u};     // a permutation-ish gather
    std::vector<uint32_t> ss = {0u, V}, info(V, 0u);
    float *d_lines, *d_geff, *d_partial; SendEntry *d_entries; uint32_t *d_ss, *d_info;
    CK(cudaMalloc(&d_lines, lines.size()*4)); CK(cudaMalloc(&d_geff, geff.size()*4));
    CK(cudaMalloc(&d_partial, size_t(chunks)*cw*kLine*4)); CK(cudaMalloc(&d_entries, V*sizeof(SendEntry)));
    CK(cudaMalloc(&d_ss, 8)); CK(cudaMalloc(&d_info, V*4));
    CK(cudaMemcpy(d_lines, lines.data(), lines.size()*4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_geff, geff.data(), geff.size()*4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_entries, entries.data(), V*sizeof(SendEntry), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_ss, ss.data(), 8, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_info, info.data(), V*4, cudaMemcpyHostToDevice));
    CK(cudaMemset(d_partial, 0, size_t(chunks)*cw*kLine*4));
    PanMixTcParams Q{d_ss, d_entries, d_info, d_lines, nullptr, d_geff, cw, chunks, d_partial};
    const int smem = kPmStages*kPmStageBytes + 1024;
    CK(cudaFuncSetAttribute(k_panmix_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    k_panmix_tc<<<chunks, 128, smem>>>(Q);
    CK(cudaGetLastError()); CK(cudaDeviceSynchronize());
    cudaEventRecord(e0);
    for(int r = 0;r < 20;++r) k_panmix_tc<<<chunks, 128, smem>>>(Q);
    cudaEventRecord(e1); CK(cudaDeviceSynchronize());
    float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
    std::vector<float> part(size_t(chunks)*cw*kLine);
    CK(cudaMemcpy(part.data(), d_partial, part.size()*4, cudaMemcpyDeviceToHost));
    double maxerr = 0, maxref = 0, sq = 0; size_t cnt = 0;
    for(uint32_t c = 0;c < cw;++c)
        for(uint32_t i = 128;i < 1024;++i)
        {
            double ref = 0, got = 0;
            for(uint32_t e = 0;e < V;++e) ref += double(lines[size_t(entries[e].voice)*kLine + i])*double(geff[size_t(e)*cw + c]);
            for(uint32_t z = 0;z < chunks;++z) got += part[(size_t(z)*cw + c)*kLine + i];
            maxerr = std::max(maxerr, std::fabs(got - ref)); maxref = std::max(maxref, std::fabs(ref));
            sq += (got - ref)*(got - ref); ++cnt;
        }
    printf("V=%u cw=%u chunks=%u  max|ref|=%.4f  max err=%.3e  rms err=%.3e  %.2f us/launch\n", V, cw, chunks,
        maxref, maxerr, std::sqrt(sq/cnt), ms*1000.0/20);
    const bool ok = maxerr < 2e-6*std::max(1.0, maxref);
    printf(ok ? "PANMIX_TC_OK\n" : "PANMIX_TC_FAIL\n");
    return ok ? 0 : 2;
}
