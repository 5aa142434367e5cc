// panmix_probe.cu — k_panmix_tc (openal-soft_b200/csrc/panmix_tc.cuh) on caller-supplied device
// buffers, for tests/test_gpu_panmix.py.  Built by openal-soft_b200/Makefile with the library's own
// NVFLAGS (-ftz=true etc.), so the kernel is the same code the mixer launches.
#include <cstdint>
#include <cuda_runtime.h>

#include "../../openal-soft_b200/csrc/panmix_tc.cuh"

using namespace b200mix;

extern "C" {

// Launches k_panmix_tc<<<chunks, 128>>> on the legacy default stream with the mixer's dynamic
// shared-memory size and waits for it.  Pointers are device pointers laid out as in
// PanMixTcParams; dline may be null.  Returns the cudaError_t of the launch / synchronisation.
__attribute__((visibility("default")))
int panmix_probe_run(const uint32_t *slot_start, const SendEntry *entries, const uint32_t *sendinfo,
    const float *xscratch, const float *dline, const float *geff, uint32_t cw, uint32_t chunks,
    float *partial)
{
    if(cw == 0u || cw > uint32_t(kPmN) || chunks == 0u) return int(cudaErrorInvalidValue);
    const int smem = kPmStages*kPmStageBytes + 1024;
    cudaError_t rc = cudaFuncSetAttribute(k_panmix_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if(rc != cudaSuccess) return int(rc);
    const PanMixTcParams Q{slot_start, entries, sendinfo, xscratch, dline, geff, cw, chunks, partial};
    k_panmix_tc<<<chunks, 128, smem, 0>>>(Q);
    rc = cudaGetLastError();
    if(rc != cudaSuccess) return int(rc);
    return int(cudaDeviceSynchronize());
}

} // extern "C"
