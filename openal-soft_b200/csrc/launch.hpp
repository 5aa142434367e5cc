// launch.hpp — the host library's kernel launch with programmatic dependent launch.
#pragma once
#include <cstddef>
#include <cstdint>

#include <cuda_runtime.h>

namespace b200mix {

// Launches fn on `stream` and counts it in `launches`.  `programmatic`: the kernel directly follows
// the one it depends on, and may be scheduled once every CTA of that one has executed
// griddepcontrol.launch_dependents; it must run griddepcontrol.wait before it reads anything
// that kernel writes.
template<typename... Args>
cudaError_t launch_ex(cudaStream_t stream, uint64_t &launches, bool programmatic, void (*fn)(Args...),
    dim3 grid, dim3 block, size_t smem, Args... args)
{
    cudaLaunchAttribute attr{};
    attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr.val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cfg.attrs = programmatic ? &attr : nullptr; cfg.numAttrs = programmatic ? 1u : 0u;
    ++launches;
    return cudaLaunchKernelEx(&cfg, fn, args...);
}

} // namespace b200mix
