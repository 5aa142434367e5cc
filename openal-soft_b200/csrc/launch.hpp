// launch.hpp — the host library's kernel launch with programmatic dependent launch, and how its
// calls report an error.
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>

#include <cuda_runtime.h>

#include "../../include/b200mix.h"

namespace b200mix {

// Every host call returns a B200MIX_* code and, when it fails, sets the device's error string `err`:
// refuse() when the call's checks reject it, fail() (or CUDA_TRY) when a CUDA call fails.
inline int refuse(std::string &err, const std::string &why) { err = why; return B200MIX_ERR_INVALID; }
inline int fail(std::string &err, const char *what, cudaError_t e) { err = std::string(what) + ": " + cudaGetErrorString(e); return B200MIX_ERR_CUDA; }
#define CUDA_TRY(err, expr) do { const cudaError_t e_ = (expr); if(e_ != cudaSuccess) return ::b200mix::fail(err, #expr, e_); } while(0)

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
