// async_ptx.cuh — thin wrappers over the sm_90a asynchronous-copy and tensor-core PTX the
// kernels use: mbarrier, the bulk ("1-D TMA") global->shared copy cp.async.bulk (SASS: UBLKCP),
// the warpgroup MMA wgmma.mma_async (SASS: HGMMA).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace b200mix {

__device__ __forceinline__ uint32_t smem_u32(const void *p)
{ return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// ---- mbarrier ---------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{ asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory"); }
// makes the initialised barriers visible to the async proxy (TMA / tensor core arrivals)
__device__ __forceinline__ void mbar_fence_init()
{ asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{ asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{ asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                 "selp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0u;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{ while(!mbar_try_wait(bar, parity)) { } }

// ---- bulk copy global -> shared (1-D TMA): 16-byte aligned, size a multiple of 16 ----------
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        :: "r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// generic-proxy writes to shared memory -> visible to the async proxy (tensor core operand reads)
__device__ __forceinline__ void fence_proxy_async_smem()
{ asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- programmatic dependent launch --------------------------------------------------------
// Blocks until every grid this one depends on has completed and its memory is visible; returns
// at once when the grid was launched without the programmatic-serialization attribute.
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// Lets the next grid on the stream (launched with the attribute) be scheduled once every CTA of
// this grid has executed it or exited.  It counts per CTA: the first thread of a CTA to run it
// marks the whole CTA, later executions in that CTA are no-ops.
__device__ __forceinline__ void griddep_launch_dependents()
{ asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---- wgmma: Hopper's warpgroup MMA (4 warps issue together, accumulators in registers) ----
// Shared-memory matrix descriptor (cute::GmmaDescriptor), no swizzle ("interleave"):
// start address, leading / stride byte offsets (all >> 4), layout type 0.
__device__ __forceinline__ uint64_t wgmma_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes)
{
    return uint64_t((saddr >> 4) & 0x3fffu) | (uint64_t((lbo_bytes >> 4) & 0x3fffu) << 16)
        | (uint64_t((sbo_bytes >> 4) & 0x3fffu) << 32);
}
// orders this thread's register and shared-memory accesses before the wgmma that follow
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// waits until at most N committed wgmma groups of this thread are still in flight
template<int N> __device__ __forceinline__ void wgmma_wait()
{ asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }
// D[64 x 16] (+)= A[smem, 64 x 8] * B[smem, 8 x 16], kind tf32, both operands K-major, fp32 accumulate.
// Thread (warp w, lane l) holds d[i] = D[16w + l/4 + 8*((i/2)%2)][8*(i/4) + 2*(l%4) + i%2].
__device__ __forceinline__ void wgmma_m64n16k8_tf32(float (&d)[8], uint64_t adesc, uint64_t bdesc, bool accumulate)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
                 "{%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(adesc), "l"(bdesc), "r"(uint32_t(accumulate)) : "memory");
}

} // namespace b200mix
