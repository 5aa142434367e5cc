// Microbenchmark: do SHFL.IDX and LDS share one per-SM bandwidth, or do they add?
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o shfl_lds shfl_lds.cu
#include <cstdio>
#include <cuda_runtime.h>

template<int MODE>   // 0: LDS only, 1: SHFL only, 2: LDS + SHFL interleaved, 3: FFMA2 only, 4: LDS + FFMA2
__global__ void __launch_bounds__(128) k(float *out, int iters, const int *idx)
{
    __shared__ float sm[4096];
    for(int i = threadIdx.x;i < 4096;i += blockDim.x) sm[i] = float(i);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    int a = (threadIdx.x*33) & 4095;
    const int src = idx[lane];
    float acc0 = 0.f, acc1 = 0.f, v0 = float(lane), v1 = float(lane+1);
    float2 f0 = make_float2(1.f, 2.f), f1 = make_float2(0.5f, 0.25f), f2 = make_float2(0.f, 0.f), f3 = f2;
    for(int it = 0;it < iters;++it)
    {
        #pragma unroll
        for(int u = 0;u < 16;++u)
        {
            if(MODE == 0 || MODE == 2 || MODE == 4)
            { acc0 += sm[(a + u*37) & 4095]; }
            if(MODE == 1 || MODE == 2)
            { acc1 += __shfl_sync(0xffffffffu, v0, (src + u) & 31); v0 += 1.0f; }
            if(MODE == 3 || MODE == 4)
            { f2 = __ffma2_rn(f0, f1, f2); f3 = __ffma2_rn(f1, f0, f3); }
        }
        a = (a + 17) & 4095;
    }
    out[blockIdx.x*blockDim.x + threadIdx.x] = acc0 + acc1 + v1 + f2.x + f2.y + f3.x + f3.y;
}

template<int MODE> float run(float *out, const int *idx, int iters)
{
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    k<MODE><<<132*4, 128>>>(out, 10, idx);
    cudaEventRecord(e0);
    k<MODE><<<132*4, 128>>>(out, iters, idx);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1); return ms;
}

int main()
{
    float *out; int *idx; cudaMalloc(&out, 132*4*128*4); cudaMalloc(&idx, 128);
    int h[32]; for(int i = 0;i < 32;++i) h[i] = (i*7 + 3) & 31;
    cudaMemcpy(idx, h, 128, cudaMemcpyHostToDevice);
    const int iters = 20000;
    const double ops = double(iters)*16*16;   // warp-instrs per SM of each kind (16 warps/SM)
    float t0 = run<0>(out, idx, iters), t1 = run<1>(out, idx, iters), t2 = run<2>(out, idx, iters);
    float t3 = run<3>(out, idx, iters), t4 = run<4>(out, idx, iters);
    int clk = 0; cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
    printf("clock %d kHz\n", clk);
    printf("LDS only      %.3f ms  -> %.2f clk per warp-LDS per SM\n", t0, t0*1e-3*clk*1e3/ops);
    printf("SHFL only     %.3f ms  -> %.2f clk per warp-SHFL per SM\n", t1, t1*1e-3*clk*1e3/ops);
    printf("LDS+SHFL      %.3f ms  (sum %.3f, max %.3f)\n", t2, t0+t1, t0 > t1 ? t0 : t1);
    printf("FFMA2 x2 only %.3f ms  -> %.2f clk per warp-FFMA2 per SM\n", t3, t3*1e-3*clk*1e3/(2*ops));
    printf("LDS+FFMA2x2   %.3f ms\n", t4);
    return 0;
}
