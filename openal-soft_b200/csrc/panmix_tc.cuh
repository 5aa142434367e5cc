// panmix_tc.cuh — the dense ambisonic pan-mix on Hopper's warpgroup tensor cores (wgmma).
//
// A device that mixes above first order (config 4a: third-order B-Format output, 16 dry
// channels) sums every voice into every channel: Dry[c][i] += line_v[i] * gain_v,c — the
// reference's MixSamples 1->many (core/mixer/mixer_c.cpp:150-186) over all voices is the
// contraction  Dry[16 x 1024] = G[16 x V] . S[V x 1024], a true dense GEMM with K = voices.
// Past the gain fade (Counter <= 64 samples, core/voice.cpp:1093) the gains are constants, so
// samples 128..1023 of every line go through wgmma.mma_async, one warpgroup per CTA:
//
//   D[M = 64 samples][N = 16 channels] += A[M x K = 8 voices] . B[K x N]      (tf32, 14 M tiles)
//
//   A = the parked lines.  They lie with the samples (M) contiguous, but wgmma takes tf32
//       shared-memory operands K-major only, so the lines are transposed on their way into
//       shared memory: 8-row x 16-byte core matrices, (m%8)*16 + (m/8)*SBO + (k/4)*LBO + (k%4)*4,
//       with LBO = 144 and SBO = 288 bytes so that the transposing scalar stores are conflict-free.
//   B = geff[entry][channel] (k_send_gains_prepare), K-major
//   D = fp32 accumulators in registers (14 tiles x 8 per thread), accumulated over ALL the
//       voices a CTA owns, transposed through shared memory into the CTA's partial row.
//
// fp32 parity from tf32 tensor cores: both operands are split  x = hi + lo  with hi = x rounded
// to tf32 and lo = x - hi (exact), and three MMAs accumulate hi.hi + lo.hi + hi.lo; the dropped
// lo.lo term and lo's own truncation are ~2^-22 relative per product, an order below the parity
// budget (tests/test_gpu_panmix.py: this kernel alone against a float64 sum, and the mixer's
// dry bus against the oracle on the tensor cores and on the SIMT path).
// Samples 0..127 (the fades) stay with k_send_mix<16>'s first tile; both kernels write disjoint
// columns of the same per-chunk partial rows, k_reduce_rows sums the chunks in fixed order.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "async_ptx.cuh"
#include "effect_kernels.cuh"

namespace b200mix {

constexpr int kPmTiles = 7;                         // staged sample tiles 1..7 of 128 (896 samples)
constexpr int kPmMmaTiles = 2*kPmTiles;             // wgmma M tiles of 64 samples
constexpr int kPmK = 8;                             // voices per MMA (tf32: 32 bytes of K)
constexpr int kPmN = 16;                            // channels (padded)
constexpr int kPmLboA = 144, kPmSboA = 288;         // A core-matrix strides (padded: conflict-free stores)
constexpr int kPmTileBytes = 16*kPmSboA;            // one A tile: 16 groups of 8 samples x 2 K halves
constexpr int kPmStageBytes = 2*kPmTiles*kPmTileBytes + 2*kPmN*kPmK*4;     // A hi, A lo, B hi, B lo
constexpr int kPmStages = 2;
constexpr int kPmOutStride = 7*128 + 4;             // epilogue rows in shared memory (conflict-free stores)
static_assert(kPmN*kPmOutStride*4 <= kPmStages*kPmStageBytes, "epilogue staging fits the stages");

struct PanMixTcParams {
    const uint32_t *slot_start;     // [2] entry range of the dry bus
    const SendEntry *entries;
    const uint32_t *sendinfo;
    const float *xscratch;          // [max_voices][1024]
    const float *dline;             // [max_voices][1024] lines of deferred (direct-filtered) voices
    const float *geff;              // [entries][cw] constant gain of every entry-channel
    uint32_t cw, chunks;
    float *partial;                 // [chunks][cw][1024]
};

// tf32 split of an fp32 value: hi = round-to-nearest at 10 mantissa bits, lo = x - hi truncated
__device__ __forceinline__ void tf32_split(float x, float &hi, float &lo)
{
    const uint32_t b = __float_as_uint(x);
    hi = __uint_as_float((b + 0x1000u) & 0xffffe000u);
    lo = __uint_as_float(__float_as_uint(x - hi) & 0xffffe000u);
}

// grid = chunks (the entry ranges k_send_mix uses), 128 threads (one warpgroup),
// kPmStages*kPmStageBytes dynamic smem
__global__ void __launch_bounds__(128, 1) k_panmix_tc(const PanMixTcParams Q)
{
    extern __shared__ __align__(1024) unsigned char pm_smem[];
    const uint32_t t = threadIdx.x, warp = t >> 5, lane = t & 31u;

    uint32_t e0 = Q.slot_start[0], e1 = Q.slot_start[1];
    {
        const uint32_t per = (e1 - e0 + Q.chunks - 1u)/Q.chunks;
        e0 = min(e0 + blockIdx.x*per, e1);
        e1 = min(e0 + per, e1);
    }
    const uint32_t nkb = (e1 - e0 + uint32_t(kPmK) - 1u)/uint32_t(kPmK);
    float *out = Q.partial + size_t(blockIdx.x)*Q.cw*kLine;

    float acc[kPmMmaTiles][8];                           // defined by the first K block's MMAs

    // this thread's voice of a K block and its sample groups (4 consecutive samples each)
    const uint32_t kk = t & 7u, gl = t >> 3;             // gl in [0,16)
    for(uint32_t kb = 0;kb < nkb;++kb)
    {
        const uint32_t st = kb % uint32_t(kPmStages);
        unsigned char *stage = pm_smem + size_t(st)*kPmStageBytes;
        // (the MMAs that read this stage, K block kb - kPmStages, were waited for by every warp below)
        // ---- A: 8 lines x 896 samples, split, transposed into K-major core matrices
        const uint32_t e = e0 + kb*uint32_t(kPmK) + kk;
        const bool live = e < e1;
        const SendEntry en = Q.entries[live ? e : e0];
        const float *line = ((Q.dline && (Q.sendinfo[en.voice] & kSiDeferred)) ? Q.dline : Q.xscratch)
            + size_t(en.voice)*kLine + 128;
        float4 v[14];
        #pragma unroll
        for(int i = 0;i < 14;++i)
            v[i] = live ? __ldg(reinterpret_cast<const float4*>(line) + gl + 16u*uint32_t(i))
                        : make_float4(0.f, 0.f, 0.f, 0.f);
        #pragma unroll
        for(int i = 0;i < 14;++i)
        {
            const uint32_t g = gl + 16u*uint32_t(i);     // [0, 224)
            float4 hi, lo;
            tf32_split(v[i].x, hi.x, lo.x); tf32_split(v[i].y, hi.y, lo.y);
            tf32_split(v[i].z, hi.z, lo.z); tf32_split(v[i].w, hi.w, lo.w);
            // samples m = 4*(g % 32) + j of tile g / 32, voice kk
            const uint32_t mg = (g & 31u) >> 1;          // group of 8 rows
            const uint32_t off = (g >> 5)*uint32_t(kPmTileBytes) + mg*uint32_t(kPmSboA)
                + ((g & 1u)*4u)*16u + (kk >> 2)*uint32_t(kPmLboA) + (kk & 3u)*4u;
            float *ph = reinterpret_cast<float*>(stage + off);
            float *pl = reinterpret_cast<float*>(stage + kPmTiles*kPmTileBytes + off);
            ph[0] = hi.x; ph[4] = hi.y; ph[8] = hi.z; ph[12] = hi.w;       // rows are 16 bytes apart
            pl[0] = lo.x; pl[4] = lo.y; pl[8] = lo.z; pl[12] = lo.w;
        }
        // ---- B: gains [n = channel][k = voice], K-major core matrices:
        //      (n % 8)*16 + (n / 8)*256 + (k / 4)*128 + (k % 4)*4
        {
            const uint32_t n = t & 15u, k = t >> 4;      // 16 x 8
            const uint32_t eb = e0 + kb*uint32_t(kPmK) + k;
            float g = 0.0f;
            if(eb < e1 && n < Q.cw) g = Q.geff[size_t(eb)*Q.cw + n];
            float hi, lo;
            tf32_split(g, hi, lo);
            const uint32_t off = (n & 7u)*16u + (n >> 3)*256u + (k >> 2)*128u + (k & 3u)*4u;
            unsigned char *bs = stage + 2*kPmTiles*kPmTileBytes;
            *reinterpret_cast<float*>(bs + off) = hi;
            *reinterpret_cast<float*>(bs + kPmN*kPmK*4 + off) = lo;
        }
        fence_proxy_async_smem();                        // generic-proxy stores -> tensor core reads
        __syncthreads();
        {
            const uint32_t sa = smem_u32(stage);
            const uint32_t sb = sa + 2u*kPmTiles*kPmTileBytes;
            const uint64_t bhi = wgmma_smem_desc(sb, 128u, 256u), blo = wgmma_smem_desc(sb + kPmN*kPmK*4, 128u, 256u);
            wgmma_fence();
            #pragma unroll
            for(int q = 0;q < kPmMmaTiles;++q)
            {
                // M tile q = samples 64q..64q+63: the 8-row groups 8(q%2).. of staged tile q/2
                const uint32_t a = sa + uint32_t(q >> 1)*kPmTileBytes + uint32_t(q & 1)*8u*kPmSboA;
                const uint64_t ahi = wgmma_smem_desc(a, kPmLboA, kPmSboA);
                const uint64_t alo = wgmma_smem_desc(a + uint32_t(kPmTiles*kPmTileBytes), kPmLboA, kPmSboA);
                wgmma_m64n16k8_tf32(acc[q], ahi, bhi, kb != 0u);
                wgmma_m64n16k8_tf32(acc[q], alo, bhi, true);
                wgmma_m64n16k8_tf32(acc[q], ahi, blo, true);
            }
            wgmma_commit();
        }
        wgmma_wait<kPmStages - 1>();                     // this warp's share of group kb - 1 is done
        __syncthreads();    // wait_group covers only this warp's MMAs: all 4 must wait before the stage is rewritten
    }
    wgmma_wait<0>();
    __syncthreads();
    // ---- epilogue: registers -> shared [channel][sample] -> the CTA's partial row (samples 128..1023)
    float *so = reinterpret_cast<float*>(pm_smem);
    #pragma unroll
    for(int q = 0;q < kPmMmaTiles;++q)
        #pragma unroll
        for(int i = 0;i < 8;++i)
        {
            const uint32_t m = uint32_t(q)*64u + warp*16u + (lane >> 2) + 8u*((uint32_t(i) >> 1) & 1u);
            const uint32_t n = uint32_t(i >> 2)*8u + (lane & 3u)*2u + (uint32_t(i) & 1u);
            so[n*uint32_t(kPmOutStride) + m] = nkb ? acc[q][i] : 0.0f;
        }
    __syncthreads();
    for(uint32_t c = 0;c < Q.cw;++c)
        for(uint32_t i = t;i < uint32_t(kPmTiles*128/4);i += 128u)
            reinterpret_cast<float4*>(out + size_t(c)*kLine + 128)[i]
                = reinterpret_cast<const float4*>(so + c*uint32_t(kPmOutStride))[i];
}

} // namespace b200mix
