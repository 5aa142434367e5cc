// effect_kernels.cuh — aux-send wet mix and the convolution effect slot on sm_90a.
//
//  k_send_mix        MixSamples of every (voice, send) into the slot wet buffers
//                    (core/voice.cpp:967-980), slot-major and in a fixed order (no atomics)
//  k_conv_input      ConvolutionState::process, input side (alc/effects/convolution.cpp:
//                    636-667): FIFO bookkeeping, 256-point FFTs of the completed 128-sample
//                    blocks into the spectrum ring, and the 128-tap time-domain head (apply_fir)
//  k_conv_mac        sum_s X[(cur+s) mod S] * H[s] for ALL blocks completed in this update in
//                    ONE pass over the filter spectra (the reference re-reads them per block)
//  k_conv_output     inverse FFTs + overlap-add (convolution.cpp:699-706)
//  k_slot_output_mix the slots' output lines -> Dry with MixSamples(Counter = samplesToDo)
//
// The FFT is an in-shared-memory radix-2 complex FFT of 256 points (cuFFT-free); only the
// RESULT has to match the reference's pffft path, the spectrum layout is our own:
// packed [re0, nyquist, re1, im1, ... re127, im127].
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "mixer_kernels.cuh"
#include "async_ptx.cuh"

namespace b200mix {

constexpr int kConvBlock = 128;     // ConvolveUpdateSamples
constexpr int kConvFft = 256;       // ConvolveUpdateSize
constexpr int kConvMaxBlocks = 9;   // blocks that can complete in one 1024-frame update
constexpr int kConvMaxChunks = 48;  // segment-range chunks of k_conv_mac (gridDim.z), partials in yspec

// ---- send mix --------------------------------------------------------------------------
struct SendMixParams {
    const uint32_t *slot_start;     // [slots+1] CSR over entries
    const SendEntry *entries;
    const uint32_t *sendinfo;       // per voice: kSi* bits, bits 8.. fade counter
    const float *xscratch;          // [max_voices][1024] resampled lines of voices with sends
    float *send_cur; const float *send_tgt;   // [max_voices][num_sends][cw]
    float *wet;                     // [slots][cw][1024]
    uint32_t frames, cw, num_sends;
    FilterRec *filt; uint32_t filt_paths;   // send filters (null: none ever set)
    const float *fscratch;          // [entries][1024] filtered lines of entries with an active filter
    // The same kernel sums the DRY bus of parked non-HRTF voices: one pseudo slot whose
    // entries are (voice, 0), gains dry_cur/dry_tgt, valid bit kSiDry, filtered line dline[v].
    uint32_t valid_bit;             // kSiSend or kSiDry
    const float *dline;             // dry bus only: [max_voices][1024] (deferred voices), else null
    uint32_t chunks;                // gridDim.z: entry ranges summed by separate CTAs
    float *partial;                 // [chunks][slots][cw][1024] when chunks > 1 (then k_reduce_rows)
    float *geff;                    // [entries][cw] gain of every entry-channel once its fade is over
                                    // (k_send_gains_prepare), 0 for entries not mixed this update
    float4 *gramp;                  // [entries][cw] {a, b, flat, L}: gain(i) = i < L ? a + b*i : flat
};

// ---- direct and send filters ------------------------------------------------------------
// DoFilters -> BiquadInterpFilter::dualProcess (core/voice.cpp:255-268,
// core/filters/biquad.cpp:254-343).  The two cascaded transposed-direct-form-II biquads are a
// serial recurrence per line, and with the EFX shelves (poles close to z = 1) its fp32
// rounding noise is amplified ~1000x: any re-association (scan, FMA contraction) moves the
// result by 1e-5 relative.  So the recurrence is evaluated exactly as the reference does —
// one thread per line, same operation order, explicit round-to-nearest mul/add/sub so the
// compiler cannot contract to FMA — and the parallelism comes from the lines: a warp takes
// 32 (voice, path) items, stages 32x32-sample tiles through shared memory (coalesced
// loads/stores, conflict-free column walks) and prefetches the next tile into registers.
// Items: [0, num_direct) = voices of `direct_order` (parked line xscratch[v] -> dline[v]),
//        [num_direct, num_direct + num_entries) = send entries (xscratch[v] -> fscratch[e]).
struct FilterRunParams {
    FilterRec *filt; uint32_t filt_paths;
    const uint32_t *sendinfo;
    const uint32_t *direct_order; uint32_t num_direct;
    const SendEntry *entries; uint32_t num_entries;
    const float *xscratch; float *dline; float *fscratch;
    uint32_t frames;
};

struct BiquadCoefs { float b0, b1, b2, a1, a2; };

__global__ void __launch_bounds__(32) k_filters(const FilterRunParams Q)
{
    __shared__ float tile[32][33];
    __shared__ const float *inp[32];
    __shared__ float *outp[32];
    const uint32_t lane = threadIdx.x;
    const uint32_t item = blockIdx.x*32u + lane;
    const uint32_t n = Q.frames;

    FilterRec *fr = nullptr;
    const float *in = nullptr; float *out = nullptr;
    if(item < Q.num_direct)
    {
        const uint32_t v = Q.direct_order[item];
        if(Q.sendinfo[v] & kSiDeferred)
        { fr = Q.filt + size_t(v)*Q.filt_paths; in = Q.xscratch + size_t(v)*kLine; out = Q.dline + size_t(v)*kLine; }
    }
    else if(item - Q.num_direct < Q.num_entries)
    {
        const uint32_t e = item - Q.num_direct;
        const SendEntry en = Q.entries[e];
        if(Q.sendinfo[en.voice] & kSiSend)
        {
            fr = Q.filt + size_t(en.voice)*Q.filt_paths + 1u + en.send;
            in = Q.xscratch + size_t(en.voice)*kLine; out = Q.fscratch + size_t(e)*kLine;
        }
    }
    bool run = false;
    if(fr)
    {
        run = fr->active != 0u;
        if(!run)
        {
            // lpfilter.clear(); hpfilter.clear() (core/voice.cpp:265-266)
            #pragma unroll
            for(int f = 0;f < 2;++f)
            {
                #pragma unroll
                for(int k = 0;k < 5;++k) fr->cur[f][k] = fr->tgt[f][k];
                fr->z[f][0] = 0.0f; fr->z[f][1] = 0.0f; fr->counter[f] = 0;
            }
        }
    }
    inp[lane] = run ? in : nullptr;
    outp[lane] = run ? out : nullptr;
    if(!__any_sync(0xffffffffu, run)) return;

    BiquadCoefs c0{1.f,0.f,0.f,0.f,0.f}, c1 = c0, t0 = c0, t1 = c0;
    float z01 = 0.f, z02 = 0.f, z11 = 0.f, z12 = 0.f;
    int counter = 0;              // remaining interpolation steps
    uint32_t steprem = 0xffffffffu;   // samples until the next coefficient step
    int maxc = 0;
    if(run)
    {
        c0 = BiquadCoefs{fr->cur[0][0], fr->cur[0][1], fr->cur[0][2], fr->cur[0][3], fr->cur[0][4]};
        c1 = BiquadCoefs{fr->cur[1][0], fr->cur[1][1], fr->cur[1][2], fr->cur[1][3], fr->cur[1][4]};
        t0 = BiquadCoefs{fr->tgt[0][0], fr->tgt[0][1], fr->tgt[0][2], fr->tgt[0][3], fr->tgt[0][4]};
        t1 = BiquadCoefs{fr->tgt[1][0], fr->tgt[1][1], fr->tgt[1][2], fr->tgt[1][3], fr->tgt[1][4]};
        z01 = fr->z[0][0]; z02 = fr->z[0][1]; z11 = fr->z[1][0]; z12 = fr->z[1][1];
        maxc = max(fr->counter[0], fr->counter[1]);
        if(maxc > 0) { counter = maxc >> 5; steprem = 32u - uint32_t(maxc & 31); }
    }
    __syncwarp();

    const uint32_t tiles = (n + 31u) >> 5;
    float nx[32];
    // prefetch tile 0: row r = item r's 32 consecutive samples, one coalesced load per row
    #pragma unroll
    for(int r = 0;r < 32;++r)
    {
        const float *p = inp[r];
        nx[r] = (p && lane < n) ? __ldg(p + lane) : 0.0f;
    }
    for(uint32_t tb = 0;tb < tiles;++tb)
    {
        #pragma unroll
        for(int r = 0;r < 32;++r) tile[r][lane] = nx[r];
        __syncwarp();
        if(tb + 1u < tiles)
        {
            const uint32_t s = (tb + 1u)*32u + lane;
            #pragma unroll
            for(int r = 0;r < 32;++r)
            {
                const float *p = inp[r];
                nx[r] = (p && s < n) ? __ldg(p + s) : 0.0f;
            }
        }
        if(run)
        {
            const uint32_t cnt = min(32u, n - tb*32u);
            uint32_t i = 0;
            while(i < cnt)
            {
                if(cnt - i >= 8u && (counter <= 0 || steprem > 8u))
                {
                    // 8 samples with constant coefficients: straight-line code, so the input
                    // products are off the recurrence's critical path
                    float xin[8], yout[8];
                    #pragma unroll
                    for(int u = 0;u < 8;++u) xin[u] = tile[lane][i + u];
                    #pragma unroll
                    for(int u = 0;u < 8;++u)
                    {
                        const float x0 = xin[u];
                        const float y0 = __fadd_rn(__fmul_rn(x0, c0.b0), z01);
                        z01 = __fadd_rn(__fsub_rn(__fmul_rn(x0, c0.b1), __fmul_rn(y0, c0.a1)), z02);
                        z02 = __fsub_rn(__fmul_rn(x0, c0.b2), __fmul_rn(y0, c0.a2));
                        const float y1 = __fadd_rn(__fmul_rn(y0, c1.b0), z11);
                        z11 = __fadd_rn(__fsub_rn(__fmul_rn(y0, c1.b1), __fmul_rn(y1, c1.a1)), z12);
                        z12 = __fsub_rn(__fmul_rn(y0, c1.b2), __fmul_rn(y1, c1.a2));
                        yout[u] = y1;
                    }
                    #pragma unroll
                    for(int u = 0;u < 8;++u) tile[lane][i + u] = yout[u];
                    if(counter > 0) steprem -= 8u;
                    i += 8u;
                    continue;
                }
                // BiquadFilter::dualProcess body (biquad.cpp:264-275)
                const float x0 = tile[lane][i];
                const float y0 = __fadd_rn(__fmul_rn(x0, c0.b0), z01);
                z01 = __fadd_rn(__fsub_rn(__fmul_rn(x0, c0.b1), __fmul_rn(y0, c0.a1)), z02);
                z02 = __fsub_rn(__fmul_rn(x0, c0.b2), __fmul_rn(y0, c0.a2));
                const float y1 = __fadd_rn(__fmul_rn(y0, c1.b0), z11);
                z11 = __fadd_rn(__fsub_rn(__fmul_rn(y0, c1.b1), __fmul_rn(y1, c1.a1)), z12);
                z12 = __fsub_rn(__fmul_rn(y0, c1.b2), __fmul_rn(y1, c1.a2));
                tile[lane][i] = y1;
                ++i;
                // BiquadInterpFilter::dualProcess stepping (biquad.cpp:293-338)
                if(counter > 0 && --steprem == 0u)
                {
                    steprem = 32u;
                    if(--counter == 0) { c0 = t0; c1 = t1; }
                    else
                    {
                        const float a = __fdiv_rn(1.0f, float(counter + 1));
                        c0.b0 = lerp_rn(c0.b0, t0.b0, a); c0.b1 = lerp_rn(c0.b1, t0.b1, a);
                        c0.b2 = lerp_rn(c0.b2, t0.b2, a); c0.a1 = lerp_rn(c0.a1, t0.a1, a);
                        c0.a2 = lerp_rn(c0.a2, t0.a2, a);
                        c1.b0 = lerp_rn(c1.b0, t1.b0, a); c1.b1 = lerp_rn(c1.b1, t1.b1, a);
                        c1.b2 = lerp_rn(c1.b2, t1.b2, a); c1.a1 = lerp_rn(c1.a1, t1.a1, a);
                        c1.a2 = lerp_rn(c1.a2, t1.a2, a);
                    }
                }
            }
        }
        __syncwarp();
        {
            const uint32_t s = tb*32u + lane;
            #pragma unroll
            for(int r = 0;r < 32;++r)
            {
                float *p = outp[r];
                if(p && s < n) p[s] = tile[r][lane];
            }
        }
        __syncwarp();
    }
    if(run)
    {
        fr->z[0][0] = z01; fr->z[0][1] = z02; fr->z[1][0] = z11; fr->z[1][1] = z12;
        if(maxc > 0)
        {
            fr->cur[0][0] = c0.b0; fr->cur[0][1] = c0.b1; fr->cur[0][2] = c0.b2; fr->cur[0][3] = c0.a1; fr->cur[0][4] = c0.a2;
            fr->cur[1][0] = c1.b0; fr->cur[1][1] = c1.b1; fr->cur[1][2] = c1.b2; fr->cur[1][3] = c1.a1; fr->cur[1][4] = c1.a2;
            // mCounter = (counter*SamplesPerStep) | samples already done in the current step
            const int nc = counter > 0 ? ((counter << 5) | int(32u - steprem)) : 0;
            fr->counter[0] = nc; fr->counter[1] = nc;
        }
    }
}

// grid (slot, tile of 128 samples, entry chunk), 256 threads = 8 warps.  A warp takes
// blocks of 32 consecutive (voice, send) entries of the chunk: one coalesced load brings the
// block's entries and their sendinfo words, which are then broadcast by shuffle, so the only
// dependent global loads inside the entry loop are the parked line (one float4 per lane,
// 4 consecutive samples) and the gains.  All wet channels of an entry are accumulated in
// registers in one pass (CH per pass).  The 8 warps' partial sums are combined through
// shared memory in warp order, chunks through k_reduce_rows: the result does not depend on
// scheduling.
template<int CH>
__global__ void __launch_bounds__(256, (CH > 4) ? 2 : 4) k_send_mix(const SendMixParams Q)
{
    __shared__ float part[8][4][128];
    const uint32_t slot = blockIdx.x;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const uint32_t i0 = blockIdx.y*128u + lane*4u;
    const uint32_t n = Q.frames;
    uint32_t e0 = Q.slot_start[slot], e1 = Q.slot_start[slot+1];
    if(Q.chunks > 1u)
    {
        const uint32_t per = (e1 - e0 + Q.chunks - 1u)/Q.chunks;
        e0 = min(e0 + blockIdx.z*per, e1);
        e1 = min(e0 + per, e1);
    }
    // the CTA's entries are split evenly over its 8 warps (contiguous ranges)
    const uint32_t wblock = (e1 - e0 + 7u)/8u;
    float *outBase = Q.chunks > 1u
        ? Q.partial + (size_t(blockIdx.z)*gridDim.x + slot)*Q.cw*kLine
        : Q.wet + size_t(slot)*Q.cw*kLine;
    for(uint32_t c0 = 0;c0 < Q.cw;c0 += CH)
    {
        float acc[CH][4];
        #pragma unroll
        for(int c = 0;c < CH;++c) { acc[c][0] = acc[c][1] = acc[c][2] = acc[c][3] = 0.0f; }
        // Tiles that start at sample 128 or later are past every fade (Counter <= 64): the gain
        // of an entry-channel is the constant k_send_gains_prepare left in geff.  Full tiles
        // only, so no per-sample bound checks: one float4 of the line, CH broadcast gains,
        // 4*CH FMAs per entry.
        const bool plainTile = blockIdx.y > 0u && (blockIdx.y + 1u)*128u <= n && (Q.cw & 3u) == 0u;
        if(plainTile)
        {
            for(uint32_t base = e0 + warp*wblock;base < min(e0 + (warp + 1u)*wblock, e1);base += 32u)
            {
                const uint32_t cnt = min(32u, min(e0 + (warp + 1u)*wblock, e1) - base);
                uint32_t myVoice = 0u, myLine = 0u;     // myLine: 0 xscratch, 1 dline, 2 fscratch
                if(lane < cnt)
                {
                    const SendEntry en = Q.entries[base + lane];
                    myVoice = en.voice;
                    if(Q.dline) myLine = (Q.sendinfo[en.voice] & kSiDeferred) ? 1u : 0u;
                    else if(Q.filt && Q.filt[size_t(en.voice)*Q.filt_paths + 1u + en.send].active) myLine = 2u;
                }
                constexpr int U = (CH > 4) ? 2 : 4;      // entries in flight per lane
                for(uint32_t u0 = 0;u0 < cnt;u0 += U)
                {
                    float4 xU[U]; float4 gU[U][CH/4];
                    #pragma unroll
                    for(int q = 0;q < U;++q)
                    {
                        const uint32_t u = min(u0 + uint32_t(q), cnt - 1u);
                        const uint32_t voice = __shfl_sync(0xffffffffu, myVoice, int(u));
                        const uint32_t which = __shfl_sync(0xffffffffu, myLine, int(u));
                        const float *line = which == 0u ? Q.xscratch + size_t(voice)*kLine
                            : (which == 1u ? Q.dline + size_t(voice)*kLine : Q.fscratch + size_t(base + u)*kLine);
                        xU[q] = *reinterpret_cast<const float4*>(line + i0);
                        const float4 *gp = reinterpret_cast<const float4*>(Q.geff + size_t(base + u)*Q.cw + c0);
                        #pragma unroll
                        for(int g4 = 0;g4 < CH/4;++g4)
                            gU[q][g4] = (c0 + uint32_t(g4)*4u < Q.cw && u0 + uint32_t(q) < cnt) ? gp[g4]
                                : make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                    #pragma unroll
                    for(int q = 0;q < U;++q)
                    {
                        const float xs[4] = {xU[q].x, xU[q].y, xU[q].z, xU[q].w};
                        #pragma unroll
                        for(int g4 = 0;g4 < CH/4;++g4)
                        {
                            const float gg[4] = {gU[q][g4].x, gU[q][g4].y, gU[q][g4].z, gU[q][g4].w};
                            #pragma unroll
                            for(int cc = 0;cc < 4;++cc)
                                #pragma unroll
                                for(int k = 0;k < 4;++k)
                                    acc[g4*4 + cc][k] = fmaf(xs[k], gg[cc], acc[g4*4 + cc][k]);
                        }
                    }
                }
            }
        }
        else
        for(uint32_t base = e0 + warp*wblock;base < min(e0 + (warp + 1u)*wblock, e1);base += 32u)
        {
            // first tile (fades) or a partial tile: gain(i) = i < L ? a + b*i : flat from the
            // ramp k_send_gains_prepare left per entry-channel (Mix_, mixer_c.cpp:150-186)
            const uint32_t cnt = min(32u, min(e0 + (warp + 1u)*wblock, e1) - base);
            uint32_t myVoice = 0u, myLine = 0u;
            if(lane < cnt)
            {
                const SendEntry en = Q.entries[base + lane];
                myVoice = en.voice;
                if(Q.dline) myLine = (Q.sendinfo[en.voice] & kSiDeferred) ? 1u : 0u;
                else if(Q.filt && Q.filt[size_t(en.voice)*Q.filt_paths + 1u + en.send].active) myLine = 2u;
            }
            for(uint32_t u = 0;u < cnt;++u)
            {
                const uint32_t voice = __shfl_sync(0xffffffffu, myVoice, int(u));
                const uint32_t which = __shfl_sync(0xffffffffu, myLine, int(u));
                const float *line = which == 0u ? Q.xscratch + size_t(voice)*kLine
                    : (which == 1u ? Q.dline + size_t(voice)*kLine : Q.fscratch + size_t(base + u)*kLine);
                float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
                if(i0 < n) x = *reinterpret_cast<const float4*>(line + i0);
                const float4 *gp = Q.gramp + size_t(base + u)*Q.cw + c0;
                float xs[4] = {x.x, x.y, x.z, x.w};
                float fi[4];
                #pragma unroll
                for(int k = 0;k < 4;++k)
                {
                    if(i0 + k >= n) xs[k] = 0.0f;
                    fi[k] = float(i0 + k);
                }
                #pragma unroll
                for(int g4 = 0;g4 < CH/4;++g4)
                {
                    float4 rp[4];
                    #pragma unroll
                    for(int cc = 0;cc < 4;++cc)
                        rp[cc] = (c0 + g4*4 + cc < Q.cw) ? gp[g4*4 + cc] : make_float4(0.f, 0.f, 0.f, 0.f);
                    #pragma unroll
                    for(int cc = 0;cc < 4;++cc)
                    {
                        #pragma unroll
                        for(int k = 0;k < 4;++k)
                        {
                            const float g = (fi[k] < rp[cc].w) ? fmaf(rp[cc].y, fi[k], rp[cc].x) : rp[cc].z;
                            acc[g4*4 + cc][k] = fmaf(xs[k], g, acc[g4*4 + cc][k]);
                        }
                    }
                }
            }
        }
        // combine the 8 warps' partials, four channels at a time, in warp order
        #pragma unroll
        for(int g4 = 0;g4 < CH/4;++g4)
        {
            #pragma unroll
            for(int cc = 0;cc < 4;++cc)
                #pragma unroll
                for(int k = 0;k < 4;++k) part[warp][cc][lane*4 + k] = acc[g4*4 + cc][k];
            __syncthreads();
            if(threadIdx.x < 128u)
            {
                const uint32_t i = blockIdx.y*128u + threadIdx.x;
                #pragma unroll
                for(uint32_t cc = 0;cc < 4u;++cc)
                {
                    const uint32_t c = c0 + uint32_t(g4)*4u + cc;
                    if(c < Q.cw && (i < n || Q.chunks > 1u))
                    {
                        float sum = part[0][cc][threadIdx.x];
                        #pragma unroll
                        for(int wv = 1;wv < 8;++wv) sum += part[wv][cc][threadIdx.x];
                        outBase[size_t(c)*kLine + i] = sum;
                    }
                }
            }
            __syncthreads();
        }
    }
}

// Gain of every (entry, channel) once its fade has ended (Mix_, mixer_c.cpp:150-186: the
// target, or silence below GainSilenceThreshold / when the voice is stopping); runs before
// k_send_mix.  One thread per entry-channel.
__global__ void k_send_gains_prepare(const SendMixParams Q, uint32_t num_entries)
{
    const uint32_t idx = blockIdx.x*blockDim.x + threadIdx.x;
    const uint32_t e = idx / Q.cw, c = idx - e*Q.cw;
    if(e >= num_entries) return;
    const SendEntry en = Q.entries[e];
    const uint32_t info = Q.sendinfo[en.voice];
    float flat = 0.0f;
    float4 ramp = make_float4(0.f, 0.f, 0.f, 0.f);
    if(info & Q.valid_bit)
    {
        const bool playing = (info & kSiPlaying) != 0;
        const uint32_t counter = (info >> 8) & 0xffu, n = Q.frames;
        const float delta = counter ? 1.0f/float(counter) : 0.0f;
        const uint32_t fadeLen = counter < n ? counter : n;
        const size_t g = (size_t(en.voice)*Q.num_sends + en.send)*Q.cw + c;
        const float tg0 = Q.send_tgt[g];
        const float cg = counter ? Q.send_cur[g] : tg0;
        const float tg = playing ? tg0 : 0.0f;
        const float step = (tg - cg)*delta;
        const bool fade = fabsf(step) > kEps;
        const bool early = fade && fadeLen < counter;
        flat = (!early && fabsf(tg) > kSilence) ? tg : 0.0f;
        // fading: cg + step*i for i < fadeLen, then flat; not fading: flat from sample 0
        ramp = fade ? make_float4(cg, step, flat, float(fadeLen)) : make_float4(0.f, 0.f, flat, 0.f);
    }
    Q.geff[size_t(e)*Q.cw + c] = flat;
    Q.gramp[size_t(e)*Q.cw + c] = ramp;
}

// New Current gains of the sends (runs after k_send_mix; one thread per entry-channel).
__global__ void k_send_gains_update(const SendMixParams Q, uint32_t num_entries)
{
    const uint32_t idx = blockIdx.x*blockDim.x + threadIdx.x;
    const uint32_t e = idx / Q.cw, c = idx - e*Q.cw;
    if(e >= num_entries) return;
    const SendEntry en = Q.entries[e];
    const uint32_t info = Q.sendinfo[en.voice];
    if(!(info & Q.valid_bit)) return;
    const bool playing = (info & kSiPlaying) != 0;
    const uint32_t counter = (info >> 8) & 0xffu, n = Q.frames;
    const float delta = counter ? 1.0f/float(counter) : 0.0f;
    const uint32_t fadeLen = counter < n ? counter : n;
    const size_t g = (size_t(en.voice)*Q.num_sends + en.send)*Q.cw + c;
    const float tg0 = Q.send_tgt[g];
    const float cg = counter ? Q.send_cur[g] : tg0;
    const float tg = playing ? tg0 : 0.0f;
    const float step = (tg - cg)*delta;
    const bool early = (fabsf(step) > kEps) && fadeLen < counter;
    Q.send_cur[g] = early ? (cg + step*float(fadeLen)) : tg;
}

// ---- 256-point complex FFT in shared memory (128 threads, radix-2 DIT) -------------------
// tw[k] = exp(-2 pi i k/256), k < 128.  data must hold the input in bit-reversed order.
__device__ __forceinline__ uint32_t bitrev8(uint32_t v) { return __brev(v) >> 24; }

__device__ __forceinline__ void fft256_inplace(float2 *data, const float2 *__restrict__ tw, int t)
{
    #pragma unroll
    for(int stage = 0;stage < 8;++stage)
    {
        const int half = 1 << stage;
        const int grp = t >> stage, pos = t & (half-1);
        const int i0 = (grp << (stage+1)) + pos, i1 = i0 + half;
        const float2 w = tw[pos << (7-stage)];
        const float2 a = data[i0], b = data[i1];
        const float2 bw = make_float2(b.x*w.x - b.y*w.y, b.x*w.y + b.y*w.x);
        __syncthreads();
        data[i0] = make_float2(a.x + bw.x, a.y + bw.y);
        data[i1] = make_float2(a.x - bw.x, a.y - bw.y);
        __syncthreads();
    }
}

struct ConvParams {
    const SlotRec *slots; const float *wet; const float2 *twiddle;
    uint32_t frames, cw, num_slots, stage;
    uint32_t chunks;                  // gridDim.z of k_conv_mac
};

// segment range of chunk z of `chunks` over `segs` segments; zcnt = chunks that are not empty
__device__ __forceinline__ uint32_t conv_chunk_len(uint32_t segs, uint32_t chunks)
{ return (segs + chunks - 1u)/chunks; }

// grid = slots, 128 threads
__global__ void __launch_bounds__(128) k_conv_input(const ConvParams Q)
{
    __shared__ float stream[kConvFft + kLine + 8];
    __shared__ float2 fbuf[kConvFft];
    __shared__ float hsm[kConvBlock];
    const SlotRec &S = Q.slots[blockIdx.x];
    if(S.type != 1u || S.stage != Q.stage) return;
    ConvRing &G = *S.ring;
    const int t = threadIdx.x;
    const uint32_t n = Q.frames, f = G.fifo, cur = G.cur, ring = S.segs + kConvMaxBlocks;
    const uint32_t nb = (f + n) / kConvBlock;
    const float *in = Q.wet + size_t(blockIdx.x)*Q.cw*kLine;          // wet channel 0
    // stream = [previous block | partial block (f) | new samples (n)]
    for(uint32_t k = t;k < kConvBlock + f;k += 128) stream[k] = S.inbuf[k];
    for(uint32_t k = t;k < n;k += 128) stream[kConvBlock + f + k] = in[k];
    __syncthreads();

    // spectra of the blocks completed by this update -> ring slots cur, cur-1, ...
    for(uint32_t b = 0;b < nb;++b)
    {
        const float *blk = stream + kConvBlock + b*kConvBlock;
        // [128 samples | 128 zeros], loaded in bit-reversed order
        for(int k = t;k < kConvFft;k += 128)
        {
            const uint32_t r = bitrev8(uint32_t(k));
            fbuf[k] = make_float2(r < uint32_t(kConvBlock) ? blk[r] : 0.0f, 0.0f);
        }
        __syncthreads();
        fft256_inplace(fbuf, Q.twiddle, t);
        const uint32_t slotIdx = (cur + ring - b) % ring;
        float2 *dst = reinterpret_cast<float2*>(S.X + size_t(slotIdx)*kConvFft);
        dst[t] = (t == 0) ? make_float2(fbuf[0].x, fbuf[128].x) : fbuf[t];
        __syncthreads();
    }

    // 128-tap time-domain head (apply_fir, convolution.cpp:205-251)
    for(uint32_t c = 0;c < S.channels;++c)
    {
        hsm[t] = S.head[c*kConvBlock + t];
        __syncthreads();
        for(uint32_t i = t;i < n;i += 128)
        {
            const float *p = stream + kConvBlock + f + i;      // newest sample of output i
            float a0 = 0.0f, a1 = 0.0f;
            #pragma unroll 8
            for(int k = 0;k < kConvBlock;k += 2)
            {
                a0 = fmaf(hsm[k], p[-k], a0);
                a1 = fmaf(hsm[k+1], p[-k-1], a1);
            }
            S.lines[size_t(c)*kLine + i] = a0 + a1;
        }
        __syncthreads();
    }

    // new mInput: [last complete block | partial block]
    const uint32_t fNew = (f + n) - nb*kConvBlock;
    float keep0 = stream[nb*kConvBlock + t];
    float keep1 = (uint32_t(t) < fNew) ? stream[(nb+1)*kConvBlock + t] : 0.0f;
    S.inbuf[t] = keep0;
    S.inbuf[kConvBlock + t] = keep1;
    if(t == 0)
    {
        G.nb_last = nb; G.f_last = f; G.cur_last = cur;
        G.fifo = fNew;
        G.cur = (cur + ring - nb) % ring;
    }
}

// grid (slots, channels, segment chunks), 128 threads = the 128 packed bins.  The filter spectra
// are the one HBM-bound stream of the effects stage (2 s IR: 767 KB per slot and channel, plus
// as much input-spectrum history).  A chunk's filter and input rows (1 KB each) are streamed
// into a 3-stage shared-memory ring by bulk copies (cp.async.bulk, the 1-D form of TMA) that
// complete on mbarriers: one thread issues the copies of the stage after next while all threads
// accumulate the current one, so HBM stays busy during the arithmetic; the chunks spread one
// slot's stream over the SMs and leave partial sums in yspec that k_conv_ifft adds in chunk
// order (deterministic).  A thread keeps the accumulators of ALL blocks completed this update
// (<= 9) in registers: X[(cur0 - b + s)] is a sliding window over the spectrum ring, so each
// segment costs ONE new input bin and ONE filter bin for up to 9 complex MACs.  Stages hold 9
// segments aligned to multiples of 9, so the window rotation is a compile-time renaming.
constexpr int kConvStages = 3;
struct ConvMacSmem {
    float2 H[kConvStages][kConvMaxBlocks][128];
    float2 X[kConvStages][kConvMaxBlocks][128];
    uint64_t full[kConvStages];
};

__global__ void __launch_bounds__(128) k_conv_mac(const ConvParams Q)
{
    constexpr int NB = kConvMaxBlocks;
    extern __shared__ __align__(128) unsigned char conv_smem_raw[];
    ConvMacSmem &M = *reinterpret_cast<ConvMacSmem*>(conv_smem_raw);
    const SlotRec &S = Q.slots[blockIdx.x];
    if(S.type != 1u || S.stage != Q.stage || blockIdx.y >= S.channels) return;
    const ConvRing &G = *S.ring;
    const uint32_t nb = G.nb_last;
    if(nb == 0) return;
    const int t = threadIdx.x;
    const uint32_t segs = S.segs, cur0 = G.cur_last, ring = segs + kConvMaxBlocks;
    const uint32_t clen = conv_chunk_len(segs, gridDim.z);
    const uint32_t s0 = blockIdx.z*clen;
    if(s0 >= segs) return;                                   // empty chunk (short IR)
    const uint32_t s1 = (s0 + clen < segs) ? s0 + clen : segs;
    const float *Xg = S.X;
    const float *Hg = S.H + size_t(blockIdx.y)*segs*kConvFft;
    // rounds of NB segments aligned to multiples of NB: the window slot (s mod NB) is static
    const uint32_t r0 = s0 - (s0 % uint32_t(NB));
    const uint32_t rounds = (s1 - r0 + uint32_t(NB) - 1u)/uint32_t(NB);

    if(t == 0)
    {
        for(int st = 0;st < kConvStages;++st) mbar_init(&M.full[st], 1u);
        mbar_fence_init();
    }
    __syncthreads();
    // producer: the rows of round r go to stage r % kConvStages
    auto issue = [&](uint32_t r) {
        const uint32_t sb = r0 + r*uint32_t(NB);
        const int st = int(r % uint32_t(kConvStages));
        uint32_t rows = 0;
        for(int u = 0;u < NB;++u) { const uint32_t s = sb + uint32_t(u); if(s >= s0 && s < s1) ++rows; }
        mbar_expect_tx(&M.full[st], rows*2u*uint32_t(kConvFft)*4u);
        for(int u = 0;u < NB;++u)
        {
            const uint32_t s = sb + uint32_t(u);
            if(s < s0 || s >= s1) continue;
            uint32_t q = cur0 + s;                 // cur0 < ring, s < segs < ring
            q = q >= ring ? q - ring : q;
            bulk_g2s(M.X[st][u], Xg + size_t(q)*kConvFft, kConvFft*4u, &M.full[st]);
            bulk_g2s(M.H[st][u], Hg + size_t(s)*kConvFft, kConvFft*4u, &M.full[st]);
        }
    };
    if(t == 0)
        for(uint32_t r = 0;r < rounds && r < uint32_t(kConvStages);++r) issue(r);

    float2 acc[NB], xw[NB];          // xw[s mod NB] holds X[(cur0 + s) mod ring]
    #pragma unroll
    for(int b = 0;b < NB;++b) acc[b] = make_float2(0.f, 0.f);
    #pragma unroll
    for(int u = 0;u < NB;++u) xw[u] = make_float2(0.f, 0.f);
    {
        // history the first segments of the range look back at: X[cur0 + s0 - d], d = 1..NB-1
        // (plain loads, in flight together with the first stages)
        const float2 *X = reinterpret_cast<const float2*>(Xg) + t;
        float2 hv[NB];
        #pragma unroll
        for(int d = 1;d < NB;++d)
        {
            const uint32_t q = (cur0 + 2u*ring + s0 - uint32_t(d)) % ring;
            hv[d] = X[size_t(q)*128];
        }
        #pragma unroll
        for(int d = 1;d < NB;++d)
        {
            const int slotIdx = int((s0 + uint32_t(NB)*8u - uint32_t(d)) % uint32_t(NB));
            #pragma unroll
            for(int u = 0;u < NB;++u) if(u == slotIdx) xw[u] = hv[d];
        }
    }
    for(uint32_t r = 0;r < rounds;++r)
    {
        const int st = int(r % uint32_t(kConvStages));
        mbar_wait(&M.full[st], (r / uint32_t(kConvStages)) & 1u);
        const uint32_t sb = r0 + r*uint32_t(NB);
        #pragma unroll
        for(int u = 0;u < NB;++u)
        {
            const uint32_t s = sb + uint32_t(u);
            if(s >= s0 && s < s1)
            {
                xw[u] = M.X[st][u][t];
                const float2 h = M.H[st][u][t];
                #pragma unroll
                for(int b = 0;b < NB;++b)
                {
                    const float2 xv = xw[(u - b + NB) % NB];   // X[cur0 + s - b]
                    if(t == 0)
                    {   // packed DC / Nyquist: two independent real products
                        acc[b].x = fmaf(xv.x, h.x, acc[b].x);
                        acc[b].y = fmaf(xv.y, h.y, acc[b].y);
                    }
                    else
                    {
                        acc[b].x = fmaf(xv.x, h.x, fmaf(-xv.y, h.y, acc[b].x));
                        acc[b].y = fmaf(xv.x, h.y, fmaf(xv.y, h.x, acc[b].y));
                    }
                }
            }
        }
        __syncthreads();                       // every thread is done with this stage
        if(t == 0 && r + uint32_t(kConvStages) < rounds) issue(r + uint32_t(kConvStages));
    }
    float2 *Y = reinterpret_cast<float2*>(S.yspec
        + (size_t(blockIdx.y)*kConvMaxChunks + blockIdx.z)*kConvMaxBlocks*kConvFft) + t;
    #pragma unroll
    for(int b = 0;b < NB;++b)
        if(uint32_t(b) < nb) Y[size_t(b)*128] = acc[b];
}

// grid (slots, channels, blocks), 128 threads: the accumulated spectrum of one completed block
// (sum of the segment chunks' partials, in chunk order) through the inverse FFT; the 256
// time-domain samples replace chunk 0's partial of that block in yspec.
__global__ void __launch_bounds__(128) k_conv_ifft(const ConvParams Q)
{
    __shared__ float2 fbuf[kConvFft];
    __shared__ float2 ysp[kConvBlock];
    const SlotRec &S = Q.slots[blockIdx.x];
    if(S.type != 1u || S.stage != Q.stage || blockIdx.y >= S.channels || blockIdx.z >= S.ring->nb_last) return;
    const int t = threadIdx.x;
    const uint32_t c = blockIdx.y, b = blockIdx.z;
    const uint32_t clen = conv_chunk_len(S.segs, Q.chunks);
    const uint32_t zcnt = (S.segs + clen - 1u)/clen;
    float2 ysum = make_float2(0.f, 0.f);
    for(uint32_t z = 0;z < zcnt;++z)
    {
        const float2 a = reinterpret_cast<const float2*>(S.yspec
            + ((size_t(c)*kConvMaxChunks + z)*kConvMaxBlocks + b)*kConvFft)[t];
        ysum.x += a.x; ysum.y += a.y;
    }
    ysp[t] = ysum;
    __syncthreads();
    // inverse FFT: ifft(x) = conj(fft(conj(x)))
    const float2 y0 = ysp[0];
    for(int k = t;k < kConvFft;k += 128)
    {
        float2 v;
        if(k == 0) v = make_float2(y0.x, 0.0f);
        else if(k == 128) v = make_float2(y0.y, 0.0f);
        else if(k < 128) { const float2 a = ysp[k]; v = make_float2(a.x, -a.y); }       // conj(x_k)
        else { const float2 a = ysp[256-k]; v = make_float2(a.x, a.y); }                // conj(conj(x_{N-k}))
        fbuf[bitrev8(uint32_t(k))] = v;
    }
    __syncthreads();
    fft256_inplace(fbuf, Q.twiddle, t);
    float *yt = S.yspec + ((size_t(c)*kConvMaxChunks + 0u)*kConvMaxBlocks + b)*kConvFft;
    yt[t] = fbuf[t].x; yt[kConvBlock + t] = fbuf[kConvBlock + t].x;
}

// grid (slots, channels), 128 threads: overlap-add of the blocks' time-domain outputs
// (convolution.cpp:699-706) into the slot's output lines.
__global__ void __launch_bounds__(128) k_conv_output(const ConvParams Q)
{
    const SlotRec &S = Q.slots[blockIdx.x];
    if(S.type != 1u || S.stage != Q.stage || blockIdx.y >= S.channels) return;
    const int t = threadIdx.x;
    const uint32_t c = blockIdx.y, n = Q.frames, nb = S.ring->nb_last, f = S.ring->f_last;
    float *ov = S.ov + size_t(c)*kConvFft;
    float *line = S.lines + size_t(c)*kLine;
    float first = ov[t], tail = ov[kConvBlock + t];
    // every thread owns sample t of each 128-sample block: no exchange between threads.
    // samples of the block that was in progress when the update started: line[i] += mOutput[f + i]
    {
        const uint32_t cnt = (kConvBlock - f < n) ? kConvBlock - f : n;
        if(uint32_t(t) >= f && uint32_t(t) - f < cnt) line[uint32_t(t) - f] += first;
    }
    for(uint32_t b = 0;b < nb;++b)
    {
        const float *yt = S.yspec + ((size_t(c)*kConvMaxChunks + 0u)*kConvMaxBlocks + b)*kConvFft;
        // O_b = y[0..128) + previous tail ; new tail = y[128..256)   (convolution.cpp:702-706)
        first = yt[t] + tail;
        tail = yt[kConvBlock + t];
        // the samples following this block boundary
        const uint32_t base = (b+1u)*kConvBlock - f;       // output index of the block start
        if(base < n)
        {
            const uint32_t cnt = (n - base < uint32_t(kConvBlock)) ? n - base : uint32_t(kConvBlock);
            if(uint32_t(t) < cnt) line[base + t] += first;
        }
    }
    ov[t] = first; ov[kConvBlock + t] = tail;
}

// Dry[o][i] += sum over slots/lines of line[i]*gain(i): MixSamples(Counter = samplesToDo)
// (ConvolutionState::NormalMix, convolution.cpp:298-304), slots and lines in index order.
struct SlotMixParams { const SlotRec *slots; float *dry; uint32_t frames, cd, num_slots, stage; float *wet; uint32_t cw; };

__global__ void __launch_bounds__(128) k_slot_output_mix(const SlotMixParams Q)
{
    // per-(slot,line) constants are staged once per CTA; the sample loop then only streams
    // the output lines (coalesced, independent loads)
    constexpr int kMaxLines = 16;
    __shared__ float s_cg[64][kMaxLines], s_tg[64][kMaxLines];
    __shared__ const float *s_line[64];
    __shared__ uint32_t s_ch[64], s_first[64], s_fade[64];
    const uint32_t o = blockIdx.y;
    const uint32_t i = blockIdx.x*128u + threadIdx.x;
    const uint32_t n = Q.frames;
    float acc = (i < n) ? Q.dry[size_t(o)*kLine + i] : 0.0f;
    const float delta = 1.0f/float(n);
    for(uint32_t sb = 0;sb < Q.num_slots;sb += 64u)
    {
        const uint32_t cnt = (Q.num_slots - sb < 64u) ? Q.num_slots - sb : 64u;
        __syncthreads();
        if(threadIdx.x < cnt)
        {
            const SlotRec &S = Q.slots[sb + threadIdx.x];
            // only this stage's slots whose output goes to the Dry mix (no target slot)
            uint32_t ch = (S.type == 0u || S.stage != Q.stage || S.target != 0xffffffffu) ? 0u
                : (S.channels < uint32_t(kMaxLines) ? S.channels : uint32_t(kMaxLines));
            uint32_t first = 0u;
            if(S.type == 2u)
            {
                // reverb: lines 0-7 belong to pipeline object 0, 8-15 to object 1; the current
                // pipeline is mixed first, then (while it rings out) the old one
                // (ReverbState::process, reverb.cpp:1843-1877)
                first = S.rv_cur*8u;
                if(ch) ch = (S.rv_mask == 3u) ? 16u : 8u;
            }
            s_ch[threadIdx.x] = ch;
            s_first[threadIdx.x] = first;
            s_fade[threadIdx.x] = S.fade_len ? min(S.fade_len, n) : n;
            s_line[threadIdx.x] = S.lines;
        }
        __syncthreads();
        // the gains of every (slot, line): one thread each, all loads independent
        for(uint32_t idx = threadIdx.x;idx < cnt*uint32_t(kMaxLines);idx += blockDim.x)
        {
            const uint32_t sl = idx / uint32_t(kMaxLines), c = idx % uint32_t(kMaxLines);
            if(c >= s_ch[sl]) continue;
            const SlotRec &S = Q.slots[sb + sl];
            const uint32_t li = (c + s_first[sl]) & (kMaxLines - 1u);
            s_cg[sl][c] = S.gains[li*32u + o];
            s_tg[sl][c] = S.gtgt[li*32u + o];
        }
        __syncthreads();
        // the slots' lines as a flat list of blocks of <= 8 lines; block b+1's samples are loaded
        // while block b is added (the adds stay in slot / line order): without the prefetch the
        // loop is one L2 round trip per slot
        uint32_t nblk = 0;
        for(uint32_t sl = 0;sl < cnt;++sl) nblk += (s_ch[sl] + 7u)/8u;
        uint32_t ps = 0, pc0 = 0;                       // the block being prefetched: (slot, first line)
        while(ps < cnt && s_ch[ps] == 0u) ++ps;
        float xn[8];
        #pragma unroll
        for(uint32_t k = 0;k < 8u;++k) xn[k] = 0.0f;
        auto load_block = [&](uint32_t sl, uint32_t c0)
        {
            const uint32_t ch = s_ch[sl], first = s_first[sl];
            const float *lines = s_line[sl];
            #pragma unroll
            for(uint32_t k = 0;k < 8u;++k)
            {
                const uint32_t li = (c0 + k + first) & (kMaxLines - 1u);
                xn[k] = (i < n && c0 + k < ch) ? lines[size_t(li)*kLine + i] : 0.0f;
            }
        };
        if(nblk) load_block(ps, pc0);
        for(uint32_t bk = 0;bk < nblk;++bk)
        {
            const uint32_t sl = ps, c0 = pc0;
            float xv[8];
            #pragma unroll
            for(uint32_t k = 0;k < 8u;++k) xv[k] = xn[k];
            // advance the prefetch cursor and issue the next block's loads
            pc0 += 8u;
            if(pc0 >= s_ch[ps]) { pc0 = 0u; ++ps; while(ps < cnt && s_ch[ps] == 0u) ++ps; }
            if(bk + 1u < nblk) load_block(ps, pc0);
            const uint32_t ch = s_ch[sl], L = s_fade[sl];
            const float dl = (L == n) ? delta : 1.0f/float(L);
            #pragma unroll
            for(uint32_t k = 0;k < 8u;++k)
            {
                const uint32_t c = c0 + k;
                if(c >= ch) break;
                const float cg = s_cg[sl][c], tg = s_tg[sl][c];
                const float step = (tg - cg)*dl;
                // MixLine (mixer_c.cpp:150-186): the ramp over the first L samples, then the target
                if(fabsf(step) > kEps && i < L) acc += xv[k]*(cg + step*float(i));
                else if(fabsf(tg) > kSilence) acc += xv[k]*tg;
            }
        }
    }
    if(i < n) Q.dry[size_t(o)*kLine + i] = acc;
}

// Slots with a target slot (EffectSlotBase::Target): their output lines are mixed into the
// target's Wet buffer before the target's stage runs.  grid (tile of 128 samples, target slot);
// the sources of one target are added in slot order (deterministic).  Full occupancy (16 CTAs per SM)
// fits in 32 registers.
__global__ void __launch_bounds__(128, 16) k_slot_target_mix(const SlotMixParams Q)
{
    const uint32_t t = blockIdx.y;
    const uint32_t i = blockIdx.x*128u + threadIdx.x;
    const uint32_t n = Q.frames;
    if(i >= n) return;
    const float delta = 1.0f/float(n);
    for(uint32_t s = 0;s < Q.num_slots;++s)
    {
        const SlotRec &S = Q.slots[s];
        if(S.type == 0u || S.stage != Q.stage || S.target != t) continue;
        uint32_t ch = S.channels, first = 0u;
        if(S.type == 2u) { first = S.rv_cur*8u; ch = (S.rv_mask == 3u) ? 16u : 8u; }
        const uint32_t L = S.fade_len ? min(S.fade_len, n) : n;
        const float dl = (L == n) ? delta : 1.0f/float(L);
        const float *gcur = S.gains;
        for(uint32_t o = 0;o < Q.cw;++o)
        {
            float acc = Q.wet[(size_t(t)*Q.cw + o)*kLine + i];
            for(uint32_t c = 0;c < ch;++c)
            {
                const uint32_t li = S.type == 2u ? ((c + first) & 15u) : c;
                const float cg = gcur[li*32u + o], tg = S.gtgt[li*32u + o];
                const float step = (tg - cg)*dl;
                const float x = S.lines[size_t(li)*kLine + i];
                if(fabsf(step) > kEps && i < L) acc += x*(cg + step*float(i));
                else if(fabsf(tg) > kSilence) acc += x*tg;
            }
            Q.wet[(size_t(t)*Q.cw + o)*kLine + i] = acc;
        }
    }
}

// Current <- Target for every slot line (the fade always completes: Counter == frames).
__global__ void k_slot_gains_commit(const SlotMixParams Q)
{
    const uint32_t s = blockIdx.x;
    const SlotRec &S = Q.slots[s];
    if(S.type == 0u) return;
    for(uint32_t k = threadIdx.x;k < S.channels*32u;k += blockDim.x)
    {
        // a reverb pipeline object that did not run this update keeps its Current gains
        if(S.type == 2u && !((S.rv_mask >> (k >> 8)) & 1u)) continue;
        S.gains[k] = S.gtgt[k];
    }
}

} // namespace b200mix

// =====================================================================================
// EAX / standard reverb: ReverbState::process for one pipeline in the Normal state
// (alc/effects/reverb.cpp:1813-1845).  One CTA per slot, 4 warps = the 4 A-format lines.
// Sample-parallel wherever the reference's data flow allows it (delay taps, all-pass
// sub-chunks bounded by the feedback delay, scatter matrices, modulated cubic taps);
// the biquad recurrences (master shelves, T60) run serially on lane 0 of each line warp.
// =====================================================================================
namespace b200mix {

struct ReverbDev {
    // parameters (b200mix_reverb_params)
    uint32_t main_len, late_in_len, early_ap_len, early_len, late_ap_len, late_len;
    uint32_t early_tap[4]; float early_tap_coeff; uint32_t late_tap[4];
    float mix_x, mix_y;
    float filter_lp[5], filter_hp[5];
    float early_ap_coeff; uint32_t early_ap_offset[4]; uint32_t early_offset[4]; float early_coeff;
    uint32_t late_offset[4]; float density_gain; float t60_mid_gain[4];
    float t60_hf[4][5], t60_lf[4][5];
    uint32_t mod_step; float mod_depth; float late_ap_coeff; uint32_t late_ap_offset[4];
    uint32_t upmix; float order_scale[2]; float split_coeff;      // MixOutAmbiUp
    // state
    float z_lp[4][2], z_hp[4][2], z_t60hf[4][2], z_t60lf[4][2];
    float z_split[2][4][3];                                        // mAmbiSplitter {lp_z1, lp_z2, ap_z1}
    uint32_t early_tap_cur[4], late_tap_cur[4]; float early_coeff_cur;
    uint32_t mod_index; uint32_t offset;
    uint32_t sync;                // (update seq << 8) | early chunks of this update that are complete
    // delay lines
    float *main_d, *late_in, *early_ap, *early_d, *late_ap, *late_d;
};

struct ReverbParamsK { const SlotRec *slots; const float *wet; const float *cubic; uint32_t frames, cw, stage, seq; };

__device__ __forceinline__ void scatter4(const float in[4], float x, float y, float out[4])
{
    // VectorPartialScatter, reverb.cpp:1396-1405
    out[0] = x*in[0] + y*(          in[1] + -in[2] + in[3]);
    out[1] = x*in[1] + y*(-in[0]          +  in[2] + in[3]);
    out[2] = x*in[2] + y*( in[0] + -in[1]          + in[3]);
    out[3] = x*in[3] + y*(-in[0] + -in[1] + -in[2]        );
}

// BiquadFilter::dualProcess (core/filters/biquad.cpp:254-283), in place, one thread; inputs and
// outputs move in 8-sample register batches so only the z-state is on the dependency chain.
__device__ __forceinline__ void dual_biquad_serial(const float *c0, const float *c1, float *z0,
    float *z1, float *buf, uint32_t n)
{
    const float b00 = c0[0], b01 = c0[1], b02 = c0[2], a01 = c0[3], a02 = c0[4];
    const float b10 = c1[0], b11 = c1[1], b12 = c1[2], a11 = c1[3], a12 = c1[4];
    float z01 = z0[0], z02 = z0[1], z11 = z1[0], z12 = z1[1];
    for(uint32_t i0 = 0;i0 < n;i0 += 8)
    {
        float x[8], y[8];
        #pragma unroll
        for(int k = 0;k < 8;++k) x[k] = (i0 + k < n) ? buf[i0+k] : 0.0f;
        #pragma unroll
        for(int k = 0;k < 8;++k)
        {
            const float x0 = x[k];
            const float y0 = x0*b00 + z01;
            const float n01 = x0*b01 - y0*a01 + z02;
            const float n02 = x0*b02 - y0*a02;
            const float y1 = y0*b10 + z11;
            const float n11 = y0*b11 - y1*a11 + z12;
            const float n12 = y0*b12 - y1*a12;
            y[k] = y1;
            if(i0 + k < n) { z01 = n01; z02 = n02; z11 = n11; z12 = n12; }
        }
        #pragma unroll
        for(int k = 0;k < 8;++k) if(i0 + k < n) buf[i0+k] = y[k];
    }
    z0[0] = z01; z0[1] = z02; z1[0] = z11; z1[1] = z12;
}

__global__ void __launch_bounds__(128) k_reverb_process(const ReverbParamsK Q)
{
    constexpr int NL = 4;
    constexpr uint32_t MAXUPD = 256;
    __shared__ float temp[NL][MAXUPD];
    __shared__ uint32_t moddel[MAXUPD];
    const SlotRec &S = Q.slots[blockIdx.x];
    if(S.type != 2u || S.stage != Q.stage || !((S.rv_mask >> blockIdx.y) & 1u)) return;
    // blockIdx.y = pipeline object (ReverbState::mPipelines[2]); both share the main delay line,
    // each early CTA writes this update's input into it itself (identical values) before reading it.
    // blockIdx.z = half: 0 runs B2A + processEarly, 1 runs processLate CONCURRENTLY on another SM.
    // The only data the late half takes from this update's early half is the late-input delay
    // line, read `late tap` (>= the late reverb delay) samples back: late chunk s may start once
    // the early chunks covering [.., base_s + todo_s - 1 - minTap] are complete (R.sync).
    ReverbDev &R = reinterpret_cast<ReverbDev*>(S.H)[blockIdx.y];
    const bool earlyHalf = blockIdx.z == 0u;
    const int tid = threadIdx.x, line = tid >> 5, lane = tid & 31;
    const uint32_t n = Q.frames;
    const uint32_t offset0 = R.offset;
    const float *wet = Q.wet + size_t(blockIdx.x)*Q.cw*kLine;
    const uint32_t numInput = Q.cw < 4u ? Q.cw : 4u;
    float *earlyOut = S.lines + size_t(blockIdx.y)*8*kLine, *lateOut = earlyOut + 4*kLine;

    // B-Format -> A-Format into the main delay (reverb.cpp:1824-1838, B2A :91-97)
    if(earlyHalf)
    {
        const float B2A[4][4] = {{0.5f, 0.5f, 0.5f, 0.5f}, {0.5f, -0.5f, -0.5f, 0.5f},
            {0.5f, 0.5f, -0.5f, -0.5f}, {0.5f, -0.5f, 0.5f, -0.5f}};
        float *dl = R.main_d + size_t(line)*R.main_len;
        // (all loads of a batch are issued before the first store: the delay lines are plain
        // pointers, so the compiler must assume a store may alias the next load)
        for(uint32_t i0 = lane;i0 < n;i0 += 8u*32u)
        {
            float w[8][4];
            #pragma unroll
            for(int u = 0;u < 8;++u)
                #pragma unroll
                for(int k = 0;k < 4;++k)
                {
                    const uint32_t i = i0 + uint32_t(u)*32u;
                    w[u][k] = (i < n && uint32_t(k) < numInput) ? wet[size_t(k)*kLine + i] : 0.0f;
                }
            #pragma unroll
            for(int u = 0;u < 8;++u)
            {
                const uint32_t i = i0 + uint32_t(u)*32u;
                float a = 0.0f;
                #pragma unroll
                for(int k = 0;k < 4;++k) if(uint32_t(k) < numInput) a = a + w[u][k]*B2A[line][k];
                if(i < n) dl[(offset0 + i) & (R.main_len-1)] = a;
            }
        }
    }
    __syncthreads();

    // ---- processEarly, reverb.cpp:1558-1660 ----
    uint32_t offset = offset0;
    float coeffCur = R.early_coeff_cur;
    uint32_t tapCur = R.early_tap_cur[line];
    uint32_t chunksDone = 0;
    for(uint32_t base = 0;earlyHalf && base < n;)
    {
        const uint32_t todo = (n-base < MAXUPD) ? n-base : MAXUPD;
        const float fadeStep = 1.0f/float(todo);
        const float c0 = coeffCur, c1 = R.early_tap_coeff;
        coeffCur = c1;
        {
            const float *input = R.main_d + size_t(line)*R.main_len;
            const uint32_t t0 = offset - tapCur, t1 = offset - R.early_tap[line];
            tapCur = R.early_tap[line];
            float v0[8], v1[8];
            #pragma unroll
            for(int u = 0;u < 8;++u)
            {
                const uint32_t i = lane + uint32_t(u)*32u;
                v0[u] = i < todo ? input[(t0+i) & (R.main_len-1)] : 0.0f;
                v1[u] = i < todo ? input[(t1+i) & (R.main_len-1)] : 0.0f;
            }
            #pragma unroll
            for(int u = 0;u < 8;++u)
            {
                const uint32_t i = lane + uint32_t(u)*32u;
                const float a = v0[u]*c0, b = v1[u]*c1;
                if(i < todo) temp[line][i] = a + (b-a)*(fadeStep*float(i));
            }
        }
        __syncwarp();
        if(lane == 0)
            dual_biquad_serial(R.filter_lp, R.filter_hp, R.z_lp[line], R.z_hp[line], temp[line], todo);
        __syncwarp();
        // Allpass4::process (reverb.cpp:1508-1538): sub-chunks no longer than the feedback delay
        {
            float *buf = R.early_ap + size_t(line)*R.early_ap_len;
            const uint32_t m = R.early_ap_len-1, off = R.early_ap_offset[line];
            const float fc = R.early_ap_coeff;
            for(uint32_t sb = 0;sb < todo;sb += off)
            {
                const uint32_t td = (todo - sb < off) ? todo - sb : off;
                float dv[8];
                #pragma unroll
                for(int u = 0;u < 8;++u)
                {
                    const uint32_t i = lane + uint32_t(u)*32u;
                    dv[u] = i < td ? buf[(offset + sb + i - off) & m] : 0.0f;
                }
                #pragma unroll
                for(int u = 0;u < 8;++u)
                {
                    const uint32_t i = lane + uint32_t(u)*32u;
                    if(i < td)
                    {
                        const float x = temp[line][sb+i];
                        const float y = dv[u] - fc*x;
                        buf[(offset + sb + i) & m] = x + fc*y;
                        temp[line][sb+i] = y;
                    }
                }
                __syncwarp();
            }
        }
        __syncthreads();
        // writeReflected (reverb.cpp:340-365)
        for(uint32_t i = tid;i < todo;i += 128)
        {
            const float s0 = temp[0][i], s1 = temp[1][i], s2 = temp[2][i], s3 = temp[3][i];
            const uint32_t o = (offset+i) & (R.early_len-1);
            R.early_d[0*size_t(R.early_len) + o] = (s0      - s1 - s2 - s3) * 0.5f;
            R.early_d[1*size_t(R.early_len) + o] = (s1 - s0      - s2 - s3) * 0.5f;
            R.early_d[2*size_t(R.early_len) + o] = (s2 - s0 - s1      - s3) * 0.5f;
            R.early_d[3*size_t(R.early_len) + o] = (s3 - s0 - s1 - s2     ) * 0.5f;
        }
        __syncthreads();
        {
            const float *dl = R.early_d + size_t(line)*R.early_len;
            const uint32_t tap = offset - R.early_offset[line];
            float dv[8];
            #pragma unroll
            for(int u = 0;u < 8;++u)
            {
                const uint32_t i = lane + uint32_t(u)*32u;
                dv[u] = i < todo ? dl[(tap+i) & (R.early_len-1)] : 0.0f;
            }
            const float ec = R.early_coeff;
            #pragma unroll
            for(int u = 0;u < 8;++u)
            {
                const uint32_t i = lane + uint32_t(u)*32u;
                if(i < todo) earlyOut[size_t(line)*kLine + base + i] = dv[u]*ec + temp[line][i];
            }
        }
        __syncthreads();
        // VectorScatter + late-input write (reverb.cpp:1649-1655)
        for(uint32_t i = tid;i < todo;i += 128)
        {
            const float in[4] = {temp[0][i], temp[1][i], temp[2][i], temp[3][i]};
            float f[4];
            scatter4(in, R.mix_x, R.mix_y, f);
            const uint32_t o = (offset+i) & (R.late_in_len-1);
            #pragma unroll
            for(int j = 0;j < NL;++j) R.late_in[size_t(j)*R.late_in_len + o] = f[j];
        }
        __syncthreads();
        base += todo; offset += todo;
        // publish: this chunk's late-input samples are in memory
        ++chunksDone;
        if(tid == 0)
        {
            __threadfence();
            asm volatile("st.release.gpu.global.u32 [%0], %1;" :: "l"(&R.sync), "r"((Q.seq << 8) | chunksDone) : "memory");
        }
    }
    if(earlyHalf)
    {
        if(lane == 0)
        {
            R.early_tap_cur[line] = tapCur;
            if(line == 0) R.early_coeff_cur = coeffCur;
        }
        return;
    }

    // ---- processLate, reverb.cpp:1696-1811 ----
    offset = offset0;
    uint32_t modIdx = R.mod_index;
    uint32_t ltapCur = R.late_tap_cur[line];
    for(uint32_t base = 0;base < n;)
    {
        uint32_t todo = R.late_offset[0] < MAXUPD ? R.late_offset[0] : MAXUPD;
        if(n-base < todo) todo = n-base;
        {
            // early chunks (of MAXUPD samples) this chunk's late-input taps reach into
            uint32_t minTap = 0xffffffffu;
            for(int j = 0;j < NL;++j)
            {
                minTap = min(minTap, R.late_tap[j]);
                minTap = min(minTap, R.late_tap_cur[j]);
            }
            const int64_t last = int64_t(base) + int64_t(todo) - 1 - int64_t(minTap);
            const uint32_t need = last < 0 ? 0u : min(uint32_t(last / int64_t(MAXUPD)) + 1u, (n + MAXUPD - 1u)/MAXUPD);
            if(need && tid == 0)
            {
                unsigned long long t0;
                asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
                for(;;)
                {
                    uint32_t v;
                    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(&R.sync) : "memory");
                    if((v >> 8) == (Q.seq & 0xffffffu) && (v & 0xffu) >= need) break;
                    unsigned long long t1;
                    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
                    if(t1 - t0 > 1000000000ull) break;          // never hang the GPU on a lost partner
                    __nanosleep(100);
                }
            }
            __syncthreads();
        }
        // Modulation::calcDelays (reverb.cpp:1662-1681)
        {
            const float depth = R.mod_depth*256.0f;
            for(uint32_t i = tid;i < todo;i += 128)
            {
                const uint32_t idx = modIdx + i*R.mod_step;
                const float x = float(idx & 0xffffffu) * (1.0f/16777216.0f);
                const float lfo = !(idx & 0x800000u) ? ((-16.0f*x*x) + (8.0f*x))
                    : ((16.0f*x*x) + (-8.0f*x) + (-16.0f*x) + 8.0f);
                const float v = (lfo+1.0f)*depth;
                moddel[i] = v > 0.0f ? uint32_t(v) : 0u;
            }
            modIdx += todo*R.mod_step;
        }
        __syncthreads();
        {
            const float *input = R.late_d + size_t(line)*R.late_len;
            const uint32_t m = R.late_len-1;
            const float midGain = R.t60_mid_gain[line];
            const uint32_t tap = offset - R.late_offset[line];
            float o[8][4], cb[8][4];
            #pragma unroll
            for(int u = 0;u < 8;++u)
            {
                const uint32_t i = lane + uint32_t(u)*32u;
                const uint32_t idelay = i < todo ? moddel[i] : 0u;
                const uint32_t delay = tap + i - (idelay>>8), doff = idelay & 255u;
                #pragma unroll
                for(int k = 0;k < 4;++k) o[u][k] = i < todo ? input[(delay - uint32_t(k)) & m] : 0.0f;
                cb[u][0] = Q.cubic[256u+doff]; cb[u][1] = Q.cubic[doff];
                cb[u][2] = Q.cubic[256u-doff]; cb[u][3] = Q.cubic[512u-doff];
            }
            #pragma unroll
            for(int u = 0;u < 8;++u)
            {
                const uint32_t i = lane + uint32_t(u)*32u;
                const float out = o[u][0]*cb[u][0] + o[u][1]*cb[u][1] + o[u][2]*cb[u][2] + o[u][3]*cb[u][3];
                if(i < todo) temp[line][i] = out*midGain;
            }
        }
        __syncwarp();
        if(lane == 0)
            dual_biquad_serial(R.t60_hf[line], R.t60_lf[line], R.z_t60hf[line], R.z_t60lf[line],
                temp[line], todo);
        __syncwarp();
        {
            const float *input = R.late_in + size_t(line)*R.late_in_len;
            const uint32_t m = R.late_in_len-1;
            const uint32_t t0 = offset - ltapCur, t1 = offset - R.late_tap[line];
            ltapCur = R.late_tap[line];
            const float fadeStep = 1.0f/float(todo);
            const float dg = R.density_gain;
            const float ds = (t0 != t1) ? dg*fadeStep : 0.0f;
            float v0[8], v1[8];
            #pragma unroll
            for(int u = 0;u < 8;++u)
            {
                const uint32_t i = lane + uint32_t(u)*32u;
                v0[u] = i < todo ? __ldcg(input + ((t0+i) & m)) : 0.0f;      // written by the early half on another SM
                v1[u] = i < todo ? __ldcg(input + ((t1+i) & m)) : 0.0f;
            }
            #pragma unroll
            for(int u = 0;u < 8;++u)
            {
                const uint32_t i = lane + uint32_t(u)*32u;
                const float fc = float(i);
                const float fade0 = dg - ds*fc, fade1 = ds*fc;
                if(i < todo) temp[line][i] = v0[u]*fade0 + v1[u]*fade1 + temp[line][i];
            }
        }
        __syncthreads();
        // VecAllpass::process (reverb.cpp:1452-1503), interleaved delay: frame*4 + line
        {
            float *buf = R.late_ap;
            const uint32_t m = R.late_ap_len-1, minOff = R.late_ap_offset[0];
            const uint32_t myOff = R.late_ap_offset[line];
            const float fc = R.late_ap_coeff;
            for(uint32_t sb = 0;sb < todo;sb += minOff)
            {
                const uint32_t td = (todo - sb < minOff) ? todo - sb : minOff;
                float dv[8];
                #pragma unroll
                for(int u = 0;u < 8;++u)
                {
                    const uint32_t i = lane + uint32_t(u)*32u;
                    dv[u] = i < td ? buf[size_t((offset + sb + i - myOff) & m)*NL + line] : 0.0f;
                }
                #pragma unroll
                for(int u = 0;u < 8;++u)
                {
                    const uint32_t i = lane + uint32_t(u)*32u;
                    if(i < td)
                    {
                        const float input = temp[line][sb+i];
                        const float out = dv[u] - fc*input;
                        buf[size_t((offset + sb + i) & m)*NL + line] = input + fc*out;
                        temp[line][sb+i] = out;
                    }
                }
                __syncthreads();
                {
                    float4 dq[2];
                    #pragma unroll
                    for(int u = 0;u < 2;++u)
                    {
                        const uint32_t i = tid + uint32_t(u)*128u;
                        dq[u] = i < td ? *reinterpret_cast<const float4*>(buf + size_t((offset + sb + i) & m)*NL)
                            : make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                    #pragma unroll
                    for(int u = 0;u < 2;++u)
                    {
                        const uint32_t i = tid + uint32_t(u)*128u;
                        if(i < td)
                        {
                            const float in[4] = {dq[u].x, dq[u].y, dq[u].z, dq[u].w};
                            float f[4];
                            scatter4(in, R.mix_x, R.mix_y, f);
                            *reinterpret_cast<float4*>(buf + size_t((offset + sb + i) & m)*NL)
                                = make_float4(f[0], f[1], f[2], f[3]);
                        }
                    }
                }
                __syncthreads();
            }
        }
        for(uint32_t i = lane;i < todo;i += 32) lateOut[size_t(line)*kLine + base + i] = temp[line][i];
        __syncthreads();
        // VectorScatterRev + feedback write (reverb.cpp:1800-1806)
        for(uint32_t i = tid;i < todo;i += 128)
        {
            const float in[4] = {temp[3][i], temp[2][i], temp[1][i], temp[0][i]};
            float f[4];
            scatter4(in, R.mix_x, R.mix_y, f);
            const uint32_t o = (offset+i) & (R.late_len-1);
            #pragma unroll
            for(int j = 0;j < NL;++j) R.late_d[size_t(j)*R.late_len + o] = f[j];
        }
        __syncthreads();
        base += todo; offset += todo;
    }

    if(lane == 0)
    {
        R.late_tap_cur[line] = ltapCur;
        if(line == 0) R.mod_index = modIdx;
    }
}

// After both halves of every pipeline: the write offset moves on (ReverbState::mOffset, reverb.cpp:1880).
__global__ void k_reverb_commit(const ReverbParamsK Q)
{
    const SlotRec &S = Q.slots[blockIdx.x];
    if(S.type != 2u || S.stage != Q.stage || !((S.rv_mask >> threadIdx.x) & 1u)) return;
    reinterpret_cast<ReverbDev*>(S.H)[threadIdx.x].offset += Q.frames;
}

// MixOutAmbiUp's front half (reverb.cpp:618-634,658-699) for higher-order devices: turns a
// pipeline's 4 early + 4 late A-format lines IN PLACE into 4 + 4 B-format rows
// (EarlyA2B / LateA2B, DoMixRow) and scales each row's HF band with its BandSplitter
// (in-place processHfScale, core/filters/splitter.cpp:99-131); k_slot_output_mix then pans the
// rows with the 8 gain rows as usual.  grid (slot, pipeline object), 8 warps = the 8 rows; the
// splitter recurrence runs on lane 0 of each warp from shared memory.
__global__ void __launch_bounds__(256) k_reverb_upmix(const ReverbParamsK Q)
{
    extern __shared__ float rows[];                 // [8][1024]
    const SlotRec &S = Q.slots[blockIdx.x];
    if(S.type != 2u || S.stage != Q.stage || !((S.rv_mask >> blockIdx.y) & 1u)) return;
    ReverbDev &R = reinterpret_cast<ReverbDev*>(S.H)[blockIdx.y];
    if(!R.upmix) return;
    const float inv_sqrt2 = 0.707106781186547524400844362104849039f;
    const float A2B[2][4][4] = {
        {{0.5f, 0.5f, 0.5f, 0.5f}, {0.5f, -0.5f, 0.5f, -0.5f}, {0.5f, -0.5f, -0.5f, 0.5f}, {0.5f, 0.5f, -0.5f, -0.5f}},
        {{0.5f, 0.5f, 0.5f, 0.5f}, {inv_sqrt2, -inv_sqrt2, 0.0f, 0.0f}, {0.0f, 0.0f, -inv_sqrt2, inv_sqrt2},
         {0.5f, 0.5f, -0.5f, -0.5f}}};
    const uint32_t n = Q.frames;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int which = warp >> 2, row = warp & 3;
    float *lines = S.lines + (size_t(blockIdx.y)*8 + size_t(which)*4)*kLine;     // this group's 4 A lines
    float *mine = rows + size_t(warp)*kLine;
    for(uint32_t i = lane;i < n;i += 32)
    {
        float acc = 0.0f;
        #pragma unroll
        for(int k = 0;k < 4;++k)
        {
            const float g = A2B[which][row][k];
            if(fabsf(g) > kSilence) acc = acc + lines[size_t(k)*kLine + i]*g;
        }
        mine[i] = acc;
    }
    __syncthreads();                                 // every row has read the A-format lines
    if(lane == 0)
    {
        const float hfscale = R.order_scale[row ? 1 : 0];
        const float ap_coeff = R.split_coeff, lp_coeff = R.split_coeff*0.5f + 0.5f;
        float lp_z1 = R.z_split[which][row][0], lp_z2 = R.z_split[which][row][1];
        float ap_z1 = R.z_split[which][row][2];
        for(uint32_t i0 = 0;i0 < n;i0 += 8)
        {
            float x[8], y[8];
            #pragma unroll
            for(int k = 0;k < 8;++k) x[k] = (i0 + k < n) ? mine[i0+k] : 0.0f;
            #pragma unroll
            for(int k = 0;k < 8;++k)
            {
                const float in0 = x[k];
                const float d0 = (in0 - lp_z1) * lp_coeff;
                const float lp_y0 = lp_z1 + d0;
                const float n1 = lp_y0 + d0;
                const float d1 = (lp_y0 - lp_z2) * lp_coeff;
                const float lp_y1 = lp_z2 + d1;
                const float n2 = lp_y1 + d1;
                const float ap_y = in0*ap_coeff + ap_z1;
                const float n3 = in0 - ap_y*ap_coeff;
                y[k] = (ap_y-lp_y1)*hfscale + lp_y1;
                if(i0 + k < n) { lp_z1 = n1; lp_z2 = n2; ap_z1 = n3; }
            }
            #pragma unroll
            for(int k = 0;k < 8;++k) if(i0 + k < n) mine[i0+k] = y[k];
        }
        R.z_split[which][row][0] = lp_z1; R.z_split[which][row][1] = lp_z2; R.z_split[which][row][2] = ap_z1;
    }
    __syncwarp();
    for(uint32_t i = lane;i < n;i += 32) lines[size_t(row)*kLine + i] = mine[i];
}

} // namespace b200mix
