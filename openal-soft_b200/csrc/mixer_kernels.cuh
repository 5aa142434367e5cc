// mixer_kernels.cuh — sm_90a kernels of the b200mix hot path (device code only).
//
// Work decomposition (DESIGN.md §3): the voice loop of ProcessContexts
// (alc/alu.cpp:2201-2206) becomes persistent launches in which a CTA holds GROUPS voice
// groups of GS threads:
//   1. k_mix_voices: per voice, rebuilds the reference's resample window chunk by chunk in
//      shared memory (LoadResampledSamples, core/voice.cpp:642-822), decoding the source
//      straight from HBM, and resamples it with a per-voice pre-combined phase table.  The
//      resampled line is parked in HBM (xscratch) or, on devices with at most 4 dry
//      channels, mixed into register accumulators of the dry bus; on those devices
//      k_mix_deferred mixes the lines of voices with an active direct filter once filtered,
//   2. k_hrtf_fir (HRTF devices): per parked HRTF voice, bulk-copied into shared memory one
//      voice ahead, builds the per-ear, gain-ramped FIR
//      inputs (DoHrtfMix, core/voice.cpp:827-902; MixHrtfBlend/MixHrtf, hrtfbase.h:17-89)
//      and runs the HRIR FIR with the outputs held in registers ACROSS all voices of the
//      group (the cross-voice reduction of `Accum[i+j] += ...` happens in registers),
// and the accumulating kernels store one partial row per CTA; k_reduce_* (for the HRIR FIR's
// rows: k_post_hrtf_reduce, with the HRTF post-mix) sums the rows in a fixed order
// (deterministic output).
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

#include "voice_structs.hpp"
#include "async_ptx.cuh"

namespace b200mix {

constexpr int kLine = 1024;          // BufferLineSize
constexpr int kHrirLen = 128;        // HrirLength
constexpr int kHist = 64;            // HrtfHistoryLength
constexpr int kEdge = 24;            // MaxResamplerEdge
constexpr int kPad = 48;             // MaxResamplerPadding
constexpr int kResBuf = kLine + 256 + kPad;   // DeviceBase::mResampleData (core/device.h:282)
constexpr int kSrcSizeMax = kResBuf - kEdge;
constexpr int kAccumLen = kLine + kHrirLen;   // HrtfAccumData (core/device.h:288)
constexpr float kSilence = 0.00001f;          // GainSilenceThreshold
constexpr float kEps = 1.1920929e-07f;

// internal voice flag bits (low 8 bits are the ABI's B200MIX_VF_*)
constexpr uint32_t kVfStatic = 1u<<2, kVfLooping = 1u<<3, kVfHrtf = 1u<<4;
constexpr uint32_t kVfFading = 1u<<8, kVfHaveBuffer = 1u<<9, kVfCoefDirty = 1u<<10;
// VoiceUpdate::flags only: mCurrentBuffer is null (B200MIX_NO_BUFFER)
constexpr uint32_t kUpNoBuffer = 1u<<11;
constexpr uint32_t kVfChannelMask = 0xffu<<16;       // B200MIX_VF_CHANNEL: buffer channel read

struct alignas(16) BufferRec {
    const void *data;
    uint32_t frames, type, channels, pad;
};

// Device-resident mirror of the mixing state of one Voice (core/voice.h:157-272).
struct alignas(16) VoiceRec {
    uint32_t state;            // 0 stopped, 1 playing, 2 stopping
    uint32_t flags;
    uint32_t buffer, resampler;
    int32_t  pos; uint32_t frac, step, loop_start;
    uint32_t loop_end; float bsinc_sf; uint32_t bsinc_m, bsinc_l;
    uint32_t bsinc_off, tgt_delay0, tgt_delay1; float tgt_gain;
    uint32_t old_delay0, old_delay1; float old_gain; uint32_t send_mask;
    uint32_t send_slot[kMaxSends]; uint32_t pad2[2];
    float prev[kPad];          // mPrevSamples[0]
    float hist[kHist];         // Hrtf.History
};

struct VoiceResult { int32_t position; uint32_t position_frac, flags, buffers_done; };

// Device-resident BiquadInterpFilter pair of one voice path (core/voice.h:50-53,70-73;
// core/filters/biquad.h:137-198): [0] = LowPass (high-shelf), [1] = HighPass (low-shelf).
// Coefficient sets are {b0,b1,b2,a1,a2}.
struct alignas(16) FilterRec {
    float cur[2][5]; float tgt[2][5];
    float z[2][2];
    int32_t counter[2];
    uint32_t active;
    uint32_t pad[5];
};
static_assert(sizeof(FilterRec) == 128, "FilterRec layout");

struct MixParams {
    VoiceRec *voices; const BufferRec *buffers;
    float2 *hrtf_tgt; float2 *hrtf_old;       // [max_voices][ir_pad]
    float *dry_cur; float *dry_tgt;           // [max_voices][cd]
    float *partial;                           // see k_reduce_*
    VoiceResult *results;
    const float *bsinc_tab[3];                // bsinc12, 24, 48
    const float *cubic_tab[2];                // spline, gaussian [32][8]
    uint32_t max_voices, frames, ir_pad, cd, num_sends;
    float *xscratch;                          // [max_voices][1024] parked resampled lines
    uint32_t *sendinfo;                       // per voice: kSi* bits, bits8.. fade counter
    const uint32_t *order;                    // mixing order: voice indices, cost-sorted
    uint32_t num_order;
    FilterRec *filt;                          // [max_voices][filt_paths] or null (no filter ever set)
    uint32_t filt_paths;                      // 1 + num_sends
    // Voices whose direct-path filter is active are resampled and parked by k_mix_voices,
    // filtered by k_filters and mixed from here by k_mix_deferred or k_hrtf_fir.
    const float *dline;                       // [max_voices][1024] filtered direct-path lines
    // streaming queues (null until the first b200mix_voice_queue): per voice
    // {count, head, loop, -} and kMaxQueue buffer ids
    uint4 *qhdr; const uint32_t *queue;
    uint32_t *claim;                         // {next order index, groups done}: zero between launches
    // callback buffers (b200mix_buffer_callback): a BufferRec whose pad is 1 + s is read as
    // cbplan[s] this update (null while no callback voice mixes; the record itself then reads
    // as an empty buffer over zeros).  That record, planned on the
    // host (callback_plan.hpp, Span), is the samples the buffer's callbacks delivered as a
    // static buffer of `frames` frames that the voice's position addresses directly:
    // LoadBufferCallback (core/voice.cpp:546-561) is then LoadBufferStatic without a loop, and
    // the voice ends, as a static one, once its position reaches `frames` (core/voice.cpp:1158-1176).
    const BufferRec *cbplan;
};

constexpr uint32_t kMaxQueue = 32, kNoLoop = 0xffffffffu;

// sendinfo bits: the line is parked for the aux sends (kSiSend), the parked dry bus (kSiDry),
// k_hrtf_fir (kSiHrtf) or the RealOut bus (kSiReal: a direct-channel voice); kSiDeferred: its
// direct filter is active, the mix reads dline
constexpr uint32_t kSiSend = 1u, kSiPlaying = 2u, kSiDeferred = 4u, kSiDirty = 8u, kSiDry = 16u,
    kSiHrtf = 32u, kSiReal = 64u;

// Named barrier of voice group id (1 or 2).  The ids are immediates: with a register id ptxas
// reserves all 16 hardware barriers for the CTA, which caps the SM at 4 such CTAs.
__device__ __forceinline__ void group_sync(int id, int count)
{
    if(id == 1) asm volatile("bar.sync 1, %0;" :: "r"(count) : "memory");
    else asm volatile("bar.sync 2, %0;" :: "r"(count) : "memory");
}

// group_sync that also returns whether pred holds on every thread of the group (bar.red.and)
__device__ __forceinline__ bool group_sync_and(int id, int count, bool pred)
{
    uint32_t all;
    if(id == 1)
        asm volatile("{ .reg .pred p, q; setp.ne.u32 p, %1, 0; bar.red.and.pred q, 1, %2, p; selp.u32 %0, 1, 0, q; }"
            : "=r"(all) : "r"(uint32_t(pred)), "r"(count) : "memory");
    else
        asm volatile("{ .reg .pred p, q; setp.ne.u32 p, %1, 0; bar.red.and.pred q, 2, %2, p; selp.u32 %0, 1, 0, q; }"
            : "=r"(all) : "r"(uint32_t(pred)), "r"(count) : "memory");
    return all != 0u;
}

// Whether v survives the 16-bit window unchanged: v = s/32768 for an integer s in [-32768, 32767].
__device__ __forceinline__ bool exact16(float v)
{
    const float s = v*32768.0f;
    return s == rintf(s) && s >= -32768.0f && s <= 32767.0f;
}

__device__ __forceinline__ void prefetch_l2(const void *p)
{ asm volatile("prefetch.global.L2 [%0];" :: "l"(p)); }

__device__ __forceinline__ uint32_t sample_bytes(uint32_t type)
{ return type == 1u ? 2u : ((type == 0u || type >= 5u) ? 1u : (type == 4u ? 8u : 4u)); }

// Pulls the lines a voice will read next update into L2: its record + HRIR two voices
// ahead (plain address arithmetic), and one voice ahead the source span its resampler
// will consume (needs that voice's header, already prefetched the round before).
__device__ __forceinline__ void prefetch_span(const char *base, size_t bytes, size_t off,
    size_t len, int t, int gs)
{
    if(off >= bytes) return;
    if(off + len > bytes) len = bytes - off;
    const size_t first = off & ~size_t(127);
    for(size_t a = first + size_t(t)*128u;a < off + len;a += size_t(gs)*128u)
        prefetch_l2(base + a);
}

__device__ __forceinline__ float load_sample(const BufferRec &b, size_t idx)
{
    // SampleInfo<T>::to_float, core/fmt_traits.h:88-131
    switch(b.type)
    {
    case 0: return (float(static_cast<const uint8_t*>(b.data)[idx]) - 128.0f) * (1.0f/128.0f);
    case 1: return float(static_cast<const int16_t*>(b.data)[idx]) * (1.0f/32768.0f);
    case 2: return float(static_cast<const int32_t*>(b.data)[idx]) * (1.0f/2147483648.0f);
    case 3: return static_cast<const float*>(b.data)[idx];
    case 4: return float(static_cast<const double*>(b.data)[idx]);
    }
    return 0.0f;
}

// CalculateBufferSize, core/voice.cpp:601-640
__device__ __forceinline__ void calc_buffer_size(uint32_t fracPos, uint32_t increment,
    uint32_t dstRemaining, uint32_t &dst, uint32_t &src)
{
    const uint32_t ext = increment <= 65536u;
    const uint64_t srcSize64 = ((uint64_t(dstRemaining - ext)*increment + fracPos) >> 16)
        + ext + kEdge;
    if(srcSize64 <= uint64_t(kSrcSizeMax)) { dst = dstRemaining; src = uint32_t(srcSize64); return; }
    const uint64_t dstSize64 = ((uint64_t(kSrcSizeMax - kEdge)<<16) - fracPos) / increment;
    if(dstSize64 < dstRemaining) { dst = uint32_t(dstSize64) & ~3u; src = kSrcSizeMax; return; }
    dst = dstRemaining; src = kSrcSizeMax;
}

__device__ __forceinline__ int32_t add_sat(int32_t a, int32_t b)
{
    long long r = (long long)a + b;
    r = r > 2147483647ll ? 2147483647ll : (r < -2147483648ll ? -2147483648ll : r);
    return int32_t(r);
}

// SampleInfo<T>::to_float, core/fmt_traits.h:88-131
__device__ __forceinline__ float to_float(uint8_t v) { return (float(v) - 128.0f) * (1.0f/128.0f); }
__device__ __forceinline__ float to_float(int16_t v) { return float(v) * (1.0f/32768.0f); }
__device__ __forceinline__ float to_float(int32_t v) { return float(v) * (1.0f/2147483648.0f); }
__device__ __forceinline__ float to_float(float v) { return v; }
__device__ __forceinline__ float to_float(double v) { return float(v); }
// ITU-T G.711 expansion == muLaw/aLawDecompressionTable (core/fmt_traits.h:12-81)
struct MulawByte { uint8_t v; };
struct AlawByte { uint8_t v; };
__device__ __forceinline__ float to_float(MulawByte b)
{
    const uint32_t u = (~uint32_t(b.v)) & 0xffu;
    const int s = int((((u & 0x0fu)<<3) + 0x84u) << ((u>>4)&7u)) - 0x84;
    return float((u & 0x80u) ? -s : s) * (1.0f/32768.0f);
}
__device__ __forceinline__ float to_float(AlawByte b)
{
    const uint32_t a = uint32_t(b.v) ^ 0x55u;
    const uint32_t e = (a>>4)&7u, m = a & 0x0fu;
    const int s = (e == 0u) ? int((m<<4) + 8u) : int(((m<<4) + 0x108u) << (e-1u));
    return float((a & 0x80u) ? s : -s) * (1.0f/32768.0f);
}

template<typename T> __device__ __forceinline__ T ld_raw(const T *p) { return __ldg(p); }
template<> __device__ __forceinline__ MulawByte ld_raw(const MulawByte *p)
{ return MulawByte{__ldg(reinterpret_cast<const uint8_t*>(p))}; }
template<> __device__ __forceinline__ AlawByte ld_raw(const AlawByte *p)
{ return AlawByte{__ldg(reinterpret_cast<const uint8_t*>(p))}; }

// word offset of the second 16-bit window copy: 16 (mod 32) banks away from the first, so lanes
// on an even and on an odd window position never meet in a bank while the warp's span stays
// within 32 samples
constexpr int kPackB = 688;
static_assert(kPackB >= (kResBuf + 8 + 1)/2 && kPackB + (kResBuf + 8 + 1)/2 <= kResBuf + 8 + 24
    && (kPackB % 32) == 16, "16-bit window copies must fit the float window's storage");

// sample k of the resample window, whichever representation it is in
__device__ __forceinline__ float win_at(const float *win, bool packed, uint32_t k)
{
    if(!packed) return win[k];
    const uint16_t y = reinterpret_cast<const uint16_t*>(win)[k];
    return float(int(y) - 32768) * (1.0f/32768.0f);
}

struct FillArgs {
    float *dst; uint32_t count, uintPos, q0, firstRun, loopStart, loopSize, lastFrame, channels;
    bool looping, pastEnd, simpleWrap;
};

// DoFilters with an inactive pair: lpfilter.clear(); hpfilter.clear() (biquad.h:152-157).
__device__ __forceinline__ void filter_clear(FilterRec &fr, int t)
{
    if(t < 10) fr.cur[t/5][t%5] = fr.tgt[t/5][t%5];
    else if(t < 14) fr.z[(t-10)>>1][(t-10)&1] = 0.0f;
    else if(t < 16) fr.counter[t-14] = 0;
}

// LoadBufferStatic (core/voice.cpp:500-544) for one window run: element k maps to buffer
// frame q(k) (loop wrap / end hold); 8 independent loads are issued before any use.
template<typename T, int GS>
__device__ __forceinline__ void fill_window(const FillArgs &A, const T *__restrict__ src, int t)
{
    for(uint32_t k0 = t;k0 < A.count;k0 += 8u*GS)
    {
        T raw[8];
        #pragma unroll
        for(int u = 0;u < 8;++u)
        {
            uint32_t k = k0 + uint32_t(u)*GS;
            k = k < A.count ? k : A.count-1u;
            uint32_t q;
            if(!A.looping) q = min(A.uintPos + k, A.lastFrame);
            else if(k < A.firstRun) q = A.q0 + k;
            else if(A.simpleWrap) q = A.loopStart + (k - A.firstRun);
            else q = A.loopStart + (k - A.firstRun)%A.loopSize;
            raw[u] = ld_raw(src + size_t(q)*A.channels);
        }
        #pragma unroll
        for(int u = 0;u < 8;++u)
        {
            const uint32_t k = k0 + uint32_t(u)*GS;
            if(k < A.count) A.dst[k] = A.pastEnd ? 0.0f : to_float(raw[u]);
        }
    }
}

// Shared-memory carve-up of one voice group of k_mix_voices.  Only the register-dry variant
// (CDR > 0) stages the resampled line here; the parking variant writes it to xscratch.
constexpr int kWinFloats = kResBuf + 8 + 24;
template<int CDR>
struct alignas(16) GroupSmem {
    static constexpr int kTabStride = kPad + 2;         // max row stride; rows use m+2 (even, half odd:
                                                        // 8-byte aligned AND conflict-free for LDS.64)
    float win[kWinFloats];
    alignas(8) float tabF[32*kTabStride];
    alignas(8) float tabD[32*kTabStride];
    float x[CDR > 0 ? kLine : 1];
    float newGain[32];                  // dry Current gains written back after the voice
    uint64_t tmaBar;                    // mbarrier of the group's source-span bulk copies
    uint32_t claimed;                   // order index the group claimed last (parking variant)
};

// What k_hrtf_fir bulk-copies for one voice: [History | resampled line] and the target HRIR,
// plus the old HRIR when the voice is dirty.
struct alignas(16) FirStage {
    float x[kHist + kLine];
    float2 coefT[kHrirLen], coefO[kHrirLen];
};
static_assert(offsetof(VoiceRec, hist) % 16 == 0 && sizeof(VoiceRec) % 16 == 0,
    "VoiceRec::hist is a bulk-copy source: 16-byte aligned");

// Shared-memory carve-up of one voice group of k_hrtf_fir.  The stage buffers alternate
// between voices: one is filled for the group's next voice while the other is read.
template<int GS, int OPT, int FP>
struct alignas(16) FirSmem {
    static constexpr int kLLen = FP + OPT*GS;           // FIR input incl. front zero pad
    static constexpr int kOLen = FP + kHist + FP + 32;  // old-coefficient pass input
    float2 lLR[kLLen];                  // {left, right} per input sample
    float2 oLR[kOLen];
    FirStage st[2];
    uint64_t bar[2];                    // mbarrier of each stage buffer's bulk copies
};

// Both ears' MACs: {a.x*b.x + c.x, a.y*b.y + c.y}, each one fused multiply-add (round to
// nearest); left and right travel together as a float2.
__device__ __forceinline__ float2 fma2_rn(float2 a, float2 b, float2 c)
{ return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }

// One FIR pass for BOTH ears: acc[r].{x,y} += sum_j c[j].{x,y} * in[FP + t0 + r - j].{x,y}
// (gather form of MixHrtfBase's scatter, hrtfbase.h:28-40).  Taps go in blocks of JB with a
// register window w[k] = in[FP + t0 - jb - (JB-1) + k].  The next block's window is this one
// moved down by JB entries, so it keeps the OPT-1 entries the two share and loads only JB new
// ones.  Blocks go in pairs, unrolled so that the window slides by register renaming (no moves):
// OPT+7 + 8 input loads per 16 taps instead of 2*(OPT+7).  Unrolling every block of the 64-tap
// variant made its code three times larger and the pass slower.
template<int OPT, int FP>
__device__ __forceinline__ void fir_pass(float2 (&acc)[OPT], const float2 *__restrict__ in,
    const float2 *__restrict__ coef, int irpad, int t0)
{
    constexpr int JB = 8;                       // taps per register-window block
    constexpr int W = OPT + JB - 1;
    for(int jb = 0;jb < irpad;jb += 2*JB)
    {
        const float2 *p = in + FP + t0 - jb - (JB-1);
        float2 w[W];
        #pragma unroll
        for(int k = 0;k < W;++k) w[k] = p[k];
        #pragma unroll
        for(int jj = 0;jj < JB;++jj)
        {
            const float2 c = coef[jb+jj];
            #pragma unroll
            for(int r = 0;r < OPT;++r)
                acc[r] = fma2_rn(c, w[r - jj + (JB-1)], acc[r]);
        }
        if(jb + JB >= irpad) break;
        #pragma unroll
        for(int k = W-1;k >= JB;--k) w[k] = w[k-JB];
        #pragma unroll
        for(int k = 0;k < JB;++k) w[k] = p[k - JB];
        #pragma unroll
        for(int jj = 0;jj < JB;++jj)
        {
            const float2 c = coef[jb+JB+jj];
            #pragma unroll
            for(int r = 0;r < OPT;++r)
                acc[r] = fma2_rn(c, w[r - jj + (JB-1)], acc[r]);
        }
    }
}

// Next voice of a parking group: groups claim order indices from a counter one at a time, so
// the cost-sorted order is spread over the groups as they free up (no static rounds).  The
// last group to run dry resets the counter pair for the next launch.
__device__ __forceinline__ uint32_t claim_voice(const MixParams &P, uint32_t &slot, int t, int bar,
    int gs, uint32_t groups)
{
    group_sync(bar, gs);                          // every thread has read the previous claim
    if(t == 0)
    {
        uint32_t oi = atomicAdd(P.claim, 1u);
        if(oi >= P.num_order && atomicAdd(P.claim + 1, 1u) == groups - 1u)
        {
            atomicExch(P.claim, 0u);
            atomicExch(P.claim + 1, 0u);
        }
        slot = oi;
    }
    group_sync(bar, gs);
    return slot;
}

// ---------------------------------------------------------------------------
// Stages of the voice loop.  Each runs on one voice group (GS threads; thread t, named
// barrier bar) and takes what it reads and writes as arguments.
// ---------------------------------------------------------------------------

// A voice that resamples nothing this update: not playing, or a zero step (a stopping voice
// then stops).  Reports its result and clears its sendinfo; returns true when it is done.
__device__ __forceinline__ bool voice_early_out(const MixParams &P, VoiceRec &rec, uint32_t v,
    uint32_t vstate, uint4 h1, int t)
{
    if(vstate != 1u && vstate != 2u)
    {
        if(t == 0)
        {
            if(P.results) P.results[v] = VoiceResult{int32_t(h1.x), h1.y, 1u<<7, 0u};
            if(P.sendinfo) P.sendinfo[v] = 0u;
        }
        return true;
    }
    if(h1.z < 1u)
    {
        if(t == 0)
        {
            if(vstate == 2u) rec.state = 0u;
            if(P.sendinfo) P.sendinfo[v] = 0u;
            if(P.results)
                P.results[v] = VoiceResult{int32_t(h1.x), h1.y, (vstate == 2u) ? (1u<<7) : 1u, 0u};
        }
        return true;
    }
    return false;
}

// Pre-combined phase table: coef(phase,pf)[j] = F[phase][j] + pf*D[phase][j]
//   BSinc      F = fil + sf*scd, D = phd + sf*spd   (mixer_c.cpp:84-105)
//   FastBSinc  F = fil,          D = phd            (mixer_c.cpp:63-82)
//   cubic      F = mCoeffs,      D = mDeltas        (mixer_c.cpp:48-61)
// Sets the tap count m, the left offset tapOff into the window and the row stride ms.
template<int GS>
__device__ __forceinline__ void build_phase_table(const MixParams &P, float *tabF, float *tabD,
    uint32_t resampler, uint32_t increment, uint4 h2, uint4 h3, int t,
    uint32_t &m, uint32_t &tapOff, uint32_t &ms)
{
    m = 0; tapOff = 0; ms = 5;
    if(resampler >= 4u)
    {
        m = h2.z;
        tapOff = kEdge - h2.w;
        const float *tab = P.bsinc_tab[(resampler-4u)>>1] + h3.x;
        const bool full = (increment > 65536u) && (resampler & 1u);
        const float sf = __uint_as_float(h2.y);
        // The sub-table of one scale is [32 phases][fil m | phd m] followed by
        // [32 phases][scd m | spd m].  A thread owns one column of the 2m-wide rows and
        // walks the 32 phases (coalesced across threads, 8 loads in flight).
        const uint32_t rowLen = 2u*m;
        const float *tab2 = tab + 64u*m;
        ms = m + 1u;
        for(uint32_t c = t;c < rowLen;c += GS)
        {
            float *dstc = (c < m) ? (tabF + c) : (tabD + (c - m));
            #pragma unroll 1
            for(uint32_t p0 = 0;p0 < 32u;p0 += 8u)
            {
                float a[8], b[8];
                #pragma unroll
                for(int u = 0;u < 8;++u)
                {
                    a[u] = __ldg(tab + (p0+u)*rowLen + c);
                    b[u] = full ? __ldg(tab2 + (p0+u)*rowLen + c) : 0.0f;
                }
                #pragma unroll
                for(int u = 0;u < 8;++u)
                    dstc[(p0+u)*ms] = full ? fmaf(sf, b[u], a[u]) : a[u];
            }
        }
    }
    else if(resampler >= 2u)
    {
        m = 4; tapOff = kEdge - 1; ms = 5;
        const float *tab = P.cubic_tab[resampler-2u];
        for(uint32_t e = t;e < 128u;e += GS)
        {
            const uint32_t pi = e>>2, j = e&3u;
            tabF[pi*ms + j] = tab[pi*8u + j];
            tabD[pi*ms + j] = tab[pi*8u + 4u + j];
        }
    }
}

// Software prefetch for the voices this group resamples next (overlaps the current voice).
template<int GS>
__device__ __forceinline__ void prefetch_next_voices(const MixParams &P, uint32_t oi, uint32_t groups,
    int t)
{
    const uint32_t o2 = oi + 2u*groups, o1 = oi + groups;
    const uint32_t v2 = o2 < P.num_order ? P.order[o2] : 0xffffffffu;
    const uint32_t v1 = o1 < P.num_order ? P.order[o1] : 0xffffffffu;
    if(v2 < P.max_voices && t < 5)
        prefetch_l2(reinterpret_cast<const char*>(&P.voices[v2]) + t*128);
    if(v1 < P.max_voices)
    {
        const VoiceRec &nx = P.voices[v1];
        if((nx.state == 1u || nx.state == 2u) && (nx.flags & kVfHaveBuffer) && nx.step >= 1u)
        {
            const BufferRec nb = P.buffers[nx.buffer];
            const size_t fb = size_t(sample_bytes(nb.type))*nb.channels;
            const size_t bytes = size_t(nb.frames)*fb;
            const uint32_t p0 = nx.pos < 0 ? 0u : uint32_t(nx.pos);
            const size_t need = size_t((uint64_t(P.frames)*nx.step + nx.frac) >> 16) + kPad;
            const char *base = static_cast<const char*>(nb.data);
            prefetch_span(base, bytes, size_t(p0)*fb, need*fb, t, GS);
            if((nx.flags & kVfLooping) && p0 + need > nx.loop_end && nx.loop_end > p0)
                prefetch_span(base, bytes, size_t(nx.loop_start)*fb,
                    (p0 + need - nx.loop_end)*fb, t, GS);
        }
    }
}

// Voice ended: hold the sample closest to 0 (core/voice.cpp:704-719).
template<int GS>
__device__ __forceinline__ void hold_end_sample(float *srcBuffer, uint32_t srcn, int t, int bar)
{
    const uint32_t avail = srcn < uint32_t(kEdge) ? srcn : uint32_t(kEdge);
    const uint32_t tofill = srcn > uint32_t(kEdge) ? srcn : uint32_t(kEdge);
    uint32_t best = 0;
    for(uint32_t i = 1;i < avail;++i)
        if(fabsf(srcBuffer[i]) < fabsf(srcBuffer[best])) best = i;
    const float held = srcBuffer[best];
    group_sync(bar, GS);
    for(uint32_t k = best+1+t;k < tofill;k += GS) srcBuffer[k] = held;
}

// The 16-bit window copies of pack_window16, built straight from a one-run int16 span that the
// bulk copy left at raw (sample 0 at halfword lead).  Span sample s becomes y = s + 32768, which
// is the raw halfword XOR 0x8000, so an A word is the funnel of two neighbouring raw words,
// XOR 0x80008000 (window position k sits at raw halfword k - kEdge - srcDelay + lead; the funnel
// covers its parity).  Positions before the span, the history from prev (floats) and the
// srcDelay zeros, are converted as pack_window16 converts them.  Only the A words are held
// across the one barrier (the B copy overlaps the raw span): B word w = y(2w+1) | y(2w+2) << 16
// is the funnel of A words w and w+1.  Each warp takes a run of 32*PER consecutive words, so a
// lane gets word w+1 (and raw word w+1) from the next lane, lane 31 from lane 0 one step later.
// Consecutive runs share one word: the earlier warp writes its A, the later one its B.  The
// result equals what pack_window16 writes for the same window; positions past the span are
// never read.
template<int GS>
__device__ __forceinline__ void pack_span16(float *win, const unsigned char *raw, uint32_t lead,
    uint32_t srcDelay, uint32_t count, int t, int bar)
{
    constexpr int NW = (kResBuf + 8 + 1)/2;                    // words of one copy
    constexpr int PER = (NW + GS - 1)/GS;                      // words per lane
    static_assert((GS/32)*(32*PER - 1) >= NW + 1, "the warps' runs must cover every word");
    const uint32_t lane = uint32_t(t) & 31u;
    const uint32_t w0 = uint32_t(t >> 5)*(32u*PER - 1u) + lane;  // the lane's word at u = 0
    const uint32_t lo = uint32_t(kEdge) + srcDelay;            // first position from the span
    const uint32_t nw = (min(lo + count + 8u, uint32_t(kResBuf + 8)) + 1u)/2u;
    // position 2w is raw halfword 2w - off: word w funnels raw words w - ceil(off/2) and the
    // next by off's parity.  Raw word w holds positions 2w-1..2w+1, so it is loaded only when
    // 2w+1 >= lo: words wholly before the span take their values from the masks below and read
    // nothing (the srcDelay zeros may be being stored there).  Words past the span read other
    // bytes of the group's storage (the phase table after the window), which the resampler's
    // reach makes irrelevant.
    const uint32_t off = lo - lead;
    const uint32_t *rw = reinterpret_cast<const uint32_t*>(raw) - int((off + 1u) >> 1);
    const uint32_t sh = (off & 1u)*16u;
    uint32_t wa[PER];
    #pragma unroll
    for(int u = 0;u < PER;++u)
    {
        const uint32_t w = w0 + uint32_t(u)*32u;
        wa[u] = (w <= nw && 2u*w + 1u >= lo) ? rw[w] : 0u;
    }
    #pragma unroll
    for(int u = 0;u < PER;++u)
    {
        const uint32_t w = w0 + uint32_t(u)*32u;
        uint32_t r1 = __shfl_sync(0xffffffffu, (u + 1 < PER && lane == 0u) ? wa[u + 1 < PER ? u + 1 : u] : wa[u],
            (lane + 1u) & 31u);
        if(u + 1 == PER && lane == 31u && w <= nw && 2u*w + 3u >= lo) r1 = rw[w + 1u];
        uint32_t a = __funnelshift_r(wa[u], r1, sh) ^ 0x80008000u;
        const int d = int(lo) - int(2u*w);                      // positions 2w, 2w+1 before lo: zeros
        const uint32_t m = (d >= 1 ? 0x0000ffffu : 0u) | (d >= 2 ? 0xffff0000u : 0u);
        a = (a & ~m) | (0x80008000u & m);
        if(u == 0 && w < uint32_t(kEdge/2))                     // history
            a = uint32_t(uint16_t(__float2int_rn(win[2u*w]*32768.0f) + 32768))
                | (uint32_t(uint16_t(__float2int_rn(win[2u*w + 1u]*32768.0f) + 32768)) << 16);
        wa[u] = a;
    }
    group_sync(bar, GS);                 // raw span and history read: the copies may overwrite them
    uint32_t *pa = reinterpret_cast<uint32_t*>(win);
    uint32_t *pb = pa + kPackB;
    #pragma unroll
    for(int u = 0;u < PER;++u)
    {
        const uint32_t w = w0 + uint32_t(u)*32u;
        const uint32_t next = __shfl_sync(0xffffffffu, (u + 1 < PER && lane == 0u) ? wa[u + 1 < PER ? u + 1 : u] : wa[u],
            (lane + 1u) & 31u);
        if(w < nw)
        {
            if(u > 0 || lane > 0u || t < 32) pa[w] = wa[u];
            if(u + 1 < PER || lane < 31u) pb[w] = __funnelshift_r(wa[u], next, 16u);
        }
    }
}

// TMA staging of the source span (the common case: a static mono int16 buffer, the span inside
// the buffer, at most one loop wrap).  The span is one or two CONTIGUOUS runs of the buffer: one
// thread issues a bulk copy (cp.async.bulk: global -> shared, completion on the group's
// mbarrier) per run into the unused tail of the window storage; the group then converts from
// shared memory.  Replaces ~1300 two-byte gathers per voice-chunk by one or two asynchronous
// copies; the lines were pulled into L2 a round earlier.  Writes count samples to
// win[kEdge+srcDelay..] and returns true, or returns false (nothing written) when the span does
// not qualify.  With pack set, a one-run span goes straight into the 16-bit window copies
// (pack_span16) and packed is set; otherwise the window is left as floats.
template<int GS>
__device__ __forceinline__ bool stage_span_tma(float *win, uint64_t *tmaBar, uint32_t &tmaPhase,
    const BufferRec &buf, uint32_t flags, bool isQueue, bool looping, uint32_t loopStart,
    uint32_t loopEnd, uint32_t uintPos, uint32_t srcDelay, uint32_t count, bool pack, bool &packed,
    int t, int bar)
{
    if(isQueue || buf.type != 1u || buf.channels != 1u || ((flags >> 16) & 0xffu) != 0u || count == 0u)
        return false;
    const uint32_t loopSize = looping ? (loopEnd - loopStart) : 1u;
    const uint32_t q0 = !looping ? uintPos : ((uintPos < loopEnd) ? uintPos
        : ((uintPos-loopStart)%loopSize + loopStart));
    const uint32_t run1 = looping ? min(count, loopEnd - q0) : count;
    const uint32_t run2 = count - run1;
    const bool fits = looping ? (run2 <= loopSize && loopEnd <= buf.frames)
                              : (uintPos + count <= buf.frames);
    if(!fits) return false;
    const int16_t *base = static_cast<const int16_t*>(buf.data);
    const uintptr_t a1 = reinterpret_cast<uintptr_t>(base + q0);
    const uintptr_t a2 = reinterpret_cast<uintptr_t>(base + loopStart);
    const uint32_t lead1 = uint32_t(a1 & 15u) >> 1, lead2 = uint32_t(a2 & 15u) >> 1;
    const uint32_t bytes1 = ((run1 + lead1)*2u + 15u) & ~15u;
    const uint32_t bytes2 = run2 ? (((run2 + lead2)*2u + 15u) & ~15u) : 0u;
    constexpr uint32_t kWinBytes = uint32_t(kWinFloats*sizeof(float));
    unsigned char *wbytes = reinterpret_cast<unsigned char*>(win);
    unsigned char *raw2 = wbytes + kWinBytes - bytes2;
    unsigned char *raw1 = raw2 - bytes1;
    if(t == 0)
    {
        fence_proxy_async_smem();
        mbar_expect_tx(tmaBar, bytes1 + bytes2);
        bulk_g2s(raw1, reinterpret_cast<const void*>(a1 & ~uintptr_t(15)), bytes1, tmaBar);
        if(run2)
            bulk_g2s(raw2, reinterpret_cast<const void*>(a2 & ~uintptr_t(15)), bytes2, tmaBar);
    }
    mbar_wait(tmaBar, tmaPhase);
    tmaPhase ^= 1u;
    if(pack && !run2)
    {
        pack_span16<GS>(win, raw1, lead1, srcDelay, count, t, bar);
        packed = true;
        return true;
    }
    float *dst = win + kEdge + srcDelay;
    const int16_t *r1 = reinterpret_cast<const int16_t*>(raw1) + lead1;
    const int16_t *r2 = reinterpret_cast<const int16_t*>(raw2) + lead2;
    constexpr int PERW = (kSrcSizeMax + GS - 1)/GS;
    float v[PERW];
    #pragma unroll
    for(int u = 0;u < PERW;++u)
    {
        const uint32_t k = uint32_t(t) + uint32_t(u)*GS;
        int16_t x = 0;
        if(k < count) x = k < run1 ? r1[k] : r2[k - run1];
        v[u] = to_float(x);
    }
    group_sync(bar, GS);                 // raw span consumed: the floats may overwrite it
    #pragma unroll
    for(int u = 0;u < PERW;++u)
    {
        const uint32_t k = uint32_t(t) + uint32_t(u)*GS;
        if(k < count) dst[k] = v[u];
    }
    return true;
}

// Gather staging of the source span: LoadBufferStatic (core/voice.cpp:500-544) as one run;
// element k maps to buffer frame q(k).  LoadBufferQueue (:546-595): one run per queue item
// crossed, then the last sample held.  Loads are issued 8 at a time before any conversion.
// Returns whether every sample came from a <= 16-bit format.
template<int GS>
__device__ __forceinline__ bool gather_span(const MixParams &P, const BufferRec &buf, uint32_t flags,
    bool isQueue, uint4 qh, const uint32_t *qitems, bool looping, uint32_t loopStart, uint32_t loopEnd,
    uint32_t uintPos, uint32_t count, float *dst, int t, int bar)
{
    uint32_t done = 0, item = qh.x ? qh.y : kNoLoop, qpos = uintPos;
    bool more = true, winInt = true;
    while(more)
    {
        BufferRec rb = buf;
        FillArgs fa;
        if(!isQueue)
        {
            const uint32_t loopSize = looping ? (loopEnd - loopStart) : 1u;
            const uint32_t q0 = !looping ? uintPos : ((uintPos < loopEnd) ? uintPos
                : ((uintPos-loopStart)%loopSize + loopStart));
            const uint32_t firstRun = looping ? (loopEnd - q0) : 0u;
            const uint32_t lastFrame = buf.frames ? buf.frames-1u : 0u;
            const bool pastEnd = !looping && !(buf.frames > uintPos);
            const bool simpleWrap = looping && count <= firstRun + loopSize;
            fa = FillArgs{dst, count, uintPos, q0, firstRun, loopStart, loopSize,
                lastFrame, buf.channels, looping, pastEnd, simpleWrap};
            done = count; more = false;
        }
        else
        {
            bool found = false;
            while(item != kNoLoop && done < count)
            {
                rb = P.buffers[qitems[item]];
                if(qpos >= rb.frames)
                {
                    qpos -= rb.frames;
                    item = (item + 1u < qh.x) ? item + 1u : qh.z;
                    continue;
                }
                found = true;
                break;
            }
            if(!found) break;
            const uint32_t run = min(count - done, rb.frames - qpos);
            fa = FillArgs{dst + done, run, qpos, qpos, 0u, 0u, 1u, rb.frames-1u,
                rb.channels, false, false, false};
            done += run; qpos = 0u;
            item = (item + 1u < qh.x) ? item + 1u : qh.z;
            more = done < count;
        }
        winInt = winInt && (rb.type <= 1u || rb.type >= 5u);
        // srcChannel of LoadSamples (core/voice.cpp:271-287); a channel the buffer
        // does not have reads channel 0
        const uint32_t ch = ((flags >> 16) & 0xffu) < rb.channels ? ((flags >> 16) & 0xffu) : 0u;
        switch(rb.type)
        {
        case 0: fill_window<uint8_t, GS>(fa, static_cast<const uint8_t*>(rb.data) + ch, t); break;
        case 1: fill_window<int16_t, GS>(fa, static_cast<const int16_t*>(rb.data) + ch, t); break;
        case 2: fill_window<int32_t, GS>(fa, static_cast<const int32_t*>(rb.data) + ch, t); break;
        case 3: fill_window<float, GS>(fa, static_cast<const float*>(rb.data) + ch, t); break;
        case 4: fill_window<double, GS>(fa, static_cast<const double*>(rb.data) + ch, t); break;
        case 5: fill_window<MulawByte, GS>(fa, static_cast<const MulawByte*>(rb.data) + ch, t); break;
        default: fill_window<AlawByte, GS>(fa, static_cast<const AlawByte*>(rb.data) + ch, t); break;
        }
    }
    if(done < count)
    {
        // queue ran out inside the window: hold the last sample (0 if none)
        group_sync(bar, GS);
        const float held = done ? dst[done-1u] : 0.0f;
        for(uint32_t k = done + t;k < count;k += GS) dst[k] = held;
    }
    return winInt;
}

// 16-bit window for the bsinc resamplers.
// u8/i16/mu-law/A-law samples are exact multiples of 2^-15, so a window of such samples (its
// history included, see exact16) can be re-stored as biased 16-bit integers y = 32768*s + 32768
// without loss.  Two copies (A: pairs (y0,y1),(y2,y3)..;
// B: pairs (y1,y2),(y3,y4)..) give every window position an aligned pair, so ONE 32-bit shared
// load feeds two taps: the resampler is bound by shared-memory wavefronts (3 per lane-tap: F, D,
// sample) and this removes half of the sample loads and their bank conflicts at pitch > 1.
// Converting back costs a PRMT and half an add per tap on the idle ALU; the 2^-15 scale is
// applied once to the result (exact), so the resampled line is unchanged bit for bit.
template<int GS>
__device__ __forceinline__ void pack_window16(float *win, uint32_t srcn, int t, int bar)
{
    constexpr int PER = (kResBuf + 8 + GS - 1)/GS;
    const uint32_t L = min(uint32_t(kEdge) + srcn + 8u, uint32_t(kResBuf + 8));
    float v[PER];
    #pragma unroll
    for(int u = 0;u < PER;++u)
    {
        const uint32_t k = uint32_t(t) + uint32_t(u)*GS;
        v[u] = k < L ? win[k] : 0.0f;
    }
    group_sync(bar, GS);
    uint16_t *pa = reinterpret_cast<uint16_t*>(win);
    uint16_t *pb = pa + 2*kPackB;
    #pragma unroll
    for(int u = 0;u < PER;++u)
    {
        const uint32_t k = uint32_t(t) + uint32_t(u)*GS;
        if(k < L)
        {
            const uint16_t y = uint16_t(__float2int_rn(v[u]*32768.0f) + 32768);
            pa[k] = y;
            if(k) pb[k-1u] = y;
        }
    }
    group_sync(bar, GS);
}

// Resamples dstn outputs of one chunk into xs[loaded..] (core/voice.cpp:764-769).
template<int GS>
__device__ __forceinline__ void resample_chunk(const float *win, const float *tabF, const float *tabD,
    float *xs, uint32_t loaded, uint32_t dstn, uint32_t increment, uint32_t fracPos,
    uint32_t resampler, uint32_t m, uint32_t tapOff, uint32_t ms, bool packedWin, int t)
{
    const float *srcBuffer = win + kEdge;
    if(increment == 65536u && fracPos == 0u)
    {
        for(uint32_t k = t;k < dstn;k += GS) xs[loaded+k] = srcBuffer[k];
    }
    else if(packedWin)
    {
        const uint32_t *wordsA = reinterpret_cast<const uint32_t*>(win);
        const uint32_t *wordsB = wordsA + kPackB;
        const float2 bias = make_float2(-8421376.0f, -8421376.0f);   // -(2^23 + 32768)
        const float2 one = make_float2(1.0f, 1.0f);
        for(uint32_t k = t;k < dstn;k += 2u*GS)
        {
            const uint32_t kB = k + GS;
            const bool hasB = kB < dstn;
            const uint64_t fpA = uint64_t(k)*increment + fracPos;
            const uint64_t fpB = uint64_t(hasB ? kB : k)*increment + fracPos;
            const uint32_t fracA = uint32_t(fpA) & 0xffffu, fracB = uint32_t(fpB) & 0xffffu;
            const float pfA = float(fracA & 2047u) * (1.0f/2048.0f);
            const float pfB = float(fracB & 2047u) * (1.0f/2048.0f);
            const float *FA = tabF + (fracA>>11)*ms, *DA = tabD + (fracA>>11)*ms;
            const float *FB = tabF + (fracB>>11)*ms, *DB = tabD + (fracB>>11)*ms;
            const uint32_t posA = tapOff + uint32_t(fpA>>16), posB = tapOff + uint32_t(fpB>>16);
            const uint32_t *wA = ((posA & 1u) ? wordsB : wordsA) + (posA >> 1);
            const uint32_t *wB = ((posB & 1u) ? wordsB : wordsA) + (posB >> 1);
            const float2 pA = make_float2(pfA, pfA), pB = make_float2(pfB, pfB);
            float2 a0 = make_float2(0.0f, 0.0f), a1 = a0, b0 = a0, b1 = a0;
            for(uint32_t j = 0;j < m;j += 4)
            {
                const uint32_t wa0 = wA[(j>>1)], wa1 = wA[(j>>1)+1u];
                const uint32_t wb0 = wB[(j>>1)], wb1 = wB[(j>>1)+1u];
                // (0x4B000000 | y) is the float 2^23 + y: subtract the bias to get 32768*s
                const float2 sA0 = fma2_rn(make_float2(__uint_as_float(__byte_perm(wa0, 0x4B00u, 0x5410u)),
                    __uint_as_float(__byte_perm(wa0, 0x4B00u, 0x5432u))), one, bias);
                const float2 sA1 = fma2_rn(make_float2(__uint_as_float(__byte_perm(wa1, 0x4B00u, 0x5410u)),
                    __uint_as_float(__byte_perm(wa1, 0x4B00u, 0x5432u))), one, bias);
                const float2 sB0 = fma2_rn(make_float2(__uint_as_float(__byte_perm(wb0, 0x4B00u, 0x5410u)),
                    __uint_as_float(__byte_perm(wb0, 0x4B00u, 0x5432u))), one, bias);
                const float2 sB1 = fma2_rn(make_float2(__uint_as_float(__byte_perm(wb1, 0x4B00u, 0x5410u)),
                    __uint_as_float(__byte_perm(wb1, 0x4B00u, 0x5432u))), one, bias);
                const float2 cA0 = fma2_rn(pA, make_float2(DA[j+0], DA[j+1]), make_float2(FA[j+0], FA[j+1]));
                const float2 cB0 = fma2_rn(pB, make_float2(DB[j+0], DB[j+1]), make_float2(FB[j+0], FB[j+1]));
                const float2 cA1 = fma2_rn(pA, make_float2(DA[j+2], DA[j+3]), make_float2(FA[j+2], FA[j+3]));
                const float2 cB1 = fma2_rn(pB, make_float2(DB[j+2], DB[j+3]), make_float2(FB[j+2], FB[j+3]));
                a0 = fma2_rn(cA0, sA0, a0);
                b0 = fma2_rn(cB0, sB0, b0);
                a1 = fma2_rn(cA1, sA1, a1);
                b1 = fma2_rn(cB1, sB1, b1);
            }
            xs[loaded+k] = ((a0.x + a1.x) + (a0.y + a1.y)) * (1.0f/32768.0f);
            if(hasB) xs[loaded+kB] = ((b0.x + b1.x) + (b0.y + b1.y)) * (1.0f/32768.0f);
        }
    }
    else if(resampler >= 2u)
    {
        const float *vals = win + tapOff;
        // two outputs per thread per pass (k and k+GS): twice the independent
        // FFMA2 chains and loads in flight per warp
        for(uint32_t k = t;k < dstn;k += 2u*GS)
        {
            const uint32_t kB = k + GS;
            const bool hasB = kB < dstn;
            const uint64_t fpA = uint64_t(k)*increment + fracPos;
            const uint64_t fpB = uint64_t(hasB ? kB : k)*increment + fracPos;
            const uint32_t fracA = uint32_t(fpA) & 0xffffu, fracB = uint32_t(fpB) & 0xffffu;
            const float pfA = float(fracA & 2047u) * (1.0f/2048.0f);
            const float pfB = float(fracB & 2047u) * (1.0f/2048.0f);
            // scalar coefficient loads from rows with an ODD stride: every lane reads
            // its own phase row without bank conflicts; pairs are packed for FFMA2
            const float *FA = tabF + (fracA>>11)*ms, *DA = tabD + (fracA>>11)*ms;
            const float *FB = tabF + (fracB>>11)*ms, *DB = tabD + (fracB>>11)*ms;
            const float *svA = vals + uint32_t(fpA>>16), *svB = vals + uint32_t(fpB>>16);
            const float2 pA = make_float2(pfA, pfA), pB = make_float2(pfB, pfB);
            float2 a0 = make_float2(0.0f, 0.0f), a1 = a0, b0 = a0, b1 = a0;
            for(uint32_t j = 0;j < m;j += 4)
            {
                // two taps per packed FFMA2: c = F + pf*D ; r += c*s
                const float2 cA0 = fma2_rn(pA, make_float2(DA[j+0], DA[j+1]), make_float2(FA[j+0], FA[j+1]));
                const float2 cB0 = fma2_rn(pB, make_float2(DB[j+0], DB[j+1]), make_float2(FB[j+0], FB[j+1]));
                const float2 cA1 = fma2_rn(pA, make_float2(DA[j+2], DA[j+3]), make_float2(FA[j+2], FA[j+3]));
                const float2 cB1 = fma2_rn(pB, make_float2(DB[j+2], DB[j+3]), make_float2(FB[j+2], FB[j+3]));
                a0 = fma2_rn(cA0, make_float2(svA[j+0], svA[j+1]), a0);
                b0 = fma2_rn(cB0, make_float2(svB[j+0], svB[j+1]), b0);
                a1 = fma2_rn(cA1, make_float2(svA[j+2], svA[j+3]), a1);
                b1 = fma2_rn(cB1, make_float2(svB[j+2], svB[j+3]), b1);
            }
            xs[loaded+k] = (a0.x + a1.x) + (a0.y + a1.y);
            if(hasB) xs[loaded+kB] = (b0.x + b1.x) + (b0.y + b1.y);
        }
    }
    else
    {
        const float *vals = srcBuffer;
        for(uint32_t k = t;k < dstn;k += GS)
        {
            const uint64_t fp = uint64_t(k)*increment + fracPos;
            const uint32_t pos = uint32_t(fp>>16), frac = uint32_t(fp) & 0xffffu;
            if(resampler == 0u) xs[loaded+k] = vals[pos];
            else
            {
                const float a = vals[pos], b = vals[pos+1];
                xs[loaded+k] = a + (b-a)*(float(frac)*(1.0f/65536.0f));
            }
        }
    }
}

// History for the next update (core/voice.cpp:772-785), then the step to the next chunk: the
// source position moves past the consumed samples and the window tail slides to the front
// (core/voice.cpp:808-809).
template<int GS>
__device__ __forceinline__ void advance_chunk(float *win, float *prev, bool packedWin, bool silent,
    bool playing, uint32_t n, uint32_t &loaded, uint32_t dstn, uint32_t increment, uint32_t &fracPos,
    int32_t &intPos, int t, int bar)
{
    const uint32_t loadEnd = loaded + dstn;
    if(!silent && playing && n > loaded && n <= loadEnd)
    {
        const uint32_t dstOffset = n - loaded;
        const uint32_t srcOffset = uint32_t((uint64_t(dstOffset)*increment + fracPos) >> 16);
        for(int k = t;k < kPad;k += GS) prev[k] = win_at(win, packedWin, srcOffset + uint32_t(k));
    }
    loaded = loadEnd;
    if(loaded < n)
    {
        fracPos += dstn*increment;
        const uint32_t srcOffset = fracPos >> 16;
        fracPos &= 0xffffu;
        if(silent) intPos = add_sat(intPos, int32_t(srcOffset));
        else
        {
            if(intPos < 0) intPos += int32_t(srcOffset);
            else intPos = add_sat(intPos, int32_t(srcOffset));
            float carry = 0.0f;
            if(t < kPad) carry = win_at(win, packedWin, srcOffset + uint32_t(t));
            float carry2 = 0.0f;
            if(GS < kPad && t + GS < kPad) carry2 = win_at(win, packedWin, srcOffset + uint32_t(t) + GS);
            group_sync(bar, GS);
            if(t < kPad) win[t] = carry;
            if(GS < kPad && t + GS < kPad) win[t + GS] = carry2;
        }
    }
}

// Auxiliary sends (core/voice.cpp:967-980): the UNFILTERED resampled line is parked in HBM;
// k_send_filters / k_send_mix take it from there slot by slot.  The parking variant (CDR == 0:
// HRTF devices, or more than 4 dry channels) mixes no voice itself: every line is parked, HRTF
// voices for k_hrtf_fir (kSiHrtf), the others for k_send_mix, which sums the dry bus like one
// more slot (kSiDry; deterministic, no atomics).  sendinfo carries what those kernels need of
// the voice's state.  A direct-channel voice's line is parked for the RealOut bus (kSiReal) by
// both variants.
template<int GS, int CDR>
__device__ __forceinline__ void park_voice(const MixParams &P, const float *xs, uint32_t v,
    uint32_t sendMask, bool defer, bool isHrtf, bool isDirect, bool playing, bool dirty, uint32_t counter, int t)
{
    const uint32_t n = P.frames;
    const bool sends = P.num_sends && sendMask;
    const bool park = sends || defer || isDirect || CDR == 0;
    if(CDR > 0 && park)
        for(uint32_t k = t;k < n;k += GS) P.xscratch[size_t(v)*kLine + k] = xs[k];
    if(t == 0)
        P.sendinfo[v] = park ? ((sends ? kSiSend : 0u)
            | (playing ? kSiPlaying : 0u) | (defer ? kSiDeferred : 0u) | (dirty ? kSiDirty : 0u)
            | ((CDR == 0 && !isHrtf && !isDirect) ? kSiDry : 0u) | (isHrtf ? kSiHrtf : 0u)
            | (isDirect ? kSiReal : 0u) | (counter << 8)) : 0u;
}

// MixSamples -> Mix_ (core/mixer.h:27-41, mixer_c.cpp:150-186,247-258) of one line into the
// register dry bus: thread t holds samples t + r*GS of every channel.  Thread 0 leaves the
// new Current gains in newGain; they are stored once every thread has read the old ones.
template<int GS, int CDR>
__device__ __forceinline__ void mix_dry(float (&accD)[CDR][kLine/GS], const float *xs, float *newGain,
    const float *cur, const float *tgt, uint32_t cd, uint32_t n, uint32_t counter, bool playing, int t)
{
    constexpr int SPT = kLine / GS;
    const float delta = counter ? 1.0f/float(counter) : 0.0f;
    const uint32_t fadeLen = counter < n ? counter : n;
    for(uint32_t c = 0;c < cd;++c)
    {
        const float cg = counter ? cur[c] : tgt[c];
        const float tg = playing ? tgt[c] : 0.0f;
        const float step = (tg - cg)*delta;
        const bool fade = fabsf(step) > kEps;
        const bool early = fade && fadeLen < counter;
        const float flat = (!early && fabsf(tg) > kSilence) ? tg : 0.0f;
        const uint32_t start = fade ? fadeLen : 0u;
        #pragma unroll
        for(int r = 0;r < SPT;++r)
        {
            const uint32_t i = t + r*GS;
            float gi = 0.0f;
            if(i < n)
                gi = (fade && i < fadeLen) ? (cg + step*float(i)) : (i >= start ? flat : 0.0f);
            const float x = xs[i < n ? i : 0];
            // one fused multiply-add, written out: left to the compiler, whether x*gi is
            // contracted into the sum depends on the kernel this is inlined into, and both
            // kernels that call this must round the same way
            if(c < uint32_t(CDR))
            {
                #pragma unroll
                for(int cc = 0;cc < CDR;++cc)
                    if(cc == int(c)) accD[cc][r] = __fmaf_rn(x, gi, accD[cc][r]);
            }
        }
        if(t == 0)
            newGain[c] = early ? (cg + step*float(fadeLen)) : tg;
    }
}

// Gains.Current write-back of mix_dry, after every thread of the group has read the old values.
__device__ __forceinline__ void store_dry_gains(float *cur, const float *newGain, uint32_t cd, int t)
{
    if(t == 0)
        for(uint32_t c = 0;c < cd;++c) cur[c] = newGain[c];
}

// Position / state update (core/voice.cpp:1116-1232), by one thread.
__device__ __forceinline__ void write_back_voice(const MixParams &P, VoiceRec &rec, uint32_t v,
    uint4 h1, uint32_t flags, uint32_t vstate, uint32_t increment, bool haveBuffer, bool isQueue,
    uint4 qh, const uint32_t *qitems, bool looping, uint32_t loopStart, uint32_t loopEnd,
    uint32_t bufFrames)
{
    uint32_t newFlags = (flags | kVfFading) & ~kVfCoefDirty;
    uint32_t newState = vstate;
    uint32_t buffersDone = 0u;
    int32_t pos = int32_t(h1.x); uint32_t frac = h1.y;
    if(vstate == 2u) newState = 0u;
    else
    {
        frac += increment*P.frames;
        const uint32_t done = frac >> 16;
        pos = add_sat(pos, int32_t(done));
        frac &= 0xffffu;
        if(haveBuffer && pos > 0 && isQueue)
        {
            // streaming source: finished items leave the queue (core/voice.cpp:1183-1196)
            uint32_t item = qh.x ? qh.y : kNoLoop;
            while(item != kNoLoop)
            {
                const uint32_t len = P.buffers[qitems[item]].frames;
                if(len > uint32_t(pos)) break;
                pos -= int32_t(len);
                ++buffersDone;
                item = (item + 1u < qh.x) ? item + 1u : qh.z;
            }
            if(item == kNoLoop) { newFlags &= ~kVfHaveBuffer; newState = 2u; }
            else if(item != qh.y) P.qhdr[v].y = item;
        }
        else if(haveBuffer && pos > 0)
        {
            if(looping)
            {
                uint32_t up = uint32_t(pos);
                if(up >= loopEnd)
                    pos = int32_t((up-loopStart)%(loopEnd-loopStart) + loopStart);
            }
            else if(uint32_t(pos) >= bufFrames)
            {
                newFlags &= ~kVfHaveBuffer;
                newState = 2u;
            }
        }
        // a voice that had no buffer to begin with stops as well: one that ran out earlier and
        // was set playing again by an update fades out on the next one (core/voice.cpp:1224-1232)
        if(!haveBuffer) newState = 2u;
        rec.pos = pos; rec.frac = frac;
    }
    rec.flags = newFlags;
    rec.state = newState;
    if(P.results)
        P.results[v] = VoiceResult{pos, frac,
            newState == 1u ? 1u : (newState == 2u ? 2u : (1u<<7)), buffersDone};
}

// One partial row per CTA: the groups' register accumulators are summed through shared memory
// in group order (deterministic), halving the rows k_reduce_rows reads.  smem must hold
// CDR*kLine floats.
template<int GS, int GROUPS, int CDR>
__device__ __forceinline__ void store_partial_row(const float (&accD)[CDR][kLine/GS], unsigned char *smem,
    float *partial, int g, int t)
{
    constexpr int SPT = kLine / GS;
    const size_t row = blockIdx.x;
    __syncthreads();                     // every group is done with its voice storage
    float *stage = reinterpret_cast<float*>(smem);
    float *pd = partial + row*(size_t(CDR)*kLine);
    if(GROUPS == 1)
    {
        #pragma unroll
        for(int c = 0;c < CDR;++c)
            #pragma unroll
            for(int r = 0;r < SPT;++r)
                pd[c*kLine + t + r*GS] = accD[c][r];
    }
    else
    {
        for(int gg = 0;gg < GROUPS;++gg)
        {
            if(g == gg)
            {
                #pragma unroll
                for(int c = 0;c < CDR;++c)
                    #pragma unroll
                    for(int r = 0;r < SPT;++r)
                    {
                        float *dst = stage + c*kLine + t + r*GS;
                        if(gg == 0) *dst = accD[c][r]; else *dst += accD[c][r];
                    }
            }
            __syncthreads();
        }
        for(int o = threadIdx.x;o < CDR*kLine;o += GS*GROUPS) pd[o] = stage[o];
    }
}

// ---------------------------------------------------------------------------
// The resample kernel.  GS threads per voice group, GROUPS groups per CTA.
//   CDR : > 0: dry channels of non-HRTF devices accumulated in registers (static voice
//         assignment, one partial row per CTA); 0: every voice's line is parked in xscratch
//         (HRTF voices for k_hrtf_fir, the rest for k_send_mix) and groups claim voices
// A voice with an active direct filter is only resampled and parked: k_filters filters its
// line, then k_mix_deferred (CDR > 0) or k_hrtf_fir mixes it.
// ---------------------------------------------------------------------------
constexpr int kMixGS = 64, kMixGroups = 2;      // the geometry both variants are built with

template<int GS, int GROUPS, int CDR>
__global__ void __launch_bounds__(GS*GROUPS, GS*GROUPS != 128 ? 1 : (CDR == 0 ? 5 : 3))
k_mix_voices(const MixParams P)
{
    using Smem = GroupSmem<CDR>;
    static_assert(CDR == 0 || sizeof(Smem)*GROUPS >= size_t(CDR)*kLine*sizeof(float),
        "the partial row is staged in the groups' storage");
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int g = threadIdx.x / GS;
    const int t = threadIdx.x % GS;
    Smem &S = reinterpret_cast<Smem*>(smem_raw)[g];
    const int bar = 1 + g;
    constexpr int SPT = kLine / GS;               // resampled samples per thread

    float accD[CDR > 0 ? CDR : 1][SPT];
    #pragma unroll
    for(int c = 0;c < (CDR > 0 ? CDR : 1);++c)
        #pragma unroll
        for(int r = 0;r < SPT;++r) accD[c][r] = 0.0f;

    const uint32_t n = P.frames;
    if(t == 0) { mbar_init(&S.tmaBar, 1u); mbar_fence_init(); }
    uint32_t tmaPhase = 0u;                       // parity of the next completion of tmaBar
    group_sync(bar, GS);

    // Voices are visited in the host's mixing order (active voices only, sorted by
    // resampler cost).  The register-dry variant sums across voices, so its assignment is
    // grid-strided (static, deterministic sums); a parking group's line depends on its voice
    // only, so it claims the next unclaimed voice.
    const uint32_t groups = gridDim.x*GROUPS;
    for(uint32_t oi = CDR > 0 ? blockIdx.x*GROUPS + g : claim_voice(P, S.claimed, t, bar, GS, groups);
        oi < P.num_order;
        oi = CDR > 0 ? oi + groups : claim_voice(P, S.claimed, t, bar, GS, groups))
    {
        // ---- header and early-outs ----
        const uint32_t v = P.order[oi];
        VoiceRec &rec = P.voices[v];
        // one batch of vector loads for the scalar part of the record
        const uint4 *hp = reinterpret_cast<const uint4*>(&rec);
        const uint4 h0 = hp[0], h1 = hp[1], h2 = hp[2], h3 = hp[3];
        const uint32_t vstate = h0.x;
        if(voice_early_out(P, rec, v, vstate, h1, t)) continue;
        const uint32_t increment = h1.z;
        const uint32_t flags = h0.y;
        const bool haveBuffer = (flags & kVfHaveBuffer) != 0;
        // callback source (pad = 1 + its plan slot): the plan's record stands in for the buffer's,
        // this update's span of the samples its callbacks delivered
        const BufferRec rb = P.buffers[haveBuffer ? h0.z : 0u];
        const BufferRec buf = (haveBuffer && rb.pad && P.cbplan) ? P.cbplan[rb.pad - 1u] : rb;
        const uint32_t cbSlot = haveBuffer ? buf.pad : 0u;
        const uint32_t loopStart = h1.w, loopEnd = h2.x;
        int32_t intPos = int32_t(h1.x);
        uint32_t fracPos = h1.y;
        bool looping = (flags & kVfLooping) != 0 && cbSlot == 0u;
        if((flags & kVfStatic) && looping && haveBuffer && intPos >= 0
            && uint32_t(intPos) >= loopEnd)
            looping = false;                                     // core/voice.cpp:1015-1019
        const uint32_t resampler = h0.w;
        // streaming source (neither IsStatic nor callback): plays the voice's buffer queue
        const bool isQueue = !(flags & kVfStatic) && P.qhdr != nullptr && cbSlot == 0u;
        const uint4 qh = isQueue ? P.qhdr[v] : make_uint4(0u, 0u, kNoLoop, 0u);
        const uint32_t *qitems = P.queue + size_t(v)*kMaxQueue;
        // mixed through its own HRIR by k_hrtf_fir (HRTF devices only)
        const bool isHrtf = CDR == 0 && P.ir_pad != 0u && (flags & kVfHrtf);
        const bool dirty = (flags & kVfCoefDirty) != 0;
        // mixed into RealOut by the RealOut bus (never HRTF: the host refuses both)
        const bool isDirect = (flags & kVfDirect) != 0;
        FilterRec *dfilt = P.filt ? P.filt + size_t(v)*P.filt_paths : nullptr;
        // a voice with an active direct filter is only resampled here; its mix is deferred
        const bool defer = dfilt && dfilt->active;
        const bool playing = vstate == 1u;

        // ---- phase table, next-voice prefetch ----
        for(int k = t;k < kPad;k += GS) S.win[k] = rec.prev[k];
        uint32_t m, tapOff, ms;                      // taps, left offset into the window, row stride
        build_phase_table<GS>(P, S.tabF, S.tabD, resampler, increment, h2, h3, t, m, tapOff, ms);
        float *xs = CDR > 0 ? S.x : P.xscratch + size_t(v)*kLine;
        if(CDR == 0) prefetch_next_voices<GS>(P, oi, groups, t);

        // ---- LoadResampledSamples, chunk by chunk (core/voice.cpp:668-811) ----
        for(uint32_t loaded = 0;loaded < n;)
        {
            uint32_t dstn, srcn;
            calc_buffer_size(fracPos, increment, n-loaded, dstn, srcn);
            uint32_t srcDelay = 0;
            bool silent = false;
            bool packedWin = false;        // the window currently holds the two 16-bit copies
            // defence in depth (the host rejects steps above MaxPitch): a chunk that cannot
            // produce any output would never end this loop
            if(dstn == 0u) { dstn = n - loaded; silent = true; }
            if(intPos < 0)
            {
                srcDelay = uint32_t(-intPos);
                if(srcDelay >= srcn) silent = true;
            }
            // window history in place / previous chunk consumed.  The history (win[0, kEdge): mPrevSamples
            // or the previous chunk's tail, each float written by its own thread) may come from a float
            // format even when the span after it is 16-bit (a queue of mixed types, a buffer re-pointed
            // without a reset): the window is packed only when the history is exact in 16 bits too.
            const bool histExact = group_sync_and(bar, GS, t >= kEdge || exact16(S.win[t]));
            if(silent)
            {
                for(uint32_t k = t;k < dstn;k += GS) xs[loaded+k] = 0.0f;
                for(uint32_t k = t;k < srcn;k += GS) S.win[kEdge+k] = 0.0f;
            }
            else
            {
                float *srcBuffer = S.win + kEdge;
                bool winInt = false;       // every sample of this window came from a <=16-bit format
                // the bsinc resamplers read the 16-bit copies when every sample is exact in them
                const bool pack = resampler >= 4u && !(increment == 65536u && fracPos == 0u) && histExact;
                if(!haveBuffer) hold_end_sample<GS>(srcBuffer, srcn, t, bar);
                else
                {
                    const uint32_t uintPos = intPos < 0 ? 0u : uint32_t(intPos);
                    const uint32_t count = srcn - srcDelay;
                    for(uint32_t k = t;k < srcDelay;k += GS) srcBuffer[k] = 0.0f;
                    winInt = stage_span_tma<GS>(S.win, &S.tmaBar, tmaPhase, buf, flags, isQueue, looping,
                            loopStart, loopEnd, uintPos, srcDelay, count, pack, packedWin, t, bar)
                        || gather_span<GS>(P, buf, flags, isQueue, qh, qitems, looping, loopStart, loopEnd,
                            uintPos, count, srcBuffer + srcDelay, t, bar);
                }
                group_sync(bar, GS);       // window complete

                if(pack && winInt && !packedWin)
                {
                    pack_window16<GS>(S.win, srcn, t, bar);
                    packedWin = true;
                }
                resample_chunk<GS>(S.win, S.tabF, S.tabD, xs, loaded, dstn, increment, fracPos,
                    resampler, m, tapOff, ms, packedWin, t);
            }
            advance_chunk<GS>(S.win, rec.prev, packedWin, silent, playing, n, loaded, dstn, increment,
                fracPos, intPos, t, bar);
        }
        group_sync(bar, GS);               // xs complete

        // ---- park, register dry mix, position / state write-back ----
        // fade bookkeeping (core/voice.cpp:1093-1112)
        const uint32_t counter = (flags & kVfFading) ? (n < 64u ? n : 64u) : 0u;
        // the send mask is read here rather than held through the chunks: the parking
        // variant has no register to spare there
        if(P.sendinfo)
            park_voice<GS, CDR>(P, xs, v, rec.send_mask, defer, isHrtf, isDirect, playing, dirty, counter, t);
        // direct-path DoFilters (core/voice.cpp:943-946) with an inactive pair: clear()
        if(dfilt && !defer) filter_clear(*dfilt, t);
        if constexpr(CDR > 0)
            if(!defer && !isDirect)
                mix_dry<GS, CDR>(accD, xs, S.newGain, P.dry_cur + size_t(v)*P.cd, P.dry_tgt + size_t(v)*P.cd,
                    P.cd, n, counter, playing, t);
        // a callback voice's span ends where its stored samples do: the static end check is
        // then the reference's (core/voice.cpp:1158-1176, see callback_plan.hpp)
        if(t == 0)
            write_back_voice(P, rec, v, h1, flags, vstate, increment, haveBuffer, isQueue, qh, qitems,
                looping, loopStart, loopEnd, buf.frames);
        group_sync(bar, GS);               // smem free for the next voice
        if(CDR > 0 && !defer && !isDirect) store_dry_gains(P.dry_cur + size_t(v)*P.cd, S.newGain, P.cd, t);
        group_sync(bar, GS);
    }

    if constexpr(CDR > 0) store_partial_row<GS, GROUPS, CDR>(accD, smem_raw, P.partial, g, t);
    else
    {
        // both groups found the claims exhausted: the HRIR FIR may be scheduled (it waits for
        // this grid's completion before it reads anything the voices wrote)
        __syncthreads();
        griddep_launch_dependents();
    }
}

// ---------------------------------------------------------------------------
// The deferred dry pass (register-dry devices).  Mixes the voices k_mix_voices parked with
// kSiDeferred (direct-channel voices, kSiReal, excepted: the RealOut bus mixes them) once
// k_filters has left their filtered line in dline.  Same static assignment
// over the order it is given (order2), the same Mix_ arithmetic and the same partial-row
// combine as k_mix_voices<GS,GROUPS,CDR>, so the sums and their order are unchanged.
// ---------------------------------------------------------------------------
template<int GROUPS, int CDR>
union DeferredSmem {
    struct { float x[kLine]; float newGain[32]; } group[GROUPS];
    float stage[CDR*kLine];                           // partial-row combine, once every group is done
};

template<int GS, int GROUPS, int CDR>
__global__ void __launch_bounds__(GS*GROUPS)
k_mix_deferred(const MixParams P)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int g = threadIdx.x / GS;
    const int t = threadIdx.x % GS;
    auto &S = reinterpret_cast<DeferredSmem<GROUPS, CDR>*>(smem_raw)->group[g];
    const int bar = 1 + g;
    constexpr int SPT = kLine / GS;

    float accD[CDR][SPT];
    #pragma unroll
    for(int c = 0;c < CDR;++c)
        #pragma unroll
        for(int r = 0;r < SPT;++r) accD[c][r] = 0.0f;

    const uint32_t n = P.frames;
    const uint32_t groups = gridDim.x*GROUPS;
    for(uint32_t oi = blockIdx.x*GROUPS + g;oi < P.num_order;oi += groups)
    {
        const uint32_t v = P.order[oi];
        const uint32_t info = P.sendinfo[v];
        if((info & (kSiDeferred | kSiReal)) != kSiDeferred) continue;
        const float *fl = P.dline + size_t(v)*kLine;
        for(uint32_t k = t;k < n;k += GS) S.x[k] = fl[k];
        group_sync(bar, GS);               // line staged
        mix_dry<GS, CDR>(accD, S.x, S.newGain, P.dry_cur + size_t(v)*P.cd, P.dry_tgt + size_t(v)*P.cd,
            P.cd, n, (info >> 8) & 0xffu, (info & kSiPlaying) != 0, t);
        group_sync(bar, GS);               // line and old gains read
        store_dry_gains(P.dry_cur + size_t(v)*P.cd, S.newGain, P.cd, t);
    }

    store_partial_row<GS, GROUPS, CDR>(accD, smem_raw, P.partial, g, t);
}

// ---------------------------------------------------------------------------
// The HRIR FIR kernel (HRTF devices).  Mixes every voice k_mix_voices parked with kSiHrtf:
// takes the line from xscratch (dline when its direct filter ran), builds DoHrtfMix's
// gain-ramped per-ear inputs (core/voice.cpp:827-902; MixHrtfBlend/MixHrtf, hrtfbase.h:17-89)
// and runs the HRIR FIR in gather form with OPT contiguous outputs per thread held in
// registers ACROSS all voices of the group (the cross-voice reduction of `Accum[i+j] += ...`
// happens in registers, not memory).  Voices are assigned statically in the mixing order and
// each CTA stores one partial row; k_post_hrtf_reduce sums the rows in a fixed order
// (deterministic output).  A group's inputs for its next voice are bulk-copied into its second
// stage buffer while the current voice is built and filtered.
//   OPT/FP : FIR outputs per thread / front pad (17/64 for ir<=64, 19/128 for ir<=128)
// ---------------------------------------------------------------------------
constexpr int kFirGS = 64, kFirGroups = 2, kFirCtasPerSm = 4;

// First order slot from oi on, in steps of stride, whose voice was parked for the HRIR FIR
// (kSiHrtf), with that voice and its sendinfo; P.num_order or more when there is none.
__device__ __forceinline__ uint32_t next_hrtf_voice(const MixParams &P, uint32_t oi, uint32_t stride,
    uint32_t &v, uint32_t &info)
{
    for(;oi < P.num_order;oi += stride)
    {
        v = P.order[oi];
        info = P.sendinfo[v];
        if(info & kSiHrtf) break;
    }
    return oi;
}

// One thread fills stage buffer B with voice v's History, line and HRIR(s) by bulk copies that
// complete on bar.  A bulk copy moves a multiple of 16 bytes, so the line's last n%4 samples are
// left to plain loads.
__device__ __forceinline__ void fir_stage_issue(const MixParams &P, FirStage &B, uint64_t *bar,
    uint32_t v, uint32_t info, uint32_t n)
{
    const uint32_t lineBytes = (n & ~3u)*4u, irBytes = P.ir_pad*8u;
    const bool dirty = (info & kSiDirty) != 0;
    const float *line = ((info & kSiDeferred) ? P.dline : P.xscratch) + size_t(v)*kLine;
    fence_proxy_async_smem();            // the group's generic accesses to B come first
    mbar_expect_tx(bar, kHist*4u + lineBytes + (dirty ? 2u : 1u)*irBytes);
    bulk_g2s(B.x, P.voices[v].hist, kHist*4u, bar);
    if(lineBytes) bulk_g2s(B.x + kHist, line, lineBytes, bar);
    bulk_g2s(B.coefT, P.hrtf_tgt + size_t(v)*P.ir_pad, irBytes, bar);
    if(dirty) bulk_g2s(B.coefO, P.hrtf_old + size_t(v)*P.ir_pad, irBytes, bar);
}

template<int OPT, int FP>
__global__ void __launch_bounds__(kFirGS*kFirGroups, kFirCtasPerSm)
k_hrtf_fir(const MixParams P)
{
    constexpr int GS = kFirGS, GROUPS = kFirGroups;
    using Smem = FirSmem<GS, OPT, FP>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int g = threadIdx.x / GS;
    const int t = threadIdx.x % GS;
    Smem &S = reinterpret_cast<Smem*>(smem_raw)[g];
    const int bar = 1 + g;
    const int t0 = OPT*t;
    const uint32_t n = P.frames;

    float2 acc[OPT];
    #pragma unroll
    for(int r = 0;r < OPT;++r) acc[r] = make_float2(0.0f, 0.0f);

    // the FIR input's front pad and the samples past the update's end are zero for every voice
    for(int i = t;i < FP;i += GS) S.lLR[i] = make_float2(0.0f, 0.0f);
    for(int i = FP + int(n) + t;i < Smem::kLLen;i += GS) S.lLR[i] = make_float2(0.0f, 0.0f);
    if(t == 0) { mbar_init(&S.bar[0], 1u); mbar_init(&S.bar[1], 1u); mbar_fence_init(); }
    group_sync(bar, GS);
    // launched right behind the resample kernel, the set-up above ran under its tail: what it
    // writes (sendinfo, the parked lines, the voice records) is read only from here on
    griddep_wait();

    const uint32_t stride = gridDim.x*GROUPS;
    uint32_t v = 0u, info = 0u;
    uint32_t oi = next_hrtf_voice(P, blockIdx.x*GROUPS + g, stride, v, info);
    if(t == 0 && oi < P.num_order) fir_stage_issue(P, S.st[0], &S.bar[0], v, info, n);
    uint32_t parity = 0u;                    // bit b: parity of stage buffer b's next completion
    for(int b = 0;oi < P.num_order;b ^= 1)
    {
        VoiceRec &rec = P.voices[v];
        const uint4 *hp = reinterpret_cast<const uint4*>(&rec);
        const uint4 h3 = hp[3], h4 = hp[4];     // in flight during the look-ahead's loads

        // the group's next voice is copied into the other stage buffer while this one mixes
        // (the previous voice's reads of it ended at the last barrier)
        uint32_t vN = 0u, infoN = 0u;
        const uint32_t oiN = next_hrtf_voice(P, oi + stride, stride, vN, infoN);
        if(t == 0 && oiN < P.num_order) fir_stage_issue(P, S.st[b^1], &S.bar[b^1], vN, infoN, n);

        FirStage &B = S.st[b];
        const bool playing = (info & kSiPlaying) != 0;
        const bool dirty = (info & kSiDirty) != 0;
        const uint32_t counter = (info >> 8) & 0xffu;

        // ---- the line's last n%4 samples, which the bulk copy leaves out ----
        const float *line = ((info & kSiDeferred) ? P.dline : P.xscratch) + size_t(v)*kLine;
        for(uint32_t k = (n & ~3u) + t;k < n;k += GS) B.x[kHist + k] = line[k];
        mbar_wait(&S.bar[b], (parity >> b) & 1u);
        parity ^= 1u << b;
        if(n & 3u) group_sync(bar, GS);

        // DoHrtfMix (core/voice.cpp:827-902), outPos == 0
        if(playing)
            for(int k = t;k < kHist;k += GS) rec.hist[k] = B.x[n + k];
        uint32_t oD0 = h4.x, oD1 = h4.y;
        float oGain = __uint_as_float(h4.z);
        const uint32_t tD0 = h3.y, tD1 = h3.z;
        const float tgtGain = __uint_as_float(h3.w);
        if(!counter) { oD0 = tD0; oD1 = tD1; oGain = tgtGain; }
        const bool sameFilter = !counter || (!dirty && oD0 == tD0 && oD1 == tD1);
        const float targetGain = tgtGain * (playing ? 1.0f : 0.0f);
        const uint32_t fademix = counter;                     // counter <= n always
        float blendNewStep = 0.0f, oldStep = 0.0f;
        bool oldOn = false, newOn = false;
        float gainA = oGain;                                  // Old.Gain entering part 2
        if(fademix)
        {
            const float gain = targetGain;                    // counter == fademix
            blendNewStep = gain / float(fademix);
            oldStep = oGain / float(fademix);
            oldOn = oGain > kSilence;
            newOn = blendNewStep*float(fademix) > kSilence;
            gainA = gain;
        }
        const uint32_t todo = n - fademix;
        const float step2 = todo ? (targetGain - gainA) / float(todo) : 0.0f;

        // FIR input sample s at lLR[FP + s]; the pad and the tail stay zero from the start
        const float *hs = B.x;                                // [History | samples]
        float2 *in = S.lLR + FP;
        for(uint32_t s = t;s < fademix;s += GS)               // the fade (at most 64 samples)
        {
            const float gnew = (newOn && s >= 1u) ? blendNewStep*float(s) : 0.0f;
            float l = hs[kHist - tD0 + s] * gnew;
            float r = hs[kHist - tD1 + s] * gnew;
            if(sameFilter && oldOn)
            {
                const float gold = oldStep*float(fademix - s);
                l += hs[kHist - oD0 + s] * gold;
                r += hs[kHist - oD1 + s] * gold;
            }
            in[s] = make_float2(l, r);
        }
        const float *xl = hs + kHist - tD0, *xr = hs + kHist - tD1;
        for(uint32_t s = fademix + t;s < n;s += GS)           // the steady ramp
        {
            const float gnew = gainA + step2*float(s - fademix);
            in[s] = make_float2(xl[s] * gnew, xr[s] * gnew);
        }
        const bool oldPass = !sameFilter && oldOn;
        if(oldPass)
            for(int i = t;i < Smem::kOLen;i += GS)
            {
                const int s = i - FP;
                float l = 0.0f, r = 0.0f;
                if(s >= 0 && uint32_t(s) < fademix)
                {
                    const float gold = oldStep*float(fademix - uint32_t(s));
                    l = hs[kHist - oD0 + s] * gold;
                    r = hs[kHist - oD1 + s] * gold;
                }
                S.oLR[i] = make_float2(l, r);
            }
        group_sync(bar, GS);

        const int irpad = int(P.ir_pad);
        fir_pass<OPT, FP>(acc, S.lLR, B.coefT, irpad, t0);
        if(oldPass && t0 < int(kHist) + irpad)      // the old HRIR is the target one unless dirty
            fir_pass<OPT, FP>(acc, S.oLR, dirty ? B.coefO : B.coefT, irpad, t0);
        if(t == 0)
        {
            rec.old_delay0 = tD0; rec.old_delay1 = tD1;
            rec.old_gain = targetGain;
        }
        group_sync(bar, GS);               // lLR, oLR and stage buffer b free for the next voices
        oi = oiN; v = vN; info = infoN;
    }

    // ---- one partial row per CTA: the groups' register accumulators are summed through
    //      shared memory in group order (deterministic), halving the rows k_post_hrtf_reduce reads
    const size_t row = blockIdx.x;
    __syncthreads();                         // every group is done with its voice storage
    griddep_launch_dependents();             // the post-process may be scheduled (it waits for the rows)
    float *stage = reinterpret_cast<float*>(smem_raw);     // >= 2*kAccumLen floats (group 0's area)
    for(int gg = 0;gg < GROUPS;++gg)
    {
        if(g == gg)
        {
            #pragma unroll
            for(int r = 0;r < OPT;++r)
            {
                const int o = t0 + r;
                if(o < kAccumLen)
                {
                    if(gg == 0) { stage[o] = acc[r].x; stage[kAccumLen + o] = acc[r].y; }
                    else { stage[o] += acc[r].x; stage[kAccumLen + o] += acc[r].y; }
                }
            }
            if(gg == 0 && GS*OPT < kAccumLen)
                for(int o = GS*OPT + t;o < kAccumLen;o += GS) { stage[o] = 0.0f; stage[kAccumLen + o] = 0.0f; }
        }
        __syncthreads();
    }
    float *pl = P.partial + row*(2*kAccumLen);
    for(int o = threadIdx.x;o < 2*kAccumLen;o += GS*GROUPS) pl[o] = stage[o];
}


// Sums `rows` partial rows of `len` floats in a fixed order into out (+= if accumulate).
// A CTA owns 8 float4 columns (one 128-byte line of every row); its 1024 threads are 128
// row segments x 8 lanes, so every thread has only rows/128 loads to chain and 72+ SMs pull
// from L2 at once; the 128 segment sums are then combined in shared memory, 4 at a time in
// fixed order.  Deterministic: the summation tree depends only on (rows, len).
constexpr int kReduceCols = 8, kReduceSegs = 128;

// The CTA's part of that sum: float4 column e4 of the rows (thread col = threadIdx.x % 8 of a
// 1024-thread CTA), summed when `live`.  Every thread of the CTA calls it; the total is
// returned to the 8 threads of segment 0 (threadIdx.x < 8).
__device__ __forceinline__ float4 reduce_rows_cta(const float *__restrict__ partial, uint32_t rows,
    uint32_t len, uint32_t e4, bool live, float4 (&sm)[kReduceSegs][kReduceCols])
{
    const uint32_t col = threadIdx.x & (kReduceCols-1), seg = threadIdx.x / kReduceCols;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    if(live)
    {
        const uint32_t per = (rows + kReduceSegs - 1u)/kReduceSegs;
        const uint32_t r0 = seg*per, r1 = (r0 + per < rows) ? r0 + per : rows;
        const float4 *p = reinterpret_cast<const float4*>(partial) + e4;
        const size_t stride4 = len/4u;
        // up to 8 rows' loads in flight at once (one L2 round trip for a segment of <= 8 rows,
        // e.g. 528 FIR rows), then added in row order
        constexpr uint32_t kBatch = 8;
        for(uint32_t r = r0;r < r1;r += kBatch)
        {
            float4 a[kBatch];
            #pragma unroll
            for(uint32_t k = 0;k < kBatch;++k)
                if(r + k < r1) a[k] = __ldg(p + size_t(r + k)*stride4);
            #pragma unroll
            for(uint32_t k = 0;k < kBatch;++k)
                if(r + k < r1) { s.x += a[k].x; s.y += a[k].y; s.z += a[k].z; s.w += a[k].w; }
        }
    }
    sm[seg][col] = s;
    __syncthreads();
    // 128 -> 32 -> 8 -> 2 -> 1 partial sums per column, each level adding 4 neighbours in order
    #pragma unroll
    for(uint32_t width = kReduceSegs/4u;width >= 1u;width /= 4u)
    {
        float4 tot = make_float4(0.f, 0.f, 0.f, 0.f);
        const bool on = seg < width;
        if(on)
        {
            tot = sm[seg*4u][col];
            #pragma unroll
            for(uint32_t k = 1;k < 4u;++k)
            {
                const float4 a = sm[seg*4u + k][col];
                tot.x += a.x; tot.y += a.y; tot.z += a.z; tot.w += a.w;
            }
        }
        __syncthreads();
        if(on) sm[seg][col] = tot;
        __syncthreads();
        if(width == 2u) break;
    }
    float4 tot = make_float4(0.f, 0.f, 0.f, 0.f);
    if(seg == 0)
    {
        tot = sm[0][col];
        const float4 b = sm[1][col];
        tot.x += b.x; tot.y += b.y; tot.z += b.z; tot.w += b.w;
    }
    return tot;
}

__global__ void __launch_bounds__(1024)
k_reduce_rows(const float *__restrict__ partial, uint32_t rows, uint32_t len,
    float *__restrict__ out, int accumulate)
{
    __shared__ float4 sm[kReduceSegs][kReduceCols];
    const uint32_t e4 = blockIdx.x*kReduceCols + (threadIdx.x & (kReduceCols-1));
    float4 tot = reduce_rows_cta(partial, rows, len, e4, e4*4u < len, sm);
    if(threadIdx.x < kReduceCols && e4*4u < len)
    {
        float4 *o = reinterpret_cast<float4*>(out) + e4;
        if(accumulate)
        {
            const float4 a = *o;
            tot.x += a.x; tot.y += a.y; tot.z += a.z; tot.w += a.w;
        }
        *o = tot;
    }
}

// The same sum for a handful of long rows (the chunk partials of k_send_mix: <= 16 rows of
// slots x channels x 1024 floats): one float4 column per thread, all rows' loads in flight at
// once, added with exactly the association k_reduce_rows' tree has for rows <= 16 (groups of
// four rows in order, then the groups in order), so both kernels give bit-identical results.
__global__ void __launch_bounds__(256)
k_reduce_few(const float *__restrict__ partial, uint32_t rows, uint32_t len,
    float *__restrict__ out, int accumulate)
{
    const uint32_t e4 = blockIdx.x*blockDim.x + threadIdx.x;
    if(e4*4u >= len) return;
    const float4 *p = reinterpret_cast<const float4*>(partial) + e4;
    const size_t stride4 = len/4u;
    float4 v[16];
    #pragma unroll
    for(uint32_t r = 0;r < 16u;++r)
        v[r] = r < rows ? __ldg(p + size_t(r)*stride4) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 g[4];
    #pragma unroll
    for(uint32_t j = 0;j < 4u;++j)
    {
        float4 t = v[4u*j];
        #pragma unroll
        for(uint32_t k = 1;k < 4u;++k)
        { t.x += v[4u*j+k].x; t.y += v[4u*j+k].y; t.z += v[4u*j+k].z; t.w += v[4u*j+k].w; }
        g[j] = t;
    }
    float4 tot = g[0];
    #pragma unroll
    for(uint32_t j = 1;j < 4u;++j) { tot.x += g[j].x; tot.y += g[j].y; tot.z += g[j].z; tot.w += g[j].w; }
    float4 *o = reinterpret_cast<float4*>(out) + e4;
    if(accumulate)
    {
        const float4 a = *o;
        tot.x += a.x; tot.y += a.y; tot.z += a.z; tot.w += a.w;
    }
    *o = tot;
}

// Applies staged parameter snapshots to the voice records (the device half of
// b200mix_voices_update).  One CTA of 64 threads per update.
struct ApplyParams {
    VoiceRec *voices; const VoiceUpdate *updates;
    const float *coeffs; const float *dry; const float *send;   // staged side arrays (or null)
    float2 *hrtf_tgt; float2 *hrtf_old; float *dry_cur, *dry_tgt, *send_cur, *send_tgt;
    uint32_t ir, ir_pad, cd, cw, num_sends;
    FilterRec *filt; uint32_t filt_paths;
    // device-side HrtfStore::getCoeffs (b200mix_voices_update_dirs): per update
    // {elevation, azimuth, distance, spread}; the attached data set
    const float4 *dirs;
    const float2 *st_fields;     // {distance, ev_count as float bits}
    const uint2 *st_elevs;       // {az_count, ir_offset}
    const float2 *st_coeffs;     // [ir_count][st_ir]
    const uint8_t *st_delays;    // [ir_count][2]
    uint32_t st_num_fields, st_ir;
    uint4 *qhdr;                 // streaming queues (null: none): a restart rewinds the head
    // direct-channel voices (null until the first b200mix_voices_update_direct): staged RealOut
    // gains [n][creal], Current / Target [max_voices][creal]
    const float *real; float *real_cur, *real_tgt; uint32_t creal;
};

// HrtfStore::getCoeffs (core/hrtf.cpp:192-260) on the device, in the exact operation order of
// the host restatement (csrc/hrtf_store.cpp: b200mix_hrtf_get_coeffs) with explicit
// round-to-nearest mul/add, so both give bit-identical HRIRs and delays.
struct HrirBlend { uint32_t idx[4]; float w[4]; float passthru; uint32_t delay[2]; };

__device__ __forceinline__ void hrir_index(uint32_t count, float v, bool elev, uint32_t &idx, float &blend)
{
    const float inv_pi = 0.318309886183790671538f;
    if(elev)
    {
        v = __fmul_rn(__fadd_rn(__fmul_rn(inv_pi, v), 0.5f), float(count-1u));
        const uint32_t i = v > 0.0f ? uint32_t(v) : 0u;
        idx = min(i, count-1u); blend = __fsub_rn(v, float(i));
    }
    else
    {
        v = __fmul_rn(__fadd_rn(__fmul_rn(inv_pi*0.5f, v), 1.0f), float(count));
        const uint32_t i = v > 0.0f ? uint32_t(v) : 0u;
        idx = i % count; blend = __fsub_rn(v, float(i));
    }
}

__device__ __forceinline__ void hrir_blend(const ApplyParams &A, const float4 dir, HrirBlend &B)
{
    const float inv_pi = 0.318309886183790671538f;
    const float elevation = dir.x, azimuth = dir.y, distance = dir.z, spread = dir.w;
    const float dirfact = __fsub_rn(1.0f, __fmul_rn(inv_pi/2.0f, spread));
    uint32_t ebase = 0, fi = 0;
    for(;fi + 1u < A.st_num_fields;++fi)
    {
        if(distance >= A.st_fields[fi].x) break;
        ebase += __float_as_uint(A.st_fields[fi].y);
    }
    const uint32_t evCount = __float_as_uint(A.st_fields[fi].y);
    uint32_t e0i; float e0b;
    hrir_index(evCount, elevation, true, e0i, e0b);
    const uint32_t e1i = min(e0i + 1u, evCount - 1u);
    const uint2 el0 = A.st_elevs[ebase + e0i], el1 = A.st_elevs[ebase + e1i];
    uint32_t a0i, a1i; float a0b, a1b;
    hrir_index(el0.x, azimuth, false, a0i, a0b);
    hrir_index(el1.x, azimuth, false, a1i, a1b);
    B.idx[0] = el0.y + a0i; B.idx[1] = el0.y + ((a0i + 1u) % el0.x);
    B.idx[2] = el1.y + a1i; B.idx[3] = el1.y + ((a1i + 1u) % el1.x);
    const float ne = __fsub_rn(1.0f, e0b);
    B.w[0] = __fmul_rn(__fmul_rn(ne, __fsub_rn(1.0f, a0b)), dirfact);
    B.w[1] = __fmul_rn(__fmul_rn(ne, a0b), dirfact);
    B.w[2] = __fmul_rn(__fmul_rn(e0b, __fsub_rn(1.0f, a1b)), dirfact);
    B.w[3] = __fmul_rn(__fmul_rn(e0b, a1b), dirfact);
    #pragma unroll
    for(int ear = 0;ear < 2;++ear)
    {
        float dsum = __fmul_rn(float(A.st_delays[B.idx[0]*2u + ear]), B.w[0]);
        dsum = __fadd_rn(dsum, __fmul_rn(float(A.st_delays[B.idx[1]*2u + ear]), B.w[1]));
        dsum = __fadd_rn(dsum, __fmul_rn(float(A.st_delays[B.idx[2]*2u + ear]), B.w[2]));
        dsum = __fadd_rn(dsum, __fmul_rn(float(A.st_delays[B.idx[3]*2u + ear]), B.w[3]));
        B.delay[ear] = uint32_t(__float2int_rn(__fmul_rn(dsum, 0.25f)));
    }
    B.passthru = __fmul_rn(0.70710678118654752440f, __fsub_rn(1.0f, dirfact));
}

// BiquadInterpFilter::reset (biquad.h:144-150) for one record; lane k < 32 writes word k.
__device__ __forceinline__ void filter_reset_word(FilterRec *fr, int k)
{
    uint32_t *w = reinterpret_cast<uint32_t*>(fr);
    uint32_t val = 0u;
    if(k == 0 || k == 5 || k == 10 || k == 15) val = __float_as_uint(1.0f);   // b0 of cur/tgt
    else if(k == 24 || k == 25) val = 0xffffffffu;                             // mCounter = -1
    w[k] = val;
}

// b200mix_voice_queue: installs a voice's buffer list (items by value in the launch
// parameters) and keeps VoiceFlag "has a current buffer" in step with it.
struct QueueSet { uint32_t voice, count, loop; uint32_t items[kMaxQueue]; };
__global__ void k_set_queue(VoiceRec *voices, uint4 *qhdr, uint32_t *queue, const QueueSet Q)
{
    const uint32_t t = threadIdx.x;
    if(t < Q.count) queue[size_t(Q.voice)*kMaxQueue + t] = Q.items[t];
    if(t == 0)
    {
        qhdr[Q.voice] = make_uint4(Q.count, 0u, Q.loop, 0u);
        uint32_t fl = voices[Q.voice].flags;
        fl = Q.count ? (fl | kVfHaveBuffer) : (fl & ~kVfHaveBuffer);
        voices[Q.voice].flags = fl;
    }
}

__global__ void k_filter_init(FilterRec *filt, size_t count)
{
    const size_t i = size_t(blockIdx.x)*blockDim.x + threadIdx.x;
    if(i < count*32u) filter_reset_word(filt + (i >> 5), int(i & 31u));
}

// The device half of b200mix_voices_filters: BiquadInterpFilter::setParams once
// SetParams has produced the new targets (biquad.cpp:36-43,123-147).
__global__ void k_apply_filter_updates(FilterRec *filt, uint32_t paths, const FilterUpdate *upd,
    uint32_t n)
{
    const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
    if(i >= n*2u) return;
    const FilterUpdate &u = upd[i >> 1];
    const int f = int(i & 1u);
    FilterRec &fr = filt[size_t(u.voice)*paths + u.path];
    const float *nt = f ? u.hp : u.lp;
    bool diff = false;
    #pragma unroll
    for(int k = 0;k < 5;++k)
    {
        diff |= !(fabsf(nt[k] - fr.tgt[f][k]) <= 0.015625f);          // check_set
        fr.tgt[f][k] = nt[k];
    }
    const int c = fr.counter[f];
    if(!diff)
    {
        if(c <= 0)
        {
            fr.counter[f] = 0;
            #pragma unroll
            for(int k = 0;k < 5;++k) fr.cur[f][k] = nt[k];
        }
    }
    else if(c >= 0) fr.counter[f] = 8*32;                            // InterpSteps*SamplesPerStep
    else
    {
        fr.counter[f] = 0;
        #pragma unroll
        for(int k = 0;k < 5;++k) fr.cur[f][k] = nt[k];
    }
    if(f == 0) fr.active = u.active ? 1u : 0u;
}

__global__ void __launch_bounds__(64) k_apply_updates(const ApplyParams A)
{
    const uint32_t u = blockIdx.x;
    const VoiceUpdate up = A.updates[u];
    VoiceRec &rec = A.voices[up.voice];
    const int t = threadIdx.x;
    const bool reset = (up.flags & (1u<<5)) != 0;
    const uint32_t oldFlags = reset ? 0u : rec.flags;
    const bool wasDirty = (oldFlags & kVfCoefDirty) != 0;
    __syncthreads();
    if(reset)
    {
        for(int k = t;k < kPad;k += 64) rec.prev[k] = 0.0f;
        for(int k = t;k < kHist;k += 64) rec.hist[k] = 0.0f;
        if(A.dry_cur) for(uint32_t c = t;c < A.cd;c += 64) A.dry_cur[size_t(up.voice)*A.cd + c] = 0.0f;
        if(A.send_cur)
            for(uint32_t c = t;c < A.num_sends*A.cw;c += 64)
                A.send_cur[size_t(up.voice)*A.num_sends*A.cw + c] = 0.0f;
        if(A.real_cur) for(uint32_t c = t;c < A.creal;c += 64) A.real_cur[size_t(up.voice)*A.creal + c] = 0.0f;
        if(A.filt)          // chandata.mDryParams = DirectParams{}; mWetParams = SendParams{} (voice.cpp:1387-1394)
            for(uint32_t k = t;k < A.filt_paths*32u;k += 64)
                filter_reset_word(A.filt + size_t(up.voice)*A.filt_paths + (k >> 5), int(k & 31u));
    }
    __shared__ HrirBlend sB;
    const bool fromDirs = A.dirs != nullptr && up.has_coeffs && A.hrtf_tgt;
    if(fromDirs)
    {
        if(t == 0) hrir_blend(A, A.dirs[u], sB);
        __syncthreads();
    }
    if(up.has_coeffs && A.hrtf_tgt)
    {
        float2 *tg = A.hrtf_tgt + size_t(up.voice)*A.ir_pad;
        float2 *ol = A.hrtf_old + size_t(up.voice)*A.ir_pad;
        const float *src = fromDirs ? nullptr : A.coeffs + size_t(u)*A.ir*2;
        for(uint32_t k = t;k < A.ir_pad;k += 64)
        {
            // keep "old" = the filter used by the last mix unless a newer target is
            // already pending (see DESIGN.md §3.6)
            if(!wasDirty && !reset) ol[k] = tg[k];
            float2 val = make_float2(0.f, 0.f);
            if(fromDirs)
            {
                if(k < A.st_ir && k < A.ir)
                {
                    val = (k == 0) ? make_float2(sB.passthru, sB.passthru) : val;
                    #pragma unroll
                    for(int c = 0;c < 4;++c)
                    {
                        const float2 sv = A.st_coeffs[size_t(sB.idx[c])*A.st_ir + k];
                        val.x = __fadd_rn(__fmul_rn(sv.x, sB.w[c]), val.x);
                        val.y = __fadd_rn(__fmul_rn(sv.y, sB.w[c]), val.y);
                    }
                }
            }
            else if(k < A.ir) val = make_float2(src[k*2], src[k*2+1]);
            tg[k] = val;
        }
    }
    if(up.has_dry && A.dry_tgt)
        for(uint32_t c = t;c < A.cd;c += 64)
            A.dry_tgt[size_t(up.voice)*A.cd + c] = A.dry[size_t(u)*A.cd + c];
    // The reference's voice has one mDryParams.Gains.Current, indexed by the channels of whichever
    // buffer its direct path feeds: a voice moved between Dry and RealOut carries the shared
    // channel indices' Current gains across; the others keep what they had.
    if(!reset && A.real_cur && ((oldFlags ^ up.flags) & kVfDirect))
    {
        float *dc = A.dry_cur + size_t(up.voice)*A.cd, *rc = A.real_cur + size_t(up.voice)*A.creal;
        const bool toReal = (up.flags & kVfDirect) != 0;
        for(uint32_t c = t;c < min(A.cd, A.creal);c += 64)
        {
            if(toReal) rc[c] = dc[c];
            else dc[c] = rc[c];
        }
    }
    if(A.real)
        for(uint32_t c = t;c < A.creal;c += 64)
            A.real_tgt[size_t(up.voice)*A.creal + c] = A.real[size_t(u)*A.creal + c];
    if(A.send && A.send_tgt)
        for(uint32_t c = t;c < A.num_sends*A.cw;c += 64)
            A.send_tgt[size_t(up.voice)*A.num_sends*A.cw + c] = A.send[size_t(u)*A.num_sends*A.cw + c];
    if(t == 0)
    {
        uint32_t fl = up.flags & (kVfStatic|kVfLooping|kVfHrtf|kVfChannelMask|kVfDirect);
        if(reset)
        {
            rec.pos = up.position; rec.frac = up.position_frac;
            fl |= kVfHaveBuffer;
            if(up.flags & (1u<<6)) fl |= kVfFading;
            rec.old_delay0 = 0; rec.old_delay1 = 0; rec.old_gain = 0.0f;
            if(A.qhdr) A.qhdr[up.voice].y = 0u;
        }
        else
        {
            fl |= oldFlags & (kVfFading|kVfHaveBuffer|kVfCoefDirty);
        }
        if(up.has_coeffs && !reset) fl |= kVfCoefDirty;
        if(up.flags & kUpNoBuffer) fl &= ~kVfHaveBuffer;
        rec.flags = fl;
        if(up.flags & (1u<<7)) rec.state = 0u;
        else if(up.flags & (1u<<1)) rec.state = 2u;
        else if(up.flags & (1u<<0)) rec.state = 1u;
        rec.buffer = up.buffer; rec.resampler = up.resampler;
        rec.loop_start = up.loop_start; rec.loop_end = up.loop_end; rec.step = up.step;
        rec.bsinc_sf = up.bsinc_sf; rec.bsinc_m = up.bsinc_m; rec.bsinc_l = up.bsinc_l;
        rec.bsinc_off = up.bsinc_off;
        rec.tgt_delay0 = fromDirs ? sB.delay[0] : up.delay0;
        rec.tgt_delay1 = fromDirs ? sB.delay[1] : up.delay1;
        rec.tgt_gain = up.gain;
        uint32_t mask = 0;
        for(int s = 0;s < kMaxSends;++s)
        {
            rec.send_slot[s] = up.send_slot[s];
            if(up.send_slot[s] != 0xffffffffu) mask |= 1u<<s;
        }
        rec.send_mask = mask;
    }
}

// Post-process for HRTF output (DeviceBase::Process(HrtfPostProcess), alc/alu.cpp:289-298
// -> MixDirectHrtfBase, hrtfbase.h:91-133).
struct PostHrtfParams {
    const float *partial;        // [rows][2][kAccumLen] the HRIR FIR's partial rows
    uint32_t rows;
    const float *carry_in;       // [2][kHrirLen]  accumulator tail from the last update
    float *carry_out;            // [2][kHrirLen]
    const float *dry;            // [cd][1024]
    float *real;                 // [real][1024]
    const float2 *dec_coef;      // [cd][dec_ir]
    const float *dec_hfscale; float *dec_state;   // state: [cd][4] = coeff, lp_z1, lp_z2, ap_z1
    float *temp;                 // [cd][1024] band-split dry
    uint32_t frames, cd, dec_ir, real_left, real_right, dry_active;
    uint32_t overwrite;          // RealOut L/R were not cleared: store instead of accumulate
};

// Stage 1 (only when the dry mix is non-silent): BandSplitter::processHfScale per dry
// channel (core/filters/splitter.cpp:64-95) — a serial recurrence.  One warp per channel:
// the lanes stage the line through shared memory (coalesced), lane 0 runs the recurrence
// with 8-sample register batches so the loads/stores stay off the dependency chain.
__global__ void __launch_bounds__(32) k_post_hrtf_split(const PostHrtfParams Q)
{
    __shared__ float line[kLine];
    const uint32_t c = blockIdx.x;
    if(c >= Q.cd) return;
    const uint32_t lane = threadIdx.x, n = Q.frames;
    const float *in = Q.dry + size_t(c)*kLine;
    float *out = Q.temp + size_t(c)*kLine;
    for(uint32_t i = lane;i < kLine;i += 32) line[i] = (i < n) ? in[i] : 0.0f;
    __syncwarp();
    if(lane == 0)
    {
        float *st = Q.dec_state + c*4;
        const float ap_coeff = st[0];
        const float lp_coeff = st[0]*0.5f + 0.5f;
        float lp_z1 = st[1], lp_z2 = st[2], ap_z1 = st[3];
        const float hfscale = Q.dec_hfscale[c];
        for(uint32_t i0 = 0;i0 < n;i0 += 8)
        {
            float x[8], y[8];
            #pragma unroll
            for(int k = 0;k < 8;++k) x[k] = line[i0+k];
            #pragma unroll
            for(int k = 0;k < 8;++k)
            {
                const float d0 = (x[k] - lp_z1) * lp_coeff;
                const float lp_y0 = lp_z1 + d0;
                const float nz1 = lp_y0 + d0*lp_coeff;
                const float d1 = (lp_y0 - lp_z2) * lp_coeff;
                const float lp_y1 = lp_z2 + d1;
                const float nz2 = lp_y1 + d1;
                const float ap_y = x[k]*ap_coeff + ap_z1;
                const float naz = x[k] - ap_y*ap_coeff;
                y[k] = (ap_y-lp_y1)*hfscale + lp_y1;
                if(i0 + k < n) { lp_z1 = nz1; lp_z2 = nz2; ap_z1 = naz; }
            }
            #pragma unroll
            for(int k = 0;k < 8;++k) line[i0+k] = y[k];
        }
        st[1] = lp_z1; st[2] = lp_z2; st[3] = ap_z1;
    }
    __syncwarp();
    for(uint32_t i = lane;i < n;i += 32) out[i] = line[i];
}

// Stage 2: total[t] = carry[t] + voices[t] + decoder FIR of the dry channels;
// RealOut L/R (+)= total[0..n); carry_out = total[n..n+128).
// voices[t] is the sum of the HRIR FIR's partial rows, summed here with k_reduce_rows' tree for
// (rows, 2*kAccumLen), so it is the same float as that kernel would store.  grid (tiles of 32
// outputs, ear), 1024 threads: the row sum first (8 float4 columns x 128 row segments), then
// thread (output o = tid % 32, channel c = tid / 32) runs channel c's decoder FIR for output o,
// and the 32 channel sums are added to the total in channel order.
constexpr uint32_t kPostTile = kReduceCols*4u, kPostMaxDry = 32u;   // B200MIX_MAX_DRY_CHANNELS
static_assert(kAccumLen % kPostTile == 0, "a tile lies within one ear's accumulator");
static_assert(kPostMaxDry*kPostTile <= 1024u, "one thread per (channel, output)");
__global__ void __launch_bounds__(1024, 1) k_post_hrtf_reduce(const PostHrtfParams Q)
{
    __shared__ float4 sm[kReduceSegs][kReduceCols];
    __shared__ float vsum[kPostTile];
    __shared__ float dsum[kPostMaxDry][kPostTile];
    const uint32_t span = Q.frames + kHrirLen;
    const uint32_t ear = blockIdx.y;
    const uint32_t t0 = blockIdx.x*kPostTile;
    // the FIR's partial rows (and, launched right behind it, everything it wrote) are complete
    griddep_wait();
    const uint32_t col = threadIdx.x & (kReduceCols-1);
    const uint32_t e4 = (ear*kAccumLen + t0)/4u + col;
    const float4 v = reduce_rows_cta(Q.partial, Q.rows, 2u*kAccumLen, e4, t0 + 4u*col < span, sm);
    if(threadIdx.x < kReduceCols)
    { vsum[4*col] = v.x; vsum[4*col + 1] = v.y; vsum[4*col + 2] = v.z; vsum[4*col + 3] = v.w; }

    const uint32_t o = threadIdx.x % kPostTile, c = threadIdx.x / kPostTile;
    const uint32_t tt = t0 + o;
    if(Q.dry_active && c < Q.cd)
    {
        const float *x = Q.temp + size_t(c)*kLine;
        const float2 *cg = Q.dec_coef + size_t(c)*Q.dec_ir;
        float s = 0.0f;
        for(uint32_t j = 0;j < Q.dec_ir;++j)           // dec_ir <= kHrirLen
        {
            const int src = int(tt) - int(j);
            const float xv = (src >= 0 && src < int(Q.frames)) ? x[src] : 0.0f;
            s = fmaf(ear ? cg[j].y : cg[j].x, xv, s);
        }
        dsum[c][o] = s;
    }
    __syncthreads();
    if(threadIdx.x >= kPostTile || tt >= span) return;
    float tot = vsum[o];
    if(tt < uint32_t(kHrirLen)) tot += Q.carry_in[ear*kHrirLen + tt];
    if(Q.dry_active)
        for(uint32_t ch = 0;ch < Q.cd;++ch) tot += dsum[ch][o];
    if(tt < Q.frames)
    {
        float *out = Q.real + size_t(ear ? Q.real_right : Q.real_left)*kLine + tt;
        *out = Q.overwrite ? tot : (*out + tot);
    }
    else
        Q.carry_out[ear*kHrirLen + (tt - Q.frames)] = tot;
}

// BFormatDec::process, single band (core/bformatdec.cpp:85-95): real[o] += G[c][o]*dry[c],
// summed in channel order like the reference's MixSamples loop.
struct PostAmbiParams {
    const float *dry; float *real; const float *gains_hf; const float *gains_lf;
    float *split_state; float *temp_hf; float *temp_lf;
    uint32_t frames, cd, real_channels, dual;
};

__global__ void k_post_ambi_split(const PostAmbiParams Q)
{
    // BandSplitter::process, core/filters/splitter.cpp:28-62 (dual-band decoders)
    const uint32_t c = blockIdx.x*blockDim.x + threadIdx.x;
    if(c >= Q.cd) return;
    float *st = Q.split_state + c*4;
    const float ap_coeff = st[0];
    const float lp_coeff = st[0]*0.5f + 0.5f;
    float lp_z1 = st[1], lp_z2 = st[2], ap_z1 = st[3];
    const float *in = Q.dry + size_t(c)*kLine;
    float *hp = Q.temp_hf + size_t(c)*kLine, *lp = Q.temp_lf + size_t(c)*kLine;
    for(uint32_t i = 0;i < Q.frames;++i)
    {
        const float x = in[i];
        const float d0 = (x - lp_z1) * lp_coeff;
        const float lp_y0 = lp_z1 + d0;
        lp_z1 = lp_y0 + d0;
        const float d1 = (lp_y0 - lp_z2) * lp_coeff;
        const float lp_y1 = lp_z2 + d1;
        lp_z2 = lp_y1 + d1;
        lp[i] = lp_y1;
        const float ap_y = x*ap_coeff + ap_z1;
        ap_z1 = x - ap_y*ap_coeff;
        hp[i] = ap_y - lp_y1;
    }
    st[1] = lp_z1; st[2] = lp_z2; st[3] = ap_z1;
}

__global__ void __launch_bounds__(128) k_post_ambi_mix(const PostAmbiParams Q)
{
    const uint32_t idx = blockIdx.x*blockDim.x + threadIdx.x;   // [out][i]
    if(idx >= Q.real_channels*Q.frames) return;
    const uint32_t o = idx / Q.frames, i = idx - o*Q.frames;
    float acc = Q.real[size_t(o)*kLine + i];
    for(uint32_t c = 0;c < Q.cd;++c)
    {
        if(Q.dual)
        {
            const float gh = Q.gains_hf[c*Q.real_channels + o];
            const float gl = Q.gains_lf[c*Q.real_channels + o];
            if(fabsf(gh) > kSilence) acc += Q.temp_hf[size_t(c)*kLine + i]*gh;
            if(fabsf(gl) > kSilence) acc += Q.temp_lf[size_t(c)*kLine + i]*gl;
        }
        else
        {
            const float gh = Q.gains_hf[c*Q.real_channels + o];
            if(fabsf(gh) > kSilence) acc += Q.dry[size_t(c)*kLine + i]*gh;
        }
    }
    Q.real[size_t(o)*kLine + i] = acc;
}

// UhjEncoderIIR::encode (core/uhjfilter.cpp:231-283): five 4-stage all-pass chains
// (core/allpass_iir.hpp:53-70), each a serial recurrence -> one thread per chain, then
// the whole block combines.  state: [5 chains][4 stages][2] + 4 delay samples.
// The two stereo matrix encoders share their structure and differ in constants and in the Dry
// channels they read: UhjEncoder* (core/uhjfilter.cpp:59-70; Dry 0,1,2 = W,X,Y) and TsmeEncoder*
// (core/tsmefilter.cpp:156-163,289-309; Dry 0,1,2,3 = W,Y,Z,X).  S = sw W + sx X [+ sz Z],
// D = j(dw W + dx X) + dy Y, Left = S + D, Right = S - D.
struct MatrixEncSpec { uint32_t w, x, y, z; float sw, sx, sz, dw, dx, dy; };   // z = ~0u: none
constexpr MatrixEncSpec kUhjEncSpec{0u, 1u, 2u, ~0u, 0.4698463f, 0.0757602682546f, 0.0f,
    -0.17101005f, 0.208149636675f, 0.267586995182f};
constexpr MatrixEncSpec kTsmeEncSpec{0u, 3u, 1u, 2u, 0.288397341271f, 0.166565447888f, 0.187684284734f,
    0.444008050325f, -0.256439256487f, 0.333238912931f};

struct PostUhjParams {
    const float *dry; float *real; float *state; float *scratch;   // scratch: not read (null)
    uint32_t frames, real_left, real_right;
    MatrixEncSpec enc;
};

__global__ void __launch_bounds__(1024) k_post_uhj(const PostUhjParams Q)
{
    constexpr float F1[4] = {0.479400865589f, 0.876218493539f, 0.976597589508f, 0.997499255936f};
    constexpr float F2[4] = {0.161758498368f, 0.733028932341f, 0.945349700329f, 0.990599156684f};
    // chain inputs and outputs live in shared memory: the serial recurrences never wait on
    // a global load (row stride 1025+8 keeps the five chain threads on different banks)
    constexpr int kRow = kLine + 9;
    __shared__ float sIn[5][kRow];
    __shared__ float sOut[5][kRow];
    const uint32_t n = Q.frames;
    const MatrixEncSpec E = Q.enc;
    const float *w = Q.dry + size_t(E.w)*kLine, *x = Q.dry + size_t(E.x)*kLine, *y = Q.dry + size_t(E.y)*kLine;
    const float *z = E.z != ~0u ? Q.dry + size_t(E.z)*kLine : nullptr;
    float *left = Q.real + size_t(Q.real_left)*kLine, *right = Q.real + size_t(Q.real_right)*kLine;
    for(uint32_t k = threadIdx.x;k < n;k += blockDim.x)
    {
        const float wk = w[k], xk = x[k];
        float sv = E.sw*wk + E.sx*xk;
        if(z) sv = sv + E.sz*z[k];
        sIn[0][k] = sv;
        sIn[1][k] = E.dw*wk + E.dx*xk;
        sIn[2][k] = y[k];
        sIn[3][k] = left[k];
        sIn[4][k] = right[k];
    }
    __syncthreads();
    // one warp per chain so the five chains run on five schedulers' worth of issue slots
    const int chain = threadIdx.x >> 5;
    if(chain < 5 && (threadIdx.x & 31) == 0)
    {
        float *st = Q.state + chain*8;
        float z0[4], z1[4], c[4];
        #pragma unroll
        for(int i = 0;i < 4;++i) { z0[i] = st[i*2]; z1[i] = st[i*2+1]; c[i] = chain == 1 ? F2[i] : F1[i]; }
        // the Filter1 chains are delayed by one sample: out[0] is last update's final output
        const int off = chain == 1 ? 0 : 1;
        const float *src = sIn[chain];
        float *dst = sOut[chain] + off;
        #pragma unroll 4
        for(uint32_t k = 0;k < n;++k)
        {
            float v = src[k];
            #pragma unroll
            for(int i = 0;i < 4;++i)
            {
                const float yy = v*c[i] + z0[i];
                z0[i] = z1[i];
                z1[i] = yy*c[i] - v;
                v = yy;
            }
            dst[k] = v;
        }
        #pragma unroll
        for(int i = 0;i < 4;++i) { st[i*2] = z0[i]; st[i*2+1] = z1[i]; }
        float *delay = Q.state + 40;
        const int di = chain == 0 ? 0 : chain == 2 ? 1 : chain == 3 ? 2 : 3;
        if(chain != 1) { sOut[chain][0] = delay[di]; delay[di] = sOut[chain][n]; }
    }
    __syncthreads();
    for(uint32_t i = threadIdx.x;i < n;i += blockDim.x)
    {
        const float dd = sOut[1][i] + E.dy*sOut[2][i];
        left[i] = sOut[0][i] + dd + sOut[3][i];
        right[i] = sOut[0][i] - dd + sOut[4][i];
    }
}

// Front image stabilizer after the ambisonic decode (StablizerPostProcess, alc/alu.cpp:330-406).
// RealOut holds only the decode here (nothing mixes into it directly), so the "direct" mid/side
// signals the reference moves out of the way first are zero and the left channel's all-pass
// (which only ever sees that zero mid signal) keeps a zero state.  One warp per serial filter:
// warp 0 the mid band splitter (BandSplitter::process), warp 1 the side signal's all-pass
// (ChannelFilters[right]), warps 2.. the all-pass of every other output channel
// (BandSplitter::processAllPass); rows staged in shared memory, operations in the reference's
// order with explicit rounding.  state: [0..2] MidFilter lp_z1, lp_z2, ap_z1; [4+i] mApZ1 of
// ChannelFilters[i].
struct StabParams {
    float *real; float *state;
    uint32_t frames, real_channels, lidx, ridx, cidx;
    float coeff;
    float mid_lf, mid_hf, center_lf, center_hf;   // cos/sin(1/3 * pi/2), cos/sin(1/4 * pi/2) by the host libm
};

__global__ void __launch_bounds__(1024) k_post_stabilizer(const StabParams Q)
{
    extern __shared__ float sRows[];            // [2 + real_channels][kLine]: tmp->LF, HF, side, others
    const uint32_t n = Q.frames, C = Q.real_channels;
    float *left = Q.real + size_t(Q.lidx)*kLine, *right = Q.real + size_t(Q.ridx)*kLine;
    float *rowLF = sRows, *rowHF = sRows + kLine, *rowSide = sRows + 2*kLine;
    for(uint32_t k = threadIdx.x;k < n;k += blockDim.x)
    {
        const float l = left[k], r = right[k];
        rowLF[k] = __fadd_rn(l, r);             // the decoded mid signal (splitter input)
        rowSide[k] = __fadd_rn(0.0f, __fsub_rn(l, r));   // side[i] (= 0) += leftout - rightout
    }
    // the other channels, in output-channel order, rows 3..
    uint32_t other = 0;
    for(uint32_t c = 0;c < C;++c)
    {
        if(c == Q.lidx || c == Q.ridx) continue;
        float *row = sRows + size_t(3u + other)*kLine;
        const float *src = Q.real + size_t(c)*kLine;
        for(uint32_t k = threadIdx.x;k < n;k += blockDim.x) row[k] = src[k];
        ++other;
    }
    __syncthreads();

    const uint32_t chain = threadIdx.x >> 5;
    const float coeff = Q.coeff;
    if((threadIdx.x & 31u) == 0u && chain < C)
    {
        if(chain == 0)
        {
            const float lp_coeff = __fadd_rn(__fmul_rn(coeff, 0.5f), 0.5f);
            float lp_z1 = Q.state[0], lp_z2 = Q.state[1], ap_z1 = Q.state[2];
            uint32_t k = 0;
            for(;k < n;)
            {
                float x[8];
                const uint32_t m = min(8u, n - k);
                #pragma unroll
                for(uint32_t j = 0;j < 8u;++j) x[j] = j < m ? rowLF[k + j] : 0.0f;
                #pragma unroll
                for(uint32_t j = 0;j < 8u;++j)
                {
                    if(j < m)
                    {
                        const float d0 = __fmul_rn(__fsub_rn(x[j], lp_z1), lp_coeff);
                        const float lp_y0 = __fadd_rn(lp_z1, d0);
                        lp_z1 = __fadd_rn(lp_y0, d0);
                        const float d1 = __fmul_rn(__fsub_rn(lp_y0, lp_z2), lp_coeff);
                        const float lp_y1 = __fadd_rn(lp_z2, d1);
                        lp_z2 = __fadd_rn(lp_y1, d1);
                        const float ap_y = __fadd_rn(__fmul_rn(x[j], coeff), ap_z1);
                        ap_z1 = __fsub_rn(x[j], __fmul_rn(ap_y, coeff));
                        rowLF[k + j] = lp_y1;
                        rowHF[k + j] = __fsub_rn(ap_y, lp_y1);
                    }
                }
                k += m;
            }
            Q.state[0] = lp_z1; Q.state[1] = lp_z2; Q.state[2] = ap_z1;
        }
        else
        {
            // chain 1: side with ChannelFilters[ridx]; chain 2+o: other channel o with its own
            uint32_t ch = Q.ridx;
            float *row = rowSide;
            if(chain >= 2u)
            {
                uint32_t o = chain - 2u, c = 0;
                for(;c < C;++c)
                {
                    if(c == Q.lidx || c == Q.ridx) continue;
                    if(o == 0u) break;
                    --o;
                }
                ch = c;
                row = sRows + size_t(3u + (chain - 2u))*kLine;
            }
            float z1 = Q.state[4u + ch];
            uint32_t k = 0;
            for(;k < n;)
            {
                float x[8];
                const uint32_t m = min(8u, n - k);
                #pragma unroll
                for(uint32_t j = 0;j < 8u;++j) x[j] = j < m ? row[k + j] : 0.0f;
                #pragma unroll
                for(uint32_t j = 0;j < 8u;++j)
                {
                    if(j < m)
                    {
                        const float y = __fadd_rn(__fmul_rn(x[j], coeff), z1);
                        z1 = __fsub_rn(x[j], __fmul_rn(y, coeff));
                        row[k + j] = y;
                    }
                }
                k += m;
            }
            Q.state[4u + ch] = z1;
        }
    }
    __syncthreads();

    // pan the mid bands between centre and left+right (alc/alu.cpp:380-405)
    const float mid_lf = Q.mid_lf, mid_hf = Q.mid_hf, center_lf = Q.center_lf, center_hf = Q.center_hf;
    float *center = Q.real + size_t(Q.cidx)*kLine;
    const float *rowCenter = nullptr;
    other = 0;
    for(uint32_t c = 0;c < C;++c)
    {
        if(c == Q.lidx || c == Q.ridx) continue;
        float *row = sRows + size_t(3u + other)*kLine;
        if(c == Q.cidx) rowCenter = row;
        else
        {
            float *dst = Q.real + size_t(c)*kLine;
            for(uint32_t k = threadIdx.x;k < n;k += blockDim.x) dst[k] = row[k];
        }
        ++other;
    }
    for(uint32_t k = threadIdx.x;k < n;k += blockDim.x)
    {
        const float lf = rowLF[k], hf = rowHF[k];
        const float m = __fadd_rn(__fadd_rn(__fmul_rn(lf, mid_lf), __fmul_rn(hf, mid_hf)), 0.0f);
        const float cc = __fadd_rn(__fmul_rn(lf, center_lf), __fmul_rn(hf, center_hf));
        const float sd = rowSide[k];
        left[k] = __fmul_rn(__fadd_rn(m, sd), 0.5f);
        right[k] = __fmul_rn(__fsub_rn(m, sd), 0.5f);
        center[k] = __fadd_rn(rowCenter[k], __fmul_rn(cc, 0.5f));
    }
}

// BS2B crossfeed after the ambisonic decode (Bs2bPostProcess, alc/alu.cpp:408-434):
// bs2b_processor::cross_feed (core/bs2b.cpp:104-163) on FrontLeft/FrontRight.  Four first-order
// recurrences (a high-shelf "direct" and a low-pass "crossfeed" path per input channel), one
// thread each on its own warp, inputs and outputs staged in shared memory; operations in the
// reference's order with explicit rounding.  coef = {a0_lo, b1_lo, a0_hi, a1_hi, b1_hi},
// state = history[2]{lo, hi}.
// `direct` (null: none): the direct-channel signal of L/R [2][1024], moved out of RealOut before
// the decode and added back after the cross-feed (alc/alu.cpp:414-433).
struct Bs2bParams { float *real; float *state; const float *coef; uint32_t frames, real_left, real_right;
    const float *direct; };

__global__ void __launch_bounds__(128) k_post_bs2b(const Bs2bParams Q)
{
    __shared__ float sIn[2][kLine];
    __shared__ float sOut[4][kLine + 8];     // L hi, L lo, R lo, R hi
    const uint32_t n = Q.frames;
    float *left = Q.real + size_t(Q.real_left)*kLine, *right = Q.real + size_t(Q.real_right)*kLine;
    for(uint32_t k = threadIdx.x;k < n;k += blockDim.x) { sIn[0][k] = left[k]; sIn[1][k] = right[k]; }
    __syncthreads();
    const int chain = threadIdx.x >> 5;
    if((threadIdx.x & 31) == 0)
    {
        const float a0lo = Q.coef[0], b1lo = Q.coef[1], a0hi = Q.coef[2], a1hi = Q.coef[3], b1hi = Q.coef[4];
        // chain 0: left hi, 1: left lo, 2: right lo, 3: right hi
        const bool hi = chain == 0 || chain == 3;
        const float *src = sIn[chain >> 1];
        float *st = Q.state + (chain >> 1)*2 + (hi ? 1 : 0);
        float z = *st;
        float *dst = sOut[chain];
        uint32_t k = 0;
        for(;k + 8u <= n;k += 8u)
        {
            float x[8];
            #pragma unroll
            for(int j = 0;j < 8;++j) x[j] = src[k + j];
            #pragma unroll
            for(int j = 0;j < 8;++j)
            {
                const float y = __fadd_rn(__fmul_rn(hi ? a0hi : a0lo, x[j]), z);
                z = hi ? __fadd_rn(__fmul_rn(a1hi, x[j]), __fmul_rn(b1hi, y)) : __fmul_rn(b1lo, y);
                dst[k + j] = y;
            }
        }
        for(;k < n;++k)
        {
            const float y = __fadd_rn(__fmul_rn(hi ? a0hi : a0lo, src[k]), z);
            z = hi ? __fadd_rn(__fmul_rn(a1hi, src[k]), __fmul_rn(b1hi, y)) : __fmul_rn(b1lo, y);
            dst[k] = y;
        }
        *st = z;
    }
    __syncthreads();
    for(uint32_t k = threadIdx.x;k < n;k += blockDim.x)
    {
        left[k] = __fadd_rn(sOut[0][k], sOut[2][k]);
        right[k] = __fadd_rn(sOut[1][k], sOut[3][k]);
    }
    if(Q.direct)
        for(uint32_t k = threadIdx.x;k < n;k += blockDim.x)
        {
            left[k] = __fadd_rn(left[k], Q.direct[k]);
            right[k] = __fadd_rn(right[k], Q.direct[kLine + k]);
        }
}

// UhjEncoder<N>::encode (core/uhjfilter.cpp:83-205), N = 256 or 512.  The reference shifts
// -0.171 W + 0.208 X by +90 degrees with a segmented FFT overlap-add (core/allpass_conv.hpp);
// that is a linear convolution with an N-tap response (every second tap zero) delivered one
// 128-sample segment late, evaluated here directly from shared memory — 64/128 k MACs per
// update.  W, X, Y and the existing Left/Right content are delayed by N/2 + 128 samples.
struct PostUhjFirParams {
    const float *dry; float *real; float *state; const float *coef;   // coef[j] = h[2j+1]
    uint32_t frames, real_left, real_right, taps;
    MatrixEncSpec enc;
};
constexpr uint32_t kUhjFirHist = 640u, kUhjFirDelay = 384u;            // state: hist | W X Y L R Z lines
constexpr uint32_t kUhjFirStateFloats = kUhjFirHist + 6u*kUhjFirDelay;

__global__ void __launch_bounds__(1024) k_post_uhj_fir(const PostUhjFirParams Q)
{
    constexpr uint32_t kSeg = 128u;
    __shared__ float sExt[kUhjFirHist + kLine];
    __shared__ float sCoef[256];
    const uint32_t n = Q.frames, N = Q.taps, hist = N + kSeg - 1u, delay = N/2u + kSeg;
    const uint32_t i = threadIdx.x;
    float *wxh = Q.state;
    const MatrixEncSpec E = Q.enc;
    const bool hasZ = E.z != ~0u;
    const float *w = Q.dry + size_t(E.w)*kLine, *x = Q.dry + size_t(E.x)*kLine, *y = Q.dry + size_t(E.y)*kLine;
    float *lines[6] = {const_cast<float*>(w), const_cast<float*>(x), const_cast<float*>(y),
        Q.real + size_t(Q.real_left)*kLine, Q.real + size_t(Q.real_right)*kLine,
        const_cast<float*>(hasZ ? Q.dry + size_t(E.z)*kLine : w)};

    if(i < hist) sExt[i] = wxh[i];
    if(i < n) sExt[hist + i] = E.dw*w[i] + E.dx*x[i];
    if(i < N/2u) sCoef[i] = Q.coef[i];
    // the delayed signals: [delay line | this update] -> value i; the tail is the new line
    float dv[6], nd[6];
    #pragma unroll
    for(int c = 0;c < 6;++c)
    {
        const float *dl = Q.state + kUhjFirHist + c*kUhjFirDelay;
        dv[c] = 0.0f; nd[c] = 0.0f;
        if(c == 5 && !hasZ) continue;
        if(i < n) dv[c] = i < delay ? dl[i] : lines[c][i - delay];
        if(i < delay) nd[c] = (n + i < delay) ? dl[n + i] : lines[c][n + i - delay];
    }
    __syncthreads();
    if(i < n)
    {
        const float *src = sExt + hist + i - kSeg - 1u;     // tap k = 2j+1 reads src[-2j]
        float acc0 = 0.0f, acc1 = 0.0f;
        for(uint32_t j = 0;j < N/2u;j += 2u)
        {
            acc0 = fmaf(sCoef[j], src[-int(2u*j)], acc0);
            acc1 = fmaf(sCoef[j + 1u], src[-int(2u*j + 2u)], acc1);
        }
        float S = E.sw*dv[0] + E.sx*dv[1];
        if(hasZ) S = S + E.sz*dv[5];
        const float D = (acc0 + acc1) + E.dy*dv[2];
        lines[3][i] = dv[3] + (S + D);
        lines[4][i] = dv[4] + (S - D);
    }
    #pragma unroll
    for(int c = 0;c < 6;++c)
        if(i < delay && (c < 5 || hasZ)) Q.state[kUhjFirHist + c*kUhjFirDelay + i] = nd[c];
    if(i < hist) wxh[i] = sExt[n + i];
}

// Output limiter: Compressor::process (core/mastering.cpp:261-379) on RealOut, one CTA.
// The reference's stages are kept, each in the most parallel form its arithmetic allows:
//  1. pre-gain, linked peak max_c|x_c| (one thread per sample);
//  2. the crest-factor detectors (:288-308) are first-order recurrences — one thread walks them
//     in the reference's order while the other warps take the logarithm and the peak hold: the
//     sliding hold (:46-105, a descending-maxima queue) IS the maximum over the last `hold`
//     detector values, so every sample takes it over a window of [history | this update];
//  3. attack/release coefficients exp(-1/t) from the crest factor, one thread per sample;
//  4. gain computer + ballistics + deviation tracking (gainCompressor, :177-259): a serial,
//     nonlinear chain (the automated knee feeds back), one thread, the reference's operation
//     order with explicitly rounded operations;
//  5. exp() of the control signal, the look-ahead FIFO (:331-358) and the gain, per sample.
struct LimiterDev {
    uint32_t flags, look_ahead, hold, num_chans;
    float pre_gain, post_gain, threshold, slope, knee, attack, release;
    float crest_coeff, gain_estimate, adapt_coeff;
    // state carried between updates
    float last_peak_sq, last_rms_sq, last_release, last_attack, last_gain_dev;
    uint32_t pad;
    float side_carry[kLine];      // mSideChain[0..look_ahead)
    float hold_hist[kLine];       // the hold's last hold-1 detector values (-inf at start)
};
struct LimiterParams { LimiterDev *lim; float *real; float *delay; uint32_t frames; };

__device__ __forceinline__ float lerp_rn(float a, float b, float mu)
{ return __fadd_rn(a, __fmul_rn(__fsub_rn(b, a), mu)); }       // lerpf, common/altypes.hpp:1197

// exp/log as the host libm rounds them (glibc's expf/logf are correctly rounded but for rare
// half-way cases): evaluated in double and rounded once.  The smoothing coefficients
// exp(-1/t) sit just below 1, where one float ulp changes the release RATE (1-a) by 1e-4
// relative — CUDA's 2-ulp expf would make the envelope drift away from the reference's.
__device__ __forceinline__ float exp_cr(float x) { return float(exp(double(x))); }
__device__ __forceinline__ float log_cr(float x) { return float(log(double(x))); }

struct LimiterChainArgs {
    LimiterDev *lim;
    const float *yg, *side, *rel, *att;     // shared memory: x_over / y_G, mSideChain, a_rel, a_att
    float *out;                             // shared memory: postGain - y_L per sample
    uint32_t n; float thr;
};

// Gain computer + ballistics + deviation tracking of gainCompressor (core/mastering.cpp:196-253),
// one thread, the reference's operation order.
template<bool AUTO_KNEE, bool AUTO_POST, bool AUTO_DECLIP>
__device__ __noinline__ void limiter_chain(const LimiterChainArgs A)
{
    LimiterDev &L = *A.lim;
    const uint32_t n = A.n;
    const float thr = A.thr, nslope = -L.slope, c_est = L.gain_estimate, a_adp = L.adapt_coeff;
    float postGain = L.post_gain;
    float y_1 = L.last_release, y_L = L.last_attack, c_dev = L.last_gain_dev;

    // one sample of the chain after the static curve
    auto ballistics = [&](float y_G, float input, float a_rel, float a_att) -> float
    {
        const float x_L = __fmul_rn(nslope, y_G);
        y_1 = fmaxf(x_L, lerp_rn(x_L, y_1, a_rel));
        y_L = lerp_rn(y_1, y_L, a_att);
        c_dev = lerp_rn(-__fadd_rn(y_L, c_est), c_dev, a_adp);
        if(AUTO_POST)
        {
            if(AUTO_DECLIP)
                c_dev = fmaxf(c_dev, __fsub_rn(__fsub_rn(__fsub_rn(input, y_L), thr), c_est));
            postGain = -__fadd_rn(c_dev, c_est);
        }
        return __fsub_rn(postGain, y_L);
    };
    // half the automated knee: 0.5*max(0, 2.5*(c_dev+c_est)) == max(0, 1.25*(c_dev+c_est))
    auto knee_half = [&]() -> float
    { return fmaxf(0.0f, __fmul_rn(1.25f, __fadd_rn(c_dev, c_est))); };
    // the static curve with a knee (:205-210); 2*knee == 4*knee_half
    auto curve = [&](float x_over, float knee_h) -> float
    {
        if(x_over <= -knee_h) return 0.0f;
        if(fabsf(x_over) < knee_h)
        {
            const float t = __fadd_rn(x_over, knee_h);
            return __fdiv_rn(__fmul_rn(t, t), __fmul_rn(4.0f, knee_h));
        }
        return x_over;
    };

    uint32_t k = 0;
    for(;k + 8u <= n;k += 8u)
    {
        float xo[8], in[8], ar[8], aa[8], o[8];
        #pragma unroll
        for(int j = 0;j < 8;++j)
        { xo[j] = A.yg[k + j]; in[j] = A.side[k + j]; ar[j] = A.rel[k + j]; aa[j] = A.att[k + j]; }
        if(!AUTO_KNEE)
        {
            // no feedback into the static curve (y_G came from phase 3): three short
            // pipelined recurrences
            #pragma unroll
            for(int j = 0;j < 8;++j) o[j] = ballistics(xo[j], in[j], ar[j], aa[j]);
        }
        else
        {
            // The automated knee feeds the deviation c_dev back into the curve, which makes
            // every sample wait for the previous one's whole chain.  But the curve only asks
            // on which side of -knee/2 the sample lies (the knee region itself is rare), and
            // the knee moves slowly: run the block with the knee frozen at its first sample's
            // value, then check every sample's decision against the knee it should have seen;
            // on any difference redo the block one sample at a time.  Exact either way.
            const float sy1 = y_1, syL = y_L, scd = c_dev, spg = postGain;
            const float kh0 = knee_half();
            float kh[8];
            #pragma unroll
            for(int j = 0;j < 8;++j)
            {
                kh[j] = knee_half();
                o[j] = ballistics(xo[j] <= -kh0 ? 0.0f : xo[j], in[j], ar[j], aa[j]);
            }
            bool bad = false;
            #pragma unroll
            for(int j = 0;j < 8;++j)
            {
                const bool below0 = xo[j] <= -kh0, below = xo[j] <= -kh[j];
                bad |= (below != below0) | (!below & (fabsf(xo[j]) < kh[j]));
            }
            if(bad)
            {
                y_1 = sy1; y_L = syL; c_dev = scd; postGain = spg;
                #pragma unroll
                for(int j = 0;j < 8;++j)
                    o[j] = ballistics(curve(xo[j], knee_half()), in[j], ar[j], aa[j]);
            }
        }
        #pragma unroll
        for(int j = 0;j < 8;++j) A.out[k + j] = o[j];
    }
    for(;k < n;++k)
    {
        const float x_over = A.yg[k];
        const float y_G = AUTO_KNEE ? curve(x_over, knee_half()) : x_over;
        A.out[k] = ballistics(y_G, A.side[k], A.rel[k], A.att[k]);
    }
    L.last_release = y_1; L.last_attack = y_L; L.last_gain_dev = c_dev;
}

__global__ void __launch_bounds__(1024) k_limiter(const LimiterParams Q)
{
    __shared__ float s_side[2*kLine];     // [carried look-ahead part | this update's detector]
    __shared__ float s_xg[2*kLine];       // [hold history | log peak of this update]
    __shared__ float s_x2[kLine];         // squared peak, later the log-domain gain
    __shared__ float s_att[kLine], s_rel[kLine];
    __shared__ float s_yg[kLine];         // x_over, or the static curve's y_G with a fixed knee
    LimiterDev &L = *Q.lim;
    const uint32_t n = Q.frames, i = threadIdx.x, la = L.look_ahead, C = L.num_chans;
    const uint32_t flags = L.flags;
    const bool autoKnee = flags & 1u, autoAtt = flags & 2u, autoRel = flags & 4u;
    const bool autoPost = flags & 8u, autoDeclip = flags & 16u;
    const uint32_t hh = L.hold > 1u ? L.hold - 1u : 0u;
    const float pre = L.pre_gain;

    // 1
    if(i < n)
    {
        float xabs = 0.0f;
        for(uint32_t c = 0;c < C;++c)
        {
            float v = Q.real[size_t(c)*kLine + i];
            if(pre != 1.0f) { v = __fmul_rn(v, pre); Q.real[size_t(c)*kLine + i] = v; }
            xabs = fmaxf(xabs, fabsf(v));
        }
        s_x2[i] = fminf(fmaxf(__fmul_rn(xabs, xabs), 0.000001f), 1000000.0f);
        s_xg[hh + i] = log_cr(fmaxf(0.000001f, xabs));
    }
    if(i < la) s_side[i] = L.side_carry[i];
    if(i < hh) s_xg[i] = L.hold_hist[i];
    __syncthreads();

    // 2
    if(i == 0 || i == 32u)
    {
        // the two detectors are independent recurrences: one thread each (different warps),
        // eight samples loaded ahead of the dependent chain
        if(autoAtt || autoRel)
        {
            const float a = L.crest_coeff;
            const bool peak = i == 0;
            float y = peak ? L.last_peak_sq : L.last_rms_sq;
            float *dst = peak ? s_att : s_rel;
            uint32_t k = 0;
            for(;k + 8u <= n;k += 8u)
            {
                float x2[8];
                #pragma unroll
                for(int j = 0;j < 8;++j) x2[j] = s_x2[k + j];
                #pragma unroll
                for(int j = 0;j < 8;++j)
                {
                    const float t = lerp_rn(x2[j], y, a);
                    y = peak ? fmaxf(x2[j], t) : t;
                    dst[k + j] = y;
                }
            }
            for(;k < n;++k)
            {
                const float x2 = s_x2[k];
                const float t = lerp_rn(x2, y, a);
                y = peak ? fmaxf(x2, t) : t;
                dst[k] = y;
            }
            if(peak) L.last_peak_sq = y; else L.last_rms_sq = y;
        }
    }
    else if(i >= 64u)
    {
        for(uint32_t k = i - 64u;k < n;k += 960u)
        {
            float m = s_xg[hh + k];
            for(uint32_t j = 0;j < hh;++j) m = fmaxf(m, s_xg[k + j]);
            s_side[la + k] = m;
        }
    }
    __syncthreads();
    if(i < hh) L.hold_hist[i] = s_xg[n + i];

    // 3
    const float thr = L.threshold;
    if(i < n)
    {
        float t_att = L.attack, t_rel = __fsub_rn(L.release, L.attack);
        float a_att, a_rel;
        if(autoAtt || autoRel)
        {
            const float crest = __fdiv_rn(s_att[i], s_rel[i]);
            if(autoAtt) t_att = __fdiv_rn(__fmul_rn(2.0f, L.attack), crest);
            if(autoRel) t_rel = __fsub_rn(__fdiv_rn(__fmul_rn(2.0f, L.release), crest), t_att);
        }
        a_att = exp_cr(__fdiv_rn(-1.0f, t_att));
        a_rel = exp_cr(__fdiv_rn(-1.0f, t_rel));
        s_att[i] = a_att; s_rel[i] = a_rel;
        // x_over; with a fixed knee the whole static curve is known here
        const float x_over = __fsub_rn(s_side[la + i], thr);
        float y_G = x_over;
        if(!autoKnee)
        {
            const float knee = L.knee, knee_h = __fmul_rn(0.5f, knee);
            if(x_over <= -knee_h) y_G = 0.0f;
            else if(fabsf(x_over) < knee_h)
            {
                const float t = __fadd_rn(x_over, knee_h);
                y_G = __fdiv_rn(__fmul_rn(t, t), __fmul_rn(2.0f, knee));
            }
        }
        s_yg[i] = y_G;
    }
    __syncthreads();

    // 4
    if(i == 0)
    {
        const LimiterChainArgs A{&L, s_yg, s_side, s_rel, s_att, s_x2, n, thr};
        // the automation flags are compile-time in the chain: a flag test inside the unrolled
        // block would cut it into short dependent pieces
        if(autoKnee)
        {
            if(autoDeclip) limiter_chain<true, true, true>(A);
            else if(autoPost) limiter_chain<true, true, false>(A);
            else limiter_chain<true, false, false>(A);
        }
        else
        {
            if(autoDeclip) limiter_chain<false, true, true>(A);
            else if(autoPost) limiter_chain<false, true, false>(A);
            else limiter_chain<false, false, false>(A);
        }
    }
    __syncthreads();

    // 5
    const float g = i < n ? exp_cr(s_x2[i]) : 0.0f;
    if(i < la) L.side_carry[i] = s_side[n + i];
    for(uint32_t c = 0;c < C;++c)
    {
        float *x = Q.real + size_t(c)*kLine;
        float *dl = Q.delay + size_t(c)*kLine;
        // stream = [delay line | this update]: output i is stream[i], the new delay line is the
        // stream's last look_ahead samples
        float v = 0.0f, nd = 0.0f;
        if(i < n) v = i < la ? dl[i] : x[i - la];
        if(i < la) nd = (n + i < la) ? dl[n + i] : x[n + i - la];
        __syncthreads();
        if(i < n) x[i] = __fmul_rn(g, v);
        if(i < la) dl[i] = nd;
    }
}

// Speaker distance compensation: ApplyDistanceComp (alc/alu.cpp:2276-2307).  Per channel a
// FIFO of `delay` samples ([delay line | this update] -> output, the rest is the new delay
// line), then the channel's gain on what comes out; channels without a delay are left alone.
struct DistCompParams { float *real; float *buf; const uint32_t *delay; const float *gain; uint32_t frames; };

__global__ void __launch_bounds__(1024) k_distance_comp(const DistCompParams Q)
{
    const uint32_t c = blockIdx.x, i = threadIdx.x, n = Q.frames, base = Q.delay[c];
    if(base < 1u) return;
    float *x = Q.real + size_t(c)*kLine, *dl = Q.buf + size_t(c)*kLine;
    float v = 0.0f, nd = 0.0f;
    if(i < n) v = i < base ? dl[i] : x[i - base];
    if(i < base) nd = (n + i < base) ? dl[n + i] : x[n + i - base];
    __syncthreads();
    if(i < n) x[i] = __fmul_rn(v, Q.gain[c]);
    if(i < base) dl[i] = nd;
}

// Output stage: ApplyDither (alc/alu.cpp:2309-2333) + Write<T> (alc/alu.cpp:2362-2390).
// The reference draws two LCG values per sample, channel after channel; sample i of channel c
// therefore uses draws 2(c*n+i)+1 and +2 from the incoming seed — reached directly with the
// LCG's closed form x_k = A^k x_0 + C(A^k-1)/(A-1) (mod 2^32), so every thread is independent.
struct OutputParams {
    const float *real; void *out;
    uint32_t frames, channels, frame_step, out_type, seed;
    float dither_depth;
};

// Also advances the host's seed past an update, whose step count needs 64 bits.
template<typename Count>
__host__ __device__ __forceinline__ uint32_t lcg_skip(uint32_t x, Count k)
{
    // k steps of x -> x*96314165 + 907633515 (dither_rng, alc/alu.cpp:444-448)
    uint32_t a = 96314165u, c = 907633515u;      // one step
    uint32_t accA = 1u, accC = 0u;               // identity
    while(k)
    {
        if(k & 1u) { accA = accA*a; accC = accC*a + c; }
        c = c*a + c; a = a*a;
        k >>= 1;
    }
    return accA*x + accC;
}

__global__ void k_output_write(const OutputParams Q)
{
    const uint32_t idx = blockIdx.x*blockDim.x + threadIdx.x;
    const uint32_t n = Q.frames;
    if(idx >= n*Q.frame_step) return;
    const uint32_t i = idx / Q.frame_step, c = idx - i*Q.frame_step;
    float val = 0.0f;
    if(c < Q.channels)
    {
        val = Q.real[size_t(c)*kLine + i];
        if(Q.dither_depth > 0.0f)
        {
            const uint32_t k = 2u*(c*n + i);
            const uint32_t r0 = lcg_skip(Q.seed, k + 1u);
            const uint32_t r1 = r0*96314165u + 907633515u;
            const double inv = 1.0/4294967295.0;
            float v = __fmul_rn(val, Q.dither_depth);
            v = __fadd_rn(v, float(double(r0)*inv - double(r1)*inv));
            val = __fmul_rn(rintf(v), __fdiv_rn(1.0f, Q.dither_depth));
        }
    }
    // SampleConv<T>, alc/alu.cpp:2335-2360 (fastf2i rounds to nearest even)
    switch(Q.out_type)
    {
    case 0: case 1:
    {
        int v = __float2int_rn(fminf(fmaxf(__fmul_rn(val, 128.0f), -128.0f), 127.0f));
        if(Q.out_type == 1) v += 128;
        static_cast<uint8_t*>(Q.out)[idx] = uint8_t(v);
        break;
    }
    case 2: case 3:
    {
        int v = __float2int_rn(fminf(fmaxf(__fmul_rn(val, 32768.0f), -32768.0f), 32767.0f));
        if(Q.out_type == 3) v += 32768;
        static_cast<uint16_t*>(Q.out)[idx] = uint16_t(v);
        break;
    }
    case 4: case 5:
    {
        const int v = __float2int_rn(fminf(fmaxf(__fmul_rn(val, 2147483648.0f), -2147483648.0f), 2147483520.0f));
        static_cast<uint32_t*>(Q.out)[idx] = Q.out_type == 5 ? uint32_t(v) + 2147483648u : uint32_t(v);
        break;
    }
    default: static_cast<float*>(Q.out)[idx] = val; break;
    }
}

} // namespace b200mix
