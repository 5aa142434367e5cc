// efx_kernels.cu — EffectState::process of the EFX effects behind b200mix_slot_efx on the GPU:
// echo, ring modulator, equalizer, compressor, dedicated, distortion
// (alc/effects/{echo,modulator,equalizer,compressor,dedicated,distortion}.cpp).
//
// Every one of these is a handful of per-sample recurrences (biquads, an envelope follower, a
// feedback delay) around trivially parallel arithmetic, and a scene has few of them: one CTA per
// slot, the recurrences each on their own thread reading and writing shared memory (so only the
// filter state is on the dependency chain), everything else spread over the CTA.  The kernel
// leaves the effect's output LINES in the slot record; the slot output mix
// (k_slot_output_mix / k_slot_target_mix) applies the pan gains with MixSamples' fade.
//
// Built with -fmad=false like the parameter kernels: the recurrences are written as the
// reference writes them and are evaluated operation for operation (no FMA contraction; the
// reference's x86-64 baseline build has none either), with flush-to-zero as the mixer thread
// runs (core/fpu_ctrl.cpp).  The one libm call inside a process() — the ring modulator's
// std::sin per sample — is evaluated in double and rounded once.
#include <cstdint>
#include <cuda_runtime.h>

#include "efx_kernels.hpp"
#include "pshift.hpp"

namespace b200mix {

namespace {

constexpr int kLine = 1024;

// BiquadFilter::process (core/filters/biquad.cpp:175-200), in place on shared memory
__device__ __forceinline__ void biquad_run(const float *c, float *z, const float *src, float *dst, uint32_t n)
{
    const float b0 = c[0], b1 = c[1], b2 = c[2], a1 = c[3], a2 = c[4];
    float z1 = z[0], z2 = z[1];
    for(uint32_t i = 0;i < n;++i)
    {
        const float x = src[i];
        const float y = x*b0 + z1;
        z1 = x*b1 - y*a1 + z2;
        z2 = x*b2 - y*a2;
        dst[i] = y;
    }
    z[0] = z1; z[1] = z2;
}

// BiquadFilter::dualProcess (core/filters/biquad.cpp:254-283)
__device__ __forceinline__ void dual_biquad_run(const float *c0, const float *c1, float *z0, float *z1,
    const float *src, float *dst, uint32_t n)
{
    const float b00 = c0[0], b01 = c0[1], b02 = c0[2], a01 = c0[3], a02 = c0[4];
    const float b10 = c1[0], b11 = c1[1], b12 = c1[2], a11 = c1[3], a12 = c1[4];
    float z01 = z0[0], z02 = z0[1], z11 = z1[0], z12 = z1[1];
    for(uint32_t i = 0;i < n;++i)
    {
        const float x0 = src[i];
        const float y0 = x0*b00 + z01;
        z01 = x0*b01 - y0*a01 + z02;
        z02 = x0*b02 - y0*a02;
        const float y1 = y0*b10 + z11;
        z11 = y0*b11 - y1*a11 + z12;
        z12 = y0*b12 - y1*a12;
        dst[i] = y1;
    }
    z0[0] = z01; z0[1] = z02; z1[0] = z11; z1[1] = z12;
}

constexpr float kDecodeCoeff = static_cast<float>(0.25 / 1.7320508075688772935);     // distortion.cpp:52
constexpr float kEncodeCoeff = static_cast<float>(0.5 * 1.7320508075688772935);      // distortion.cpp:62
__constant__ float kB2A[4][4] = {{0.25f,  kDecodeCoeff,  kDecodeCoeff,  kDecodeCoeff},
                                 {0.25f, -kDecodeCoeff, -kDecodeCoeff,  kDecodeCoeff},
                                 {0.25f,  kDecodeCoeff, -kDecodeCoeff, -kDecodeCoeff},
                                 {0.25f, -kDecodeCoeff,  kDecodeCoeff, -kDecodeCoeff}};
__constant__ float kA2B[4][4] = {{1.0f, 1.0f, 1.0f, 1.0f},
                                 {kEncodeCoeff, -kEncodeCoeff,  kEncodeCoeff, -kEncodeCoeff},
                                 {kEncodeCoeff, -kEncodeCoeff, -kEncodeCoeff,  kEncodeCoeff},
                                 {kEncodeCoeff,  kEncodeCoeff, -kEncodeCoeff, -kEncodeCoeff}};

// grid = slots, 128 threads, dynamic shared memory: 2*kEfxMaxLines + 1 lines (input copies + work)
// ---- frequency shifter helpers: 1024-point complex FFT in double, one warp per transform, data in
// shared memory (complex_fft, common/alcomplex.cpp:110-197 computes the same radix-2 DIT butterflies
// with recursively multiplied twiddles; direct table twiddles differ in the last bits of a double
// only) and the discrete Hilbert transform built on it (complex_hilbert, :199-215).
__device__ double2 g_fs_tw[512];          // exp(+i 2 pi k / 1024)
__device__ float g_fs_hann[1024];         // gHannWindow<1024>, common/hann_window.hpp:11-26

__global__ void k_efx_tables()
{
    const uint32_t k = threadIdx.x;
    if(k < 512u)
    {
        double sn, cs;
        sincospi(double(k) / 512.0, &sn, &cs);
        g_fs_tw[k] = make_double2(cs, sn);
        const double v = ::sin((double(k) + 1.0) * (3.14159265358979323846 / 1025.0));
        const float w = float(v * v);
        g_fs_hann[k] = w; g_fs_hann[1023u - k] = w;
    }
}

__device__ __forceinline__ void fft1024_warp(double2 *x, uint32_t lane, double sign)
{
    for(uint32_t i = lane;i < 1024u;i += 32u)
    {
        const uint32_t j = __brev(i) >> 22;
        if(i < j) { const double2 a = x[i]; x[i] = x[j]; x[j] = a; }
    }
    __syncwarp();
    for(uint32_t s = 0;s < 10u;++s)
    {
        const uint32_t half = 1u << s;
        for(uint32_t b = lane;b < 512u;b += 32u)
        {
            const uint32_t j = b & (half - 1u), k = ((b >> s) << (s + 1u)) + j;
            const double2 w = g_fs_tw[j * (512u >> s)];
            const double wi = w.y * sign;
            const double2 v = x[k + half];
            const double2 tmp = make_double2(v.x*w.x - v.y*wi, v.x*wi + v.y*w.x);
            const double2 u = x[k];
            x[k + half] = make_double2(u.x - tmp.x, u.y - tmp.y);
            x[k] = make_double2(u.x + tmp.x, u.y + tmp.y);
        }
        __syncwarp();
    }
}

__device__ __forceinline__ void hilbert1024_warp(double2 *x, uint32_t lane)
{
    fft1024_warp(x, lane, 1.0);                       // inverse_fft
    const double inv = 1.0 / 1024.0;
    for(uint32_t i = lane;i < 1024u;i += 32u)
    {
        double2 v = x[i];
        if(i == 0u || i == 512u) { v.x *= inv; v.y *= inv; }
        else if(i < 512u) { v.x *= inv*2.0; v.y *= inv*2.0; }
        else v = make_double2(0.0, 0.0);
        x[i] = v;
    }
    __syncwarp();
    fft1024_warp(x, lane, -1.0);                      // forward_fft
}

__global__ void __launch_bounds__(128) k_efx_process(const EfxRunParams Q)
{
    extern __shared__ float sm[];
    const SlotRec &S = Q.slots[blockIdx.x];
    if(S.type < B200MIX_EFFECT_ECHO || S.stage != Q.stage) return;
    EfxDev &E = *reinterpret_cast<EfxDev*>(S.H);
    const EfxParams &P = E.p;
    const uint32_t t = threadIdx.x, n = Q.frames;
    const float *wet = Q.wet + size_t(blockIdx.x)*Q.cw*kLine;
    float *lines = S.lines;
    const uint32_t nin = min(P.in_channels, Q.cw);
    float *sIn = sm;                                   // [kEfxMaxLines][1024]
    float *sWork = sm + kEfxMaxLines*kLine;            // [.. ][1024]

    switch(P.type)
    {
    case B200MIX_EFFECT_DEDICATED:
        // MixSamples(samplesIn[0], ...): the line IS wet channel 0 (dedicated.cpp:105-109)
        for(uint32_t i = t;i < n;i += blockDim.x) lines[i] = wet[i];
        break;

    case B200MIX_EFFECT_ECHO:
    {
        // EchoState::process (echo.cpp:133-171).  Inside a chunk no longer than the shorter tap
        // delay every tap read refers to samples written before the chunk: the reads, the
        // delay-line write and the output lines are sample-parallel; only the damping filter on
        // the feedback tap is a recurrence (one thread, shared memory).
        const uint32_t mask = P.echo_len - 1u;
        float *buf = E.echo_buf;
        uint32_t offset = E.echo_offset;
        for(uint32_t base = 0;base < n;)
        {
            const uint32_t td = min(n - base, P.echo_tap[0]);
            for(uint32_t i = t;i < td;i += blockDim.x)
            {
                const float o1 = buf[(offset + i - P.echo_tap[0]) & mask];
                const float o2 = buf[(offset + i - P.echo_tap[1]) & mask];
                lines[base + i] = o1;
                lines[kLine + base + i] = o2;
                sWork[i] = o2;
            }
            __syncthreads();
            if(t == 0) biquad_run(P.echo_filter, E.echo_z, sWork, sWork, td);
            __syncthreads();
            for(uint32_t i = t;i < td;i += blockDim.x)
                buf[(offset + i) & mask] = wet[base + i] + sWork[i] * P.echo_feed;
            __threadfence_block();
            __syncthreads();
            offset += td; base += td;
        }
        if(t == 0) E.echo_offset = offset & mask;
        break;
    }

    case B200MIX_EFFECT_MODULATOR:
    {
        // ModulatorState::process (modulator.cpp:157-199)
        const uint32_t range = P.mod_range, index0 = E.mod_index;
        for(uint32_t i = t;i < n;i += blockDim.x)
        {
            const uint32_t idx = (index0 + i) % range;
            float m = 1.0f;
            if(P.mod_wave == 1u) m = float(::sin(double(float(idx) * P.mod_scale)));
            else if(P.mod_wave == 2u) m = float(idx)*P.mod_scale - 1.0f;
            else if(P.mod_wave == 3u) m = float(float(idx)*P.mod_scale < 0.5f)*2.0f - 1.0f;
            sWork[kLine*kEfxMaxLines + i] = m;         // mModSamples: the extra work row
        }
        for(uint32_t c = 0;c < nin;++c)
            for(uint32_t i = t;i < n;i += blockDim.x) sIn[c*kLine + i] = wet[size_t(c)*kLine + i];
        __syncthreads();
        if(t < nin && P.line_on[t]) biquad_run(P.mod_hp, E.chan_z[t][0], sIn + t*kLine, sWork + t*kLine, n);
        __syncthreads();
        const float *mod = sWork + kLine*kEfxMaxLines;
        for(uint32_t c = 0;c < P.lines;++c)
            for(uint32_t i = t;i < n;i += blockDim.x)
                lines[size_t(c)*kLine + i] = (c < nin && P.line_on[c]) ? sWork[c*kLine + i] * mod[i] : 0.0f;
        if(t == 0) E.mod_index = (index0 + n) % range;
        break;
    }

    case B200MIX_EFFECT_EQUALIZER:
    {
        // EqualizerState::process (equalizer.cpp:165-183): two DualBiquad passes per channel
        for(uint32_t c = 0;c < nin;++c)
            for(uint32_t i = t;i < n;i += blockDim.x) sIn[c*kLine + i] = wet[size_t(c)*kLine + i];
        __syncthreads();
        if(t < nin && P.line_on[t])
        {
            dual_biquad_run(P.eq[0], P.eq[1], E.chan_z[t][0], E.chan_z[t][1], sIn + t*kLine, sWork + t*kLine, n);
            dual_biquad_run(P.eq[2], P.eq[3], E.chan_z[t][2], E.chan_z[t][3], sWork + t*kLine, sWork + t*kLine, n);
        }
        __syncthreads();
        for(uint32_t c = 0;c < P.lines;++c)
            for(uint32_t i = t;i < n;i += blockDim.x)
                lines[size_t(c)*kLine + i] = (c < nin && P.line_on[c]) ? sWork[c*kLine + i] : 0.0f;
        break;
    }

    case B200MIX_EFFECT_COMPRESSOR:
    {
        // CompressorState::process (compressor.cpp:111-177): envelope follower on channel 0
        for(uint32_t i = t;i < n;i += blockDim.x) sIn[i] = wet[i];
        __syncthreads();
        if(t == 0)
        {
            float env = E.comp_env;
            const float am = P.comp_attack, rm = P.comp_release;
            for(uint32_t i = 0;i < n;++i)
            {
                float amplitude = 1.0f;
                if(P.comp_enabled)
                {
                    amplitude = fabsf(sIn[i]);
                    amplitude = amplitude < 0.5f ? 0.5f : (2.0f < amplitude ? 2.0f : amplitude);
                }
                if(amplitude > env) { const float e = env*am; env = amplitude < e ? amplitude : e; }
                else if(amplitude < env) { const float e = env*rm; env = e < amplitude ? amplitude : e; }
                sWork[i] = 1.0f / env;
            }
            E.comp_env = env;
        }
        __syncthreads();
        for(uint32_t c = 0;c < P.lines;++c)
            for(uint32_t i = t;i < n;i += blockDim.x)
                lines[size_t(c)*kLine + i] = (c < nin && P.line_on[c]) ? wet[size_t(c)*kLine + i] * sWork[i] : 0.0f;
        break;
    }

    case B200MIX_EFFECT_DISTORTION:
    {
        // DistortionState::process (distortion.cpp:198-303), first-order devices
        const uint32_t numInput = min(nin, 4u);
        // B-Format -> A-Format, accumulated in input order like the reference's transform loop
        for(uint32_t i = t;i < n;i += blockDim.x)
            for(uint32_t c = 0;c < 4u;++c)
            {
                float a = 0.0f;
                for(uint32_t k = 0;k < numInput;++k) a = a + wet[size_t(k)*kLine + i]*kB2A[c][k];
                sIn[c*kLine + i] = a;
            }
        // mBBuffer rows 4..7 of sIn accumulate the result
        for(uint32_t i = t;i < 4u*kLine;i += blockDim.x) sIn[4*kLine + i] = 0.0f;
        __syncthreads();
        const float fc = P.dist_edge;
        for(uint32_t base = 0;base < n;)
        {
            const uint32_t todo = min(uint32_t(kLine), (n - base)*4u);
            for(uint32_t c = 0;c < 4u;++c)
            {
                float *t0 = sWork, *t1 = sWork + kLine;
                // zero stuffing x4 (keeps the signal's power)
                for(uint32_t i = t;i < todo;i += blockDim.x)
                    t0[i] = !(i & 3u) ? sIn[c*kLine + (i >> 2) + base] * 4.0f : 0.0f;
                __syncthreads();
                if(t == 0) biquad_run(P.dist_lp, E.chan_z[c][0], t0, t1, todo);
                __syncthreads();
                // three waveshaper steps
                for(uint32_t i = t;i < todo;i += blockDim.x)
                {
                    float smp = t1[i];
                    smp = ( 1.0f + fc) * smp/(1.0f + fc*fabsf(smp));
                    smp = (-1.0f - fc) * smp/(1.0f + fc*fabsf(smp));
                    smp = ( 1.0f + fc) * smp/(1.0f + fc*fabsf(smp));
                    t0[i] = smp;
                }
                __syncthreads();
                if(t == 0) biquad_run(P.dist_bp, E.chan_z[c][1], t0, t1, todo);
                __syncthreads();
                // A-Format -> B-Format, decimated (every fourth sample)
                for(uint32_t i = t;i < (todo >> 2);i += blockDim.x)
                    for(uint32_t k = 0;k < 4u;++k)
                        sIn[(4u + k)*kLine + base + i] = sIn[(4u + k)*kLine + base + i] + t1[i*4u]*kA2B[k][c];
                __syncthreads();
            }
            base += todo >> 2;
        }
        for(uint32_t c = 0;c < 4u;++c)
            for(uint32_t i = t;i < n;i += blockDim.x)
                lines[size_t(c)*kLine + i] = P.line_on[c] ? sIn[(4u + c)*kLine + i] : 0.0f;
        break;
    }
    case B200MIX_EFFECT_CHORUS:
    {
        // ChorusState::process (chorus.cpp:326-425), first-order devices.  The feedback tap sits
        // only (mDelay + 2^15) >> 16 samples back — a per-sample recurrence through the delay
        // line: one thread per A-format line, the line's delay buffer in shared memory.
        static const float dc = kDecodeCoeff, ec = kEncodeCoeff;
        const float B2A[4][4] = {{0.25f, dc, dc, dc}, {0.25f, dc, -dc, -dc}, {0.25f, -dc, -dc, dc}, {0.25f, -dc, dc, -dc}};
        const float A2B[4][4] = {{1.0f, 1.0f, 1.0f, 1.0f}, {ec, ec, -ec, -ec}, {ec, -ec, -ec, ec}, {ec, -ec, ec, -ec}};
        const uint32_t numInput = min(nin, 4u);
        for(uint32_t i = t;i < n;i += blockDim.x)
            for(uint32_t c = 0;c < 4u;++c)
            {
                float a = 0.0f;
                for(uint32_t k = 0;k < numInput;++k) a = a + wet[size_t(k)*kLine + i]*B2A[c][k];
                sIn[c*kLine + i] = a;
            }
        // mModDelays[0] / [1] (calcTriangleDelays / calcSinusoidDelays, chorus.cpp:235-323)
        uint32_t *md = reinterpret_cast<uint32_t*>(sWork);          // rows 0,1
        const uint32_t range = P.cho_lfo_range, lfo0 = E.cho_lfo_offset;
        for(uint32_t i = t;i < 2u*n;i += blockDim.x)
        {
            const uint32_t side = i / n, k = i - side*n;
            const uint32_t off = ((side ? lfo0 + P.cho_lfo_disp : lfo0) % range + k) % range;
            const float offset_norm = float(off) * P.cho_lfo_scale;
            const float v = P.cho_wave == 1u ? (1.0f - fabsf(2.0f - offset_norm)) * P.cho_depth
                                              : float(::sin(double(offset_norm))) * P.cho_depth;
            md[side*kLine + k] = uint32_t(__float2int_rn(v) + P.cho_delay);        // fastf2i: round to nearest even
        }
        const uint32_t len = P.cho_len, mask = len - 1u;
        const bool inSmem = 4u*len <= 12u*uint32_t(kLine);
        float *dl = inSmem ? sWork + 4*kLine : E.cho_buf;              // rows 4..15 when it fits
        if(inSmem) for(uint32_t i = t;i < 4u*len;i += blockDim.x) dl[i] = E.cho_buf[i];
        __syncthreads();
        if(t < 4u)
        {
            float *d = dl + size_t(t)*len;
            const uint32_t *mds = md + (t < 2u ? 0 : kLine);
            const float fb = P.cho_feedback;
            const uint32_t avgdelay = (uint32_t(P.cho_delay) + 32768u) >> 16;
            uint32_t offset = E.cho_offset;
            float *tmp = sIn + (4u + t)*kLine;                         // mTempLine of this line
            for(uint32_t i = 0;i < n;++i)
            {
                d[offset & mask] = sIn[t*kLine + i];
                const uint32_t moddelay = mds[i];
                const uint32_t delay = offset - (moddelay >> 8), phase = moddelay & 255u;
                const float sample = d[(delay+1u) & mask]*Q.cubic[256u + phase] + d[delay & mask]*Q.cubic[phase]
                    + d[(delay-1u) & mask]*Q.cubic[256u - phase] + d[(delay-2u) & mask]*Q.cubic[512u - phase];
                d[offset & mask] += d[(offset - avgdelay) & mask] * fb;
                ++offset;
                tmp[i] = sample;
            }
        }
        __syncthreads();
        for(uint32_t c = 0;c < 4u;++c)
            for(uint32_t i = t;i < n;i += blockDim.x)
            {
                float b = 0.0f;
                for(uint32_t k = 0;k < 4u;++k) b = b + sIn[(4u + k)*kLine + i]*A2B[c][k];
                lines[size_t(c)*kLine + i] = P.line_on[c] ? b : 0.0f;
            }
        if(inSmem) for(uint32_t i = t;i < 4u*len;i += blockDim.x) E.cho_buf[i] = dl[i];
        if(t == 0) { E.cho_offset += n; E.cho_lfo_offset = (lfo0 + n) % range; }
        break;
    }

    case B200MIX_EFFECT_AUTOWAH:
    {
        // AutowahState::process (autowah.cpp:136-205): envelope follower on channel 0 (a
        // recurrence), the per-sample filter terms from it (parallel), then one peaking filter
        // with per-sample coefficients per channel (a recurrence per channel)
        for(uint32_t c = 0;c < nin;++c)
            for(uint32_t i = t;i < n;i += blockDim.x) sIn[c*kLine + i] = wet[size_t(c)*kLine + i];
        __syncthreads();
        float *env = sWork + kEfxMaxLines*kLine;                       // the extra row
        if(t == 0)
        {
            float env_delay = E.wah_env;
            for(uint32_t i = 0;i < n;++i)
            {
                const float sample = P.wah_peak_gain * fabsf(sIn[i]);
                const float a = (sample > env_delay) ? P.wah_attack : P.wah_release;
                env_delay = sample + (env_delay - sample)*a;            // lerpf(sample, env_delay, a)
                env[i] = env_delay;
            }
            E.wah_env = env_delay;
        }
        __syncthreads();
        float *cosw = sWork + (kEfxMaxLines - 1)*kLine, *alpha = sWork + (kEfxMaxLines - 2)*kLine;
        for(uint32_t i = t;i < n;i += blockDim.x)
        {
            const float f = P.wah_bandwidth*env[i] + P.wah_freq_min;
            const float w0 = (f < 0.46f ? f : 0.46f) * (3.14159265358979323846f*2.0f);
            cosw[i] = float(::cos(double(w0)));
            alpha[i] = float(::sin(double(w0)))*(0.5f/5.0f);
        }
        __syncthreads();
        if(t < nin && t < kEfxMaxLines - 2u && P.line_on[t])
        {
            float z1 = E.chan_z[t][0][0], z2 = E.chan_z[t][0][1];
            const float rg = P.wah_res_gain;
            const float *src = sIn + t*kLine;
            float *dst = sWork + t*kLine;
            for(uint32_t i = 0;i < n;++i)
            {
                const float al = alpha[i], cw = cosw[i], input = src[i];
                const float b0 = 1.0f + al*rg, b1 = -2.0f * cw, b2 = 1.0f - al*rg;
                const float a0 = 1.0f / (1.0f + al/rg), a1 = -2.0f * cw, a2 = 1.0f - al/rg;
                const float output = input*(b0*a0) + z1;
                z1 = input*(b1*a0) - output*(a1*a0) + z2;
                z2 = input*(b2*a0) - output*(a2*a0);
                dst[i] = output;
            }
            E.chan_z[t][0][0] = z1; E.chan_z[t][0][1] = z2;
        }
        __syncthreads();
        for(uint32_t c = 0;c < P.lines;++c)
            for(uint32_t i = t;i < n;i += blockDim.x)
                lines[size_t(c)*kLine + i] = (c < nin && c < kEfxMaxLines - 2u && P.line_on[c]) ? sWork[c*kLine + i] : 0.0f;
        break;
    }
    case B200MIX_EFFECT_VMORPHER:
    {
        // VmorpherState::process (vmorpher.cpp:272-330): per 256-sample chunk the LFO, then per
        // channel two banks of four formant filters (state-variable, vmorpher.cpp:106-140) —
        // eight independent recurrences per channel, one thread each — whose band outputs are
        // accumulated in formant order, blended by the LFO and mixed with MixSamples' gain ramp
        // of that chunk (Counter = the samples left in the update).
        for(uint32_t c = 0;c < nin;++c)
            for(uint32_t i = t;i < n;i += blockDim.x) sIn[c*kLine + i] = wet[size_t(c)*kLine + i];
        float *lfo = sWork + kEfxMaxLines*kLine;                       // the extra row: mLfo
        __shared__ float vmCur[kEfxMaxLines];
        if(t < kEfxMaxLines) vmCur[t] = E.vm_cur[t];
        const uint32_t step = P.vm_step, wave = P.vm_wave, index0 = E.vm_index;
        for(uint32_t i = t;i < n;i += blockDim.x)
        {
            const uint32_t idx = (index0 + step*(i + 1u)) & 0xffffffu;
            float v;
            if(wave == 0u) v = 0.5f;
            else if(wave == 1u) v = float(::sin(double(float(idx) * (3.14159265358979323846f*2.0f / 16777216.0f))))*0.5f + 0.5f;
            else if(wave == 2u) v = fabsf(float(idx)*(2.0f/16777216.0f) - 1.0f);
            else v = float(idx) / 16777216.0f;
            lfo[i] = v;
        }
        __syncthreads();
        constexpr uint32_t kChunk = 256u, kGroup = 8u;                  // channels per pass: 8 ch x 8 filters x 256
        for(uint32_t base = 0;base < n;base += kChunk)
        {
            const uint32_t td = min(kChunk, n - base);
            const uint32_t counter = n - base;
            for(uint32_t c0 = 0;c0 < nin;c0 += kGroup)
            {
                if(t < kGroup*8u)
                {
                    const uint32_t c = c0 + (t >> 3), v = (t >> 2) & 1u, f = t & 3u;
                    if(c < nin && P.vm_target[c] != 0xffffffffu)
                    {
                        const float g = P.vm_coeff[v][f], gain = P.vm_fgain[v][f];
                        const float h = 1.0f / (1.0f + (g*(1.0f/5.0f)) + (g*g));
                        const float coeff = (1.0f/5.0f) + g;
                        float s1 = E.vm_s[c][v][f][0], s2 = E.vm_s[c][v][f][1];
                        const float *src = sIn + c*kLine + base;
                        float *dst = sWork + size_t(t)*kChunk;
                        for(uint32_t k = 0;k < td;++k)
                        {
                            const float in = src[k];
                            const float H = (in - coeff*s1 - s2)*h;
                            const float B = g*H + s1;
                            const float L = g*B + s2;
                            s1 = g*H + B;
                            s2 = g*B + L;
                            dst[k] = B*gain;
                        }
                        E.vm_s[c][v][f][0] = s1; E.vm_s[c][v][f][1] = s2;
                    }
                }
                __syncthreads();
                for(uint32_t e = t;e < kGroup*td;e += blockDim.x)
                {
                    const uint32_t cl = e / td, k = e - cl*td, c = c0 + cl;
                    if(c >= nin) continue;
                    float outv = 0.0f;
                    if(P.vm_target[c] != 0xffffffffu)
                    {
                        const float *bg = sWork + size_t(cl)*8u*kChunk + k;
                        const float A = (((0.0f + bg[0]) + bg[kChunk]) + bg[2u*kChunk]) + bg[3u*kChunk];
                        const float Bv = (((0.0f + bg[4u*kChunk]) + bg[5u*kChunk]) + bg[6u*kChunk]) + bg[7u*kChunk];
                        const float blended = A + (Bv - A)*lfo[base + k];             // lerpf
                        // MixLine (mixer_c.cpp:150-186) with fade_len = td, Counter = counter
                        const float cur = vmCur[c], tg = P.vm_tgain[c];
                        const float stp = (tg - cur) * (1.0f / float(counter));
                        if(fabsf(stp) > 1.1920929e-07f) outv = blended * (cur + stp*float(k));
                        else if(fabsf(tg) > 0.00001f) outv = blended * tg;
                    }
                    lines[size_t(c)*kLine + base + k] = outv;
                }
                __syncthreads();
            }
            if(t < nin && P.vm_target[t] != 0xffffffffu)
            {
                const float cur = vmCur[t], tg = P.vm_tgain[t];
                const float stp = (tg - cur) * (1.0f / float(counter));
                vmCur[t] = (fabsf(stp) > 1.1920929e-07f && td < counter) ? cur + stp*float(td) : tg;
            }
            __syncthreads();
        }
        if(t < kEfxMaxLines) E.vm_cur[t] = vmCur[t];
        if(t == 0) E.vm_index = (index0 + step*n) & 0xffffffu;
        break;
    }
    case B200MIX_EFFECT_FSHIFTER:
    {
        // FshifterState::process (fshifter.cpp:235-366), first-order devices.  One warp per A-format
        // line: B2A into the input FIFO, every 256 samples one STFT frame (Hann window, analytic
        // signal through the Hilbert transform, window again, overlap-add), then the analytic
        // signal is rotated by the phase accumulator and encoded back to B-Format.
        static const float dc = kDecodeCoeff, ec = kEncodeCoeff;
        const float B2A[4][4] = {{0.25f, dc, dc, dc}, {0.25f, dc, -dc, -dc}, {0.25f, -dc, -dc, dc}, {0.25f, -dc, dc, -dc}};
        const float A2B[4][4] = {{1.0f, 1.0f, 1.0f, 1.0f}, {ec, ec, -ec, -ec}, {ec, -ec, -ec, ec}, {ec, -ec, ec, -ec}};
        double2 *ana = reinterpret_cast<double2*>(sIn);                 // [4][1024] mAnalytic, one per warp
        double2 *outd = reinterpret_cast<double2*>(sWork);              // [4][1024] mOutdata
        const uint32_t c = t >> 5, lane = t & 31u;
        double *infifo = E.fs_in + size_t(c)*1024u;
        double2 *outfifo = E.fs_outfifo + size_t(c)*256u;
        double2 *accum = E.fs_accum + size_t(c)*1024u;
        double2 *myAna = ana + size_t(c)*1024u, *myOut = outd + size_t(c)*1024u;
        uint32_t count = E.fs_count, pos = E.fs_pos;
        const uint32_t numInput = min(nin, 4u);
        __syncthreads();                                                // everybody has read count / pos
        for(uint32_t base = 0;base < n;)
        {
            const uint32_t todo = min(256u - count, n - base);
            for(uint32_t i = lane;i < todo;i += 32u)
            {
                double a = 0.0;
                for(uint32_t k = 0;k < numInput;++k)
                    a = a + double(wet[size_t(k)*kLine + base + i]) * double(B2A[c][k]);
                infifo[pos + count + i] = a;
                myOut[base + i] = outfifo[count + i];
            }
            __syncwarp();
            count += todo; base += todo;
            if(count < 256u) break;
            count = 0u; pos = (pos + 256u) & 1023u;
            for(uint32_t k = lane;k < 1024u;k += 32u)
                myAna[k] = make_double2(infifo[(pos + k) & 1023u] * double(g_fs_hann[k]), 0.0);
            __syncwarp();
            hilbert1024_warp(myAna, lane);
            for(uint32_t k = lane;k < 1024u;k += 32u)
            {
                const double sc = (2.0/4.0) * double(g_fs_hann[k]);
                const double2 v = myAna[k];
                const uint32_t q = (pos + k) & 1023u;
                double2 acc = accum[q];
                acc.x += sc*v.x; acc.y += sc*v.y;
                accum[q] = acc;
            }
            __syncwarp();
            for(uint32_t j = lane;j < 256u;j += 32u)
            {
                outfifo[j] = accum[pos + j];
                accum[pos + j] = make_double2(0.0, 0.0);
            }
            __syncwarp();
        }
        __syncthreads();
        float *temp = reinterpret_cast<float*>(sIn);                    // [4][1024] mTempLine per line
        {
            const uint32_t pstep = P.fs_phase_step[c], ph0 = E.fs_phase[c];
            const double sign = double(P.fs_sign[c]);
            for(uint32_t i = lane;i < n;i += 32u)
            {
                const uint32_t pidx = (ph0 + pstep*i) & 0xffffu;
                const double phase = double(pidx) * (3.14159265358979323846*2.0 / 65536.0);
                const double2 in = myOut[i];
                temp[c*kLine + i] = float(in.x*::cos(phase) + in.y*::sin(phase)*sign);
            }
            __syncwarp();
            if(lane == 0u) E.fs_phase[c] = (ph0 + pstep*n) & 0xffffu;
        }
        __syncthreads();
        for(uint32_t i4 = 0;i4 < 4u;++i4)
            for(uint32_t i = t;i < n;i += blockDim.x)
            {
                float b = 0.0f;
                for(uint32_t k = 0;k < 4u;++k) b = b + temp[k*kLine + i]*A2B[i4][k];
                lines[size_t(i4)*kLine + i] = P.line_on[i4] ? b : 0.0f;
            }
        if(t == 0u) { E.fs_count = count; E.fs_pos = pos; }
        break;
    }
    default: break;
    }
}

// PshifterState::process (pshifter.cpp:207-472), devices up to second order: a kernel of its own
// beside k_efx_process (same grid, same shared-memory carve-up; launched only while a pitch
// shifter slot exists).  One warp per wet channel (4 at a time): FIFO exchange, and every 128
// samples one STFT frame — the frame arithmetic is csrc/pshift.hpp (lane-strided, also run on the
// host by the CPU tests).  Channel 0's analysis fixes mLastPhase / mSumPhase of the frame before the
// other channels read them; the next frame's channel 0 waits for every reader of this one.
__global__ void __launch_bounds__(128) k_efx_pshift(const EfxRunParams Q)
{
    extern __shared__ float sm[];
    const SlotRec &S = Q.slots[blockIdx.x];
    if(S.type < B200MIX_EFFECT_ECHO || S.stage != Q.stage) return;
    EfxDev &E = *reinterpret_cast<EfxDev*>(S.H);
    const EfxParams &P = E.p;
    if(P.type != B200MIX_EFFECT_PSHIFTER) return;
    const uint32_t t = threadIdx.x, n = Q.frames;
    const float *wet = Q.wet + size_t(blockIdx.x)*Q.cw*kLine;
    float *lines = S.lines;
    const uint32_t nin = min(P.in_channels, Q.cw);
    float *sIn = sm;
    float *sWork = sm + kEfxMaxLines*kLine;
    namespace ps = pshift;
    static_assert(sizeof(ps::Cplx) == sizeof(double2), "transform buffers share the double2 layout");
    const uint32_t w = t >> 5;
    const ps::Lanes L{t & 31u, 32u};
    ps::Cplx *X = reinterpret_cast<ps::Cplx*>(sIn) + size_t(w)*ps::kSize;          // [4][1024] complex doubles = sIn
    float *re = sWork + size_t(w)*2u*544u, *im = re + 544u;                       // [4][2][513 (+pad)]
    const ps::Cplx *tw = reinterpret_cast<const ps::Cplx*>(g_fs_tw);
    const uint32_t numInput = min(nin, ps::kMaxLines);
    const uint32_t shift_i = P.ps_shift_i; const float shift = P.ps_shift;
    uint32_t count = E.ps_count, pos = E.ps_pos;
    __syncthreads();                                                // everybody has read count / pos
    for(uint32_t base = 0;base < n;)
    {
        const uint32_t todo = min(ps::kStep - count, n - base);
        for(uint32_t c = w;c < numInput;c += 4u)
            ps::fifo_exchange(E.ps_fifo + size_t(c)*ps::kSize + pos + count, wet + size_t(c)*kLine + base,
                lines + size_t(c)*kLine + base, todo, L);
        count += todo; base += todo;
        if(count < ps::kStep) break;
        count = 0u; pos = (pos + ps::kStep) & (ps::kSize - 1u);
        for(uint32_t c0 = 0;c0 < numInput;c0 += 4u)
        {
            const uint32_t c = c0 + w;
            const bool on = c < numInput;
            float *fifo = E.ps_fifo + size_t(c)*ps::kSize, *accum = E.ps_accum + size_t(c)*ps::kSize;
            if(on) ps::analyse_frame(X, tw, fifo, g_fs_hann, pos, re, im, L);
            if(c == 0u)
            {
                ps::bins_channel0(re, im, E.ps_last, shift, L);
                ps::synthesise_bins<true>(X, re, im, E.ps_sum, shift_i, L);
            }
            if(c0 == 0u) __syncthreads();                           // mLastPhase / mSumPhase of this frame are final
            if(on && c != 0u)
            {
                ps::bins_channelN(re, im, E.ps_last, L);
                ps::synthesise_bins<false>(X, re, im, E.ps_sum, shift_i, L);
            }
            if(on) ps::resynthesise_frame(X, tw, fifo, accum, g_fs_hann, pos, L);
        }
        __syncthreads();                                            // every channel has read this frame's phases
    }
    for(uint32_t c = numInput;c < P.lines;++c)
        for(uint32_t i = t;i < n;i += blockDim.x) lines[size_t(c)*kLine + i] = 0.0f;
    if(t == 0u) { E.ps_count = count; E.ps_pos = pos; }
}

} // namespace

constexpr int kEfxSmem = int((2u*kEfxMaxLines + 1u)*kLine*sizeof(float));

cudaError_t efx_kernels_init()
{
    k_efx_tables<<<1, 512>>>();            // twiddles + Hann window of the frequency shifter (per CUDA device)
    if(cudaError_t e = cudaDeviceSynchronize(); e != cudaSuccess) return e;
    if(cudaError_t e = cudaFuncSetAttribute(k_efx_pshift, cudaFuncAttributeMaxDynamicSharedMemorySize, kEfxSmem); e != cudaSuccess) return e;
    return cudaFuncSetAttribute(k_efx_process, cudaFuncAttributeMaxDynamicSharedMemorySize, kEfxSmem);
}

cudaError_t launch_efx_process(const EfxRunParams &Q, uint32_t num_slots, cudaStream_t stream)
{
    k_efx_process<<<num_slots, 128, kEfxSmem, stream>>>(Q);
    return cudaGetLastError();
}

cudaError_t launch_efx_pshift(const EfxRunParams &Q, uint32_t num_slots, cudaStream_t stream)
{
    k_efx_pshift<<<num_slots, 128, kEfxSmem, stream>>>(Q);
    return cudaGetLastError();
}

} // namespace b200mix
