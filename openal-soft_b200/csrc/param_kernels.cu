// param_kernels.cu — the parameter ("ALU") stage of point sources ON THE GPU (SURVEY §8f #1):
// CalcVoiceParams -> CalcAttnVoiceParams + CalcPanningAndFilters (alc/alu.cpp:1512-1657,
// 1712-2010) for the sources an application moved this update.  b200mix_sources_update ships the
// source PROPERTIES (what alSourcefv set) and the listener; these kernels produce exactly what
// b200mix_voices_update_dirs + b200mix_voices_filters would have received from the host's
// b200mix_calc_voices — step and BsincPrepare state, HRIR direction, HRTF gain or dry pan gains,
// send gains, the four shelf designs per path — as staged VoiceUpdate / FilterUpdate records that
// the existing k_apply_updates / k_apply_filter_updates then scatter.
//
// The arithmetic is param_math.hpp, the same source text the host helpers compile.  This file is
// built with -fmad=false (and without -ftz): plain float expressions keep the host's operation
// sequence, division and square root are IEEE; libm calls are evaluated in double and rounded
// once (DeviceMath).  Results equal b200mix_calc_voice's bit for bit except where the host libm's
// float function is not correctly rounded (<= 1 ulp; tests/test_gpu_params.py measures it).
#include <cstdint>
#include <cuda_runtime.h>

#include "param_kernels.hpp"

namespace b200mix {

namespace {

struct DeviceMath {
    __device__ static float sqrt(float x) { return ::sqrtf(x); }
    __device__ static float pow(float a, float b) { return float(::pow(double(a), double(b))); }
    __device__ static float acos(float x) { return float(::acos(double(x))); }
    __device__ static float asin(float x) { return float(::asin(double(x))); }
    __device__ static float atan2(float y, float x) { return float(::atan2(double(y), double(x))); }
    __device__ static float sin(float x) { return float(::sin(double(x))); }
    __device__ static float cos(float x) { return float(::cos(double(x))); }
    __device__ static float copysign(float a, float b) { return ::copysignf(a, b); }
    __device__ static long lrint(float x) { return long(__float2ll_rn(x)); }
    __device__ static float infinity() { return __int_as_float(0x7f800000); }
};

// One thread per source: everything up to the per-path HF/LF gains.
__global__ void __launch_bounds__(64) k_calc_voices(const CalcVoicesParams Q)
{
    const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
    if(i >= Q.n) return;
    const b200mix_source_voice sv = Q.voices[i];
    const b200mix_source_props &P = Q.props[i];

    b200mix_source_result r;
    pm::calc_source_params<DeviceMath>(P, Q.listener, Q.num_sends, sv.buffer_rate, Q.device_rate, r);

    b200mix_voice_env env;
    env.struct_size = sizeof(env);
    env.device_rate = Q.device_rate; env.num_sends = Q.num_sends; env.render_mode = Q.render_mode;
    env.wet_stride = Q.cw;
    env.dry.channels = Q.dry_channels; env.dry.scale = Q.dry_scale; env.dry.index = Q.dry_index;
    for(uint32_t s = 0;s < B200MIX_MAX_SENDS;++s)
    {
        env.wet[s].channels = Q.wet_channels[s];
        env.wet[s].scale = Q.wet_scale[s]; env.wet[s].index = Q.wet_index[s];
    }
    float dir[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    float dry[B200MIX_MAX_DRY_CHANNELS];
    float *send = Q.send ? Q.send + size_t(i)*Q.num_sends*Q.cw : nullptr;
    float hrtf_gain = 0.0f; bool is_hrtf = false;
    for(uint32_t c = 0;c < Q.cd;++c) dry[c] = 0.0f;
    const bool ok = pm::calc_panning<DeviceMath>(P, r, env, &hrtf_gain, &is_hrtf, dir, dry, send);

    VoiceUpdate u;
    u.voice = sv.voice; u.buffer = sv.buffer; u.resampler = sv.resampler;
    u.flags = (sv.flags & ~uint32_t(B200MIX_VF_HRTF | kVfDirect)) | (is_hrtf ? uint32_t(B200MIX_VF_HRTF) : 0u);
    if(!ok) u.flags = (u.flags & ~3u) | uint32_t(B200MIX_VF_STOPPED);      // a bad mix map: silence the voice
    u.position = sv.position; u.position_frac = sv.position_frac;
    u.loop_start = sv.loop_start; u.loop_end = sv.loop_end;
    u.step = r.step;
    u.bsinc_sf = 0.0f; u.bsinc_m = 0u; u.bsinc_l = 0u; u.bsinc_off = 0u;
    if(sv.resampler >= B200MIX_RESAMPLER_FAST_BSINC12 && sv.resampler <= B200MIX_RESAMPLER_BSINC48)
    {
        const pm::BsincPrep st = pm::prepare_bsinc<DeviceMath>(
            Q.bsinc[(sv.resampler - B200MIX_RESAMPLER_FAST_BSINC12) >> 1], r.step);
        u.bsinc_sf = st.sf; u.bsinc_m = st.m; u.bsinc_l = st.l; u.bsinc_off = st.offset;
    }
    u.delay0 = 0u; u.delay1 = 0u; u.gain = hrtf_gain;
    for(uint32_t s = 0;s < uint32_t(kMaxSends);++s)
        u.send_slot[s] = s < Q.num_sends ? sv.send_slot[s] : B200MIX_NO_SLOT;
    u.has_coeffs = (is_hrtf && Q.ir) ? 1u : 0u;
    u.has_dry = is_hrtf ? 0u : 1u;
    Q.updates[i] = u;
    Q.dirs[i] = make_float4(dir[0], dir[1], dir[2], dir[3]);
    if(Q.dry) for(uint32_t c = 0;c < Q.cd;++c) Q.dry[size_t(i)*Q.cd + c] = dry[c];
    if(Q.gains_hflf)
    {
        float *g = Q.gains_hflf + size_t(i)*(1u + B200MIX_MAX_SENDS)*2u;
        g[0] = r.dry_gain_hf; g[1] = r.dry_gain_lf;
        for(uint32_t s = 0;s < B200MIX_MAX_SENDS;++s) { g[2+2*s] = r.wet_gain_hf[s]; g[3+2*s] = r.wet_gain_lf[s]; }
    }
}

// One thread per (source, path): the path's two shelf designs (alc/alu.cpp:1619-1656).
__global__ void __launch_bounds__(64) k_design_filters(const CalcVoicesParams Q)
{
    const uint32_t idx = blockIdx.x*blockDim.x + threadIdx.x;
    const uint32_t paths = 1u + Q.num_sends;
    const uint32_t i = idx / paths, path = idx - i*paths;
    if(i >= Q.n) return;
    const float *g = Q.gains_hflf + size_t(i)*(1u + B200MIX_MAX_SENDS)*2u + 2u*path;
    b200mix_voice_filter f;
    f.voice = Q.voices[i].voice;
    pm::design_filter<DeviceMath>(Q.props[i], Q.device_rate, path, g[0], g[1], f);
    FilterUpdate o;
    o.voice = f.voice; o.path = f.path; o.active = f.active;
    for(int k = 0;k < 5;++k) { o.lp[k] = f.lowpass[k]; o.hp[k] = f.highpass[k]; }
    Q.fupd[idx] = o;
}

} // namespace

cudaError_t launch_calc_voices(const CalcVoicesParams &Q, bool filters, cudaStream_t stream)
{
    k_calc_voices<<<(Q.n + 63u)/64u, 64, 0, stream>>>(Q);
    if(filters)
    {
        const uint32_t tot = Q.n*(1u + Q.num_sends);
        k_design_filters<<<(tot + 63u)/64u, 64, 0, stream>>>(Q);
    }
    return cudaGetLastError();
}

} // namespace b200mix
