// output_stage.hpp — the host's state of the output stage: the post-process after the mix (HRTF,
// ambisonic decode with the front stabilizer or BS2B, UHJ / TSME), the limiter, distance
// compensation and the interleaved output, with every device array they keep between updates.
// It decides in one place which of their kernels an update launches and with what state.  Host code.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/b200mix.h"
#include "mixer_kernels.cuh"
#include "device_memory.hpp"
#include "launch.hpp"

namespace b200mix {

static_assert(kPostMaxDry == B200MIX_MAX_DRY_CHANNELS, "k_post_hrtf_reduce: one thread per dry channel");

class OutputStage {
public:
    // What every update may use: the HRTF accumulator carry, the decoders' band-split scratch, the
    // interleaved output's staging, a UHJ / TSME device's IIR encoder state.  `err`: the device's
    // error string, which outlives the stage.
    int init(const b200mix_device_desc &dd, cudaStream_t stream, std::string &err)
    {
        dd_ = dd; s_ = stream; err_ = &err;
        const size_t temp = size_t(std::max(dd.dry_channels, 1u))*kLine;
        for(DevArray<float> &c : carry_) CUDA_TRY(*err_, c.alloc(2*kHrirLen, s_));
        CUDA_TRY(*err_, temp_.alloc(temp, s_));
        CUDA_TRY(*err_, temp2_.alloc(temp, s_));
        CUDA_TRY(*err_, d_outbuf_.alloc(size_t(kLine)*64*4));
        CUDA_TRY(*err_, h_outbuf_.alloc(size_t(kLine)*64*4));
        if(dd.post_process == B200MIX_POST_UHJ || dd.post_process == B200MIX_POST_TSME)
            CUDA_TRY(*err_, uhj_.state.alloc(64, s_));
        return B200MIX_OK;
    }

    // Why an update cannot run yet, or null.
    const char *missing() const
    {
        if(dd_.post_process == B200MIX_POST_HRTF && !hrtf_.channels) return "HRTF decoder not set";
        return dd_.post_process == B200MIX_POST_AMBIDEC && !ambi_.in ? "ambisonic decoder not set" : nullptr;
    }

    // The HRTF post-process stores RealOut's L/R (its only channels) instead of adding to them, so
    // the update need not clear RealOut (unless direct-channel voices were mixed into it).
    bool overwrites_real() const
    { return dd_.post_process == B200MIX_POST_HRTF && dd_.real_channels == 2 && dd_.real_left != dd_.real_right; }

    bool has_stabilizer() const { return stab_.center != B200MIX_NO_SLOT; }

    // ---- setters, on the mixer's GPU: each checks its arguments, derives the new state on the host,
    // allocates and fills it into a local and commits it, so a refused or failed call changes nothing.

    // DirectHrtfState: coeffs [cd][ir][2], hf_scale [cd], splitter [cd].
    int set_hrtf_decoder(uint32_t channels, uint32_t ir, const float *coeffs, const float *hf_scale,
        const float *splitter)
    {
        if(channels != dd_.dry_channels || ir > B200MIX_HRIR_LENGTH || !coeffs || !hf_scale || !splitter
            || dd_.post_process != B200MIX_POST_HRTF)
            return refuse(*err_, "set_hrtf_decoder: bad arguments");
        HrtfDecoder next{channels, ir};
        std::vector<float> st(size_t(channels)*4, 0.0f);
        for(uint32_t c = 0;c < channels;++c) st[c*4] = splitter[c];
        CUDA_TRY(*err_, fill(next.coef, reinterpret_cast<const float2*>(coeffs), size_t(channels)*ir));
        CUDA_TRY(*err_, fill(next.hfscale, hf_scale, channels));
        CUDA_TRY(*err_, fill(next.state, st.data(), st.size()));
        return commit(hrtf_, next);
    }

    // BFormatDec: gains [cd][real] (gains_lf null: single band).
    int set_ambi_decoder(uint32_t in_channels, const float *gains_hf, const float *gains_lf, float xover_coeff)
    {
        if(in_channels != dd_.dry_channels || !gains_hf || dd_.post_process != B200MIX_POST_AMBIDEC)
            return refuse(*err_, "set_ambi_decoder: bad arguments");
        const size_t n = size_t(in_channels)*dd_.real_channels;
        AmbiDecoder next{in_channels, gains_lf != nullptr};
        std::vector<float> st(size_t(in_channels)*4, 0.0f);
        for(uint32_t c = 0;c < in_channels;++c) st[c*4] = xover_coeff;
        CUDA_TRY(*err_, fill(next.hf, gains_hf, n));
        if(gains_lf) CUDA_TRY(*err_, fill(next.lf, gains_lf, n));
        CUDA_TRY(*err_, fill(next.state, st.data(), st.size()));
        return commit(ambi_, next);
    }

    // 0 = the IIR encoder, 256 / 512 = UhjEncoder<N>; either starts from a cleared state.  *delay
    // (nullable): EncoderBase::getDelay().
    int set_uhj_encoder(uint32_t filter_length, uint32_t *delay)
    {
        if((dd_.post_process != B200MIX_POST_UHJ && dd_.post_process != B200MIX_POST_TSME) || dd_.dry_channels < 3
            || (filter_length != 0 && filter_length != 256 && filter_length != 512))
            return refuse(*err_, "set_uhj_encoder: needs a UHJ device and a length of 0, 256 or 512");
        UhjEncoder next{filter_length};
        CUDA_TRY(*err_, next.state.alloc(64, s_));
        std::vector<float> coef(256, 0.0f);
        if(filter_length)
        {
            CUDA_TRY(*err_, next.fir_state.alloc(kUhjFirStateFloats, s_));
            // SegmentedFilter's desired response (core/allpass_conv.hpp:56-75): Blackman-Nuttall
            // windowed 2/(pi k) at the odd taps
            const uint32_t half = filter_length/2u;
            const double pi = 3.14159265358979323846;
            for(uint32_t i = 0;i < half;++i)
            {
                const int k = int(half) - int(i*2u + 1u);
                const double w = 2.0*pi/double(half - 1u) * double(i);
                const double window = 0.3635819 - 0.4891775*std::cos(w) + 0.1365995*std::cos(2.0*w)
                    - 0.0106411*std::cos(3.0*w);
                coef[i] = float(window * 2.0 / (pi * double(k)));
            }
            CUDA_TRY(*err_, fill(next.fir_coef, coef.data(), coef.size()));
        }
        if(int rc = commit(uhj_, next)) return rc;
        if(delay) *delay = filter_length ? filter_length/2u + 128u : 1u;
        return B200MIX_OK;
    }

    // B200MIX_NO_SLOT removes it; the filter states start cleared.
    int set_front_stabilizer(uint32_t center_channel, float splitter_coeff)
    {
        Stabilizer next{center_channel, splitter_coeff};
        if(center_channel != B200MIX_NO_SLOT)
        {
            if(dd_.post_process != B200MIX_POST_AMBIDEC || center_channel >= dd_.real_channels || !stereo()
                || center_channel == dd_.real_left || center_channel == dd_.real_right || dd_.real_channels > 32u)
                return refuse(*err_, "set_front_stabilizer: needs an ambisonic-decode device with left, right and centre outputs");
            CUDA_TRY(*err_, next.state.alloc(4 + 32, s_));
            CUDA_TRY(*err_, cudaFuncSetAttribute(k_post_stabilizer, cudaFuncAttributeMaxDynamicSharedMemorySize,
                int(size_t(2u + dd_.real_channels)*kLine*sizeof(float))));
        }
        return commit(stab_, next);
    }

    // Level 0 removes it; the filter history starts cleared.
    int set_bs2b(uint32_t level)
    {
        if(level > 6 || dd_.post_process != B200MIX_POST_AMBIDEC || !stereo())
            return refuse(*err_, "set_bs2b: needs a stereo ambisonic-decode device and a level of 0..6");
        Bs2b next{level};
        float h[9] = {};
        if(level)
        {
            // init(), core/bs2b.cpp:41-91 (same float expressions, host libm)
            static const float tab[6][4] = {
                {360.0f,  501.0f, 0.398107170553497f, 0.205671765275719f},
                {500.0f,  711.0f, 0.459726988530872f, 0.228208484414988f},
                {700.0f, 1021.0f, 0.530884444230988f, 0.250105790667544f},
                {360.0f,  494.0f, 0.316227766016838f, 0.168236228897329f},
                {500.0f,  689.0f, 0.354813389233575f, 0.187169483835901f},
                {700.0f,  975.0f, 0.398107170553497f, 0.205671765275719f}};
            const float Fc_lo = tab[level-1][0], Fc_hi = tab[level-1][1];
            const float G_lo = tab[level-1][2], G_hi = tab[level-1][3];
            const float pi = 3.14159265358979323846f;
            const float g = 1.0f / (1.0f - G_hi + G_lo);
            float x = std::exp(-pi*2.0f*Fc_lo/float(dd_.sample_rate));
            h[4+1] = x; h[4+0] = G_lo * (1.0f - x) * g;
            x = std::exp(-pi*2.0f*Fc_hi/float(dd_.sample_rate));
            h[4+4] = x; h[4+2] = (1.0f - G_hi * (1.0f - x)) * g; h[4+3] = -x * g;
            CUDA_TRY(*err_, fill(next.buf, h, 9));
            CUDA_TRY(*err_, next.direct.alloc(2*kLine, s_));
        }
        return commit(bs2b_, next);
    }

    // Null removes it.  Compressor::Create (core/mastering.cpp:108-166): the same float/double
    // expressions, by the host's libm, so the derived constants are the reference's bit for bit.
    int set_limiter(const b200mix_limiter_desc *p, uint32_t *look_ahead)
    {
        if(p && p->struct_size != sizeof(*p)) return refuse(*err_, "set_limiter: struct_size");
        Limiter next;
        LimiterDev h{};
        if(p)
        {
            const float rate = float(dd_.sample_rate);
            auto clampf = [](float v, float lo, float hi) { return v < lo ? lo : (hi < v ? hi : v); };
            h.look_ahead = uint32_t(clampf(std::round(p->look_ahead_time*rate), 0.0f, float(kLine) - 1.0f));
            const uint32_t hold = uint32_t(clampf(std::round(p->hold_time*rate), 0.0f, float(kLine) - 1.0f));
            h.flags = p->auto_flags & 31u;
            if(!(h.flags & B200MIX_LIM_AUTO_POSTGAIN)) h.flags &= ~uint32_t(B200MIX_LIM_AUTO_DECLIP);
            h.num_chans = dd_.real_channels;
            h.pre_gain = std::pow(10.0f, p->pre_gain_db / 20.0f);
            h.post_gain = float(std::log(10.0)/20.0 * double(p->post_gain_db));
            h.threshold = float(std::log(10.0)/20.0 * double(p->threshold_db));
            h.slope = 1.0f/std::max(1.0f, p->ratio) - 1.0f;
            h.knee = float(std::max(0.0, std::log(10.0)/20.0 * double(p->knee_db)));
            h.attack = std::max(1.0f, p->attack_time * rate);
            h.release = std::max(1.0f, p->release_time * rate);
            if(h.flags & B200MIX_LIM_AUTO_KNEE) h.slope = -1.0f;
            // the hold needs a look-ahead and more than one sample (:141-153)
            h.hold = (h.look_ahead > 0 && hold > 1) ? hold : 0u;
            h.crest_coeff = std::exp(-1.0f / (0.200f * rate));
            h.gain_estimate = h.threshold * -0.5f * h.slope;
            h.adapt_coeff = std::exp(-1.0f / (2.0f * rate));
            for(float &v : h.hold_hist) v = -INFINITY;
            CUDA_TRY(*err_, fill(next.lim, &h, 1));
            CUDA_TRY(*err_, next.delay.alloc(size_t(std::max(dd_.real_channels, 1u))*kLine, s_));
        }
        if(int rc = commit(limiter_, next)) return rc;
        if(look_ahead) *look_ahead = h.look_ahead;
        return B200MIX_OK;
    }

    // The first `channels` RealOut channels' delays (< kLine) and gains; 0 channels removes it.
    int set_distance_comp(uint32_t channels, const uint32_t *delays, const float *gains)
    {
        DistComp next;
        std::vector<uint32_t> hd(dd_.real_channels, 0u);
        std::vector<float> hg(dd_.real_channels, 1.0f);
        if(channels)
        {
            if(channels > dd_.real_channels || !delays || !gains) return refuse(*err_, "set_distance_comp: bad arguments");
            for(uint32_t c = 0;c < channels;++c)
            {
                if(delays[c] >= kLine) return refuse(*err_, "set_distance_comp: delay >= 1024");
                hd[c] = delays[c]; hg[c] = gains[c];
            }
            CUDA_TRY(*err_, fill(next.delay, hd.data(), hd.size()));
            CUDA_TRY(*err_, fill(next.gain, hg.data(), hg.size()));
            CUDA_TRY(*err_, next.buf.alloc(size_t(dd_.real_channels)*kLine, s_));
        }
        return commit(dc_, next);
    }

    // The post-process (alc/alu.cpp:2252-2256) of the dry mix into RealOut.  The HRTF device's also
    // sums the HRIR FIR's partial rows; it starts under the FIR's tail when the FIR was the last
    // launch (`fir_done`: the launch count once the FIR was launched).  `dry_active`: the dry mix
    // may be non-silent.  `direct`: direct-channel voices were mixed into RealOut ahead of it.
    int post(const float *dry, float *real, const float *partial, uint32_t rows, bool dry_active,
        bool direct, uint64_t fir_done, uint32_t frames, uint64_t &launches)
    {
        switch(dd_.post_process)
        {
        case B200MIX_POST_HRTF:
        {
            PostHrtfParams Q{.partial = partial, .rows = rows, .carry_in = carry_[carry_idx_],
                .carry_out = carry_[carry_idx_^1], .dry = dry, .real = real, .dec_coef = hrtf_.coef,
                .dec_hfscale = hrtf_.hfscale, .dec_state = hrtf_.state, .temp = temp_, .frames = frames,
                .cd = dd_.dry_channels, .dec_ir = hrtf_.ir, .real_left = dd_.real_left, .real_right = dd_.real_right,
                .dry_active = dry_active};
            if(dry_active)
                CUDA_TRY(*err_, launch_ex(s_, launches, false, k_post_hrtf_split, dim3(dd_.dry_channels), dim3(32), 0, Q));
            Q.overwrite = overwrites_real() && !direct ? 1u : 0u;
            // straight behind the HRIR FIR (no kernel of the dry bus, sends, effects or band split in
            // between), it is scheduled under the FIR's last CTAs
            CUDA_TRY(*err_, launch_ex(s_, launches, launches == fir_done, k_post_hrtf_reduce,
                dim3((frames + kHrirLen + kPostTile - 1)/kPostTile, 2), dim3(1024), 0, Q));
            carry_idx_ ^= 1;
            break;
        }
        case B200MIX_POST_AMBIDEC:
        {
            const PostAmbiParams Q{.dry = dry, .real = real, .gains_hf = ambi_.hf, .gains_lf = ambi_.lf,
                .split_state = ambi_.state, .temp_hf = temp_, .temp_lf = temp2_, .frames = frames,
                .cd = dd_.dry_channels, .real_channels = dd_.real_channels, .dual = ambi_.dual};
            // BS2B filters the decode only: the direct L/R signal is moved out first (alc/alu.cpp:414-423)
            const bool bs2bDirect = direct && stab_.center == B200MIX_NO_SLOT && bs2b_.level;
            if(bs2bDirect)
                for(uint32_t k = 0;k < 2;++k)
                {
                    float *ch = real + size_t(k ? dd_.real_right : dd_.real_left)*kLine;
                    CUDA_TRY(*err_, cudaMemcpyAsync(bs2b_.direct + k*kLine, ch, frames*sizeof(float),
                        cudaMemcpyDeviceToDevice, s_));
                    CUDA_TRY(*err_, cudaMemsetAsync(ch, 0, frames*sizeof(float), s_));
                }
            if(ambi_.dual) CUDA_TRY(*err_, launch_ex(s_, launches, false, k_post_ambi_split, dim3(1), dim3(32), 0, Q));
            CUDA_TRY(*err_, launch_ex(s_, launches, false, k_post_ambi_mix, dim3((dd_.real_channels*frames + 127)/128),
                dim3(128), 0, Q));
            // with both installed, the stabilizer runs and BS2B does not (a device with a stabilizer
            // takes no direct-channel voices)
            if(stab_.center != B200MIX_NO_SLOT)
            {
                const float halfPi = 3.14159265358979323846f*0.5f;
                const StabParams S{.real = real, .state = stab_.state, .frames = frames,
                    .real_channels = dd_.real_channels, .lidx = dd_.real_left, .ridx = dd_.real_right,
                    .cidx = stab_.center, .coeff = stab_.coeff,
                    .mid_lf = std::cos(1.0f/3.0f * halfPi), .mid_hf = std::cos(1.0f/4.0f * halfPi),
                    .center_lf = std::sin(1.0f/3.0f * halfPi), .center_hf = std::sin(1.0f/4.0f * halfPi)};
                CUDA_TRY(*err_, launch_ex(s_, launches, false, k_post_stabilizer, dim3(1), dim3(32u*dd_.real_channels),
                    size_t(2u + dd_.real_channels)*kLine*sizeof(float), S));
            }
            else if(bs2b_.level)
            {
                const Bs2bParams B{real, bs2b_.buf, bs2b_.buf + 4, frames, dd_.real_left, dd_.real_right,
                    bs2bDirect ? bs2b_.direct.get() : nullptr};
                CUDA_TRY(*err_, launch_ex(s_, launches, false, k_post_bs2b, dim3(1), dim3(128), 0, B));
            }
            break;
        }
        case B200MIX_POST_UHJ: case B200MIX_POST_TSME:
        {
            const MatrixEncSpec spec = dd_.post_process == B200MIX_POST_TSME ? kTsmeEncSpec : kUhjEncSpec;
            if(uhj_.fir)
                CUDA_TRY(*err_, launch_ex(s_, launches, false, k_post_uhj_fir, dim3(1), dim3(1024), 0, PostUhjFirParams{dry,
                    real, uhj_.fir_state, uhj_.fir_coef, frames, dd_.real_left, dd_.real_right, uhj_.fir, spec}));
            else
                CUDA_TRY(*err_, launch_ex(s_, launches, false, k_post_uhj, dim3(1), dim3(1024), 0, PostUhjParams{dry, real,
                    uhj_.state, nullptr /* scratch: k_post_uhj reads none */, frames, dd_.real_left, dd_.real_right, spec}));
            break;
        }
        }
        return B200MIX_OK;
    }

    // The nonlinear output stage on RealOut: the limiter, then speaker distance compensation
    // (alc/alu.cpp:2446-2450).
    int finish(float *real, uint32_t frames, uint64_t &launches)
    {
        if(limiter_.lim)
            CUDA_TRY(*err_, launch_ex(s_, launches, false, k_limiter, dim3(1), dim3(1024), 0,
                LimiterParams{limiter_.lim, real, limiter_.delay, frames}));
        if(dc_.delay)
            CUDA_TRY(*err_, launch_ex(s_, launches, false, k_distance_comp, dim3(dd_.real_channels), dim3(1024), 0,
                DistCompParams{real, dc_.buf, dc_.delay, dc_.gain, frames}));
        return B200MIX_OK;
    }

    // Dither and conversion of RealOut into the staging (k_output_write), and its copy to the host.
    int interleave(const float *real, uint32_t frames, uint32_t frame_step, uint32_t out_type,
        float dither_depth, uint32_t seed, uint64_t &launches)
    {
        static const size_t sz[] = {1, 1, 2, 2, 4, 4, 4};
        const OutputParams Q{.real = real, .out = d_outbuf_, .frames = frames, .channels = dd_.real_channels,
            .frame_step = frame_step, .out_type = out_type, .seed = seed, .dither_depth = dither_depth};
        const uint32_t total = frames*frame_step;
        CUDA_TRY(*err_, launch_ex(s_, launches, false, k_output_write, dim3((total + 255)/256), dim3(256), 0, Q));
        out_bytes_ = size_t(total)*sz[out_type];
        CUDA_TRY(*err_, cudaMemcpyAsync(h_outbuf_, d_outbuf_, out_bytes_, cudaMemcpyDeviceToHost, s_));
        return B200MIX_OK;
    }

    // The last interleave()'s output, once the stream has synchronised.
    void copy_interleaved(void *out) const { std::memcpy(out, h_outbuf_, out_bytes_); }

private:
    // The parts a setter replaces whole.  The decoders' `state` is [cd][4] = BandSplitter coeff,
    // lp_z1, lp_z2, ap_z1; the stabilizer's [0..2] MidFilter, [4+i] ChannelFilters[i].mApZ1; BS2B's
    // `buf` [0..3] history, [4..8] coefficients.
    struct HrtfDecoder { uint32_t channels{0}, ir{0}; DevArray<float2> coef; DevArray<float> hfscale, state; };
    struct AmbiDecoder { uint32_t in{0}; bool dual{false}; DevArray<float> hf, lf, state; };
    struct UhjEncoder { uint32_t fir{0}; DevArray<float> state, fir_state, fir_coef; };   // fir 0: IIR
    struct Stabilizer { uint32_t center{B200MIX_NO_SLOT}; float coeff{0.0f}; DevArray<float> state; };
    struct Bs2b { uint32_t level{0}; DevArray<float> buf, direct; };   // level 0: off; direct: [2][1024] L/R moved out
    struct Limiter { DevArray<LimiterDev> lim; DevArray<float> delay; };   // DeviceBase::Limiter, Compressor::mDelay
    struct DistComp { DevArray<uint32_t> delay; DevArray<float> gain, buf; };   // DeviceBase::ChannelDelays

    bool stereo() const
    { return dd_.real_left != dd_.real_right && dd_.real_left < dd_.real_channels && dd_.real_right < dd_.real_channels; }

    // A new array holding `count` elements of host memory, copied on the stream: the setter's
    // commit() waits for the copy, so the source must live until then.
    template<typename T>
    cudaError_t fill(DevArray<T> &a, const T *src, size_t count)
    {
        const cudaError_t e = a.alloc(count);
        return e != cudaSuccess || !count ? e : cudaMemcpyAsync(a.get(), src, count*sizeof(T), cudaMemcpyHostToDevice, s_);
    }

    // Once the stream is idle (queued kernels may still read the part being replaced, and the new
    // part's fills have landed), `next` replaces `part`.
    template<typename Part>
    int commit(Part &part, Part &next)
    {
        CUDA_TRY(*err_, cudaStreamSynchronize(s_));
        part = std::move(next);
        return B200MIX_OK;
    }

    b200mix_device_desc dd_{};
    cudaStream_t s_{nullptr};
    std::string *err_{nullptr};
    HrtfDecoder hrtf_; AmbiDecoder ambi_; UhjEncoder uhj_; Stabilizer stab_; Bs2b bs2b_;   // channels / in 0: not set
    Limiter limiter_; DistComp dc_;
    DevArray<float> carry_[2];                       // [2][kHrirLen] HRTF accumulator carry, ping-pong
    int carry_idx_{0};
    DevArray<float> temp_, temp2_;                   // [cd][1024] band-split dry (HF, LF)
    DevArray<char> d_outbuf_; PinnedArray<char> h_outbuf_;   // interleaved output staging
    size_t out_bytes_{0};
};


} // namespace b200mix
