// slot_table.hpp — the effect slots from install to launch: each slot's record (the device's copy is
// uploaded from the table) and the memory it points into, the host halves of the reverb's pipeline
// state machine and of the EFX effects, and run(), which launches an update's slot kernels.  Host code.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "../../include/b200mix.h"
#include "effect_kernels.cuh"
#include "efx_kernels.hpp"
#include "device_memory.hpp"
#include "launch.hpp"
#include "resampler_tables.hpp"

namespace b200mix {

class SlotTable {
public:
    // ReverbState's PipelineState (reverb.cpp:1243-1280, 1840-1878); StartFade is Fading from the start
    enum class Pipeline { Fading, Cleanup, Normal };
    struct Reverb {
        int cur{0};                             // current pipeline object
        Pipeline state{Pipeline::Normal};
        uint32_t fade[2]{1u, 1u};               // mFadeSampleCount per pipeline object
        uint32_t offset{0};                     // mOffset
        ReverbDev h[2]{};                       // host mirrors of the device's ReverbDev[2]

        // ReverbPipeline::clear (reverb.cpp:550-566) on object `obj`'s mirror: the parameters
        // clear() resets, and the filter and tap state (z_lp up to offset); the caller clears the delay lines
        void clear(int obj)
        {
            ReverbDev &r = h[obj];
            std::memset(r.early_tap, 0, sizeof(r.early_tap)); std::memset(r.late_tap, 0, sizeof(r.late_tap));
            r.early_tap_coeff = 0.0f; r.mod_step = 1u; r.mod_depth = 0.0f;
            std::memset(r.z_lp, 0, offsetof(ReverbDev, offset) - offsetof(ReverbDev, z_lp));
            r.offset = offset;
        }
    };
    // An EFX effect's last parameters, and the phase indices update() rescales (mIndex, mLfoOffset)
    struct Efx { EfxParams p{}; uint32_t mod_index{0}, mod_range{1}, lfo_offset{0}, lfo_range{1}; };
    struct Slot {
        SlotRec rec{};                          // type 0: no effect; the target outlives the effect
        Reverb rv;
        Efx efx;
        std::vector<DevArray<char>> mem;        // what the record and the effect's device state point into
    };

    // The slots of a device with sends, their device records, the twiddles and gCubicTable (the reverb's
    // modulation taps); a device without sends has no slots.  `err`: the device's error string.
    int init(const b200mix_device_desc &dd, uint32_t num_sms, cudaStream_t stream, std::string &err)
    {
        dd_ = dd; num_sms_ = num_sms; s_ = stream; err_ = &err;
        if(!dd.max_slots || !dd.wet_channels || !dd.num_sends) return B200MIX_OK;
        slots_.resize(dd.max_slots); recs_.resize(dd.max_slots);
        CUDA_TRY(*err_, d_slots_.alloc(dd.max_slots, s_));
        CUDA_TRY(*err_, cudaFuncSetAttribute(k_conv_mac, cudaFuncAttributeMaxDynamicSharedMemorySize, int(sizeof(ConvMacSmem))));
        CUDA_TRY(*err_, cudaFuncSetAttribute(k_reverb_upmix, cudaFuncAttributeMaxDynamicSharedMemorySize, int(8*kLine*sizeof(float))));
        std::vector<float2> tw(128);
        for(int k = 0;k < 128;++k)
        {
            const double a = -2.0*3.14159265358979323846*double(k)/256.0;
            tw[k] = make_float2(float(std::cos(a)), float(std::sin(a)));
        }
        const std::vector<float> cf = BuildCubicFilter();
        CUDA_TRY(*err_, cubic_.alloc(cf.size()));
        CUDA_TRY(*err_, b200mix::upload(cubic_, cf, s_));
        CUDA_TRY(*err_, twiddle_.alloc(tw.size()));
        CUDA_TRY(*err_, b200mix::upload(twiddle_, tw, s_));
        return B200MIX_OK;
    }
    uint32_t size() const { return uint32_t(slots_.size()); }
    bool active() const { return active_; }                 // a slot has an effect
    bool ever_installed() const { return installed_; }      // since create: the slots may have fed Dry

    // ---- setters: each checks the whole call before it writes anything, then builds the new state in
    // locals and commits it once the device has it, so a refused or failed call changes nothing.

    int disable(uint32_t sl)
    {
        if(sl >= size()) return refuse(*err_, "slot_disable: bad slot");
        return exchange(slots_[sl], empty(sl));
    }

    int convolution(uint32_t sl, uint32_t ir_channels, uint32_t ir_frames, const float *ir)
    {
        if(sl >= size() || !ir_channels || ir_channels > 16 || !ir_frames || !ir)
            return refuse(*err_, "slot_convolution: bad arguments (or the device has no sends/slots)");
        // mNumConvolveSegs (alc/effects/convolution.cpp:375-376)
        const uint32_t nseg = std::max<uint32_t>((ir_frames + kConvBlock - 1)/kConvBlock, 2u) - 1u;

        // Filter spectra: segment s holds taps [128(s+1), 128(s+2)), zero padded to 256,
        // transformed in f64 and scaled by 1/256 (convolution.cpp:425-468); layout is ours.
        std::vector<float> H(size_t(ir_channels)*nseg*kConvFft, 0.0f), head(size_t(ir_channels)*kConvBlock, 0.0f);
        std::vector<double> cs(kConvFft), sn(kConvFft);
        for(int k = 0;k < kConvFft;++k)
        {
            cs[k] = std::cos(2.0*3.14159265358979323846*k/kConvFft);
            sn[k] = std::sin(2.0*3.14159265358979323846*k/kConvFft);
        }
        for(uint32_t c = 0;c < ir_channels;++c)
        {
            const float *h = ir + size_t(c)*ir_frames;
            for(uint32_t k = 0;k < uint32_t(kConvBlock) && k < ir_frames;++k) head[c*kConvBlock + k] = h[k];
            for(uint32_t sg = 0;sg < nseg;++sg)
            {
                const size_t base = size_t(kConvBlock)*(sg + 1);
                float *dst = H.data() + (size_t(c)*nseg + sg)*kConvFft;
                const uint32_t cnt = base < ir_frames ? std::min<uint32_t>(kConvBlock, uint32_t(ir_frames - base)) : 0u;
                for(int bin = 0;bin <= kConvBlock;++bin)
                {
                    double re = 0.0, im = 0.0;
                    for(uint32_t j = 0;j < cnt;++j)
                    {
                        const int ph = int((uint64_t(bin)*j) % kConvFft);
                        re += double(h[base + j])*cs[ph];
                        im -= double(h[base + j])*sn[ph];
                    }
                    const double sc = 1.0/double(kConvFft);
                    if(bin == 0) dst[0] = float(re*sc);
                    else if(bin == kConvBlock) dst[1] = float(re*sc);
                    else { dst[bin*2] = float(re*sc); dst[bin*2+1] = float(im*sc); }
                }
            }
        }
        Slot next = empty(sl);
        SlotRec &r = next.rec;
        r.type = B200MIX_EFFECT_CONVOLUTION; r.channels = ir_channels; r.frames = ir_frames; r.segs = nseg;
        if(int rc = alloc(next, r.ring, 1)) return rc;
        if(int rc = alloc(next, r.H, size_t(ir_channels)*nseg*kConvFft)) return rc;
        if(int rc = alloc(next, r.X, size_t(nseg + kConvMaxBlocks)*kConvFft)) return rc;
        if(int rc = alloc(next, r.head, size_t(ir_channels)*kConvBlock)) return rc;
        if(int rc = alloc(next, r.inbuf, kConvFft)) return rc;
        if(int rc = alloc(next, r.ov, size_t(ir_channels)*kConvFft)) return rc;
        if(int rc = alloc(next, r.yspec, size_t(ir_channels)*kConvMaxChunks*kConvMaxBlocks*kConvFft)) return rc;
        if(int rc = alloc(next, r.lines, size_t(ir_channels)*kLine)) return rc;
        if(int rc = alloc(next, r.gains, size_t(ir_channels)*32)) return rc;
        if(int rc = alloc(next, r.gtgt, size_t(ir_channels)*32)) return rc;
        CUDA_TRY(*err_, cudaMemcpyAsync(r.H, H.data(), H.size()*sizeof(float), cudaMemcpyHostToDevice, s_));
        CUDA_TRY(*err_, cudaMemcpyAsync(r.head, head.data(), head.size()*sizeof(float), cudaMemcpyHostToDevice, s_));
        return exchange(slots_[sl], std::move(next));
    }

    int reverb(uint32_t sl, const b200mix_reverb_params *p)
    {
        if(sl >= size() || !p || p->struct_size != sizeof(*p))
            return refuse(*err_, "slot_reverb: bad arguments (or the device has no sends/slots)");
        if(int rc = check_reverb(p)) return rc;
        Slot next = empty(sl);
        SlotRec &r = next.rec;
        Reverb &R = next.rv;
        r.type = B200MIX_EFFECT_REVERB; r.channels = 16;       // 2 pipeline objects x (4 early + 4 late) lines
        float *main_d = nullptr;
        if(int rc = alloc(next, main_d, size_t(4)*p->main_len)) return rc;
        for(int obj = 0;obj < 2;++obj)
        {
            ReverbDev &h = R.h[obj];
            h.main_len = p->main_len; h.late_in_len = p->late_in_len; h.early_ap_len = p->early_ap_len;
            h.early_len = p->early_len; h.late_ap_len = p->late_ap_len; h.late_len = p->late_len;
            // a pipeline that has not been updated yet is in ReverbPipeline::clear()'s state
            fill_reverb(h, p);
            R.clear(obj);
            h.main_d = main_d;
            if(int rc = alloc(next, h.late_in, size_t(4)*p->late_in_len)) return rc;
            if(int rc = alloc(next, h.early_ap, size_t(4)*p->early_ap_len)) return rc;
            if(int rc = alloc(next, h.early_d, size_t(4)*p->early_len)) return rc;
            if(int rc = alloc(next, h.late_ap, size_t(4)*p->late_ap_len)) return rc;
            if(int rc = alloc(next, h.late_d, size_t(4)*p->late_len)) return rc;
        }
        // deviceUpdate leaves DeviceClear; the first update is a full one: it switches to pipeline
        // object 1 and goes straight to Normal (reverb.cpp:1243-1280)
        R.cur = 1;
        fill_reverb(R.h[1], p);
        R.fade[1] = p->fade_samples; R.fade[0] = 1u;
        ReverbDev *dev = nullptr;
        if(int rc = alloc(next, dev, 2)) return rc;
        r.H = reinterpret_cast<float*>(dev);
        if(int rc = alloc(next, r.lines, size_t(16)*kLine)) return rc;
        if(int rc = alloc(next, r.gains, size_t(16)*32)) return rc;
        if(int rc = alloc(next, r.gtgt, size_t(16)*32)) return rc;
        CUDA_TRY(*err_, cudaMemcpyAsync(dev, R.h, 2*sizeof(ReverbDev), cudaMemcpyHostToDevice, s_));
        return exchange(slots_[sl], std::move(next));
    }

    // New reverb parameters with the installed line lengths: a full update cross-fades to the other
    // pipeline object (reverb.cpp:1275-1279), else the current object takes them.
    int reverb_update(uint32_t sl, const b200mix_reverb_params *p, uint32_t full_update)
    {
        if(sl >= size() || !p || p->struct_size != sizeof(*p) || slots_[sl].rec.type != B200MIX_EFFECT_REVERB)
            return refuse(*err_, "slot_reverb_update: no reverb installed on this slot / bad arguments");
        if(int rc = check_reverb(p)) return rc;
        Slot &S = slots_[sl];
        const ReverbDev &h0 = S.rv.h[0];
        if(p->main_len != h0.main_len || p->late_in_len != h0.late_in_len || p->early_ap_len != h0.early_ap_len
            || p->early_len != h0.early_len || p->late_ap_len != h0.late_ap_len || p->late_len != h0.late_len)
            return refuse(*err_, "slot_reverb_update: line lengths differ from the installed ones");
        ReverbDev *dev = reinterpret_cast<ReverbDev*>(S.rec.H);
        Reverb R = S.rv;
        if(full_update)
        {
            R.state = Pipeline::Fading;
            R.cur ^= 1;
            const int old = R.cur ^ 1;
            R.h[old].early_tap_coeff = 0.0f;
            CUDA_TRY(*err_, cudaMemcpyAsync(&dev[old].early_tap_coeff, &R.h[old].early_tap_coeff, sizeof(float),
                cudaMemcpyHostToDevice, s_));
            // the object coming back into use has not advanced mOffset while it was idle
            R.h[R.cur].offset = R.offset;
            CUDA_TRY(*err_, cudaMemcpyAsync(&dev[R.cur].offset, &R.h[R.cur].offset, sizeof(uint32_t),
                cudaMemcpyHostToDevice, s_));
        }
        fill_reverb(R.h[R.cur], p);
        R.fade[R.cur] = p->fade_samples;
        // the parameter prefix of ReverbDev (everything before the filter states)
        CUDA_TRY(*err_, cudaMemcpyAsync(dev + R.cur, &R.h[R.cur], offsetof(ReverbDev, z_lp), cudaMemcpyHostToDevice, s_));
        CUDA_TRY(*err_, cudaStreamSynchronize(s_));
        S.rv = R;
        refresh();                                      // the up-mix flag follows the parameters
        return B200MIX_OK;
    }

    // An EFX effect (echo .. pitch shifter): EffectState::update on the installed effect when its kind
    // and delay lines stay, else EffectState::deviceUpdate on a new one.
    int efx(uint32_t sl, const b200mix_efx_props *props, const b200mix_efx_target *target)
    {
        if(sl >= size() || !props || !target || props->struct_size != sizeof(*props)
            || target->struct_size != sizeof(*target) || props->type < B200MIX_EFFECT_ECHO
            || props->type > B200MIX_EFFECT_PSHIFTER)
            return refuse(*err_, "slot_efx: bad arguments (or the device has no sends/slots)");
        if(target->wet_channels != dd_.wet_channels
            || target->out_channels != (slots_[sl].rec.target != B200MIX_NO_SLOT ? dd_.wet_channels : dd_.dry_channels))
            return refuse(*err_, "slot_efx: the target maps do not match the device's wet / output mix");
        EfxParams P;
        if(int rc = efx_update(*props, *target, P))
        { *err_ = rc == B200MIX_ERR_UNSUPPORTED ? "slot_efx: not supported in this configuration (see b200mix.h)"
            : "slot_efx: bad properties / maps"; return rc; }
        if(P.type == B200MIX_EFFECT_AUTOWAH && P.lines > kEfxMaxLines - 2u)
        { *err_ = "slot_efx: autowah handles up to 14 wet channels"; return B200MIX_ERR_UNSUPPORTED; }
        if(!efx_ready_) { CUDA_TRY(*err_, efx_kernels_init()); efx_ready_ = true; }
        Slot &S = slots_[sl];
        if(S.rec.type != props->type || S.efx.p.lines != P.lines || S.efx.p.echo_len != P.echo_len
            || S.efx.p.cho_len != P.cho_len)
        {
            // EffectState::deviceUpdate: new state, cleared
            Slot next = empty(sl);
            SlotRec &r = next.rec;
            EfxDev h{};
            h.p = P; h.comp_env = 1.0f;
            r.type = props->type; r.channels = P.lines; r.fade_len = P.fade_len;
            EfxDev *dev = nullptr;
            if(int rc = alloc(next, dev, 1)) return rc;
            if(int rc = alloc(next, r.lines, size_t(P.lines)*kLine)) return rc;
            if(int rc = alloc(next, r.gains, size_t(P.lines)*32)) return rc;
            if(int rc = alloc(next, r.gtgt, size_t(P.lines)*32)) return rc;
            if(P.echo_len) { if(int rc = alloc(next, h.echo_buf, P.echo_len)) return rc; }
            if(P.cho_len) { if(int rc = alloc(next, h.cho_buf, size_t(4)*P.cho_len)) return rc; }
            if(P.type == B200MIX_EFFECT_FSHIFTER)
            {   // FshifterState::deviceUpdate (fshifter.cpp:140-148): cleared FIFOs, mPos = HilSize - HilStep
                if(int rc = alloc(next, h.fs_in, size_t(4)*1024)) return rc;
                if(int rc = alloc(next, h.fs_outfifo, size_t(4)*256)) return rc;
                if(int rc = alloc(next, h.fs_accum, size_t(4)*1024)) return rc;
                h.fs_count = 0u; h.fs_pos = 1024u - 256u;
            }
            if(P.type == B200MIX_EFFECT_PSHIFTER)
            {   // PshifterState::deviceUpdate (pshifter.cpp:131-145): cleared FIFOs and phases, mPos = StftSize - StftStep
                if(int rc = alloc(next, h.ps_fifo, size_t(9)*1024)) return rc;
                if(int rc = alloc(next, h.ps_accum, size_t(9)*1024)) return rc;
                if(int rc = alloc(next, h.ps_last, size_t(513))) return rc;
                if(int rc = alloc(next, h.ps_sum, size_t(513))) return rc;
                h.ps_count = 0u; h.ps_pos = 1024u - 128u;
            }
            r.H = reinterpret_cast<float*>(dev);
            CUDA_TRY(*err_, cudaMemcpyAsync(dev, &h, sizeof(h), cudaMemcpyHostToDevice, s_));
            if(int rc = efx_gains(r, P)) return rc;
            next.efx = Efx{P, 0u, P.mod_range ? P.mod_range : 1u, 0u, P.cho_lfo_range ? P.cho_lfo_range : 1u};
            return exchange(slots_[sl], std::move(next));
        }
        EfxDev *dev = reinterpret_cast<EfxDev*>(S.rec.H);
        Efx H = S.efx;
        // EffectState::update: new parameters, state kept.  The ring modulator rescales its
        // phase index to the new range (modulator.cpp:117-118); the host mirrors the index
        CUDA_TRY(*err_, cudaMemcpyAsync(&dev->p, &P, sizeof(EfxParams), cudaMemcpyHostToDevice, s_));
        if(props->type == B200MIX_EFFECT_MODULATOR)
        {
            H.mod_index = uint32_t(uint64_t(H.mod_index) * P.mod_range_new / H.mod_range);
            H.mod_range = P.mod_range;
            CUDA_TRY(*err_, cudaMemcpyAsync(&dev->mod_index, &H.mod_index, sizeof(uint32_t), cudaMemcpyHostToDevice, s_));
        }
        if(props->type == B200MIX_EFFECT_CHORUS)
        {
            // mLfoOffset follows the LFO range (chorus.cpp:185-211)
            H.lfo_offset = P.cho_rate_on ? H.lfo_offset * P.cho_lfo_range_new / H.lfo_range : 0u;
            H.lfo_range = P.cho_lfo_range;
            CUDA_TRY(*err_, cudaMemcpyAsync(&dev->cho_lfo_offset, &H.lfo_offset, sizeof(uint32_t), cudaMemcpyHostToDevice,
                s_));
        }
        if(props->type == B200MIX_EFFECT_FSHIFTER)
        {   // a direction switched off zeroes that side's phase accumulators (fshifter.cpp:189-192,205-208)
            static const uint32_t zero = 0u;
            for(int c = 0;c < 4;++c)
                if(P.fs_reset_phase[c])
                    CUDA_TRY(*err_, cudaMemcpyAsync(&dev->fs_phase[c], &zero, sizeof(uint32_t), cudaMemcpyHostToDevice, s_));
        }
        if(props->type == B200MIX_EFFECT_VMORPHER)
            // update() installs newly constructed formant filters: their histories restart at 0
            // (vmorpher.cpp:252-260)
            CUDA_TRY(*err_, cudaMemsetAsync(dev->vm_s, 0, sizeof(EfxDev::vm_s), s_));
        SlotRec rec = S.rec;
        rec.fade_len = P.fade_len;
        if(int rc = upload_records(sl, &rec)) return rc;
        if(int rc = efx_gains(S.rec, P)) return rc;
        CUDA_TRY(*err_, cudaStreamSynchronize(s_));
        H.p = P;
        S.efx = H; S.rec.fade_len = P.fade_len;
        return B200MIX_OK;
    }

    int target(uint32_t sl, uint32_t target)
    {
        if(sl >= size() || (target != B200MIX_NO_SLOT && target >= size()))
            return refuse(*err_, "slot_target: slot out of range");
        uint32_t hops = 0;
        for(uint32_t t = target;t != B200MIX_NO_SLOT;t = slots_[t].rec.target)
            if(t == sl || ++hops > size())
                return refuse(*err_, "slot_target: the chain would loop");
        SlotRec rec = slots_[sl].rec;
        rec.target = target;
        return exchange(slots_[sl].rec, rec);
    }

    int output_gains(uint32_t sl, uint32_t lines, const float *gains)
    {
        if(sl >= size() || !slots_[sl].rec.type || !gains) return refuse(*err_, "slot_output_gains: bad arguments");
        const Slot &S = slots_[sl];
        const bool reverb = S.rec.type == B200MIX_EFFECT_REVERB;
        if(lines != (reverb ? 8u : S.rec.channels)) return refuse(*err_, "slot_output_gains: wrong line count");
        // gains address the slot's output target: the Dry mix or the target slot's Wet mix
        const uint32_t width = S.rec.target != B200MIX_NO_SLOT ? dd_.wet_channels : dd_.dry_channels;
        std::vector<float> g(size_t(lines)*32, 0.0f);
        for(uint32_t c = 0;c < lines;++c)
            for(uint32_t o = 0;o < width;++o)
                g[c*32 + o] = gains[c*width + o];
        // a reverb's gains are those of its CURRENT pipeline object (update3DPanning, reverb.cpp:1293-1296)
        float *dst = S.rec.gtgt + (reverb ? size_t(S.rv.cur)*8*32 : 0);
        CUDA_TRY(*err_, cudaMemcpyAsync(dst, g.data(), g.size()*sizeof(float), cudaMemcpyHostToDevice, s_));
        CUDA_TRY(*err_, cudaStreamSynchronize(s_));
        return B200MIX_OK;
    }

    // One update's slot work once `wet` holds the sends: every slot advances, then, per stage of the slot
    // graph, the effect kernels, the output mix into `dry` and the target mix into `wet`; then the gains commit.
    int run(uint32_t frames, float *wet, float *dry, uint64_t &launches)
    {
        if(!active_) return B200MIX_OK;
        bool upload = false;
        for(uint32_t sl = 0;sl < size();++sl)
            if(int rc = advance(sl, frames, upload)) return rc;
        if(upload)
            if(int rc = upload_records()) return rc;
        const uint32_t ns = dd_.max_slots;
        ConvParams CP{};
        CP.slots = d_slots_; CP.wet = wet; CP.twiddle = twiddle_;
        CP.frames = frames; CP.cw = dd_.wet_channels; CP.num_slots = ns; CP.chunks = conv_chunks_;
        SlotMixParams SP{};
        SP.slots = d_slots_; SP.dry = dry; SP.frames = frames; SP.cd = dd_.dry_channels;
        SP.num_slots = ns; SP.wet = wet; SP.cw = dd_.wet_channels;
        for(uint32_t st = 0;st < stages_;++st)
        {
            if(reverb_)
            {
                ReverbParamsK RP{};
                RP.slots = d_slots_; RP.wet = wet; RP.cubic = cubic_;
                RP.frames = frames; RP.cw = dd_.wet_channels; RP.stage = st;
                RP.seq = ++reverb_seq_;
                CUDA_TRY(*err_, launch_ex(s_, launches, false, k_reverb_process, dim3(ns, 2, 2), dim3(128), 0, RP));
                CUDA_TRY(*err_, launch_ex(s_, launches, false, k_reverb_commit, dim3(ns), dim3(2), 0, RP));
                if(upmix_)
                    CUDA_TRY(*err_, launch_ex(s_, launches, false, k_reverb_upmix, dim3(ns, 2), dim3(256), 8*kLine*sizeof(float), RP));
            }
            CP.stage = st; SP.stage = st;
            if(efx_)
            {
                EfxRunParams EQ{d_slots_, wet, frames, dd_.wet_channels, st, cubic_};
                CUDA_TRY(*err_, launch_efx_process(EQ, ns, s_));
                ++launches;
                if(pshift_)
                {
                    CUDA_TRY(*err_, launch_efx_pshift(EQ, ns, s_));
                    ++launches;
                }
            }
            if(conv_)
            {
                CUDA_TRY(*err_, launch_ex(s_, launches, false, k_conv_input, dim3(ns), dim3(128), 0, CP));
                CUDA_TRY(*err_, launch_ex(s_, launches, false, k_conv_mac, dim3(ns, conv_ch_, CP.chunks), dim3(128),
                    sizeof(ConvMacSmem), CP));
                CUDA_TRY(*err_, launch_ex(s_, launches, false, k_conv_ifft, dim3(ns, conv_ch_, kConvMaxBlocks), dim3(128), 0, CP));
                CUDA_TRY(*err_, launch_ex(s_, launches, false, k_conv_output, dim3(ns, conv_ch_), dim3(128), 0, CP));
            }
            CUDA_TRY(*err_, launch_ex(s_, launches, false, k_slot_output_mix, dim3((frames + 127)/128, dd_.dry_channels),
                dim3(128), 0, SP));
            if(targets_)
                CUDA_TRY(*err_, launch_ex(s_, launches, false, k_slot_target_mix, dim3((frames + 127)/128, ns), dim3(128), 0, SP));
        }
        CUDA_TRY(*err_, launch_ex(s_, launches, false, k_slot_gains_commit, dim3(ns), dim3(64), 0, SP));
        return B200MIX_OK;
    }

private:
    // Processing stages (alc/alu.cpp:2211-2251: every slot before its target): stage = (longest
    // chain length) - (hops from the slot to a slot that outputs to Dry).  Sets the stage of every
    // record, and the flags and grids the update launch reads.  Allocates nothing.
    void refresh()
    {
        const uint32_t ns = size();
        auto hops = [&](uint32_t sl) {
            uint32_t n = 0;
            for(uint32_t t = slots_[sl].rec.target;t != B200MIX_NO_SLOT && n <= ns;t = slots_[t].rec.target) ++n;
            return n;
        };
        uint32_t maxd = 0;
        active_ = targets_ = reverb_ = upmix_ = efx_ = pshift_ = conv_ = false;
        conv_ch_ = conv_chunks_ = 1u;
        for(uint32_t sl = 0;sl < ns;++sl)
            if(slots_[sl].rec.type) { maxd = std::max(maxd, hops(sl)); targets_ |= hops(sl) != 0; }
        stages_ = maxd + 1u;
        uint32_t convWork = 0, convSegs = 0;
        for(uint32_t sl = 0;sl < ns;++sl)
        {
            SlotRec &r = slots_[sl].rec;
            r.stage = r.type ? maxd - std::min(hops(sl), maxd) : 0u;
            active_ |= r.type != B200MIX_EFFECT_NONE;
            reverb_ |= r.type == B200MIX_EFFECT_REVERB;
            upmix_ |= r.type == B200MIX_EFFECT_REVERB && (slots_[sl].rv.h[0].upmix || slots_[sl].rv.h[1].upmix);
            efx_ |= r.type >= B200MIX_EFFECT_ECHO;
            pshift_ |= r.type == B200MIX_EFFECT_PSHIFTER;
            if(r.type == B200MIX_EFFECT_CONVOLUTION)
            { conv_ch_ = std::max(conv_ch_, r.channels); convWork += r.channels; convSegs = std::max(convSegs, r.segs); }
        }
        // segment chunks of k_conv_mac: ~4 CTAs (of 128 threads) per SM over all convolution
        // slot-channels, at least 18 segments per chunk
        conv_ = convWork != 0;
        if(conv_)
            conv_chunks_ = std::max(1u, std::min(std::min(uint32_t(kConvMaxChunks), (convSegs + 17u)/18u),
                (4u*num_sms_ + convWork - 1u)/convWork));
    }

    // Refreshes the table and uploads every record (slot `sl`'s as `rec`, when given), then waits.
    int upload_records(uint32_t sl = 0, const SlotRec *rec = nullptr)
    {
        refresh();
        for(uint32_t i = 0;i < size();++i) recs_[i] = slots_[i].rec;
        if(rec) recs_[sl] = *rec;
        CUDA_TRY(*err_, b200mix::upload(d_slots_, recs_, s_));
        return B200MIX_OK;
    }

    // `next` takes the place of `cur` (a slot, or its record) and the table is uploaded with it; on
    // failure the table is as it was.  On success `next` holds what `cur` held, so the memory of an
    // effect that is replaced is freed only once no record on the device points into it.
    template<typename T>
    int exchange(T &cur, T next)
    {
        std::swap(cur, next);
        if(const int rc = upload_records()) { std::swap(cur, next); refresh(); return rc; }
        installed_ |= active_;
        return B200MIX_OK;
    }

    // Slot `sl` without its effect: the target stays.
    Slot empty(uint32_t sl) const { Slot S; S.rec.target = slots_[sl].rec.target; return S; }

    // `count` zeroed T, held by `S`
    template<typename T>
    int alloc(Slot &S, T *&p, size_t count)
    {
        DevArray<char> a;
        CUDA_TRY(*err_, a.alloc(count*sizeof(T), s_));
        p = reinterpret_cast<T*>(a.get());
        S.mem.push_back(std::move(a));
        return B200MIX_OK;
    }

    // The EFX output gains: Target, and Current too when update() snaps them.
    int efx_gains(const SlotRec &r, const EfxParams &P)
    {
        CUDA_TRY(*err_, cudaMemcpyAsync(r.gtgt, P.gains, size_t(P.lines)*32*sizeof(float), cudaMemcpyHostToDevice, s_));
        if(P.snap_gains)
            CUDA_TRY(*err_, cudaMemcpyAsync(r.gains, P.gains, size_t(P.lines)*32*sizeof(float), cudaMemcpyHostToDevice, s_));
        return B200MIX_OK;
    }

    int check_reverb(const b200mix_reverb_params *p)
    {
        auto pow2 = [](uint32_t v) { return v >= 4u && !(v & (v-1u)); };
        if(!pow2(p->main_len) || !pow2(p->late_in_len) || !pow2(p->early_ap_len) || !pow2(p->early_len)
            || !pow2(p->late_ap_len) || !pow2(p->late_len) || !p->late_offset[0] || !p->late_ap_offset[0])
            return refuse(*err_, "slot_reverb: line lengths must be powers of two, feedback delays non-zero");
        for(int j = 0;j < 4;++j)
            if(!p->early_ap_offset[j] || p->late_ap_offset[j] < p->late_ap_offset[0])
                return refuse(*err_, "slot_reverb: all-pass delays must be non-zero, late all-pass sorted");
        return B200MIX_OK;
    }

    // b200mix_reverb_params -> the parameter part of a ReverbDev (state and pointers untouched)
    static void fill_reverb(ReverbDev &h, const b200mix_reverb_params *p)
    {
        std::memcpy(h.early_tap, p->early_tap, sizeof(h.early_tap)); h.early_tap_coeff = p->early_tap_coeff;
        std::memcpy(h.late_tap, p->late_tap, sizeof(h.late_tap));
        h.mix_x = p->mix_x; h.mix_y = p->mix_y;
        std::memcpy(h.filter_lp, p->filter_lp, sizeof(h.filter_lp));
        std::memcpy(h.filter_hp, p->filter_hp, sizeof(h.filter_hp));
        h.early_ap_coeff = p->early_ap_coeff;
        std::memcpy(h.early_ap_offset, p->early_ap_offset, sizeof(h.early_ap_offset));
        std::memcpy(h.early_offset, p->early_offset, sizeof(h.early_offset));
        h.early_coeff = p->early_coeff;
        std::memcpy(h.late_offset, p->late_offset, sizeof(h.late_offset));
        h.density_gain = p->density_gain;
        std::memcpy(h.t60_mid_gain, p->t60_mid_gain, sizeof(h.t60_mid_gain));
        std::memcpy(h.t60_hf, p->t60_hf, sizeof(h.t60_hf)); std::memcpy(h.t60_lf, p->t60_lf, sizeof(h.t60_lf));
        h.mod_step = p->mod_step; h.mod_depth = p->mod_depth; h.late_ap_coeff = p->late_ap_coeff;
        std::memcpy(h.late_ap_offset, p->late_ap_offset, sizeof(h.late_ap_offset));
        h.upmix = p->upmix ? 1u : 0u; h.order_scale[0] = p->order_scale[0]; h.order_scale[1] = p->order_scale[1];
        h.split_coeff = p->splitter_coeff;
    }

    // One update of `frames` for slot `sl`, before its kernels run: ReverbState::process's pipeline
    // state machine (reverb.cpp:1840-1878), the ring modulator's and chorus' phase indices.  `upload`:
    // the slot's record changed.
    int advance(uint32_t sl, uint32_t frames, bool &upload)
    {
        Slot &S = slots_[sl];
        if(S.rec.type == B200MIX_EFFECT_MODULATOR) S.efx.mod_index = (S.efx.mod_index + frames) % S.efx.mod_range;
        if(S.rec.type == B200MIX_EFFECT_CHORUS) S.efx.lfo_offset = (S.efx.lfo_offset + frames) % S.efx.lfo_range;
        if(S.rec.type != B200MIX_EFFECT_REVERB) return B200MIX_OK;
        Reverb &R = S.rv;
        const int old = R.cur ^ 1;
        uint32_t mask = 1u << R.cur;
        if(R.state == Pipeline::Cleanup)
        {
            // ReverbPipeline::clear (reverb.cpp:550-566) of the old object: its mirror, then on the device
            // its delay lines, its ReverbDev from the mirror and its output gains
            R.clear(old);
            R.state = Pipeline::Normal;
            const ReverbDev &h = R.h[old];
            CUDA_TRY(*err_, cudaMemsetAsync(h.late_in, 0, size_t(4)*h.late_in_len*sizeof(float), s_));
            CUDA_TRY(*err_, cudaMemsetAsync(h.early_ap, 0, size_t(4)*h.early_ap_len*sizeof(float), s_));
            CUDA_TRY(*err_, cudaMemsetAsync(h.early_d, 0, size_t(4)*h.early_len*sizeof(float), s_));
            CUDA_TRY(*err_, cudaMemsetAsync(h.late_ap, 0, size_t(4)*h.late_ap_len*sizeof(float), s_));
            CUDA_TRY(*err_, cudaMemsetAsync(h.late_d, 0, size_t(4)*h.late_len*sizeof(float), s_));
            CUDA_TRY(*err_, cudaMemcpyAsync(reinterpret_cast<ReverbDev*>(S.rec.H) + old, &h, sizeof(ReverbDev),
                cudaMemcpyHostToDevice, s_));
            CUDA_TRY(*err_, cudaMemsetAsync(S.rec.gtgt + size_t(old)*8*32, 0, size_t(8)*32*sizeof(float), s_));
            CUDA_TRY(*err_, cudaMemsetAsync(S.rec.gains + size_t(old)*8*32, 0, size_t(8)*32*sizeof(float), s_));
            // the mirror was read by a pageable-memory copy above: wait before it changes again
            CUDA_TRY(*err_, cudaStreamSynchronize(s_));
        }
        else if(R.state == Pipeline::Fading)
        {
            // the old pipeline's final mix fades its gains to silence
            if(frames >= R.fade[old])
            {
                R.fade[old] = 0; R.state = Pipeline::Cleanup;
                CUDA_TRY(*err_, cudaMemsetAsync(S.rec.gtgt + size_t(old)*8*32, 0, size_t(8)*32*sizeof(float), s_));
            }
            else R.fade[old] -= frames;
            mask |= 1u << old;
        }
        R.offset += frames;
        upload |= S.rec.rv_mask != mask || S.rec.rv_cur != uint32_t(R.cur);
        S.rec.rv_mask = mask; S.rec.rv_cur = uint32_t(R.cur);
        return B200MIX_OK;
    }

    b200mix_device_desc dd_{};
    uint32_t num_sms_{1};
    cudaStream_t s_{nullptr};
    std::string *err_{nullptr};
    std::vector<Slot> slots_;
    std::vector<SlotRec> recs_;                 // the records as uploaded
    DevArray<SlotRec> d_slots_;
    DevArray<float2> twiddle_;                  // k_conv_* FFT twiddles
    DevArray<float> cubic_;                     // gCubicTable (reverb modulation taps)
    bool efx_ready_{false};                     // efx_kernels_init has run (first efx())
    bool installed_{false};                     // ever_installed()
    uint32_t reverb_seq_{0};                    // update counter of k_reverb_process' early/late hand-off (24 bits used)
    // derived by refresh()
    uint32_t stages_{1};
    bool active_{false}, targets_{false}, reverb_{false}, upmix_{false}, efx_{false}, pshift_{false};
    bool conv_{false}; uint32_t conv_ch_{1}, conv_chunks_{1};  // k_conv_* grids: channels, segment chunks
};

} // namespace b200mix
