// slot_table.hpp — the host's state of every effect slot: the record the device's copy is uploaded
// from, and the host halves of the reverb's pipeline state machine and of the EFX effects.  refresh()
// derives the stages and every flag and grid the update launch reads; advance() runs one update's host
// state and says what the caller has to do on the stream.  Host code only.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../include/b200mix.h"
#include "effect_kernels.cuh"
#include "efx_math.hpp"

namespace b200mix {

struct SlotTable {
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
    };
    // What advance() asks of the caller for one slot: clear reverb pipeline object `clear`
    // (delay lines, device mirror, gains), silence object `silence`'s target gains, upload the records.
    struct Due { int clear{-1}, silence{-1}; bool upload{false}; };

    // derived by refresh()
    uint32_t stages{1};
    bool active{false}, targets{false}, reverb{false}, upmix{false}, efx{false}, pshift{false};
    bool conv{false}; uint32_t conv_ch{1}, conv_chunks{1};     // k_conv_* grids: channels, segment chunks

    void init(uint32_t slots, uint32_t sms) { s_.assign(slots, Slot{}); num_sms_ = sms; refresh(); }
    uint32_t size() const { return uint32_t(s_.size()); }
    Slot &operator[](uint32_t sl) { return s_[sl]; }

    // The slot loses its effect; its target stays.
    void release(uint32_t sl) { const uint32_t t = s_[sl].rec.target; s_[sl] = Slot{}; s_[sl].rec.target = t; }

    // Processing stages (alc/alu.cpp:2211-2251: every slot before its target): stage = (longest
    // chain length) - (hops from the slot to a slot that outputs to Dry).  Sets the stage of every
    // record, and the flags and grids the update launch reads.
    void refresh()
    {
        const uint32_t ns = size();
        std::vector<uint32_t> depth(ns, 0);
        uint32_t maxd = 0;
        active = targets = reverb = upmix = efx = pshift = conv = false;
        conv_ch = conv_chunks = 1u;
        for(uint32_t sl = 0;sl < ns;++sl)
        {
            uint32_t hops = 0;
            for(uint32_t t = s_[sl].rec.target;t != B200MIX_NO_SLOT && hops <= ns;t = s_[t].rec.target) ++hops;
            depth[sl] = hops;
            if(s_[sl].rec.type) { maxd = std::max(maxd, hops); if(hops) targets = true; }
        }
        stages = maxd + 1u;
        uint32_t convWork = 0, convSegs = 0;
        for(uint32_t sl = 0;sl < ns;++sl)
        {
            SlotRec &r = s_[sl].rec;
            r.stage = r.type ? maxd - std::min(depth[sl], maxd) : 0u;
            active |= r.type != B200MIX_EFFECT_NONE;
            reverb |= r.type == B200MIX_EFFECT_REVERB;
            upmix |= r.type == B200MIX_EFFECT_REVERB && (s_[sl].rv.h[0].upmix || s_[sl].rv.h[1].upmix);
            efx |= r.type >= B200MIX_EFFECT_ECHO;
            pshift |= r.type == B200MIX_EFFECT_PSHIFTER;
            if(r.type == B200MIX_EFFECT_CONVOLUTION)
            { conv_ch = std::max(conv_ch, r.channels); convWork += r.channels; convSegs = std::max(convSegs, r.segs); }
        }
        // segment chunks of k_conv_mac: ~4 CTAs (of 128 threads) per SM over all convolution
        // slot-channels, at least 18 segments per chunk
        conv = convWork != 0;
        if(conv)
            conv_chunks = std::max(1u, std::min(std::min(uint32_t(kConvMaxChunks), (convSegs + 17u)/18u),
                (4u*num_sms_ + convWork - 1u)/convWork));
    }

    // One update of `frames` for slot `sl`, before its kernels run: ReverbState::process's pipeline
    // state machine (reverb.cpp:1840-1878), the ring modulator's and chorus' phase indices.
    Due advance(uint32_t sl, uint32_t frames)
    {
        Slot &S = s_[sl];
        Due due;
        if(S.rec.type == B200MIX_EFFECT_MODULATOR) S.efx.mod_index = (S.efx.mod_index + frames) % S.efx.mod_range;
        if(S.rec.type == B200MIX_EFFECT_CHORUS) S.efx.lfo_offset = (S.efx.lfo_offset + frames) % S.efx.lfo_range;
        if(S.rec.type != B200MIX_EFFECT_REVERB) return due;
        Reverb &R = S.rv;
        const int old = R.cur ^ 1;
        uint32_t mask = 1u << R.cur;
        if(R.state == Pipeline::Cleanup)
        {
            R.clear(old);
            due.clear = old; R.state = Pipeline::Normal;
        }
        else if(R.state == Pipeline::Fading)
        {
            // the old pipeline's final mix fades its gains to silence
            if(frames >= R.fade[old]) { due.silence = old; R.fade[old] = 0; R.state = Pipeline::Cleanup; }
            else R.fade[old] -= frames;
            mask |= 1u << old;
        }
        R.offset += frames;
        due.upload = S.rec.rv_mask != mask || S.rec.rv_cur != uint32_t(R.cur);
        S.rec.rv_mask = mask; S.rec.rv_cur = uint32_t(R.cur);
        return due;
    }

private:
    std::vector<Slot> s_;
    uint32_t num_sms_{1};
};

} // namespace b200mix
