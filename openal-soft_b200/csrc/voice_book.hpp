// voice_book.hpp — the host's mirror of every voice, and the lists the mixing kernels walk.
//
// The lists fix the order of every cross-voice sum, so each has one rule:
//   order         the active voices, stable-sorted by cost key, descending (the mixing order)
//   order2        the voices of `order` with an active direct filter (all of them once the GPU
//                 parameter stage decides filter activity: k_filters and k_mix_deferred then look
//                 at every voice's kSiDeferred bit)
//   dry_entries   the active voices that mix into Dry (neither HRTF nor direct) in index order
//                 (the parked dry bus)
//   real_entries  the active direct-channel voices in index order (the RealOut bus)
//   slot_start / entries   per slot, its (voice, send) pairs: voices, then sends, in index order
// The setters mark the lists a change affects; refresh() rebuilds those and says which, for the
// caller to upload.  Host code only.
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../include/b200mix.h"
#include "voice_structs.hpp"

namespace b200mix {

struct VoiceBook {
    // One voice as an update leaves it: active (not B200MIX_VF_STOPPED), its mixing-order cost key
    // (resampler taps per output), HRTF (mixes through its own HRIR, not the dry bus), its aux slot
    // per send, the static buffer it plays (or B200MIX_NO_SLOT), RESET (clears the direct filter),
    // DIRECT (mixes into RealOut, not the dry bus).
    struct State { bool active; uint32_t cost; bool hrtf; const uint32_t *send_slot; uint32_t buffer; bool reset;
        bool direct; };
    struct Rebuilt { bool order, order2, dry, sends, real; };

    uint32_t num_sends{0}, max_slots{0};
    std::vector<uint8_t> active, hrtf, dfilt, direct;   // dfilt: direct filter active
    std::vector<uint32_t> cost, vbuf;              // vbuf: static buffer an active voice plays
    std::vector<uint32_t> send_slot;               // [voice][num_sends]
    std::vector<uint32_t> bufrefs;                 // active static voices per buffer
    uint32_t voice_hi{0};                          // 1 + highest voice index ever set
    bool dry_active{false};                        // a voice has fed the dry bus
    bool dev_filters{false};                       // filter activity is decided on the device

    std::vector<uint32_t> order, order2, slot_start;
    std::vector<SendEntry> dry_entries, entries, real_entries;
    uint32_t max_slot_entries{0};
    bool order_dirty{true}, order2_dirty{false}, dry_dirty{true}, sends_dirty{true}, real_dirty{false};

    void init(uint32_t max_voices, uint32_t max_buffers, uint32_t sends, uint32_t slots)
    {
        num_sends = sends; max_slots = slots;
        active.assign(max_voices, 0); hrtf.assign(max_voices, 0); dfilt.assign(max_voices, 0);
        direct.assign(max_voices, 0);
        cost.assign(max_voices, 0); vbuf.assign(max_voices, B200MIX_NO_SLOT);
        send_slot.assign(size_t(max_voices)*num_sends, B200MIX_NO_SLOT);
        bufrefs.assign(std::max(max_buffers, 1u), 0u);
    }

    void set(uint32_t v, const State &s)
    {
        for(uint32_t k = 0;k < num_sends;++k)
        {
            uint32_t &m = send_slot[size_t(v)*num_sends + k];
            const uint32_t slot = s.active ? s.send_slot[k] : B200MIX_NO_SLOT;
            if(m != slot) { m = slot; sends_dirty = true; }
        }
        if(s.active && !s.hrtf && !s.direct) dry_active = true;
        if(hrtf[v] != s.hrtf) { hrtf[v] = s.hrtf; dry_dirty = true; }
        if(direct[v] != s.direct) { direct[v] = s.direct; dry_dirty = real_dirty = true; }
        if(active[v] != s.active || cost[v] != s.cost) order_dirty = true;
        if(direct[v] && active[v] != s.active) real_dirty = true;
        active[v] = s.active; cost[v] = s.cost;
        voice_hi = std::max(voice_hi, v + 1u);
        const uint32_t nb = s.active ? s.buffer : B200MIX_NO_SLOT;
        if(vbuf[v] != nb)
        {
            if(vbuf[v] != B200MIX_NO_SLOT) --bufrefs[vbuf[v]];
            if(nb != B200MIX_NO_SLOT) ++bufrefs[nb];
            vbuf[v] = nb;
        }
        if(s.reset) set_direct_filter(v, false);
    }
    bool has_direct() const
    {
        for(uint32_t v = 0;v < voice_hi;++v) if(active[v] && direct[v]) return true;
        return false;
    }
    void set_direct_filter(uint32_t v, bool on) { if(dfilt[v] != on) { dfilt[v] = on; order2_dirty = true; } }
    void set_device_filters() { order2_dirty |= !dev_filters; dev_filters = true; }

    // order2 is kept once the device has filters, the dry entries once it parks its dry bus, the
    // send CSR while it mixes sends; the RealOut entries whenever a direct voice changes.
    Rebuilt refresh(bool filters, bool dry, bool sends)
    {
        Rebuilt r{order_dirty, false, false, false, real_dirty};
        if(r.order)
        {
            order.clear();
            for(uint32_t v = 0;v < voice_hi;++v) if(active[v]) order.push_back(v);
            std::stable_sort(order.begin(), order.end(), [this](uint32_t a, uint32_t b) { return cost[a] > cost[b]; });
            order_dirty = false; order2_dirty = dry_dirty = true;
        }
        r.order2 = filters && order2_dirty; r.dry = dry && dry_dirty; r.sends = sends && sends_dirty;
        if(r.order2)
        {
            order2.clear();
            for(uint32_t v : order) if(dev_filters || dfilt[v]) order2.push_back(v);
            order2_dirty = false;
        }
        if(r.dry)
        {
            dry_entries.clear();
            for(uint32_t v = 0;v < voice_hi;++v)
                if(active[v] && !hrtf[v] && !direct[v]) dry_entries.push_back(SendEntry{v, 0u});
            dry_dirty = false;
        }
        if(r.real)
        {
            real_entries.clear();
            for(uint32_t v = 0;v < voice_hi;++v) if(active[v] && direct[v]) real_entries.push_back(SendEntry{v, 0u});
            real_dirty = false;
        }
        if(r.sends)
        {
            slot_start.assign(max_slots + 1, 0);
            entries.clear();
            max_slot_entries = 0;
            for(uint32_t sl = 0;sl < max_slots;++sl)
            {
                slot_start[sl] = uint32_t(entries.size());
                for(uint32_t v = 0;v < voice_hi;++v)
                    for(uint32_t k = 0;k < num_sends;++k)
                        if(send_slot[size_t(v)*num_sends + k] == sl) entries.push_back(SendEntry{v, k});
                max_slot_entries = std::max(max_slot_entries, uint32_t(entries.size()) - slot_start[sl]);
            }
            slot_start[max_slots] = uint32_t(entries.size());
            sends_dirty = false;
        }
        return r;
    }
};

} // namespace b200mix
