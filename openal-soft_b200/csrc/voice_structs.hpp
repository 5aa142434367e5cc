// voice_structs.hpp — plain records shared by the mixer kernels (mixer_kernels.cuh) and the
// parameter kernel (param_kernels.cu): what b200mix_voices_update / b200mix_sources_update stage
// for k_apply_updates and k_apply_filter_updates, and the bus mixes' (voice, send) entries.
#pragma once
#include <cstdint>

namespace b200mix {

constexpr int kMaxSends = 6;

struct alignas(16) VoiceUpdate {   // staged by b200mix_voices_update
    uint32_t voice, flags, buffer, resampler;
    int32_t  position; uint32_t position_frac, loop_start, loop_end;
    uint32_t step; float bsinc_sf; uint32_t bsinc_m, bsinc_l;
    uint32_t bsinc_off, delay0, delay1; float gain;
    uint32_t send_slot[kMaxSends]; uint32_t has_coeffs, has_dry;
};

struct FilterUpdate {      // == b200mix_voice_filter
    uint32_t voice, path, active; float lp[5], hp[5];
};

struct SendEntry { uint32_t voice, send; };   // a voice's send (0 on the dry bus)

} // namespace b200mix
