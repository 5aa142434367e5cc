// voice_structs.hpp — plain records shared by the mixer kernels (mixer_kernels.cuh), the
// parameter kernel (param_kernels.cu) and the EFX kernels (efx_kernels.cu): what
// b200mix_voices_update / b200mix_sources_update stage for k_apply_updates and
// k_apply_filter_updates, the bus mixes' (voice, send) entries, and the effect slot records.
#pragma once
#include <cstdint>

namespace b200mix {

// A convolution slot's input ring (ConvolutionState::mInput / mCurrentSegment).  Device only:
// k_conv_input alone writes it, every update; the other k_conv_* kernels read the last update's part.
struct ConvRing {
    uint32_t cur, fifo;                        // spectra-ring position, FIFO fill
    uint32_t nb_last, f_last, cur_last;        // last update: blocks completed, fill and position at its start
};

// One effect slot as the kernels see it.  The host writes every field (SlotTable); what a kernel
// carries from one update to the next lives behind the pointers (ring, H, lines, gains), so the
// host may upload any record at any time without overwriting device state.
struct SlotRec {
    uint32_t type, channels, frames, segs;     // type: b200mix_effect; segs = mNumConvolveSegs
    uint32_t rv_cur, rv_mask;                  // reverb: current pipeline object; objects to run now
    uint32_t stage;                            // processing stage: every slot runs before its target
    uint32_t target{0xffffffffu};              // slot whose Wet takes the output, or 0xffffffff (Dry)
    uint32_t fade_len;                         // MixSamples Counter of the output mix: 0 = samplesToDo, else min(n, fade_len)
    ConvRing *ring;   // convolution: the input ring
    float *H;         // convolution: [channels][segs][256] filter spectra (pre-scaled by 1/256);
                      // reverb: its ReverbDev[2]; EFX: its EfxDev
    float *X;         // [segs+kConvMaxBlocks][256] input spectra ring (our own ring: long enough that
                      //                        a whole update's blocks never overwrite live history)
    float *head;      // [channels][128]        first 128 IR taps
    float *inbuf;     // [256]                  mInput
    float *ov;        // [channels][256]        mOutput
    float *yspec;     // [channels][kConvMaxChunks][kConvMaxBlocks][256] partial sums per segment chunk
    float *lines;     // [channels][1024]       this update's output lines
    float *gains;     // [channels][32]         Current gains
    float *gtgt;      // [channels][32]         Target gains
};

constexpr int kMaxSends = 6;

// VoiceUpdate / VoiceRec flag of a direct-channel voice (direct path RealOut); set by
// b200mix_voices_update_direct only, never taken from the caller's flags.
constexpr uint32_t kVfDirect = 1u<<12;

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
