// efx_kernels.hpp — interface between the library's host side (b200mix.cu) and the EFX effect
// kernels (efx_kernels.cu, compiled separately with -fmad=false).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "efx_math.hpp"
#include "voice_structs.hpp"

namespace b200mix {

// Device-resident effect state: the parameters update() produced + what process() carries over.
struct EfxDev {
    EfxParams p;
    float *echo_buf;                       // EchoState::mSampleBuffer [echo_len]
    uint32_t echo_offset; float echo_z[2]; // mOffset, mFilter z1/z2
    uint32_t mod_index;                    // ModulatorState::mIndex
    float comp_env;                        // CompressorState::mEnvFollower
    float *cho_buf;                        // ChorusState::mDelayBuffers [4][cho_len]
    uint32_t cho_offset, cho_lfo_offset;   // mOffset, mLfoOffset
    float wah_env;                         // AutowahState::mEnvDelay
    uint32_t vm_index; float vm_cur[kEfxMaxLines];   // VmorpherState::mIndex, OutParams::mCurrentGain
    float vm_s[kEfxMaxLines][2][4][2];     // FormantFilter::mS1/mS2 [channel][vowel][formant]
    // frequency shifter (double precision like the reference): mInFIFO [4][1024], mOutFIFO [4][256] complex,
    // mOutputAccum [4][1024] complex; mCount, mPos, mPhase[4]
    double *fs_in; double2 *fs_outfifo; double2 *fs_accum;
    uint32_t fs_count, fs_pos, fs_phase[4];
    float chan_z[kEfxMaxLines][4][2];      // per-channel biquad histories (modulator [0], equalizer [0..3],
                                           // distortion [0] low-pass, [1] band-pass)
    // pitch shifter: ProcessParams::mFIFO / mOutputAccum [9][1024], mLastPhase / mSumPhase [513]; mCount, mPos
    float *ps_fifo, *ps_accum, *ps_last, *ps_sum;
    uint32_t ps_count, ps_pos;
};

// k_efx_process / k_efx_pshift run the slots of type >= B200MIX_EFFECT_ECHO: their EfxDev is SlotRec::H
struct EfxRunParams { const SlotRec *slots; const float *wet; uint32_t frames, cw, stage; const float *cubic; /* gCubicTable [513] */ };

cudaError_t efx_kernels_init();            // per CUDA device: dynamic shared memory opt-in
cudaError_t launch_efx_process(const EfxRunParams &Q, uint32_t num_slots, cudaStream_t stream);
cudaError_t launch_efx_pshift(const EfxRunParams &Q, uint32_t num_slots, cudaStream_t stream);   // the pitch shifter's own kernel

} // namespace b200mix
