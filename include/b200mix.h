/* b200mix.h — C ABI of the Hopper (sm_90a) mixer backend for OpenAL Soft.
 *
 * This is the drop-in boundary: one level above the reference's per-kernel
 * function pointers, it replaces the body of DeviceBase::renderSamples(unsigned)
 * between "parameters updated" and "RealOut ready" —
 *   the voice loop      alc/alu.cpp:2201-2206  (Voice::mix, core/voice.cpp:988-1233)
 *   the slot loop       alc/alu.cpp:2252-2256  (EffectState::process)
 *   the post-process    alc/alu.cpp:2439-2443  (DeviceBase::Process, alc/alu.cpp:284-312)
 * The host keeps ProcessParamUpdates (alc/alu.cpp:2153), clocks, events and
 * Write<T>.  Everything here is plain C: pointers and sizes, no C++/torch types.
 * All float data is IEEE fp32.  All functions return B200MIX_OK (0) or a
 * negative error; b200mix_last_error() gives the text.  A failing render is
 * what the host turns into DeviceBase::handleDisconnect (alc/alu.cpp:2521).
 *
 * Threading follows the reference: create/destroy/buffer_* from API threads
 * (serialised by the host's BufferLock), everything else from the single mixer
 * thread of the device.  No entry point is re-entrant per device.
 */
#ifndef B200MIX_H
#define B200MIX_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define B200MIX_API __declspec(dllexport)
#else
#define B200MIX_API __attribute__((visibility("default")))
#endif

/* ---- constants mirrored from the reference ------------------------------ */
#define B200MIX_LINE_SIZE        1024u /* BufferLineSize          core/bufferline.h:11 */
#define B200MIX_HRIR_LENGTH       128u /* HrirLength              core/mixer/hrtfdefs.h:19 */
#define B200MIX_HRTF_HISTORY       64u /* HrtfHistoryLength       core/mixer/hrtfdefs.h:15 */
#define B200MIX_MAX_SENDS           6u /* MaxSendCount            core/voice.h:31 */
#define B200MIX_MAX_DRY_CHANNELS   32u /* MaxOutputChannels       core/devformat.h:81 */
#define B200MIX_MAX_WET_CHANNELS   25u /* MaxAmbiChannels         core/ambidefs.h:19 */
#define B200MIX_RESAMPLER_PADDING  48u /* MaxResamplerPadding     core/resampler_limits.h:8 */
#define B200MIX_NO_SLOT   0xffffffffu
#define B200MIX_NO_LOOP   0xffffffffu
#define B200MIX_NO_BUFFER 0xffffffffu
#define B200MIX_MAX_QUEUE          32u /* items of a streaming queue the mixer looks ahead over */

enum { B200MIX_OK = 0, B200MIX_ERR_INVALID = -1, B200MIX_ERR_CUDA = -2,
       B200MIX_ERR_NOMEM = -3, B200MIX_ERR_UNSUPPORTED = -4 };

/* enum class Resampler, core/mixer/defs.h:31-44 (same order and values). */
enum b200mix_resampler {
    B200MIX_RESAMPLER_POINT = 0, B200MIX_RESAMPLER_LINEAR, B200MIX_RESAMPLER_SPLINE,
    B200MIX_RESAMPLER_GAUSSIAN, B200MIX_RESAMPLER_FAST_BSINC12, B200MIX_RESAMPLER_BSINC12,
    B200MIX_RESAMPLER_FAST_BSINC24, B200MIX_RESAMPLER_BSINC24, B200MIX_RESAMPLER_FAST_BSINC48,
    B200MIX_RESAMPLER_BSINC48
};

/* enum FmtType, core/storage_formats.h. */
enum b200mix_sample_type {
    B200MIX_FMT_U8 = 0, B200MIX_FMT_I16, B200MIX_FMT_I32, B200MIX_FMT_F32, B200MIX_FMT_F64,
    B200MIX_FMT_MULAW, B200MIX_FMT_ALAW,
    B200MIX_FMT_IMA4, B200MIX_FMT_MSADPCM     /* only through b200mix_buffer_data_adpcm */
};

/* PostProcess variant of DeviceBase (core/device.h:200-222). */
enum b200mix_post_process {
    B200MIX_POST_NONE = 0,   /* RealOut aliases Dry (e.g. ALC_BFORMAT3D_SOFT output) */
    B200MIX_POST_AMBIDEC,    /* BFormatDec::process        core/bformatdec.cpp:60-97 */
    B200MIX_POST_HRTF,       /* MixDirectHrtf              core/mixer/hrtfbase.h:91-133 */
    B200MIX_POST_UHJ,        /* UhjEncoderIIR::encode      core/uhjfilter.cpp:231-283 */
    B200MIX_POST_TSME        /* TsmeEncoderIIR::encode     core/tsmefilter.cpp:280-329 (4 dry channels W,Y,Z,X) */
};

typedef struct b200mix_device b200mix_device;

/* What aluInitRenderer / UpdateDeviceParams decided (alc/panning.cpp:1220-1438). */
typedef struct b200mix_device_desc {
    uint32_t struct_size;     /* sizeof(b200mix_device_desc) */
    int32_t  cuda_device;     /* ordinal; -1 = current */
    uint32_t sample_rate;     /* DeviceBase::mSampleRate */
    uint32_t dry_channels;    /* Dry.Buffer.size()  (C_d) */
    uint32_t real_channels;   /* RealOut.Buffer.size() */
    uint32_t wet_channels;    /* per-slot Wet.Buffer.size() (C_w); 0 = no sends */
    uint32_t num_sends;       /* DeviceBase::NumAuxSends */
    uint32_t ir_size;         /* DeviceBase::mIrSize (0 when no HRTF) */
    uint32_t post_process;    /* enum b200mix_post_process */
    uint32_t real_left;       /* RealOut.ChannelIndex[FrontLeft]  (HRTF/UHJ output) */
    uint32_t real_right;      /* RealOut.ChannelIndex[FrontRight] */
    uint32_t max_voices;      /* capacity of the voice array */
    uint32_t max_buffers;     /* capacity of the buffer table */
    uint32_t max_slots;       /* capacity of the aux-slot table */
} b200mix_device_desc;

B200MIX_API int b200mix_create(const b200mix_device_desc *desc, b200mix_device **out);
B200MIX_API void b200mix_destroy(b200mix_device *dev);
/* Text of the last error on this device (or the last create failure if dev==NULL). */
B200MIX_API const char *b200mix_last_error(const b200mix_device *dev);
/* Library/ABI version: (major<<16)|minor. */
B200MIX_API uint32_t b200mix_version(void);

/* ---- post-process constant data ----------------------------------------- */
/* DirectHrtfState (core/hrtf.h:84-110): per dry channel the pre-summed
 * virtual-speaker HRIR, the HF scale and the band-splitter coefficient.
 * ir_size is DirectHrtfState::mIrSize (may exceed the per-voice ir_size, <=128);
 * coeffs is [channels][ir_size][2].  Refused between b200mix_render_begin and _render_end. */
B200MIX_API int b200mix_set_hrtf_decoder(b200mix_device *dev, uint32_t channels,
    uint32_t ir_size, const float *coeffs, const float *hf_scale, const float *splitter_coeff);
/* BFormatDec (core/bformatdec.h): gains_hf/gains_lf are [in_channels][real_channels];
 * gains_lf==NULL selects the single-band decoder; xover_coeff is the splitter's mCoeff.
 * Refused between b200mix_render_begin and _render_end. */
B200MIX_API int b200mix_set_ambi_decoder(b200mix_device *dev, uint32_t in_channels,
    const float *gains_hf, const float *gains_lf, float xover_coeff);

/* ---- buffers: BufferStorage (core/buffer_storage.h:52-75) ---------------- */
/* Uploads an immutable copy (AL semantics: a buffer cannot change while attached). */
B200MIX_API int b200mix_buffer_data(b200mix_device *dev, uint32_t buffer, uint32_t sample_type,
    uint32_t channels, uint32_t frames, const void *data, size_t bytes);
/* Block-compressed buffers (AL_EXT_IMA4, AL_SOFT_MSADPCM): `blocks` blocks of
 * samples_per_block sample frames each (BufferStorage::mBlockAlign; AL's defaults are 65 for
 * IMA4 and 64 for MSADPCM), laid out exactly as alBufferData receives them.  The reference
 * decodes these inside the mixer (LoadSamples<IMA4Data>/<MSADPCMData>, core/voice.cpp:289-484);
 * both are integer recurrences, so the library decodes once here to the identical int16
 * samples and the mixer streams those.  The buffer then has blocks*samples_per_block frames. */
B200MIX_API int b200mix_buffer_data_adpcm(b200mix_device *dev, uint32_t buffer, uint32_t sample_type,
    uint32_t channels, uint32_t samples_per_block, uint32_t blocks, const void *data, size_t bytes);
B200MIX_API int b200mix_buffer_free(b200mix_device *dev, uint32_t buffer);

/* ---- auxiliary effect slots: EffectSlotBase + EffectState (core/effectslot.h:50-82,
 *      core/effects/base.h:197-222) ------------------------------------------------ */
enum b200mix_effect { B200MIX_EFFECT_NONE = 0, B200MIX_EFFECT_CONVOLUTION = 1, B200MIX_EFFECT_REVERB = 2,
    /* the EFX effects behind b200mix_slot_efx */
    B200MIX_EFFECT_ECHO = 3,          /* EchoState        alc/effects/echo.cpp */
    B200MIX_EFFECT_MODULATOR = 4,     /* ModulatorState   alc/effects/modulator.cpp (ring modulator) */
    B200MIX_EFFECT_EQUALIZER = 5,     /* EqualizerState   alc/effects/equalizer.cpp */
    B200MIX_EFFECT_COMPRESSOR = 6,    /* CompressorState  alc/effects/compressor.cpp */
    B200MIX_EFFECT_DEDICATED = 7,     /* DedicatedState   alc/effects/dedicated.cpp (dialogue / LFE) */
    B200MIX_EFFECT_DISTORTION = 8,    /* DistortionState  alc/effects/distortion.cpp */
    B200MIX_EFFECT_CHORUS = 9,        /* ChorusState      alc/effects/chorus.cpp (AL_EFFECT_CHORUS and AL_EFFECT_FLANGER) */
    B200MIX_EFFECT_AUTOWAH = 10,      /* AutowahState     alc/effects/autowah.cpp */
    B200MIX_EFFECT_VMORPHER = 11,     /* VmorpherState    alc/effects/vmorpher.cpp (vocal morpher) */
    B200MIX_EFFECT_FSHIFTER = 12,     /* FshifterState    alc/effects/fshifter.cpp (frequency shifter) */
    B200MIX_EFFECT_PSHIFTER = 13      /* PshifterState    alc/effects/pshifter.cpp (pitch shifter) */
};

/* ConvolutionState::deviceUpdate (alc/effects/convolution.cpp:318-471): installs the
 * device-rate impulse response (planar [ir_channels][ir_frames] floats; the host applies
 * the reference's polyphase resampling first when the IR buffer's rate differs) on aux
 * slot `slot` and resets its history.  The slot reads wet channel 0 of its input
 * (alc/effects/convolution.cpp:636) and mixes ir_channels output lines into the Dry mix. */
B200MIX_API int b200mix_slot_convolution(b200mix_device *dev, uint32_t slot, uint32_t ir_channels,
    uint32_t ir_frames, const float *ir);
/* Result of EffectState::update for the slot's output mix: Target gains
 * [lines][dry_channels] (ConvolutionState::ChannelData::Target); Current is kept on the
 * device and fades to Target over the whole update like MixSamples(..., Counter=samplesToDo). */
B200MIX_API int b200mix_slot_output_gains(b200mix_device *dev, uint32_t slot, uint32_t lines,
    const float *gains);
/* EAX / standard reverb (alc/effects/reverb.cpp).  The host's ReverbState::update
 * (reverb.cpp:1222-1351, with updateDelayLine/updateLines/updateModulator/CalcMatrixCoeffs)
 * stays the parameter stage; this struct is its RESULT for the current pipeline, i.e. the
 * state ReverbState::process consumes.  Biquads are {b0, b1, b2, a1, a2} (a0 pre-applied).
 * Tap/offset values are in samples.  Line lengths come from ReverbState::allocLines. */
typedef struct b200mix_reverb_params {
    uint32_t struct_size;
    uint32_t main_len, late_in_len, early_ap_len, early_len, late_ap_len, late_len; /* per line, pow2 */
    uint32_t early_tap[4];        /* mEarlyDelayTap[j][1] */
    float    early_tap_coeff;     /* mEarlyDelayCoeff[1] */
    uint32_t late_tap[4];         /* mLateDelayTap[j][1] */
    float    mix_x, mix_y;        /* mMixX, mMixY */
    float    filter_lp[5], filter_hp[5];   /* mFilter[*].Lp / .Hp */
    float    early_ap_coeff;      /* mEarly.Allpass.Coeff */
    uint32_t early_ap_offset[4];  /* mEarly.Allpass.Offset */
    uint32_t early_offset[4];     /* mEarly.Offset */
    float    early_coeff;         /* mEarly.Coeff */
    uint32_t late_offset[4];      /* mLate.Offset */
    float    density_gain;        /* mLate.DensityGain */
    float    t60_mid_gain[4];     /* mLate.T60[j].mMidGain */
    float    t60_hf[4][5], t60_lf[4][5];   /* mLate.T60[j].mHFFilter / mLFFilter */
    uint32_t mod_step;            /* mLate.Mod.Step */
    float    mod_depth;           /* mLate.Mod.Depth */
    float    late_ap_coeff;       /* mLate.VecAp.Coeff */
    uint32_t late_ap_offset[4];   /* mLate.VecAp.Offset */
    uint32_t fade_samples;        /* mFadeSampleCount of this pipeline: how long it keeps ringing
                                     out once a later full update has replaced it */
    /* MixOutAmbiUp (reverb.cpp:658-699), used when the device mixes above first order
     * (ReverbState::mUpmixOutput, :834-850): the A-format lines are first turned into four
     * B-format rows (EarlyA2B/LateA2B), each row's HF band is scaled for the device order by a
     * BandSplitter, and the 8 output gain rows then pan those B-format rows. */
    uint32_t upmix;               /* mUpmixOutput */
    float    order_scale[2];      /* mOrderScales[0], [1] */
    float    splitter_coeff;      /* mAmbiSplitter[*][*].mCoeff */
} b200mix_reverb_params;

/* Host helpers, no GPU: the source half of the parameter stage for point sources.
 * b200mix_calc_source_params restates CalcAttnVoiceParams (alc/alu.cpp:1712-2010): listener
 * transform, distance model, cones, gain limits, air absorption and the send decay adjustment,
 * doppler, the resampler step and the source spread.  b200mix_listener_params is ContextParams
 * (core/context.h:67-84; matrix row-major as al::Matrix), b200mix_source_props the VoiceProps
 * fields that function reads (core/voice.h:101-157) with the slot values it takes from
 * EffectSlotBase (core/effectslot.h:70-75) folded into each send.  The result feeds
 * CalcPanningAndFilters' steps (alc/alu.cpp:1519-1656), each of which has its helper:
 *   HRTF device: hrtf_elevation/hrtf_azimuth/distance/spread -> b200mix_hrtf_get_coeffs or
 *     b200mix_voices_update_dirs, hrtf_gain = dry_gain;
 *   other devices: b200mix_ambi_coeffs(pos or b200mix_pairwise_azimuth(pos), spread) ->
 *     b200mix_pan_gains(Dry map, dry_gain);
 *   sends: b200mix_ambi_coeffs(pos, spread) -> b200mix_pan_gains(slot Wet map, wet_gain[i]);
 *   filters: b200mix_biquad_coeffs(HighShelf, hf_reference/rate, gain_hf, 1) and
 *     (LowShelf, lf_reference/rate, gain_lf, 1), active iff gain_hf != 1 || gain_lf != 1.
 * b200mix_pairwise_azimuth is ScaleAzimuthFront3_2 (alc/alu.cpp:675-708), used when the device
 * renders stereo pair-wise (RenderMode::Pairwise).  Everything is bit-identical to the reference
 * (the ReverseX/Y/Z, nfc-scale and half-angle-cone compatibility options at their defaults). */
typedef struct b200mix_listener_params {
    uint32_t struct_size;
    float position[3];
    float matrix[16];
    float velocity[3];
    float gain, meters_per_unit, air_absorption_gain_hf, doppler_factor, speed_of_sound;
    uint32_t source_distance_model;     /* ContextParams::SourceDistanceModel */
    uint32_t distance_model;            /* enum DistanceModel order: Disable, Inverse, InverseClamped,
                                           Linear, LinearClamped, Exponent, ExponentClamped */
} b200mix_listener_params;
/* ContextProps (core/context.h:46-64) -> b200mix_calc_listener_params = CalcContextParams
 * (alc/alu.cpp:508-555); gain_boost is ContextBase::mGainBoost (1 unless volume-adjust is set). */
typedef struct b200mix_listener_props {
    uint32_t struct_size;
    float position[3], velocity[3], orient_at[3], orient_up[3];
    float gain, gain_boost, meters_per_unit, air_absorption_gain_hf;
    float doppler_factor, doppler_velocity, speed_of_sound;
    uint32_t source_distance_model, distance_model;
} b200mix_listener_props;
typedef struct b200mix_source_send {
    float gain, gain_hf, hf_reference, gain_lf, lf_reference;   /* VoiceProps::SendData */
    uint32_t active;                    /* Slot != null && EffectType != None */
    float slot_room_rolloff, slot_decay_time, slot_air_absorption_gain_hf;   /* EffectSlotBase */
} b200mix_source_send;
typedef struct b200mix_source_props {
    uint32_t struct_size;
    float pitch, gain, outer_gain, min_gain, max_gain, inner_angle, outer_angle;
    float ref_distance, max_distance, rolloff_factor;
    float position[3], velocity[3], direction[3];
    uint32_t head_relative, distance_model;
    uint32_t dry_gain_hf_auto, wet_gain_auto, wet_gain_hf_auto;
    float outer_gain_hf, air_absorption_factor, room_rolloff_factor, doppler_factor, radius;
    struct { float gain, gain_hf, hf_reference, gain_lf, lf_reference; } direct;
    b200mix_source_send sends[B200MIX_MAX_SENDS];
    float orient_at[3], orient_up[3];   /* VoiceProps::OrientAt/OrientUp (B-Format sources) */
} b200mix_source_props;
typedef struct b200mix_source_result {
    uint32_t step;                      /* Voice::mStep */
    float pos[3];                       /* unit vector to the source, listener space */
    float distance, spread;
    float hrtf_elevation, hrtf_azimuth; /* CalcHrtfPanning's src_ev / src_az */
    float dry_gain, dry_gain_hf, dry_gain_lf;                   /* drygain {Base, HF, LF} */
    float wet_gain[B200MIX_MAX_SENDS], wet_gain_hf[B200MIX_MAX_SENDS], wet_gain_lf[B200MIX_MAX_SENDS];
} b200mix_source_result;
B200MIX_API int b200mix_calc_source_params(const b200mix_source_props *props,
    const b200mix_listener_params *listener, uint32_t num_sends, uint32_t buffer_rate,
    uint32_t device_rate, b200mix_source_result *result);
B200MIX_API int b200mix_calc_listener_params(const b200mix_listener_props *props,
    b200mix_listener_params *listener);
B200MIX_API int b200mix_pairwise_azimuth(const float pos[3], float out[3]);

/* Host helper, no GPU: the rate conversion of a convolution effect's impulse response.
 * ConvolutionState::deviceUpdate (alc/effects/convolution.cpp:356-361,417-431) runs an IR whose
 * buffer rate differs from the device's through PPhaseResampler (common/polyphase_resampler.cpp,
 * Kaiser-windowed sinc, 180 dB rejection, double precision) and stores it as float; this is that
 * conversion for one channel, bit-identical.  out_frames is normally
 * b200mix_resampled_ir_frames(src, dst, in_frames) = ceil(in_frames*dst/src); the result feeds
 * b200mix_slot_convolution. */
B200MIX_API int64_t b200mix_resampled_ir_frames(uint32_t src_rate, uint32_t dst_rate, uint32_t frames);
B200MIX_API int b200mix_resample_ir(uint32_t src_rate, uint32_t dst_rate, const float *in,
    uint32_t in_frames, float *out, uint32_t out_frames);

/* Host helpers, no GPU: the reverb's own parameter stage.  b200mix_efx_reverb is ReverbProps
 * (core/effects/base.h:62-86, the AL_EAXREVERB_* properties after the AL layer's clamping).
 * b200mix_reverb_params_from_efx restates ReverbState::deviceUpdate/allocLines
 * (alc/effects/reverb.cpp:728-851) and ReverbState::update (:1222-1351) for one pipeline:
 * every field of b200mix_reverb_params, and — when gains is not NULL — the 8 output gain rows
 * [4 early, 4 late][out_channels] of update3DPanning (:1151-1220) on the target mix described by
 * b200mix_reverb_target.  All values are bit-identical to the reference's.
 * b200mix_reverb_full_update_needed(prev, next) is the fullUpdate test of :1243-1262 (prev NULL:
 * the first update after deviceUpdate, always full). */
typedef struct b200mix_efx_reverb {
    uint32_t struct_size;
    float density, diffusion, gain, gain_hf, gain_lf, decay_time, decay_hf_ratio, decay_lf_ratio;
    float reflections_gain, reflections_delay, reflections_pan[3];
    float late_reverb_gain, late_reverb_delay, late_reverb_pan[3];
    float echo_time, echo_depth, modulation_time, modulation_depth;
    float air_absorption_gain_hf, hf_reference, lf_reference, room_rolloff_factor;
    uint32_t decay_hf_limit;
} b200mix_efx_reverb;
typedef struct b200mix_reverb_target {
    uint32_t struct_size;
    uint32_t sample_rate;           /* DeviceBase::mSampleRate */
    uint32_t device_ambi_order;     /* DeviceBase::mAmbiOrder (above 1: MixOutAmbiUp) */
    uint32_t device_2d;             /* DeviceBase::m2DMixing */
    float    xover_freq;            /* DeviceBase::mXOverFreq (400 Hz by default, core/device.h:238) */
    float    slot_gain;             /* EffectSlotBase::Gain */
    float    reverb_boost;          /* ReverbBoost (alc/effects/base.h:11; 1 unless the reverb/boost option is set) */
    uint32_t out_channels;          /* target.Main->Buffer.size(): Dry, or the target slot's Wet */
    const float *out_scale;         /* target.Main->AmbiMap[c].Scale */
    const uint32_t *out_index;      /* target.Main->AmbiMap[c].Index */
} b200mix_reverb_target;
B200MIX_API int b200mix_reverb_params_from_efx(const b200mix_efx_reverb *props,
    const b200mix_reverb_target *target, struct b200mix_reverb_params *params, float *gains);
B200MIX_API int b200mix_reverb_full_update_needed(const b200mix_efx_reverb *prev,
    const b200mix_efx_reverb *next);

/* ReverbState::deviceUpdate + the first (full) update: allocates and clears the delay
 * lines of both pipelines and installs the parameters.  Output mix gains (8 lines: 4 early
 * then 4 late, EarlyReflections::Gains / LateReverb::Gains) go through
 * b200mix_slot_output_gains and always address the CURRENT pipeline.
 * Both output paths are implemented: MixOutPlain (first-order devices) and MixOutAmbiUp. */
B200MIX_API int b200mix_slot_reverb(b200mix_device *dev, uint32_t slot,
    const b200mix_reverb_params *params);
/* A later ReverbState::update (alc/effects/reverb.cpp:1222-1351) on an installed reverb.
 * params = the post-update values of the pipeline that is current AFTER the update (line
 * lengths must equal the installed ones).
 * full_update == 0: the values are applied to the current pipeline in place; its state is kept
 *   and changed delay taps / tap coefficient cross-fade over the next block exactly as
 *   processEarly/processLate do.
 * full_update != 0 (density, diffusion, decay times, modulation or reference frequencies
 *   changed, reverb.cpp:1243-1262): the reference switches to its other pipeline; the old one
 *   gets its input tap coefficient faded to zero and keeps ringing out beside the new one for
 *   its fade_samples, then its output gains fade to zero and it is cleared
 *   (ReverbState::process :1840-1878, ReverbPipeline::clear :550-566).  The library runs that
 *   state machine; send the new pipeline's output gains with b200mix_slot_output_gains. */
B200MIX_API int b200mix_slot_reverb_update(b200mix_device *dev, uint32_t slot,
    const b200mix_reverb_params *params, uint32_t full_update);

/* The other EFX effects (SURVEY §8f #4): EffectState::deviceUpdate + update + process of
 *   echo        alc/effects/echo.cpp:82-157         (two-tap delay line, damped feedback, L/R spread)
 *   modulator   alc/effects/modulator.cpp:96-199    (ring modulator: sine / saw / square carrier, high-pass)
 *   equalizer   alc/effects/equalizer.cpp:112-183   (low shelf, two peaking bands, high shelf per channel)
 *   compressor  alc/effects/compressor.cpp:80-177   (envelope follower on channel 0 -> gain on all)
 *   dedicated   alc/effects/dedicated.cpp:62-109    (dialogue to front-centre / LFE)
 *   distortion  alc/effects/distortion.cpp:113-303  (B2A, 4x oversampled low-pass -> waveshaper -> band-pass, A2B)
 *   chorus      alc/effects/chorus.cpp:132-425      (chorus and flanger: LFO-modulated cubic taps + feedback, B2A/A2B)
 *   autowah     alc/effects/autowah.cpp:94-205      (envelope follower -> per-sample peaking filter)
 *   vmorpher    alc/effects/vmorpher.cpp:100-330    (two 4-band formant filter banks blended by an LFO)
 *   fshifter    alc/effects/fshifter.cpp:92-366     (analytic signal by a 1024-point STFT Hilbert transform in double,
 *                                                    rotated by a phase accumulator; first-order devices)
 *   pshifter    alc/effects/pshifter.cpp:84-472     (phase vocoder: 1024-point STFT, hop 128, up to 9 wet channels that
 *                                                    follow the phase of channel 0; devices up to second order)
 * b200mix_efx_props carries the effect's PROPERTIES (the EffectProps variant of
 * core/effects/base.h:62-178 after the AL layer's clamping); b200mix_efx_target what update() reads
 * from the slot and its output target: EffectSlotBase::Gain, the target mix's AmbiMap
 * (target.Main: the Dry mix, or the target slot's Wet mix) and the slot's own Wet.AmbiMap
 * indices (setAmbiMixParams, core/device.h:126-147).  The library runs the reference's update()
 * arithmetic on the host (same float expressions, host libm: bit-identical coefficients) and
 * process() on the GPU.  The first call on a slot (or a change of `type`) is deviceUpdate +
 * update: the effect state is created and cleared; later calls are update(): parameters and
 * gain targets change, delay lines / filter histories / current gains are kept.
 * B200MIX_ERR_UNSUPPORTED: more than 16 wet channels; dedicated effects that resolve to a RealOut
 * channel (FrontCenter / LFE present: the reference then writes RealOut, not the mix);
 * distortion / chorus / frequency shifter on a device mixing above first order, the pitch shifter above
 * second order (their up-samplers). */
typedef struct b200mix_efx_props {
    uint32_t struct_size;
    uint32_t type;                      /* enum b200mix_effect, >= B200MIX_EFFECT_ECHO */
    struct { float delay, lr_delay, damping, feedback, spread; } echo;                    /* EchoProps */
    struct { float frequency, high_pass_cutoff; uint32_t waveform; } modulator;           /* 0 sinusoid, 1 sawtooth, 2 square */
    struct { float low_cutoff, low_gain, mid1_center, mid1_gain, mid1_width,
             mid2_center, mid2_gain, mid2_width, high_cutoff, high_gain; } equalizer;     /* EqualizerProps */
    struct { uint32_t on_off; } compressor;                                               /* CompressorProps */
    struct { uint32_t target; float gain; } dedicated;                                    /* 0 dialogue, 1 LFE */
    struct { float edge, gain, lowpass_cutoff, eq_center, eq_bandwidth; } distortion;     /* DistortionProps */
    struct { uint32_t waveform; int32_t phase; float rate, depth, feedback, delay; } chorus; /* ChorusProps (0 sinusoid, 1 triangle) */
    struct { float attack_time, release_time, resonance, peak_gain; } autowah;            /* AutowahProps */
    struct { float rate; uint32_t phoneme_a, phoneme_b;     /* VMorpherPhenome: 0 A, 1 E, 2 I, 3 O, 4 U, 5.. (no formants) */
             int32_t phoneme_a_coarse_tuning, phoneme_b_coarse_tuning;
             uint32_t waveform; } vmorpher;                 /* VmorpherProps (0 sinusoid, 1 triangle, 2 sawtooth) */
    struct { float frequency; uint32_t left_direction, right_direction; } fshifter;  /* FshifterProps (0 down, 1 up, 2 off) */
    struct { int32_t coarse_tune, fine_tune; } pshifter;                                  /* PshifterProps (semitones, cents) */
} b200mix_efx_props;
typedef struct b200mix_efx_target {
    uint32_t struct_size;
    uint32_t sample_rate;               /* DeviceBase::mSampleRate */
    float    slot_gain;                 /* EffectSlotBase::Gain */
    uint32_t out_channels;              /* target.Main->Buffer.size() */
    const float *out_scale;             /* target.Main->AmbiMap[c].Scale */
    const uint32_t *out_index;          /* target.Main->AmbiMap[c].Index */
    uint32_t wet_channels;              /* slot->Wet.Buffer.size() (== the device's wet_channels) */
    const uint32_t *wet_index;          /* slot->Wet.AmbiMap[c].Index */
    uint32_t real_center, real_lfe;     /* RealOut.ChannelIndex[FrontCenter] / [LFE] or B200MIX_NO_SLOT */
    uint32_t device_ambi_order;         /* DeviceBase::mAmbiOrder */
} b200mix_efx_target;
B200MIX_API int b200mix_slot_efx(b200mix_device *dev, uint32_t slot, const b200mix_efx_props *props,
    const b200mix_efx_target *target);

/* EffectSlotBase::Target (AL_SOFT_effect_target, core/effectslot.h:64; alc/alu.cpp:626-633): the
 * slot's effect output is mixed into `target`'s Wet buffer instead of the Dry mix
 * (B200MIX_NO_SLOT restores Dry).  A targeting slot's output gains are then
 * [lines][wet_channels].  Slots run in the reference's order — every slot before its target
 * (alc/alu.cpp:2211-2251); chains must be acyclic. */
B200MIX_API int b200mix_slot_target(b200mix_device *dev, uint32_t slot, uint32_t target);

/* Detaches the effect (EffectSlotType::None): the slot's wet input is ignored. */
B200MIX_API int b200mix_slot_disable(b200mix_device *dev, uint32_t slot);

/* ---- voices: the post-ALU snapshot of Voice (core/voice.h:157-272) ------- */
enum {
    B200MIX_VF_PLAYING   = 1u<<0, /* Voice::Playing */
    B200MIX_VF_STOPPING  = 1u<<1, /* Voice::Stopping: fade to silence this update, then stop */
    B200MIX_VF_STATIC    = 1u<<2, /* VoiceFlag::IsStatic */
    B200MIX_VF_LOOPING   = 1u<<3, /* mLoopBuffer != nullptr */
    B200MIX_VF_HRTF      = 1u<<4, /* VoiceFlag::HasHrtf: direct path is the per-voice HRIR */
    B200MIX_VF_RESET     = 1u<<5, /* fresh voice (Voice::prepare): zero histories, take position,
                                     clear IsFading */
    B200MIX_VF_FADING    = 1u<<6, /* with RESET: start with IsFading set (al/source.cpp:775,2714) */
    B200MIX_VF_STOPPED   = 1u<<7, /* Voice::Stopped: remove from the active set */
    B200MIX_VF_DIRECT    = 1u<<8  /* direct channels (AL_DIRECT_CHANNELS_SOFT): the direct path is
                                     RealOut (mDirect.Buffer = RealOut.Buffer).  Only
                                     b200mix_voices_update_direct takes it (and requires it); the
                                     other update calls ignore the bit and mix the voice into Dry
                                     or through its HRIR */
};
/* Multi-channel sources: the reference mixes every buffer channel as its own mixing channel
 * with its own panning/HRIR (Voice::mChans[c], core/voice.h:236-257; LoadSamples' srcChannel,
 * core/voice.cpp:271-287).  Here each mixing channel is a voice of its own: same buffer,
 * position and step, its own targets, and the buffer channel it reads in bits 16..23. */
#define B200MIX_VF_CHANNEL(c)  (((uint32_t)(c) & 0xffu) << 16)

typedef struct b200mix_voice_params {
    uint32_t voice;           /* index in the device voice array, < max_voices */
    uint32_t flags;           /* B200MIX_VF_* */
    uint32_t buffer;          /* buffer id of mCurrentBuffer (static sources); B200MIX_NO_BUFFER =
                               * mCurrentBuffer is null (alSourceStop / rewind, alc/alu.cpp:2069-2083):
                               * the voice holds its near-zero sample while it fades
                               * (core/voice.cpp:704-719) */
    uint32_t resampler;       /* enum b200mix_resampler (VoiceProps::mResampler) */
    int32_t  position;        /* mPosition      (RESET only) */
    uint32_t position_frac;   /* mPositionFrac  (RESET only) */
    uint32_t loop_start;      /* VoiceBufferItem::mLoopStart */
    uint32_t loop_end;        /* VoiceBufferItem::mLoopEnd */
    uint32_t step;            /* mStep, 16.16 fixed point */
    uint32_t hrtf_delay[2];   /* Hrtf.Target.Delay */
    float    hrtf_gain;       /* Hrtf.Target.Gain */
    uint32_t send_slot[B200MIX_MAX_SENDS]; /* aux slot id per send or B200MIX_NO_SLOT */
} b200mix_voice_params;

/* Applies n parameter snapshots.  Side arrays are indexed like params[]:
 *   hrtf_coeffs [n][ir_size][2]              Hrtf.Target.Coeffs (HRTF voices; may be NULL)
 *   dry_gains   [n][dry_channels]            mDryParams.Gains.Target (non-HRTF; may be NULL)
 *   send_gains  [n][num_sends][wet_channels] mWetParams[s].Gains.Target (may be NULL)
 * A NULL side array leaves the corresponding targets unchanged. */
B200MIX_API int b200mix_voices_update(b200mix_device *dev, uint32_t n,
    const b200mix_voice_params *params, const float *hrtf_coeffs, const float *dry_gains,
    const float *send_gains);

struct b200mix_voice_filter;     /* defined with b200mix_voices_filters below */
/* CalcVoiceParams for a point source in one call (host, no GPU): b200mix_calc_source_params
 * followed by CalcPanningAndFilters' steps (alc/alu.cpp:1196-1226,1318-1361,1619-1656).  Fills, for
 * the voice that plays the source: voice->step, voice->hrtf_gain and the HRTF flag; on HRTF
 * devices (render_mode 2) dir = {elevation, azimuth, distance, spread} for
 * b200mix_voices_update_dirs, otherwise dry_gains[dry.channels] (render_mode 1 = pair-wise stereo);
 * send_gains[num_sends][wet_stride]; filters[1 + num_sends] for b200mix_voices_filters.  The other
 * fields of *voice (buffer, positions, flags, send_slot) are the caller's.  A source exactly at
 * the listener takes the reference's no-distance path (front-centre position, distance = inf for
 * the HRIR lookup, :1268-1310,1420-1466).  Bit-identical to the reference's voices (tests/test_source_params.py). */
typedef struct b200mix_mix_map { uint32_t channels; const float *scale; const uint32_t *index; } b200mix_mix_map;
typedef struct b200mix_voice_env {
    uint32_t struct_size;
    uint32_t device_rate, num_sends;
    uint32_t render_mode;               /* DeviceBase::mRenderMode: 0 Normal, 1 Pairwise, 2 Hrtf */
    uint32_t wet_stride;                /* floats per send in send_gains (>= every wet map's channels) */
    b200mix_mix_map dry;                /* DeviceBase::Dry.AmbiMap */
    b200mix_mix_map wet[B200MIX_MAX_SENDS];   /* the send's slot Wet.AmbiMap; channels 0 = no slot */
} b200mix_voice_env;
B200MIX_API int b200mix_calc_voice(const b200mix_source_props *props,
    const b200mix_listener_params *listener, const b200mix_voice_env *env, uint32_t buffer_rate,
    b200mix_voice_params *voice, float dir[4], float *dry_gains, float *send_gains,
    struct b200mix_voice_filter *filters);

/* b200mix_calc_voice over n independent sources, split over `threads` host threads (the caller's
 * included; 0 or 1 = in the calling thread).  Arrays are indexed like props[]: voices[n],
 * buffer_rates[n], dirs[n][4], dry_gains[n][dry.channels], send_gains[n][num_sends][wet_stride],
 * filters[n][1 + num_sends] — the layout b200mix_voices_update(_dirs) and b200mix_voices_filters
 * take.  Returns the first error any source produced. */
B200MIX_API int b200mix_calc_voices(uint32_t n, const b200mix_source_props *props,
    const b200mix_listener_params *listener, const b200mix_voice_env *env, const uint32_t *buffer_rates,
    b200mix_voice_params *voices, float *dirs, float *dry_gains, float *send_gains,
    struct b200mix_voice_filter *filters, uint32_t threads);

/* The same for a multi-channel source that is not spatialized (stereo music and the like:
 * CalcNonAttnVoiceParams, alc/alu.cpp:1658-1710, then the no-distance branches of
 * CalcHrtfPanning / CalcNormalPanning, :1268-1310,1420-1466): one mixing channel per buffer
 * channel (one ABI voice each, B200MIX_VF_CHANNEL(c)) at the layout's speaker position.  Returns
 * the channel count (or < 0); per channel c: hrtf_gains[c] and dirs[c][4] on HRTF devices,
 * dry_gains[c][dry.channels] otherwise, send_gains[c][num_sends][wet_stride]; *step and
 * filters[1 + num_sends] are shared by all channels.  setup: the buffer's channel layout,
 * VoiceProps::StereoPan (radians, {pi/6, -pi/6} by default) and ::Panning, and the index of the
 * LFE channel in the Dry mix when the Dry mix is the output mix itself (else B200MIX_NO_SLOT). */
enum b200mix_channel_layout { B200MIX_LAYOUT_STEREO = 2, B200MIX_LAYOUT_REAR, B200MIX_LAYOUT_QUAD,
    B200MIX_LAYOUT_X51, B200MIX_LAYOUT_X61, B200MIX_LAYOUT_X71 };
typedef struct b200mix_channel_setup {
    uint32_t struct_size;
    uint32_t layout;                    /* enum b200mix_channel_layout */
    float stereo_pan[2];
    float panning;
    uint32_t lfe_dry_index;
    uint32_t spatialized;               /* AL_SOURCE_SPATIALIZE_SOFT forced on: CalcAttnVoiceParams, the
                                           channels drawn toward the source (alc/alu.cpp:1228-1266,1363-1418) */
} b200mix_channel_setup;
B200MIX_API int b200mix_calc_voice_channels(const b200mix_source_props *props,
    const b200mix_listener_params *listener, const b200mix_voice_env *env, uint32_t buffer_rate,
    const b200mix_channel_setup *setup, uint32_t *step, float *hrtf_gains, float *dirs,
    float *dry_gains, float *send_gains, struct b200mix_voice_filter *filters);

/* And for a B-Format source of order 1..4 (ambient beds: AL_FORMAT_BFORMAT2D/3D_*, AL_SOFT_bformat_hoa)
 * that is not spatialized, on a device that mixes at most the source's order: CalcNonAttnVoiceParams,
 * then CalcAmbisonicPanning at no distance (alc/alu.cpp:911-1077 with coverage 1): the source's
 * orientation (and the listener's, unless head-relative) rotates the sound field — first order by
 * the orientation vectors, the bands above it by AmbiRotator's recursion up to the device's order
 * (alc/alu.cpp:799-889) —, the buffer's channel order and normalisation are folded in, and each
 * mixed buffer channel becomes one non-HRTF voice whose dry/send gains are a row of that matrix.
 * Only the buffer's leading channels up to the device's order are mixed (Voice::prepare,
 * core/voice.cpp:1246-1248): returns that count ((o+1)^2, or 2*o+1 for 2D, o = min(source order,
 * device order)) or < 0; B200MIX_ERR_UNSUPPORTED when the device
 * mixes above the source's order, or mixes a 2D bed periphonically from second order on (the
 * reference then up-samples and band-splits the source, alc/alu.cpp:1001-1036,
 * core/voice.cpp:1082-1089). */
typedef struct b200mix_bformat_setup {
    uint32_t struct_size;
    uint32_t is_2d;                     /* FmtBFormat2D (W, X, Y) instead of FmtBFormat3D */
    uint32_t layout;                    /* AmbiLayout: 0 FuMa, 1 ACN */
    uint32_t scaling;                   /* AmbiScaling: 0 FuMa, 1 SN3D, 2 N3D */
    uint32_t device_ambi_order;         /* DeviceBase::mAmbiOrder */
    uint32_t source_ambi_order;         /* Voice::mAmbiOrder (AL_UNPACK_AMBISONIC_ORDER_SOFT), 1..4; 0 reads as 1 */
    uint32_t device_2d_mixing;          /* DeviceBase::m2DMixing */
} b200mix_bformat_setup;
B200MIX_API int b200mix_calc_voice_bformat(const b200mix_source_props *props,
    const b200mix_listener_params *listener, const b200mix_voice_env *env, uint32_t buffer_rate,
    const b200mix_bformat_setup *setup, uint32_t *step, float *dry_gains, float *send_gains,
    struct b200mix_voice_filter *filters);

/* Streaming sources: the VoiceBufferItem list behind alSourceQueueBuffers
 * (core/voice.h:84-99; LoadBufferQueue core/voice.cpp:546-595; queue advance :1183-1196).
 * A voice updated WITHOUT B200MIX_VF_STATIC plays this list instead of `buffer`:
 * buffers[0] is the current item (mCurrentBuffer), the following ones its mNext chain;
 * loop_index is the item playback continues with after the last one (mLoopBuffer: 0 for a
 * looping source) or B200MIX_NO_LOOP.  position/position_frac count from the start of the
 * current item.  Every update reports how many items were finished in
 * b200mix_voice_result.buffers_done (AsyncBufferCompleteEvent); the mixer advances its own
 * head, and the host re-sends the list (from the then-current item) whenever the
 * application queues or unqueues buffers.  At most B200MIX_MAX_QUEUE items are looked at;
 * count 0 detaches the queue (the voice ends like one whose buffer ran out). */
B200MIX_API int b200mix_voice_queue(b200mix_device *dev, uint32_t voice, uint32_t count,
    const uint32_t *buffers, uint32_t loop_index);

/* Callback buffers (AL_SOFT_callback_buffer, alBufferCallbackSOFT): the application supplies
 * the samples while the source plays.  b200mix_buffer_callback makes `buffer` such a buffer
 * (BufferStorage::mCallback / mUserData, al/buffer.cpp:447-511).  A voice whose `buffer` names
 * it is a callback voice: STATIC must be clear, its queue is ignored, looping too, and it joins
 * with B200MIX_VF_RESET (InitVoice, al/source.cpp:659-662).  All channel voices of one source
 * share the buffer and must agree on step, position and state (else voices_update fails with
 * B200MIX_ERR_INVALID).  B200MIX_VF_RESET on any of them returns the state to 0,0,0.
 *
 * The library calls `callback` on the calling thread inside b200mix_render, _render_device,
 * _render_interleaved and _render_begin, before the update is launched, and nowhere else.  It
 * makes the reference's calls (core/voice.cpp:726-753): per chunk of the update, the missing
 * whole blocks, written at storage + num_blocks*bytes_per_block; a short return ends the
 * stream.  After the update it drops the blocks the voice has passed by moving the rest to
 * the front of `storage` (core/voice.cpp:1155-1180), so `storage` always holds the bytes the
 * reference's buffer holds.  When the stream runs out the voice ends like a static voice at
 * the end of its buffer (Stopping, no buffer).  IMA4 / MSADPCM blocks are decoded on the host
 * as b200mix_buffer_data_adpcm does.  num_blocks / block_offset / stopped give the state to
 * continue from (Voice::mNumCallbackBlocks, mCallbackBlockOffset, CallbackStopped; 0,0,0 for a
 * new stream): to carry a stream over to a new device, register the buffer there after the
 * voices' RESET update.  storage_bytes must be at least the reference's callback storage
 * (al/buffer.cpp:468-473: ceil(((1024 + 256)*10 + 24) / samples_per_block) blocks), which no
 * request passes.  At most 16 channels.  Callback voices are updated with b200mix_voices_update
 * only: b200mix_sources_update refuses them (B200MIX_ERR_UNSUPPORTED), since it computes the
 * step on the GPU, out of the planner's sight.  A callback buffer's voices must live on the
 * device that registered it (sharded sets add no special handling).
 * buffer_data / buffer_free on the id end its callback registration (refused while a voice
 * plays it). */
typedef int (*b200mix_callback_fn)(void *userptr, void *sampledata, int numbytes); /* ALBUFFERCALLBACKTYPESOFT */
typedef struct b200mix_callback_buffer {
    uint32_t struct_size;
    uint32_t sample_type, channels;                 /* enum b200mix_sample_type, incl. IMA4 / MSADPCM */
    uint32_t samples_per_block, bytes_per_block;    /* Voice::mSamplesPerBlock / mBytesPerBlock (1 and the
                                                       frame size for PCM) */
    b200mix_callback_fn callback; void *userptr;    /* VoiceBufferItem::mCallback / mUserData */
    void *storage; size_t storage_bytes;            /* the bytes the callback writes into (BufferStorage) */
    uint32_t num_blocks, block_offset, stopped;     /* state to resume from; 0,0,0 for a new stream */
} b200mix_callback_buffer;
B200MIX_API int b200mix_buffer_callback(b200mix_device *dev, uint32_t buffer, const b200mix_callback_buffer *cb);
/* The buffer's state after the last update (and its callbacks). */
B200MIX_API int b200mix_buffer_callback_state(b200mix_device *dev, uint32_t buffer,
    uint32_t *num_blocks, uint32_t *block_offset, uint32_t *stopped);

/* Direct and send filters: DoFilters -> BiquadInterpFilter::dualProcess
 * (core/voice.cpp:255-268, core/filters/biquad.cpp:254-343).  One entry is the RESULT of
 * the parameter stage's filter block for one path of one voice (alc/alu.cpp:1619-1656):
 * FilterActive plus the two mTargetCoeffs {b0,b1,b2,a1,a2} that
 * lowpass.setParamsFromSlope(HighShelf, hfNorm, gainHF, 1) and
 * highpass.setParamsFromSlope(LowShelf, lfNorm, gainLF, 1) produced.  The library keeps
 * the filter state (z1/z2, current coefficients, mCounter) on the device and applies
 * BiquadInterpFilter::setParams' rule itself: a target that moved by more than 1/64 in
 * any coefficient starts the 8x32-sample interpolation, otherwise Current snaps to Target
 * once the counter has run out.  Forward every setParams call of the reference (once per
 * CalcVoiceParams of that voice); a voice that never had a filter set costs nothing.
 * B200MIX_VF_RESET returns every path of the voice to BiquadInterpFilter's initial state. */
typedef struct b200mix_voice_filter {
    uint32_t voice;
    uint32_t path;            /* 0 = direct (mDryParams), 1+s = send s (mWetParams[s]) */
    uint32_t active;          /* mDirect.FilterActive / mSend[s].FilterActive */
    float    lowpass[5];      /* LowPass.mTargetCoeffs  (high-shelf) */
    float    highpass[5];     /* HighPass.mTargetCoeffs (low-shelf) */
} b200mix_voice_filter;

B200MIX_API int b200mix_voices_filters(b200mix_device *dev, uint32_t n,
    const b200mix_voice_filter *filters);

/* Host helpers, no GPU: the panning half of the parameter stage.
 * b200mix_ambi_coeffs = CalcDirectionCoeffs(dir, spread) (core/mixer.h:68-73 -> CalcAmbiCoeffs,
 * core/mixer.cpp:16-91, core/ambidefs.h:219-272): the 25 N3D/ACN encoder coefficients of the unit
 * vector dir (OpenAL axes), widened by `spread` radians (0..tau).
 * b200mix_pan_gains = ComputePanGains (core/mixer.cpp:93-102) on a mix whose AmbiMap is
 * {scale[c], index[c]} for c < channels (DeviceBase::Dry.AmbiMap or an effect slot's Wet.AmbiMap,
 * core/device.h:109-121): gains[c] = scale[c]*coeffs[index[c]]*ingain, the rest up to gains_len
 * zero — what goes into dry_gains / send_gains of b200mix_voices_update.  Both are bit-identical
 * to the reference's results. */
#define B200MIX_MAX_AMBI_CHANNELS 25u /* MaxAmbiChannels core/ambidefs.h:18-19 */
B200MIX_API int b200mix_ambi_coeffs(const float dir[3], float spread,
    float coeffs[B200MIX_MAX_AMBI_CHANNELS]);
B200MIX_API int b200mix_pan_gains(uint32_t channels, const float *scale, const uint32_t *index,
    const float coeffs[B200MIX_MAX_AMBI_CHANNELS], float ingain, float *gains, uint32_t gains_len);

/* Host helper, no GPU: the reference's built-in decoders for mono (0), stereo (1), quad (2), 5.1
 * (3), 6.1 (4) and 7.1 (5) output — InitPanning (alc/panning.cpp:542-577,718-845) — as the arguments of b200mix_create
 * (dry_channels, real_channels, B200MIX_POST_AMBIDEC) and b200mix_set_ambi_decoder, plus the Dry
 * mix's AmbiMap for the panning helpers.  hq_mode = the decoder/hq-mode option (default on: the
 * quad decoder is dual-band).  gains_* are [dry_channels][real_channels].  Bit-identical to a
 * reference device of that format. */
typedef struct b200mix_builtin_decoder_out {
    uint32_t struct_size;
    uint32_t ambi_order, is_2d, dry_channels, real_channels, dual_band;
    float map_scale[5]; uint32_t map_index[5];
    float gains_hf[5*8], gains_lf[5*8];
    float xover_coeff;
} b200mix_builtin_decoder_out;
B200MIX_API int b200mix_builtin_decoder(uint32_t layout, uint32_t hq_mode, uint32_t sample_rate,
    b200mix_builtin_decoder_out *out);

/* Host helper, no GPU: the output gains of a convolution effect whose impulse response is a
 * plain channel layout — ConvolutionState::update (alc/effects/convolution.cpp:541-620).  layout:
 * 1 = mono, else enum b200mix_channel_layout (stereo ... 7.1); pairwise: the device renders stereo
 * pair-wise (RenderMode::Pairwise); slot_gain: EffectSlotBase::Gain; {channels, scale, index}: the
 * target mix's AmbiMap.  gains receives one row of gains_stride floats per IR channel (the LFE row
 * is zero) for b200mix_slot_output_gains; returns the row count.  Bit-identical to the reference. */
B200MIX_API int b200mix_convolution_gains(uint32_t layout, uint32_t pairwise, float slot_gain,
    uint32_t channels, const float *scale, const uint32_t *index, float *gains, uint32_t gains_stride);

/* Host helper, no GPU: BiquadFilter::SetParams via setParamsFromSlope
 * (core/filters/biquad.h:92-97, biquad.cpp:48-129).  type follows enum BiquadType:
 * 0 HighShelf, 1 LowShelf, 2 Peaking, 3 LowPass, 4 HighPass, 5 BandPass.
 * coeffs receives {b0,b1,b2,a1,a2} with a0 pre-applied. */
B200MIX_API int b200mix_biquad_coeffs(uint32_t type, float f0norm, float gain, float slope,
    float coeffs[5]);

typedef struct b200mix_voice_result {
    int32_t  position;        /* new mPosition */
    uint32_t position_frac;   /* new mPositionFrac */
    uint32_t flags;           /* B200MIX_VF_PLAYING / _STOPPING / _STOPPED after this update */
    uint32_t buffers_done;    /* for AsyncBufferCompleteEvent (queues; 0 for static) */
} b200mix_voice_result;

/* ---- the hot path -------------------------------------------------------- */
/* One mix update of `frames` (1..1024) sample frames:
 * zero MixBuffer, mix every active voice, run the aux slots, post-process.
 * real_out[c] (c < real_channels) are HOST pointers to >= frames floats each
 * (the planar RealOut the host's Write<T> then converts/interleaves).
 * results (nullable) receives max_voices entries. */
B200MIX_API int b200mix_render(b200mix_device *dev, uint32_t frames, float *const *real_out,
    b200mix_voice_result *results);

/* Same update with the output left in device memory (for callers that keep
 * going on the GPU, and for device-timed benchmarking): *real_out_dev is a
 * device pointer to [real_channels][1024] floats valid until the next call. */
B200MIX_API int b200mix_render_device(b200mix_device *dev, uint32_t frames,
    const float **real_out_dev);

/* Output stage on the device: ApplyDither (alc/alu.cpp:2309-2333) followed by the
 * interleaving Write<T> (alc/alu.cpp:2362-2390, SampleConv :2335-2360) of the same update
 * b200mix_render performs.  out receives frames*frame_step samples of out_type (enum DevFmtType
 * order below); frame_step >= real_channels, extra channels get SampleConv<T>(0).
 * dither_depth is DeviceBase::DitherDepth (0 = off; 32768 for 16-bit output), *dither_seed
 * DeviceBase::DitherSeed (22222 at device open), advanced exactly as the reference's LCG.
 * With a limiter installed (b200mix_set_limiter) it runs ahead of the dither, as in
 * DeviceBase::renderSamples (alc/alu.cpp:2446). */
enum b200mix_out_type { B200MIX_OUT_I8 = 0, B200MIX_OUT_U8, B200MIX_OUT_I16, B200MIX_OUT_U16,
    B200MIX_OUT_I32, B200MIX_OUT_U32, B200MIX_OUT_F32 };
B200MIX_API int b200mix_render_interleaved(b200mix_device *dev, uint32_t frames, void *out,
    uint32_t out_type, uint32_t frame_step, float dither_depth, uint32_t *dither_seed,
    b200mix_voice_result *results);

/* The output gain limiter: Compressor (core/mastering.h:25-117, core/mastering.cpp).  The
 * fields are Compressor::Params (core/mastering.h:88-114) — NumChans and SampleRate come from
 * the device — and b200mix_set_limiter derives the state exactly as Compressor::Create
 * (core/mastering.cpp:108-166).  The reference's device limiter (CreateDeviceLimiter,
 * alc/alc.cpp:1079-1091) is {auto_flags = all five, look_ahead_time 0.001, hold_time 0.002,
 * 0 dB pre/post gain, ratio INFINITY, knee 0, attack 0.02, release 0.2} with threshold_db
 * from the output type (alc/alc.cpp:1750-1770).  Once installed, every render applies
 * Compressor::process (core/mastering.cpp:261-379) to RealOut after the post-process stage and
 * before dither/conversion (alc/alu.cpp:2446), keeping its look-ahead delay, peak hold and
 * envelope state in device memory.  desc == NULL removes it (device->Limiter = nullptr).
 * *look_ahead (nullable) receives Compressor::getLookAhead() in samples. */
enum { B200MIX_LIM_AUTO_KNEE = 1u, B200MIX_LIM_AUTO_ATTACK = 2u, B200MIX_LIM_AUTO_RELEASE = 4u,
    B200MIX_LIM_AUTO_POSTGAIN = 8u, B200MIX_LIM_AUTO_DECLIP = 16u };
typedef struct b200mix_limiter_desc {
    uint32_t struct_size;
    uint32_t auto_flags;        /* B200MIX_LIM_AUTO_* (Compressor::FlagBits) */
    float look_ahead_time;      /* seconds */
    float hold_time;            /* seconds */
    float pre_gain_db;
    float post_gain_db;
    float threshold_db;
    float ratio;                /* INFINITY for true limiting */
    float knee_db;
    float attack_time;          /* seconds */
    float release_time;         /* seconds */
} b200mix_limiter_desc;
B200MIX_API int b200mix_set_limiter(b200mix_device *dev, const b200mix_limiter_desc *desc,
    uint32_t *look_ahead);

/* Which encoder a B200MIX_POST_UHJ / B200MIX_POST_TSME device runs (UhjEncodeQuality /
 * TsmeEncodeQuality, alc/alc.cpp:564-597; core/uhjfilter.h, core/tsmefilter.hpp): filter_length
 * 0 = UhjEncoderIIR / TsmeEncoderIIR (the default), 256 / 512 = UhjEncoder<N> / TsmeEncoder<N>
 * (core/uhjfilter.cpp:83-205, core/tsmefilter.cpp:137-278: the +90 degree shift as an N-tap
 * linear-phase FIR, every other signal delayed by N/2 + 128 samples).  Resets the encoder state; *delay (nullable) receives
 * EncoderBase::getDelay() in samples. */
B200MIX_API int b200mix_set_uhj_encoder(b200mix_device *dev, uint32_t filter_length,
    uint32_t *delay);

/* BS2B headphone crossfeed on a stereo B200MIX_POST_AMBIDEC device: Bs2bPostProcess
 * (alc/alu.cpp:408-434; set up at alc/panning.cpp:1421-1432 from the cf_level option) =
 * the ambisonic decode followed by Bs2b::bs2b_processor::cross_feed (core/bs2b.cpp:104-163) on
 * FrontLeft/FrontRight, with the coefficients of core/bs2b.cpp:41-91 for `level` 1..6
 * (Bs2b::LowCLevel .. HighECLevel) at the device rate.  level 0 removes it.  Clears the
 * filter history. */
B200MIX_API int b200mix_set_bs2b(b200mix_device *dev, uint32_t level);

/* Front image stabilizer on a B200MIX_POST_AMBIDEC device with FrontLeft, FrontRight and a
 * FrontCenter output the decoder does not feed: StablizerPostProcess (alc/alu.cpp:330-406; set up
 * by InitPanning/CreateStablizer, alc/panning.cpp:160-172,806-834, front-stablizer option).  After
 * the decode the mid signal L+R is band-split (BandSplitter::process, crossover 5 kHz), part of it
 * is moved to the centre channel, and every other channel passes the splitter's all-pass
 * (BandSplitter::processAllPass) to stay in phase.  splitter_coeff is
 * FrontStablizer::MidFilter.mCoeff (BandSplitter::init(5000/rate), core/filters/splitter.cpp:15-26).
 * center_channel = B200MIX_NO_SLOT removes it.  Clears the filter states. */
B200MIX_API int b200mix_set_front_stabilizer(b200mix_device *dev, uint32_t center_channel,
    float splitter_coeff);

/* Speaker distance compensation: ApplyDistanceComp (alc/alu.cpp:2276-2307) with the per-channel
 * delays and gains InitDistanceComp derived from a custom decoder's speaker distances
 * (alc/panning.cpp:301-371: DistanceComp::ChanData{Buffer.size(), Gain} per RealOut channel).
 * Runs after the limiter and before dither/conversion (alc/alu.cpp:2449-2450).  delays[c] in
 * samples (< 1024 = DistanceComp::MaxDelay, core/device.h:88), 0 = channel untouched (the
 * reference skips channels without a buffer, gain included).  channels == 0 removes it. */
B200MIX_API int b200mix_set_distance_comp(b200mix_device *dev, uint32_t channels,
    const uint32_t *delays, const float *gains);

/* The same update in two halves, for voice-sharded multi-GPU mixing (SURVEY §8e): effects
 * consume the SUMMED wet input of all ranks, so the host reduces the wet buffers between
 * the halves.  b200mix_render_begin clears the mix buffers, mixes this device's voices and
 * finishes its aux sends; *wet_dev is then a DEVICE pointer to the slots' Wet buffers
 * [max_slots][wet_channels][1024] (wet_floats floats) — sum it across ranks in place, on
 * the stream b200mix_stream() returns (e.g. ncclAllReduce).  b200mix_render_end runs the
 * effect slots installed on THIS device (a rank installs only the slots it owns), mixes
 * their output into Dry and post-processes; real_out/results as for b200mix_render (both
 * may be NULL), *real_out_dev (nullable) gets the device pointer like b200mix_render_device.
 * The post-process is linear, so the ranks' RealOut blocks sum to the single-device result. */
B200MIX_API int b200mix_render_begin(b200mix_device *dev, uint32_t frames, float **wet_dev,
    size_t *wet_floats);
B200MIX_API int b200mix_render_end(b200mix_device *dev, float *const *real_out,
    b200mix_voice_result *results, const float **real_out_dev);

/* ---- voice-sharded device sets (SURVEY §8e): one device per GPU, one process per device ----
 * Voices are independent until they add into the mix buffers (core/voice.cpp:962,978;
 * hrtfbase.h:28), so the host deals its voices over `world` devices (each holds only its own
 * voices and buffers) and the LIBRARY performs the two exchanges of an update inside
 * b200mix_render / _render_device / _render_interleaved, on the device's own stream:
 *   1. after the voice loop: the slots' Wet buffers are reduce-scattered — slot s is OWNED by
 *      rank s mod world, which installs its effect (b200mix_slot_*) and receives the sum of
 *      every rank's sends to it (effects consume the summed input, alc/alu.cpp:2252-2256);
 *   2. after the post-process (linear, alc/alu.cpp:2439-2443): the RealOut blocks are summed
 *      onto rank 0; the nonlinear output stage (limiter, distance compensation, dither,
 *      conversion) then runs on rank 0 only.  On the other ranks real_out receives that
 *      rank's partial mix.
 * Two transports:
 *   - peer stores over NVLink (default): b200mix_shard_init allocates this device's receive
 *     block and returns its CUDA IPC handle (B200MIX_SHARD_HANDLE_BYTES); the host gathers the
 *     handles of all ranks by whatever means it has (MPI, a socket, torch.distributed) and
 *     passes the rank-ordered array to b200mix_shard_connect.  Each update a rank writes its
 *     block straight into the receiver's memory and publishes an epoch flag; the receiver sums
 *     in rank order (bit-reproducible).  A peer that stops answering makes render fail with
 *     B200MIX_ERR_CUDA after a time-out instead of hanging.
 *   - NCCL: b200mix_shard_nccl_id (rank 0) creates the ncclUniqueId (128 bytes) the host
 *     broadcasts; b200mix_shard_nccl joins the communicator; an update is one ncclAllReduce of
 *     the Wet buffers (when the device has slots) and one ncclReduce of RealOut.  NCCL is
 *     dlopen()ed (libnccl.so.2): B200MIX_ERR_UNSUPPORTED when it is not installed.
 * b200mix_render_begin/_end are for hosts that exchange the wet buffers themselves and are
 * refused on a sharded device.  b200mix_shard_last_us: with b200mix_profile on, the device time
 * of the last update's two exchanges in microseconds (<0: none). */
#define B200MIX_SHARD_HANDLE_BYTES 64u
#define B200MIX_NCCL_ID_BYTES     128u
B200MIX_API int b200mix_shard_init(b200mix_device *dev, uint32_t rank, uint32_t world, void *handle_out);
B200MIX_API int b200mix_shard_connect(b200mix_device *dev, const void *handles);
B200MIX_API int b200mix_shard_nccl_id(void *id_out);
B200MIX_API int b200mix_shard_nccl(b200mix_device *dev, uint32_t rank, uint32_t world, const void *nccl_id);
B200MIX_API int b200mix_shard_last_us(b200mix_device *dev, float *wet_us, float *real_us);

/* ---- host-side parameter helpers (no GPU involved) -------------------------- */
/* The HRTF data set and the per-voice HRIR lookup of the parameter stage:
 * LoadHrtf03 (core/hrtf_loader.cpp:583-721, "MinPHR03" files such as hrtf/Default HRTF.mhr)
 * and HrtfStore::getCoeffs (core/hrtf.cpp:192-260).  coeffs is [ir_size][2]. */
typedef struct b200mix_hrtf b200mix_hrtf;
B200MIX_API int b200mix_hrtf_load(const void *mhr_data, size_t bytes, b200mix_hrtf **out);
B200MIX_API void b200mix_hrtf_free(b200mix_hrtf *hrtf);
B200MIX_API int b200mix_hrtf_info(const b200mix_hrtf *hrtf, uint32_t *sample_rate, uint32_t *ir_size,
    uint32_t *ir_count);
B200MIX_API int b200mix_hrtf_get_coeffs(const b200mix_hrtf *hrtf, float elevation, float azimuth,
    float distance, float spread, float *coeffs, uint32_t delays[2]);

/* The HRTF decoder of a first-order device from the data set alone (host, no GPU): the
 * virtual-speaker set-up of InitHrtfPanning (alc/panning.cpp:847-1137, hrtf-mode full / ambi1)
 * through DirectHrtfState::build (core/hrtf.cpp:265-366) — what b200mix_set_hrtf_decoder takes.
 * voice_ir_size = DeviceBase::mIrSize (0: the data set's).  coeffs must hold 4*128*2 floats and is
 * filled as [4][*ir_size][2]; returns the channel count (4).  Bit-identical to the reference's
 * DirectHrtfState; B200MIX_ERR_UNSUPPORTED for other ambisonic orders (their decoder matrices
 * are not restated yet). */
B200MIX_API int b200mix_hrtf_build_decoder(const b200mix_hrtf *hrtf, uint32_t ambi_order,
    uint32_t voice_ir_size, uint32_t *ir_size, float *coeffs, float hf_scale[4], float *splitter_coeff);

/* Device-side parameter stage (SURVEY §8f #1): with a data set attached, voices can be
 * updated with their DIRECTIONS instead of pre-blended HRIRs — dirs is [n][4] floats
 * {elevation, azimuth, distance, spread} exactly as CalcHrtfPanning hands them to
 * HrtfStore::getCoeffs (alc/alu.cpp, core/hrtf.cpp:192-260).  The 4-HRIR blend and the
 * delays are then computed on the GPU (16 bytes per moved voice cross the bus instead of
 * ir_size*8), bit-identically to b200mix_hrtf_get_coeffs.  params[i].hrtf_delay is ignored;
 * non-HRTF voices in the same call ignore their dirs row.  The data set's ir_size must not
 * exceed the device's. */
B200MIX_API int b200mix_hrtf_attach(b200mix_device *dev, const b200mix_hrtf *hrtf);
/* The whole parameter stage of point sources on the GPU: CalcVoiceParams ->
 * CalcAttnVoiceParams + CalcPanningAndFilters (alc/alu.cpp:1512-1657,1712-2010).  The host sends,
 * for every source the application touched, its PROPERTIES (b200mix_source_props, what
 * alSourcefv set — the same struct b200mix_calc_voice takes), the listener and the device's mix
 * maps; a kernel computes per source what b200mix_calc_voice computes on a host core — listener
 * transform, distance model, cones, air absorption, send decay, doppler -> step and
 * BsincPrepare, spread, the HRIR direction (then blended from the attached data set exactly as
 * b200mix_voices_update_dirs does) or the dry pan gains, the send gains, and the high-/low-shelf
 * pair of every path with BiquadInterpFilter::setParams' rule — and writes the voice records
 * directly.  What stays with the host is what the AL layer decides: which voice plays the
 * source, its buffer / queue, start offset, loop points, resampler and send slots
 * (b200mix_source_voice; flags as in b200mix_voice_params — the HRTF flag is set by the
 * library from env->render_mode).  env->dry / env->wet[] point at HOST arrays (copied).
 * Requires b200mix_hrtf_attach when env->render_mode == 2.  The arithmetic is the same source
 * text as the host helpers' (csrc/param_math.hpp) compiled without FMA contraction, libm calls in
 * double rounded once: voices come out bit-identical to b200mix_calc_voice's except where the host
 * libm is not correctly rounded (<= 1 ulp). */
typedef struct b200mix_source_voice {
    uint32_t voice;           /* index in the device voice array */
    uint32_t flags;           /* B200MIX_VF_* (HRTF is decided by the library) */
    uint32_t buffer;          /* buffer id (static sources) */
    uint32_t resampler;       /* enum b200mix_resampler */
    int32_t  position;        /* mPosition      (RESET only) */
    uint32_t position_frac;   /* mPositionFrac  (RESET only) */
    uint32_t loop_start, loop_end;
    uint32_t buffer_rate;     /* BufferStorage::mSampleRate (the step is pitch * buffer_rate / device_rate) */
    uint32_t send_slot[B200MIX_MAX_SENDS];
} b200mix_source_voice;
B200MIX_API int b200mix_sources_update(b200mix_device *dev, uint32_t n, const b200mix_source_voice *voices,
    const b200mix_source_props *props, const b200mix_listener_params *listener,
    const b200mix_voice_env *env);
/* Reads back what the parameter stage left in a voice's record (tests): step, the BsincPrepare
 * state {sf, m, l, offset as float bits}, HRTF target gain and delays, dry target gains
 * [dry_channels], send target gains [num_sends][wet_channels], and the filter targets of every
 * path [1 + num_sends] x {active, lowpass[5], highpass[5]} (11 floats, active as 0/1).  Any
 * pointer may be NULL. */
B200MIX_API int b200mix_get_voice_targets(b200mix_device *dev, uint32_t voice, uint32_t *step,
    float bsinc[4], float *hrtf_gain, uint32_t hrtf_delay[2], float *hrtf_coeffs, float *dry_gains,
    float *send_gains, float *filters);
B200MIX_API int b200mix_voices_update_dirs(b200mix_device *dev, uint32_t n,
    const b200mix_voice_params *params, const float *dirs, const float *dry_gains,
    const float *send_gains);
/* Direct-channel voices (CalcDirectPanning, alc/alu.cpp:1142-1195): every entry carries
 * B200MIX_VF_DIRECT and not B200MIX_VF_HRTF, and its direct path mixes into RealOut ahead of the
 * post-process:
 *   real_gains [n][real_channels]           mDryParams.Gains.Target by RealOut channel (may be NULL)
 *   send_gains [n][num_sends][wet_channels] as in b200mix_voices_update (may be NULL)
 * A NULL side array leaves those targets unchanged.  The direct filter (path 0 of
 * b200mix_voices_filters) and the sends work as for any voice.  A voice keeps one set of Current
 * gains whichever mix it feeds, as the reference's voice does: switched between this call and
 * b200mix_voices_update(_dirs) while it plays, it fades from the gains it last had at each
 * channel index.  A later b200mix_voices_update(_dirs) of the voice returns it to the Dry / HRTF
 * path.
 * B200MIX_ERR_UNSUPPORTED, with nothing applied, where the reference never mixes direct
 * channels (RealOut.RemixMap is empty or RealOut is the Dry mix): B200MIX_POST_NONE, UHJ and
 * TSME devices; and, not supported here: sharded device sets and devices with a front
 * stabilizer (while a direct voice is active, b200mix_set_front_stabilizer and joining a set of
 * more than one device through b200mix_shard_init / b200mix_shard_nccl are refused the same way).  The
 * BS2B and HRTF post-processes leave the direct signal unfiltered, as the reference's do.
 * b200mix_sources_update has no direct mode. */
B200MIX_API int b200mix_voices_update_direct(b200mix_device *dev, uint32_t n,
    const b200mix_voice_params *params, const float *real_gains, const float *send_gains);

/* ---- introspection (tests, profiling) ------------------------------------ */
/* Copies the Dry mix of the last update: [dry_channels][1024]. */
B200MIX_API int b200mix_get_dry(b200mix_device *dev, float *dry);
/* Copies resampler tables as the device holds them (bit-compared with the
 * reference's in tests): which = enum b200mix_resampler; returns float count. */
B200MIX_API int64_t b200mix_get_resampler_table(b200mix_device *dev, uint32_t which,
    float *out, size_t max_floats);
/* Taps per output sample a voice with this resampler and step costs (BsincPrepare's m,
 * alc/alu.cpp:140-165; 4 cubic, 2 linear, 1 point) and, in *full (nullable), whether the bsinc
 * runs with scale interpolation (step > 1.0, Resample_BSinc instead of _FastBSinc) — the terms
 * of SURVEY §8(d)'s algorithmic flop count.  < 0 on bad arguments. */
B200MIX_API int b200mix_resampler_taps(b200mix_device *dev, uint32_t resampler, uint32_t step,
    uint32_t *full);
/* Kernel timing for roofline reports: when enabled, the voice loop of every update (the
 * resample kernel through the HRIR FIR kernel, with the direct filters between them) is
 * bracketed by CUDA events on the device's stream; b200mix_last_mix_kernel_ms returns the
 * duration of the most recent one (synchronises the stream), <0 if unavailable. */
B200MIX_API int b200mix_profile(b200mix_device *dev, int enable);
/* With b200mix_profile(dev, 2) every update also records stage marks; this returns the
 * durations (ms) of the last update's 8 stages: 0 clear, 1 resample kernel, 2 direct filters
 * + deferred dry pass + HRIR FIR kernel, 3 row reduction, 4 parked dry bus, 5 aux sends,
 * 6 effect slots + slot output mix, 7 post-process.  Returns the stage count, <0 if
 * unavailable. */
B200MIX_API int b200mix_last_stage_ms(b200mix_device *dev, float *ms, uint32_t count);
B200MIX_API float b200mix_last_mix_kernel_ms(b200mix_device *dev);
/* Number of CUDA kernels this device has launched so far. */
B200MIX_API uint64_t b200mix_launch_count(const b200mix_device *dev);
/* CUDA stream the device launches on (a cudaStream_t), for event timing. */
B200MIX_API void *b200mix_stream(b200mix_device *dev);

#ifdef __cplusplus
}
#endif
#endif /* B200MIX_H */
