"""ctypes mirror of include/b200mix.h (structs + constants) shared by the tests,
the reference harness wrapper and bench.py.  Pure declarations, no compute."""
import ctypes as C

LINE = 1024
HRIR_LENGTH = 128
HRTF_HISTORY = 64
MAX_SENDS = 6
MAX_DRY = 32
MAX_WET = 25
PADDING = 48
NO_SLOT = 0xFFFFFFFF
NO_LOOP = 0xFFFFFFFF
MAX_QUEUE = 32


def vf_channel(c):
    """B200MIX_VF_CHANNEL(c): the buffer channel a voice reads."""
    return (int(c) & 0xff) << 16


(RS_POINT, RS_LINEAR, RS_SPLINE, RS_GAUSSIAN, RS_FAST_BSINC12, RS_BSINC12, RS_FAST_BSINC24,
 RS_BSINC24, RS_FAST_BSINC48, RS_BSINC48) = range(10)
FMT_U8, FMT_I16, FMT_I32, FMT_F32, FMT_F64, FMT_MULAW, FMT_ALAW, FMT_IMA4, FMT_MSADPCM = range(9)
POST_NONE, POST_AMBIDEC, POST_HRTF, POST_UHJ, POST_TSME = range(5)
VF_PLAYING, VF_STOPPING, VF_STATIC, VF_LOOPING, VF_HRTF, VF_RESET, VF_FADING, VF_STOPPED = (
    1 << i for i in range(8))


class DeviceDesc(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("cuda_device", C.c_int32),
                ("sample_rate", C.c_uint32), ("dry_channels", C.c_uint32),
                ("real_channels", C.c_uint32), ("wet_channels", C.c_uint32),
                ("num_sends", C.c_uint32), ("ir_size", C.c_uint32),
                ("post_process", C.c_uint32), ("real_left", C.c_uint32),
                ("real_right", C.c_uint32), ("max_voices", C.c_uint32),
                ("max_buffers", C.c_uint32), ("max_slots", C.c_uint32)]


class VoiceParams(C.Structure):
    _fields_ = [("voice", C.c_uint32), ("flags", C.c_uint32), ("buffer", C.c_uint32),
                ("resampler", C.c_uint32), ("position", C.c_int32),
                ("position_frac", C.c_uint32), ("loop_start", C.c_uint32),
                ("loop_end", C.c_uint32), ("step", C.c_uint32),
                ("hrtf_delay", C.c_uint32 * 2), ("hrtf_gain", C.c_float),
                ("send_slot", C.c_uint32 * MAX_SENDS)]


class VoiceFilter(C.Structure):
    _fields_ = [("voice", C.c_uint32), ("path", C.c_uint32), ("active", C.c_uint32),
                ("lowpass", C.c_float * 5), ("highpass", C.c_float * 5)]


class VoiceResult(C.Structure):
    _fields_ = [("position", C.c_int32), ("position_frac", C.c_uint32),
                ("flags", C.c_uint32), ("buffers_done", C.c_uint32)]


# b200mix_callback_fn (ALBUFFERCALLBACKTYPESOFT): int (*)(void *userptr, void *sampledata, int numbytes)
CALLBACK_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int)


class CallbackBuffer(C.Structure):
    """b200mix_callback_buffer (alBufferCallbackSOFT)."""
    _fields_ = [("struct_size", C.c_uint32), ("sample_type", C.c_uint32), ("channels", C.c_uint32),
                ("samples_per_block", C.c_uint32), ("bytes_per_block", C.c_uint32),
                ("callback", CALLBACK_FN), ("userptr", C.c_void_p),
                ("storage", C.c_void_p), ("storage_bytes", C.c_size_t),
                ("num_blocks", C.c_uint32), ("block_offset", C.c_uint32), ("stopped", C.c_uint32)]


class EfxReverb(C.Structure):
    """b200mix_efx_reverb (ReverbProps, core/effects/base.h:62-86)."""
    _fields_ = [("struct_size", C.c_uint32),
                ("density", C.c_float), ("diffusion", C.c_float), ("gain", C.c_float), ("gain_hf", C.c_float),
                ("gain_lf", C.c_float), ("decay_time", C.c_float), ("decay_hf_ratio", C.c_float),
                ("decay_lf_ratio", C.c_float), ("reflections_gain", C.c_float), ("reflections_delay", C.c_float),
                ("reflections_pan", C.c_float * 3), ("late_reverb_gain", C.c_float),
                ("late_reverb_delay", C.c_float), ("late_reverb_pan", C.c_float * 3), ("echo_time", C.c_float),
                ("echo_depth", C.c_float), ("modulation_time", C.c_float), ("modulation_depth", C.c_float),
                ("air_absorption_gain_hf", C.c_float), ("hf_reference", C.c_float), ("lf_reference", C.c_float),
                ("room_rolloff_factor", C.c_float), ("decay_hf_limit", C.c_uint32)]


class ReverbTarget(C.Structure):
    """b200mix_reverb_target."""
    _fields_ = [("struct_size", C.c_uint32), ("sample_rate", C.c_uint32), ("device_ambi_order", C.c_uint32),
                ("device_2d", C.c_uint32), ("xover_freq", C.c_float), ("slot_gain", C.c_float),
                ("reverb_boost", C.c_float), ("out_channels", C.c_uint32), ("out_scale", C.c_void_p),
                ("out_index", C.c_void_p)]


class LimiterDesc(C.Structure):
    """b200mix_limiter_desc (Compressor::Params, core/mastering.h:88-114)."""
    _fields_ = [("struct_size", C.c_uint32), ("auto_flags", C.c_uint32),
                ("look_ahead_time", C.c_float), ("hold_time", C.c_float),
                ("pre_gain_db", C.c_float), ("post_gain_db", C.c_float),
                ("threshold_db", C.c_float), ("ratio", C.c_float), ("knee_db", C.c_float),
                ("attack_time", C.c_float), ("release_time", C.c_float)]


LIM_AUTO_ALL = 31


def device_limiter(threshold_db: float) -> "LimiterDesc":
    """The reference's device limiter (CreateDeviceLimiter, alc/alc.cpp:1079-1091)."""
    return LimiterDesc(C.sizeof(LimiterDesc), LIM_AUTO_ALL, 0.001, 0.002, 0.0, 0.0, threshold_db,
                       float("inf"), 0.0, 0.02, 0.2)


class ReverbParams(C.Structure):
    _fields_ = [("struct_size", C.c_uint32),
                ("main_len", C.c_uint32), ("late_in_len", C.c_uint32), ("early_ap_len", C.c_uint32),
                ("early_len", C.c_uint32), ("late_ap_len", C.c_uint32), ("late_len", C.c_uint32),
                ("early_tap", C.c_uint32 * 4), ("early_tap_coeff", C.c_float),
                ("late_tap", C.c_uint32 * 4), ("mix_x", C.c_float), ("mix_y", C.c_float),
                ("filter_lp", C.c_float * 5), ("filter_hp", C.c_float * 5),
                ("early_ap_coeff", C.c_float), ("early_ap_offset", C.c_uint32 * 4),
                ("early_offset", C.c_uint32 * 4), ("early_coeff", C.c_float),
                ("late_offset", C.c_uint32 * 4), ("density_gain", C.c_float),
                ("t60_mid_gain", C.c_float * 4),
                ("t60_hf", (C.c_float * 5) * 4), ("t60_lf", (C.c_float * 5) * 4),
                ("mod_step", C.c_uint32), ("mod_depth", C.c_float),
                ("late_ap_coeff", C.c_float), ("late_ap_offset", C.c_uint32 * 4),
                ("fade_samples", C.c_uint32), ("upmix", C.c_uint32), ("order_scale", C.c_float * 2),
                ("splitter_coeff", C.c_float)]


def reverb_params_from(raw) -> "ReverbParams":
    """ReverbParams from stored bytes (fixtures written before a field was appended are
    zero-extended; struct_size is refreshed)."""
    raw = bytes(raw)
    n = C.sizeof(ReverbParams)
    p = ReverbParams.from_buffer_copy(raw[:n].ljust(n, b"\0"))
    p.struct_size = n
    return p


# ---- host parameter stage (b200mix_calc_listener_params / _source_params / _voice*) ----
class ListenerParams(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("position", C.c_float * 3), ("matrix", C.c_float * 16),
                ("velocity", C.c_float * 3), ("gain", C.c_float), ("meters_per_unit", C.c_float),
                ("air_absorption_gain_hf", C.c_float), ("doppler_factor", C.c_float),
                ("speed_of_sound", C.c_float), ("source_distance_model", C.c_uint32),
                ("distance_model", C.c_uint32)]


class ListenerProps(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("position", C.c_float * 3), ("velocity", C.c_float * 3),
                ("orient_at", C.c_float * 3), ("orient_up", C.c_float * 3), ("gain", C.c_float),
                ("gain_boost", C.c_float), ("meters_per_unit", C.c_float), ("air_absorption_gain_hf", C.c_float),
                ("doppler_factor", C.c_float), ("doppler_velocity", C.c_float), ("speed_of_sound", C.c_float),
                ("source_distance_model", C.c_uint32), ("distance_model", C.c_uint32)]


class SourceSend(C.Structure):
    _fields_ = [("gain", C.c_float), ("gain_hf", C.c_float), ("hf_reference", C.c_float),
                ("gain_lf", C.c_float), ("lf_reference", C.c_float), ("active", C.c_uint32),
                ("slot_room_rolloff", C.c_float), ("slot_decay_time", C.c_float),
                ("slot_air_absorption_gain_hf", C.c_float)]


class SourceDirect(C.Structure):
    _fields_ = [("gain", C.c_float), ("gain_hf", C.c_float), ("hf_reference", C.c_float),
                ("gain_lf", C.c_float), ("lf_reference", C.c_float)]


class SourceProps(C.Structure):
    _fields_ = [("struct_size", C.c_uint32)] + [(n, C.c_float) for n in (
        "pitch", "gain", "outer_gain", "min_gain", "max_gain", "inner_angle", "outer_angle", "ref_distance",
        "max_distance", "rolloff_factor")] + [("position", C.c_float * 3), ("velocity", C.c_float * 3),
        ("direction", C.c_float * 3), ("head_relative", C.c_uint32), ("distance_model", C.c_uint32),
        ("dry_gain_hf_auto", C.c_uint32), ("wet_gain_auto", C.c_uint32), ("wet_gain_hf_auto", C.c_uint32),
        ("outer_gain_hf", C.c_float), ("air_absorption_factor", C.c_float), ("room_rolloff_factor", C.c_float),
        ("doppler_factor", C.c_float), ("radius", C.c_float), ("direct", SourceDirect),
        ("sends", SourceSend * MAX_SENDS), ("orient_at", C.c_float * 3), ("orient_up", C.c_float * 3)]


class SourceResult(C.Structure):
    _fields_ = [("step", C.c_uint32), ("pos", C.c_float * 3), ("distance", C.c_float), ("spread", C.c_float),
                ("hrtf_elevation", C.c_float), ("hrtf_azimuth", C.c_float), ("dry_gain", C.c_float),
                ("dry_gain_hf", C.c_float), ("dry_gain_lf", C.c_float), ("wet_gain", C.c_float * MAX_SENDS),
                ("wet_gain_hf", C.c_float * MAX_SENDS), ("wet_gain_lf", C.c_float * MAX_SENDS)]


class MixMap(C.Structure):
    _fields_ = [("channels", C.c_uint32), ("scale", C.c_void_p), ("index", C.c_void_p)]


class VoiceEnv(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("device_rate", C.c_uint32), ("num_sends", C.c_uint32),
                ("render_mode", C.c_uint32), ("wet_stride", C.c_uint32), ("dry", MixMap),
                ("wet", MixMap * MAX_SENDS)]


class SourceVoice(C.Structure):
    """b200mix_source_voice: what the host still decides per voice for b200mix_sources_update."""
    _fields_ = [("voice", C.c_uint32), ("flags", C.c_uint32), ("buffer", C.c_uint32), ("resampler", C.c_uint32),
                ("position", C.c_int32), ("position_frac", C.c_uint32), ("loop_start", C.c_uint32),
                ("loop_end", C.c_uint32), ("buffer_rate", C.c_uint32), ("send_slot", C.c_uint32 * MAX_SENDS)]


(EFFECT_NONE, EFFECT_CONVOLUTION, EFFECT_REVERB, EFFECT_ECHO, EFFECT_MODULATOR, EFFECT_EQUALIZER,
 EFFECT_COMPRESSOR, EFFECT_DEDICATED, EFFECT_DISTORTION, EFFECT_CHORUS, EFFECT_AUTOWAH, EFFECT_VMORPHER,
 EFFECT_FSHIFTER, EFFECT_PSHIFTER) = range(14)


class _EfxEcho(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("delay", "lr_delay", "damping", "feedback", "spread")]


class _EfxModulator(C.Structure):
    _fields_ = [("frequency", C.c_float), ("high_pass_cutoff", C.c_float), ("waveform", C.c_uint32)]


class _EfxEqualizer(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("low_cutoff", "low_gain", "mid1_center", "mid1_gain", "mid1_width",
                                          "mid2_center", "mid2_gain", "mid2_width", "high_cutoff", "high_gain")]


class _EfxCompressor(C.Structure):
    _fields_ = [("on_off", C.c_uint32)]


class _EfxDedicated(C.Structure):
    _fields_ = [("target", C.c_uint32), ("gain", C.c_float)]


class _EfxDistortion(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("edge", "gain", "lowpass_cutoff", "eq_center", "eq_bandwidth")]


class _EfxChorus(C.Structure):
    _fields_ = [("waveform", C.c_uint32), ("phase", C.c_int32), ("rate", C.c_float), ("depth", C.c_float),
                ("feedback", C.c_float), ("delay", C.c_float)]


class _EfxAutowah(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("attack_time", "release_time", "resonance", "peak_gain")]


class _EfxVmorpher(C.Structure):
    _fields_ = [("rate", C.c_float), ("phoneme_a", C.c_uint32), ("phoneme_b", C.c_uint32),
                ("phoneme_a_coarse_tuning", C.c_int32), ("phoneme_b_coarse_tuning", C.c_int32), ("waveform", C.c_uint32)]


class _EfxFshifter(C.Structure):
    _fields_ = [("frequency", C.c_float), ("left_direction", C.c_uint32), ("right_direction", C.c_uint32)]


class _EfxPshifter(C.Structure):
    _fields_ = [("coarse_tune", C.c_int32), ("fine_tune", C.c_int32)]


class EfxProps(C.Structure):
    """b200mix_efx_props: the EFX effect's properties (EffectProps, core/effects/base.h)."""
    _fields_ = [("struct_size", C.c_uint32), ("type", C.c_uint32), ("echo", _EfxEcho), ("modulator", _EfxModulator),
                ("equalizer", _EfxEqualizer), ("compressor", _EfxCompressor), ("dedicated", _EfxDedicated),
                ("distortion", _EfxDistortion), ("chorus", _EfxChorus), ("autowah", _EfxAutowah),
                ("vmorpher", _EfxVmorpher), ("fshifter", _EfxFshifter), ("pshifter", _EfxPshifter)]


class EfxTarget(C.Structure):
    """b200mix_efx_target: what EffectState::update reads from the slot and its output target."""
    _fields_ = [("struct_size", C.c_uint32), ("sample_rate", C.c_uint32), ("slot_gain", C.c_float),
                ("out_channels", C.c_uint32), ("out_scale", C.c_void_p), ("out_index", C.c_void_p),
                ("wet_channels", C.c_uint32), ("wet_index", C.c_void_p), ("real_center", C.c_uint32),
                ("real_lfe", C.c_uint32), ("device_ambi_order", C.c_uint32)]


def efx_defaults(effect_type):
    """The EFX defaults of include/AL/efx.h (AL_*_DEFAULT_*) for one effect type."""
    p = EfxProps()
    p.struct_size = C.sizeof(EfxProps)
    p.type = effect_type
    p.echo = _EfxEcho(0.1, 0.1, 0.5, 0.5, -1.0)
    p.modulator = _EfxModulator(440.0, 800.0, 0)
    p.equalizer = _EfxEqualizer(200.0, 1.0, 500.0, 1.0, 1.0, 3000.0, 1.0, 1.0, 6000.0, 1.0)
    p.compressor = _EfxCompressor(1)
    p.dedicated = _EfxDedicated(0, 1.0)
    p.distortion = _EfxDistortion(0.2, 0.05, 8000.0, 3600.0, 3600.0)
    p.chorus = _EfxChorus(1, 90, 1.1, 0.1, 0.25, 0.016)
    p.autowah = _EfxAutowah(0.06, 0.06, 1000.0, 11.22)
    p.vmorpher = _EfxVmorpher(1.41, 0, 10, 0, 0, 0)       # phoneme A -> ER, sinusoid
    p.fshifter = _EfxFshifter(0.0, 0, 0)                  # 0 Hz, both sides down
    p.pshifter = _EfxPshifter(12, 0)                      # one octave up
    return p


class ChannelSetup(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("layout", C.c_uint32), ("stereo_pan", C.c_float * 2),
                ("panning", C.c_float), ("lfe_dry_index", C.c_uint32), ("spatialized", C.c_uint32)]


class BFormatSetup(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("is_2d", C.c_uint32), ("layout", C.c_uint32),
                ("scaling", C.c_uint32), ("device_ambi_order", C.c_uint32),
                ("source_ambi_order", C.c_uint32), ("device_2d_mixing", C.c_uint32)]
