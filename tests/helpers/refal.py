"""ctypes driver for the UNMODIFIED reference (oracle/_ref/libopenal_ref.so) through
its public loopback API (include/AL/alext.h:318-345), plus the state/kernel taps
of oracle/ref_harness.cpp.  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "openal-soft_b200"))
from pyb200mix import abi  # noqa: E402

REF_DIR = os.path.join(ROOT, "oracle", "_ref")

# AL / ALC enums (include/AL/al.h, alc.h, alext.h, efx.h)
AL_NONE = 0
AL_SOURCE_RELATIVE = 0x202
AL_PITCH = 0x1003
AL_POSITION = 0x1004
AL_LOOPING = 0x1007
AL_BUFFER = 0x1009
AL_GAIN = 0x100A
AL_SOURCE_STATE = 0x1010
AL_PLAYING = 0x1012
AL_ROLLOFF_FACTOR = 0x1021
AL_FORMAT_MONO8 = 0x1100
AL_FORMAT_MONO16 = 0x1101
AL_FORMAT_MONO_FLOAT32 = 0x10010
AL_FORMAT_STEREO16 = 0x1103
AL_DISTANCE_MODEL = 0xD000
AL_SOURCE_RESAMPLER_SOFT = 0x1212
AL_SOURCE_SPATIALIZE_SOFT = 0x1214
AL_SAMPLE_OFFSET = 0x1025
AL_AUXILIARY_SEND_FILTER = 0x20006
AL_EFFECT_TYPE = 0x8001
AL_EFFECT_EAXREVERB = 0x8000
AL_EFFECT_CONVOLUTION_SOFT = 0xA000
AL_EFFECTSLOT_GAIN = 0x0002
AL_EFFECTSLOT_EFFECT = 0x0001
AL_FILTER_NULL = 0
AL_DIRECT_FILTER = 0x20005
AL_FILTER_TYPE = 0x8001
AL_FILTER_LOWPASS = 0x0001
AL_FILTER_HIGHPASS = 0x0002
AL_FILTER_BANDPASS = 0x0003
AL_LOWPASS_GAIN = 0x0001
AL_LOWPASS_GAINHF = 0x0002
AL_BANDPASS_GAIN = 0x0001
AL_BANDPASS_GAINLF = 0x0002
AL_BANDPASS_GAINHF = 0x0003
ALC_FREQUENCY = 0x1007
ALC_MONO_SOURCES = 0x1010
ALC_STEREO_SOURCES = 0x1011
ALC_FORMAT_CHANNELS_SOFT = 0x1990
ALC_FORMAT_TYPE_SOFT = 0x1991
ALC_FLOAT_SOFT = 0x1406
ALC_SHORT_SOFT = 0x1402
ALC_UNSIGNED_BYTE_SOFT = 0x1401
ALC_STEREO_SOFT = 0x1501
ALC_QUAD_SOFT = 0x1503
ALC_5POINT1_SOFT = 0x1504
ALC_BFORMAT3D_SOFT = 0x1507
ALC_HRTF_SOFT = 0x1992
ALC_HRTF_STATUS_SOFT = 0x1993
ALC_AMBISONIC_LAYOUT_SOFT = 0x1997
ALC_AMBISONIC_SCALING_SOFT = 0x1998
ALC_AMBISONIC_ORDER_SOFT = 0x1999
ALC_ACN_SOFT = 1
ALC_N3D_SOFT = 2
ALC_OUTPUT_MODE_SOFT = 0x19AC
ALC_STEREO_BASIC_SOFT = 0x19AE
ALC_STEREO_UHJ_SOFT = 0x19AF
ALC_STEREO_HRTF_SOFT = 0x19B2
ALC_MAX_AUXILIARY_SENDS = 0x20003
ALC_OUTPUT_LIMITER_SOFT = 0x199A


class VoiceState(C.Structure):
    _fields_ = [("play_state", C.c_int32), ("is_fading", C.c_uint32), ("position", C.c_int32),
                ("position_frac", C.c_uint32), ("buffer_frames", C.c_uint32),
                ("buffer_type", C.c_uint32), ("buffer_channels", C.c_uint32),
                ("bsinc_m", C.c_uint32), ("bsinc_l", C.c_uint32), ("bsinc_sf", C.c_float),
                ("buffer_data", C.c_void_p),
                ("prev_samples", C.c_float * abi.PADDING),
                ("hrtf_history", C.c_float * abi.HRTF_HISTORY),
                ("old_coeffs", (C.c_float * 2) * abi.HRIR_LENGTH),
                ("old_delay", C.c_uint32 * 2), ("old_gain", C.c_float),
                ("cur_dry_gains", C.c_float * abi.MAX_DRY),
                ("cur_send_gains", (C.c_float * abi.MAX_WET) * abi.MAX_SENDS)]


def available() -> bool:
    return (os.path.exists(os.path.join(REF_DIR, "libopenal_ref.so"))
            and os.path.exists(os.path.join(REF_DIR, "libref_harness.so")))


_libs = None


def libs(conf_text: str | None = None):
    """Loads the reference once per process.  conf_text (alsoft.conf syntax) must be
    given on the FIRST call: the reference reads ALSOFT_CONF at its first use."""
    global _libs
    if _libs is not None:
        return _libs
    # outside the tree, which may be read-only
    fd, conf_path = tempfile.mkstemp(prefix="alsoft_", suffix=".conf")
    with os.fdopen(fd, "w") as f:
        f.write(conf_text or "[general]\n")
    os.environ["ALSOFT_CONF"] = conf_path
    import atexit
    atexit.register(lambda: os.path.exists(conf_path) and os.remove(conf_path))
    os.environ.setdefault("ALSOFT_LOGLEVEL", "1")
    al = C.CDLL(os.path.join(REF_DIR, "libopenal_ref.so"), mode=C.RTLD_GLOBAL)
    hz = C.CDLL(os.path.join(REF_DIR, "libref_harness.so"))
    al.alcLoopbackOpenDeviceSOFT.restype = C.c_void_p
    al.alcLoopbackOpenDeviceSOFT.argtypes = [C.c_char_p]
    al.alcCreateContext.restype = C.c_void_p
    al.alcCreateContext.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
    al.alcMakeContextCurrent.argtypes = [C.c_void_p]
    al.alcDestroyContext.argtypes = [C.c_void_p]
    al.alcCloseDevice.argtypes = [C.c_void_p]
    al.alcGetIntegerv.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int)]
    al.alcRenderSamplesSOFT.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    al.alcGetError.argtypes = [C.c_void_p]
    al.alGenBuffers.argtypes = [C.c_int, C.POINTER(C.c_uint)]
    al.alGenSources.argtypes = [C.c_int, C.POINTER(C.c_uint)]
    al.alBufferData.argtypes = [C.c_uint, C.c_int, C.c_void_p, C.c_int, C.c_int]
    al.alSourcei.argtypes = [C.c_uint, C.c_int, C.c_int]
    al.alSourcef.argtypes = [C.c_uint, C.c_int, C.c_float]
    al.alSource3f.argtypes = [C.c_uint, C.c_int, C.c_float, C.c_float, C.c_float]
    al.alSource3i.argtypes = [C.c_uint, C.c_int, C.c_int, C.c_int, C.c_int]
    al.alSourceQueueBuffers.argtypes = [C.c_uint, C.c_int, C.POINTER(C.c_uint)]
    al.alSourcePlayv.argtypes = [C.c_int, C.POINTER(C.c_uint)]
    al.alSourceStopv.argtypes = [C.c_int, C.POINTER(C.c_uint)]
    al.alDistanceModel.argtypes = [C.c_int]
    al.alGetSourcei.argtypes = [C.c_uint, C.c_int, C.POINTER(C.c_int)]
    al.alcDevicePauseSOFT.argtypes = [C.c_void_p]
    hz.refh_device_desc.argtypes = [C.c_void_p, C.POINTER(abi.DeviceDesc)]
    hz.refh_hrtf_decoder.argtypes = [C.c_void_p, C.POINTER(C.c_uint32)] + [C.c_void_p] * 3
    hz.refh_ambi_decoder.argtypes = [C.c_void_p] + [C.c_void_p] * 3 + [C.POINTER(C.c_int)]
    hz.refh_voice_count.argtypes = [C.c_void_p]
    hz.refh_snapshot_voices.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_uint32, C.c_void_p]
    hz.refh_slot_count.argtypes = [C.c_void_p]
    hz.refh_slot_wet_channels.argtypes = [C.c_void_p, C.c_int]
    hz.refh_mono_line_gains.argtypes = [C.c_void_p, C.c_float, C.c_void_p]
    hz.refh_mono_line_gains_slot.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_void_p]
    hz.refh_dither_depth.argtypes = [C.c_void_p]
    hz.refh_dither_depth.restype = C.c_float
    hz.refh_limiter_desc.argtypes = [C.c_void_p, C.c_void_p]
    hz.refh_distance_comp.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    hz.refh_front_stabilizer.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    hz.refh_set_snapshot_channel.argtypes = [C.c_int]
    hz.refh_set_snapshot_channel.restype = None
    hz.refh_voice_filters.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    hz.refh_biquad_coeffs.argtypes = [C.c_int, C.c_float, C.c_float, C.c_float, C.c_void_p]
    hz.refh_biquad_coeffs.restype = None
    al.alFilteri.argtypes = [C.c_uint, C.c_int, C.c_int]
    al.alFilterf.argtypes = [C.c_uint, C.c_int, C.c_float]
    for fn in ("alGenEffects", "alGenAuxiliaryEffectSlots", "alGenFilters"):
        getattr(al, fn).argtypes = [C.c_int, C.POINTER(C.c_uint)]
    al.alEffecti.argtypes = [C.c_uint, C.c_int, C.c_int]
    al.alEffectf.argtypes = [C.c_uint, C.c_int, C.c_float]
    al.alAuxiliaryEffectSloti.argtypes = [C.c_uint, C.c_int, C.c_int]
    al.alAuxiliaryEffectSlotf.argtypes = [C.c_uint, C.c_int, C.c_float]
    hz.refh_get_hrtf_accum.argtypes = [C.c_void_p, C.c_void_p]
    hz.refh_get_dry.argtypes = [C.c_void_p, C.c_void_p]
    hz.refh_resample.argtypes = [C.c_uint32, C.c_int, C.c_uint32, C.c_uint32, C.c_void_p,
                                 C.c_uint32, C.c_void_p, C.c_uint32]
    hz.refh_bsinc_state.argtypes = [C.c_uint32, C.c_uint32, C.POINTER(C.c_float),
                                    C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                    C.POINTER(C.c_uint32)]
    hz.refh_bsinc_table.restype = C.c_int64
    hz.refh_bsinc_table.argtypes = [C.c_uint32, C.c_void_p, C.c_size_t]
    hz.refh_cubic_table.argtypes = [C.c_int, C.c_void_p]
    hz.refh_cubic_filter.argtypes = [C.c_void_p]
    _libs = (al, hz)
    return _libs


class RefDevice:
    """A loopback device + context on the reference.  Stereo float32 by default."""

    def __init__(self, attrs: dict, conf_text: str | None = None):
        self.al, self.hz = libs(conf_text)
        self.dev = self.al.alcLoopbackOpenDeviceSOFT(None)
        assert self.dev, "alcLoopbackOpenDeviceSOFT failed"
        a = {ALC_FORMAT_CHANNELS_SOFT: ALC_STEREO_SOFT, ALC_FORMAT_TYPE_SOFT: ALC_FLOAT_SOFT,
             ALC_FREQUENCY: 48000}
        a.update(attrs)
        flat = []
        for k, v in a.items():
            flat += [k, v]
        flat.append(0)
        arr = (C.c_int * len(flat))(*flat)
        self.ctx = self.al.alcCreateContext(self.dev, arr)
        assert self.ctx, f"alcCreateContext failed: {self.al.alcGetError(self.dev):#x}"
        self.al.alcMakeContextCurrent(self.ctx)
        self.buffers = []
        self.sources = []
        self._keep = []
        self.desc = abi.DeviceDesc()
        rc = self.hz.refh_device_desc(self.dev, C.byref(self.desc))
        assert rc == 0, f"refh_device_desc {rc}"
        self.out_channels = 2

    def close(self):
        self.al.alcMakeContextCurrent(None)
        self.al.alcDestroyContext(self.ctx)
        self.al.alcCloseDevice(self.dev)

    def hrtf_enabled(self) -> bool:
        v = C.c_int(0)
        self.al.alcGetIntegerv(self.dev, ALC_HRTF_STATUS_SOFT, 1, C.byref(v))
        return v.value == 1

    def add_voice(self, pcm: np.ndarray, rate: int, pitch: float, pos, gain: float,
                  resampler: int | None, looping: bool = True, fmt=AL_FORMAT_MONO16):
        b = C.c_uint(0)
        s = C.c_uint(0)
        self.al.alGenBuffers(1, C.byref(b))
        pcm = np.ascontiguousarray(pcm)
        self.al.alBufferData(b, fmt, pcm.ctypes.data, pcm.nbytes, rate)
        self.al.alGenSources(1, C.byref(s))
        self.al.alSourcei(s, AL_BUFFER, b.value)
        self.al.alSourcei(s, AL_LOOPING, 1 if looping else 0)
        self.al.alSourcef(s, AL_PITCH, pitch)
        self.al.alSourcef(s, AL_GAIN, gain)
        self.al.alSource3f(s, AL_POSITION, *[float(x) for x in pos])
        if resampler is not None:
            self.al.alSourcei(s, AL_SOURCE_RESAMPLER_SOFT, resampler)
        err = self.al.alGetError()
        assert err == 0, f"AL error {err:#x}"
        self.buffers.append(b.value)
        self.sources.append(s.value)
        self._keep.append(pcm)
        return s.value

    def add_queue_voice(self, pcms, rate: int, pitch: float, pos, gain: float,
                        resampler: int | None, looping: bool = False, fmt=AL_FORMAT_MONO16):
        """A streaming source: alSourceQueueBuffers with one buffer per PCM array."""
        ids = (C.c_uint * len(pcms))()
        self.al.alGenBuffers(len(pcms), ids)
        for i, pcm in enumerate(pcms):
            pcm = np.ascontiguousarray(pcm)
            self.al.alBufferData(ids[i], fmt, pcm.ctypes.data, pcm.nbytes, rate)
            self._keep.append(pcm)
        s = C.c_uint(0)
        self.al.alGenSources(1, C.byref(s))
        self.al.alSourceQueueBuffers(s, len(pcms), ids)
        self.al.alSourcei(s, AL_LOOPING, 1 if looping else 0)
        self.al.alSourcef(s, AL_PITCH, pitch)
        self.al.alSourcef(s, AL_GAIN, gain)
        self.al.alSource3f(s, AL_POSITION, *[float(x) for x in pos])
        if resampler is not None:
            self.al.alSourcei(s, AL_SOURCE_RESAMPLER_SOFT, resampler)
        err = self.al.alGetError()
        assert err == 0, f"AL error {err:#x}"
        self.buffers += list(ids)
        self.sources.append(s.value)
        return s.value

    def add_convolution_slot(self, ir_pcm: np.ndarray, rate: int, slot_gain: float = 1.0,
                             fmt=AL_FORMAT_MONO_FLOAT32):
        """examples/alconvolve.c:448-450: IR buffer on an aux slot + the convolution effect."""
        b = C.c_uint(0)
        e = C.c_uint(0)
        s = C.c_uint(0)
        ir_pcm = np.ascontiguousarray(ir_pcm)
        self.al.alGenBuffers(1, C.byref(b))
        self.al.alBufferData(b, fmt, ir_pcm.ctypes.data, ir_pcm.nbytes, rate)
        self.al.alGenEffects(1, C.byref(e))
        self.al.alEffecti(e, AL_EFFECT_TYPE, AL_EFFECT_CONVOLUTION_SOFT)
        self.al.alGenAuxiliaryEffectSlots(1, C.byref(s))
        self.al.alAuxiliaryEffectSloti(s, AL_BUFFER, b.value)
        self.al.alAuxiliaryEffectSlotf(s, AL_EFFECTSLOT_GAIN, slot_gain)
        self.al.alAuxiliaryEffectSloti(s, AL_EFFECTSLOT_EFFECT, e.value)
        err = self.al.alGetError()
        assert err == 0, f"AL error {err:#x} creating convolution slot"
        self._keep.append(ir_pcm)
        return s.value

    def add_reverb_slot(self, eax: bool = True, props: dict | None = None, slot_gain: float = 1.0):
        """examples/alreverb.c: an (EAX) reverb effect on an aux slot; props = {AL_param: float}."""
        e = C.c_uint(0)
        s = C.c_uint(0)
        self.al.alGenEffects(1, C.byref(e))
        self.al.alEffecti(e, AL_EFFECT_TYPE, AL_EFFECT_EAXREVERB if eax else 0x0001)
        for k, v in (props or {}).items():
            self.al.alEffectf(e, k, float(v))
        self.al.alGenAuxiliaryEffectSlots(1, C.byref(s))
        self.al.alAuxiliaryEffectSlotf(s, AL_EFFECTSLOT_GAIN, slot_gain)
        self.al.alAuxiliaryEffectSloti(s, AL_EFFECTSLOT_EFFECT, e.value)
        err = self.al.alGetError()
        assert err == 0, f"AL error {err:#x} creating reverb slot"
        self._slot_effect = getattr(self, "_slot_effect", {})
        self._slot_effect[s.value] = e.value
        return s.value

    def add_efx_slot(self, al_type: int, fprops: dict | None = None, iprops: dict | None = None,
                     slot_gain: float = 1.0):
        """Any EFX effect on an aux slot: fprops {AL_param: float} via alEffectf, iprops via alEffecti."""
        e = C.c_uint(0)
        s = C.c_uint(0)
        self.al.alGenEffects(1, C.byref(e))
        self.al.alEffecti(e, AL_EFFECT_TYPE, al_type)
        for k, v in (fprops or {}).items():
            self.al.alEffectf(e, k, float(v))
        for k, v in (iprops or {}).items():
            self.al.alEffecti(e, k, int(v))
        self.al.alGenAuxiliaryEffectSlots(1, C.byref(s))
        self.al.alAuxiliaryEffectSlotf(s, AL_EFFECTSLOT_GAIN, slot_gain)
        self.al.alAuxiliaryEffectSloti(s, AL_EFFECTSLOT_EFFECT, e.value)
        err = self.al.alGetError()
        assert err == 0, f"AL error {err:#x} creating effect slot {al_type:#x}"
        self._slot_effect = getattr(self, "_slot_effect", {})
        self._slot_effect[s.value] = e.value
        return s.value

    def change_efx(self, slot: int, fprops: dict | None = None, iprops: dict | None = None):
        """Changes properties of the slot's effect and re-applies it (EffectState::update)."""
        e = self._slot_effect[slot]
        for k, v in (fprops or {}).items():
            self.al.alEffectf(e, k, float(v))
        for k, v in (iprops or {}).items():
            self.al.alEffecti(e, k, int(v))
        self.al.alAuxiliaryEffectSloti(slot, AL_EFFECTSLOT_EFFECT, e)
        err = self.al.alGetError()
        assert err == 0, f"AL error {err:#x} changing effect"

    def dry_ambi_map(self):
        """DeviceBase::Dry.AmbiMap: (scale [n] f32, index [n] u32)."""
        self.hz.refh_dry_ambi_map.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        sc = np.zeros(64, dtype=np.float32)
        ix = np.zeros(64, dtype=np.uint32)
        n = self.hz.refh_dry_ambi_map(self.dev, sc.ctypes.data, ix.ctypes.data)
        return sc[:n].copy(), ix[:n].copy()

    def slot_ambi_map(self, idx: int):
        """The idx-th active slot's Wet.AmbiMap: (scale, index)."""
        self.hz.refh_slot_ambi_map.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        sc = np.zeros(64, dtype=np.float32)
        ix = np.zeros(64, dtype=np.uint32)
        n = self.hz.refh_slot_ambi_map(self.ctx, idx, sc.ctypes.data, ix.ctypes.data)
        assert n > 0, n
        return sc[:n].copy(), ix[:n].copy()

    def device_ambi_order(self) -> int:
        self.hz.refh_device_ambi.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32),
                                             C.POINTER(C.c_float)]
        o, d2, xo = C.c_uint32(), C.c_uint32(), C.c_float()
        self.hz.refh_device_ambi(self.dev, C.byref(o), C.byref(d2), C.byref(xo))
        return int(o.value)

    def change_reverb(self, slot: int, props: dict):
        """Changes properties of the slot's reverb effect and re-applies it (ReverbState::update)."""
        e = self._slot_effect[slot]
        for k, v in props.items():
            self.al.alEffectf(e, k, float(v))
        self.al.alAuxiliaryEffectSloti(slot, AL_EFFECTSLOT_EFFECT, e)
        err = self.al.alGetError()
        assert err == 0, f"AL error {err:#x} changing reverb"

    def reverb_params(self, idx: int):
        if not hasattr(self, "_rv"):
            self._rv = C.CDLL(os.path.join(REF_DIR, "libref_reverb_tap.so"))
            self._rv.refh_reverb_params.argtypes = [C.c_void_p, C.c_int, C.POINTER(abi.ReverbParams),
                                                    C.c_void_p, C.POINTER(C.c_int)]
        p = abi.ReverbParams()
        gains = np.zeros((8, self.desc.dry_channels), dtype=np.float32)
        st = C.c_int(0)
        rc = self._rv.refh_reverb_params(self.ctx, idx, C.byref(p), gains.ctypes.data, C.byref(st))
        assert rc == 0, f"refh_reverb_params -> {rc}"
        return p, gains, st.value

    def make_filter(self, gain: float, gain_hf: float, gain_lf: float | None = None) -> int:
        """A low-pass (gain, gainHF) or, with gain_lf, band-pass EFX filter object."""
        f = C.c_uint(0)
        self.al.alGenFilters(1, C.byref(f))
        if gain_lf is None:
            self.al.alFilteri(f, AL_FILTER_TYPE, AL_FILTER_LOWPASS)
            self.al.alFilterf(f, AL_LOWPASS_GAIN, gain)
            self.al.alFilterf(f, AL_LOWPASS_GAINHF, gain_hf)
        else:
            self.al.alFilteri(f, AL_FILTER_TYPE, AL_FILTER_BANDPASS)
            self.al.alFilterf(f, AL_BANDPASS_GAIN, gain)
            self.al.alFilterf(f, AL_BANDPASS_GAINHF, gain_hf)
            self.al.alFilterf(f, AL_BANDPASS_GAINLF, gain_lf)
        err = self.al.alGetError()
        assert err == 0, f"AL error {err:#x} creating filter"
        return f.value

    def set_direct_filter(self, source: int, filt: int):
        self.al.alSourcei(source, AL_DIRECT_FILTER, filt)
        err = self.al.alGetError()
        assert err == 0, f"AL error {err:#x} setting direct filter"

    def voice_filters(self, nv: int):
        """[(voice, path, active, lowpass[5], highpass[5])] for voices < nv and every path
        (0 = direct, 1+s = send s < num_sends), plus the mCounter pairs."""
        out, counters = [], []
        ns = self.desc.num_sends
        for v in range(nv):
            co = np.zeros((7, 2, 5), dtype=np.float32)
            act = (C.c_int * 7)()
            cnt = (C.c_int * 14)()
            rc = self.hz.refh_voice_filters(self.ctx, v, co.ctypes.data, act, cnt)
            assert rc == 0
            for p in range(1 + ns):
                out.append((v, p, act[p], co[p, 0].copy(), co[p, 1].copy()))
                counters.append((cnt[2 * p], cnt[2 * p + 1]))
        return out, counters

    def try_reverb(self, idx: int) -> bool:
        """True if active slot idx holds a reverb."""
        if not hasattr(self, "_rv"):
            self.reverb_params.__func__  # noqa: B018  (make sure the attribute exists)
            self._rv = C.CDLL(os.path.join(REF_DIR, "libref_reverb_tap.so"))
            self._rv.refh_reverb_params.argtypes = [C.c_void_p, C.c_int, C.POINTER(abi.ReverbParams),
                                                    C.c_void_p, C.POINTER(C.c_int)]
        p = abi.ReverbParams()
        gains = np.zeros((8, abi.MAX_WET), dtype=np.float32)
        st = C.c_int(0)
        return self._rv.refh_reverb_params(self.ctx, idx, C.byref(p), gains.ctypes.data, C.byref(st)) == 0

    def connect_send(self, source: int, slot: int, send: int = 0, filt: int = AL_FILTER_NULL):
        self.al.alSource3i(source, AL_AUXILIARY_SEND_FILTER, slot, send, filt)
        err = self.al.alGetError()
        assert err == 0, f"AL error {err:#x} connecting send"

    def dither_depth(self) -> float:
        return float(self.hz.refh_dither_depth(self.dev))

    def front_stabilizer(self):
        """(FrontCenter index, splitter coefficient) of StablizerPostProcess, or None."""
        co = C.c_float(0.0)
        idx = self.hz.refh_front_stabilizer(self.dev, C.byref(co))
        return (idx, co.value) if idx >= 0 else None

    def distance_comp(self):
        """(delays uint32[real], gains float32[real]) of DeviceBase::ChannelDelays, or None."""
        dl = np.zeros(64, dtype=np.uint32)
        g = np.zeros(64, dtype=np.float32)
        n = self.hz.refh_distance_comp(self.dev, dl.ctypes.data, g.ctypes.data)
        return (dl[:n].copy(), g[:n].copy()) if n else None

    def limiter_desc(self):
        """(abi.LimiterDesc, look-ahead) of the device's limiter, or None when it has none."""
        from pyb200mix import abi
        d = abi.LimiterDesc()
        rc = self.hz.refh_limiter_desc(self.dev, C.byref(d))
        return (d, rc - 1) if rc else None

    def set_slot_target(self, slot: int, target: int):
        self.al.alAuxiliaryEffectSloti(slot, 0x199C, target)      # AL_EFFECTSLOT_TARGET_SOFT
        err = self.al.alGetError()
        assert err == 0, f"AL error {err:#x} setting slot target"

    def mono_line_gains_slot(self, target_idx: int, slot_gain: float) -> np.ndarray:
        out = np.zeros(abi.MAX_WET, dtype=np.float32)
        n = self.hz.refh_mono_line_gains_slot(self.ctx, target_idx, slot_gain, out.ctypes.data)
        assert n > 0, n
        return out[:n].copy()

    def slot_info(self):
        n = self.hz.refh_slot_count(self.ctx)
        return n, [self.hz.refh_slot_wet_channels(self.ctx, i) for i in range(n)]

    def mono_line_gains(self, slot_gain: float) -> np.ndarray:
        out = np.zeros(self.desc.dry_channels, dtype=np.float32)
        self.hz.refh_mono_line_gains(self.dev, slot_gain, out.ctypes.data)
        return out

    def play_all(self):
        arr = (C.c_uint * len(self.sources))(*self.sources)
        self.al.alSourcePlayv(len(self.sources), arr)

    def render(self, frames: int = 1024, channels: int | None = None, dtype=np.float32) -> np.ndarray:
        """Returns planar [channels][frames] (de-interleaved) of the device's sample type."""
        ch = channels or self.out_channels
        buf = np.zeros((frames, ch), dtype=dtype)
        self.al.alcRenderSamplesSOFT(self.dev, buf.ctypes.data, frames)
        return np.ascontiguousarray(buf.T)

    # ---- taps ----
    def snapshot(self, wet_channels: int = 0, channel: int = 0):
        """channel: which mixing channel (Voice::mChans[channel]) of every voice to read."""
        self.hz.refh_set_snapshot_channel(channel)
        n = self.hz.refh_voice_count(self.ctx)
        d = self.desc
        params = (abi.VoiceParams * max(n, 1))()
        state = (VoiceState * max(n, 1))()
        coeffs = np.zeros((max(n, 1), max(d.ir_size, 1), 2), dtype=np.float32)
        dry = np.zeros((max(n, 1), d.dry_channels), dtype=np.float32)
        send = np.zeros((max(n, 1), max(d.num_sends, 1), max(wet_channels, 1)), dtype=np.float32)
        got = self.hz.refh_snapshot_voices(self.ctx, params, coeffs.ctypes.data, dry.ctypes.data,
                                           send.ctypes.data if wet_channels else None,
                                           wet_channels, state)
        assert got == n
        return n, params, coeffs[:n], dry[:n], send[:n], state

    def hrtf_accum(self) -> np.ndarray:
        out = np.zeros((abi.LINE + abi.HRIR_LENGTH, 2), dtype=np.float32)
        self.hz.refh_get_hrtf_accum(self.dev, out.ctypes.data)
        return out

    def dry(self) -> np.ndarray:
        out = np.zeros((self.desc.dry_channels, abi.LINE), dtype=np.float32)
        self.hz.refh_get_dry(self.dev, out.ctypes.data)
        return out

    def hrtf_decoder(self):
        ir = C.c_uint32(0)
        n = self.hz.refh_hrtf_decoder(self.dev, C.byref(ir), None, None, None)
        assert n == self.desc.dry_channels, (n, self.desc.dry_channels)
        coeffs = np.zeros((n, ir.value, 2), dtype=np.float32)
        hf = np.zeros(n, dtype=np.float32)
        sc = np.zeros(n, dtype=np.float32)
        self.hz.refh_hrtf_decoder(self.dev, C.byref(ir), coeffs.ctypes.data, hf.ctypes.data,
                                  sc.ctypes.data)
        return coeffs, hf, sc

    def ambi_decoder(self):
        d = self.desc
        hfm = np.zeros((d.dry_channels, d.real_channels), dtype=np.float32)
        lfm = np.zeros((d.dry_channels, d.real_channels), dtype=np.float32)
        xo = C.c_float(0)
        dual = C.c_int(0)
        got = self.hz.refh_ambi_decoder(self.dev, hfm.ctypes.data, lfm.ctypes.data,
                                        C.byref(xo), C.byref(dual))
        assert got == d.dry_channels, (got, d.dry_channels)
        return hfm, (lfm if dual.value else None), xo.value
