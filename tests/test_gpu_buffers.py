"""-m gpu: a refused buffer or callback-voice call changes nothing.

Each case makes one call that the device refuses with B200MIX_ERR_INVALID:
- a short buffer_data on a registered callback buffer that no voice plays;
- buffer_data, buffer_free and buffer_callback on a static buffer that an active voice plays;
- a buffer_callback whose block size does not match its format, on a buffer that has data;
- a voices_update whose first entry moves a static voice from buffer A to B, and whose second entry gives
  channel 0 of a two-channel callback source a step that its channel 1 does not get.
Over the next four updates the device renders RealOut bit for bit as a twin that never saw the call,
makes the same callback requests, reports the same callback-buffer states and holds the same buffers."""
import ctypes as C

import numpy as np
import pytest

from helpers import mixlib, synth
from helpers.mixlib import MixDevice
from pyb200mix import abi, scene
from test_gpu_callback import Stream, _bind

pytestmark = pytest.mark.gpu

ERR_INVALID = -1                       # B200MIX_ERR_INVALID
# static A (voice 0 plays it), static B, a two-channel stream (voices 1 and 2), a mono stream no voice plays
BUF_A, BUF_B, BUF_CB, BUF_IDLE = 0, 1, 2, 3
STATIC = abi.VF_PLAYING | abi.VF_STATIC | abi.VF_LOOPING
STEP = 0x11000


def _voice(voice, buffer, flags, step=STEP):
    p = abi.VoiceParams()
    p.voice, p.buffer, p.resampler, p.flags, p.step = voice, buffer, abi.RS_SPLINE, flags, step
    p.loop_start, p.loop_end = 0, scene.BUFFER_FRAMES
    for s in range(abi.MAX_SENDS):
        p.send_slot[s] = abi.NO_SLOT
    return p


def _gains(n):
    return (np.random.default_rng(43).standard_normal((n, 3)) * 0.3).astype(np.float32)


def _stream(k, channels):
    return Stream(np.random.default_rng(60 + k), k, abi.FMT_I16, channels, 1, 20000)


def _device(L):
    desc = synth.stereo_desc(4)
    desc.max_buffers = 4
    dev = MixDevice(mixlib.product(), desc)
    dev.set_ambi_decoder((np.random.default_rng(8).standard_normal((3, 2)) * 0.5).astype(np.float32), None, 0.0)
    for b in (BUF_A, BUF_B):
        dev.buffer_data(b, abi.FMT_I16, scene.voice_buffer_fast(b))
    streams = [_stream(0, 2), _stream(1, 1)]
    for b, s in zip((BUF_CB, BUF_IDLE), streams):
        assert L.b200mix_buffer_callback(dev.h, b, C.byref(s.desc())) == 0
    dev.voices_update([_voice(0, BUF_A, STATIC | abi.VF_RESET)]
                      + [_voice(1 + c, BUF_CB, abi.VF_PLAYING | abi.VF_RESET | abi.vf_channel(c)) for c in (0, 1)],
                      None, _gains(3), None)
    return dev, streams


def _refused_call(L, dev, case):
    pcm = scene.voice_buffer_fast(5)
    if case == "short_data_on_callback_buffer":
        return L.b200mix_buffer_data(dev.h, BUF_IDLE, abi.FMT_I16, 1, len(pcm), pcm.ctypes.data, pcm.nbytes - 2)
    if case == "data_on_played_buffer":
        return L.b200mix_buffer_data(dev.h, BUF_A, abi.FMT_I16, 1, len(pcm), pcm.ctypes.data, pcm.nbytes)
    if case == "free_played_buffer":
        return L.b200mix_buffer_free(dev.h, BUF_A)
    if case == "callback_block_size":
        d = _stream(2, 1).desc()
        d.bytes_per_block += 1
        return L.b200mix_buffer_callback(dev.h, BUF_B, C.byref(d))
    if case == "callback_on_played_buffer":
        return L.b200mix_buffer_callback(dev.h, BUF_A, C.byref(_stream(2, 1).desc()))
    assert case == "callback_voices_disagree"
    vp = (abi.VoiceParams * 2)(_voice(0, BUF_B, STATIC | abi.VF_RESET),
                               _voice(1, BUF_CB, abi.VF_PLAYING | abi.vf_channel(0), STEP + 0x800))
    return dev.m.voices_update(dev.h, 2, vp, None, _gains(2).ctypes.data, None)


def _state(L, dev, buffer):
    got = [C.c_uint32() for _ in range(3)]
    rc = L.b200mix_buffer_callback_state(dev.h, buffer, *[C.byref(g) for g in got])
    return rc, [g.value for g in got]


@pytest.mark.parametrize("case", ["short_data_on_callback_buffer", "data_on_played_buffer", "free_played_buffer",
                                  "callback_block_size", "callback_on_played_buffer", "callback_voices_disagree"])
def test_rejected_buffer_call_changes_nothing(case):
    L = mixlib.product().lib
    _bind(L)
    L.b200mix_buffer_free.argtypes = [C.c_void_p, C.c_uint32]
    devs = []
    try:
        devs += [_device(L) for _ in range(2)]
        for dev, _ in devs:
            dev.render()
        assert _refused_call(L, devs[0][0], case) == ERR_INVALID
        seen = []
        for dev, streams in devs:
            updates = []
            for _ in range(4):
                updates.append((dev.render(), [_state(L, dev, b) for b in (BUF_CB, BUF_IDLE)]))
            seen.append((updates, [s.log for s in streams]))
        (ours, our_logs), (twin, twin_logs) = seen
        assert np.abs(twin[-1][0]).max() > 1e-4 and twin_logs[0]
        for u, ((out, states), (tout, tstates)) in enumerate(zip(ours, twin)):
            assert out.tobytes() == tout.tobytes(), u
            assert states == tstates, u
        assert our_logs == twin_logs
        holds = [[L.b200mix_buffer_free(dev.h, b) for b in (BUF_A, BUF_B, BUF_CB)] for dev, _ in devs]
        assert holds[0] == holds[1] == [ERR_INVALID, 0, ERR_INVALID]
    finally:
        for dev, _ in devs:
            dev.close()
