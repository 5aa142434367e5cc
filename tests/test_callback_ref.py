"""The library's callback-buffer planner (openal-soft_b200/csrc/callback_plan.hpp, built for the host)
against the UNMODIFIED reference (oracle/_ref/libopenal_ref.so) playing the same callback buffers
through its public API (alBufferCallbackSOFT, alcRenderSamplesSOFT on a loopback device): every
callback request the reference makes, and with the same answers the same requests from the planner,
update by update, over ragged update sizes, pitches up to MaxPitch, PCM and IMA4 blocks, and
streams that run out (the source then stops).  No GPU involved."""
import ctypes as C

import numpy as np
import pytest

from helpers import refal
from test_callback_plan import REQUEST_FN, Update, _lib

pytestmark = pytest.mark.skipif(not refal.available(), reason="compiled reference not built")

AL_FORMAT_MONO16, AL_FORMAT_STEREO_FLOAT32, AL_FORMAT_MONO_IMA4 = 0x1101, 0x10011, 0x1300
AL_STOPPED = 0x1014
CB_TYPE = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int)
# (AL format, samples per block, bytes per block)
FORMATS = {"mono16": (AL_FORMAT_MONO16, 1, 2), "stereo_f32": (AL_FORMAT_STEREO_FLOAT32, 1, 8),
           "ima4": (AL_FORMAT_MONO_IMA4, 65, 36)}


@pytest.mark.parametrize("fmt", list(FORMATS))
@pytest.mark.parametrize("pitch", [1.0, 0.75, 1.5, 3.0, 10.0])
def test_planner_requests_equal_the_reference(fmt, pitch):
    al_fmt, spb, bpb = FORMATS[fmt]
    dev = refal.RefDevice({})
    al = dev.al
    al.alBufferCallbackSOFT.argtypes = [C.c_uint, C.c_int, C.c_int, CB_TYPE, C.c_void_p]
    rng = np.random.default_rng(int(pitch * 100) + len(fmt))
    frame_seq = [1024, 7, 333, 1, 1024, 555, 64, 1024, 1000, 17, 1024, 1024, 512, 1024]
    # streams: one that outlasts the scene, one that runs out part way
    total_need = int(sum(frame_seq) * pitch / spb) + 64
    streams = [total_need * bpb + 5, int(total_need * 0.4) * bpb + int(rng.integers(0, bpb))]
    logs, fed, cbs, sources = [], [], [], []
    for k, nbytes in enumerate(streams):
        data = rng.integers(0, 256, nbytes, dtype=np.uint8)
        log, cur = [], [0]

        def cb(user, dst, numbytes, data=data, log=log, cur=cur):
            got = min(numbytes, len(data) - cur[0])
            C.memmove(dst, data[cur[0]:cur[0] + got].ctypes.data, got)
            cur[0] += got
            log.append((int(dst), numbytes, got))
            return got
        fn = CB_TYPE(cb)
        b, s = C.c_uint(0), C.c_uint(0)
        al.alGenBuffers(1, C.byref(b))
        al.alBufferCallbackSOFT(b, al_fmt, 48000, fn, None)
        al.alGenSources(1, C.byref(s))
        al.alSourcei(s, refal.AL_BUFFER, b.value)
        al.alSourcef(s, refal.AL_PITCH, pitch)
        assert al.alGetError() == 0
        logs.append(log); fed.append(cur); cbs.append(fn); sources.append(s.value)
    arr = (C.c_uint * len(sources))(*sources)
    al.alSourcePlayv(len(sources), arr)

    lib = _lib()
    storage = (((1024 + 256) * 10 + 24 + spb - 1) // spb) * bpb
    step = min(int(np.float32(pitch) * np.float32(65536.0)), 10 << 16)
    plans = [Update(0, 0, 0, 0, 0, step, 1, 1) for _ in streams]
    pfed = [0] * len(streams)
    storage_base = [None] * len(streams)
    ended = [False] * len(streams)
    for u, frames in enumerate(frame_seq):
        marks = [len(log) for log in logs]
        dev.render(frames)
        for k, nbytes in enumerate(streams):
            got_ref = logs[k][marks[k]:]
            if got_ref and storage_base[k] is None:
                storage_base[k] = got_ref[0][0]           # the first request writes at offset 0
            ref_reqs = [(ptr - storage_base[k], need, got) for ptr, need, got in got_ref]
            mine = []

            @REQUEST_FN
            def request(offset, need, k=k, mine=mine):
                got = min(int(need), streams[k] - pfed[k])
                pfed[k] += got
                mine.append((int(offset), int(need), got))
                return got
            assert lib.cbplan_run(C.byref(plans[k]), spb, bpb, frames, storage, request) == 0
            assert mine == ref_reqs, f"{fmt} pitch {pitch} stream {k} update {u} ({frames} frames)"
            ended[k] = ended[k] or bool(plans[k].ends)
    st = C.c_int(0)
    for k, s in enumerate(sources):
        al.alGetSourcei(s, refal.AL_SOURCE_STATE, C.byref(st))
        assert (st.value == AL_STOPPED) == ended[k], (k, st.value, ended[k])
    assert ended[1] and not ended[0]
    dev.close()
