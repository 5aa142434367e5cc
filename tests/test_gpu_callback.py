"""-m gpu: callback-buffer sources (b200mix_buffer_callback, AL_SOFT_callback_buffer) on the GPU.

A callback stream renders exactly as a static voice on the whole blocks its callback delivers: the
reference reads storage[cb_offset..] where cb_offset - position never changes within an update, and
holds the last stored sample only once the callback has returned short, after which nothing more is
stored (tests/test_callback_plan.py checks this on random voices).  So the library, playing the
streams through callbacks, is compared with the CPU oracle playing those blocks as static buffers:
audio within test_gpu_parity's bounds, positions and flags identical.  The callbacks' requests, the
buffer state and the bytes left in each storage are compared every update with the restatement of
the reference in tests/test_callback_plan.py (whose planner tests/test_callback_ref.py holds to the
live reference's own callback requests)."""
import ctypes as C

import numpy as np
import pytest

from helpers import mixlib, synth
from helpers.mixlib import MixDevice
from pyb200mix import abi, scene
from test_callback_plan import reference_update

pytestmark = pytest.mark.gpu

RMS_TOL, MAX_TOL = 1e-6, 1e-5          # test_gpu_parity.py's bounds against the oracle
SIZES = {abi.FMT_U8: 1, abi.FMT_I16: 2, abi.FMT_I32: 4, abi.FMT_F32: 4, abi.FMT_F64: 8, abi.FMT_MULAW: 1,
         abi.FMT_ALAW: 1}
# (sample type, channels, samples per block)
FORMATS = [(abi.FMT_I16, 1, 1), (abi.FMT_F32, 2, 1), (abi.FMT_U8, 1, 1), (abi.FMT_MULAW, 1, 1),
           (abi.FMT_IMA4, 1, 65), (abi.FMT_MSADPCM, 2, 64), (abi.FMT_I16, 2, 1), (abi.FMT_ALAW, 1, 1)]
PITCHES = [0.7, 1.0, 1.7, 3.3, 10.0, 1.0, 0.45, 2.2]


def _block_bytes(fmt, ch, spb):
    if fmt == abi.FMT_IMA4:
        return ((spb - 1) // 2 + 4) * ch
    if fmt == abi.FMT_MSADPCM:
        return ((spb - 2) // 2 + 7) * ch
    return SIZES[fmt] * ch


def _stream_bytes(rng, fmt, ch, nbytes):
    """A seeded signal of nbytes bytes in the format (ADPCM: random blocks, which decode to a valid
    bounded signal)."""
    if fmt in (abi.FMT_IMA4, abi.FMT_MSADPCM, abi.FMT_U8, abi.FMT_MULAW, abi.FMT_ALAW):
        return rng.integers(0, 256, nbytes, dtype=np.uint8)
    n = nbytes // SIZES[fmt]
    x = 0.5 * np.sin(np.arange(n) * float(rng.uniform(0.01, 0.2))) + 0.1 * rng.standard_normal(n)
    if fmt == abi.FMT_I16:
        return (np.clip(x, -1, 1) * 32000).astype(np.int16).view(np.uint8)
    return x.astype(np.float32).view(np.uint8)


class Stream:
    """One callback source: its stream bytes, the ctypes callback with its log, its storage."""

    def __init__(self, rng, k, fmt, ch, spb, total_blocks):
        self.fmt, self.ch, self.spb = fmt, ch, spb
        self.bpb = _block_bytes(fmt, ch, spb)
        self.data = _stream_bytes(rng, fmt, ch, total_blocks * self.bpb + int(rng.integers(0, self.bpb)))
        # PrepareCallback's storage (al/buffer.cpp:468-473)
        self.storage = (C.c_uint8 * ((((1024 + 256) * 10 + 24 + spb - 1) // spb) * self.bpb))()
        self.fed, self.log = 0, []

        def cb(user, dst, numbytes):
            got = min(numbytes, len(self.data) - self.fed)
            C.memmove(dst, self.data[self.fed:self.fed + got].ctypes.data, got)
            self.fed += got
            self.log.append((int(dst) - C.addressof(self.storage), numbytes, got))
            return got
        self.fn = abi.CALLBACK_FN(cb)
        # the reference restatement's view of the same stream
        self.model = {"num_blocks": 0, "block_offset": 0, "stopped": 0}
        self.mfed, self.counted, self.mvoice = 0, 0, None

    def model_answer(self, offset, need):
        got = min(need, len(self.data) - self.mfed)
        self.mfed += got
        return got

    def desc(self):
        d = abi.CallbackBuffer()
        d.struct_size = C.sizeof(abi.CallbackBuffer)
        d.sample_type, d.channels = self.fmt, self.ch
        d.samples_per_block, d.bytes_per_block = self.spb, self.bpb
        d.callback, d.userptr = self.fn, None
        d.storage, d.storage_bytes = C.addressof(self.storage), C.sizeof(self.storage)
        return d


def _bind(lib):
    lib.b200mix_buffer_callback.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(abi.CallbackBuffer)]
    lib.b200mix_buffer_callback_state.argtypes = [C.c_void_p, C.c_uint32] + [C.POINTER(C.c_uint32)] * 3
    lib.b200mix_launch_count.argtypes = [C.c_void_p]
    lib.b200mix_launch_count.restype = C.c_uint64


def _run(hrtf, n_sources, n_static, updates, seed, static_lib=None):
    """static_lib: the implementation that plays the streams as static buffers (the oracle)."""
    rng = np.random.default_rng(seed)
    ir = 64
    nv_max = 2 * n_sources + n_static
    desc = synth.hrtf_desc(nv_max, ir) if hrtf else synth.stereo_desc(nv_max)
    desc.max_buffers = 2 * nv_max
    streams, voices = [], []           # voices: (voice index, source k, channel)
    for k in range(n_sources):
        fmt, ch, spb = FORMATS[k % len(FORMATS)]
        pitch = PITCHES[k % len(PITCHES)]
        # every fifth stream runs out mid-scene (short return -> the voice ends), the rest outlast it
        need = int(updates * 1024 * pitch / spb) + 40
        total = int(need * rng.uniform(0.2, 0.8)) if k % 5 == 2 else need + 64
        streams.append(Stream(rng, k, fmt, ch, spb, max(total, 1)))
        for c in range(ch):
            voices.append((len(voices), k, c))
    n_cb_voices = len(voices)
    params, coeffs, dry = synth.voice_set(rng, n_cb_voices + n_static, ir, hrtf=hrtf,
                                          dry_channels=desc.dry_channels, looping=True,
                                          resampler=list(range(10)))
    start_frac = [0 if k % 3 else int(rng.integers(0, 65536)) for k in range(n_sources)]
    for v, k, c in voices:
        p = params[v]
        p.position, p.position_frac = 0, start_frac[k]    # the channels of a source move together
        p.step = min(int(PITCHES[k % len(PITCHES)] * 65536), 10 << 16)
        p.flags = abi.VF_PLAYING | abi.VF_RESET | abi.vf_channel(c) | (abi.VF_HRTF if hrtf else 0)
    for p, v in zip(params, range(len(params))):
        if v >= n_cb_voices:
            p.buffer = 2 * nv_max - 1 - (v - n_cb_voices)
    frame_seq = [1024, 7, 333, 1, 1024, 555, 1024, 64, 1024, 1000, 17, 1024][:updates]

    out = {}
    for which in ("oracle", "product"):
        lib = (static_lib or mixlib.oracle()) if which == "oracle" else mixlib.product()
        dev = MixDevice(lib, desc)
        if hrtf:
            dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7), desc.dry_channels))
        else:
            g = np.random.default_rng(8).standard_normal((desc.dry_channels, desc.real_channels))
            dev.set_ambi_decoder(g.astype(np.float32), None, 0.0)
        for v in range(n_cb_voices, n_cb_voices + n_static):
            dev.buffer_data(params[v].buffer, abi.FMT_I16, scene.voice_buffer_fast(v))
        vp = [abi.VoiceParams.from_buffer_copy(bytes(p)) for p in params]
        for v, k, c in voices:
            s = streams[k]
            if which == "oracle":
                blocks = len(s.data) // s.bpb
                raw = s.data[:blocks * s.bpb]
                if s.fmt in (abi.FMT_IMA4, abi.FMT_MSADPCM):
                    if c == 0:
                        dev.buffer_data_adpcm(k, s.fmt, s.spb, blocks, raw, channels=s.ch)
                elif c == 0:
                    dev.buffer_data(k, s.fmt, raw.view({1: np.uint8, 2: np.int16, 4: np.float32,
                                                        8: np.float64}[SIZES[s.fmt]]).reshape(-1, s.ch),
                                    channels=s.ch)
                vp[v].flags |= abi.VF_STATIC
                vp[v].flags &= ~abi.VF_LOOPING
            else:
                if c == 0:
                    _bind(lib.lib)
                    assert lib.lib.b200mix_buffer_callback(dev.h, k, C.byref(s.desc())) == 0
                vp[v].flags &= ~abi.VF_LOOPING
            vp[v].buffer = k
        dev.voices_update(vp, coeffs if hrtf else None, dry, None)
        audio, results, launches = [], [], []
        for u, frames in enumerate(frame_seq):
            if u == 7:
                # replay source 2 from the top (RESET of a running or ended stream, the application
                # rewinding its stream), and re-register source 3 with the state read back (resume)
                # a restarted voice comes with its targets (a RESET voice is a fresh one)
                idx = [v for v, k, c in voices if k == 2]
                dev.voices_update([vp[v] for v in idx], coeffs[idx] if hrtf else None, dry[idx], None)
                s2 = streams[2]
                s2.fed = 0
                if which == "product":
                    s2.mfed, s2.counted = 0, 0
                    s2.model = {"num_blocks": 0, "block_offset": 0, "stopped": 0}
                    s2.mvoice = {"pos": 0, "frac": start_frac[2], "step": params[voices[[k for _, k, _ in voices].index(2)][0]].step,
                                 "state": 1, "have": True}
                    got = [C.c_uint32() for _ in range(3)]
                    assert lib.lib.b200mix_buffer_callback_state(dev.h, 3, *[C.byref(g) for g in got]) == 0
                    d3 = streams[3].desc()
                    d3.num_blocks, d3.block_offset, d3.stopped = (g.value for g in got)
                    assert lib.lib.b200mix_buffer_callback(dev.h, 3, C.byref(d3)) == 0
            if u == 5:
                # stop one source: a Stopping fade, then stopped
                upd = []
                for v, k, c in voices:
                    if k == 1:
                        q = abi.VoiceParams.from_buffer_copy(bytes(vp[v]))
                        q.flags = (q.flags & ~(abi.VF_PLAYING | abi.VF_RESET)) | abi.VF_STOPPING
                        upd.append(q)
                if upd:
                    dev.voices_update(upd, None, None, None)
            if which == "product":
                before = lib.lib.b200mix_launch_count(dev.h)
                logs_before = [len(s.log) for s in streams]
            o, res = dev.render(frames, want_results=True)
            audio.append(o)
            results.append([(res[v].position, res[v].position_frac, res[v].flags) for v in range(nv_max)])
            if which == "product":
                launches.append(lib.lib.b200mix_launch_count(dev.h) - before)
                # the callbacks, the state and the storage against the reference restatement
                rep = {}
                for v, k, c in voices:
                    rep.setdefault(k, v)
                for k, s in enumerate(streams):
                    v = rep[k]
                    mv = s.mvoice
                    if mv is None:
                        mv = s.mvoice = {"pos": params[v].position, "frac": params[v].position_frac,
                                         "step": params[v].step, "state": 1, "have": True}
                    if u == 5 and k == 1 and mv["state"] == 1:
                        mv["state"] = 2
                    requests, _ = reference_update(s.model, mv, s.spb, s.bpb, frames, s.model_answer)
                    assert s.log[logs_before[k]:] == requests, (k, u)
                    # whole blocks delivered so far: the storage holds the last num_blocks of them
                    s.counted += sum(got // s.bpb for _, need, got in requests if got <= need)
                    got = [C.c_uint32() for _ in range(3)]
                    assert lib.lib.b200mix_buffer_callback_state(dev.h, k, *[C.byref(g) for g in got]) == 0
                    assert [g.value for g in got] == [s.model["num_blocks"], s.model["block_offset"],
                                                      s.model["stopped"]], (k, u)
                    if mv["have"]:
                        kept = s.model["num_blocks"] * s.bpb
                        start = (s.counted - s.model["num_blocks"]) * s.bpb
                        assert bytes(s.storage)[:kept] == s.data[start:start + kept].tobytes(), (k, u)
        dev.close()
        out[which] = (audio, results, launches)
    return out, n_cb_voices, streams


def _compare(out, rms_tol=RMS_TOL, max_tol=MAX_TOL):
    (ao, ro, _), (ap, rp, _) = out["oracle"], out["product"]
    for u, (o, p) in enumerate(zip(ao, ap)):
        err = p.astype(np.float64) - o.astype(np.float64)
        rms, mx = float(np.sqrt((err ** 2).mean())), float(np.abs(err).max())
        assert rms <= rms_tol and mx <= max_tol, f"update {u}: rms {rms:.3e} max {mx:.3e}"
        assert ro[u] == rp[u], f"update {u}: voice results differ"
    assert max(np.abs(o).max() for o in ao) > 1e-3, "silent scene"


@pytest.mark.parametrize("hrtf", [True, False], ids=["hrtf", "dry"])
def test_callback_sources_vs_oracle(hrtf):
    out, ncb, streams = _run(hrtf, n_sources=24, n_static=12, updates=12, seed=77 + hrtf)
    _compare(out)
    # streams that ran out ended (Stopping, then stopped) like a static voice at its end
    assert any(s.model["stopped"] for s in streams)


def test_many_callback_voices_equal_static_voices():
    """550 callback voices over every format and resampler, pitches up to 10, ragged updates and
    streams that end, beside 64 static voices: the same scene with the streams as static buffers on
    the same library mixes the same samples in the same order (test_gpu_parity pins that static path
    to the oracle at scale; against the oracle directly, ~600 full-scale noise streams differ from it
    by float summation order alone)."""
    out, ncb, streams = _run(True, n_sources=400, n_static=64, updates=6, seed=5, static_lib=mixlib.product())
    assert ncb >= 500
    _compare(out, rms_tol=1e-7, max_tol=1e-7)
    assert any(s.model["stopped"] for s in streams)


def test_sources_update_refuses_callback_buffers():
    """The GPU parameter stage computes steps the host planner cannot see: it refuses callback voices."""
    from test_gpu_params import _lib as params_lib, _listener, _props
    L = params_lib()
    _bind(L)
    desc = synth.stereo_desc(4, dry_channels=3)
    dev = MixDevice(mixlib.product(), desc)
    dev.set_ambi_decoder((np.random.default_rng(8).standard_normal((3, 2)) * 0.5).astype(np.float32), None, 0.0)
    s = Stream(np.random.default_rng(1), 0, abi.FMT_I16, 1, 1, 100)
    assert L.b200mix_buffer_callback(dev.h, 0, C.byref(s.desc())) == 0
    dscale, dindex = np.ones(3, dtype=np.float32), np.arange(3, dtype=np.uint32)
    env = abi.VoiceEnv()
    env.struct_size = C.sizeof(env)
    env.device_rate, env.num_sends, env.render_mode, env.wet_stride = 48000, 0, 0, 0
    env.dry = abi.MixMap(3, dscale.ctypes.data, dindex.ctypes.data)
    sv = (abi.SourceVoice * 1)()
    sv[0].voice, sv[0].buffer, sv[0].buffer_rate = 0, 0, 48000
    sv[0].flags = abi.VF_PLAYING | abi.VF_RESET
    for k in range(abi.MAX_SENDS):
        sv[0].send_slot[k] = abi.NO_SLOT
    props = _props(np.random.default_rng(2), 1, 0, True)
    lis = _listener(L, np.random.default_rng(3))
    assert L.b200mix_sources_update(dev.h, 1, sv, props, C.byref(lis), C.byref(env)) == -4   # UNSUPPORTED
    dev.render(256)                                    # nothing was bound: the device still mixes
    dev.close()


def test_callback_scene_launches_no_extra_kernels():
    """A callback voice costs a host plan and one copy per update, no kernel launch of its own."""
    out, _, _ = _run(True, n_sources=8, n_static=8, updates=4, seed=3)
    launches = out["product"][2]
    desc = synth.hrtf_desc(32, 64)
    rng = np.random.default_rng(3)
    params, coeffs, dry = synth.voice_set(rng, 24, 64)
    lib = mixlib.product()
    _bind(lib.lib)
    dev = MixDevice(lib, desc)
    dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7), desc.dry_channels))
    for i in range(24):
        dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
    dev.voices_update(params, coeffs, dry, None)

    def count():
        out = []
        for frames in (1024, 7, 333, 1):
            before = lib.lib.b200mix_launch_count(dev.h)
            dev.render(frames)
            out.append(lib.lib.b200mix_launch_count(dev.h) - before)
        return out
    static = count()
    assert launches == static
    # a callback buffer that no voice plays changes nothing, nor does its removal
    s = Stream(np.random.default_rng(4), 0, abi.FMT_I16, 1, 1, 100)
    assert lib.lib.b200mix_buffer_callback(dev.h, 31, C.byref(s.desc())) == 0
    assert count() == static
    lib.lib.b200mix_buffer_free.argtypes = [C.c_void_p, C.c_uint32]
    assert lib.lib.b200mix_buffer_free(dev.h, 31) == 0
    assert count() == static and not s.log
    dev.close()
