"""-m gpu: the host library's ownership of device memory, upload arenas and events.

- Teardown: devices that configure every part the library allocates (lazily or not) go through
  create / configure / render / destroy 20 times; the free device memory must come back.
- Growth: each upload arena and scratch array grows mid-stream, and the scene still matches the
  CPU oracle within test_gpu_parity's bounds (positions and flags identical).
- Rejected updates: a voices_update / voices_update_dirs / sources_update call with one bad entry
  changes neither what the device renders nor which buffers its voices hold; an output-stage setter
  refused for a bad argument or between render_begin and render_end changes nothing either.
- Device guard (two or more GPUs): the output-stage setters allocate on the mixer's GPU whichever
  GPU is current, so a mixer on the last GPU renders what the same scene renders on GPU 0."""
import ctypes as C
import os

import numpy as np
import pytest

from helpers import golden, mixlib, synth
from helpers.mixlib import MixDevice
from pyb200mix import abi, scene
from pyb200mix.abi import SourceVoice, VoiceEnv, MixMap
from test_gpu_callback import Stream, _bind, _compare, _run
from test_gpu_params import _lib as params_lib, _listener, _props

pytestmark = pytest.mark.gpu

RMS_TOL, MAX_TOL = 1e-6, 1e-5          # test_gpu_parity.py's bounds against the oracle
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MHR = os.path.join(ROOT, "openal-soft_b200", "data", "Default HRTF.mhr")


def _L():
    L = params_lib()
    _bind(L)
    L.b200mix_profile.argtypes = [C.c_void_p, C.c_int]
    L.b200mix_hrtf_free.argtypes = [C.c_void_p]
    return L


def _filters():
    lp, hp = np.zeros(5, dtype=np.float32), np.zeros(5, dtype=np.float32)
    prod = mixlib.product()
    assert prod.biquad_coeffs(0, 5000.0 / 48000.0, 0.35, 1.0, lp.ctypes.data) == 0
    assert prod.biquad_coeffs(1, 250.0 / 48000.0, 1.0, 1.0, hp.ctypes.data) == 0
    return lp, hp


def _env(keep, cd, num_sends, cw, mode):
    dscale, dindex = np.ones(cd, dtype=np.float32), np.arange(cd, dtype=np.uint32)
    wscale, windex = np.ones(max(cw, 1), dtype=np.float32), np.arange(max(cw, 1), dtype=np.uint32)
    keep += [dscale, dindex, wscale, windex]
    env = VoiceEnv()
    env.struct_size = C.sizeof(env)
    env.device_rate, env.num_sends, env.render_mode, env.wet_stride = 48000, num_sends, mode, cw
    env.dry = MixMap(cd, dscale.ctypes.data, dindex.ctypes.data)
    for s in range(num_sends):
        env.wet[s] = MixMap(cw, wscale.ctypes.data, windex.ctypes.data)
    return env


def _source_voices(first, n, buffers, num_sends, reset):
    sv = (SourceVoice * n)()
    for i in range(n):
        r = sv[i]
        r.voice, r.buffer, r.buffer_rate = first + i, i % buffers, 48000
        r.flags = abi.VF_PLAYING | abi.VF_STATIC | abi.VF_LOOPING | (abi.VF_RESET if reset else 0)
        r.resampler = (abi.RS_SPLINE, abi.RS_LINEAR, abi.RS_BSINC12)[i % 3]
        r.loop_start, r.loop_end = 0, scene.BUFFER_FRAMES
        for s in range(abi.MAX_SENDS):
            r.send_slot[s] = 0 if s < num_sends else abi.NO_SLOT
    return sv


# ---- teardown ------------------------------------------------------------------------------

def _hrtf_everything(L, hrtf):
    """A 131 072-voice HRTF device with every part that allocates: sends and filters, convolution,
    reverb, pitch and frequency shifter slots, queues, a callback buffer, an attached HRTF data set,
    the GPU parameter stage, stage profiling, limiter, distance compensation, interleaved output."""
    nv, play, nbuf = 131072, 256, 64
    desc = synth.hrtf_desc(nv, 64)
    desc.num_sends, desc.wet_channels, desc.max_slots, desc.max_buffers = 1, 4, 4, nbuf + 1
    dev = MixDevice(mixlib.product(), desc)
    keep = []
    dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
    assert L.b200mix_hrtf_attach(dev.h, hrtf) == 0
    for i in range(nbuf):
        dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
    rng = np.random.default_rng(3)
    dev.slot_convolution(0, (rng.standard_normal((4, 300)) * 0.1).astype(np.float32),
                         np.eye(4, dtype=np.float32) * 0.5)
    fx = golden.load("hrtf_bsinc24_reverb_v6")
    dev.slot_reverb(1, abi.reverb_params_from(fx["reverb_params"].tobytes()), fx["reverb_gains"])
    ones, idx = np.ones(4, dtype=np.float32), np.arange(4, dtype=np.uint32)
    dev.slot_efx(2, abi.efx_defaults(abi.EFFECT_PSHIFTER), 0.7, ones, idx, idx)
    dev.slot_efx(3, abi.efx_defaults(abi.EFFECT_FSHIFTER), 0.7, ones, idx, idx)
    params, coeffs, dry = synth.voice_set(rng, play, 64)
    send = (rng.standard_normal((play, 1, 4)) * 0.3).astype(np.float32)
    for k, p in enumerate(params):
        p.buffer = k % nbuf
        p.send_slot[0] = k % 4
    params[1].flags &= ~(abi.VF_STATIC | abi.VF_LOOPING)          # a streaming voice
    params[1].loop_start = params[1].loop_end = params[1].position = 0
    stream = Stream(np.random.default_rng(4), 0, abi.FMT_I16, 1, 1, 4000)
    keep.append(stream)
    assert L.b200mix_buffer_callback(dev.h, nbuf, C.byref(stream.desc())) == 0
    params[0].buffer = nbuf                                         # a callback voice
    params[0].flags &= ~(abi.VF_STATIC | abi.VF_LOOPING)
    params[0].position, params[0].position_frac = 0, 0
    dev.voices_update(params, coeffs, dry, send)
    dev.voice_queue(1, [2, 3], abi.NO_LOOP)
    lp, hp = _filters()
    dev.voices_filters((k, 0, 1, lp, hp) for k in range(2, play, 3))
    assert L.b200mix_profile(dev.h, 2) == 0
    dev.set_limiter(abi.device_limiter(-3.0))
    dev.set_distance_comp([3, 5], [1.0, 0.9])
    outs = [dev.render()]
    env = _env(keep, 4, 1, 4, 2)
    sv = _source_voices(play, 64, nbuf, 1, True)
    rc = L.b200mix_sources_update(dev.h, 64, sv, _props(rng, 64, 1, False), C.byref(_listener(L, rng)), C.byref(env))
    assert rc == 0, L.b200mix_last_error(dev.h)
    outs.append(dev.render_interleaved(1024, 6, 0.0, 0)[0].T)
    outs.append(dev.render(333))
    return dev, keep, outs


def _ambi_stabilizer():
    desc = synth.stereo_desc(4096, dry_channels=4)
    desc.real_channels = 3
    dev = MixDevice(mixlib.product(), desc)
    rng = np.random.default_rng(5)
    dev.set_ambi_decoder((rng.standard_normal((4, 3)) * 0.5).astype(np.float32), None, 0.0)
    dev.set_bs2b(3)
    dev.set_front_stabilizer(2, -0.9123257)
    return dev


def _uhj_fir():
    desc = synth.stereo_desc(4096, dry_channels=3)
    desc.post_process = abi.POST_UHJ
    dev = MixDevice(mixlib.product(), desc)
    dev.set_uhj_encoder(256)
    return dev


def _play_dry(dev, n=64):
    rng = np.random.default_rng(6)
    cd = dev.desc.dry_channels
    params, _, dry = synth.voice_set(rng, n, 0, hrtf=False, dry_channels=cd, resampler=abi.RS_SPLINE)
    for i in range(n):
        dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
    dev.voices_update(params, None, dry, None)
    return [dev.render(), dev.render(777), dev.render()]


def test_teardown_returns_device_memory():
    """20 cycles of create / configure / render three updates / destroy: the free device memory after
    the last cycle is no more than one device's footprint below its value after the first (a leaked
    per-voice array of the 131 072-voice device would cost >= 10 GB over the cycles; the GPU is
    shared, so this catches large leaks, not small ones)."""
    torch = pytest.importorskip("torch")
    if not os.path.exists(MHR):
        pytest.skip("HRTF data set not staged (run build())")
    L = _L()
    data = open(MHR, "rb").read()
    hrtf = C.c_void_p()
    assert L.b200mix_hrtf_load(data, len(data), C.byref(hrtf)) == 0
    free, footprint = [], 0
    try:
        for cycle in range(20):
            before = torch.cuda.mem_get_info()[0]
            dev, keep, outs = _hrtf_everything(L, hrtf)
            if cycle == 0:
                torch.cuda.synchronize()
                footprint = before - torch.cuda.mem_get_info()[0]
            assert all(np.isfinite(o).all() for o in outs) and np.abs(outs[0]).max() > 1e-4
            dev.close()
            del keep
            for make in (_ambi_stabilizer, _uhj_fir):
                dev = make()
                outs = _play_dry(dev)
                assert all(np.isfinite(o).all() for o in outs) and np.abs(outs[-1]).max() > 1e-4
                dev.close()
            torch.cuda.synchronize()
            free.append(torch.cuda.mem_get_info()[0])
    finally:
        L.b200mix_hrtf_free(hrtf)
    assert footprint > 1 << 30, footprint           # the device's per-voice arrays are counted
    assert free[-1] >= free[0] - footprint, (free[0], free[-1], footprint)


# ---- growth --------------------------------------------------------------------------------

def test_upload_arenas_and_scratch_grow_mid_stream():
    """voices_update at n = 1, 300, then above the initial 4096-voice arena; voices_filters at the same
    rising n; a slot whose send entries pass 128 (the send partial rows grow) and whose filtered
    entries grow the send filter scratch: against the oracle, update by update."""
    nv, nbuf = 5000, 64
    rng = np.random.default_rng(12)
    desc = synth.stereo_desc(nv)
    desc.num_sends, desc.wet_channels, desc.max_slots, desc.max_buffers = 1, 4, 1, nbuf
    params, _, dry = synth.voice_set(rng, nv, 0, hrtf=False, dry_channels=desc.dry_channels,
                                     resampler=[abi.RS_LINEAR, abi.RS_SPLINE, abi.RS_POINT])
    send = (rng.standard_normal((nv, 1, 4)) * 0.2 / np.sqrt(nv / 64)).astype(np.float32)
    dry *= 1.0 / np.sqrt(nv / 64)
    for k, p in enumerate(params):
        p.buffer = k % nbuf
        p.send_slot[0] = 0
    ir = (rng.standard_normal((4, 200)) * 0.1).astype(np.float32)
    lp, hp = _filters()
    steps = ((1, 1024), (300, 333), (nv, 1024), (0, 1024))
    outs = {}
    for which, lib in (("oracle", mixlib.oracle()), ("product", mixlib.product())):
        dev = MixDevice(lib, desc)
        dev.set_ambi_decoder((np.random.default_rng(8).standard_normal((desc.dry_channels, 2)) * 0.5
                              ).astype(np.float32), None, 0.0)
        for i in range(nbuf):
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
        dev.slot_convolution(0, ir, np.eye(4, desc.dry_channels, dtype=np.float32) * 0.5)
        audio, results = [], []
        for n, frames in steps:
            if n:
                dev.voices_update(params[:n], None, dry[:n], send[:n])
                dev.voices_filters([(k, 0, 1, lp, hp) for k in range(0, n, 2)]
                                   + [(k, 1, 1, lp, hp) for k in range(1, n, 3)])
            o, res = dev.render(frames, want_results=True)
            audio.append(o)
            results.append([(res[v].position, res[v].position_frac, res[v].flags) for v in range(nv)])
        dev.close()
        outs[which] = (audio, results, None)
    _compare(outs, RMS_TOL, MAX_TOL)


def test_callback_arenas_grow_mid_stream():
    """Callback buffers whose stored blocks grow from update to update (both alternating arenas grow)
    against the oracle playing the delivered blocks as static buffers."""
    out, _, _ = _run(False, n_sources=8, n_static=4, updates=12, seed=21)
    _compare(out)


def test_sources_update_arena_grows_mid_stream():
    """b200mix_sources_update at n = 1, 300, 900 (its pinned input arena and device scratch grow)
    mixes what the host parameter stage (b200mix_calc_voices + voices_update) mixes."""
    L = _L()
    nv, nbuf, cd = 900, 64, 3
    desc = synth.stereo_desc(nv, dry_channels=cd)
    desc.max_buffers = nbuf
    keep = []
    env = _env(keep, cd, 0, 0, 0)
    devs = []
    for _ in range(2):
        dev = MixDevice(mixlib.product(), desc)
        dev.set_ambi_decoder((np.random.default_rng(8).standard_normal((cd, 2)) * 0.5).astype(np.float32), None, 0.0)
        for i in range(nbuf):
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
        devs.append(dev)
    host_dev, gpu_dev = devs
    outs = [[], []]
    for u, n in enumerate((1, 300, nv)):
        lis = _listener(L, np.random.default_rng(50 + u))
        props = _props(np.random.default_rng(70 + u), n, 0, True)
        sv = _source_voices(0, n, nbuf, 0, True)         # voices new to an update start with RESET
        vp = (abi.VoiceParams * n)()
        for i in range(n):
            for f in ("voice", "buffer", "flags", "resampler", "position", "position_frac", "loop_start",
                      "loop_end"):
                setattr(vp[i], f, getattr(sv[i], f))
            for s in range(abi.MAX_SENDS):
                vp[i].send_slot[s] = abi.NO_SLOT
        rates = np.full(n, 48000, dtype=np.uint32)
        dirs = np.zeros((n, 4), dtype=np.float32)
        dry = np.zeros((n, cd), dtype=np.float32)
        send = np.zeros((n, 1), dtype=np.float32)
        filt = (abi.VoiceFilter * n)()
        assert L.b200mix_calc_voices(n, props, C.byref(lis), C.byref(env), rates.ctypes.data, vp, dirs.ctypes.data,
                                     dry.ctypes.data, send.ctypes.data, filt, 1) == 0
        host_dev.voices_update(vp, None, dry, None)
        rc = L.b200mix_sources_update(gpu_dev.h, n, sv, props, C.byref(lis), C.byref(env))
        assert rc == 0, L.b200mix_last_error(gpu_dev.h)
        for k, dev in enumerate(devs):
            outs[k].append(dev.render(1024 if u != 1 else 333))
    for dev in devs:
        dev.close()
    a, b = np.concatenate(outs[0], axis=1), np.concatenate(outs[1], axis=1)
    assert np.abs(a).max() > 1e-3
    err = a.astype(np.float64) - b
    assert np.sqrt((err ** 2).mean()) <= RMS_TOL and np.abs(err).max() <= MAX_TOL, np.abs(err).max()


# ---- rejected updates ----------------------------------------------------------------------

ERR_INVALID = -1                       # B200MIX_ERR_INVALID
BUF_A, BUF_B, BUF_C = 0, 1, 2


def _rejection_device(L, entry, hrtf):
    """Two convolution slots; voice 0 plays static buffer A into slot 0, voice 1 plays buffer C."""
    desc = synth.hrtf_desc(4, 64) if entry == "voices_update_dirs" else synth.stereo_desc(4)
    desc.num_sends, desc.wet_channels, desc.max_slots, desc.max_buffers = 1, 4, 2, 3
    cd = desc.dry_channels
    dev = MixDevice(mixlib.product(), desc)
    if entry == "voices_update_dirs":
        dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
        assert L.b200mix_hrtf_attach(dev.h, hrtf) == 0
    else:
        dev.set_ambi_decoder((np.random.default_rng(8).standard_normal((cd, 2)) * 0.5).astype(np.float32), None, 0.0)
    for b in (BUF_A, BUF_B, BUF_C):
        dev.buffer_data(b, abi.FMT_I16, scene.voice_buffer_fast(b))
    rng = np.random.default_rng(31)
    for slot in (0, 1):
        dev.slot_convolution(slot, (rng.standard_normal((4, 300)) * 0.1).astype(np.float32),
                             np.eye(4, cd, dtype=np.float32) * 0.5)
    return dev


def _apply(L, dev, entry, records, keep):
    """One update call of the entry point under test; returns its result code."""
    n, cd = len(records), dev.desc.dry_channels
    if entry == "sources_update":
        sv = (SourceVoice * n)(*records)
        env = _env(keep, cd, 1, 4, 0)
        return L.b200mix_sources_update(dev.h, n, sv, _props(np.random.default_rng(41), n, 1, True),
                                        C.byref(_listener(L, np.random.default_rng(42))), C.byref(env))
    vp = (abi.VoiceParams * n)(*records)
    send = np.full((n, 1, 4), 0.4, dtype=np.float32)
    if entry == "voices_update_dirs":
        dirs = np.tile(np.array([[0.2, 0.8, 1.5, 0.0]], dtype=np.float32), (n, 1))
        return L.b200mix_voices_update_dirs(dev.h, n, vp, dirs.ctypes.data, None, send.ctypes.data)
    dry = (np.random.default_rng(43).standard_normal((n, cd)) * 0.3).astype(np.float32)
    return dev.m.voices_update(dev.h, n, vp, None, dry.ctypes.data, send.ctypes.data)


def _record(entry, voice, buffer, slot):
    r = SourceVoice() if entry == "sources_update" else abi.VoiceParams()
    r.voice, r.buffer, r.resampler = voice, buffer, abi.RS_SPLINE
    r.flags = abi.VF_PLAYING | abi.VF_STATIC | abi.VF_LOOPING | abi.VF_RESET
    if entry == "voices_update_dirs":
        r.flags |= abi.VF_HRTF
    r.loop_start, r.loop_end = 0, scene.BUFFER_FRAMES
    for s in range(abi.MAX_SENDS):
        r.send_slot[s] = slot if s == 0 else abi.NO_SLOT
    if entry == "sources_update":
        r.buffer_rate = 48000
    else:
        r.step, r.hrtf_gain = 0x11000, 0.5
    return r


@pytest.mark.parametrize("entry,reject", [
    ("voices_update", "empty_loop"), ("voices_update", "step"), ("voices_update", "hrtf_delay"),
    ("voices_update_dirs", "empty_loop"), ("voices_update_dirs", "step"), ("sources_update", "empty_loop")])
def test_rejected_update_changes_nothing(entry, reject):
    """A call whose entry 0 moves voice 0 from buffer A / slot 0 to buffer B / slot 1 and whose entry 1
    is rejected returns B200MIX_ERR_INVALID and changes nothing: four updates render RealOut bit for
    bit as a twin that never saw the call, and buffer A is still held by its voice while B is not."""
    if entry == "voices_update_dirs" and not os.path.exists(MHR):
        pytest.skip("HRTF data set not staged (run build())")
    L = _L()
    L.b200mix_buffer_free.argtypes = [C.c_void_p, C.c_uint32]
    data = open(MHR, "rb").read() if entry == "voices_update_dirs" else None
    hrtf = C.c_void_p()
    if data:
        assert L.b200mix_hrtf_load(data, len(data), C.byref(hrtf)) == 0
    keep, outs, devs = [], [], []
    try:
        devs += [_rejection_device(L, entry, hrtf) for _ in range(2)]
        for dev in devs:
            rc = _apply(L, dev, entry, [_record(entry, 0, BUF_A, 0), _record(entry, 1, BUF_C, abi.NO_SLOT)], keep)
            assert rc == 0, L.b200mix_last_error(dev.h)
            outs.append([dev.render()])
        bad = _record(entry, 1, BUF_C, abi.NO_SLOT)
        if reject == "empty_loop":
            bad.loop_end = bad.loop_start
        elif reject == "step":
            bad.step = (10 << 16) + 1
        else:
            bad.hrtf_delay[0] = abi.HRTF_HISTORY
        moved = _record(entry, 0, BUF_B, 1)
        assert _apply(L, devs[0], entry, [moved, bad], keep) == ERR_INVALID
        for dev, out in zip(devs, outs):
            out += [dev.render() for _ in range(4)]
        assert np.abs(outs[1][-1]).max() > 1e-4
        for a, b in zip(*outs):
            assert a.tobytes() == b.tobytes()
        assert L.b200mix_buffer_free(devs[0].h, BUF_A) == ERR_INVALID
        assert L.b200mix_buffer_free(devs[0].h, BUF_B) == 0
    finally:
        for dev in devs:
            dev.close()
        if data:
            L.b200mix_hrtf_free(hrtf)


def _output_device(kind):
    """ambi: 3 RealOut channels, a dual-band decoder, the front stabilizer, a limiter and distance
    compensation; uhj: the FIR-256 encoder and a limiter; hrtf: its decoder.  64 voices play, a third of
    them through the dry mix on the HRTF device."""
    rng = np.random.default_rng(5)
    if kind == "hrtf":
        dev = MixDevice(mixlib.product(), synth.hrtf_desc(64, 64))
        dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
        params, coeffs, dry = synth.voice_set(rng, 64, 64)
        for k in range(1, 64, 3):
            params[k].flags &= ~abi.VF_HRTF
    else:
        desc = synth.stereo_desc(64, dry_channels=4 if kind == "ambi" else 3)
        if kind == "ambi":
            desc.real_channels = 3
        else:
            desc.post_process = abi.POST_UHJ
        dev = MixDevice(mixlib.product(), desc)
        if kind == "ambi":
            gains = (rng.standard_normal((2, 4, 3)) * 0.5).astype(np.float32)
            dev.set_ambi_decoder(gains[0], gains[1], -0.9123257)
            dev.set_front_stabilizer(2, -0.9123257)
            dev.set_distance_comp([3, 5, 1], [1.0, 0.9, 0.8])
        else:
            dev.set_uhj_encoder(256)
        dev.set_limiter(abi.device_limiter(-6.0))
        params, coeffs, dry = synth.voice_set(rng, 64, 0, hrtf=False, dry_channels=desc.dry_channels,
                                              resampler=abi.RS_SPLINE)
        coeffs = None
    for i in range(64):
        dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
    dev.voices_update(params, coeffs, dry, None)
    return dev


def _output_call(dev, call):
    """One output-stage call through the C ABI; returns its result code."""
    m, h = dev.m, dev.h
    rng = np.random.default_rng(11)
    lim = abi.device_limiter(-3.0)
    if call == "limiter_struct_size":
        lim.struct_size += 4
    gains = (rng.standard_normal((4, 3)) * 0.5).astype(np.float32)
    cd = 3 if call == "hrtf_decoder_channels" else 4
    dec = synth.decoder(rng, channels=cd)
    delays = np.array([3, 5, 1024 if call == "distance_comp_delay" else 1, 2], dtype=np.uint32)
    dc_gains = np.array([1.0, 0.9, 0.8, 0.7], dtype=np.float32)
    calls = {
        "distance_comp_delay": lambda: m.set_distance_comp(h, 3, delays.ctypes.data, dc_gains.ctypes.data),
        "distance_comp_channels": lambda: m.set_distance_comp(h, 4, delays.ctypes.data, dc_gains.ctypes.data),
        "limiter_struct_size": lambda: m.set_limiter(h, C.byref(lim), None),
        "bs2b_level_7": lambda: m.set_bs2b(h, 7),
        "stabilizer_on_left": lambda: m.set_front_stabilizer(h, dev.desc.real_left, -0.9),
        "uhj_length_128": lambda: m.set_uhj_encoder(h, 128, None),
        "ambi_decoder_channels": lambda: m.set_ambi_decoder(h, 3, gains[:3].ctypes.data, None, 0.0),
        "hrtf_decoder_channels": lambda: m.set_hrtf_decoder(h, cd, dec[0].shape[1], dec[0].ctypes.data,
                                                            dec[1].ctypes.data, dec[2].ctypes.data),
        # accepted outside a render
        "hrtf_decoder": lambda: m.set_hrtf_decoder(h, cd, dec[0].shape[1], dec[0].ctypes.data, dec[1].ctypes.data,
                                                   dec[2].ctypes.data),
        "ambi_decoder": lambda: m.set_ambi_decoder(h, 4, gains.ctypes.data, gains.ctypes.data, -0.8),
        "uhj_encoder": lambda: m.set_uhj_encoder(h, 512, None),
        "front_stabilizer": lambda: m.set_front_stabilizer(h, 2, -0.8),
        "bs2b": lambda: m.set_bs2b(h, 3),
        "distance_comp": lambda: m.set_distance_comp(h, 2, delays.ctypes.data, dc_gains.ctypes.data),
        "limiter": lambda: m.set_limiter(h, C.byref(lim), None),
    }
    return calls[call]()


@pytest.mark.parametrize("kind,call,mid_render", [
    ("ambi", "distance_comp_delay", False), ("ambi", "distance_comp_channels", False),
    ("ambi", "limiter_struct_size", False), ("ambi", "bs2b_level_7", False), ("ambi", "stabilizer_on_left", False),
    ("uhj", "uhj_length_128", False), ("ambi", "ambi_decoder_channels", False),
    ("hrtf", "hrtf_decoder_channels", False),
    ("hrtf", "hrtf_decoder", True), ("ambi", "ambi_decoder", True), ("uhj", "uhj_encoder", True),
    ("ambi", "front_stabilizer", True), ("ambi", "bs2b", True), ("ambi", "distance_comp", True),
    ("uhj", "limiter", True)])
def test_rejected_output_stage_call_changes_nothing(kind, call, mid_render):
    """An output-stage setter refused with B200MIX_ERR_INVALID, for a bad argument or between render_begin
    and render_end (with arguments it accepts outside a render), changes nothing: RealOut of the update it
    interrupts and of four more is bit for bit a twin's that never saw the call."""
    devs = [_output_device(kind) for _ in range(2)]
    try:
        outs = [[dev.render()] for dev in devs]
        if mid_render:
            for dev in devs:
                dev.render_begin()
        assert _output_call(devs[0], call) == ERR_INVALID
        if mid_render:
            assert "render_begin is pending" in devs[0].last_error()
            for dev, out in zip(devs, outs):
                out.append(dev.render_end())
        for dev, out in zip(devs, outs):
            out += [dev.render() for _ in range(4)]
        assert np.abs(outs[1][-1]).max() > 1e-4
        for a, b in zip(*outs):
            assert a.tobytes() == b.tobytes()
        if mid_render:
            assert _output_call(devs[0], call) == 0, devs[0].last_error()
    finally:
        for dev in devs:
            dev.close()


# ---- device guard --------------------------------------------------------------------------

def test_output_stage_setters_allocate_on_the_mixers_gpu():
    """A mixer on the last GPU, GPU 0 current before each output-stage setter: RealOut equals the
    same scene's on GPU 0 bit for bit."""
    torch = pytest.importorskip("torch")
    ngpu = torch.cuda.device_count()
    if ngpu < 2:
        pytest.skip("needs two or more GPUs")

    def ambi(dev):
        dev.set_ambi_decoder((np.random.default_rng(5).standard_normal((4, 3)) * 0.5).astype(np.float32), None, 0.0)

    ambi_desc = synth.stereo_desc(64, dry_channels=4)
    ambi_desc.real_channels = 3
    uhj_desc = synth.stereo_desc(64, dry_channels=3)
    uhj_desc.post_process = abi.POST_UHJ
    limiter = abi.device_limiter(-6.0)
    scenes = [(ambi_desc, [ambi, lambda dev: dev.set_bs2b(3), lambda dev: dev.set_front_stabilizer(2, -0.9123257),
                           lambda dev: dev.set_limiter(limiter),
                           lambda dev: dev.set_distance_comp([3, 5, 1], [1.0, 0.9, 0.8])]),
              (uhj_desc, [lambda dev: dev.set_uhj_encoder(256), lambda dev: dev.set_limiter(limiter)])]

    def scene_out(gpu):
        outs = []
        for desc, setters in scenes:
            desc.cuda_device = gpu
            dev = MixDevice(mixlib.product(), desc)
            for setter in setters:
                torch.cuda.set_device(0)
                setter(dev)
            outs += _play_dry(dev)
            dev.close()
        return outs

    a, b = scene_out(ngpu - 1), scene_out(0)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    assert max(np.abs(x).max() for x in a) > 1e-4
