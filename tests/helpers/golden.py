"""Replays a committed golden fixture (tests/golden/*.npz, produced from the compiled
reference by tests/golden/make_golden.py) on a b200mix-surface implementation."""
import ctypes as C
import glob
import os

import numpy as np

from pyb200mix import abi, scene
from .mixlib import MixDevice

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "golden")


# The pitch shifter's fixtures: their GPU replay lives in tests/test_gpu_zz_pshifter.py, which sorts
# last, so that under `pytest -x` it cannot hide the other GPU tests.  The CPU tests treat them like any other.
LATE = ("efx_pshifter_hrtf_v5", "efx_pshifter_down_stereo_v4")


def names():
    return sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, "*.npz")))


def kernel_set_gap(fx):
    """How far the reference's own two kernel sets (SSE vs plain C) are apart on this scene:
    (rms, max).  Effects with poles near z = 1 (the ring modulator's 50 Hz high-pass, the
    equalizer's shelves) amplify the kernels' last-bit differences by orders of magnitude; a
    comparison with `out_sse` cannot be tighter than the reference is with itself."""
    d = fx["out_sse"].astype(np.float64) - fx["out_c"].astype(np.float64)
    return float(np.sqrt((d ** 2).mean())), float(np.abs(d).max())


def load(name):
    return dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz")))


def replay(mixlib, fx, updates=None, frames=abi.LINE):
    """Returns (out [U][ch][frames], final voice results)."""
    V, hrtf, rs, U, looping, buf_frames = [int(x) for x in fx["meta"]]
    desc = abi.DeviceDesc.from_buffer_copy(fx["desc"].tobytes())
    stereo_src = "params_c1" in fx
    desc.max_voices = V * (2 if stereo_src else 1)
    desc.max_buffers = V * (len(fx["queue_lens"]) if "queue_lens" in fx else 1)
    desc.max_slots = 0
    taps = int(fx["conv_taps"]) if "conv_taps" in fx else 0
    reverb = "reverb_params" in fx
    chain = "chain_conv_idx" in fx
    if taps or reverb:
        desc.max_slots = 1
        desc.wet_channels = int(fx["wet_channels"])
    if chain:
        desc.max_slots = 2
        desc.wet_channels = int(fx["wet_channels"])
    efx = "efx_props" in fx
    if efx:
        desc.max_slots = 1
        desc.wet_channels = int(fx["wet_channels"])
    dev = MixDevice(mixlib, desc)
    try:
        if desc.post_process == abi.POST_HRTF:
            dev.set_hrtf_decoder(fx["dec_coeffs"], fx["dec_hf"], fx["dec_sc"])
        elif desc.post_process == abi.POST_AMBIDEC:
            dev.set_ambi_decoder(fx["amb_hf"], fx.get("amb_lf"), float(fx["amb_xover"]))
        fmt = str(fx["fmt"]) if "fmt" in fx else "i16"
        qlens = [int(x) for x in fx["queue_lens"]] if "queue_lens" in fx else None
        if "adpcm_blocks" in fx:
            for i in range(V):
                kind = "ima4" if i % 2 == 0 else "msadpcm"
                dev.buffer_data_adpcm(i, scene.FORMATS[kind][0], scene.ADPCM_BLOCK[kind][0],
                                      int(fx["adpcm_blocks"]), scene.adpcm_blocks(i, kind, int(fx["adpcm_blocks"])))
        elif qlens:
            for i in range(V * len(qlens)):
                dev.buffer_data(i, scene.FORMATS[fmt][0], scene.voice_buffer_fmt(i, qlens[i % len(qlens)], fmt))
        elif stereo_src:
            for i in range(V):
                lr = np.stack([scene.voice_buffer_fmt(2 * i, buf_frames, fmt),
                               scene.voice_buffer_fmt(2 * i + 1, buf_frames, fmt)], axis=1)
                dev.buffer_data(i, scene.FORMATS[fmt][0], np.ascontiguousarray(lr), channels=2)
        else:
            for i in range(V):
                dev.buffer_data(i, scene.FORMATS[fmt][0], scene.voice_buffer_fmt(i, buf_frames, fmt))
        if taps:
            rng = np.random.default_rng(taps)      # same IR as tests/golden/make_golden.py:conv_ir
            ir = (rng.standard_normal(taps) * np.exp(-np.arange(taps) / (taps / 5.0)) * 0.05).astype(np.float32)
            dev.slot_convolution(0, ir[None, :], fx["conv_gains"][None, :])
        if reverb:
            dev.slot_reverb(0, abi.reverb_params_from(fx["reverb_params"].tobytes()),
                            fx["reverb_gains"])
        def set_efx(raw):
            # fixtures written before an effect was added hold a shorter b200mix_efx_props: the new
            # sub-structs are unused by their effect type, zero-extend
            props = abi.EfxProps.from_buffer_copy(bytes(raw).ljust(C.sizeof(abi.EfxProps), b"\0"))
            props.struct_size = C.sizeof(abi.EfxProps)
            dev.slot_efx(0, props, float(fx["efx_slot_gain"]), fx["efx_out_scale"], fx["efx_out_index"],
                         fx["efx_wet_index"], int(fx["efx_ambi_order"]))
        if efx:
            set_efx(fx["efx_props"])
        if chain:
            a, b = int(fx["chain_conv_idx"]), int(fx["chain_reverb_idx"])
            dev.slot_target(a, b)
            n600 = int(fx["conv_taps_chain"])
            rng = np.random.default_rng(n600)      # make_golden.py:conv_ir
            ir = (rng.standard_normal(n600) * np.exp(-np.arange(n600) / (n600 / 5.0)) * 0.05).astype(np.float32)
            dev.slot_convolution(a, ir[None, :], fx["chain_conv_gains"][None, :])
            dev.slot_reverb(b, abi.reverb_params_from(fx["chain_reverb_params"].tobytes()), fx["chain_reverb_gains"])
        params = (abi.VoiceParams * V).from_buffer_copy(fx["params"].tobytes())
        plist = []
        for k in range(V):
            q = abi.VoiceParams()
            C.memmove(C.byref(q), C.byref(params[k]), C.sizeof(q))
            q.buffer = k
            # the snapshot was taken after the reference's first update: restart the voice
            q.flags = (q.flags & ~(abi.VF_STOPPING | abi.VF_STOPPED)) | abi.VF_PLAYING | abi.VF_RESET
            q.position = 0
            q.position_frac = 0
            plist.append(q)
        coeffs, dry = fx["coeffs"], fx["dry"]
        if stereo_src:
            # one voice per mixing channel: voice 2k+c = channel c of source k, in the order the
            # reference mixes them (voice by voice, channel by channel)
            params1 = (abi.VoiceParams * V).from_buffer_copy(fx["params_c1"].tobytes())
            both = []
            for k in range(V):
                for c, src in ((0, plist[k]), (1, params1[k])):
                    q = abi.VoiceParams()
                    C.memmove(C.byref(q), C.byref(plist[k]), C.sizeof(q))
                    q.voice = 2 * k + c
                    q.hrtf_delay[0], q.hrtf_delay[1] = src.hrtf_delay[0], src.hrtf_delay[1]
                    q.hrtf_gain = src.hrtf_gain
                    q.flags |= abi.vf_channel(c)
                    both.append(q)
            plist = both
            coeffs = np.stack([fx["coeffs"], fx["coeffs_c1"]], axis=1).reshape((2 * V,) + fx["coeffs"].shape[1:])
            dry = np.stack([fx["dry"], fx["dry_c1"]], axis=1).reshape((2 * V,) + fx["dry"].shape[1:])
        dev.voices_update(plist, coeffs, dry, fx["send"] if (taps or reverb or chain or efx) else None)
        if qlens:
            for k in range(V):
                ids = [k * len(qlens) + j for j in range(len(qlens))]
                dev.voice_queue(k, ids, 0 if (plist[k].flags & abi.VF_LOOPING) else abi.NO_LOOP)
        if "stab_center" in fx:
            dev.set_front_stabilizer(int(fx["stab_center"]), float(fx["stab_coeff"]))
        if "uhj_fir" in fx:
            n = int(fx["uhj_fir"])
            assert dev.set_uhj_encoder(n) == n // 2 + 128
        if "distcomp_delays" in fx:
            dev.set_distance_comp(fx["distcomp_delays"], fx["distcomp_gains"])
        if "limiter_desc" in fx:
            la = dev.set_limiter(abi.LimiterDesc.from_buffer_copy(fx["limiter_desc"].tobytes()))
            assert la == int(fx["limiter_look_ahead"]), (la, int(fx["limiter_look_ahead"]))
        outs = []
        res = None
        seed = 22222            # DitherRNGSeed, alc/alc.cpp:329
        for u in range(updates or U):
            if "filt_meta" in fx:
                # the reference's filter targets during update u, every path of every voice
                dev.voices_filters((int(m[0]), int(m[1]), int(m[2]), c[0], c[1])
                                   for m, c in zip(fx["filt_meta"][u], fx["filt_coef"][u]))
            if "mv_params" in fx and u > 0:
                # the reference recomputed the moved sources' targets before this update: resend
                # the voices whose snapshot differs from the previous one
                mp = (abi.VoiceParams * V).from_buffer_copy(fx["mv_params"][u].tobytes())
                mprev = (abi.VoiceParams * V).from_buffer_copy(fx["mv_params"][u - 1].tobytes())
                sel = []
                for k in range(V):
                    same = (np.array_equal(fx["mv_coeffs"][u][k], fx["mv_coeffs"][u - 1][k])
                            and np.array_equal(fx["mv_dry"][u][k], fx["mv_dry"][u - 1][k])
                            and mp[k].hrtf_gain == mprev[k].hrtf_gain
                            and list(mp[k].hrtf_delay) == list(mprev[k].hrtf_delay))
                    if not same:
                        sel.append(k)
                if sel:
                    ql = []
                    for k in sel:
                        q = abi.VoiceParams()
                        C.memmove(C.byref(q), C.byref(mp[k]), C.sizeof(q))
                        q.buffer = k
                        q.flags = (q.flags & ~(abi.VF_STOPPING | abi.VF_STOPPED | abi.VF_RESET)) | abi.VF_PLAYING
                        ql.append(q)
                    dev.voices_update(ql, fx["mv_coeffs"][u][sel], fx["mv_dry"][u][sel], None)
            if efx:
                for k, uu in enumerate(fx["efx_step_updates"]):
                    if int(uu) == u:
                        set_efx(fx["efx_step_props"][k])
            if "rv_state" in fx and u > 0:
                # replay the reference's ReverbState::update calls: a flipped mCurrentPipeline bit
                # marks a full update; otherwise changed values are applied in place
                st, prev = int(fx["rv_state"][u]), int(fx["rv_state"][u - 1])
                full = (st >> 8) != (prev >> 8)
                changed = full or not np.array_equal(fx["rv_params"][u], fx["rv_params"][u - 1]) \
                    or not np.array_equal(fx["rv_gains"][u], fx["rv_gains"][u - 1])
                if changed:
                    dev.slot_reverb_update(0, abi.reverb_params_from(fx["rv_params"][u].tobytes()), full,
                                           fx["rv_gains"][u])
            if "out_type" in fx:
                o, res, seed = dev.render_interleaved(frames, int(fx["out_type"]), float(fx["dither_depth"]), seed)
                o = np.ascontiguousarray(o.T)        # planar like the fixture
            else:
                o, res = dev.render(frames, want_results=True)
            outs.append(o)
        out = np.stack(outs)
        if "undefined_head" in fx:
            # samples the reference itself leaves undefined (zeroed in the fixture, see
            # make_golden.py): the first update's head of every delayed channel
            for c, n in enumerate(fx["undefined_head"]):
                out[0, c, :int(n)] = 0
        return out, res
    finally:
        dev.close()
