"""-m gpu parity tests proper: the CUDA mixer through the C ABI (libb200mix.so) against
(1) the committed golden vectors rendered by the compiled reference,
(2) the CPU oracle on seeded synthetic descriptors at larger sizes,
(3) size-independent properties at BASELINE.json's config-2 size.
Tolerance (north_star): RMS <= 1e-5 and max-abs <= 1e-4 on float32 output; we hold the
CUDA path to a 10x tighter bound against the oracle since both follow the same math."""
import ctypes as C

import numpy as np
import pytest

from helpers import golden, mixlib, synth
from helpers.mixlib import MixDevice
from pyb200mix import abi, scene

pytestmark = pytest.mark.gpu

RMS_TOL, MAX_TOL = 1e-6, 1e-5


def _check(out, ref, what="", rms_tol=RMS_TOL, max_tol=MAX_TOL):
    err = out.astype(np.float64) - ref.astype(np.float64)
    rms = float(np.sqrt((err ** 2).mean()))
    mx = float(np.abs(err).max())
    assert rms <= rms_tol and mx <= max_tol, f"{what}: rms {rms:.3e} max {mx:.3e}"
    assert np.abs(ref).max() > 1e-4, "reference output is silent"


@pytest.mark.parametrize("name", [n for n in golden.names() if n not in golden.LATE])
def test_golden_vectors_from_reference(name):
    golden_case(name)


def golden_case(name):
    fx = golden.load(name)
    out, res = golden.replay(mixlib.product(), fx)
    if "out_type" in fx:
        # integer output (dither + Write<T>): the float mix ahead of the rounding differs from the
        # reference's in the last bits, so a sample may land on the neighbouring integer — never
        # further, and rarely (the dither noise itself is reproduced exactly)
        for key in ("out_sse", "out_c"):
            diff = np.abs(out.astype(np.int64) - fx[key].astype(np.int64))
            assert diff.max() <= 1, (name, key, int(diff.max()))
            assert (diff != 0).mean() <= 0.01, (name, key, float((diff != 0).mean()))
        assert np.ptp(fx["out_c"].astype(np.int64)) > 8
    else:
        gap_rms, gap_max = golden.kernel_set_gap(fx)      # the reference against itself (SSE vs C)
        max_tol = max(MAX_TOL, 2 * gap_max)
        if name.startswith(("efx_chorus", "efx_flanger")):
            # The sinusoid LFO is rounded to a 24.8 fixed-point delay per sample (fastf2i,
            # chorus.cpp:300-323).  glibc's sinf is not correctly rounded (<= 0.56 ulp); the kernel's
            # sine is (double sin, rounded once), so on isolated samples the delay lands 1/256 sample
            # away and the cubic-interpolated tap differs by ~slope/256.  RMS keeps the 10x-tighter
            # bar; the peak gets north_star's own budget (1e-4).
            max_tol = max(max_tol, 1e-4)
        _check(out, fx["out_sse"], name + " vs reference SSE kernels", max(RMS_TOL, 2 * gap_rms), max_tol)
        _check(out, fx["out_c"], name + " vs reference C kernels", max(RMS_TOL, 2 * gap_rms), max_tol)
    # voice bookkeeping agrees with the oracle (positions are integers: exact)
    out_o, res_o = golden.replay(mixlib.oracle(), fx)
    V = int(fx["meta"][0])
    for k in range(V):
        assert (res[k].position, res[k].position_frac, res[k].flags, res[k].buffers_done) == \
            (res_o[k].position, res_o[k].position_frac, res_o[k].flags, res_o[k].buffers_done), k


def _run_pair(desc_fn, nv, updates, **kw):
    rng = np.random.default_rng(1234 + nv)
    ir = kw.pop("ir", 64)
    hrtf = kw.pop("hrtf", True)
    desc = desc_fn(nv, ir) if hrtf else desc_fn(nv)
    params, coeffs, dry = synth.voice_set(rng, nv, ir, hrtf=hrtf, dry_channels=desc.dry_channels, **kw)
    frames = kw.get("frames", scene.BUFFER_FRAMES)
    outs = []
    for lib in (mixlib.oracle(), mixlib.product()):
        dev = MixDevice(lib, desc)
        if desc.post_process == abi.POST_HRTF:
            dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7), desc.dry_channels))
        else:
            g = np.random.default_rng(8).standard_normal((desc.dry_channels, desc.real_channels))
            dev.set_ambi_decoder(g.astype(np.float32), None, 0.0)
        for i in range(nv):
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i, frames))
        dev.voices_update(params, coeffs if hrtf else None, dry, None)
        o = []
        for u in range(updates):
            if u == 2:
                # move a quarter of the voices: new coefficients, delays, gains (MixHrtfBlend path)
                rng2 = np.random.default_rng(99)
                sub = [p for k, p in enumerate(params) if k % 4 == 1]
                c2 = (rng2.standard_normal((len(sub), max(ir, 1), 2)) * 0.2).astype(np.float32)
                d2 = (rng2.standard_normal((len(sub), desc.dry_channels)) * 0.3).astype(np.float32)
                sub2 = []
                for p in sub:
                    q = abi.VoiceParams.from_buffer_copy(bytes(p))
                    q.flags &= ~abi.VF_RESET
                    q.hrtf_delay[0] = (q.hrtf_delay[0] + 5) % 64
                    q.hrtf_gain *= 0.7
                    sub2.append(q)
                dev.voices_update(sub2, c2 if hrtf else None, d2, None)
            o.append(dev.render())
        dev.close()
        outs.append(np.stack(o))
    return outs


@pytest.mark.parametrize("resampler", [abi.RS_BSINC24, abi.RS_SPLINE, abi.RS_FAST_BSINC12,
                                       abi.RS_BSINC48, abi.RS_LINEAR, abi.RS_POINT, abi.RS_GAUSSIAN])
def test_hrtf_vs_oracle_synthetic(resampler):
    o, p = _run_pair(synth.hrtf_desc, 96, 4, resampler=resampler)
    _check(p, o, f"hrtf resampler {resampler}")


def test_hrtf_ir128_vs_oracle():
    o, p = _run_pair(synth.hrtf_desc, 40, 3, ir=128)
    _check(p, o, "ir=128")


def test_hrtf_oneshot_and_high_pitch_vs_oracle():
    o, p = _run_pair(synth.hrtf_desc, 48, 6, looping=False, frames=6000, pitch_lo=0.3, pitch_hi=9.5)
    _check(p, o, "one-shot, pitch up to 9.5")


@pytest.mark.parametrize("resampler", [abi.RS_SPLINE, abi.RS_BSINC24])
def test_dry_mix_vs_oracle(resampler):
    o, p = _run_pair(synth.stereo_desc, 64, 4, hrtf=False, resampler=resampler)
    _check(p, o, "plain dry mix (config 1 shape)")


def test_partial_update_sizes_vs_oracle():
    rng = np.random.default_rng(5)
    nv, ir = 24, 64
    desc = synth.hrtf_desc(nv, ir)
    params, coeffs, dry = synth.voice_set(rng, nv, ir)
    outs = []
    for lib in (mixlib.oracle(), mixlib.product()):
        dev = MixDevice(lib, desc)
        dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
        for i in range(nv):
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
        dev.voices_update(params, coeffs, dry, None)
        o = [dev.render(f) for f in (1024, 37, 512, 1, 1000, 64)]
        dev.close()
        outs.append(np.concatenate(o, axis=1))
    _check(outs[1], outs[0], "ragged update sizes")


LIMITER_DESCS = {
    # the reference's device limiter (CreateDeviceLimiter, alc/alc.cpp:1079-1091), 16-bit threshold
    "device": abi.device_limiter(-0.00053),
    # a plain 4:1 compressor: nothing automated, soft knee, pre/post gain, no hold
    "manual": abi.LimiterDesc(C.sizeof(abi.LimiterDesc), 0, 0.002, 0.0, 3.0, -1.5, -9.0, 4.0, 6.0, 0.005, 0.1),
    # automation without look-ahead (no delay lines, no hold)
    "no_lookahead": abi.LimiterDesc(C.sizeof(abi.LimiterDesc), abi.LIM_AUTO_ALL, 0.0, 0.002, 0.0, 0.0, -3.0,
                                    float("inf"), 0.0, 0.02, 0.2),
}


@pytest.mark.parametrize("kind", sorted(LIMITER_DESCS))
def test_limiter_vs_oracle_ragged_updates(kind):
    """Compressor::process on a mix driven past full scale, with update sizes below and above the
    look-ahead (48) and hold (96) lengths; the unlimited mix is checked to be much louder."""
    rng = np.random.default_rng(21)
    nv, ir = 16, 64
    desc = synth.hrtf_desc(nv, ir)
    params, coeffs, dry = synth.voice_set(rng, nv, ir)
    for p in params:
        p.hrtf_gain *= 12.0
    sizes = (1024, 37, 512, 1, 1000, 64, 20, 20, 100, 1024)
    outs = []
    for lib, lim in ((mixlib.oracle(), True), (mixlib.product(), True), (mixlib.product(), False)):
        dev = MixDevice(lib, desc)
        dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
        for i in range(nv):
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
        dev.voices_update(params, coeffs, dry, None)
        if lim:
            la = dev.set_limiter(LIMITER_DESCS[kind])
            assert la == round(LIMITER_DESCS[kind].look_ahead_time * desc.sample_rate)
        o = [dev.render(f) for f in sizes]
        if lim:
            dev.set_limiter(None)      # device->Limiter = nullptr
        dev.close()
        outs.append(np.concatenate(o, axis=1))
    # the tolerances are for full-scale output: a compressor that leaves the mix above 1.0 is
    # judged relative to its peak
    scale = max(1.0, float(np.abs(outs[0]).max()))
    _check(outs[1] / scale, outs[0] / scale, f"limiter {kind}")
    assert np.abs(outs[2]).max() > 2.0 * np.abs(outs[1]).max()


def test_distance_comp_vs_oracle_ragged_updates():
    """ApplyDistanceComp after an ambisonic decode: per-channel FIFOs longer and shorter than the
    update sizes, a channel without delay (left untouched, gain included), then removal."""
    rng = np.random.default_rng(31)
    nv = 12
    desc = synth.stereo_desc(nv)
    params, coeffs, dry = synth.voice_set(rng, nv, 0, hrtf=False, dry_channels=desc.dry_channels)
    delays = np.array([700, 0][:desc.real_channels] + [13] * max(desc.real_channels - 2, 0), dtype=np.uint32)
    gains = np.array([0.6, 0.25][:desc.real_channels] + [0.9] * max(desc.real_channels - 2, 0), dtype=np.float32)
    sizes = (1024, 37, 512, 1, 1000, 64, 5, 1024)
    outs = []
    for lib in (mixlib.oracle(), mixlib.product()):
        dev = MixDevice(lib, desc)
        g = np.random.default_rng(8).standard_normal((desc.dry_channels, desc.real_channels))
        dev.set_ambi_decoder(g.astype(np.float32), None, 0.0)
        for i in range(nv):
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
        dev.voices_update(params, None, dry, None)
        dev.set_distance_comp(delays, gains)
        o = [dev.render(f) for f in sizes]
        dev.set_distance_comp(None, None)
        o.append(dev.render(256))
        dev.close()
        outs.append(np.concatenate(o, axis=1))
    _check(outs[1], outs[0], "distance compensation")
    # channel 0 starts with 700 samples of (zeroed) delay line
    assert not outs[1][0, :700].any() and outs[1][0, 700:1024].any()


@pytest.mark.parametrize("post,taps", [(abi.POST_UHJ, 0), (abi.POST_UHJ, 256), (abi.POST_UHJ, 512),
                                       (abi.POST_TSME, 0), (abi.POST_TSME, 256), (abi.POST_TSME, 512)])
def test_matrix_encoders_vs_oracle_ragged_updates(post, taps):
    """Uhj/TsmeEncoderIIR (taps 0) and Uhj/TsmeEncoder<256/512> on a 3- / 4-channel dry mix, update
    sizes below and above the encoder delay (N/2 + 128) and the FIR history."""
    rng = np.random.default_rng(41 + taps + post)
    nv = 12
    desc = synth.stereo_desc(nv, dry_channels=4 if post == abi.POST_TSME else 3)
    desc.post_process = post
    params, coeffs, dry = synth.voice_set(rng, nv, 0, hrtf=False, dry_channels=desc.dry_channels)
    sizes = (1024, 37, 512, 1, 1000, 64, 300, 5, 1024)
    outs = []
    for lib in (mixlib.oracle(), mixlib.product()):
        dev = MixDevice(lib, desc)
        for i in range(nv):
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
        dev.voices_update(params, None, dry, None)
        assert dev.set_uhj_encoder(taps) == (taps // 2 + 128 if taps else 1)
        o = [dev.render(f) for f in sizes]
        dev.close()
        outs.append(np.concatenate(o, axis=1))
    _check(outs[1], outs[0], f"matrix encoder {post} {taps}")
    if taps:
        d = taps // 2 + 128
        assert not outs[1][:, :128].any() and outs[1][:, d:d + 512].any()


@pytest.mark.parametrize("level", [1, 3, 6])
def test_bs2b_crossfeed_vs_oracle_ragged_updates(level):
    """Bs2bPostProcess: ambisonic decode + BS2B crossfeed (the oracle's filter is bit-exact with
    the reference's Bs2b::bs2b_processor, tests/test_oracle_vs_ref.py), ragged updates, removal."""
    rng = np.random.default_rng(51 + level)
    nv = 12
    desc = synth.stereo_desc(nv)
    params, coeffs, dry = synth.voice_set(rng, nv, 0, hrtf=False, dry_channels=desc.dry_channels)
    sizes = (1024, 37, 512, 1, 1000, 64, 7, 1024)
    outs = []
    for lib, lev in ((mixlib.oracle(), level), (mixlib.product(), level), (mixlib.product(), 0)):
        dev = MixDevice(lib, desc)
        g = np.random.default_rng(8).standard_normal((desc.dry_channels, desc.real_channels))
        dev.set_ambi_decoder(g.astype(np.float32), None, 0.0)
        for i in range(nv):
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
        dev.voices_update(params, None, dry, None)
        dev.set_bs2b(lev)
        o = [dev.render(f) for f in sizes]
        dev.close()
        outs.append(np.concatenate(o, axis=1))
    _check(outs[1], outs[0], f"bs2b level {level}")
    assert np.abs(outs[1] - outs[2]).max() > 1e-3       # the crossfeed did change the output


def test_front_stabilizer_vs_oracle_ragged_updates():
    """StablizerPostProcess on a 6-channel decode (the oracle is bit-exact with the reference on
    the 5.1 golden): mid band split, centre feed, all-pass on the other channels; then removal."""
    rng = np.random.default_rng(61)
    nv = 12
    desc = synth.stereo_desc(nv, dry_channels=4)
    desc.real_channels = 6
    params, coeffs, dry = synth.voice_set(rng, nv, 0, hrtf=False, dry_channels=desc.dry_channels)
    sizes = (1024, 37, 512, 1, 1000, 64, 7, 1024)
    outs = []
    for lib, on in ((mixlib.oracle(), True), (mixlib.product(), True), (mixlib.product(), False)):
        dev = MixDevice(lib, desc)
        g = np.random.default_rng(8).standard_normal((desc.dry_channels, desc.real_channels)) * 0.5
        g[:, 2] = 0.0          # the decoder leaves the centre speaker to the stabilizer
        dev.set_ambi_decoder(g.astype(np.float32), None, 0.0)
        for i in range(nv):
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
        dev.voices_update(params, None, dry, None)
        if on:
            dev.set_front_stabilizer(2, -0.49314544)
        o = [dev.render(f) for f in sizes]
        if on:
            dev.set_front_stabilizer(abi.NO_SLOT, 0.0)
            o.append(dev.render(128))
        dev.close()
        outs.append(np.concatenate(o, axis=1))
    _check(outs[1], outs[0], "front stabilizer")
    assert np.abs(outs[1][2]).max() > 1e-3 and not outs[2][2].any()     # only the stabilizer feeds the centre


def test_config2_size_linearity_and_subsample():
    """BASELINE config 2 size (4096 HRTF voices, bsinc24): the oracle only mixes a
    deterministic 1/16 subsample; the full mix is checked by linearity — the sum of
    the 16 disjoint sub-mixes equals the full mix (same inputs, fp32 reassociation only)."""
    nv, ir, k = 4096, 64, 16
    rng = np.random.default_rng(2024)
    desc = synth.hrtf_desc(nv, ir)
    params, coeffs, dry = synth.voice_set(rng, nv, ir)
    dec = synth.decoder(np.random.default_rng(7))
    pcm = [scene.voice_buffer_fast(i) for i in range(nv)]

    def run(lib, subset):
        dev = MixDevice(lib, desc)
        dev.set_hrtf_decoder(*dec)
        for i in subset:
            dev.buffer_data(i, abi.FMT_I16, pcm[i])
        dev.voices_update([params[i] for i in subset], coeffs[subset], dry[subset], None)
        o = np.stack([dev.render() for _ in range(3)])
        dev.close()
        return o

    full = run(mixlib.product(), list(range(nv)))
    parts = [run(mixlib.product(), list(range(r, nv, k))) for r in range(k)]
    _check(np.sum(parts, axis=0), full, "linearity: sum of 16 sub-mixes == full mix")
    sub = list(range(0, nv, k))
    _check(parts[0], run(mixlib.oracle(), sub), "1/16 subsample vs oracle")
    assert np.sqrt((full ** 2).mean()) > 1e-3


def test_convolution_slot_vs_oracle_long_ir_and_ragged_updates():
    """Aux sends -> convolution slot (2 IR channels, 20000 taps = 156 FFT segments), ragged
    update sizes so FFT blocks complete mid-update; HRTF voices + a non-silent Dry mix."""
    rng = np.random.default_rng(77)
    nv, ir = 40, 64
    desc = synth.hrtf_desc(nv, ir)
    desc.num_sends = 2
    desc.wet_channels = 4
    desc.max_slots = 3
    params, coeffs, dry = synth.voice_set(rng, nv, ir)
    send = (rng.standard_normal((nv, 2, 4)) * 0.3).astype(np.float32)
    for k, p in enumerate(params):
        p.send_slot[0] = k % 3 if k % 5 else abi.NO_SLOT
        p.send_slot[1] = (k + 1) % 3 if k % 2 else abi.NO_SLOT
    taps = [20000, 300, 1153]
    irs = [(rng.standard_normal((2 if s == 0 else 1, t)) * np.exp(-np.arange(t) / (t / 4.0)) * 0.03
            ).astype(np.float32) for s, t in enumerate(taps)]
    gains = [(rng.standard_normal((x.shape[0], desc.dry_channels)) * 0.5).astype(np.float32) for x in irs]
    outs = []
    for lib in (mixlib.oracle(), mixlib.product()):
        dev = MixDevice(lib, desc)
        dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
        for i in range(nv):
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
        for s in range(3):
            dev.slot_convolution(s, irs[s], gains[s])
        dev.voices_update(params, coeffs, dry, send)
        o = [dev.render(f) for f in (1024, 100, 1024, 28, 640, 1024, 1, 255, 1024)]
        dev.close()
        outs.append(np.concatenate(o, axis=1))
    _check(outs[1], outs[0], "convolution slots")


def test_reverb_slots_vs_oracle_ragged_updates():
    """EAX reverb slots driven by the reference's own parameter blocks (taken from two golden
    fixtures: default preset and min-density + modulation), ragged update sizes."""
    rng = np.random.default_rng(5150)
    nv, ir = 24, 64
    desc = synth.hrtf_desc(nv, ir)
    desc.num_sends = 1
    desc.wet_channels = 4
    desc.max_slots = 2
    params, coeffs, dry = synth.voice_set(rng, nv, ir)
    send = (rng.standard_normal((nv, 1, 4)) * 0.3).astype(np.float32)
    for k, p in enumerate(params):
        p.send_slot[0] = k % 2
    fxs = [golden.load("hrtf_bsinc24_reverb_v6"), golden.load("hrtf_spline_reverb_dens0_mod_v4")]
    outs = []
    for lib in (mixlib.oracle(), mixlib.product()):
        dev = MixDevice(lib, desc)
        dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
        for i in range(nv):
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
        for s, fx in enumerate(fxs):
            dev.slot_reverb(s, abi.reverb_params_from(fx["reverb_params"].tobytes()),
                            fx["reverb_gains"])
        dev.voices_update(params, coeffs, dry, send)
        o = [dev.render(f) for f in (1024, 300, 1024, 17, 1024, 1024, 700, 1024)]
        dev.close()
        outs.append(np.concatenate(o, axis=1))
    _check(outs[1], outs[0], "reverb slots")


def _shelf_pair(lib, gain_hf, gain_lf):
    """What alc/alu.cpp:1630-1631 hands the filters: high-shelf at 5 kHz, low-shelf at 250 Hz."""
    lp = np.zeros(5, dtype=np.float32)
    hp = np.zeros(5, dtype=np.float32)
    assert lib.biquad_coeffs(0, 5000.0 / 48000.0, gain_hf, 1.0, lp.ctypes.data) == 0
    assert lib.biquad_coeffs(1, 250.0 / 48000.0, gain_lf, 1.0, hp.ctypes.data) == 0
    return lp, hp


@pytest.mark.parametrize("hrtf", [True, False])
def test_direct_and_send_filters_vs_oracle_ragged_updates(hrtf):
    """DoFilters on the direct path and on a send, with targets changing between ragged
    updates so coefficient interpolation starts, straddles update boundaries mid-step,
    restarts while running, and filters get detached (clear) and re-attached."""
    rng = np.random.default_rng(2024)
    nv, ir = 40, 64
    desc = synth.hrtf_desc(nv, ir) if hrtf else synth.stereo_desc(nv)
    desc.num_sends = 1
    desc.wet_channels = 4
    desc.max_slots = 1
    params, coeffs, dry = synth.voice_set(rng, nv, ir if hrtf else 0, hrtf=hrtf,
                                          dry_channels=desc.dry_channels)
    send = (rng.standard_normal((nv, 1, 4)) * 0.3).astype(np.float32)
    for k, p in enumerate(params):
        p.send_slot[0] = 0 if k % 3 else abi.NO_SLOT
    fx = golden.load("hrtf_bsinc24_reverb_v6")
    sizes = (1024, 37, 512, 1, 1000, 64, 1024, 333, 1024)
    # (update index, voice stride/offset, path, gainHF, gainLF)
    script = {0: [(2, 0, 0, 0.2, 1.0), (3, 1, 1, 0.1, 0.5), (5, 2, 0, 0.7, 0.3)],
              1: [(2, 0, 0, 0.9, 1.0), (4, 1, 0, 0.05, 1.0)],
              2: [(2, 0, 0, 0.3, 0.6), (3, 1, 1, 1.0, 1.0)],
              4: [(5, 2, 0, 1.0, 1.0), (3, 1, 1, 0.4, 1.0)],
              6: [(4, 1, 0, 0.6, 0.9), (5, 2, 0, 0.25, 1.0)]}
    outs = []
    for lib in (mixlib.oracle(), mixlib.product()):
        dev = MixDevice(lib, desc)
        if hrtf:
            dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
        else:
            dev.set_ambi_decoder((np.random.default_rng(3).standard_normal((desc.dry_channels, 2)) * 0.5
                                  ).astype(np.float32), None, 0.0)
        for i in range(nv):
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
        dev.slot_reverb(0, abi.reverb_params_from(fx["reverb_params"].tobytes()),
                        np.ascontiguousarray(fx["reverb_gains"][:, :desc.dry_channels]))
        dev.voices_update(params, coeffs if hrtf else None, dry, send)
        o = []
        for u, f in enumerate(sizes):
            ents = []
            for stride, off, path, ghf, glf in script.get(u, []):
                lp, hp = _shelf_pair(mixlib.product(), ghf, glf)
                for v in range(off, nv, stride):
                    if path == 1 and params[v].send_slot[0] == abi.NO_SLOT:
                        continue
                    ents.append((v, path, int(ghf != 1.0 or glf != 1.0), lp, hp))
            # one entry per (voice, path) per call: later script lines win
            uniq = {(e[0], e[1]): e for e in ents}
            if uniq:
                dev.voices_filters(uniq.values())
            o.append(dev.render(f))
        dev.close()
        outs.append(np.concatenate(o, axis=1))
    # The EFX low-shelf at 250 Hz has poles at |z| ~ 0.98: the fp32 recurrence amplifies its own
    # rounding noise ~1000x (a 0.25-amplitude line is only good to ~4e-6 in the reference itself),
    # and that noise decorrelates as soon as the input differs in the last bit (the CUDA resampler
    # uses FMA).  The CUDA filter runs the reference's exact operation order; what is left is this
    # noise floor, so the bound here is 3x the usual one — still 3x inside north_star's tolerance.
    _check(outs[1], outs[0], "direct + send filters", rms_tol=3e-6, max_tol=3e-5)


def _cuda_view(ptr, count):
    import torch

    class _W:
        pass
    w = _W()
    w.__cuda_array_interface__ = {"shape": (count,), "typestr": "<f4", "data": (ptr, False), "version": 2}
    return torch.as_tensor(w, device=torch.device("cuda", 0))


def test_two_device_slot_ownership_equals_single_device():
    """SURVEY §8e on one GPU: two b200mix devices stand for two ranks — voices split in
    halves, each reverb slot installed only on its owner, the Wet buffers summed between
    render_begin and render_end (what ncclAllReduce does across GPUs), RealOut blocks added.
    The result must equal one device mixing everything."""
    import ctypes as C
    import torch
    rng = np.random.default_rng(77)
    nv, ir = 32, 64
    desc = synth.hrtf_desc(nv, ir)
    desc.num_sends = 1
    desc.wet_channels = 4
    desc.max_slots = 2
    params, coeffs, dry = synth.voice_set(rng, nv, ir)
    send = (rng.standard_normal((nv, 1, 4)) * 0.3).astype(np.float32)
    for k, p in enumerate(params):
        p.send_slot[0] = k % 2
    fxs = [golden.load("hrtf_bsinc24_reverb_v6"), golden.load("hrtf_spline_reverb_dens0_mod_v4")]
    sizes = (1024, 300, 1024, 1024, 17, 1024)
    lib = mixlib.product()
    lib.lib.b200mix_stream.restype = C.c_void_p
    lib.lib.b200mix_stream.argtypes = [C.c_void_p]

    def make(voices, owned):
        dev = MixDevice(lib, desc)
        dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
        for i in voices:
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
        for s, fx in enumerate(fxs):
            if s in owned:
                dev.slot_reverb(s, abi.reverb_params_from(fx["reverb_params"].tobytes()),
                                fx["reverb_gains"])
        dev.voices_update([params[i] for i in voices], coeffs[voices], dry[voices], send[voices])
        return dev

    single = make(list(range(nv)), {0, 1})
    ref = np.concatenate([single.render(f) for f in sizes], axis=1)
    # begin/end on one device is the same update as render
    single2 = make(list(range(nv)), {0, 1})
    o = []
    for f in sizes:
        single2.render_begin(f)
        o.append(single2.render_end())
    assert np.array_equal(np.concatenate(o, axis=1), ref)
    single.close()
    single2.close()

    ranks = [make(list(range(0, nv // 2)), {0}), make(list(range(nv // 2, nv)), {1})]
    outs = []
    for f in sizes:
        wets = []
        for dev in ranks:
            ptr, cnt = dev.render_begin(f)
            wets.append(_cuda_view(ptr, cnt))
        torch.cuda.synchronize()
        total = wets[0] + wets[1]
        for w in wets:
            w.copy_(total)
        torch.cuda.synchronize()
        outs.append(sum(dev.render_end() for dev in ranks))
    for dev in ranks:
        dev.close()
    _check(np.concatenate(outs, axis=1), ref, "two-device slot ownership")


def test_device_side_hrir_lookup_is_bit_identical_to_host_helper():
    """SURVEY §8f #1: b200mix_voices_update_dirs computes HrtfStore::getCoeffs on the GPU.
    Two devices mix the same scene — one fed HRIRs from the host helper (itself pinned to the
    reference's ALU in test_hrtf_params.py), one fed only directions — through moving voices
    and ragged updates; the outputs must be identical to the bit."""
    import ctypes as C
    import os
    mhr = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       "openal-soft_b200", "data", "Default HRTF.mhr")
    if not os.path.exists(mhr):
        pytest.skip("HRTF data set not staged (run build())")
    lib = mixlib.product().lib
    lib.b200mix_hrtf_load.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p)]
    lib.b200mix_hrtf_get_coeffs.argtypes = [C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_float,
                                            C.c_void_p, C.POINTER(C.c_uint32)]
    lib.b200mix_hrtf_free.argtypes = [C.c_void_p]
    lib.b200mix_hrtf_attach.argtypes = [C.c_void_p, C.c_void_p]
    lib.b200mix_voices_update_dirs.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p]
    data = open(mhr, "rb").read()
    hs = C.c_void_p()
    assert lib.b200mix_hrtf_load(data, len(data), C.byref(hs)) == 0
    rng = np.random.default_rng(4242)
    nv, ir = 48, 64
    desc = synth.hrtf_desc(nv, ir)
    params, _, dry = synth.voice_set(rng, nv, ir)

    def directions(seed):
        r = np.random.default_rng(seed)
        d = np.zeros((nv, 4), dtype=np.float32)
        d[:, 0] = r.uniform(-np.pi / 2, np.pi / 2, nv)        # elevation
        d[:, 1] = r.uniform(-np.pi, np.pi, nv)                # azimuth
        d[:, 2] = r.uniform(0.05, 3.0, nv)                    # distance (field selection)
        d[:, 3] = r.uniform(0.0, np.pi, nv) * (r.random(nv) < 0.3)   # spread on a third
        d[0] = [np.pi / 2, 0.0, 1.0, 0.0]                     # poles and seams
        d[1] = [-np.pi / 2, np.pi, 1.0, 0.0]
        d[2] = [0.0, -np.pi, 1.0, 2 * np.pi]
        return d

    def host_lookup(dirs, plist):
        coeffs = np.zeros((len(plist), ir, 2), dtype=np.float32)
        dl = (C.c_uint32 * 2)()
        for k, p in enumerate(plist):
            e, a, dist, sp = [float(x) for x in dirs[k]]
            assert lib.b200mix_hrtf_get_coeffs(hs, e, a, dist, sp, coeffs[k].ctypes.data, dl) == 0
            p.hrtf_delay[0], p.hrtf_delay[1] = dl[0], dl[1]
        return coeffs

    devs = [MixDevice(mixlib.product(), desc), MixDevice(mixlib.product(), desc)]
    assert lib.b200mix_hrtf_attach(devs[1].h, hs) == 0
    for dev in devs:
        dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
        for i in range(nv):
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
    outs = [[], []]
    for u, f in enumerate((1024, 1024, 300, 1024, 64, 1024)):
        if u in (0, 2, 3):
            dirs = directions(100 + u)
            sub = list(range(nv)) if u == 0 else list(range(u, nv, 3))
            plist = []
            for k in sub:
                q = abi.VoiceParams.from_buffer_copy(bytes(params[k]))
                if u:
                    q.flags &= ~abi.VF_RESET
                plist.append(q)
            coeffs = host_lookup(dirs[sub], plist)
            devs[0].voices_update(plist, coeffs, dry[sub], None)
            arr = (abi.VoiceParams * len(plist))(*plist)
            dsub = np.ascontiguousarray(dirs[sub])
            dd = np.ascontiguousarray(dry[sub])
            assert lib.b200mix_voices_update_dirs(devs[1].h, len(plist), arr, dsub.ctypes.data,
                                                  dd.ctypes.data, None) == 0
        for j, dev in enumerate(devs):
            outs[j].append(dev.render(f))
    for dev in devs:
        dev.close()
    lib.b200mix_hrtf_free(hs)
    a, b = np.concatenate(outs[0], axis=1), np.concatenate(outs[1], axis=1)
    assert np.abs(a).max() > 1e-4
    assert np.array_equal(a, b), f"max diff {np.abs(a - b).max():.3e}"


@pytest.mark.parametrize("hrtf", [True, False])
def test_streaming_queues_vs_oracle(hrtf):
    """LoadBufferQueue + queue advance: short items (several crossed per window), loop back to
    a middle item, queues that run out (Stopping fade), a start position beyond the first
    item, re-queuing mid-stream, ragged updates; audio AND per-update voice results
    (position, state, buffers_done) must match the oracle."""
    rng = np.random.default_rng(909)
    nv, ir = 20, 64
    desc = synth.hrtf_desc(nv, ir) if hrtf else synth.stereo_desc(nv)
    nbuf = nv * 4
    desc.max_buffers = nbuf
    params, coeffs, dry = synth.voice_set(rng, nv, ir if hrtf else 0, hrtf=hrtf,
                                          dry_channels=desc.dry_channels, pitch_lo=0.4, pitch_hi=3.0)
    lens = [int(x) for x in rng.integers(40, 2500, size=nbuf)]
    for k, p in enumerate(params):
        p.flags &= ~abi.VF_STATIC
        p.flags &= ~abi.VF_LOOPING
        p.position = int(rng.integers(0, 3000)) if k % 5 == 0 else 0
        p.loop_start, p.loop_end = 0, 0

    def queue_of(k, phase):
        ids = [k * 4 + j for j in range(4)]
        if phase == 1:
            ids = ids[::-1][:3]
        loop = abi.NO_LOOP if k % 3 == 0 else (k % 3 - 1)       # none / item 0 / item 1
        return ids, loop

    outs, results = [], []
    for lib in (mixlib.oracle(), mixlib.product()):
        dev = MixDevice(lib, desc)
        if hrtf:
            dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
        else:
            dev.set_ambi_decoder((np.random.default_rng(3).standard_normal((desc.dry_channels, 2)) * 0.5
                                  ).astype(np.float32), None, 0.0)
        for i in range(nbuf):
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i, lens[i]))
        dev.voices_update(params, coeffs if hrtf else None, dry, None)
        for k in range(nv):
            dev.voice_queue(k, *queue_of(k, 0))
        o, rs = [], []
        for u, f in enumerate((1024, 37, 1024, 512, 1024, 1, 1000, 1024, 1024)):
            if u == 3:
                # the application re-queues: a new list from the current item on
                for k in range(1, nv, 4):
                    dev.voice_queue(k, *queue_of(k, 1))
            out, res = dev.render(f, want_results=True)
            o.append(out)
            rs.append([(res[k].position, res[k].position_frac, res[k].flags, res[k].buffers_done)
                       for k in range(nv)])
        dev.close()
        outs.append(np.concatenate(o, axis=1))
        results.append(rs)
    assert results[0] == results[1]
    assert sum(r[3] for upd in results[0] for r in upd) > 10        # items really were consumed
    _check(outs[1], outs[0], "streaming queues")


def test_reverb_parameter_changes_vs_oracle_ragged_updates():
    """ReverbState::update while playing: the reference's own parameter blocks of the cross-fade
    golden (full updates, an in-place one, the old pipeline ringing out and being cleared, a full
    update while the previous fade still runs) replayed with ragged update sizes, so fade counts
    run out mid-way and pipelines are re-entered at odd offsets."""
    fx = golden.load("hrtf_spline_reverb_xfade_v4")
    rng = np.random.default_rng(31337)
    nv, ir = 16, 64
    desc = synth.hrtf_desc(nv, ir)
    desc.num_sends = 1
    desc.wet_channels = 4
    desc.max_slots = 1
    params, coeffs, dry = synth.voice_set(rng, nv, ir)
    send = (rng.standard_normal((nv, 1, 4)) * 0.3).astype(np.float32)
    for p in params:
        p.send_slot[0] = 0
    sizes = (1024, 300, 1024, 17, 1024, 1024, 700, 1024, 1, 1024, 1024, 512, 1024, 1024, 1024, 90, 1024, 1024)
    U = len(sizes)
    assert U == fx["rv_state"].shape[0]
    outs = []
    for lib in (mixlib.oracle(), mixlib.product()):
        dev = MixDevice(lib, desc)
        dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
        for i in range(nv):
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
        dev.slot_reverb(0, abi.reverb_params_from(fx["rv_params"][0].tobytes()), fx["rv_gains"][0])
        dev.voices_update(params, coeffs, dry, send)
        o = []
        for u, f in enumerate(sizes):
            if u > 0:
                st, prev = int(fx["rv_state"][u]), int(fx["rv_state"][u - 1])
                full = (st >> 8) != (prev >> 8)
                if full or not np.array_equal(fx["rv_params"][u], fx["rv_params"][u - 1]) \
                        or not np.array_equal(fx["rv_gains"][u], fx["rv_gains"][u - 1]):
                    dev.slot_reverb_update(0, abi.reverb_params_from(fx["rv_params"][u].tobytes()), full,
                                           fx["rv_gains"][u])
            o.append(dev.render(f))
        dev.close()
        outs.append(np.concatenate(o, axis=1))
    _check(outs[1], outs[0], "reverb parameter changes")


EFX_CASES = {
    "echo": (abi.EFFECT_ECHO, lambda p: (setattr(p.echo, "delay", 0.013), setattr(p.echo, "lr_delay", 0.021),
                                         setattr(p.echo, "feedback", 0.7), setattr(p.echo, "spread", 0.6)),
             lambda p: (setattr(p.echo, "delay", 0.0004), setattr(p.echo, "damping", 0.9))),
    "modulator": (abi.EFFECT_MODULATOR, lambda p: (setattr(p.modulator, "frequency", 523.0),
                                                   setattr(p.modulator, "high_pass_cutoff", 600.0)),
                  lambda p: (setattr(p.modulator, "frequency", 77.0), setattr(p.modulator, "waveform", 2))),
    "equalizer": (abi.EFFECT_EQUALIZER, lambda p: (setattr(p.equalizer, "low_gain", 0.2), setattr(p.equalizer, "mid1_gain", 5.0),
                                                   setattr(p.equalizer, "high_gain", 3.0)),
                  lambda p: (setattr(p.equalizer, "mid2_gain", 0.15), setattr(p.equalizer, "mid2_width", 0.2))),
    "compressor": (abi.EFFECT_COMPRESSOR, lambda p: None, lambda p: setattr(p.compressor, "on_off", 0)),
    "dedicated": (abi.EFFECT_DEDICATED, lambda p: setattr(p.dedicated, "gain", 0.7), lambda p: setattr(p.dedicated, "gain", 0.1)),
    "distortion": (abi.EFFECT_DISTORTION, lambda p: (setattr(p.distortion, "edge", 0.8), setattr(p.distortion, "gain", 0.4)),
                   lambda p: (setattr(p.distortion, "edge", 0.1), setattr(p.distortion, "eq_center", 5000.0))),
    "chorus": (abi.EFFECT_CHORUS, lambda p: (setattr(p.chorus, "waveform", 0), setattr(p.chorus, "rate", 3.3),
                                             setattr(p.chorus, "depth", 0.6), setattr(p.chorus, "feedback", 0.5)),
               lambda p: (setattr(p.chorus, "waveform", 1), setattr(p.chorus, "rate", 0.9), setattr(p.chorus, "phase", -120),
                          setattr(p.chorus, "delay", 0.003), setattr(p.chorus, "feedback", -0.7))),
    "autowah": (abi.EFFECT_AUTOWAH, lambda p: (setattr(p.autowah, "resonance", 200.0), setattr(p.autowah, "peak_gain", 3000.0)),
                lambda p: (setattr(p.autowah, "attack_time", 0.005), setattr(p.autowah, "resonance", 40.0))),
    "fshifter": (abi.EFFECT_FSHIFTER, lambda p: (setattr(p.fshifter, "frequency", 300.0), setattr(p.fshifter, "left_direction", 0),
                                                 setattr(p.fshifter, "right_direction", 1)),
                 lambda p: (setattr(p.fshifter, "frequency", 2500.0), setattr(p.fshifter, "left_direction", 2))),
    "vmorpher": (abi.EFFECT_VMORPHER, lambda p: (setattr(p.vmorpher, "rate", 5.0), setattr(p.vmorpher, "phoneme_a", 0),
                                                 setattr(p.vmorpher, "phoneme_b", 2), setattr(p.vmorpher, "waveform", 1)),
                 lambda p: (setattr(p.vmorpher, "phoneme_a", 3), setattr(p.vmorpher, "phoneme_a_coarse_tuning", 7),
                            setattr(p.vmorpher, "waveform", 0), setattr(p.vmorpher, "rate", 0.7))),
}


@pytest.mark.parametrize("kind", sorted(EFX_CASES))
def test_efx_effects_vs_oracle_ragged_updates(kind):
    """The EFX effects behind b200mix_slot_efx (alc/effects/*.cpp) against the oracle: two slots
    of the effect — one mixing into Dry, one chained into the other (EffectSlotBase::Target) —
    ragged update sizes, a property change (EffectState::update) mid-run."""
    efx_case(kind, *EFX_CASES[kind])


def efx_case(kind, typ, setup, change, product=None, perturb=None):
    """The two-slot chain of `typ` through the C ABI, `product` (default: the CUDA library) against
    the oracle.  `perturb`, if given, changes the send gains the product run uses."""
    rng = np.random.default_rng(300 + typ)
    nv, ir = 12, 64
    desc = synth.hrtf_desc(nv, ir)
    desc.num_sends, desc.wet_channels, desc.max_slots = 1, 4, 2
    params, coeffs, dry = synth.voice_set(rng, nv, ir)
    send = (rng.standard_normal((nv, 1, 4)) * 0.4).astype(np.float32)
    for k, p in enumerate(params):
        p.send_slot[0] = k % 2
    dscale = np.array([1.0, 0.9, 1.1, 0.8], dtype=np.float32)
    dindex = np.array([0, 1, 2, 3], dtype=np.uint32)
    wscale = np.ones(4, dtype=np.float32)
    windex = np.array([0, 1, 2, 3], dtype=np.uint32)
    sizes = (1024, 100, 1024, 7, 640, 1024, 333, 1024)

    def run(lib, send_gains):
        dev = MixDevice(lib, desc)
        dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
        for i in range(nv):
            dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
        props = abi.efx_defaults(typ)
        setup(props)
        dev.slot_target(1, 0)                     # slot 1 feeds slot 0's Wet mix
        dev.slot_efx(0, props, 0.8, dscale, dindex, windex)
        dev.slot_efx(1, props, 0.6, wscale, windex, windex)
        dev.voices_update(params, coeffs, dry, send_gains)
        o = []
        for u, f in enumerate(sizes):
            if u == 4:
                change(props)
                dev.slot_efx(0, props, 0.8, dscale, dindex, windex)
                dev.slot_efx(1, props, 0.5, wscale, windex, windex)
            o.append(dev.render(f))
        dev.close()
        return np.concatenate(o, axis=1)

    ref = run(mixlib.oracle(), send)
    out = run(product() if product else mixlib.product(), perturb(send) if perturb else send)
    # Conditioning: the waveshaper (small-signal gain (1+fc)^3), the high-gain peaking filters and
    # the envelope-driven wah amplify last-bit differences of their INPUT (the send mix sums in a
    # different order on the GPU) by orders of magnitude.  The oracle itself, fed send gains two
    # ulps away, moves by `sens`; the comparison cannot be tighter than a few times that.
    ptb = run(mixlib.oracle(), (send * np.float32(1.0 + 3e-7)).astype(np.float32))
    d = ptb.astype(np.float64) - ref.astype(np.float64)
    sens_rms, sens_max = float(np.sqrt((d ** 2).mean())), float(np.abs(d).max())
    _check(out, ref, f"efx {kind} vs oracle", max(3e-6, 3.0 * sens_rms), max(3e-5, 3.0 * sens_max))
