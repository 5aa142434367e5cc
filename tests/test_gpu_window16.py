"""-m gpu: the bsinc resampler's 16-bit window, through the C ABI against the CPU oracle.

The resample kernel builds the two 16-bit window copies straight from an int16 span that a bulk
copy staged.  These scenes reach the cases that path must get right: spans at every 16-byte lead
(0..7) with even and odd window origins, negative start positions (leading zeros), one-run and
wrapping loop spans, a buffer that ends inside the window, pitches that need two chunks,
bsinc12/24/48 and fast bsinc.  The lines go through the HRIR FIR at sizes from 8 to 128 (both FIR
variants), with coefficient changes mid-run (the old-filter pass), gain fades and voices that stop
(VF_STOPPING) with and without new HRIRs, and the update after the stops."""
import numpy as np
import pytest

from helpers import mixlib, synth
from helpers.mixlib import MixDevice
from pyb200mix import abi, scene

pytestmark = pytest.mark.gpu

RMS_TOL, MAX_TOL = 1e-6, 1e-5          # relative to the reference block's peak
NV = 80
FRAMES = 6000
RESAMPLERS = [abi.RS_BSINC12, abi.RS_BSINC24, abi.RS_BSINC48,
              abi.RS_FAST_BSINC12, abi.RS_FAST_BSINC24, abi.RS_FAST_BSINC48]


def _voices(rng, ir):
    params, coeffs, dry = synth.voice_set(rng, NV, ir, resampler=RESAMPLERS, frames=FRAMES)
    for i, p in enumerate(params):
        kind = i % 5
        lead = i % 8                                   # buffers start 16-byte aligned
        pitch = float(rng.uniform(0.6, 2.4))           # above ~1.27 an update takes two chunks
        p.step = int(pitch * 65536.0)
        p.position_frac = int(rng.integers(0, 65536))
        p.loop_start, p.loop_end = 0, FRAMES
        if kind == 0:                                  # one-run span, loop far ahead
            p.position = 1000 + 8 * int(rng.integers(0, 200)) + lead
        elif kind == 1:                                # the loop wraps inside the window
            p.position = 2000 + lead
            p.loop_start, p.loop_end = 96 + int(rng.integers(0, 8)), 2000 + lead + int(rng.integers(40, 900))
        elif kind == 2:                                # not looping: the buffer ends in the window
            p.flags &= ~abi.VF_LOOPING
            p.position = FRAMES - 8 * int(rng.integers(20, 120)) - lead
        elif kind == 3:                                # starts later: leading zeros (srcDelay)
            p.position = -int(rng.integers(1, 1400))
        else:                                          # not looping, span well inside
            p.flags &= ~abi.VF_LOOPING
            p.position = 8 * int(rng.integers(0, 300)) + lead
    return params, coeffs, dry


def _render(lib, ir, seed):
    rng = np.random.default_rng(seed)
    params, coeffs, dry = _voices(rng, ir)
    moved = list(range(0, NV, 3))
    stopped = list(range(1, NV, 3))
    new_coeffs = coeffs.copy()
    new_coeffs[moved] = coeffs[moved][:, ::-1, :] * 0.5
    dev = MixDevice(lib, synth.hrtf_desc(NV, ir))
    dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
    for i in range(NV):
        dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i, FRAMES))
    dev.voices_update(params, coeffs, dry, None)
    outs = []
    for u in range(3):
        if u == 1:
            # new HRIRs, delays and gains without a reset: 64-sample fades, old-filter pass;
            # every other one of these stops as well (its old HRIR fades out)
            upd = []
            for k in moved:
                p = params[k]
                p.flags &= ~abi.VF_RESET
                if k % 2:
                    p.flags = (p.flags & ~abi.VF_PLAYING) | abi.VF_STOPPING
                p.hrtf_delay[0] = (p.hrtf_delay[0] + 5) % 64
                p.hrtf_gain *= 0.7
                upd.append(p)
            dev.voices_update(upd, new_coeffs[moved], dry[moved], None)
            # stopped with no new parameters
            upd = []
            for k in stopped:
                p = params[k]
                p.flags = (p.flags & ~(abi.VF_RESET | abi.VF_PLAYING)) | abi.VF_STOPPING
                upd.append(p)
            dev.voices_update(upd, None, dry[stopped], None)
        # u == 2: the stopped voices leave only their carried tails
        outs.append(dev.render(1024))
    dev.close()
    return outs


@pytest.mark.parametrize("ir", [8, 40, 64, 72, 100, 128])
def test_window16_vs_oracle(ir):
    seed = 1000 + ir
    got = _render(mixlib.product(), ir, seed)
    ref = _render(mixlib.oracle(), ir, seed)
    for u, (o, r) in enumerate(zip(got, ref)):
        peak = float(np.abs(r).max())
        assert peak > 1e-4, f"update {u}: reference output is silent"
        err = (o.astype(np.float64) - r.astype(np.float64)) / peak
        rms, mx = float(np.sqrt((err ** 2).mean())), float(np.abs(err).max())
        assert rms <= RMS_TOL and mx <= MAX_TOL, f"ir {ir} update {u}: rms {rms:.3e} max {mx:.3e}"
