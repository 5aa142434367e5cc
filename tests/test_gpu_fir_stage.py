"""-m gpu: the HRIR FIR kernel's staging, through the C ABI against the CPU oracle.

k_hrtf_fir bulk-copies each voice's [History | line] and HRIRs into one of two stage buffers
while the group's previous voice is mixed, and builds the FIR input as a fade region and a
steady ramp.  These scenes reach what that must get right:
  - update sizes that are not a multiple of 4 frames (the last n%4 samples are loaded
    separately), down to 1 and 3 frames;
  - HRTF voices interleaved in the mixing order with non-HRTF voices and with one-shot voices
    that have ended (silent), which the look-ahead to a group's next voice skips;
  - voices with an active direct filter (the line comes from the filtered lines) next to plain
    ones;
  - fades with new HRIRs (the old HRIR is staged too), with new delays only (the old-filter pass
    runs on the target HRIR) and with new gains only (one merged pass);
  - voices that stop (VF_STOPPING) with no new parameters, with new HRIRs (some of them through
    a direct filter), with new delays and with new gains, and the update after, which mixes
    only their carried tails;
  - 40 voices, fewer than the kernel has voice groups (one voice per group, none to look ahead
    to), and 3000, which gives groups two or three order slots on a 132-SM H100;
  - HRIR lengths 8, 40, 64, 72 and 128 (both FIR variants).
tests/test_hrtf_stop.py holds stopping voices to a float64 restatement as well."""
import numpy as np
import pytest

from helpers import mixlib, synth
from helpers.mixlib import MixDevice
from pyb200mix import abi, scene

pytestmark = pytest.mark.gpu

RMS_TOL, MAX_TOL = 1e-6, 1e-5          # relative to the reference block's peak
FRAMES = 6000
NBUF = 64
SIZES = [1023, 3, 1, 517, 1024, 770]


def _copy(p):
    return abi.VoiceParams.from_buffer_copy(bytes(p))


def _render(lib, nv, ir, seed):
    rng = np.random.default_rng(seed)
    params, coeffs, dry = synth.voice_set(rng, nv, ir, hrtf=False, frames=FRAMES)
    hrtf = rng.random(nv) < 0.5
    for k, p in enumerate(params):
        p.buffer = k % NBUF
        if hrtf[k]:
            p.flags |= abi.VF_HRTF
        if k % 9 == 4:                                # one-shot that ends in the first update
            p.flags &= ~abi.VF_LOOPING
            p.position = FRAMES - int(rng.integers(100, 600))
    live = [k for k in range(nv) if k % 9 != 4]
    new_hrir = [k for k in live if k % 5 == 1]
    new_delay = [k for k in live if k % 5 == 2]
    new_gain = [k for k in live if k % 5 == 3]
    filtered = [k for k in live if k % 3 == 0]
    stop_plain = [k for k in live if k % 10 == 4]          # stopped with no new parameters
    stop_hrir = [k for k in live if k % 10 == 9]           # stopped with new HRIRs
    stopping = set(k for k in live if k % 20 in (2, 3))    # stopped with the last new delay / gain
    lp = np.zeros(5, dtype=np.float32)
    hp = np.zeros(5, dtype=np.float32)
    prod = mixlib.product()
    assert prod.biquad_coeffs(0, 5000.0 / 48000.0, 0.35, 1.0, lp.ctypes.data) == 0
    assert prod.biquad_coeffs(1, 250.0 / 48000.0, 1.0, 1.0, hp.ctypes.data) == 0

    desc = synth.hrtf_desc(nv, ir)
    desc.max_buffers = NBUF
    dev = MixDevice(lib, desc)
    dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
    for b in range(NBUF):
        dev.buffer_data(b, abi.FMT_I16, scene.voice_buffer_fast(b, FRAMES))
    dev.voices_update(params, coeffs, dry, None)

    def moved(idx, change, stop=()):
        out = []
        for k in idx:
            q = _copy(params[k])
            q.flags &= ~abi.VF_RESET
            if k in stop:                                 # fades out over this update
                q.flags = (q.flags & ~abi.VF_PLAYING) | abi.VF_STOPPING
            change(q)
            params[k] = q
            out.append(q)
        return out

    def same(q):
        pass

    def delay(q):
        q.hrtf_delay[1] = (q.hrtf_delay[1] + 7) % 64

    def gain(q):
        q.hrtf_gain *= 1.3

    def hrir(q):
        q.hrtf_delay[0] = (q.hrtf_delay[0] + 5) % 64
        q.hrtf_gain *= 0.7

    outs = []
    for u, frames in enumerate(SIZES):
        if u == 1:
            # new HRIRs, delays and gains: 64-sample fades with the old HRIR
            coeffs[new_hrir] = coeffs[new_hrir][:, ::-1, :] * 0.5
            dev.voices_update(moved(new_hrir, hrir), coeffs[new_hrir], dry[new_hrir], None)
            # stopping voices: a 64-sample (or n-sample) fade of the old HRIR to silence
            dev.voices_update(moved(stop_plain, same, stop_plain), None, dry[stop_plain], None)
        if u == 2:
            # same HRIRs: new delays (old-filter pass on the target HRIR), new gains (merged pass)
            dev.voices_update(moved(new_delay, delay), None, dry[new_delay], None)
            dev.voices_update(moved(new_gain, gain), None, dry[new_gain], None)
        if u == 3:
            # direct filters: these lines come from the filtered lines; some fade as well, some
            # stop with new HRIRs (the old HRIR is staged and faded out)
            dev.voices_filters((k, 0, 1, lp, hp) for k in filtered)
            coeffs[new_hrir] = coeffs[new_hrir] * 0.8
            dev.voices_update(moved(new_hrir, hrir), coeffs[new_hrir], dry[new_hrir], None)
            coeffs[stop_hrir] = coeffs[stop_hrir][:, ::-1, :] * 0.9
            dev.voices_update(moved(stop_hrir, hrir, stop_hrir), coeffs[stop_hrir], dry[stop_hrir], None)
        if u == 4:
            # some stop with their new delays or gains; the last update mixes the stopped voices'
            # carried tails only
            dev.voices_update(moved(new_delay, delay, stopping), None, dry[new_delay], None)
            dev.voices_update(moved(new_gain, gain, stopping), None, dry[new_gain], None)
        outs.append(dev.render(frames))
    dev.close()
    return outs


@pytest.mark.parametrize("ir", [8, 40, 64, 72, 128])
@pytest.mark.parametrize("nv", [40, 3000])
def test_fir_stage_vs_oracle(nv, ir):
    seed = 7000 + nv + ir
    # the updates are checked as one block: the 1- and 3-frame ones alone have a peak of a
    # few samples, against which the fp32 re-association of the voices' sums is not small
    got = np.concatenate(_render(mixlib.product(), nv, ir, seed), axis=1)
    ref = np.concatenate(_render(mixlib.oracle(), nv, ir, seed), axis=1)
    peak = float(np.abs(ref).max())
    assert peak > 1e-4, "reference output is silent"
    err = (got.astype(np.float64) - ref.astype(np.float64)) / peak
    rms, mx = float(np.sqrt((err ** 2).mean())), float(np.abs(err).max())
    assert rms <= RMS_TOL and mx <= MAX_TOL, f"nv {nv} ir {ir}: rms {rms:.3e} max {mx:.3e}"
