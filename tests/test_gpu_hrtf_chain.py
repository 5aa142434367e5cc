"""-m gpu: the HRTF update's kernel chain, through the C ABI against the CPU oracle.

On an HRTF device an update runs k_mix_voices (resample and park) -> k_hrtf_fir (one partial
row per CTA) -> k_post_hrtf_reduce, which sums the rows with k_reduce_rows' fixed tree and
finishes the HRTF post-mix (carry, decoder FIR of the band-split dry channels, RealOut L/R) in
the same kernel.  The FIR and the post-process are launched as programmatic dependents of the
kernel before them when nothing else is enqueued in between.  These scenes reach:
  - HRTF-only scenes, and scenes with a live dry mix (k_post_hrtf_split and the decoder FIR);
  - update sizes 1, 3, 64, 65, 1000 and 1024 in a row, so the accumulator carry crosses
    updates of every shape, and the post-process' tiles end mid-tile;
  - HRIR lengths 8, 64 and 128 (both FIR variants);
  - direct filters on (k_filters runs between the resample kernel and the FIR, which is then
    launched as an ordinary kernel);
  - profile levels 0, 1 and 2 (events between the kernels of the chain);
  - b200mix_render_device, and b200mix_render into host buffers.
1200 voices give the FIR its full grid on a 132-SM H100 (528 rows, more than the reduce's 128
row segments)."""
import ctypes as C
import functools

import numpy as np
import pytest

from helpers import mixlib, synth
from helpers.mixlib import MixDevice
from pyb200mix import abi, scene

pytestmark = pytest.mark.gpu

RMS_TOL, MAX_TOL = 1e-6, 1e-5          # relative to the reference block's peak
# HRTF-only scenes: no decoder signal adds to the peak, and the fp32 re-association of 1200
# voices' FIR sums alone measures up to 1.9e-6 RMS / 1.6e-5 max of the peak at HRIR length 128
# on an H100, the same to the bit with a separate row-sum kernel before the post-mix
RMS_TOL_HRTF, MAX_TOL_HRTF = 3e-6, 3e-5
NV = 1200
FRAMES = 6000
NBUF = 64
SIZES = [1, 3, 64, 65, 1000, 1024]


def _prod_fn(name, restype, argtypes):
    fn = getattr(mixlib.product().lib, name)
    fn.restype, fn.argtypes = restype, argtypes
    return fn


def _device_out(dev, frames):
    """b200mix_render_device, then RealOut [real_channels][frames] copied from the device."""
    import torch
    ptr = C.c_void_p()
    render_device = _prod_fn("b200mix_render_device", C.c_int,
                             [C.c_void_p, C.c_uint32, C.POINTER(C.c_void_p)])
    assert render_device(dev.h, frames, C.byref(ptr)) == 0, dev.last_error()
    ch = dev.desc.real_channels
    torch.cuda.synchronize()                 # the update ran on the mixer's own stream

    class _Block:
        __cuda_array_interface__ = {"shape": (ch, abi.LINE), "typestr": "<f4",
                                    "data": (ptr.value, False), "strides": None, "version": 2}
    out = torch.as_tensor(_Block(), device="cuda").cpu().numpy()
    return out[:, :frames].copy()


def _render(lib, ir, dry_live, filters, level=1, device_out=False, seed=0):
    rng = np.random.default_rng(9100 + ir + 7*dry_live + 13*filters + seed)
    params, coeffs, dry = synth.voice_set(rng, NV, ir, hrtf=False, frames=FRAMES)
    for k, p in enumerate(params):
        p.buffer = k % NBUF
        if not dry_live or k % 3 != 1:
            p.flags |= abi.VF_HRTF
    desc = synth.hrtf_desc(NV, ir)
    desc.max_buffers = NBUF
    dev = MixDevice(lib, desc)
    if lib is mixlib.product():
        assert _prod_fn("b200mix_profile", C.c_int, [C.c_void_p, C.c_int])(dev.h, level) == 0
    dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
    for b in range(NBUF):
        dev.buffer_data(b, abi.FMT_I16, scene.voice_buffer_fast(b, FRAMES))
    dev.voices_update(params, coeffs, dry, None)
    if filters:
        lp = np.zeros(5, dtype=np.float32)
        hp = np.zeros(5, dtype=np.float32)
        prod = mixlib.product()
        assert prod.biquad_coeffs(0, 5000.0 / 48000.0, 0.35, 1.0, lp.ctypes.data) == 0
        assert prod.biquad_coeffs(1, 250.0 / 48000.0, 1.0, 1.0, hp.ctypes.data) == 0
        dev.voices_filters((k, 0, 1, lp, hp) for k in range(0, NV, 4))
    outs = []
    for u, frames in enumerate(SIZES):
        if u == 3:
            # new gains on a third of the voices: the FIR's fades run in the 65-frame update
            moved = []
            for k in range(0, NV, 3):
                q = abi.VoiceParams.from_buffer_copy(bytes(params[k]))
                q.flags &= ~abi.VF_RESET
                q.hrtf_gain *= 0.6
                params[k] = q
                moved.append(q)
            dev.voices_update(moved, None, dry[0:NV:3], None)
        if device_out and lib is mixlib.product():
            outs.append(_device_out(dev, frames))
        else:
            outs.append(dev.render(frames))
    dev.close()
    return np.concatenate(outs, axis=1)


@functools.lru_cache(maxsize=None)
def _oracle(ir, dry_live, filters):
    return _render(mixlib.oracle(), ir, dry_live, filters)


def _check(got, ref, what, dry_live):
    peak = float(np.abs(ref).max())
    assert peak > 1e-4, "reference output is silent"
    err = (got.astype(np.float64) - ref.astype(np.float64)) / peak
    rms, mx = float(np.sqrt((err ** 2).mean())), float(np.abs(err).max())
    rtol, mtol = (RMS_TOL, MAX_TOL) if dry_live else (RMS_TOL_HRTF, MAX_TOL_HRTF)
    assert rms <= rtol and mx <= mtol, f"{what}: rms {rms:.3e} max {mx:.3e}"


@pytest.mark.parametrize("dry_live", [False, True], ids=["hrtf_only", "dry_live"])
@pytest.mark.parametrize("ir", [8, 64, 128])
def test_chain_vs_oracle(ir, dry_live):
    _check(_render(mixlib.product(), ir, dry_live, False), _oracle(ir, dry_live, False),
           f"ir {ir} dry_live {dry_live}", dry_live)


@pytest.mark.parametrize("dry_live", [False, True], ids=["hrtf_only", "dry_live"])
def test_chain_direct_filters_vs_oracle(dry_live):
    _check(_render(mixlib.product(), 64, dry_live, True), _oracle(64, dry_live, True),
           f"filters dry_live {dry_live}", dry_live)


@pytest.mark.parametrize("device_out", [False, True], ids=["render", "render_device"])
@pytest.mark.parametrize("level", [0, 1, 2])
def test_chain_profile_levels_vs_oracle(level, device_out):
    ref = _oracle(64, True, False)
    got = _render(mixlib.product(), 64, True, False, level=level, device_out=device_out)
    _check(got, ref, f"profile {level} device_out {device_out}", True)
    # the events between the kernels change nothing: bit-identical to the level-1 host render
    assert np.array_equal(got, _render(mixlib.product(), 64, True, False))


def test_hrtf_update_launches():
    """An HRTF-only update with no parameter changes is three kernels: resample, HRIR FIR and
    the post-process with the FIR rows' sum folded in."""
    rng = np.random.default_rng(11)
    params, coeffs, dry = synth.voice_set(rng, 256, 64)
    dev = MixDevice(mixlib.product(), synth.hrtf_desc(256, 64))
    dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
    for i in range(256):
        dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
    dev.voices_update(params, coeffs, dry, None)
    count = _prod_fn("b200mix_launch_count", C.c_uint64, [C.c_void_p])
    dev.render(1024)
    per = []
    for frames in (1024, 65, 1024):
        before = count(dev.h)
        dev.render(frames)
        per.append(count(dev.h) - before)
    dev.close()
    assert per == [3, 3, 3], per
