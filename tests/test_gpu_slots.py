"""-m gpu: effect slots changed while the device renders.

- A slot change leaves a running convolution alone: calls on OTHER slots (a target set to what it
  already is, disabling a slot that never had an effect, an EFX update with unchanged properties)
  between ragged updates leave RealOut bit-identical to a device that made none of them.
- Disable: from the next update on, a device renders (and launches) what a device that never had
  the slot does.
- Re-install: one slot taken through every kind of effect without a render in between renders (and
  launches) what a fresh device with only the last install does."""
import ctypes as C

import numpy as np
import pytest

from helpers import golden, mixlib, synth
from helpers.mixlib import MixDevice
from pyb200mix import abi, scene

pytestmark = pytest.mark.gpu

SIZES = (1024, 100, 1024, 28, 640, 1024, 1, 255, 1024)
DSCALE = np.array([1.0, 0.9, 1.1, 0.8], dtype=np.float32)
INDEX = np.arange(4, dtype=np.uint32)


def _launches(dev):
    fn = dev.m.lib.b200mix_launch_count
    fn.restype, fn.argtypes = C.c_uint64, [C.c_void_p]
    return fn(dev.h)


def _device(desc, seed=41):
    """A device whose voices send to every slot in turn (send 0)."""
    rng = np.random.default_rng(seed)
    nv, hrtf = desc.max_voices, desc.ir_size > 0
    params, coeffs, dry = synth.voice_set(rng, nv, desc.ir_size, hrtf=hrtf, dry_channels=desc.dry_channels)
    send = (rng.standard_normal((nv, 1, desc.wet_channels)) * 0.3).astype(np.float32)
    for k, p in enumerate(params):
        p.send_slot[0] = k % desc.max_slots
    dev = MixDevice(mixlib.product(), desc)
    if hrtf:
        dev.set_hrtf_decoder(*synth.decoder(np.random.default_rng(7)))
    for i in range(nv):
        dev.buffer_data(i, abi.FMT_I16, scene.voice_buffer_fast(i))
    return dev, (params, coeffs if hrtf else None, dry, send)


def _echo(dev, slot, feedback=0.5):
    props = abi.efx_defaults(abi.EFFECT_ECHO)
    props.echo.delay, props.echo.feedback = 0.013, feedback
    dev.slot_efx(slot, props, 0.7, DSCALE, INDEX, INDEX)
    return props


def _reverb(dev, slot, upmix):
    fx = golden.load("hrtf_bsinc24_reverb_v6")
    params = abi.reverb_params_from(fx["reverb_params"].tobytes())
    params.upmix = upmix
    dev.slot_reverb(slot, params, fx["reverb_gains"])


def _conv(dev, slot, taps=5000):
    rng = np.random.default_rng(0xC0)
    ir = (rng.standard_normal((2, taps)) * np.exp(-np.arange(taps) / (taps / 4.0)) * 0.03).astype(np.float32)
    dev.slot_convolution(slot, ir, (rng.standard_normal((2, 4)) * 0.5).astype(np.float32))


def _render(dev, sizes):
    """RealOut of each update, and the kernels each update launched."""
    out, per = [], []
    for f in sizes:
        before = _launches(dev)
        out.append(dev.render(f))
        per.append(_launches(dev) - before)
    return out, per


def _post_none_desc(slots):
    desc = synth.stereo_desc(32, dry_channels=4)
    desc.real_channels, desc.post_process = 4, abi.POST_NONE
    desc.num_sends, desc.wet_channels, desc.max_slots = 1, 4, slots
    return desc


def test_slot_change_leaves_running_convolution_alone():
    desc = synth.hrtf_desc(24, 64)
    desc.num_sends, desc.wet_channels, desc.max_slots = 1, 4, 3
    outs = []
    for change in (True, False):
        dev, voices = _device(desc)
        _conv(dev, 0)
        props = _echo(dev, 1)                     # slot 2 never gets an effect
        dev.voices_update(*voices)
        o, _ = _render(dev, SIZES[:3])            # 2148 frames: the FIFO holds 100 samples
        if change:
            dev.slot_target(1, abi.NO_SLOT)
            assert dev.m.slot_disable(dev.h, 2) == 0
            dev.slot_efx(1, props, 0.7, DSCALE, INDEX, INDEX)
        o += _render(dev, SIZES[3:])[0]
        dev.close()
        outs.append(np.concatenate(o, axis=1))
    assert np.abs(outs[1]).max() > 1e-4
    assert np.array_equal(outs[0], outs[1])


def test_disable_renders_as_if_the_slot_never_was():
    desc = _post_none_desc(2)
    runs = []
    for had in (True, False):
        dev, voices = _device(desc, seed=43)
        _echo(dev, 0)
        if had:
            _reverb(dev, 1, 0)
        dev.voices_update(*voices)
        _render(dev, SIZES[:3])
        if had:
            assert dev.m.slot_disable(dev.h, 1) == 0
        runs.append(_render(dev, SIZES[3:]))
        dev.close()
    (with_out, with_n), (without_out, without_n) = runs
    assert with_n == without_n
    assert np.abs(np.concatenate(without_out, axis=1)).max() > 1e-4
    for a, b in zip(with_out, without_out):
        assert np.array_equal(a, b)


def test_reinstall_through_every_kind_equals_fresh_install():
    desc = _post_none_desc(1)
    runs = []
    for chain in (True, False):
        dev, voices = _device(desc, seed=47)
        if chain:
            _conv(dev, 0)
            _reverb(dev, 0, 1)
            dev.slot_efx(0, abi.efx_defaults(abi.EFFECT_PSHIFTER), 0.7, DSCALE, INDEX, INDEX)
            _echo(dev, 0)
            _echo(dev, 0, feedback=0.3)           # in place: same delay lines
        _reverb(dev, 0, 0)
        dev.voices_update(*voices)
        runs.append(_render(dev, SIZES))
        dev.close()
    (chain_out, chain_n), (fresh_out, fresh_n) = runs
    assert chain_n == fresh_n
    assert np.abs(np.concatenate(fresh_out, axis=1)).max() > 1e-4
    for a, b in zip(chain_out, fresh_out):
        assert np.array_equal(a, b)
