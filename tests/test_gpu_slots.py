"""-m gpu: effect slots changed while the device renders.

- A slot change leaves a running convolution alone: calls on OTHER slots (a target set to what it
  already is, disabling a slot that never had an effect, an EFX update with unchanged properties)
  between ragged updates leave RealOut bit-identical to a device that made none of them.
- Disable: from the next update on, a device renders (and launches) what a device that never had
  the slot does.
- Re-install: one slot taken through every kind of effect without a render in between renders (and
  launches) what a fresh device with only the last install does.
- A refused slot call changes nothing: after it, the device renders (and launches) what its twin that
  never made the call does, and it reports the refusal's code and message."""
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


ERR_INVALID = -1


def _reverb_params(**changes):
    fx = golden.load("hrtf_bsinc24_reverb_v6")
    params = abi.reverb_params_from(fx["reverb_params"].tobytes())
    for k, v in changes.items():
        setattr(params, k, v)
    params.struct_size = C.sizeof(abi.ReverbParams)
    return params, fx["reverb_gains"]


def _raw_efx(dev, slot, out_channels=4, struct_size=None):
    """b200mix_slot_efx with an echo and maps of `out_channels` outputs; its return code."""
    props = abi.efx_defaults(abi.EFFECT_ECHO)
    props.struct_size = C.sizeof(abi.EfxProps) if struct_size is None else struct_size
    scale, index = np.ones(out_channels, dtype=np.float32), np.arange(out_channels, dtype=np.uint32)
    t = abi.EfxTarget()
    t.struct_size, t.sample_rate, t.slot_gain = C.sizeof(abi.EfxTarget), dev.desc.sample_rate, 0.7
    t.out_channels, t.out_scale, t.out_index = out_channels, scale.ctypes.data, index.ctypes.data
    t.wet_channels, t.wet_index = len(INDEX), INDEX.ctypes.data
    t.real_center, t.real_lfe, t.device_ambi_order = abi.NO_SLOT, abi.NO_SLOT, 1
    return dev.m.slot_efx(dev.h, slot, C.byref(props), C.byref(t))


def _raw_gains(dev, slot, lines):
    g = np.ones((lines, 4), dtype=np.float32)
    return dev.m.slot_output_gains(dev.h, slot, lines, g.ctypes.data)


# (call, the refusal's message); slots: 0 convolution, 1 reverb mid-fade, 2 echo into slot 1, 3 empty
REFUSED = {
    "disable_out_of_range": (lambda dev: dev.m.slot_disable(dev.h, 4), "slot_disable: bad slot"),
    "convolution_17_channels": (
        lambda dev: dev.m.slot_convolution(dev.h, 0, 17, 64, np.ones((17, 64), dtype=np.float32).ctypes.data),
        "slot_convolution: bad arguments (or the device has no sends/slots)"),
    "reverb_line_not_pow2": (
        lambda dev: dev.m.slot_reverb(dev.h, 1, C.byref(_reverb_params(late_len=3000)[0])),
        "slot_reverb: line lengths must be powers of two, feedback delays non-zero"),
    "reverb_update_other_lengths": (
        lambda dev: dev.m.slot_reverb_update(dev.h, 1, C.byref(_reverb_params(main_len=65536)[0]), 1),
        "slot_reverb_update: line lengths differ from the installed ones"),
    "reverb_update_on_echo": (
        lambda dev: dev.m.slot_reverb_update(dev.h, 2, C.byref(_reverb_params()[0]), 0),
        "slot_reverb_update: no reverb installed on this slot / bad arguments"),
    "efx_maps_mismatch": (lambda dev: _raw_efx(dev, 2, out_channels=3),
                          "slot_efx: the target maps do not match the device's wet / output mix"),
    "efx_struct_size": (lambda dev: _raw_efx(dev, 2, struct_size=C.sizeof(abi.EfxProps) - 4),
                        "slot_efx: bad arguments (or the device has no sends/slots)"),
    "target_loop": (lambda dev: dev.m.slot_target(dev.h, 1, 2), "slot_target: the chain would loop"),
    "output_gains_line_count": (lambda dev: _raw_gains(dev, 1, 7), "slot_output_gains: wrong line count"),
    "output_gains_empty_slot": (lambda dev: _raw_gains(dev, 3, 2), "slot_output_gains: bad arguments"),
}


@pytest.mark.parametrize("case", sorted(REFUSED))
def test_rejected_slot_call_changes_nothing(case):
    call, message = REFUSED[case]
    desc = _post_none_desc(4)
    runs = []
    for refuse in (True, False):
        dev, voices = _device(desc, seed=53)
        _conv(dev, 0)                              # 5000 taps
        _reverb(dev, 1, 0)
        dev.slot_target(2, 1)
        _echo(dev, 2)
        dev.voices_update(*voices)
        _render(dev, (512,))
        params, gains = _reverb_params(fade_samples=4000)
        dev.slot_reverb_update(1, params, True, gains)
        _render(dev, (700,))                       # the reverb is mid-fade
        if refuse:
            assert call(dev) == ERR_INVALID
            assert dev.last_error() == message
        runs.append(_render(dev, SIZES[1:6]))
        dev.close()
    (refused_out, refused_n), (twin_out, twin_n) = runs
    assert refused_n == twin_n
    assert np.abs(np.concatenate(twin_out, axis=1)).max() > 1e-4
    for a, b in zip(refused_out, twin_out):
        assert a.tobytes() == b.tobytes()
