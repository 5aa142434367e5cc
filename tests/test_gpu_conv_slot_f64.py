"""-m gpu: the convolution slot (k_conv_input, k_conv_mac, k_conv_ifft, k_conv_output, then
k_slot_output_mix / k_slot_target_mix) in isolation against the float64 model of
helpers/convslot.py, per output sample within C_BOUND * 2^-24 * S.

The device has no voices and no post-process; each convolution slot's input is written into its
wet channel 0 between render_begin and render_end, with loud noise in the wet channels it must
ignore, and RealOut (= the Dry mix) is read back.  The cases cover every IR length edge around the
128-sample block and the 9- and 18-segment boundaries up to 480 000 taps, IR channels 1-16, Dry
mixes of 4, 16 and 32 channels, update sizes 1-1024 (runs of 1-frame updates, 128 consecutive
1023-frame updates), ring wraps, gains changed every update, re-installs, disables and a
convolution slot feeding another.  The chunk plan of k_conv_mac depends on the SM count and on
which slots are installed together; test_chunk_plan_reaches_every_category checks that these
cases reach every kind of plan on the device in hand.
"""
import numpy as np
import pytest

from helpers import convslot as cs
from helpers import mixlib

pytestmark = pytest.mark.gpu

_CASES = {f.__name__: f for f in cs.GPU_CASES}


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_chunk_plan_reaches_every_category():
    sms = _sms()
    got = set()
    for f in cs.GPU_CASES:
        s = f()
        for slots in s.slot_sets():
            chunks, plans, cats = cs.categories(list(slots), sms)
            got |= cats
            print(f"{sms} SMs: {s.name}: conv_chunks {chunks}, (segs, clen, zcnt, rounds) "
                  + " ".join(f"({p['segs']},{p['clen']},{p['zcnt']},{p['rounds']})" for p in plans))
    assert got == set(cs.CATEGORIES), set(cs.CATEGORIES) - got


@pytest.mark.parametrize("case", sorted(_CASES))
def test_conv_slot_vs_f64(case):
    s = _CASES[case]()
    out = cs.run(s, mixlib.product())
    r = cs.check(s, out)
    assert np.isfinite(out).all()
    print(f"{s.name}: {s.frames} frames, err/(2^-24 S) = {r:.3f} (C = {cs.C_BOUND:g})")
