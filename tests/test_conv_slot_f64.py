"""The convolution slot's float64 model and bound (helpers/convslot.py) without a GPU:

  - the CPU oracle, driven through the same harness (input written into the Wet buffers
    between render_begin and render_end, RealOut read back), sits far inside the bound on the
    ragged, gain and lifecycle schedules for IRs up to 2433 taps;
  - each defect a convolution kernel could have, applied to the model, exceeds the bound by at
    least 10x on the test's own inputs: so the GPU file would catch it;
  - the restated chunk plan reaches every category the GPU file asserts, for 132 and 114 SMs.
"""
import numpy as np
import pytest

from helpers import convslot as cs
from helpers import mixlib

_ORACLE = {f().name: f for f in cs.ORACLE_CASES}


@pytest.mark.parametrize("name", sorted(_ORACLE))
def test_oracle_within_bound(name):
    s = _ORACLE[name]()
    r = cs.check(s, cs.run(s, mixlib.oracle()))
    # the oracle rounds a float64 direct sum to float32 once per line: a few units of 2^-24 S
    assert r <= cs.C_BOUND / 4, r
    print(f"{name}: oracle err/(2^-24 S) = {r:.3f}")


def _sensitivity_case(defect):
    if defect == "drop one chunk":
        # chunk 20 of the 480 000-tap slot on the long case's own plan (48 chunks of 79 segments)
        s = cs.case_long()
        chunks, plans, _ = cs.categories([v for v in s.slot_sets()[0]], 132)
        p = plans[0]
        assert chunks == cs.MAX_CHUNKS and p["segs"] == 3749 and p["clen"] == 79
        s0 = p["starts"][20]
        return [(s, (s0, s0 + p["clen"]))]
    cases = [(cs.case_gains(), None), (cs.case_lengths(max_taps=2433, dry=4), None)]
    if defect == "drop last segment":
        # the last of 3749 segments: the smallest share of a flat IR the GPU file runs
        cases.append((cs.case_long(), None))
    return cases


@pytest.mark.parametrize("defect", cs.DEFECTS)
def test_defect_exceeds_bound_tenfold(defect):
    for s, chunk in _sensitivity_case(defect):
        ref, bound = cs.model(s)
        bad, _ = cs.model(s, defect=defect, chunk=chunk, spot_check=False)
        r = cs.ratio(bad, ref, bound)
        print(f"{s.name}: {defect}: err/(2^-24 S) = {r:.3g} = {r / cs.C_BOUND:.3g} x the bound")
        assert r >= 10 * cs.C_BOUND, (s.name, defect, r)


def test_model_is_exact_on_tagged_impulses():
    """With one tap per segment and unit impulses, every output sample is one tap or a sum of
    a few: the model's float64 answer is exact, and float32 rounding of it is within the bound."""
    s = cs.case_tagged(one_frame_updates=40)
    ref, bound = cs.model(s)
    assert cs.ratio(ref.astype(np.float32), ref, bound) <= 1.0
    # the same output one sample late is far outside
    bad = ref.copy()
    bad[0, 1:] = ref[0, :-1]
    assert cs.ratio(bad, ref, bound) > 1e3 * cs.C_BOUND


@pytest.mark.parametrize("sms", [132, 114])
def test_chunk_plan_categories(sms):
    got = set()
    for f in cs.GPU_CASES:
        for slots in f().slot_sets():
            got |= cs.categories(list(slots), sms)[2]
    assert got == set(cs.CATEGORIES), set(cs.CATEGORIES) - got


def test_chunk_plan_restatement():
    """SlotTable::refresh's numbers for the shapes the GPU file names."""
    # tools/bench_effects.py --effect conv on a 132-SM H100: 32 mono slots of 96 000 taps
    chunks, plans, _ = cs.categories([(cs.nseg(96000), 1)] * 32, 132)
    assert (chunks, plans[0]["clen"], plans[0]["zcnt"], plans[0]["rounds"]) == (17, 45, 17, 5)
    # the previous long-IR test's shape: 20 000 taps x 2 beside 300 and 1153 taps
    chunks, plans, _ = cs.categories([(cs.nseg(20000), 2), (cs.nseg(300), 1), (cs.nseg(1153), 1)], 132)
    assert chunks == 9 and [p["clen"] for p in plans] == [18, 1, 1]
    assert [cs.nseg(t) for t in cs.IR_LENGTHS + (96000, 480000)] == \
        [1, 1, 1, 1, 1, 1, 1, 2, 2, 3, 8, 9, 10, 18, 19, 100, 156, 749, 3749]
    assert cs.conv_chunks([(3749, 2)], 132) == 48 and cs.conv_chunks([(18, 16)], 132) == 1
