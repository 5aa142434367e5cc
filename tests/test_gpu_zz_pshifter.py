"""The pitch shifter (PshifterState, alc/effects/pshifter.cpp; k_efx_pshift) through the C ABI on
the GPU: the two fixtures rendered by the compiled reference, and two slots (one chained into the
other) against the oracle with ragged update sizes and a re-tune mid-run.

The kernel's frame arithmetic (csrc/pshift.hpp) is held to the oracle bit for bit on the host
(tests/test_pshift_host.py) and the oracle to the reference (tests/test_oracle_golden.py).  The file
sorts last so that under `pytest -x` it cannot hide the other GPU tests."""
import numpy as np
import pytest

from helpers import golden, mixlib
from pyb200mix import abi
import test_gpu_parity as parity


@pytest.mark.gpu
@pytest.mark.parametrize("name", golden.LATE)
def test_pitch_shifter_golden_vectors_from_reference(name):
    parity.golden_case(name)


PSHIFT_CASES = {
    "up": (abi.EFFECT_PSHIFTER, lambda p: (setattr(p.pshifter, "coarse_tune", 7), setattr(p.pshifter, "fine_tune", 30)),
           lambda p: (setattr(p.pshifter, "coarse_tune", 12), setattr(p.pshifter, "fine_tune", 0))),
    "down": (abi.EFFECT_PSHIFTER, lambda p: (setattr(p.pshifter, "coarse_tune", -4), setattr(p.pshifter, "fine_tune", -30)),
             lambda p: (setattr(p.pshifter, "coarse_tune", -12), setattr(p.pshifter, "fine_tune", 0))),
}


@pytest.mark.gpu
@pytest.mark.parametrize("kind", sorted(PSHIFT_CASES))
def test_pitch_shifter_vs_oracle_ragged_updates(kind):
    parity.efx_case("pshifter " + kind, *PSHIFT_CASES[kind])


@pytest.mark.parametrize("kind", sorted(PSHIFT_CASES))
def test_pitch_shifter_scene_is_audible_and_well_conditioned(kind):
    """No GPU: the scene of the test above run on the oracle against itself with ONE voice's send
    gains moved by one ulp, for every voice, inside the same bound the GPU comparison uses.  The
    shifter picks the dominant analysis bin per synthesis bin, a discontinuous choice: in a scene with
    a near-tie, summing the sends in another order (as the GPU does) legitimately flips it, and the
    comparison with the oracle would then measure the tie, not the kernel."""
    def nudge(v):
        def f(send):
            s = send.copy()
            s[v] = np.nextafter(s[v], np.float32(np.inf))
            return s
        return f
    for v in range(12):
        parity.efx_case("pshifter " + kind, *PSHIFT_CASES[kind], product=mixlib.oracle, perturb=nudge(v))
