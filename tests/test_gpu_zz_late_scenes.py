"""Drop-in scenes of higher-order B-Format beds (tests/test_gpu_dropin.py's
comparison, libopenal_b200.so + libb200mix.so against the stock reference): second- / third-order
B-Format beds (AL_SOFT_bformat_hoa) on first-order devices, and beds up to fourth order on
ALC_BFORMAT3D_SOFT devices of order 2 / 3 (the reference's AmbiRotator turning them).  The CPU half of the same scenes —
the patched reference driving the oracle behind the ABI — is green in tests/test_seam_cpu.py; the
file sorts last so that under `pytest -x` it cannot hide validated tests."""
import pytest

import test_gpu_dropin as dropin


@pytest.mark.gpu
@pytest.mark.parametrize("voices,updates,hrtf,fx", [(12, 6, 1, "hoa"), (12, 6, 0, "hoa"), (12, 6, 0, "hoadev2"), (12, 6, 0, "hoadev3")])
def test_late_scenes_render_through_libb200mix(voices, updates, hrtf, fx, tmp_path):
    dropin.test_patched_reference_renders_through_libb200mix(voices, updates, hrtf, fx, tmp_path)
