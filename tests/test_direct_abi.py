"""The direct-channel entry point of the C ABI as the header and the library present it (no GPU)."""
import ctypes as C
import os
import re

from helpers import mixlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_declares_direct_voices_and_version_1_3():
    text = open(os.path.join(ROOT, "include", "b200mix.h")).read()
    assert re.search(r"B200MIX_VF_DIRECT\s*=\s*1u<<8\b", text)
    assert re.search(r"B200MIX_API int b200mix_voices_update_direct\(b200mix_device \*dev, uint32_t n,\s*"
                     r"const b200mix_voice_params \*params, const float \*real_gains, const float \*send_gains\);",
                     text)
    lib = C.CDLL(mixlib.PRODUCT_SO)
    assert hasattr(lib, "b200mix_voices_update_direct")
    lib.b200mix_version.restype = C.c_uint32
    assert lib.b200mix_version() == (1 << 16) | 3


def test_direct_update_of_no_device_is_refused():
    lib = C.CDLL(mixlib.PRODUCT_SO)
    f = lib.b200mix_voices_update_direct
    f.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    assert f(None, 1, None, None, None) == -1
