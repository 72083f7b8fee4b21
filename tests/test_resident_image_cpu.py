"""Device-resident image entry points without a device: exported, argument types declared by ctypes_api, NULL handles
and bad arguments refused before any device work, and no CPU fallback (open returns UHDR_CODEC_ERROR with a CUDA
message)."""
import ctypes as C
import os

import numpy as np
import pytest

import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A

ROOT = T.ROOT
NAMES = ("uhdr_b200_image_open_dev", "uhdr_b200_image_info", "uhdr_b200_image_render_dev", "uhdr_b200_image_release")


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    L = A.declare_resident_image(C.CDLL(T.GPU_SO))
    L.uhdr_b200_last_error.restype = C.c_char_p
    return L


def _apple():
    return np.frombuffer(open(os.path.join(ROOT, "tests", "golden", "apple_gainmap_new.jpg"), "rb").read(), np.uint8).copy()


def test_exported_and_declared(lib):
    for n in NAMES:
        assert hasattr(lib, n), n
        assert getattr(lib, n).argtypes, n


def test_null_handles_and_bad_arguments(lib):
    buf = _apple()
    h = C.c_void_p(99)
    assert lib.uhdr_b200_image_open_dev(buf.ctypes.data, buf.size, 1, None) == 3
    assert lib.uhdr_b200_image_open_dev(None, 0, 1, C.byref(h)) == 3 and not h.value
    for k in (0, 3, 5, 16, -1):
        h = C.c_void_p(99)
        assert lib.uhdr_b200_image_open_dev(buf.ctypes.data, buf.size, k, C.byref(h)) == 3, k
        assert not h.value, k
    d = [C.c_uint() for _ in range(4)]
    assert lib.uhdr_b200_image_info(None, *[C.byref(x) for x in d], None, None) == 3
    px = np.zeros(64 * 8, np.uint8)
    dest = A.raw_image(A.FMT_RGBAF16, -1, -1, -1, 8, 8, [px], [8])
    assert lib.uhdr_b200_image_render_dev(None, A.CT_LINEAR, 4.0, 0, 0, C.byref(dest), None) == 3
    assert lib.uhdr_b200_image_release(None) == 3
    assert b"CUDA" not in lib.uhdr_b200_last_error()
    h = C.c_void_p(99)
    assert lib.uhdr_b200_image_open_dev(buf.ctypes.data, buf.size // 50, 2, C.byref(h)) != 0 and not h.value


def test_open_without_device_is_a_cuda_error(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    buf = _apple()
    for k in (1, 2, 4, 8):
        h = C.c_void_p(99)
        assert lib.uhdr_b200_image_open_dev(buf.ctypes.data, buf.size, k, C.byref(h)) == 1, k
        assert b"CUDA" in lib.uhdr_b200_last_error() and not h.value, k
