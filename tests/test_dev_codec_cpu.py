"""No-GPU checks of the whole-file device codec entry points (uhdr_b200_decode_dev, uhdr_b200_encode_dev,
uhdr_b200_jpeg_encode_dev): exported, descriptors checked before any device work, and without a device a loud
CUDA error rather than a fallback."""
import ctypes as C
import os

import numpy as np
import pytest

import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("uhdr_b200_decode_dev", "uhdr_b200_encode_dev", "uhdr_b200_jpeg_encode_dev")


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    L = C.CDLL(T.GPU_SO)
    L.uhdr_b200_decode_dev.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p]
    L.uhdr_b200_encode_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p,
                                       C.c_size_t, C.c_void_p, C.c_void_p]
    L.uhdr_b200_jpeg_encode_dev.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                            C.c_void_p, C.c_void_p]
    L.uhdr_b200_last_error.restype = C.c_char_p
    return L


def _file():
    return open(os.path.join(ROOT, "tests", "golden", "apple_gainmap_new.jpg"), "rb").read()


def _size(lib, data):
    T.UhdrApi(lib)
    dec = C.c_void_p(lib.uhdr_create_decoder())
    buf = np.frombuffer(data, np.uint8).copy()
    ci = A.CompressedImage(buf.ctypes.data, len(data), len(data), -1, -1, -1)
    assert lib.uhdr_dec_set_image(dec, C.byref(ci)).error_code == 0
    assert lib.uhdr_dec_probe(dec).error_code == 0
    r = (lib.uhdr_dec_get_image_width(dec), lib.uhdr_dec_get_image_height(dec),
         lib.uhdr_dec_get_gainmap_width(dec), lib.uhdr_dec_get_gainmap_height(dec))
    lib.uhdr_release_decoder(dec)
    return r


class Args:
    """well-formed arguments of the three calls; the plane pointers are host memory, so they only pass the checks
    that come before the device is needed"""

    def __init__(self, lib):
        data = _file()
        self.data = np.frombuffer(data, np.uint8).copy()
        w, h, gw, gh = _size(lib, data)
        self.px = np.zeros(w * h * 8, np.uint8)
        self.gm = np.zeros(gw * gh * 4, np.uint8)
        self.dest = A.raw_image(A.FMT_RGBAF16, -1, -1, -1, w, h, [self.px], [w])
        self.gdesc = A.raw_image(-1, -1, -1, -1, gw, gh, [self.gm], [gw])
        self.md = A.GainmapMetadata()
        ew, eh = 64, 32
        self.hb, self.sb = T.make_p010(ew, eh), T.make_yuv420(ew, eh)
        self.hdr, self.k1 = A.p010_image(self.hb, ew, eh, A.CG_BT2100, A.CT_HLG, A.CR_LIMITED)
        self.sdr, self.k2 = A.yuv420_image(self.sb, ew, eh, A.CG_BT709)
        self.cfg = A.default_gm_config()
        self.out = np.zeros(1 << 20, np.uint8)
        self.n = C.c_size_t()

    def decode(self, lib, ct=A.CT_LINEAR, size=None, dest=None):
        return lib.uhdr_b200_decode_dev(self.data.ctypes.data, self.data.size if size is None else size, ct, A.FLT_MAX,
                                        C.byref(dest or self.dest), C.byref(self.gdesc), C.byref(self.md), None)

    def encode(self, lib, hdr=None, sdr=None, q=95):
        return lib.uhdr_b200_encode_dev(C.byref(hdr or self.hdr), C.byref(sdr or self.sdr), C.byref(self.cfg), q, None, 0,
                                        self.out.ctypes.data, self.out.size, C.byref(self.n), None)

    def jpeg(self, lib, img=None):
        return lib.uhdr_b200_jpeg_encode_dev(C.byref(img or self.sdr), 90, None, 0, self.out.ctypes.data, self.out.size,
                                             C.byref(self.n), None)


def test_exported(lib):
    assert all(hasattr(lib, n) for n in NAMES)


def test_bad_descriptors_are_invalid_param(lib):
    a = Args(lib)
    assert lib.uhdr_b200_decode_dev(None, 0, A.CT_LINEAR, A.FLT_MAX, C.byref(a.dest), None, None, None) == 3
    assert lib.uhdr_b200_decode_dev(a.data.ctypes.data, a.data.size, A.CT_LINEAR, A.FLT_MAX, None, None, None, None) == 3
    assert a.decode(lib, ct=A.CT_HLG) == 3                  # RGBA half float wants LINEAR
    wrong = A.RawImage.from_buffer_copy(a.dest)
    wrong.w -= 2
    assert a.decode(lib, dest=wrong) == 3                    # not the primary image's size
    pitch = A.RawImage.from_buffer_copy(a.dest)
    pitch.stride[0] = pitch.w - 1
    assert a.decode(lib, dest=pitch) == 3
    null = A.RawImage.from_buffer_copy(a.dest)
    null.planes[0] = None
    assert a.decode(lib, dest=null) == 3
    odd = A.RawImage.from_buffer_copy(a.dest)
    odd.planes[0] = a.px.ctypes.data + 2                      # a half-float pixel is 8 bytes
    assert a.decode(lib, dest=odd) == 3
    assert lib.uhdr_b200_encode_dev(None, None, C.byref(a.cfg), 95, None, 0, a.out.ctypes.data, a.out.size,
                                    C.byref(a.n), None) == 3
    bad = A.RawImage.from_buffer_copy(a.hdr)
    bad.ct = A.CT_SRGB
    assert a.encode(lib, hdr=bad) == 3
    small = A.RawImage.from_buffer_copy(a.sdr)
    small.w, small.h = 32, 16
    assert a.encode(lib, sdr=small) == 3                      # resolutions mismatch
    assert a.encode(lib, q=101) == 3
    for field, value in (("min_content_boost", 0.0), ("max_content_boost", float("inf")), ("target_disp_peak_nits", 100.0),
                         ("gamma", -1.0), ("scale_factor", 129), ("preset", 7)):
        a.cfg = A.default_gm_config(**{field: value})
        assert a.encode(lib) == 3, field
    a.cfg = A.default_gm_config(min_content_boost=4.0, max_content_boost=2.0)
    assert a.encode(lib) == 3
    a.cfg = A.default_gm_config()
    assert lib.uhdr_b200_jpeg_encode_dev(None, 90, None, 0, a.out.ctypes.data, a.out.size, C.byref(a.n), None) == 3
    nop = A.RawImage.from_buffer_copy(a.sdr)
    nop.planes[1] = None
    assert a.jpeg(lib, nop) == 3
    assert b"CUDA" not in lib.uhdr_b200_last_error()


def test_truncated_file_gives_the_uhdr_decode_code(lib):
    a = Args(lib)
    T.UhdrApi(lib)
    dec = C.c_void_p(lib.uhdr_create_decoder())
    cut = bytes(a.data[:a.data.size // 3])
    buf = np.frombuffer(cut, np.uint8).copy()
    ci = A.CompressedImage(buf.ctypes.data, len(cut), len(cut), -1, -1, -1)
    assert lib.uhdr_dec_set_image(dec, C.byref(ci)).error_code == 0
    want = lib.uhdr_decode(dec).error_code
    lib.uhdr_release_decoder(dec)
    assert want != 0 and a.decode(lib, size=len(cut)) == want


def test_no_cpu_fallback(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    a = Args(lib)
    for call in (a.decode, a.encode, a.jpeg):
        assert call(lib) == 1, call
        assert b"CUDA" in lib.uhdr_b200_last_error()
