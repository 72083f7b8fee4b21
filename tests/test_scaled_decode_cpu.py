"""Reduced-size decoding (1/2, 1/4, 1/8) without a GPU: the C restatement (oracle/jpeg_scaled_oracle.c) pinned bit for
bit to the real libjpeg-turbo decoding with scale_denom = k (oracle/jpeg_scaled_ref.c), over gray / 4:4:4 / 4:2:0
(and the 4:2:2 geometry) streams written by Pillow; the exported entry points, their argument checks, and a loud CUDA
error instead of a CPU fallback."""
import ctypes as C
import os

import numpy as np
import pytest

import scaled_testlib as S
import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A

pytest.importorskip("PIL.Image")

ROOT = T.ROOT
SMALL = [(1, 1), (7, 9), (17, 33)]


@pytest.fixture(scope="module")
def harness():
    if not S.have_harness():
        pytest.skip("no libjpeg-turbo binary to build the harness against")
    return S


def _same(data, k, case):
    info, ref = S.harness_decode(data, k)
    g, mine = S.oracle_scaled(data, k)
    assert info[0:2] == g[0:2], (case, info, g)
    for c in range(info[2]):
        assert info[4 + 3 * c:7 + 3 * c] == g[2 + 3 * c:5 + 3 * c], (case, c, info, g)
        assert (ref[c] == mine[c]).all(), (case, c, int((ref[c] != mine[c]).sum()))
    return info


@pytest.mark.parametrize("layout", ["gray", "444", "420"])
@pytest.mark.parametrize("w,h", SMALL)
def test_restatement_every_quality_small(harness, layout, w, h):
    for q in range(1, 101):
        data = S.pil_jpeg(S.image(w, h, "noise" if q % 2 else "smooth", seed=q), q, layout)
        for k in S.SCALES:
            _same(data, k, (layout, w, h, q, k))


@pytest.mark.parametrize("layout", ["gray", "444", "420"])
@pytest.mark.parametrize("w,h", [(1000, 722), (4080, 3072)])
def test_restatement_large(harness, layout, w, h):
    qs = (1, 10, 50, 75, 90, 95, 100) if w < 2000 else (5, 95)
    for q in qs:
        data = S.pil_jpeg(S.image(w, h, "noise" if q < 50 else "smooth", seed=q), q, layout)
        for k in S.SCALES:
            _same(data, k, (layout, w, h, q, k))


@pytest.mark.parametrize("layout", ["gray", "444", "420"])
@pytest.mark.parametrize("w,h", SMALL + [(1000, 722)])
def test_restatement_16bit_dqt_and_restart_markers(harness, layout, w, h):
    a = S.image(w, h, "noise", seed=w)
    wide = S.pil_jpeg(a, None, layout, qtables=S.wide_qtables())
    assert b"\xff\xdb" in wide
    s = wide.index(b"\xff\xdb")
    assert wide[s + 4] >> 4 == 1, "expected a 16-bit DQT"
    for data, case in ((wide, "dqt16"), (S.pil_jpeg(a, 90, layout, restart_marker_blocks=3), "rst3"),
                       (S.pil_jpeg(a, 30, layout, restart_marker_rows=1), "rst_rows")):
        for k in S.SCALES:
            _same(data, k, (layout, w, h, case, k))


def test_geometry_rules(harness):
    """4:2:0 comes out 4:4:4 at k > 1 (chroma through the next larger IDCT), 4:2:2 keeps half-width chroma"""
    for layout, want in (("420", {2: (4, 8), 4: (2, 4), 8: (1, 2)}), ("444", {2: (4, 4), 4: (2, 2), 8: (1, 1)}),
                         ("422", {2: (4, 4), 4: (2, 2), 8: (1, 1)})):
        data = S.pil_jpeg(S.image(99, 51, "smooth"), 80, layout)
        for k, (sy, sc) in want.items():
            info = _same(data, k, (layout, k))
            assert info[0:2] == [-(-99 // k), -(-51 // k)]
            assert info[4] == sy and info[7] == sc, (layout, k, info)
            full = info[8] == info[0] and info[9] == info[1]
            assert full == (layout != "422"), (layout, k, info)
    assert S.scaled_geometry(S.pil_jpeg(S.image(8, 8, "smooth"), 80, "gray"), 3)[0] == -1


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    L = A.declare_scaled_decode(C.CDLL(T.GPU_SO))
    L.uhdr_b200_last_error.restype = C.c_char_p
    return L


def _apple():
    return open(os.path.join(ROOT, "tests", "golden", "apple_gainmap_new.jpg"), "rb").read()


def test_exported(lib):
    for n in ("uhdr_b200_scaled_dims", "uhdr_b200_decode_scaled_dev", "uhdr_b200_jpeg_decode_scaled"):
        assert hasattr(lib, n), n


def test_scaled_dims(lib):
    data = _apple()
    buf = np.frombuffer(data, np.uint8).copy()
    d = [C.c_uint() for _ in range(4)]
    assert lib.uhdr_b200_scaled_dims(buf.ctypes.data, buf.size, 1, *[C.byref(x) for x in d]) == 0
    full = [x.value for x in d]
    for k in (2, 4, 8):
        assert lib.uhdr_b200_scaled_dims(buf.ctypes.data, buf.size, k, *[C.byref(x) for x in d]) == 0
        assert [x.value for x in d] == [-(-v // k) for v in full], k
    for k in (0, 3, 16, -2):
        assert lib.uhdr_b200_scaled_dims(buf.ctypes.data, buf.size, k, *[C.byref(x) for x in d]) == 3, k
    assert lib.uhdr_b200_scaled_dims(None, 0, 2, *[C.byref(x) for x in d]) == 3
    assert lib.uhdr_b200_scaled_dims(buf.ctypes.data, buf.size // 50, 2, *[C.byref(x) for x in d]) != 0


def _dest(lib, data, k, fmt=A.FMT_RGBAF16):
    buf = np.frombuffer(data, np.uint8).copy()
    d = [C.c_uint() for _ in range(4)]
    assert lib.uhdr_b200_scaled_dims(buf.ctypes.data, buf.size, k, *[C.byref(x) for x in d]) == 0
    w, h, gw, gh = [x.value for x in d]
    px = np.zeros(w * h * 8, np.uint8)
    gm = np.zeros(gw * gh * 4, np.uint8)
    return buf, (px, gm), A.raw_image(fmt, -1, -1, -1, w, h, [px], [w]), A.raw_image(-1, -1, -1, -1, gw, gh, [gm], [gw])


def test_bad_arguments_are_invalid_param(lib):
    """checked before any device work: these codes come back without a GPU too"""
    data = _apple()
    buf, keep, dest, gdesc = _dest(lib, data, 2)
    md = A.GainmapMetadata()
    call = lib.uhdr_b200_decode_scaled_dev
    for k in (0, 3, 5, 16, -1):
        assert call(buf.ctypes.data, buf.size, k, A.CT_LINEAR, A.FLT_MAX, C.byref(dest), C.byref(gdesc), C.byref(md), None) == 3
    assert call(None, 0, 2, A.CT_LINEAR, A.FLT_MAX, C.byref(dest), None, None, None) == 3
    assert call(buf.ctypes.data, buf.size, 2, A.CT_HLG, A.FLT_MAX, C.byref(dest), None, None, None) == 3
    assert call(buf.ctypes.data, buf.size, 2, A.CT_LINEAR, 0.5, C.byref(dest), None, None, None) == 3
    _b, _k, full, _g = _dest(lib, data, 1)
    assert call(buf.ctypes.data, buf.size, 2, A.CT_LINEAR, A.FLT_MAX, C.byref(full), None, None, None) == 3   # 1/1 size
    wrong = A.RawImage.from_buffer_copy(gdesc)
    wrong.w += 1
    assert call(buf.ctypes.data, buf.size, 2, A.CT_LINEAR, A.FLT_MAX, C.byref(dest), C.byref(wrong), None, None) == 3
    pitch = A.RawImage.from_buffer_copy(dest)
    pitch.stride[0] = pitch.w - 1
    assert call(buf.ctypes.data, buf.size, 2, A.CT_LINEAR, A.FLT_MAX, C.byref(pitch), None, None, None) == 3
    out = np.zeros(1 << 20, np.uint8)
    o = A.raw_image(-1, -1, -1, -1, 0, 0, [out], [0])
    for k in (0, 3, 9):
        assert lib.uhdr_b200_jpeg_decode_scaled(buf.ctypes.data, buf.size, 0, k, C.byref(o), out.size) == 3
    assert b"CUDA" not in lib.uhdr_b200_last_error()


def test_no_cpu_fallback(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    data = _apple()
    buf, keep, dest, gdesc = _dest(lib, data, 4)
    for k in (2, 4, 8):
        _b, _k2, dest, gdesc = _dest(lib, data, k)
        rc = lib.uhdr_b200_decode_scaled_dev(buf.ctypes.data, buf.size, k, A.CT_LINEAR, A.FLT_MAX, C.byref(dest),
                                             C.byref(gdesc), None, None)
        assert rc == 1 and b"CUDA" in lib.uhdr_b200_last_error(), k
    jpg = S.pil_jpeg(S.image(64, 32, "smooth"), 90, "420")
    jb = np.frombuffer(jpg, np.uint8).copy()
    out = np.zeros(1 << 16, np.uint8)
    o = A.raw_image(-1, -1, -1, -1, 0, 0, [out], [0])
    assert lib.uhdr_b200_jpeg_decode_scaled(jb.ctypes.data, jb.size, 0, 2, C.byref(o), out.size) == 1
    assert b"CUDA" in lib.uhdr_b200_last_error()
