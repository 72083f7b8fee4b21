"""uhdr_b200_transcode without a device: the 4:2:0 checker (tests/cpp/turbo_ycc420.c) pinned to Pillow's libjpeg-turbo, the
reference composition run end to end, and the argument errors refused before any device work."""
import ctypes as C
import io

import numpy as np
import pytest

import scaled_testlib as S
import transcode_testlib as X
import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A

EXIF = b"Exif\x00\x00MM\x00\x2a\x00\x00\x00\x08\x00\x00\x00\x00\x00\x00"


@pytest.fixture(scope="module")
def ref(oracle_libs):
    if not oracle_libs.ref_is_turbo() or not S.have_harness() or X.turbo_lib() is None:
        pytest.skip("reference build on libjpeg-turbo not available")
    return oracle_libs.Ref().lib


def _segments(jpg):
    """(marker, bytes) up to and including the SOS segment, the scan as the last entry"""
    out, p = [], 2
    while True:
        m, n = jpg[p + 1], (jpg[p + 2] << 8) | jpg[p + 3]
        if m == 0xDA:
            return out + [(m, jpg[p:])]
        out.append((m, jpg[p:p + 2 + n]))
        p += 2 + n


@pytest.mark.parametrize("w,h", [(1, 1), (17, 15), (31, 33), (33, 17), (47, 31), (15, 1), (1, 15), (129, 65), (160, 96)])
@pytest.mark.parametrize("quality", [1, 50, 75, 95, 100])
def test_ycc420_checker_equals_pillow(ref, w, h, quality):
    """Pillow writes a mode "YCbCr" image at 4:2:0 through the same jpeg_write_scanlines path: every table and the
    scan agree, only the JFIF segment (density) is Pillow's own"""
    from PIL import Image
    a = np.random.RandomState(w * 131 + h).randint(0, 256, (h, w, 3)).astype(np.uint8)
    b = io.BytesIO()
    Image.frombytes("YCbCr", (w, h), a.tobytes()).save(b, "JPEG", quality=quality, subsampling=2)
    mine = X.turbo_420([a[:, :, 0], a[:, :, 1], a[:, :, 2]], quality, b"")
    strip = lambda s: [x for x in _segments(s) if x[0] != 0xE0]  # noqa: E731
    assert strip(mine) == strip(b.getvalue())


def test_ycc420_checker_writes_icc(ref):
    a = S.image(40, 24, "smooth")
    icc = b"ICC_PROFILE\x00\x01\x01" + bytes(range(200))
    out = X.turbo_420([a[:, :, 0], a[:, :, 1], a[:, :, 2]], 75, icc)
    assert X.icc_of(out) == icc


@pytest.mark.parametrize("k", [1, 2, 4, 8])
@pytest.mark.parametrize("base_420", [0, 1])
def test_composition_end_to_end(ref, k, base_420):
    """the reference's API-4 accepts the re-encoded pair and the reference decodes the result at the 1/k size"""
    f = X.api4_file(ref, X.metadata(), 455, 333, "444", "444", 4, exif=EXIF)
    out = X.composition(ref, f, k, 75, 60, base_420, keep_exif=1)
    assert isinstance(out, bytes), out
    p = X._probe(ref, out)
    assert p["dims"][:2] == ((455 + k - 1) // k, (333 + k - 1) // k)
    assert p["exif"] == EXIF
    px, gm, md, cg = T.UhdrApi(ref).decode(out)
    assert px.shape[0] == (333 + k - 1) // k
    sub = _segments(p["base_image"])
    sof = [s for m, s in sub if m == 0xC0][0]
    assert sof[11] == (0x22 if base_420 else 0x11)   # luma sampling factors


def _lib():
    return A.declare_transcode(C.CDLL(T.GPU_SO))


def test_export_and_struct_layout():
    lib = _lib()
    assert lib.uhdr_b200_transcode is not None
    assert C.sizeof(A.TranscodeConfig) == 20
    hdr = open(T.ROOT + "/include/uhdr_b200.h").read()
    body = hdr[hdr.index("typedef struct uhdr_b200_transcode_config"):hdr.index("} uhdr_b200_transcode_config_t;")]
    assert [n for n, _ in A.TranscodeConfig._fields_] == [l.split()[1].rstrip(";") for l in body.splitlines()[1:]]


def test_argument_errors_without_device(ref):
    lib = _lib()
    f = X.api4_file(ref, X.metadata(), 64, 48)
    cfg = A.TranscodeConfig(2, 75, 75, 0, 0)
    out = np.zeros(1 << 16, np.uint8)
    n = C.c_size_t()
    buf = np.frombuffer(f, np.uint8).copy()
    d, o = buf.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)
    assert lib.uhdr_b200_transcode(None, len(f), C.byref(cfg), o, out.size, C.byref(n)) == A.CODEC_INVALID_PARAM
    assert lib.uhdr_b200_transcode(d, len(f), None, o, out.size, C.byref(n)) == A.CODEC_INVALID_PARAM
    assert lib.uhdr_b200_transcode(d, len(f), C.byref(cfg), None, out.size, C.byref(n)) == A.CODEC_INVALID_PARAM
    assert lib.uhdr_b200_transcode(d, len(f), C.byref(cfg), o, out.size, None) == A.CODEC_INVALID_PARAM
    for bad in (A.TranscodeConfig(3, 75, 75, 0, 0), A.TranscodeConfig(0, 75, 75, 0, 0), A.TranscodeConfig(16, 75, 75, 0, 0),
                A.TranscodeConfig(1, 101, 75, 0, 0), A.TranscodeConfig(1, 75, -1, 0, 0)):
        assert X.transcode(lib, f, bad.k, bad.base_quality, bad.gainmap_quality)[0] == A.CODEC_INVALID_PARAM
    # not a JPEG/R: the probe's error, before any device work
    junk = b"\xff\xd8" + b"\x00" * 100
    u = C.c_uint()
    A.declare_scaled_decode(lib)
    probe_rc = lib.uhdr_b200_scaled_dims(junk, len(junk), 1, C.byref(u), C.byref(u), C.byref(u), C.byref(u))
    assert probe_rc != A.CODEC_OK and X.transcode(lib, junk, 1, 75, 75)[0] == probe_rc


def test_no_device_is_a_cuda_error(ref):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is present")
    lib = _lib()
    f = X.api4_file(ref, X.metadata(), 64, 48)
    rc, out, _ = X.transcode(lib, f, 2, 75, 75)
    assert rc == A.CODEC_ERROR and out is None
    assert b"CUDA" in T.gpu_err(T.Gpu())
