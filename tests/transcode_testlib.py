"""Helpers of the transcoding tests: the reference composition uhdr_b200_transcode must equal byte for byte, the call
itself, and JPEG/R inputs of every kind (reference API-4 files built from Pillow JPEGs).

The composition (include/uhdr_b200.h, uhdr_b200_transcode):
  1. each JPEG of the file decoded by libjpeg-turbo with scale_denom = k, raw_data_out (oracle/jpeg_scaled_ref.c);
  2. re-encoded by the reference's JpegEncoderHelper::compressImage (ref_jpeg_encode) with strides equal to the
     plane widths, in the format the planes form, with that JPEG's own ICC payload -- or, for base_420 and a 4:4:4
     base, by libjpeg-turbo's scanline encoder at 4:2:0 (tests/cpp/turbo_ycc420.c);
  3. keep_exif: the primary image's EXIF segment inserted right after SOI of the new base;
  4. the reference's API-4 with the primary image's ICC gamut and the file's metadata.
"""
import ctypes as C
import glob
import io
import os
import subprocess
import tempfile

import numpy as np

import scaled_testlib as S
import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A
from test_api4_cpu import _api4
from test_probe_cpu import _probe

ISO_NS = b"urn:iso:std:iso:ts:21496:-1"


def app_payload(jpg, marker, sig):
    """payload (after the length field) of the first APPn `marker` whose payload starts with sig, else b''"""
    p = 2
    while p + 4 <= len(jpg) and jpg[p] == 0xFF and jpg[p + 1] != 0xDA:
        n = (jpg[p + 2] << 8) | jpg[p + 3]
        if jpg[p + 1] == marker and jpg[p + 4:p + 4 + len(sig)] == sig:
            return jpg[p + 4:p + 2 + n]
        p += 2 + n
    return b""


def icc_of(jpg):
    return app_payload(jpg, 0xE2, b"ICC_PROFILE\x00")


def planes_format(planes):
    if len(planes) == 1:
        return A.FMT_Y400
    (h, w), (ch, cw) = planes[0].shape, planes[1].shape
    if (cw, ch) == (w, h):
        return A.FMT_YUV444
    if (cw, ch) == ((w + 1) // 2, (h + 1) // 2):
        return A.FMT_YUV420
    if (cw, ch) == ((w + 1) // 2, h):
        return A.FMT_YUV422
    raise ValueError("sampling the encoder does not write")


def ref_compress(ref, planes, quality, icc):
    """JpegEncoderHelper::compressImage of tight planes"""
    planes = [np.ascontiguousarray(p) for p in planes]
    h, w = planes[0].shape
    img = A.raw_image(planes_format(planes), -1, -1, -1, w, h, planes, [p.shape[1] for p in planes])
    cap = w * h * 6 + (1 << 16) + len(icc)
    out = np.zeros(cap, np.uint8)
    n = C.c_size_t()
    ib = (C.c_uint8 * len(icc)).from_buffer_copy(icc) if icc else None
    rc = ref.ref_jpeg_encode(C.byref(img), quality, ib, C.c_size_t(len(icc)), out.ctypes.data_as(C.c_void_p),
                             C.c_size_t(cap), C.byref(n))
    assert rc == 0, rc
    return bytes(out[:n.value])


_turbo = []


def turbo_lib():
    """tests/cpp/turbo_ycc420.c built into a temporary directory against the libjpeg-turbo binary next to the reference
    build (oracle/_ref/), or None when there is none"""
    if not _turbo:
        S.ensure_built()
        ref_dir = os.path.join(T.ROOT, "oracle", "_ref")
        turbo = sorted(glob.glob(os.path.join(ref_dir, "libjpeg-*.so.62*")))
        if not turbo:
            _turbo.append(None)
        else:
            so = os.path.join(tempfile.mkdtemp(prefix="turbo_ycc420_"), "libturbo_ycc420.so")
            subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-Wall", "-I",
                                   os.path.join(T.ROOT, "oracle", "ref_turbo"),
                                   os.path.join(T.ROOT, "tests", "cpp", "turbo_ycc420.c"), turbo[0],
                                   "-Wl,-rpath," + ref_dir, "-o", so])
            _turbo.append(C.CDLL(so))
    return _turbo[0]


def turbo_420(planes, quality, icc):
    """libjpeg-turbo's scanline encoder at 4:2:0 from full-size YCbCr planes (tests/cpp/turbo_ycc420.c)"""
    L = turbo_lib()
    y, cb, cr = (np.ascontiguousarray(p) for p in planes)
    h, w = y.shape
    cap = w * h * 4 + (1 << 16) + len(icc)
    out = np.zeros(cap, np.uint8)
    n = C.c_size_t()
    ib = (C.c_uint8 * len(icc)).from_buffer_copy(icc) if icc else None
    rc = L.tyc_encode_ycc420(*(p.ctypes.data_as(C.c_void_p) for p in (y, cb, cr)), w, h, quality, ib,
                             C.c_size_t(len(icc)), out.ctypes.data_as(C.c_void_p), C.c_size_t(cap), C.byref(n))
    assert rc == 0, rc
    return bytes(out[:n.value])


def composition(ref, data, k, base_quality, gainmap_quality, base_420=0, keep_exif=0):
    """the reference pieces' file for these settings (bytes), or the error tuple of the failing API-4 step"""
    p = _probe(ref, data)
    assert "error" not in p, p
    base, gm, md = p["base_image"], p["gainmap_image"], p["md"]
    if ISO_NS not in gm:   # XMP-only metadata: the reference leaves use_base_cg uninitialised
        md.use_base_cg = 1
    _, bp = S.harness_decode(base, k, 0)
    _, gp = S.harness_decode(gm, k, 0)
    bicc, gicc = icc_of(base), icc_of(gm)
    if base_420 and planes_format(bp) == A.FMT_YUV422:
        return ("base_420", A.CODEC_UNSUPPORTED)
    if base_420 and planes_format(bp) == A.FMT_YUV444:
        nb = turbo_420(bp, base_quality, bicc)
    else:
        nb = ref_compress(ref, bp, base_quality, bicc)
    ng = ref_compress(ref, gp, gainmap_quality, gicc)
    exif = app_payload(base, 0xE1, b"Exif\x00\x00")
    if keep_exif and exif:
        nb = nb[:2] + b"\xff\xe1" + (len(exif) + 2).to_bytes(2, "big") + exif + nb[2:]
    cg = ref.ref_icc_gamut(C.c_char_p(bicc), C.c_size_t(len(bicc))) if bicc else A.CG_UNSPEC
    return _api4(ref, nb, ng, md, cg)


def transcode(lib, data, k, base_quality, gainmap_quality, base_420=0, keep_exif=0, cap=None):
    """uhdr_b200_transcode -> (rc, bytes or None, out_size)"""
    A.declare_transcode(lib)
    cfg = A.TranscodeConfig(k, base_quality, gainmap_quality, base_420, keep_exif)
    cap = len(data) * 2 + (1 << 20) if cap is None else cap
    out = np.full(max(cap, 1), 0xA5, np.uint8)
    n = C.c_size_t(0)
    buf = np.frombuffer(data, np.uint8).copy()
    rc = lib.uhdr_b200_transcode(buf.ctypes.data_as(C.c_void_p), C.c_size_t(len(data)), C.byref(cfg),
                                 out.ctypes.data_as(C.c_void_p), C.c_size_t(cap), C.byref(n))
    if rc:
        assert (out == 0xA5).all(), "a failing call wrote into out"
        return rc, None, n.value
    return rc, bytes(out[:n.value]), n.value


# ---- inputs ------------------------------------------------------------------------------------------------------
def pil_bytes(a, layout, quality=90, icc=None, **kw):
    from PIL import Image
    b = io.BytesIO()
    if icc:
        kw["icc_profile"] = icc
    if layout == "gray":
        Image.fromarray(a if a.ndim == 2 else a[:, :, 0]).save(b, "JPEG", quality=quality, **kw)
    else:
        Image.fromarray(a).save(b, "JPEG", quality=quality, subsampling=S.SUBSAMPLING[layout], **kw)
    return b.getvalue()


def ref_icc(ref, cg):
    """the ICC profile the reference writes for an sRGB image of gamut cg, without the 14-byte marker prefix"""
    buf = (C.c_uint8 * 8192)()
    n = ref.ref_icc_profile(A.CT_SRGB, cg, buf, 8192)
    assert n > 0
    return bytes(buf[14:n])


def api4_file(ref, md, w, h, base_layout="420", map_layout="gray", map_scale=1, seed=1, base_icc_cg=A.CG_P3,
              map_icc_cg=None, exif=None, base_cg=A.CG_BT709, **pil):
    """a JPEG/R assembled by the reference's API-4 from Pillow JPEGs; pil: extra Image.save arguments (restart
    markers, optimize) for both JPEGs"""
    a = S.image(w, h, "smooth", seed)
    mw, mh = max(1, w // map_scale), max(1, h // map_scale)
    m = S.image(mw, mh, "smooth", seed + 1)
    kw = dict(pil)
    if exif:
        kw["exif"] = exif
    base = pil_bytes(a, base_layout, 88, ref_icc(ref, base_icc_cg) if base_icc_cg is not None else None, **kw)
    gm = pil_bytes(m, map_layout, 85, ref_icc(ref, map_icc_cg) if map_icc_cg is not None else None, **pil)
    out = _api4(ref, base, gm, md, base_cg)
    assert isinstance(out, bytes), out
    return out


def metadata(use_base_cg=1):
    md = A.GainmapMetadata()
    for c in range(3):
        md.max_content_boost[c] = 4.0
        md.min_content_boost[c] = 1.0
        md.gamma[c] = 1.0
        md.offset_sdr[c] = md.offset_hdr[c] = 1.0 / 64
    md.hdr_capacity_min, md.hdr_capacity_max, md.use_base_cg = 1.0, 4.0, use_base_cg
    return md
