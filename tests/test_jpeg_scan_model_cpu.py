"""Pins the scan model (tests/jpeg_scan_model.py) on the CPU, no device needed.

  * A plain bit writer over the model's per-block codes rebuilds libjpeg-turbo's scan bytes exactly: Pillow's
    bundled libjpeg-turbo (gray, 4:4:4, 4:2:2, 4:2:0), the reference's JpegEncoderHelper on libjpeg-turbo when that
    build is present, and the C restatement (raw 4:2:0 / 4:2:2 / 4:4:4 planes, RGB888, Y400) -- small ragged images at
    qualities 1, 50 and 100, noise and worst-case content.  That fixes the scan order, dummy blocks, DC prediction
    and the code of every block.
  * On larger streams the block bits, padded to a byte, plus one stuffed zero per 0xFF equal the scan length, and the
    CTA plan partitions the blocks and bits.
  * uhdr_b200_jpeg_encode_stats is declared and reads zeros in a process without a device.
"""
import ctypes as C
import io
import os
import subprocess
import sys

import numpy as np
import pytest

import jpeg_scan_model as M
import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A

QUALITIES = (1, 50, 100)
SIZES = [(8, 8), (17, 9), (37, 21), (64, 48), (70, 34)]


def _content(kind, h, w, ch, seed):
    rs = np.random.RandomState(seed)
    if kind == "noise":
        a = rs.randint(0, 256, (h, w, ch))
    elif kind == "binary":   # 0/255 noise: the longest block strings
        a = rs.randint(0, 2, (h, w, ch)) * 255
    else:                    # "checker": alternating 0/255 blocks, DC swings of category 11 at q100
        yy, xx = np.mgrid[0:h, 0:w]
        a = np.repeat((((yy // 8 + xx // 8) % 2) * 255)[..., None], ch, 2)
        a[..., 1:] = 255 - a[..., 1:]
    return np.ascontiguousarray(a.astype(np.uint8))


def _check(model, data):
    assert M.write_scan(model) == data[model.scan_offset:-2]


@pytest.fixture(scope="module")
def olib(oracle_libs):
    return oracle_libs.Oracle().lib


@pytest.mark.parametrize("mode,subsampling", [("L", None), ("RGB", 0), ("RGB", 1), ("RGB", 2)])
def test_bit_writer_equals_pillow_libjpeg_turbo(olib, mode, subsampling):
    PIL = pytest.importorskip("PIL.Image")
    for i, (w, h) in enumerate(SIZES):
        for kind in ("noise", "binary", "checker"):
            a = _content(kind, h, w, 1 if mode == "L" else 3, seed=i)
            for q in QUALITIES:
                b = io.BytesIO()
                kw = {} if subsampling is None else {"subsampling": subsampling}
                PIL.fromarray(a[..., 0] if mode == "L" else a, mode).save(b, "JPEG", quality=q, **kw)
                data = b.getvalue()
                m = M.ScanModel(data, olib)
                assert m.ncomp == (1 if mode == "L" else 3)
                _check(m, data)


def _raw(fmt, w, h, kind, seed):
    """a raw image of the encoder's input layouts -> (RawImage, arrays kept alive)"""
    if fmt in (A.FMT_Y400, A.FMT_RGB888):
        a = _content(kind, h, w, 1 if fmt == A.FMT_Y400 else 3, seed)
        return A.raw_image(fmt, -1, -1, 1, w, h, [a], [w]), a
    cw = w if fmt == A.FMT_YUV444 else (w + 1) // 2
    chh = (h + 1) // 2 if fmt == A.FMT_YUV420 else h
    p = [_content(kind, h, w, 1, seed)[..., 0].copy()] + [_content(kind, chh, cw, 1, seed + k)[..., 0].copy() for k in (1, 2)]
    return A.raw_image(fmt, 1, 3, 1, w, h, p, [w, cw, cw]), p


FMTS = [A.FMT_Y400, A.FMT_YUV420, A.FMT_YUV422, A.FMT_YUV444, A.FMT_RGB888]


@pytest.mark.parametrize("fmt", FMTS)
def test_bit_writer_equals_encoder_streams(olib, fmt):
    """the encoder's layouts (raw planes as JpegEncoderHelper takes them): the C restatement, and the reference's
    helper on libjpeg-turbo where that build is present"""
    turbo = C.CDLL(T.REF_TURBO_SO) if os.path.exists(T.REF_TURBO_SO) else None
    for i, (w, h) in enumerate(SIZES[1:] + [(18, 18)]):
        for kind in ("noise", "binary", "checker"):
            img, keep = _raw(fmt, w, h, kind, seed=10 + i)
            for q in QUALITIES:
                streams = [T.oracle_encode(olib, img, q)]
                if turbo is not None and (fmt != A.FMT_YUV420 or (w % 2 == 0 and h % 2 == 0)):
                    cap = w * h * 8 + 65536
                    out = np.zeros(cap, np.uint8)
                    n = C.c_size_t()
                    if turbo.ref_jpeg_encode(C.byref(img), q, None, C.c_size_t(0), out.ctypes.data_as(C.c_void_p),
                                             C.c_size_t(cap), C.byref(n)) == 0:
                        streams.append(bytes(out[:n.value]))
                for data in streams:
                    _check(M.ScanModel(data, olib), data)


@pytest.mark.parametrize("fmt,w,h,kind,q", [(A.FMT_RGB888, 1000, 722, "binary", 100), (A.FMT_YUV420, 1282, 722, "noise", 100),
                                            (A.FMT_Y400, 2050, 1030, "checker", 100), (A.FMT_YUV422, 998, 510, "noise", 7)])
def test_lengths_and_plan_of_larger_streams(olib, fmt, w, h, kind, q):
    img, keep = _raw(fmt, w, h, kind, seed=w)
    data = T.oracle_encode(olib, img, q)
    m = M.ScanModel(data, olib)
    nff = int((m.raw == 0xFF).sum())
    assert (m.total_bits + 7) // 8 + nff == len(data) - 2 - m.scan_offset
    for bpt in (1, 2, 3, 8):
        P = m.plan(bpt)
        assert P["ncta"] == -(-m.nblocks // (256 * bpt))
        assert int(P["total"].sum()) == m.total_bits
        assert (P["start"][1:] == np.cumsum(P["total"])[:-1]).all()
        ff = m.ff_bytes(P)
        assert len(ff["pos"]) == nff
        # a byte that straddles a CTA boundary holds that boundary
        b = np.sort(P["start"][1:])
        for p in ff["pos"][ff["two_ctas"]]:
            k = np.searchsorted(b, 8 * p, "right")
            assert k < len(b) and b[k] < 8 * p + 8
    cs = m.cases()
    assert cs["ac_max"] == int(m.ac_lengths().max()) and cs["ac_max"] > 0


def test_locate_names_cta_window_and_block(olib):
    img, keep = _raw(A.FMT_Y400, 512, 64, "binary", 3)
    data = T.oracle_encode(olib, img, 100)
    m = M.ScanModel(data, olib)
    assert "headers" in m.locate(10, 1)
    s = m.locate(len(data) - 3, 1)
    assert f"CTA {m.plan(1)['ncta'] - 1} of" in s and f"scan block {m.nblocks - 1}" in s


def test_encode_stats_declared_and_zero_without_device():
    """uhdr_b200_jpeg_encode_stats: declared through ctypes_api, ten zeros in a process that has no device (an
    encode there fails with a CUDA error and plans nothing)"""
    import __graft_entry__ as g
    g.build()
    code = (
        "import ctypes as C, numpy as np, sys\n"
        f"sys.path.insert(0, {T.ROOT!r})\n"
        "from libultrahdr_b200 import ctypes_api as A\n"
        f"L = A.declare_jpeg_encode_stats(C.CDLL({T.GPU_SO!r}))\n"
        "assert A.jpeg_encode_stats(L) == (0, (0,) * 8, 0)\n"
        "g = np.zeros((16, 16), np.uint8)\n"
        "img = A.raw_image(A.FMT_Y400, -1, -1, 1, 16, 16, [g], [16])\n"
        "out = np.zeros(65536, np.uint8); n = C.c_size_t()\n"
        "rc = L.uhdr_b200_jpeg_encode(C.byref(img), 90, None, C.c_size_t(0), out.ctypes.data_as(C.c_void_p), C.c_size_t(65536), C.byref(n))\n"
        "assert rc != 0, rc\n"
        "assert A.jpeg_encode_stats(L) == (0, (0,) * 8, 0)\n"
        "print('ok')\n")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-2000:]
