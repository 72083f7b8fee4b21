"""Helpers of the reduced-size decoding tests: the two CPU checkers built by oracle/scaled.mk and Pillow-written
test streams.

  * ``harness_decode`` -- the real libjpeg-turbo with scale_denom = k (oracle/jpeg_scaled_ref.c)
  * ``oracle_scaled``  -- the C restatement (oracle/jpeg_scaled_oracle.c)
"""
import ctypes as C
import io
import os
import subprocess

import numpy as np

import uhdr_testlib as T

ROOT = T.ROOT
SCALED_ORACLE_SO = os.path.join(ROOT, "oracle", "_ref", "libjpeg_scaled_oracle.so")
SCALED_REF_SO = os.path.join(ROOT, "oracle", "_ref", "libjpeg_scaled_ref.so")
SCALES = (1, 2, 4, 8)
SUBSAMPLING = {"444": 0, "422": 1, "420": 2}


def _stale(so, src):
    return not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(os.path.join(ROOT, "oracle", src))


def ensure_built():
    if _stale(SCALED_ORACLE_SO, "jpeg_scaled_oracle.c") or _stale(SCALED_REF_SO, "jpeg_scaled_ref.c"):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "scaled.mk", "all"],
                              stdout=subprocess.DEVNULL)


_libs = {}


def _lib(path):
    if path not in _libs:
        ensure_built()
        _libs[path] = C.CDLL(path)
    return _libs[path]


def have_harness():
    ensure_built()
    return os.path.exists(SCALED_REF_SO)


def harness_decode(data, k, mode=0):
    """libjpeg-turbo at scale 1/k.  mode 0 -> (info, [plane c: (downsampled_height, downsampled_width) u8]);
    mode 1 -> (info, (out_h, out_w, 4) u8 RGBA).  info: [out_w, out_h, ncomp, min_s, then (s, w, h) per component;
    [15] the warnings libjpeg-turbo raised]"""
    L = _lib(SCALED_REF_SO)
    buf = (C.c_uint8 * len(data)).from_buffer_copy(data)
    ci = (C.c_int * 16)()
    rc = L.jsr_decode(buf, C.c_size_t(len(data)), k, mode, None, C.c_size_t(0), ci)
    assert rc == 0, rc
    info = list(ci)
    if mode == 1:
        out = np.zeros((info[1], info[0], 4), np.uint8)
    else:
        out = np.zeros(sum(info[5 + 3 * c] * info[6 + 3 * c] for c in range(info[2])), np.uint8)
    rc = L.jsr_decode(buf, C.c_size_t(len(data)), k, mode, out.ctypes.data_as(C.c_void_p), C.c_size_t(out.size), ci)
    assert rc == 0, rc
    info = list(ci)   # now with [15], the warnings of the decode itself
    if mode == 1:
        return info, out
    planes, o = [], 0
    for c in range(info[2]):
        w, h = info[5 + 3 * c], info[6 + 3 * c]
        planes.append(out[o:o + w * h].reshape(h, w))
        o += w * h
    return info, planes


def oracle_scaled(data, k):
    """the restatement at scale 1/k -> (geometry [out_w, out_h, then (s, w, h) per component], cropped planes)"""
    L = _lib(SCALED_ORACLE_SO)
    h = T.JoHeader()
    buf = (C.c_uint8 * len(data)).from_buffer_copy(data)
    assert L.jo_read_header(buf, C.c_size_t(len(data)), C.byref(h)) == 0
    f = h.frame
    coefs = [np.zeros((f.comp[c].hblocks * f.comp[c].wblocks, 64), np.int16) for c in range(f.ncomp)]
    cp = (C.c_void_p * 3)(*([c.ctypes.data for c in coefs] + [None] * (3 - f.ncomp)))
    assert L.jo_decode_coefs(buf, C.c_size_t(len(data)), C.byref(h), cp) == 0
    g = (C.c_int * 12)()
    assert L.jso_scaled_geometry(C.byref(f), k, g) == 0
    g = list(g)
    planes = [np.zeros((f.comp[c].hblocks * g[2 + 3 * c], f.comp[c].wblocks * g[2 + 3 * c]), np.uint8)
              for c in range(f.ncomp)]
    pp = (C.c_void_p * 3)(*([p.ctypes.data for p in planes] + [None] * (3 - f.ncomp)))
    assert L.jso_inverse_scaled(C.byref(h), k, cp, pp) == 0
    return g, [planes[c][:g[4 + 3 * c], :g[3 + 3 * c]] for c in range(f.ncomp)]


def scaled_geometry(data, k):
    L = _lib(SCALED_ORACLE_SO)
    h = T.JoHeader()
    buf = (C.c_uint8 * len(data)).from_buffer_copy(data)
    assert L.jo_read_header(buf, C.c_size_t(len(data)), C.byref(h)) == 0
    g = (C.c_int * 12)()
    rc = L.jso_scaled_geometry(C.byref(h.frame), k, g)
    return rc, list(g)


def image(w, h, kind, seed=7):
    rs = np.random.RandomState(seed)
    if kind == "noise":
        return rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    a = np.stack([(128 + 100 * np.sin(xx / 23.0 + k) * np.cos(yy / 17.0)) for k in range(3)], -1)
    return (a + rs.randint(-8, 9, a.shape)).clip(0, 255).astype(np.uint8)


def pil_jpeg(a, quality, layout, qtables=None, **restart):
    from PIL import Image
    b = io.BytesIO()
    kw = dict(restart)
    if qtables is not None:
        kw["qtables"] = qtables
    else:
        kw["quality"] = quality
    if layout == "gray":
        Image.fromarray(a[:, :, 0]).save(b, "JPEG", **kw)
    else:
        Image.fromarray(a).save(b, "JPEG", subsampling=SUBSAMPLING[layout], **kw)
    return b.getvalue()


def wide_qtables(seed=3):
    """quantiser tables with entries above 255: Pillow writes them as 16-bit DQT"""
    rs = np.random.RandomState(seed)
    t = [list(rs.randint(1, 1200, 64)), list(rs.randint(1, 1200, 64))]
    t[0][0] = t[1][0] = 300
    return t
