"""The whole-file codec on device images (uhdr_b200_decode_dev, uhdr_b200_encode_dev, uhdr_b200_jpeg_encode_dev):
files, pixels, gain maps and metadata equal the reference's at 0 tolerance; pitched and offset planes whose padding
is never read or written; stream order against the caller's queued work; back-to-back and concurrent calls; and
the host entry points' error codes with the destination untouched."""
import ctypes as C
import os
import threading
import time

import numpy as np
import pytest

import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SENT = 0xA5
BPP = {A.FMT_RGBAF16: 8, A.FMT_RGBA1010102: 4, A.FMT_RGBA8888: 4}
OUTPUTS = [(A.FMT_RGBAF16, A.CT_LINEAR), (A.FMT_RGBA1010102, A.CT_HLG), (A.FMT_RGBA1010102, A.CT_PQ),
           (A.FMT_RGBA8888, A.CT_SRGB)]


@pytest.fixture(scope="module")
def lib(gpu):
    L = gpu.lib
    L.uhdr_b200_decode_dev.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p]
    L.uhdr_b200_encode_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p,
                                       C.c_size_t, C.c_void_p, C.c_void_p]
    L.uhdr_b200_jpeg_encode_dev.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                            C.c_void_p, C.c_void_p]
    return L


@pytest.fixture(scope="module")
def ref(oracle_libs):
    if not oracle_libs.have_ref():
        pytest.skip("reference build not available")
    return oracle_libs.Ref().lib


# ---- device planes -------------------------------------------------------------------------------------------
class Plane:
    """rows (h, width bytes) in a sentinel-filled device buffer: `stride` elements of `esz` bytes per row, the plane
    starting `off` elements in, 64 guard bytes after it"""

    def __init__(self, torch, rows, esz, stride, off, fill=SENT):
        self.rows = rows
        h, wb = rows.shape
        self.pitch, self.start = stride * esz, off * esz
        self.buf = torch.full((self.start + h * self.pitch + 64,), fill, dtype=torch.uint8, device="cuda")
        self.buf[self.start:self.start + h * self.pitch].view(h, self.pitch)[:, :wb] = torch.from_numpy(rows).cuda()
        self.ptr = self.buf.data_ptr() + self.start
        self.stride = stride
        self.before = self.buf.cpu().numpy().copy()


def dev_image(torch, host, stride_pad=0, off=0, fill=0xFF, stride_mult=1):
    """device copy of a host descriptor's planes: stride = plane width + stride_pad, rounded up to a multiple of
    stride_mult; planes `off` elements into their buffers, padding filled with `fill`"""
    fmt, w, h = host.fmt, host.w, host.h
    geo = {A.FMT_P010: [(w, h, 2), (w, h // 2, 2)], A.FMT_YUV420: [(w, h, 1), (w // 2, h // 2, 1), (w // 2, h // 2, 1)],
           A.FMT_RGBA1010102: [(w, h, 4)], A.FMT_RGBAF16: [(w, h, 8)], A.FMT_RGBA8888: [(w, h, 4)],
           A.FMT_Y400: [(w, h, 1)], A.FMT_RGB888: [(w, h, 3)]}[fmt]
    planes = []
    img = A.RawImage()
    img.fmt, img.cg, img.ct, img.range, img.w, img.h = fmt, host.cg, host.ct, host.range, w, h
    for i, (pw, ph, esz) in enumerate(geo):
        n = pw * ph * esz
        src = np.ctypeslib.as_array(C.cast(host.planes[i], C.POINTER(C.c_uint8)), (host.stride[i] * esz * (ph - 1) + pw * esz,))
        rows = np.stack([src[r * host.stride[i] * esz: r * host.stride[i] * esz + pw * esz] for r in range(ph)]) if n else src
        p = Plane(torch, rows, esz, -(-(pw + stride_pad) // stride_mult) * stride_mult, off, fill)
        planes.append(p)
        img.planes[i] = p.ptr
        img.stride[i] = p.stride
    return img, planes


def unchanged(planes):
    return all((p.buf.cpu().numpy() == p.before).all() for p in planes)


# ---- reference and host-side twins ---------------------------------------------------------------------------
def ref_encode(lib, hdr, sdr, q=95, cfg=None, exif=None):
    """uhdr_encode with every setting of uhdr_b200_gm_config_t the C API has; -> bytes or the error code"""
    cfg = cfg or A.default_gm_config()
    T.UhdrApi(lib)   # declares the result types
    L = lib
    L.uhdr_enc_set_exif_data.restype = A.ErrorInfo
    enc = C.c_void_p(L.uhdr_create_encoder())
    try:
        steps = [lambda: L.uhdr_enc_set_raw_image(enc, C.byref(hdr), A.HDR_IMG)]
        if sdr is not None:
            steps.append(lambda: L.uhdr_enc_set_raw_image(enc, C.byref(sdr), A.SDR_IMG))
        steps += [lambda: L.uhdr_enc_set_quality(enc, q, A.BASE_IMG),
                  lambda: L.uhdr_enc_set_quality(enc, cfg.quality, A.GAIN_MAP_IMG),
                  lambda: L.uhdr_enc_set_gainmap_scale_factor(enc, cfg.scale_factor),
                  lambda: L.uhdr_enc_set_using_multi_channel_gainmap(enc, cfg.multichannel),
                  lambda: L.uhdr_enc_set_gainmap_gamma(enc, cfg.gamma),
                  lambda: L.uhdr_enc_set_preset(enc, cfg.preset)]
        if exif is not None:
            eb = np.frombuffer(exif, np.uint8).copy()
            blk = A.MemBlock(eb.ctypes.data, len(exif), len(exif))
            steps.append(lambda: L.uhdr_enc_set_exif_data(enc, C.byref(blk)))
        steps.append(lambda: L.uhdr_encode(enc))
        for s in steps:
            e = s()
            if e.error_code:
                return int(e.error_code)
        o = L.uhdr_get_encoded_stream(enc).contents
        return C.string_at(o.data, o.data_sz)
    finally:
        L.uhdr_release_encoder(enc)


def encode_dev(lib, hdr_d, sdr_d, q=95, cfg=None, exif=None, stream=0):
    cfg = cfg or A.default_gm_config()
    cap = hdr_d.w * hdr_d.h * 6 + (1 << 20)
    out = np.zeros(cap, np.uint8)
    n = C.c_size_t()
    eb = np.frombuffer(exif, np.uint8).copy() if exif else None
    rc = lib.uhdr_b200_encode_dev(C.byref(hdr_d), C.byref(sdr_d) if sdr_d is not None else None, C.byref(cfg), q,
                                  None if eb is None else eb.ctypes.data, len(exif) if exif else 0,
                                  out.ctypes.data, cap, C.byref(n), stream)
    return rc, bytes(out[:n.value])


class DevDecode:
    """sentinel-filled destination (stride, offset in pixels) and gain-map buffers for one decode_dev call"""

    def __init__(self, torch, data, fmt, ct, stride_pad=0, off=0, gm_pad=0, w=None, h=None):
        info = probe(data)
        self.w, self.h = w or info[0], h or info[1]
        self.gw, self.gh = info[2], info[3]
        self.fmt, self.ct, self.bpp = fmt, ct, BPP[fmt]
        self.stride = self.w + stride_pad
        self.off = off
        self.dst = torch.full(((off + self.h * self.stride) * self.bpp + 64,), SENT, dtype=torch.uint8, device="cuda")
        self.gstride = self.gw + gm_pad
        self.gbuf = torch.full((self.gh * self.gstride * 4 + 64,), SENT, dtype=torch.uint8, device="cuda")
        self.desc = A.raw_image(fmt, -1, -1, -1, self.w, self.h, [], [])
        self.desc.planes[0] = self.dst.data_ptr() + off * self.bpp
        self.desc.stride[0] = self.stride
        self.gdesc = A.raw_image(-1, -1, -1, -1, self.gw, self.gh, [], [])
        self.gdesc.planes[0] = self.gbuf.data_ptr()
        self.gdesc.stride[0] = self.gstride
        self.md = A.GainmapMetadata()
        self.data = np.frombuffer(data, np.uint8).copy()

    def run(self, lib, stream=0, boost=A.FLT_MAX):
        return lib.uhdr_b200_decode_dev(self.data.ctypes.data, self.data.size, self.ct, boost, C.byref(self.desc),
                                        C.byref(self.gdesc), C.byref(self.md), stream)

    def pixels(self):
        """-> (pixel rows, every other byte of the buffer is the sentinel)"""
        d = self.dst.cpu().numpy()
        s, pitch, wb = self.off * self.bpp, self.stride * self.bpp, self.w * self.bpp
        body = d[s:s + self.h * pitch].reshape(self.h, pitch)
        rest_ok = (d[:s] == SENT).all() and (d[s + self.h * pitch:] == SENT).all() and (body[:, wb:] == SENT).all()
        return body[:, :wb].copy(), rest_ok

    def gainmap(self):
        g = self.gbuf.cpu().numpy()
        gb = 1 if self.gdesc.fmt == A.FMT_Y400 else 4
        body = g[:self.gh * self.gstride * gb].reshape(self.gh, self.gstride * gb)
        rest_ok = (body[:, self.gw * gb:] == SENT).all() and (g[self.gh * self.gstride * gb:] == SENT).all()
        return body[:, :self.gw * gb].copy(), rest_ok

    def untouched(self):
        return (self.dst.cpu().numpy() == SENT).all() and (self.gbuf.cpu().numpy() == SENT).all()


_probe_dec = {}


def probe(data):
    key = hash(data)
    if key not in _probe_dec:
        L = T.Gpu().lib
        T.UhdrApi(L)
        dec = C.c_void_p(L.uhdr_create_decoder())
        buf = np.frombuffer(data, np.uint8).copy()
        ci = A.CompressedImage(buf.ctypes.data, len(data), len(data), -1, -1, -1)
        assert L.uhdr_dec_set_image(dec, C.byref(ci)).error_code == 0
        assert L.uhdr_dec_probe(dec).error_code == 0
        _probe_dec[key] = (L.uhdr_dec_get_image_width(dec), L.uhdr_dec_get_image_height(dec),
                           L.uhdr_dec_get_gainmap_width(dec), L.uhdr_dec_get_gainmap_height(dec))
        L.uhdr_release_decoder(dec)
    return _probe_dec[key]


def host_decode_rc(lib, data, fmt, ct):
    T.UhdrApi(lib)
    dec = C.c_void_p(lib.uhdr_create_decoder())
    try:
        buf = np.frombuffer(data, np.uint8).copy()
        ci = A.CompressedImage(buf.ctypes.data, len(data), len(data), -1, -1, -1)
        for e in (lib.uhdr_dec_set_image(dec, C.byref(ci)), lib.uhdr_dec_set_out_img_format(dec, fmt),
                  lib.uhdr_dec_set_out_color_transfer(dec, ct), lib.uhdr_decode(dec)):
            if e.error_code:
                return int(e.error_code)
        return 0
    finally:
        lib.uhdr_release_decoder(dec)


def _frames(w, h, kind="smooth", seed=T.SEED):
    hb = T.make_p010(w, h, kind, seed)
    sb = T.make_yuv420(w, h, kind, seed + 1)
    hdr, k1 = A.p010_image(hb, w, h, A.CG_BT2100, A.CT_HLG, A.CR_LIMITED)
    sdr, k2 = A.yuv420_image(sb, w, h, A.CG_BT709)
    return hdr, sdr, (hb, sb, k1, k2)


def _packed(w, h, hdr_kind):
    if hdr_kind == "f16":
        hb = T.make_rgbaf16(w, h)
        hdr = A.raw_image(A.FMT_RGBAF16, A.CG_BT2100, A.CT_LINEAR, A.CR_FULL, w, h, [hb], [w])
    else:
        hb = T.make_rgba1010102(w, h)
        hdr = A.raw_image(A.FMT_RGBA1010102, A.CG_BT2100, A.CT_PQ, A.CR_FULL, w, h, [hb], [w])
    sb = T.make_rgba8888(w, h)
    sdr = A.raw_image(A.FMT_RGBA8888, A.CG_BT709, A.CT_SRGB, A.CR_FULL, w, h, [sb], [w])
    return hdr, sdr, (hb, sb)


def _ref_decode(ref, data, fmt, ct):
    return T.UhdrApi(ref).decode(data, fmt, ct)


def _check_decode(lib, ref, data, fmt, ct, xmp=False, **kw):
    import torch
    d = DevDecode(torch, data, fmt, ct, **kw)
    rc = d.run(lib)
    assert rc == 0, T.gpu_err(T.Gpu())
    torch.cuda.synchronize()
    px, ok = d.pixels()
    gm, gok = d.gainmap()
    pb, gb, mb, cgb = _ref_decode(ref, data, fmt, ct)
    assert ok and gok, "bytes outside the planes were written"
    assert (px == pb).all(), (fmt, ct, int((px != pb).sum()))
    assert (gm == gb).all(), (fmt, ct)
    assert d.desc.cg == cgb
    if xmp:   # the reference leaves use_base_cg uninitialised on its XMP branch
        from test_xmp_cpu import _vals
        assert _vals(d.md, False) == _vals(mb, False)
    else:
        assert T.md_equal(d.md, mb)


# ---- decode ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h,scale,mc", [(w, h, s, m) for (w, h) in ((3840, 2160), (1000, 722))
                                           for (s, m) in ((1, 1), (2, 0), (4, 1))] + [(7680, 4320, 4, 1)])
def test_decode_dev_equals_reference(lib, ref, w, h, scale, mc):
    hdr, sdr, keep = _frames(w, h)
    data = ref_encode(ref, hdr, sdr, 95, A.default_gm_config(scale_factor=scale, multichannel=mc))
    assert isinstance(data, bytes)
    for i, (fmt, ct) in enumerate(OUTPUTS):
        # pitched destinations: an odd stride for the 4-byte formats, a plane one pixel into its buffer
        _check_decode(lib, ref, data, fmt, ct, stride_pad=(3 if BPP[fmt] == 4 else 8), off=i % 2, gm_pad=5)


@pytest.mark.parametrize("name", ["apple_gainmap_new.jpg", "apple_gainmap_old.jpg"])
def test_decode_dev_apple_files(lib, ref, name):
    data = open(os.path.join(GOLDEN, name), "rb").read()
    for fmt, ct in OUTPUTS:
        _check_decode(lib, ref, data, fmt, ct, xmp=True, stride_pad=1, off=1, gm_pad=3)


def test_decode_dev_restart_interval_file(lib, ref):
    from test_gpu_restart_decode import _dri_jpegr
    data = _dri_jpegr(lib)[0]
    for fmt, ct in OUTPUTS:
        _check_decode(lib, ref, data, fmt, ct, stride_pad=7, off=1, gm_pad=1)


# ---- encode ------------------------------------------------------------------------------------------------------
ENC_CASES = [
    # (w, h, sdr kind, cfg, base q, exif)
    (3840, 2160, "709", {}, 95, None),
    (1920, 1080, "p3", {"scale_factor": 2}, 50, b"Exif\0\0" + bytes(range(64))),
    # generateGainMap flags outside the C API: uhdr_encode's values are used whatever the config says
    (1000, 722, "709", {"sdr_is_601": 1, "use_luminance": 0}, 95, None),
    (1000, 722, "709", {"scale_factor": 4, "multichannel": 0, "preset": A.USAGE_REALTIME}, 95, None),
    (998, 722, "p3", {"gamma": 2.2, "quality": 50}, 95, b"Exif\0\0MM"),
    (998, 722, "709", {"preset": A.USAGE_REALTIME, "multichannel": 0, "scale_factor": 2}, 50, None),
    (1920, 1080, "rgba", {}, 95, None),
    (1000, 722, "rgba_f16", {"scale_factor": 2, "multichannel": 0}, 95, b"Exif\0\0II"),
    (1920, 1080, "api0", {}, 95, None),
    (998, 722, "api0_1010102", {"scale_factor": 4}, 50, None),
    (1000, 722, "api0_f16", {"multichannel": 0}, 95, None),
]


def _enc_inputs(kind, w, h):
    if kind in ("709", "p3", "api0"):
        hdr, sdr, keep = _frames(w, h, "noise" if w < 1024 else "smooth")
        if kind == "p3":
            sdr.cg = A.CG_P3
        return hdr, (None if kind == "api0" else sdr), keep
    hdr, sdr, keep = _packed(w, h, "f16" if kind.endswith("f16") else "1010102")
    return hdr, (None if kind.startswith("api0") else sdr), keep


@pytest.mark.parametrize("case", range(len(ENC_CASES)))
def test_encode_dev_equals_reference(lib, ref, case):
    import torch
    w, h, kind, cfgkw, q, exif = ENC_CASES[case]
    hdr, sdr, keep = _enc_inputs(kind, w, h)
    cfg = A.default_gm_config(**cfgkw)
    want = ref_encode(ref, hdr, sdr, q, cfg, exif)
    assert isinstance(want, bytes), want
    # planes at odd element offsets, strides past the width, padding 0xFF
    hd, hp = dev_image(torch, hdr, stride_pad=5, off=1)
    sd, sp = dev_image(torch, sdr, stride_pad=3, off=3) if sdr is not None else (None, [])
    rc, got = encode_dev(lib, hd, sd, q, cfg, exif)
    assert rc == 0, T.gpu_err(T.Gpu())
    assert len(got) == len(want) and got == want, (case, len(got), len(want))
    assert unchanged(hp + sp), "an input was modified"


@pytest.mark.parametrize("w,h,pad", [(1920, 1080, 0), (998, 722, 5)])
def test_encode_dev_display_p3_plane_in_place(lib, ref, w, h, pad):
    """A Display-P3 SDR intent reaches the block stage unconverted.  8-byte aligned rows whose width is a multiple of
    8 are read where they are (1920x1080, tight); at 998 wide the block stage would read the 0xFF bytes past the
    width, so the plane is staged first."""
    import torch
    hdr, sdr, keep = _frames(w, h, "noise")
    sdr.cg = A.CG_P3
    want = ref_encode(ref, hdr, sdr)
    assert isinstance(want, bytes), want
    hd, hp = dev_image(torch, hdr)
    sd, sp = dev_image(torch, sdr, stride_pad=pad, stride_mult=8)
    assert all(sd.stride[i] % 8 == 0 and sd.planes[i] % 8 == 0 for i in range(3))
    rc, got = encode_dev(lib, hd, sd)
    assert rc == 0, T.gpu_err(T.Gpu())
    assert got == want
    assert unchanged(hp + sp)


# ---- compressImage on the device -------------------------------------------------------------------------------
def test_jpeg_encode_dev_of_a_device_gain_map(lib, oracle_libs):
    """generateGainMap -> compressImage without leaving HBM == the reference's compressImage of that map"""
    import torch
    o = oracle_libs.Oracle().lib
    w, h = 1000, 722
    hdr, sdr, keep = _frames(w, h, "noise")
    hd, hp = dev_image(torch, hdr, stride_pad=2, off=1)
    sd, sp = dev_image(torch, sdr, stride_pad=2, off=1)
    for mc, scale in ((1, 1), (0, 2), (1, 4)):
        mw, mh, ch = w // scale, h // scale, 3 if mc else 1
        gm_t = torch.full((mh * (mw + 3) * ch + 64,), SENT, dtype=torch.uint8, device="cuda")
        gm_d = A.raw_image(-1, -1, -1, -1, mw, mh, [], [])
        gm_d.planes[0] = gm_t.data_ptr()
        gm_d.stride[0] = mw + 3
        md = A.GainmapMetadata()
        cfg = A.default_gm_config(scale_factor=scale, multichannel=mc)
        assert lib.uhdr_b200_generate_gainmap_dev(C.byref(sd), C.byref(hd), C.byref(cfg), C.byref(md), C.byref(gm_d), None) == 0
        cap = 1 << 22
        out = np.zeros(cap, np.uint8)
        n = C.c_size_t()
        rc = lib.uhdr_b200_jpeg_encode_dev(C.byref(gm_d), 85, None, 0, out.ctypes.data, cap, C.byref(n), None)
        assert rc == 0, T.gpu_err(T.Gpu())
        torch.cuda.synchronize()
        gm = gm_t.cpu().numpy()[:mh * (mw + 3) * ch].reshape(mh, (mw + 3) * ch)[:, :mw * ch]
        # the reference compresses its map from a zero-initialised buffer with 64-pixel aligned rows
        s = -(-mw // 64) * 64
        padded = np.zeros((mh, s * ch), np.uint8)
        padded[:, :mw * ch] = gm
        img = A.raw_image(gm_d.fmt, -1, -1, 1, mw, mh, [padded], [s])
        got = bytes(out[:n.value])
        assert got == T.oracle_encode(o, img, 85, None, T.GM_COMMENT), (mc, scale)
        assert got == T.gpu_jpeg_encode(T.Gpu(), img, 85), (mc, scale)


@pytest.mark.parametrize("fmt,w,h", [(A.FMT_Y400, 960, 540), (A.FMT_Y400, 72, 33), (A.FMT_YUV420, 1280, 720),
                                     (A.FMT_YUV420, 320, 240), (A.FMT_RGB888, 100, 61), (A.FMT_RGB888, 960, 540)])
def test_jpeg_encode_dev_tight_and_pitched(lib, gpu, oracle_libs, fmt, w, h):
    """tight strides equal the reference; pitched / offset planes with 0xFF padding equal the host entry point"""
    import torch
    from test_gpu_jpeg_api import _img
    o = oracle_libs.Oracle().lib
    img, keep = _img(fmt, w, h, "noise")
    icc = bytes(range(40))
    gm = fmt in (A.FMT_RGB888, A.FMT_Y400)
    want = T.oracle_encode(o, img, 90, icc, T.GM_COMMENT if gm else None)
    assert T.gpu_jpeg_encode(gpu, img, 90, icc) == want
    iccb = (C.c_uint8 * len(icc)).from_buffer_copy(icc)
    # tight; pitched and offset; 8-byte aligned rows with 0xFF bytes past the width
    for pad, off, mult in ((0, 0, 1), (5, 1, 1), (13, 3, 1), (3, 0, 8)):
        d, planes = dev_image(torch, img, stride_pad=pad, off=off, stride_mult=mult)
        cap = w * h * 6 + (1 << 16)
        out = np.zeros(cap, np.uint8)
        n = C.c_size_t()
        rc = lib.uhdr_b200_jpeg_encode_dev(C.byref(d), 90, C.cast(iccb, C.c_void_p), len(icc), out.ctypes.data, cap,
                                           C.byref(n), None)
        assert rc == 0, T.gpu_err(gpu)
        assert bytes(out[:n.value]) == want, (fmt, w, h, pad, off, mult)
        assert unchanged(planes)


# ---- stream order -----------------------------------------------------------------------------------------------
def _sleep_cycles(ms):
    return int(2e6 * ms)   # H100 SM clocks are below 2 GHz: at least `ms` milliseconds


def test_decode_dev_waits_for_caller_work_on_the_device_not_the_host(lib, ref):
    import torch
    hdr, sdr, keep = _frames(1000, 722)
    data = ref_encode(ref, hdr, sdr, 95, A.default_gm_config(scale_factor=2))
    fmt, ct = A.FMT_RGBAF16, A.CT_LINEAR
    d = DevDecode(torch, data, fmt, ct, stride_pad=4)
    assert d.run(lib) == 0      # warm-up
    torch.cuda.synchronize()
    want, _ = d.pixels()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        torch.cuda._sleep(_sleep_cycles(300))
        d.dst.zero_()
    t0 = time.perf_counter()
    rc = d.run(lib, st.cuda_stream)
    dt = time.perf_counter() - t0
    assert rc == 0
    st.synchronize()
    px, _ = d.pixels()
    assert (px == want).all(), "the write went ahead of the caller's zero_()"
    assert dt < 0.15, ("the call waited for the caller's stream", dt)


def test_encode_dev_reads_inputs_after_caller_work(lib, ref):
    import torch
    w, h = 1000, 722
    hdr, sdr, keep = _frames(w, h, "noise")
    want = ref_encode(ref, hdr, sdr)
    hd, hp = dev_image(torch, hdr, stride_pad=2)
    sd, sp = dev_image(torch, sdr, stride_pad=2)
    real = [p.buf.clone() for p in hp + sp]
    for p in hp + sp:
        p.buf.fill_(0x3C)
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        torch.cuda._sleep(_sleep_cycles(200))
        for p, r in zip(hp + sp, real):
            p.buf.copy_(r)
    rc, got = encode_dev(lib, hd, sd, stream=st.cuda_stream)
    assert rc == 0
    assert got == want


def test_eight_back_to_back_decodes_one_sync(lib, ref):
    import torch
    files = []
    for i in range(8):
        hdr, sdr, keep = _frames(640 + 16 * i, 368 + 8 * i, "noise" if i % 2 else "smooth", seed=T.SEED + i)
        files.append(ref_encode(ref, hdr, sdr, 90, A.default_gm_config(scale_factor=1 + i % 3, multichannel=i % 2)))
    st = torch.cuda.Stream()
    outs = []
    for i, data in enumerate(files):
        fmt, ct = OUTPUTS[i % 4]
        outs.append(DevDecode(torch, data, fmt, ct, stride_pad=i + 1, gm_pad=i))
    torch.cuda.synchronize()   # the sentinel fills ran on the current stream
    # the caller's stream is busy first: every write waits, and each call's scratch is still needed by the
    # previous call's writes when the next call starts
    with torch.cuda.stream(st):
        torch.cuda._sleep(_sleep_cycles(100))
    for d in outs:
        assert d.run(lib, st.cuda_stream) == 0
    st.synchronize()
    for data, d in zip(files, outs):
        px, ok = d.pixels()
        gm, gok = d.gainmap()
        pb, gb, mb, cgb = _ref_decode(ref, data, d.fmt, d.ct)
        assert ok and gok and (px == pb).all() and (gm == gb).all() and T.md_equal(d.md, mb)


def test_four_threads_decode_and_encode_at_once(lib, ref):
    import torch
    jobs = []
    for i in range(4):
        w, h = 640 + 32 * i, 368 + 16 * i
        hdr, sdr, keep = _frames(w, h, "noise", seed=T.SEED + 10 + i)
        want_file = ref_encode(ref, hdr, sdr, 90)
        want_px = _ref_decode(ref, want_file, A.FMT_RGBA1010102, A.CT_PQ)
        jobs.append((hdr, sdr, keep, want_file, want_px))
    errors = []

    def work(i):
        try:
            hdr, sdr, keep, want_file, (pb, gb, mb, cgb) = jobs[i]
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                hd, hp = dev_image(torch, hdr, stride_pad=1)
                sd, sp = dev_image(torch, sdr, stride_pad=1)
                st.synchronize()
                for _ in range(3):
                    d = DevDecode(torch, want_file, A.FMT_RGBA1010102, A.CT_PQ, stride_pad=3)
                    st.synchronize()
                    assert d.run(lib, st.cuda_stream) == 0
                    rc, got = encode_dev(lib, hd, sd, 90, stream=st.cuda_stream)
                    assert rc == 0 and got == want_file, i
                    st.synchronize()
                    px, ok = d.pixels()
                    assert ok and (px == pb).all(), i
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    th = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors


# ---- errors -------------------------------------------------------------------------------------------------------
def test_decode_dev_errors_match_uhdr_decode(lib, ref):
    import torch
    hdr, sdr, keep = _frames(640, 368)
    data = ref_encode(ref, hdr, sdr)
    # a bad format / transfer pair
    d = DevDecode(torch, data, A.FMT_RGBAF16, A.CT_HLG)
    assert d.run(lib) == host_decode_rc(lib, data, A.FMT_RGBAF16, A.CT_HLG) == 3
    torch.cuda.synchronize()
    assert d.untouched()
    # dimensions that are not the image's
    d = DevDecode(torch, data, A.FMT_RGBAF16, A.CT_LINEAR, w=638)
    assert d.run(lib) == 3 and d.untouched()
    # a host pointer as the destination plane
    d = DevDecode(torch, data, A.FMT_RGBAF16, A.CT_LINEAR)
    host = np.zeros(640 * 368 * 8, np.uint8)
    d.desc.planes[0] = host.ctypes.data
    assert d.run(lib) == 3 and d.untouched() and not host.any()
    # a truncated file
    cut = data[:len(data) // 2]
    d = DevDecode(torch, data, A.FMT_RGBAF16, A.CT_LINEAR)
    d.data = np.frombuffer(cut, np.uint8).copy()
    rc = d.run(lib)
    assert rc != 0 and rc == host_decode_rc(lib, cut, A.FMT_RGBAF16, A.CT_LINEAR)
    torch.cuda.synchronize()
    assert d.untouched()


def test_encode_dev_errors_match_uhdr_encode(lib, ref):
    import torch
    hdr, sdr, keep = _frames(640, 368)
    hd, hp = dev_image(torch, hdr)
    sd, sp = dev_image(torch, sdr)
    bad = A.RawImage.from_buffer_copy(hd)
    bad.ct = A.CT_SRGB   # P010 with an SDR transfer
    hbad = A.RawImage.from_buffer_copy(hdr)
    hbad.ct = A.CT_SRGB
    assert encode_dev(lib, bad, sd)[0] == ref_encode(lib, hbad, sdr) == 3
    small = A.RawImage.from_buffer_copy(sd)
    small.w = 320
    assert encode_dev(lib, hd, small)[0] == 3
    hostp = A.RawImage.from_buffer_copy(hd)
    hostp.planes[0] = keep[0].ctypes.data
    assert encode_dev(lib, hostp, sd)[0] == 3
    assert unchanged(hp + sp)
