"""Reduced-size decoding on the GPU (uhdr_b200_jpeg_decode_scaled, uhdr_b200_decode_scaled_dev) at 0 tolerance:
planes and RGBA equal to libjpeg-turbo's scale_denom = k decode (oracle/jpeg_scaled_ref.c) with both entropy
decoders; whole files equal to that decode followed by the reference's applyGainMap; k = 1 equal to
uhdr_b200_decode_dev; pitched destinations whose guard bytes stay untouched; stream order, concurrency, the
unsupported 4:2:2 case, and the reduced-IDCT kernel on the route for k > 1 only."""
import ctypes as C
import os
import threading
import time

import numpy as np
import pytest

import scaled_testlib as S
import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A
from test_api4_cpu import _api4
from test_gpu_dev_codec import BPP, OUTPUTS, _frames, _sleep_cycles, ref_encode

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(T.ROOT, "tests", "golden")
GUARD = 0xFF
UNSUPPORTED = 6
SIZES = [(1, 1), (7, 9), (17, 33), (1000, 722), (4080, 3072), (7680, 4320)]


@pytest.fixture(scope="module")
def lib(gpu):
    L = A.declare_scaled_decode(gpu.lib)
    L.uhdr_b200_decode_dev.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p]
    L.uhdr_b200_last_error.restype = C.c_char_p
    if not S.have_harness():
        pytest.skip("no libjpeg-turbo harness")
    return L


@pytest.fixture(scope="module")
def ref(oracle_libs):
    if not oracle_libs.have_ref():
        pytest.skip("reference build not available")
    return oracle_libs.Ref()


# ---- one JPEG: planes and RGBA -------------------------------------------------------------------------------------
def stage_decode(lib, data, mode, k, cap):
    buf = np.zeros(cap, np.uint8)
    out = A.raw_image(-1, -1, -1, -1, 0, 0, [buf], [0])
    src = np.frombuffer(data, np.uint8).copy()
    rc = lib.uhdr_b200_jpeg_decode_scaled(src.ctypes.data, src.size, mode, k, C.byref(out), cap)
    return rc, out, buf


def _planes(out, buf, dims):
    res = []
    for c, (w, h) in enumerate(dims):
        off = out.planes[c] - buf.ctypes.data
        s = out.stride[c]
        res.append(buf[off:off + s * h].reshape(h, s)[:, :w])
    return res


def check_jpeg(lib, data, case):
    for k in S.SCALES:
        info, ref = S.harness_decode(data, k)
        dims = [(info[5 + 3 * c], info[6 + 3 * c]) for c in range(info[2])]
        rc, out, buf = stage_decode(lib, data, 0, k, info[0] * info[1] * 3 + 2 * (info[0] + 16) * (info[1] + 16) + 4096)
        assert rc == 0, (case, k, lib.uhdr_b200_last_error())
        assert (out.w, out.h) == (info[0], info[1]), (case, k)
        if k > 1:
            assert out.fmt == (A.FMT_Y400 if info[2] == 1 else A.FMT_YUV444), (case, k, out.fmt)
        for c, (p, r) in enumerate(zip(_planes(out, buf, dims), ref)):
            assert (p == r).all(), (case, k, c, int((p != r).sum()))
        if info[2] == 3:
            _i, rgba = S.harness_decode(data, k, 1)
            rc, out, buf = stage_decode(lib, data, 1, k, info[0] * info[1] * 4)
            assert rc == 0 and out.fmt == A.FMT_RGBA8888, (case, k)
            got = buf[:info[0] * info[1] * 4].reshape(info[1], info[0], 4)
            assert (got == rgba).all(), (case, k, "rgba", int((got != rgba).any(-1).sum()))


@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("layout", ["gray", "444", "420"])
def test_planes_equal_libjpeg_turbo(lib, layout, w, h):
    combos = [(95, "smooth"), (40, "noise")] if w * h < 4000 * 3000 else [(90, "smooth")]
    for q, kind in combos:
        data = S.pil_jpeg(S.image(w, h, kind, seed=w + q), q, layout)
        check_jpeg(lib, data, (layout, w, h, q, kind))


@pytest.mark.parametrize("w,h", [(17, 33), (1000, 722), (4080, 3072)])
@pytest.mark.parametrize("layout", ["gray", "444", "420"])
def test_planes_host_entropy_decoder_and_restart_markers(lib, layout, w, h):
    """the host-decoder route (jpeg_inverse_scaled_dev), forced and through a stream the device decoder declines"""
    a = S.image(w, h, "smooth", seed=3)
    prev = lib.uhdr_b200_set_entropy_decoder(1)
    try:
        check_jpeg(lib, S.pil_jpeg(a, 85, layout), (layout, w, h, "host"))
        check_jpeg(lib, S.pil_jpeg(a, None, layout, qtables=S.wide_qtables()), (layout, w, h, "host", "dqt16"))
    finally:
        lib.uhdr_b200_set_entropy_decoder(prev)
    check_jpeg(lib, S.pil_jpeg(a, 85, layout, restart_marker_blocks=5), (layout, w, h, "rst"))


# ---- whole files ----------------------------------------------------------------------------------------------------
def split_jpegr(d):
    """the two JPEG streams of a JPEG/R file: SOI .. EOI, skipping marker segments and entropy-coded data"""
    out, p = [], 0
    while len(out) < 2:
        p = d.index(b"\xff\xd8", p)
        s, q = p, p + 2
        while True:
            if d[q] != 0xFF:
                q += 1
                continue
            m = d[q + 1]
            if m == 0xFF:
                q += 1
                continue
            if m == 0xD9:
                q += 2
                break
            q += 2 + ((d[q + 2] << 8) | d[q + 3])
            if m == 0xDA:
                while True:
                    q = d.index(b"\xff", q)
                    n = d[q + 1]
                    if n == 0 or 0xD0 <= n <= 0xD7:
                        q += 2
                    elif n == 0xFF:
                        q += 1
                    else:
                        break
        out.append(d[s:q])
        p = q
    return out


def scaled_dims(lib, data, k):
    buf = np.frombuffer(data, np.uint8).copy()
    d = [C.c_uint() for _ in range(4)]
    rc = lib.uhdr_b200_scaled_dims(buf.ctypes.data, buf.size, k, *[C.byref(x) for x in d])
    assert rc == 0, lib.uhdr_b200_last_error()
    return [x.value for x in d]


class ScaledDecode:
    """0xFF-guarded, pitched and offset destination and gain-map buffers for one decode at 1/k"""

    def __init__(self, torch, lib, data, k, fmt, ct, stride_pad=3, off=1, gm_pad=5):
        self.k, self.fmt, self.ct, self.bpp = k, fmt, ct, BPP[fmt]
        self.w, self.h, self.gw, self.gh = scaled_dims(lib, data, k)
        self.stride, self.off, self.gstride = self.w + stride_pad, off, self.gw + gm_pad
        self.dst = torch.full(((off + self.h * self.stride) * self.bpp + 64,), GUARD, dtype=torch.uint8, device="cuda")
        self.gbuf = torch.full((self.gh * self.gstride * 4 + 64,), GUARD, dtype=torch.uint8, device="cuda")
        self.desc = A.raw_image(fmt, -1, -1, -1, self.w, self.h, [], [])
        self.desc.planes[0] = self.dst.data_ptr() + off * self.bpp
        self.desc.stride[0] = self.stride
        self.gdesc = A.raw_image(-1, -1, -1, -1, self.gw, self.gh, [], [])
        self.gdesc.planes[0] = self.gbuf.data_ptr()
        self.gdesc.stride[0] = self.gstride
        self.md = A.GainmapMetadata()
        self.data = np.frombuffer(data, np.uint8).copy()

    def run(self, lib, stream=0, boost=A.FLT_MAX, dense=False):
        if dense:
            return lib.uhdr_b200_decode_dev(self.data.ctypes.data, self.data.size, self.ct, boost, C.byref(self.desc),
                                            C.byref(self.gdesc), C.byref(self.md), stream)
        return lib.uhdr_b200_decode_scaled_dev(self.data.ctypes.data, self.data.size, self.k, self.ct, boost,
                                               C.byref(self.desc), C.byref(self.gdesc), C.byref(self.md), stream)

    def pixels(self):
        d = self.dst.cpu().numpy()
        s, pitch, wb = self.off * self.bpp, self.stride * self.bpp, self.w * self.bpp
        body = d[s:s + self.h * pitch].reshape(self.h, pitch)
        ok = (d[:s] == GUARD).all() and (d[s + self.h * pitch:] == GUARD).all() and (body[:, wb:] == GUARD).all()
        return body[:, :wb].copy(), ok

    def gainmap(self):
        g = self.gbuf.cpu().numpy()
        gb = 1 if self.gdesc.fmt == A.FMT_Y400 else 4
        body = g[:self.gh * self.gstride * gb].reshape(self.gh, self.gstride * gb)
        ok = (body[:, self.gw * gb:] == GUARD).all() and (g[self.gh * self.gstride * gb:] == GUARD).all()
        return body[:, :self.gw * gb].copy(), ok

    def untouched(self):
        return (self.dst.cpu().numpy() == GUARD).all() and (self.gbuf.cpu().numpy() == GUARD).all()


def icc_gamut(ref, jpg):
    """the reference's reading (IccHelper::readIccColorGamut) of a JPEG's first ICC_PROFILE APP2 payload, as the
    decoder reads it into the decoded image's gamut; -1 without one"""
    i = 2
    while i + 4 <= len(jpg) and jpg[i] == 0xFF and jpg[i + 1] != 0xDA:
        n = (jpg[i + 2] << 8) | jpg[i + 3]
        if jpg[i + 1] == 0xE2 and jpg[i + 4:i + 16] == b"ICC_PROFILE\0":
            payload = jpg[i + 4:i + 2 + n]
            return ref.lib.ref_icc_gamut((C.c_uint8 * len(payload)).from_buffer_copy(payload), C.c_size_t(len(payload)))
        i += 2 + n
    return A.CG_UNSPEC


def expected(ref, data, k, fmt, ct, md, boost=A.FLT_MAX):
    """libjpeg-turbo at 1/k for both JPEGs, then the reference's applyGainMap -> (pixel rows, gain-map rows)"""
    base, gm = split_jpegr(data)
    cg, gm_cg = icc_gamut(ref, base), icc_gamut(ref, gm)
    info, planes = S.harness_decode(base, k)
    ginfo, gplanes = S.harness_decode(gm, k, 0 if split_ncomp(gm) == 1 else 1)
    if ginfo[2] == 1:
        gmap = gplanes[0][:, :, None].copy()
    else:
        gmap = gplanes
    w, h = info[0], info[1]
    if ct == A.CT_SRGB:
        _i, rgba = S.harness_decode(base, k, 1)
        return rgba.reshape(h, w * 4), gmap.reshape(gmap.shape[0], -1)
    keep = [np.ascontiguousarray(p) for p in planes]
    if len(keep) == 1:
        sdr = A.raw_image(A.FMT_Y400, cg, A.CT_SRGB, A.CR_FULL, w, h, keep, [w])
    else:
        fmt_in = A.FMT_YUV444 if planes[1].shape == planes[0].shape else A.FMT_YUV420
        sdr = A.raw_image(fmt_in, cg, A.CT_SRGB, A.CR_FULL, w, h, keep, [p.shape[1] for p in keep])
    gimg = T.gm_image(np.ascontiguousarray(gmap), gm_cg)
    px = ref.apply(sdr, gimg, md, ct, boost)
    return px.view(np.uint8).reshape(h, w * BPP[fmt]), gmap.reshape(gmap.shape[0], -1)


def split_ncomp(jpg):
    s = jpg.index(b"\xff\xc0") if b"\xff\xc0" in jpg else jpg.index(b"\xff\xc1")
    return jpg[s + 9]


def check_file(lib, ref, data, ks=(2, 4, 8), outputs=OUTPUTS, **kw):
    import torch
    for k in ks:
        for i, (fmt, ct) in enumerate(outputs):
            d = ScaledDecode(torch, lib, data, k, fmt, ct, off=i % 2, **kw)
            rc = d.run(lib)
            assert rc == 0, (k, fmt, ct, lib.uhdr_b200_last_error())
            torch.cuda.synchronize()
            px, ok = d.pixels()
            gm, gok = d.gainmap()
            assert ok and gok, ("bytes outside the planes were written", k, fmt, ct)
            want_px, want_gm = expected(ref, data, k, fmt, ct, d.md)
            assert (gm == want_gm).all(), (k, fmt, ct, "gain map")
            assert (px == want_px).all(), (k, fmt, ct, int((px != want_px).sum()))


@pytest.mark.parametrize("w,h,scale,mc", [(w, h, s, m) for (w, h) in ((3840, 2160), (4080, 3072), (1000, 722))
                                           for (s, m) in ((1, 1), (2, 0), (4, 1))] + [(7680, 4320, 4, 1), (7680, 4320, 1, 0)])
def test_decode_scaled_dev_equals_harness_plus_reference_apply(lib, ref, w, h, scale, mc):
    hdr, sdr, keep = _frames(w, h)
    data = ref_encode(ref.lib, hdr, sdr, 95, A.default_gm_config(scale_factor=scale, multichannel=mc))
    assert isinstance(data, bytes)
    check_file(lib, ref, data)


@pytest.mark.parametrize("name", ["apple_gainmap_new.jpg", "apple_gainmap_old.jpg"])
def test_apple_files(lib, ref, name):
    check_file(lib, ref, open(os.path.join(GOLDEN, name), "rb").read(), stride_pad=1, gm_pad=3)


def test_restart_interval_file(lib, ref):
    from test_gpu_restart_decode import _dri_jpegr
    check_file(lib, ref, _dri_jpegr(lib)[0], stride_pad=7, gm_pad=1)


def test_k1_equals_decode_dev(lib, ref):
    import torch
    for scale, mc in ((1, 1), (4, 0)):
        hdr, sdr, keep = _frames(1000, 722, "noise")
        data = ref_encode(ref.lib, hdr, sdr, 90, A.default_gm_config(scale_factor=scale, multichannel=mc))
        for fmt, ct in OUTPUTS:
            a = ScaledDecode(torch, lib, data, 1, fmt, ct)
            b = ScaledDecode(torch, lib, data, 1, fmt, ct)
            assert a.run(lib) == 0 and b.run(lib, dense=True) == 0
            torch.cuda.synchronize()
            assert (a.dst.cpu().numpy() == b.dst.cpu().numpy()).all(), (fmt, ct)
            assert (a.gbuf.cpu().numpy() == b.gbuf.cpu().numpy()).all(), (fmt, ct)
            assert bytes(a.md) == bytes(b.md) and a.desc.cg == b.desc.cg


def _route(lib, fn):
    """names of the kernels `fn` launches (the stage hook synchronises its workspace, which collects the timings)"""
    lib.uhdr_b200_set_kernel_timing(1)
    buf = C.create_string_buffer(1 << 16)
    try:
        lib.uhdr_b200_kernel_timing_report(buf, C.c_size_t(len(buf)), 1)
        fn()
        lib.uhdr_b200_kernel_timing_report(buf, C.c_size_t(len(buf)), 1)
    finally:
        lib.uhdr_b200_set_kernel_timing(0)
    return {ln.split()[0] for ln in buf.value.decode().splitlines() if ln.strip()}


def test_reduced_idct_on_the_route_for_k_above_1_only(lib, ref):
    hdr, sdr, keep = _frames(1000, 722)
    data = ref_encode(ref.lib, hdr, sdr, 95, A.default_gm_config(scale_factor=2, multichannel=1))
    base, gm = split_jpegr(data)
    for k in S.SCALES:
        def both():
            for jpg, mode in ((base, 0), (gm, 1)):
                assert stage_decode(lib, jpg, mode, k, 1 << 23)[0] == 0, (k, mode)
        names = _route(lib, both)
        assert ("idct_scaled" in names) == (k > 1), (k, names)
        # 4:2:0 primary: its chroma runs through the 8x8 IDCT at k = 1 and 2; at 4 and 8 every component is reduced
        assert ("idct_dequant" in names) == (k <= 2), (k, names)


# ---- stream order, threads, errors ------------------------------------------------------------------------------------
def test_writes_wait_for_the_callers_stream(lib, ref):
    import torch
    hdr, sdr, keep = _frames(1000, 722)
    data = ref_encode(ref.lib, hdr, sdr, 95, A.default_gm_config(scale_factor=2))
    d = ScaledDecode(torch, lib, data, 4, A.FMT_RGBA1010102, A.CT_PQ, stride_pad=4)
    assert d.run(lib) == 0
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


def test_four_threads(lib, ref):
    import torch
    jobs = []
    for i in range(4):
        hdr, sdr, keep = _frames(640 + 32 * i, 368 + 16 * i, "noise", seed=T.SEED + 20 + i)
        jobs.append(ref_encode(ref.lib, hdr, sdr, 90, A.default_gm_config(scale_factor=1 + i % 2, multichannel=i % 2)))
    wants = {}
    for i, data in enumerate(jobs):
        d = ScaledDecode(torch, lib, data, 2 << (i % 3), A.FMT_RGBAF16, A.CT_LINEAR)
        assert d.run(lib) == 0
        torch.cuda.synchronize()
        wants[i] = d.pixels()[0]
    errors = []

    def work(i):
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                for _ in range(3):
                    d = ScaledDecode(torch, lib, jobs[i], 2 << (i % 3), A.FMT_RGBAF16, A.CT_LINEAR)
                    st.synchronize()
                    assert d.run(lib, st.cuda_stream) == 0
                    st.synchronize()
                    px, ok = d.pixels()
                    assert ok and (px == wants[i]).all(), i
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    th = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors


def test_422_is_unsupported_above_k1_and_writes_nothing(lib, ref):
    import torch
    md = A.GainmapMetadata()
    for i in range(3):
        md.max_content_boost[i], md.min_content_boost[i], md.gamma[i] = 4.0, 1.0, 1.0
        md.offset_sdr[i] = md.offset_hdr[i] = 1.0 / 64
    md.hdr_capacity_min, md.hdr_capacity_max, md.use_base_cg = 1.0, 4.0, 1
    a = S.image(640, 360, "smooth")
    for base_layout, gm_layout in (("422", "gray"), ("420", "422")):
        data = _api4(lib, S.pil_jpeg(a, 90, base_layout), S.pil_jpeg(a[::2, ::2], 90, gm_layout), md, A.CG_BT709)
        assert isinstance(data, bytes), data
        for k in (2, 4, 8):
            for fmt, ct in OUTPUTS:   # a gain-map destination is passed: SRGB output decodes the map too
                d = ScaledDecode(torch, lib, data, k, fmt, ct)
                torch.cuda.synchronize()
                assert d.run(lib) == UNSUPPORTED, (base_layout, gm_layout, k, fmt, ct)
                torch.cuda.synchronize()
                assert d.untouched(), (base_layout, gm_layout, k, fmt, ct)
        d = ScaledDecode(torch, lib, data, 1, A.FMT_RGBAF16, A.CT_LINEAR)
        assert d.run(lib) == 0
        torch.cuda.synchronize()
    info, _ = S.harness_decode(S.pil_jpeg(a, 90, "422"), 2)
    rc, out, buf = stage_decode(lib, S.pil_jpeg(a, 90, "422"), 0, 2, 1 << 22)
    assert rc == UNSUPPORTED and info[8] != info[0]


def test_bad_scale_and_sizes_write_nothing(lib, ref):
    import torch
    hdr, sdr, keep = _frames(640, 368)
    data = ref_encode(ref.lib, hdr, sdr)
    d = ScaledDecode(torch, lib, data, 2, A.FMT_RGBAF16, A.CT_LINEAR)
    torch.cuda.synchronize()
    for k in (0, 3, 16):
        d.k = k
        assert d.run(lib) == 3, k
    d.k = 4   # buffers sized for 1/2
    assert d.run(lib) == 3
    torch.cuda.synchronize()
    assert d.untouched()
