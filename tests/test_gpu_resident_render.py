"""Device-resident images (uhdr_b200_image_open_dev / _render_dev / _release) on the GPU, at 0 tolerance:
full-frame renders equal uhdr_b200_decode_scaled_dev / uhdr_b200_decode_dev for every k, output and boost; any
rectangle equals that crop of the full decode (and, for a few, of the reference's uhdr_decode); the apply route a
region takes; pitched and offset destinations with untouched padding; stream order, table slots, release and threads;
errors that write nothing; and the memory an 8K image holds."""
import ctypes as C
import os
import sys
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
INVALID, UNSUPPORTED = 3, 6


@pytest.fixture(scope="module")
def lib(gpu):
    L = A.declare_resident_image(A.declare_scaled_decode(gpu.lib))
    L.uhdr_b200_decode_dev.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p]
    L.uhdr_b200_last_error.restype = C.c_char_p
    L.uhdr_b200_apply_stats.argtypes = [C.POINTER(C.c_ulonglong)]
    L.uhdr_b200_trim_cache.restype = C.c_size_t
    return L


def torch():
    import torch as t
    return t


# ---- helpers --------------------------------------------------------------------------------------------------------
class Dest:
    """a guarded device destination of w x h pixels: stride = w + pad pixels, the plane `off` pixels into the buffer"""

    def __init__(self, fmt, w, h, pad=0, off=0):
        t = torch()
        self.fmt, self.w, self.h, self.bpp, self.off, self.stride = fmt, w, h, BPP[fmt], off, w + pad
        self.buf = t.full(((off + h * self.stride) * self.bpp + 64,), GUARD, dtype=t.uint8, device="cuda")
        self.desc = A.raw_image(fmt, -1, -1, -1, w, h, [], [])
        self.desc.planes[0] = self.buf.data_ptr() + off * self.bpp
        self.desc.stride[0] = self.stride

    def body(self):
        """-> (h, w * bpp) device view, whether every byte outside it still holds the guard"""
        s, pitch, wb = self.off * self.bpp, self.stride * self.bpp, self.w * self.bpp
        rows = self.buf[s:s + self.h * pitch].view(self.h, pitch)
        ok = bool((self.buf[:s] == GUARD).all()) and bool((self.buf[s + self.h * pitch:] == GUARD).all()) and \
            bool((rows[:, wb:] == GUARD).all())
        return rows[:, :wb], ok

    def untouched(self):
        return bool((self.buf == GUARD).all())


class Image:
    def __init__(self, lib, data, k):
        self.lib, self.k = lib, k
        self.data = np.frombuffer(data, np.uint8).copy()
        h = C.c_void_p()
        rc = lib.uhdr_b200_image_open_dev(self.data.ctypes.data, self.data.size, k, C.byref(h))
        assert rc == 0, (rc, lib.uhdr_b200_last_error())
        self.h = h
        d = [C.c_uint() for _ in range(4)]
        self.md = A.GainmapMetadata()
        self.bytes = C.c_size_t()
        assert lib.uhdr_b200_image_info(h, *[C.byref(x) for x in d], C.byref(self.md), C.byref(self.bytes)) == 0
        self.w, self.hh, self.gw, self.gh = [x.value for x in d]

    def render(self, dest, ct, boost, x, y, stream=0):
        return self.lib.uhdr_b200_image_render_dev(self.h, ct, boost, x, y, C.byref(dest.desc), stream)

    def close(self):
        if self.h:
            assert self.lib.uhdr_b200_image_release(self.h) == 0
            self.h = None


def full_decode(lib, data, k, fmt, ct, boost, dense=False):
    """uhdr_b200_decode_scaled_dev (dense: uhdr_b200_decode_dev) -> (device rows, descriptor)"""
    buf = np.frombuffer(data, np.uint8).copy()
    d = [C.c_uint() for _ in range(4)]
    assert lib.uhdr_b200_scaled_dims(buf.ctypes.data, buf.size, k, *[C.byref(x) for x in d]) == 0
    dst = Dest(fmt, d[0].value, d[1].value)
    if dense:
        rc = lib.uhdr_b200_decode_dev(buf.ctypes.data, buf.size, ct, boost, C.byref(dst.desc), None, None, None)
    else:
        rc = lib.uhdr_b200_decode_scaled_dev(buf.ctypes.data, buf.size, k, ct, boost, C.byref(dst.desc), None, None, None)
    assert rc == 0, (k, fmt, ct, lib.uhdr_b200_last_error())
    torch().cuda.synchronize()
    return dst.body()[0], dst.desc


def boosts(md):
    lo, hi = max(1.0, md.hdr_capacity_min), max(1.0, md.hdr_capacity_max)
    return sorted({1.0, lo, float(np.sqrt(lo * hi)), hi, A.FLT_MAX})


def allowed_ks(lib, data):
    """the k the file's sampling allows: every k unless decode_scaled_dev refuses it"""
    out = [1]
    for k in (2, 4, 8):
        buf = np.frombuffer(data, np.uint8).copy()
        d = [C.c_uint() for _ in range(4)]
        assert lib.uhdr_b200_scaled_dims(buf.ctypes.data, buf.size, k, *[C.byref(x) for x in d]) == 0
        dst = Dest(A.FMT_RGBAF16, d[0].value, d[1].value)
        rc = lib.uhdr_b200_decode_scaled_dev(buf.ctypes.data, buf.size, k, A.CT_LINEAR, 4.0, C.byref(dst.desc), None,
                                             None, None)
        assert rc in (0, UNSUPPORTED), rc
        if rc == 0:
            out.append(k)
    torch().cuda.synchronize()
    return out


def apply_stats(lib):
    st = (C.c_ulonglong * 4)()
    lib.uhdr_b200_apply_stats(st)
    return np.array(list(st), np.int64)


_files = {}


def encoded(lib, w, h, scale, mc):
    key = (w, h, scale, mc)
    if key not in _files:
        hdr, sdr, keep = _frames(w, h, "noise" if w < 1000 else "smooth", seed=T.SEED + w + scale)
        data = ref_encode(lib, hdr, sdr, 92, A.default_gm_config(scale_factor=scale, multichannel=mc))
        assert isinstance(data, bytes), data
        _files[key] = data
    return _files[key]


def resize_file(lib):
    """a map whose aspect ratio (1.6) differs from the base image's (16:9): applyGainMap resizes it"""
    md = A.GainmapMetadata()
    for i in range(3):
        md.max_content_boost[i], md.min_content_boost[i], md.gamma[i] = 6.0, 1.0, 1.0
        md.offset_sdr[i] = md.offset_hdr[i] = 1.0 / 64
    md.hdr_capacity_min, md.hdr_capacity_max, md.use_base_cg = 1.0, 6.0, 1
    a = S.image(640, 360, "smooth", seed=5)
    gm = S.image(320, 200, "noise", seed=6)
    data = _api4(lib, S.pil_jpeg(a, 90, "420"), S.pil_jpeg(gm, 90, "444"), md, A.CG_BT709)
    assert isinstance(data, bytes), data
    return data


def restart_file(lib):
    from test_gpu_restart_decode import _dri_jpegr
    return _dri_jpegr(lib)[0]


def golden(name):
    return open(os.path.join(GOLDEN, name), "rb").read()


FILES = [("enc", w, h, s, m) for (w, h) in ((3840, 2160), (1920, 1080), (998, 722)) for (s, m) in ((1, 1), (2, 0), (4, 1))] \
    + [("apple_gainmap_old.jpg",), ("apple_gainmap_new.jpg",), ("restart",), ("resize",)]


def load(lib, spec):
    if spec[0] == "enc":
        return encoded(lib, *spec[1:])
    if spec[0] == "restart":
        return restart_file(lib)
    if spec[0] == "resize":
        return resize_file(lib)
    return golden(spec[0])


def _id(spec):
    return "-".join(str(s) for s in spec)


# ---- 1. full frame --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("spec", FILES, ids=_id)
def test_full_frame_equals_decode(lib, spec):
    data = load(lib, spec)
    for k in allowed_ks(lib, data):
        img = Image(lib, data, k)
        try:
            for fmt, ct in OUTPUTS:
                for boost in (boosts(img.md) if ct != A.CT_SRGB else [A.FLT_MAX]):
                    want, wdesc = full_decode(lib, data, k, fmt, ct, boost)
                    d = Dest(fmt, img.w, img.hh, pad=k % 3, off=k % 2)
                    assert img.render(d, ct, boost, 0, 0) == 0, lib.uhdr_b200_last_error()
                    got, ok = d.body()
                    assert ok, ("padding written", k, fmt, ct, boost)
                    assert torch().equal(got, want), (k, fmt, ct, boost, int((got != want).sum()))
                    assert (d.desc.cg, d.desc.ct, d.desc.range) == (wdesc.cg, wdesc.ct, wdesc.range), (k, ct)
                    if k == 1:
                        dense, _ = full_decode(lib, data, 1, fmt, ct, boost, dense=True)
                        assert torch().equal(got, dense), (fmt, ct, boost)
        finally:
            img.close()


# ---- 2. regions equal crops -----------------------------------------------------------------------------------------
def rects(w, h, scale, seed):
    """(x, y, rw, rh): corners, a full row and column, origins of every residue mod 4 with odd and even rows, origins
    off the map grid with rectangles crossing map cells, edge-touching ones, widths % 4 != 0, 50 seeded random ones"""
    r = [(0, 0, 1, 1), (w - 1, 0, 1, 1), (0, h - 1, 1, 1), (w - 1, h - 1, 1, 1), (0, h // 2, w, 1), (w // 3, 0, 1, h)]
    for ox in range(4):
        for oy in (0, 1, 2, 3):
            x, y = min(8 + ox, w - 1), min(6 + oy, h - 1)
            r.append((x, y, min(36, w - x), min(10, h - y)))
    s = max(scale, 2)
    for x, y in ((s + 1, s - 1), (2 * s - 1, 3 * s + 1), (s // 2, s // 2 + 1)):
        x, y = min(x, w - 1), min(y, h - 1)
        r.append((x, y, min(3 * s + 2, w - x), min(2 * s + 3, h - y)))
    r += [(w - min(w, 37), min(5, h - 1), min(w, 37), h - min(5, h - 1)), (min(4, w - 1), h - min(h, 9), w - min(4, w - 1),
                                                                              min(h, 9))]
    r += [(0, 0, min(w, 6), min(h, 4)), (min(4, w - 1), min(2, h - 1), min(w - min(4, w - 1), 13), min(h - min(2, h - 1), 6))]
    rs = np.random.RandomState(seed)
    for _ in range(50):
        rw, rh = int(rs.randint(1, min(w, 300) + 1)), int(rs.randint(1, min(h, 200) + 1))
        r.append((int(rs.randint(0, w - rw + 1)), int(rs.randint(0, h - rh + 1)), rw, rh))
    return r


REGION_FILES = [("enc", 1920, 1080, 1, 1), ("enc", 998, 722, 2, 0), ("enc", 998, 722, 4, 1), ("apple_gainmap_new.jpg",),
                ("resize",), ("restart",)]


@pytest.mark.parametrize("spec", REGION_FILES, ids=_id)
def test_regions_equal_crops(lib, spec):
    data = load(lib, spec)
    scale = spec[3] if spec[0] == "enc" else 2
    for k in allowed_ks(lib, data):
        img = Image(lib, data, k)
        try:
            for oi, (fmt, ct) in enumerate(OUTPUTS):
                bl = boosts(img.md)
                boost = bl[len(bl) // 2] if ct != A.CT_SRGB else A.FLT_MAX
                full, _ = full_decode(lib, data, k, fmt, ct, boost)
                bpp = BPP[fmt]
                for i, (x, y, rw, rh) in enumerate(rects(img.w, img.hh, max(1, scale // k), seed=17 * k + oi)):
                    d = Dest(fmt, rw, rh, pad=i % 3, off=i % 2)
                    assert img.render(d, ct, boost, x, y) == 0, (x, y, rw, rh, lib.uhdr_b200_last_error())
                    got, ok = d.body()
                    want = full[y:y + rh, x * bpp:(x + rw) * bpp]
                    assert ok, ("padding written", k, fmt, ct, (x, y, rw, rh))
                    assert torch().equal(got, want), (k, fmt, ct, (x, y, rw, rh), int((got != want).sum()))
        finally:
            img.close()


def test_regions_equal_reference_uhdr_decode(lib, oracle_libs):
    if not oracle_libs.have_ref():
        pytest.skip("reference build not available")
    ref = T.UhdrApi(oracle_libs.Ref().lib)
    for data in (encoded(lib, 998, 722, 2, 0), golden("apple_gainmap_new.jpg")):
        img = Image(lib, data, 1)
        try:
            for fmt, ct in OUTPUTS:
                for boost in (1.0, A.FLT_MAX):
                    px, _gm, _md, _cg = ref.decode(data, fmt, ct, boost)
                    bpp = BPP[fmt]
                    for x, y, rw, rh in ((0, 0, 1, 1), (img.w - 7, img.hh - 5, 7, 5), (3, 1, 129, 33), (64, 30, 256, 96)):
                        d = Dest(fmt, rw, rh, pad=1, off=1)
                        assert img.render(d, ct, boost, x, y) == 0
                        got, ok = d.body()
                        assert ok and (got.cpu().numpy() == px[y:y + rh, x * bpp:(x + rw) * bpp]).all(), \
                            (fmt, ct, boost, (x, y, rw, rh))
        finally:
            img.close()


# ---- 3. routes ------------------------------------------------------------------------------------------------------
def _route(lib, img, fmt, ct, x, y, w, h):
    before = apply_stats(lib)
    d = Dest(fmt, w, h)
    assert img.render(d, ct, 4.0, x, y) == 0, lib.uhdr_b200_last_error()
    torch().cuda.synchronize()
    return tuple(apply_stats(lib) - before)


def test_routes(lib):
    img = Image(lib, encoded(lib, 1920, 1080, 1, 1), 1)
    try:
        assert _route(lib, img, A.FMT_RGBAF16, A.CT_LINEAR, 64, 32, 256, 128) == (1, 0, 0, 0)   # k_apply_lin1
        assert _route(lib, img, A.FMT_RGBAF16, A.CT_LINEAR, 0, 0, 1920, 1080) == (1, 0, 0, 0)
        assert _route(lib, img, A.FMT_RGBA1010102, A.CT_PQ, 4, 2, 64, 8) == (0, 1, 0, 0)        # k_apply_fast
        for x, y, w, h in ((1, 0, 64, 8), (2, 2, 64, 8), (4, 1, 64, 8), (4, 2, 62, 8), (4, 2, 64, 7)):
            assert _route(lib, img, A.FMT_RGBAF16, A.CT_LINEAR, x, y, w, h) == (0, 0, 1, 0), (x, y, w, h)
    finally:
        img.close()
    for scale, mc in ((2, 0), (4, 1)):   # 1920 and 1080 are multiples of both: integer scales
        img = Image(lib, encoded(lib, 1920, 1080, scale, mc), 1)
        try:
            for ct in (A.CT_HLG, A.CT_PQ):
                assert _route(lib, img, A.FMT_RGBA1010102, ct, 8, 6, 128, 64) == (0, 1, 0, 0), (scale, ct)
                assert _route(lib, img, A.FMT_RGBA1010102, ct, 3, 6, 128, 64) == (0, 0, 1, 0), (scale, ct)
            assert _route(lib, img, A.FMT_RGBAF16, A.CT_LINEAR, 12, 10, 96, 40) == (0, 1, 0, 0), scale
        finally:
            img.close()
    for k in (2, 4, 8):
        img = Image(lib, encoded(lib, 1920, 1080, 1, 1), k)
        try:
            assert _route(lib, img, A.FMT_RGBAF16, A.CT_LINEAR, 8, 4, 64, 16) == (0, 0, 1, 0), k
        finally:
            img.close()
    before = apply_stats(lib)
    img = Image(lib, resize_file(lib), 1)   # the resize happens once, at open
    try:
        assert tuple(apply_stats(lib) - before) == (0, 0, 0, 1)
        assert _route(lib, img, A.FMT_RGBAF16, A.CT_LINEAR, 0, 0, img.w, img.hh) == (1, 0, 0, 0)
    finally:
        img.close()


# ---- 5. ordering and lifetime ---------------------------------------------------------------------------------------
def _file_with_headroom(lib):
    return encoded(lib, 998, 722, 1, 1)


def test_render_waits_for_the_callers_stream_not_the_host(lib):
    t = torch()
    data = _file_with_headroom(lib)
    want, _ = full_decode(lib, data, 1, A.FMT_RGBA1010102, A.CT_PQ, A.FLT_MAX)
    img = Image(lib, data, 1)
    try:
        d = Dest(A.FMT_RGBA1010102, img.w, img.hh, pad=2)
        st = t.cuda.Stream()
        with t.cuda.stream(st):
            t.cuda._sleep(_sleep_cycles(300))
            d.buf.zero_()
        t0 = time.perf_counter()
        rc = img.render(d, A.CT_PQ, A.FLT_MAX, 0, 0, st.cuda_stream)
        dt = time.perf_counter() - t0
        assert rc == 0
        st.synchronize()
        got, _ = d.body()
        assert t.equal(got, want), "the render went ahead of the caller's zero_()"
        assert dt < 0.15, ("the call waited for the caller's stream", dt)
    finally:
        img.close()


def test_table_slots_are_not_clobbered_across_streams(lib):
    t = torch()
    data = _file_with_headroom(lib)
    want1, _ = full_decode(lib, data, 1, A.FMT_RGBAF16, A.CT_LINEAR, 1.0)
    want_max, _ = full_decode(lib, data, 1, A.FMT_RGBAF16, A.CT_LINEAR, A.FLT_MAX)
    assert not t.equal(want1, want_max)
    img = Image(lib, data, 1)
    try:
        a, b = Dest(A.FMT_RGBAF16, img.w, img.hh), Dest(A.FMT_RGBAF16, img.w, img.hh)
        s1, s2 = t.cuda.Stream(), t.cuda.Stream()
        with t.cuda.stream(s1):
            t.cuda._sleep(_sleep_cycles(200))
        assert img.render(a, A.CT_LINEAR, 1.0, 0, 0, s1.cuda_stream) == 0
        assert img.render(b, A.CT_LINEAR, A.FLT_MAX, 0, 0, s2.cuda_stream) == 0
        t.cuda.synchronize()
        assert t.equal(a.body()[0], want1), "render A lost its boost-1 tables"
        assert t.equal(b.body()[0], want_max)
    finally:
        img.close()


def test_64_boosts_on_two_streams(lib):
    t = torch()
    data = encoded(lib, 998, 722, 2, 0)
    img = Image(lib, data, 1)
    try:
        lo, hi = max(1.0, img.md.hdr_capacity_min), img.md.hdr_capacity_max
        bs = [float(lo * (hi / lo) ** (i / 63.0)) for i in range(64)]
        wants = [full_decode(lib, data, 1, A.FMT_RGBA1010102, A.CT_HLG, b)[0] for b in bs]
        ss = [t.cuda.Stream(), t.cuda.Stream()]
        ds = [Dest(A.FMT_RGBA1010102, 200, 120, pad=i % 3) for i in range(64)]
        for i, b in enumerate(bs):
            assert img.render(ds[i], A.CT_HLG, b, 100 + i, 50, ss[i % 2].cuda_stream) == 0
        t.cuda.synchronize()
        for i in range(64):
            assert t.equal(ds[i].body()[0], wants[i][50:170, (100 + i) * 4:(300 + i) * 4]), i
    finally:
        img.close()


def test_release_right_after_a_pending_render(lib):
    t = torch()
    data = encoded(lib, 1920, 1080, 1, 1)
    want, _ = full_decode(lib, data, 1, A.FMT_RGBAF16, A.CT_LINEAR, 3.0)
    img = Image(lib, data, 1)
    d = Dest(A.FMT_RGBAF16, img.w, img.hh)
    st = t.cuda.Stream()
    with t.cuda.stream(st):
        t.cuda._sleep(_sleep_cycles(100))
    assert img.render(d, A.CT_LINEAR, 3.0, 0, 0, st.cuda_stream) == 0
    img.close()
    # the released memory goes back to the cache: reusing it at once must not disturb the render
    again = Image(lib, data, 1)
    again.close()
    st.synchronize()
    assert t.equal(d.body()[0], want)


def test_two_images_two_threads(lib):
    t = torch()
    jobs = [(encoded(lib, 998, 722, 1, 1), A.FMT_RGBAF16, A.CT_LINEAR), (encoded(lib, 998, 722, 4, 1), A.FMT_RGBA1010102,
                                                                         A.CT_PQ)]
    wants = [full_decode(lib, d, 1, f, c, 2.5)[0] for d, f, c in jobs]
    errors = []

    def work(i):
        try:
            data, fmt, ct = jobs[i]
            img = Image(lib, data, 1)
            st = t.cuda.Stream()
            try:
                for j in range(20):
                    x, y = 17 * j, 11 * j
                    d = Dest(fmt, 300, 200, pad=j % 2)
                    st.synchronize()
                    assert img.render(d, ct, 2.5, x, y, st.cuda_stream) == 0
                    st.synchronize()
                    bpp = BPP[fmt]
                    assert t.equal(d.body()[0], wants[i][y:y + 200, x * bpp:(x + 300) * bpp]), (i, j)
            finally:
                img.close()
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    th = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors


# ---- 6. errors write nothing ----------------------------------------------------------------------------------------
def test_bad_renders_write_nothing(lib):
    t = torch()
    img = Image(lib, encoded(lib, 998, 722, 2, 0), 1)
    try:
        d = Dest(A.FMT_RGBAF16, 64, 32)
        cases = [(A.CT_LINEAR, 4.0, img.w - 63, 0), (A.CT_LINEAR, 4.0, 0, img.hh - 31), (A.CT_LINEAR, 4.0, 1 << 31, 0),
                 (A.CT_HLG, 4.0, 0, 0), (A.CT_SRGB, 4.0, 0, 0), (A.CT_LINEAR, 0.5, 0, 0), (A.CT_LINEAR, float("nan"), 0, 0)]
        for ct, b, x, y in cases:
            assert img.render(d, ct, b, x, y) == INVALID, (ct, b, x, y)
        for w, h in ((0, 32), (64, 0)):
            z = Dest(A.FMT_RGBAF16, 64, 32)
            z.desc.w, z.desc.h = w, h
            assert img.render(z, A.CT_LINEAR, 4.0, 0, 0) == INVALID
        narrow = Dest(A.FMT_RGBAF16, 64, 32)
        narrow.desc.stride[0] = 63
        assert img.render(narrow, A.CT_LINEAR, 4.0, 0, 0) == INVALID
        host = np.full(64 * 32 * 8, GUARD, np.uint8)
        hd = A.raw_image(A.FMT_RGBAF16, -1, -1, -1, 64, 32, [host], [64])
        assert lib.uhdr_b200_image_render_dev(img.h, A.CT_LINEAR, 4.0, 0, 0, C.byref(hd), None) == INVALID
        assert (host == GUARD).all()
        if t.cuda.device_count() > 1:
            other = t.full((64 * 32 * 8,), GUARD, dtype=t.uint8, device="cuda:1")
            od = A.raw_image(A.FMT_RGBAF16, -1, -1, -1, 64, 32, [], [])
            od.planes[0], od.stride[0] = other.data_ptr(), 64
            assert lib.uhdr_b200_image_render_dev(img.h, A.CT_LINEAR, 4.0, 0, 0, C.byref(od), None) == INVALID
            assert bool((other == GUARD).all())
        t.cuda.synchronize()
        assert d.untouched() and narrow.untouched()
        assert lib.uhdr_b200_image_render_dev(None, A.CT_LINEAR, 4.0, 0, 0, C.byref(d.desc), None) == INVALID
        assert img.render(d, A.CT_LINEAR, 4.0, img.w - 64, img.hh - 32) == 0   # the same buffer, in bounds
    finally:
        img.close()


def _decode_code(lib, data, k):
    buf = np.frombuffer(data, np.uint8).copy()
    dims = [C.c_uint(64) for _ in range(4)]
    lib.uhdr_b200_scaled_dims(buf.ctypes.data, buf.size, k, *[C.byref(x) for x in dims])
    d = Dest(A.FMT_RGBAF16, dims[0].value, dims[1].value)
    return lib.uhdr_b200_decode_scaled_dev(buf.ctypes.data, buf.size, k, A.CT_LINEAR, 4.0, C.byref(d.desc), None, None,
                                           None)


def _open_code(lib, data, k):
    buf = np.frombuffer(data, np.uint8).copy()
    h = C.c_void_p(1234)
    rc = lib.uhdr_b200_image_open_dev(buf.ctypes.data, buf.size, k, C.byref(h))
    if rc == 0:
        lib.uhdr_b200_image_release(h)
    else:
        assert not h.value, "a failed open leaves a handle"
    return rc


def test_open_errors_match_decode(lib):
    data = encoded(lib, 998, 722, 2, 0)
    plain = S.pil_jpeg(S.image(320, 240, "smooth"), 90, "420")
    for bad in (data[:len(data) // 2], plain, data[:100]):
        for k in (1, 2):
            want = _decode_code(lib, bad, k)
            assert want != 0 and _open_code(lib, bad, k) == want, (k, want)
    for k in (0, 3, 16):
        assert _open_code(lib, data, k) == INVALID
    md = A.GainmapMetadata()
    for i in range(3):
        md.max_content_boost[i], md.min_content_boost[i], md.gamma[i] = 4.0, 1.0, 1.0
        md.offset_sdr[i] = md.offset_hdr[i] = 1.0 / 64
    md.hdr_capacity_min, md.hdr_capacity_max, md.use_base_cg = 1.0, 4.0, 1
    a = S.image(640, 360, "smooth")
    f422 = _api4(lib, S.pil_jpeg(a, 90, "422"), S.pil_jpeg(a[::2, ::2], 90, "gray"), md, A.CG_BT709)
    for k in (2, 4, 8):
        assert _decode_code(lib, f422, k) == UNSUPPORTED and _open_code(lib, f422, k) == UNSUPPORTED, k
    assert _open_code(lib, f422, 1) == 0
    torch().cuda.synchronize()


# ---- 7. memory ------------------------------------------------------------------------------------------------------
def test_8k_device_bytes(lib):
    sys.path.insert(0, T.ROOT)
    import bench
    p8, y8 = bench.make_frame(bench.W8K, bench.H8K, 7)
    h8, s8, _k = bench.frame_descs(p8, y8, bench.W8K, bench.H8K)
    data = T.UhdrApi(lib).encode(h8, s8)   # its released handle parks blocks; the image must not take a larger one
    img = Image(lib, data, 1)
    try:
        w, h = img.w, img.hh
        planes = w * h + 2 * ((w + 1) // 2) * ((h + 1) // 2)
        gmap = img.gw * img.gh * 4
        assert (w, h, img.gw, img.gh) == (7680, 4320, 7680, 4320)
        assert planes + gmap <= img.bytes.value <= 1.05 * (planes + gmap), (img.bytes.value, planes, gmap)
        want, _ = full_decode(lib, data, 1, A.FMT_RGBAF16, A.CT_LINEAR, A.FLT_MAX)
        d = Dest(A.FMT_RGBAF16, 1920, 1080)
        assert img.render(d, A.CT_LINEAR, A.FLT_MAX, 2880, 1620) == 0
        torch().cuda.synchronize()
        assert torch().equal(d.body()[0], want[1620:2700, 2880 * 8:4800 * 8])
    finally:
        img.close()
