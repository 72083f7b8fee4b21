"""Every applyGainMap route on the GPU against the CPU checker, bit exact (RGBA half-float bits, 1010102 words and
the destination gamut).

apply_gainmap_dev (engine.cu) picks one of three kernels; each route below is reached on purpose and the test asserts
which one ran through uhdr_b200_apply_stats (launches of k_apply_lin1, k_apply_fast, k_apply_gainmap, k_resize_map):

  A  k_apply_lin1: YUV420 base, map scale 1, linear output; 1 / 3 / 4-byte maps x gamut modes (none, base side,
     HDR side); w % 256 in {4, 252}, h % 8 in {2, 6}; tile counts below, near and far above the resident CTAs
  B  k_apply_fast at scale 1: PQ and HLG outputs
  C  k_apply_fast at scales 2, 3, 4, 5, 8, 16, all outputs; maps of w/s x floor(h/s) (the bottom rows clamp) and
     w/s x (h/s + 1) (within the 1 % aspect tolerance)
  D  k_apply_gainmap at integer scales: 17, 32, w % 4 != 0, odd h, gamma != 1, and (device-pointer API) a base
     pitch that is not a multiple of 4, a plane pointer one byte off, an odd destination pitch
  E  k_apply_gainmap at non-integer scales 1.5, 2.5, 3.2 and 0.5 (a map larger than the image)
  F  the gain map resized first (aspect ratio off by more than 1 %), then A or B
  G  YUV444, YUV422, RGB888 (which the reference runs through its BT.601 step: isPixelFormatRgb is false for it)
     and RGBA8888 bases at odd sizes

Inputs noise does not reach: a 4096 x 4096 base in which every (Y, U, V) triple occurs once, under a map whose
bytes cover every value with every luma value; IDW edge plants (all-255, all-0, 0/255 checkerboards, unique bytes
in the last map row and column); display boost and metadata matrices; non-finite intermediate values
(max_content_boost = FLT_MAX); every rule of the metadata validation; every gain byte under gamma != 1.
"""
import ctypes as C
import itertools
import threading

import numpy as np
import pytest

import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A

pytestmark = pytest.mark.gpu

LIN1, FAST, GEN = (1, 0, 0, 0), (0, 1, 0, 0), (0, 0, 1, 0)
OUTS = (A.CT_LINEAR, A.CT_PQ, A.CT_HLG)
F32 = np.float32


# ------------------------------------------------------------------------------------------------
# helpers
# ------------------------------------------------------------------------------------------------
def _stats(lib):
    st = (C.c_ulonglong * 4)()
    lib.uhdr_b200_apply_stats(st)
    return tuple(st)


class Route:
    """`n`: growth of uhdr_b200_apply_stats over the block (lin1, fast, generic, resize launches)"""

    def __init__(self, lib):
        self.lib = lib

    def __enter__(self):
        self.n0 = _stats(self.lib)
        return self

    def __exit__(self, *exc):
        self.n = tuple(b - a for a, b in zip(self.n0, _stats(self.lib)))
        return False


def with_resize(route):
    return route[:3] + (1,)


def _base(fmt, w, h, seed=0, pad=0):
    """seeded noise base image (host planes, rows of w + pad pixels) -> (RawImage, planes)"""
    rs = np.random.RandomState(T.SEED + 300 + seed)
    if fmt in (A.FMT_YUV420, A.FMT_YUV422, A.FMT_YUV444):
        cw = w if fmt == A.FMT_YUV444 else (w + 1) // 2
        chh = (h + 1) // 2 if fmt == A.FMT_YUV420 else h
        planes = [rs.randint(0, 256, (h, w + pad)).astype(np.uint8)] + \
                 [rs.randint(0, 256, (chh, cw + pad)).astype(np.uint8) for _ in range(2)]
        strides = [w + pad, cw + pad, cw + pad]
    else:
        bpp = 3 if fmt == A.FMT_RGB888 else 4
        p = rs.randint(0, 256, (h, w + pad, bpp)).astype(np.uint8)
        if bpp == 4:
            p[..., 3] = 255
        planes, strides = [p], [w + pad]
    return A.raw_image(fmt, A.CG_BT709, A.CT_SRGB, A.CR_FULL, w, h, planes, strides), planes


def _map(mw, mh, bpp, seed=0):
    rs = np.random.RandomState(T.SEED + 400 + seed)
    g = rs.randint(0, 256, (mh, mw, bpp)).astype(np.uint8)
    if bpp == 4:
        g[..., 3] = 255
    return g


def _md(mx=(8.0, 6.0, 4.0), mn=(0.5, 0.7, 1.0), gamma=(1.0, 1.0, 1.0), osdr=(1 / 64,) * 3, ohdr=(1 / 64,) * 3,
        cmin=1.0, cmax=8.0, use_base_cg=0):
    m = A.GainmapMetadata()
    for i in range(3):
        m.max_content_boost[i], m.min_content_boost[i], m.gamma[i] = mx[i], mn[i], gamma[i]
        m.offset_sdr[i], m.offset_hdr[i] = osdr[i], ohdr[i]
    m.hdr_capacity_min, m.hdr_capacity_max, m.use_base_cg = cmin, cmax, use_base_cg
    return m


def _apply(impl, sdr, gi, md, ct, boost=A.FLT_MAX):
    """-> (rc, pixels, destination gamut)"""
    w, h = sdr.w, sdr.h
    if ct == A.CT_LINEAR:
        out, fmt = np.zeros((h, w, 4), np.uint16), A.FMT_RGBAF16
    else:
        out, fmt = np.zeros((h, w), np.uint32), A.FMT_RGBA1010102
    dst = A.raw_image(fmt, -1, ct, A.CR_FULL, w, h, [out], [w])
    fn = impl.f("apply_gainmap")
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p]
    rc = fn(C.byref(sdr), C.byref(gi), C.byref(md), ct, fmt, boost, C.byref(dst))
    return rc, out, dst.cg


def _diff(a, b):
    if (a == b).all():
        return ""
    idx = np.argwhere(a != b)
    i = tuple(idx[0])
    return f"{len(idx)} values differ, first at {i}: {a[i]:#x} != {b[i]:#x}"


def _compare(gpu, checker, sdr, gi, md, ct, boost=A.FLT_MAX, route=None):
    """'' when the GPU equals the checker bit for bit (and took `route`), else a description"""
    with Route(gpu.lib) as r:
        rc, a, cga = _apply(gpu, sdr, gi, md, ct, boost)
    assert rc == 0, T.gpu_err(gpu)
    rc2, b, cgb = _apply(checker, sdr, gi, md, ct, boost)
    assert rc2 == 0, rc2
    if route is not None:
        assert r.n == route, (r.n, route)
    d = _diff(a, b)
    if cga != cgb:
        d += f" dest cg {cga} != {cgb}"
    return d


def _resizes(w, h, mw, mh):
    """the reference's 1 % aspect-ratio test (jpegr.cpp:1652-1660), in float"""
    pa, ga = F32(w) / F32(h), F32(mw) / F32(mh)
    return F32(abs(pa - ga)) / pa > F32(0.01)


# gamut mode -> (map gamut, use_base_cg) over a BT.709 base: identity, conversion on the base side, on the HDR side
GAMUT_MODES = {0: (A.CG_BT709, 0), 1: (A.CG_BT2100, 0), 2: (A.CG_BT2100, 1)}


def _run_cases(gpu, checker, cases):
    """cases: (label, sdr, map array, map gamut, metadata, output, boost, route)"""
    bad = []
    for label, sdr, gm, mcg, md, ct, boost, route in cases:
        gm = np.ascontiguousarray(gm)   # the descriptor points into it: keep it referenced
        d = _compare(gpu, checker, sdr, T.gm_image(gm, mcg), md, ct, boost, route)
        if d:
            bad.append((label, d))
    assert not bad, bad[:10]


# ------------------------------------------------------------------------------------------------
# 1. routes
# ------------------------------------------------------------------------------------------------
SIZES_A = [(260, 10), (508, 30), (1028, 722), (2052, 462), (3844, 2166)]


def cases_a():
    out = []
    for i, (w, h) in enumerate(SIZES_A):
        sdr, keep = _base(A.FMT_YUV420, w, h, i)
        combos = list(itertools.product((1, 3, 4), GAMUT_MODES)) if w < 3000 else [(1, 0), (3, 1), (4, 2)]
        for bpp, g in combos:
            mcg, ubc = GAMUT_MODES[g]
            out.append(((w, h, bpp, g), sdr, _map(w, h, bpp, i), mcg, _md(use_base_cg=ubc), A.CT_LINEAR, A.FLT_MAX,
                        LIN1, keep))
    return out


def cases_b():
    out = []
    w, h = 1028, 722
    sdr, keep = _base(A.FMT_YUV420, w, h, 1)
    for ct, bpp, g in itertools.product((A.CT_PQ, A.CT_HLG), (1, 3, 4), GAMUT_MODES):
        mcg, ubc = GAMUT_MODES[g]
        out.append(((ct, bpp, g), sdr, _map(w, h, bpp, bpp), mcg, _md(use_base_cg=ubc), ct, 2.5, FAST, keep))
    return out


def cases_c():
    out, k = [], 0
    for w, h, scales in ((960, 722, (2, 3, 4, 5, 8, 16)), (1000, 722, (4,))):
        sdr, keep = _base(A.FMT_YUV420, w, h, w)
        for s in scales:
            for mh in (h // s, h // s + 1):
                if _resizes(w, h, w // s, mh):
                    continue
                for ct in OUTS:
                    bpp = (1, 3, 4)[k % 3]
                    mcg, ubc = GAMUT_MODES[k % 3]
                    k += 1
                    out.append(((w, h, s, mh, ct, bpp), sdr, _map(w // s, mh, bpp, k), mcg, _md(use_base_cg=ubc), ct,
                                A.FLT_MAX, FAST, keep))
    return out


def cases_d():
    out = []
    geo = [(1088, 680, 17), (1024, 640, 32), (1002, 722, 1), (1002, 722, 2), (1000, 721, 1)]
    for i, (w, h, s) in enumerate(geo):
        sdr, keep = _base(A.FMT_YUV420, w, h, 10 + i)
        for j, ct in enumerate(OUTS):
            bpp = (1, 3, 4)[(i + j) % 3]
            out.append(((w, h, s, ct, bpp), sdr, _map(w // s, h // s, bpp, i), A.CG_BT2100, _md(), ct, A.FLT_MAX, GEN,
                        keep))
    # gamma != 1 takes the generic kernel at every scale; scale 1 only here (scale 4: test_gamma_scaled)
    sdr, keep = _base(A.FMT_YUV420, 1028, 722, 20)
    for ct in OUTS:
        out.append((("gamma", ct), sdr, _map(1028, 722, 3, 20), A.CG_P3, _md(gamma=(2.2, 0.7, 1.0)), ct, A.FLT_MAX,
                    GEN, keep))
    return out


def cases_e():
    out = []
    w, h = 960, 720
    sdr, keep = _base(A.FMT_YUV420, w, h, 30)
    for i, (mw, mh) in enumerate(((640, 480), (384, 288), (300, 225), (1920, 1440))):
        for bpp in (1, 3):
            ct = OUTS[(i + bpp) % 3]
            out.append(((mw, mh, bpp, ct), sdr, _map(mw, mh, bpp, i), A.CG_BT2100, _md(use_base_cg=i % 2), ct, 2.5, GEN,
                        keep))
    return out


def cases_g():
    out = []
    for i, (fmt, (w, h)) in enumerate(itertools.product((A.FMT_YUV444, A.FMT_YUV422, A.FMT_RGB888, A.FMT_RGBA8888),
                                                        ((321, 181), (320, 180)))):
        sdr, keep = _base(fmt, w, h, 40 + i)
        for (mw, mh), ct in zip(((w, h), (214, 121), (w // 4, h // 4)), OUTS):
            assert not _resizes(w, h, mw, mh)
            bpp = (1, 3, 4)[i % 3]
            out.append(((fmt, w, h, mw, mh, ct), sdr, _map(mw, mh, bpp, i), A.CG_P3, _md(use_base_cg=i % 2), ct,
                        A.FLT_MAX, GEN, keep))
    return out


ROUTES = {"A_lin1": cases_a, "B_fast_scale1": cases_b, "C_fast_scaled": cases_c, "D_generic_integer": cases_d,
          "E_generic_fractional": cases_e, "G_other_bases": cases_g}


@pytest.mark.parametrize("route", sorted(ROUTES))
def test_route(gpu, checker, route):
    cases = ROUTES[route]()   # holds the base planes the descriptors point into
    _run_cases(gpu, checker, [c[:8] for c in cases])


def test_route_f_resized(gpu, oracle_libs):
    """F: resize_image first (the C restatement does not cover it), then k_apply_lin1 or k_apply_fast"""
    if not oracle_libs.have_ref():
        pytest.skip("reference build not available")
    ref = oracle_libs.Ref()
    w, h = 1024, 512
    sdr, keep = _base(A.FMT_YUV420, w, h, 50)
    cases = []
    for i, (mw, mh, bpp) in enumerate(((100, 80, 4), (77, 13, 1), (300, 100, 3), (512, 512, 4))):
        assert _resizes(w, h, mw, mh)
        for ct in OUTS:
            route = with_resize(LIN1 if ct == A.CT_LINEAR else FAST)
            cases.append(((mw, mh, bpp, ct), sdr, _map(mw, mh, bpp, i), A.CG_BT2100, _md(use_base_cg=i % 2), ct,
                          A.FLT_MAX, route))
    _run_cases(gpu, ref, cases)


# ------------------------------------------------------------------------------------------------
# 2. the base-pixel x gain-code lattice
# ------------------------------------------------------------------------------------------------
LAT = 4096


@pytest.fixture(scope="module")
def lattice():
    """4096 x 4096 YUV420 in which every (Y, U, V) occurs exactly once: chroma sample c carries
    (U, V) = (c mod 65536) as (low byte, high byte), its four luma samples are 4k .. 4k+3 with k = c div 65536.
    Map: RGBA, bytes r = P0[U], g = P1[V], b = P2[(U + V) mod 256] (fixed permutations), so under every luma value
    each channel takes every byte."""
    c = np.arange((LAT // 2) ** 2, dtype=np.int64).reshape(LAT // 2, LAT // 2)
    uv, k = c % 65536, c // 65536
    u, v = (uv & 255).astype(np.uint8), (uv >> 8).astype(np.uint8)
    y = np.empty((LAT, LAT), np.uint8)
    for dy, dx in itertools.product((0, 1), (0, 1)):
        y[dy::2, dx::2] = 4 * k + 2 * dy + dx
    rs = np.random.RandomState(T.SEED + 500)
    P = [rs.permutation(256).astype(np.uint8) for _ in range(3)]
    ui, vi = u.astype(np.int64), v.astype(np.int64)
    cm = np.stack([P[0][ui], P[1][vi], P[2][(ui + vi) % 256], np.full_like(u, 255)], -1)
    gm = np.ascontiguousarray(np.repeat(np.repeat(cm, 2, 0), 2, 1))
    return y, u, v, gm


def _lattice_check(gpu, checker, lattice, ct, ubc, route, dev_pitch=0):
    y, u, v, gm = lattice
    sdr = A.raw_image(A.FMT_YUV420, A.CG_BT709, A.CT_SRGB, A.CR_FULL, LAT, LAT, [y, u, v], [LAT, LAT // 2, LAT // 2])
    gi = T.gm_image(gm, A.CG_BT2100)
    md = _md(mx=(24.0, 7.5, 3.0), mn=(0.25, 0.9, 1.0 / 3), osdr=(1 / 64, 1e-7, 0.0), ohdr=(0.0, 1 / 64, 1e-7),
             cmin=1.0, cmax=24.0, use_base_cg=ubc)
    rc2, want, _ = _apply(checker, sdr, gi, md, ct)
    assert rc2 == 0
    if dev_pitch:
        got = _apply_dev(gpu, sdr, [y, u, v], gm, md, ct, pitch=(LAT + dev_pitch, LAT // 2 + dev_pitch), route=route)
    else:
        with Route(gpu.lib) as r:
            rc, got, _ = _apply(gpu, sdr, gi, md, ct)
        assert rc == 0, T.gpu_err(gpu)
        assert r.n == route, r.n
    d = _diff(got, want)
    assert not d, d


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_lattice_lin1(gpu, checker, lattice, mode):
    """A on the lattice; mode 0 uses a BT.709 map (no gamut step), 1 / 2 a BT.2100 one with use_base_cg 0 / 1"""
    y, u, v, gm = lattice
    sdr = A.raw_image(A.FMT_YUV420, A.CG_BT709, A.CT_SRGB, A.CR_FULL, LAT, LAT, [y, u, v], [LAT, LAT // 2, LAT // 2])
    gi = T.gm_image(gm, A.CG_BT709 if mode == 0 else A.CG_BT2100)
    md = _md(mx=(24.0, 7.5, 3.0), mn=(0.25, 0.9, 1.0 / 3), osdr=(1 / 64, 1e-7, 0.0), ohdr=(0.0, 1 / 64, 1e-7),
             cmin=1.0, cmax=24.0, use_base_cg=1 if mode == 2 else 0)
    d = _compare(gpu, checker, sdr, gi, md, A.CT_LINEAR, A.FLT_MAX, LIN1)
    assert not d, d


def test_lattice_fast_pq(gpu, checker, lattice):
    _lattice_check(gpu, checker, lattice, A.CT_PQ, 0, FAST)


def test_lattice_generic(gpu, checker, lattice):
    """base rows of 4096 + 2 bytes through the device-pointer API: the generic kernel on the same lattice"""
    _lattice_check(gpu, checker, lattice, A.CT_LINEAR, 1, GEN, dev_pitch=2)


# ------------------------------------------------------------------------------------------------
# 3. IDW edges
# ------------------------------------------------------------------------------------------------
def _plants(mw, mh, bpp):
    base = np.full((mh, mw, bpp), 100, np.uint8)
    edge = base.copy()
    edge[:, -1] = 250
    edge[-1, :] = 7
    edge[-1, -1] = 255
    chk = np.where(((np.arange(mh)[:, None] + np.arange(mw)[None, :]) % 2 == 0)[..., None], 255, 0)
    chk = np.broadcast_to(chk, (mh, mw, bpp)).astype(np.uint8)
    return {"all255": np.full((mh, mw, bpp), 255, np.uint8), "all0": np.zeros((mh, mw, bpp), np.uint8),
            "checker": chk, "checker_inv": 255 - chk, "edge": edge}


IDW_SCALES = [2, 3, 4, 5, 8, 16, 1.5, 2.5, 3.2, 0.5]


@pytest.mark.parametrize("s", IDW_SCALES, ids=[str(s) for s in IDW_SCALES])
def test_idw_edges(gpu, checker, s):
    integer = float(s).is_integer()
    w, h = 960, 722 if integer else 720
    mw, mh = (w // s, h // s) if integer else (int(w / s), int(h / s))
    assert not _resizes(w, h, mw, mh)
    sdr, keep = _base(A.FMT_YUV420, w, h, 60)
    cases = []
    for bpp in (1, 4):
        for name, gm in _plants(mw, mh, bpp).items():
            for ct in (A.CT_LINEAR, A.CT_PQ):
                cases.append(((s, bpp, name, ct), sdr, gm, A.CG_BT709, _md(), ct, A.FLT_MAX, FAST if integer else GEN))
    _run_cases(gpu, checker, cases)


# ------------------------------------------------------------------------------------------------
# 4. display boost and metadata
# ------------------------------------------------------------------------------------------------
# route -> (w, h, map scale, output, expected kernel)
MD_ROUTES = {"A": (1028, 90, 1, A.CT_LINEAR, LIN1), "B": (1028, 90, 1, A.CT_PQ, FAST),
             "C": (1024, 88, 4, A.CT_HLG, FAST), "C_lin": (1024, 88, 4, A.CT_LINEAR, FAST)}


def _md_cases(route):
    w, h, s, ct, kern = MD_ROUTES[route]
    sdr, keep = _base(A.FMT_YUV420, w, h, 70)
    g3, g1 = _map(w // s, h // s, 3, 70), _map(w // s, h // s, 1, 71)
    cases = []
    # boost below, at, between and above [hdr_capacity_min, hdr_capacity_max]
    for cmin in (1.0, 2.0):
        cmax = 8.0
        for boost in (0.5, 1.0, cmin, (cmin * cmax) ** 0.5, 7.999, cmax, 20.0, A.FLT_MAX):
            cases.append((("boost", cmin, boost), sdr, g3, A.CG_BT2100, _md(cmin=cmin, cmax=cmax), ct, boost, kern))
    # offsets, one and three channels, metadata identical across channels or not
    offs = [(0.0,) * 3, (1e-7,) * 3, (1 / 64,) * 3, (0.0, 1e-7, 1 / 64), (1 / 64, 0.0, 1e-7)]
    for (osdr, ohdr), gm in itertools.product(itertools.product(offs, offs[::2]), (g1, g3)):
        cases.append((("offsets", osdr, ohdr, gm.shape[2]), sdr, gm, A.CG_P3, _md(osdr=osdr, ohdr=ohdr), ct, 3.0, kern))
    same = dict(mx=(6.0,) * 3, mn=(0.5,) * 3, osdr=(1e-7,) * 3, ohdr=(1e-7,) * 3)
    for gm in (g1, g3):
        cases.append((("identical", gm.shape[2]), sdr, gm, A.CG_BT709, _md(**same), ct, A.FLT_MAX, kern))
    # base gamut x map gamut x use_base_cg
    for bcg, mcg, ubc in itertools.product((A.CG_BT709, A.CG_P3, A.CG_BT2100), (-1, 0, 1, 2), (0, 1)):
        b, k2 = _base(A.FMT_YUV420, w, h, 70)
        b.cg = bcg
        keep.append(k2)
        cases.append((("gamut", bcg, mcg, ubc), b, g3, mcg, _md(use_base_cg=ubc), ct, 4.0, kern))
    return cases, keep


@pytest.mark.parametrize("route", sorted(MD_ROUTES))
def test_boost_and_metadata(gpu, checker, route):
    cases, keep = _md_cases(route)
    _run_cases(gpu, checker, cases)


# ------------------------------------------------------------------------------------------------
# 5. non-finite intermediate values: max_content_boost = FLT_MAX puts +inf into the gain table
# ------------------------------------------------------------------------------------------------
NF_CASES = [  # (label, base format, w, h, map (mw, mh), outputs, kernel)
    ("lin1", A.FMT_YUV420, 1028, 90, (1028, 90), (A.CT_LINEAR,), LIN1),
    ("fast_s1", A.FMT_YUV420, 1028, 90, (1028, 90), (A.CT_PQ, A.CT_HLG), FAST),
    ("fast_s2", A.FMT_YUV420, 1024, 88, (512, 44), OUTS, FAST),
    ("fast_s4", A.FMT_YUV420, 1024, 88, (256, 22), OUTS, FAST),
    ("generic_s17", A.FMT_YUV420, 1088, 68, (64, 4), OUTS, GEN),
    ("generic_s1.5", A.FMT_YUV420, 960, 90, (640, 60), OUTS, GEN),
    ("generic_rgba", A.FMT_RGBA8888, 1028, 90, (1028, 90), OUTS, GEN),
]


def _black_planted(fmt, w, h, seed):
    """noise base with black blocks (RGB 0 after the YUV step): 0 * inf in the gain step"""
    sdr, planes = _base(fmt, w, h, seed)
    if fmt == A.FMT_YUV420:
        for yy in range(0, h - 8, 24):
            for xx in range(0, w - 8, 40):
                planes[0][yy:yy + 8, xx:xx + 8] = 0
                planes[1][yy // 2:yy // 2 + 4, xx // 2:xx // 2 + 4] = 128
                planes[2][yy // 2:yy // 2 + 4, xx // 2:xx // 2 + 4] = 128
    else:
        for yy in range(0, h - 8, 24):
            for xx in range(0, w - 8, 40):
                planes[0][yy:yy + 8, xx:xx + 8, :3] = 0
    return sdr, planes


@pytest.mark.parametrize("case", NF_CASES, ids=[c[0] for c in NF_CASES])
def test_non_finite(gpu, checker, case):
    """Black base pixels with offsets of 0 give 0 * inf = NaN; use_base_cg = 1 with a gamut conversion gives
    inf - inf.  Both pass the reference's clamps (comparisons) and reach floatToHalf as x86's default NaN."""
    label, fmt, w, h, (mw, mh), outs, kern = case
    sdr, keep = _black_planted(fmt, w, h, 80)
    cases = []
    for bpp in (1, 3):
        gm = _map(mw, mh, bpp, 80 + bpp)
        gm[::2, ::3] = 255   # the +inf entry of every channel's table
        for ubc, mcg in ((0, A.CG_BT709), (1, A.CG_BT2100), (0, A.CG_BT2100)):
            md = _md(mx=(A.FLT_MAX,) * 3, mn=(1.0,) * 3, osdr=(0.0,) * 3, ohdr=(0.0,) * 3, cmin=1.0, cmax=16.0,
                     use_base_cg=ubc)
            for ct in outs:
                cases.append(((bpp, ubc, mcg, ct), sdr, gm, mcg, md, ct, A.FLT_MAX, kern))
    # the case must contain NaN channels in the reference's output, else it tests nothing
    lab, s0, gm0, mcg0, md0, ct0, b0, _k = cases[0]
    if ct0 == A.CT_LINEAR:
        rc, ref, _ = _apply(checker, s0, T.gm_image(gm0, mcg0), md0, ct0, b0)
        assert rc == 0 and np.isnan(ref.view(np.float16)).any()
    _run_cases(gpu, checker, cases)


# ------------------------------------------------------------------------------------------------
# 6. invalid metadata (uhdr_validate_gainmap_metadata_descriptor)
# ------------------------------------------------------------------------------------------------
NAN, INF = float("nan"), float("inf")
BAD_MD = {
    "max_lt_min": dict(mx=(8.0, 0.5, 4.0), mn=(0.5, 0.6, 1.0)),
    "min_zero": dict(mn=(0.0, 0.7, 1.0)),
    "min_negative": dict(mx=(8.0, 6.0, 4.0), mn=(0.5, 0.7, -1.0)),
    "gamma_zero": dict(gamma=(1.0, 0.0, 1.0)),
    "gamma_negative": dict(gamma=(-2.2, -2.2, -2.2)),
    "offset_sdr_negative": dict(osdr=(0.0, 0.0, -1e-3)),
    "offset_hdr_negative": dict(ohdr=(-1e-7, 0.0, 0.0)),
    "capacity_equal": dict(cmin=2.0, cmax=2.0),
    "capacity_max_below_min": dict(cmin=4.0, cmax=2.0),
    "capacity_min_below_1": dict(cmin=0.5, cmax=8.0),
    "nan_max": dict(mx=(NAN, 6.0, 4.0)),
    "inf_max": dict(mx=(INF, INF, INF)),
    "inf_gamma": dict(gamma=(1.0, 1.0, INF)),
    "nan_offset": dict(osdr=(1 / 64, NAN, 1 / 64)),
    "inf_offset_hdr": dict(ohdr=(INF, 0.0, 0.0)),
    "nan_capacity_max": dict(cmax=NAN),
    "inf_capacity_max": dict(cmax=INF),
}


def test_invalid_metadata(gpu, oracle_libs):
    """One case per validation rule, plus NaN / inf fields: the GPU's host-buffer and device-pointer entry points
    refuse with the reference's error code and launch nothing."""
    if not oracle_libs.have_ref():
        pytest.skip("reference build not available")
    import torch
    ref = oracle_libs.Ref()
    w, h = 260, 10
    sdr, keep = _base(A.FMT_YUV420, w, h, 90)
    gm = _map(w, h, 3, 90)
    gi = T.gm_image(gm, A.CG_BT2100)
    bad = []
    for name, kw in BAD_MD.items():
        md = _md(**kw)
        for ct in (A.CT_LINEAR, A.CT_PQ):
            rc_ref = _apply(ref, sdr, gi, md, ct)[0]
            with Route(gpu.lib) as r:
                rc = _apply(gpu, sdr, gi, md, ct)[0]
            if rc_ref == 0 or rc != rc_ref or r.n != (0, 0, 0, 0):
                bad.append((name, ct, rc, rc_ref, r.n))
        # device-pointer API: the same code, nothing enqueued
        dev = _dev_images(torch, sdr, keep, gm, A.CG_BT2100, A.CT_LINEAR, w, h)
        with Route(gpu.lib) as r:
            rc = gpu.lib.uhdr_b200_apply_gainmap_dev(C.byref(dev["sdr"]), C.byref(dev["map"]), C.byref(md), A.CT_LINEAR,
                                                     C.c_float(A.FLT_MAX), C.byref(dev["dst"]), None)
        torch.cuda.synchronize()
        if rc != _apply(ref, sdr, gi, md, A.CT_LINEAR)[0] or r.n != (0, 0, 0, 0):
            bad.append((name, "dev", rc, r.n))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------
# 7. gamma != 1: every gain byte
# ------------------------------------------------------------------------------------------------
GAMMAS = [0.5, 0.7, 1 / 2.2, 2.2, 3.0]


def test_gamma_every_byte(gpu, checker):
    """At scale 1 the gain input is one of 256 values per channel (b / 255.0f): every byte under every gamma, a
    different gamma per channel, bit exact (the device's pow(double) must give the reference's LUT index)."""
    w, h = 1024, 64
    sdr, keep = _base(A.FMT_YUV420, w, h, 100)
    xx = np.arange(w)[None, :] + np.arange(h)[:, None]
    cases = []
    for i, g in enumerate(GAMMAS):
        gammas = (g, GAMMAS[(i + 1) % 5], GAMMAS[(i + 2) % 5])
        gm3 = np.stack([(xx * 7 + c * 85) % 256 for c in range(3)], -1).astype(np.uint8)
        for gm in (gm3, gm3[..., :1]):
            for ct in (A.CT_LINEAR, A.CT_PQ):
                cases.append(((gammas, gm.shape[2], ct), sdr, gm, A.CG_BT2100, _md(gamma=gammas), ct, 3.0, GEN))
    _run_cases(gpu, checker, cases)


def test_gamma_scaled(gpu, checker):
    """gamma != 1 at scales 2 and 4: the IDW sum is continuous, so pow(double) on the device and in glibc may put a
    tie on different sides; the bound of test_apply_gamma_metadata, with the measured count printed"""
    w, h = 1024, 512
    sdr, keep = _base(A.FMT_YUV420, w, h, 101)
    for s, g, ct in ((2, 2.2, A.CT_LINEAR), (4, 0.5, A.CT_LINEAR), (4, 3.0, A.CT_PQ)):
        gm = _map(w // s, h // s, 3, s)
        gi = T.gm_image(gm, A.CG_BT2100)
        md = _md(gamma=(g, g, g))
        with Route(gpu.lib) as r:
            rc, a, _ = _apply(gpu, sdr, gi, md, ct)
        assert rc == 0 and r.n == GEN, r.n
        b = _apply(checker, sdr, gi, md, ct)[1]
        n = int((a != b).sum())
        print(f"gamma {g} scale {s} out {ct}: {n} of {a.size} values differ")
        assert n <= 1e-5 * a.size, n


# ------------------------------------------------------------------------------------------------
# 8. device-pointer API
# ------------------------------------------------------------------------------------------------
SENTINEL = 0xA5


def _dev_images(torch, sdr, planes, gm, mcg, ct, w, h, pitch=None, offset=0, map_pitch=None, dst_pitch=None):
    """device copies of a YUV420 base (rows of pitch[0] / pitch[1] bytes, the Y plane `offset` bytes into its
    allocation), a map (rows of map_pitch pixels) and a destination (rows of dst_pitch pixels, all SENTINEL bytes)"""
    py, pc = pitch or (w, (w + 1) // 2)
    ys = torch.full((h * py + offset + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    yv = ys[offset:offset + h * py].view(h, py)
    yv[:, :w] = torch.from_numpy(np.ascontiguousarray(planes[0][:h, :w])).cuda()
    cs = []
    for p in planes[1:]:
        t = torch.full((p.shape[0], pc), SENTINEL, dtype=torch.uint8, device="cuda")
        t[:, :p.shape[1]] = torch.from_numpy(np.ascontiguousarray(p[:, :(w + 1) // 2])).cuda()
        cs.append(t)
    mh, mw, bpp = gm.shape
    mp = map_pitch or mw
    mt = torch.zeros((mh, mp * bpp), dtype=torch.uint8, device="cuda")
    mt[:, :mw * bpp] = torch.from_numpy(gm.reshape(mh, mw * bpp)).cuda()
    esz = 8 if ct == A.CT_LINEAR else 4
    dp = dst_pitch or w
    dt = torch.full((h, dp * esz), SENTINEL, dtype=torch.uint8, device="cuda")
    sd = A.RawImage()
    sd.fmt, sd.cg, sd.ct, sd.range, sd.w, sd.h = A.FMT_YUV420, sdr.cg, A.CT_SRGB, A.CR_FULL, w, h
    sd.planes[0], sd.planes[1], sd.planes[2] = ys.data_ptr() + offset, cs[0].data_ptr(), cs[1].data_ptr()
    sd.stride[0], sd.stride[1], sd.stride[2] = py, pc, pc
    md_ = A.RawImage()
    md_.fmt = {1: A.FMT_Y400, 3: A.FMT_RGB888, 4: A.FMT_RGBA8888}[bpp]
    md_.cg, md_.ct, md_.range, md_.w, md_.h = mcg, -1, -1, mw, mh
    md_.planes[0], md_.stride[0] = mt.data_ptr(), mp
    dd = A.RawImage()
    dd.fmt = A.FMT_RGBAF16 if ct == A.CT_LINEAR else A.FMT_RGBA1010102
    dd.w, dd.h = w, h
    dd.planes[0], dd.stride[0] = dt.data_ptr(), dp
    return {"sdr": sd, "map": md_, "dst": dd, "keep": (ys, cs, mt), "dst_t": dt, "esz": esz}


def _apply_dev(gpu, sdr, planes, gm, md, ct, pitch=None, offset=0, map_pitch=None, dst_pitch=None, route=None,
               mcg=A.CG_BT2100):
    """uhdr_b200_apply_gainmap_dev on a side stream -> the pixels, as _apply returns them; asserts that no padding
    byte of the destination was written"""
    import torch
    w, h = sdr.w, sdr.h
    dev = _dev_images(torch, sdr, planes, gm, mcg, ct, w, h, pitch, offset, map_pitch, dst_pitch)
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    with Route(gpu.lib) as r:
        rc = gpu.lib.uhdr_b200_apply_gainmap_dev(C.byref(dev["sdr"]), C.byref(dev["map"]), C.byref(md), ct,
                                                 C.c_float(A.FLT_MAX), C.byref(dev["dst"]), C.c_void_p(st.cuda_stream))
        assert rc == 0, T.gpu_err(gpu)
        st.synchronize()
    if route is not None:
        assert r.n == route, (r.n, route)
    got = dev["dst_t"].cpu().numpy()
    esz = dev["esz"]
    assert (got[:, w * esz:] == SENTINEL).all(), "bytes past the destination width were written"
    px = np.ascontiguousarray(got[:, :w * esz])
    return px.view(np.uint16).reshape(h, w, 4) if ct == A.CT_LINEAR else px.view(np.uint32).reshape(h, w)


DEV_CASES = {
    # name -> (w, h, map scale, output, base pitches, Y offset, map pitch, destination pitch, kernel)
    "lin1_pitched": (1028, 722, 1, A.CT_LINEAR, (1088, 576), 0, 1040, 1040, LIN1),
    "fast_s4_pitched": (1028, 722, 4, A.CT_PQ, (1088, 576), 0, 300, 1032, FAST),
    "fast_s2_linear_pitched": (1028, 722, 2, A.CT_LINEAR, (1088, 576), 0, 520, 1032, FAST),
    "generic_base_pitch": (1028, 722, 1, A.CT_LINEAR, (1030, 515), 0, 1040, 1040, GEN),
    "generic_plane_offset": (1028, 722, 1, A.CT_LINEAR, (1088, 576), 1, 1040, 1040, GEN),
    "generic_odd_dst_pitch": (1028, 722, 1, A.CT_LINEAR, (1088, 576), 0, 1040, 1029, GEN),
    "generic_odd_dst_pitch_hlg": (1028, 722, 4, A.CT_HLG, (1088, 576), 0, 257, 1031, GEN),
}


@pytest.mark.parametrize("name", sorted(DEV_CASES))
def test_dev_api(gpu, checker, name):
    w, h, s, ct, pitch, off, mp, dp, kern = DEV_CASES[name]
    sdr, planes = _base(A.FMT_YUV420, w, h, 110)
    gm = _map(w // s, h // s, 4 if s == 1 else 3, 110)
    md = _md(use_base_cg=1)
    want = _apply(checker, sdr, T.gm_image(gm, A.CG_BT2100), md, ct)[1]
    got = _apply_dev(gpu, sdr, planes, gm, md, ct, pitch, off, mp, dp, kern)
    d = _diff(got, want)
    assert not d, d


# ------------------------------------------------------------------------------------------------
# 9. concurrency
# ------------------------------------------------------------------------------------------------
def test_concurrent_apply(gpu, checker):
    """four host threads call uhdr_b200_apply_gainmap at once, each on another route, three times each"""
    jobs = []
    for i, (w, h, mw, mh, bpp, ct, gamma, kern) in enumerate((
            (1028, 722, 1028, 722, 4, A.CT_LINEAR, 1.0, LIN1), (1024, 720, 256, 180, 3, A.CT_PQ, 1.0, FAST),
            (960, 720, 640, 480, 1, A.CT_LINEAR, 1.0, GEN), (1028, 722, 1028, 722, 3, A.CT_HLG, 2.2, GEN))):
        sdr, keep = _base(A.FMT_YUV420, w, h, 120 + i)
        gm = _map(mw, mh, bpp, 120 + i)
        gi = T.gm_image(gm, A.CG_BT2100)
        md = _md(gamma=(gamma,) * 3)
        want = _apply(checker, sdr, gi, md, ct)[1]
        jobs.append((sdr, keep, gm, gi, md, ct, want, kern))
    errs, gate = [], threading.Barrier(len(jobs))

    def work(i):
        sdr, keep, gm, gi, md, ct, want, kern = jobs[i]
        try:
            gate.wait()
            for _ in range(3):
                rc, got, _ = _apply(gpu, sdr, gi, md, ct)
                assert rc == 0
                d = _diff(got, want)
                assert not d, d
        except BaseException as e:  # noqa: BLE001
            errs.append((i, repr(e)))
            gate.abort()

    with Route(gpu.lib) as r:
        th = [threading.Thread(target=work, args=(i,)) for i in range(len(jobs))]
        for t in th:
            t.start()
        for t in th:
            t.join()
    assert not errs, errs
    assert r.n == (3, 3, 6, 0), r.n


# ------------------------------------------------------------------------------------------------
# 10. uhdr_decode end to end
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", [(1000, 722), (998, 722), (1024, 576)])
def test_decode_end_to_end(gpu, oracle_libs, w, h):
    """files the reference encodes at map scale 1 / 2 / 4 with 1 and 3 channels, decoded to all three outputs with
    and without a display boost: pixels, map and metadata equal the reference's decode"""
    if not oracle_libs.have_ref():
        pytest.skip("reference build not available")
    ref = T.UhdrApi(oracle_libs.Ref().lib)
    mine = T.UhdrApi(gpu.lib)
    hb, sb = T.make_p010(w, h, "smooth"), T.make_yuv420(w, h, "noise", seed=T.SEED + 130)
    hdr, k1 = A.p010_image(hb, w, h, A.CG_BT2100, A.CT_HLG, A.CR_LIMITED)
    sdr, k2 = A.yuv420_image(sb, w, h, A.CG_BT709)
    bad = []
    for scale, multi in itertools.product((1, 2, 4), (0, 1)):
        data = ref.encode(hdr, sdr, scale=scale, multichannel=multi)
        for (fmt, ct), boost in itertools.product(((A.FMT_RGBAF16, A.CT_LINEAR), (A.FMT_RGBA1010102, A.CT_PQ),
                                                   (A.FMT_RGBA1010102, A.CT_HLG)), (None, 2.5)):
            with Route(gpu.lib) as r:
                px, gm, md, cg = mine.decode(data, fmt, ct, boost)
            rpx, rgm, rmd, rcg = ref.decode(data, fmt, ct, boost)
            assert sum(r.n[:3]) == 1, r.n
            if not ((px == rpx).all() and (gm == rgm).all() and T.md_equal(md, rmd) and cg == rcg):
                bad.append((scale, multi, ct, boost, int((px != rpx).sum())))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------
# 11. toneMap at partial tiles
# ------------------------------------------------------------------------------------------------
def _tm_groups(lib):
    st = (C.c_ulonglong * 2)()
    lib.uhdr_b200_tonemap_stats(st)
    return st[0]


@pytest.mark.parametrize("w,h", [(1000, 722), (260, 10), (3844, 2166)])
def test_tonemap_partial_tiles(gpu, checker, w, h):
    """k_tonemap_fast with w % 256 != 0 and h % 8 != 0 over several tile columns"""
    bad = []
    for ct, cg, kind in ((A.CT_HLG, A.CG_BT2100, "noise"), (A.CT_PQ, A.CG_P3, "smooth")):
        hb = T.make_p010(w, h, kind, seed=T.SEED + 140)
        hdr, keep = A.p010_image(hb, w, h, cg, ct, A.CR_LIMITED)
        g0 = _tm_groups(gpu.lib)
        a = gpu.tonemap(hdr)[0]
        assert _tm_groups(gpu.lib) - g0 == (w // 2) * (h // 2), "the fast tone-map kernel did not run"
        b = checker.tonemap(hdr)[0]
        if not (a == b).all():
            bad.append((ct, cg, int((a != b).sum())))
    assert not bad, bad


def test_tonemap_dev_pitched(gpu, checker):
    """uhdr_b200_tonemap_dev with pitched P010 source and YUV420 destination planes: equal to the checker, the fast
    kernel ran, and no padding byte of the destination was written"""
    import torch
    w, h = 1000, 722
    hb = T.make_p010(w, h, "noise", seed=T.SEED + 141)
    hdr_h, keep = A.p010_image(hb, w, h, A.CG_BT2100, A.CT_HLG, A.CR_LIMITED)
    want = checker.tonemap(hdr_h)[0]
    P, PY, PC = w + 64, w + 56, w // 2 + 30
    n = w * h

    def plane(arr, rows, cols, pitch, fill, dtype):
        t = np.full((rows, pitch), fill, dtype)
        t[:, :cols] = arr.reshape(rows, cols)
        return torch.from_numpy(t.view(np.int16) if dtype == np.uint16 else t).cuda()

    src = [plane(hb[:n], h, w, P, 0xFFFF, np.uint16), plane(hb[n:], h // 2, w, P, 0xFFFF, np.uint16)]
    dst = [torch.full((h, PY), SENTINEL, dtype=torch.uint8, device="cuda")] + \
          [torch.full((h // 2, PC), SENTINEL, dtype=torch.uint8, device="cuda") for _ in range(2)]
    hd = A.RawImage()
    hd.fmt, hd.cg, hd.ct, hd.range, hd.w, hd.h = A.FMT_P010, A.CG_BT2100, A.CT_HLG, A.CR_LIMITED, w, h
    hd.planes[0], hd.planes[1] = src[0].data_ptr(), src[1].data_ptr()
    hd.stride[0], hd.stride[1] = P, P
    sd = A.RawImage()
    sd.fmt, sd.w, sd.h = A.FMT_YUV420, w, h
    for i in range(3):
        sd.planes[i] = dst[i].data_ptr()
    sd.stride[0], sd.stride[1], sd.stride[2] = PY, PC, PC
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    g0 = _tm_groups(gpu.lib)
    assert gpu.lib.uhdr_b200_tonemap_dev(C.byref(hd), C.byref(sd), C.c_void_p(st.cuda_stream)) == 0, T.gpu_err(gpu)
    st.synchronize()
    assert _tm_groups(gpu.lib) - g0 == (w // 2) * (h // 2)
    got = [d.cpu().numpy() for d in dst]
    for d, cols in zip(got, (w, w // 2, w // 2)):
        assert (d[:, cols:] == SENTINEL).all(), "bytes past the plane width were written"
    c = (w // 2) * (h // 2)
    assert (got[0][:, :w].ravel() == want[:n]).all()
    assert (got[1][:, :w // 2].ravel() == want[n:n + c]).all()
    assert (got[2][:, :w // 2].ravel() == want[n + c:]).all()


def test_tonemap_yuv444_10(gpu, checker):
    """30bppYCbCr444 -> YCbCr444 (the generic tone-map kernel)"""
    w, h = 322, 182
    rs = np.random.RandomState(T.SEED + 142)
    planes = [rs.randint(64, 941, (h, w)).astype(np.uint16)] + [rs.randint(64, 961, (h, w)).astype(np.uint16)
                                                                 for _ in range(2)]
    outs = []
    for impl in (gpu, checker):
        hdr = A.raw_image(A.FMT_YUV444_10, A.CG_BT2100, A.CT_PQ, A.CR_LIMITED, w, h, planes, [w, w, w])
        o = [np.zeros((h, w), np.uint8) for _ in range(3)]
        sdr = A.raw_image(A.FMT_YUV444, -1, -1, -1, w, h, o, [w, w, w])
        rc = impl.f("tonemap")(C.byref(hdr), C.byref(sdr))
        outs.append((rc, o, (sdr.cg, sdr.ct, sdr.range)))
    (rc1, a, ma), (rc2, b, mb) = outs
    if rc2 != 0:
        pytest.skip(f"the checker does not take 30bppYCbCr444 (rc {rc2})")
    assert rc1 == 0, T.gpu_err(gpu)
    assert ma == mb, (ma, mb)
    for i in range(3):
        d = _diff(a[i], b[i])
        assert not d, (i, d)
