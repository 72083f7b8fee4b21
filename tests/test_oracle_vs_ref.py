"""Pins the C restatement (oracle/uhdr_oracle.c) against the reference's OWN sources compiled in
place (oracle/_ref, built by oracle/Makefile when /root/reference is present): bit-exact LUTs,
tables, gain maps, metadata, decoded pixels, tone-mapped and re-encoded planes."""
import itertools

import numpy as np
import pytest

import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A

W, H = 96, 64


@pytest.fixture(scope="module")
def pair(oracle_libs):
    if not oracle_libs.have_ref():
        pytest.skip("oracle/_ref not built (needs the reference sources)")
    return oracle_libs.Ref(), oracle_libs.Oracle()


def test_luts_bitwise(pair):
    R, O = pair
    for w in range(5):
        assert (R.lut(w).view(np.uint32) == O.lut(w).view(np.uint32)).all(), w


def test_idw_and_gain_lut(pair):
    import ctypes as C
    R, O = pair
    for s in (1, 2, 3, 4, 8):
        for v in range(4):
            a = np.zeros(s * s * 4, np.float32)
            b = np.zeros(s * s * 4, np.float32)
            R.lib.ref_idw_weights(s, v, a.ctypes.data_as(C.c_void_p))
            O.lib.uo_idw_weights(s, v, b.ctypes.data_as(C.c_void_p))
            assert (a.view(np.uint32) == b.view(np.uint32)).all(), (s, v)
    md = A.GainmapMetadata()
    for i, (mx, mn) in enumerate(((65.1, 4.9e-5), (845.9, 2.7e-3), (1283.8, 4.9e-5))):
        md.max_content_boost[i], md.min_content_boost[i], md.gamma[i] = mx, mn, 1.0
    for wgt in (1.0, 0.37):
        a = np.zeros(3072, np.float32)
        b = np.zeros(3072, np.float32)
        R.lib.ref_gain_lut.argtypes = [C.c_void_p, C.c_float, C.c_void_p]
        O.lib.uo_gain_lut.argtypes = [C.c_void_p, C.c_float, C.c_void_p]
        R.lib.ref_gain_lut(C.byref(md), wgt, a.ctypes.data_as(C.c_void_p))
        O.lib.uo_gain_lut(C.byref(md), wgt, b.ctypes.data_as(C.c_void_p))
        assert (a.view(np.uint32) == b.view(np.uint32)).all()


def _inputs(kind, hct, hcg, scg, hfmt="p010"):
    if hfmt == "p010":
        hb = T.make_p010(W, H, kind)
        hdr, k = A.p010_image(hb, W, H, hcg, hct, A.CR_LIMITED)
    elif hfmt == "1010102":
        hb = T.make_rgba1010102(W, H)
        hdr, k = A.raw_image(A.FMT_RGBA1010102, hcg, hct, A.CR_FULL, W, H, [hb], [W]), hb
    else:
        hb = T.make_rgbaf16(W, H)
        hdr, k = A.raw_image(A.FMT_RGBAF16, hcg, A.CT_LINEAR, A.CR_FULL, W, H, [hb], [W]), hb
    sb = T.make_yuv420(W, H, kind)
    sdr, k2 = A.yuv420_image(sb, W, H, scg)
    return hdr, sdr, (hb, sb, k, k2)


def test_generate_matrix(pair):
    R, O = pair
    bad = []
    for kind, hct, hcg, scg, multi, scale, preset in itertools.product(
            ["noise", "black"], [A.CT_HLG, A.CT_PQ], [0, 1, 2], [0, 1, 2], [0, 1], [1, 4], [0, 1]):
        hdr, sdr, keep = _inputs(kind, hct, hcg, scg)
        cfg = A.default_gm_config(scale_factor=scale, multichannel=multi, preset=preset)
        g1, m1 = R.generate(sdr, hdr, cfg)
        g2, m2 = O.generate(sdr, hdr, cfg)
        if not ((g1 == g2).all() and T.md_equal(m1, m2)):
            bad.append((kind, hct, hcg, scg, multi, scale, preset))
    assert not bad, bad[:5]


def test_generate_other_formats_and_options(pair):
    R, O = pair
    for hfmt, ct in (("1010102", A.CT_PQ), ("f16", A.CT_LINEAR)):
        for kw in ({}, {"multichannel": 0, "use_luminance": 0}, {"preset": 0, "gamma": 2.2}, {"gamma": 1.5},
                   {"sdr_is_601": 1, "scale_factor": 2}, {"min_content_boost": 0.5, "max_content_boost": 6.0}):
            hdr, sdr, keep = _inputs("noise", ct, 2, 0, hfmt)
            cfg = A.default_gm_config(**kw)
            g1, m1 = R.generate(sdr, hdr, cfg)
            g2, m2 = O.generate(sdr, hdr, cfg)
            assert (g1 == g2).all() and T.md_equal(m1, m2), (hfmt, kw)


def test_code_lattice(pair):
    """Every HDR and SDR luma code with full-range chroma (uhdr_testlib.make_code_lattice), with clean and dirty
    P010 low bits: limited-range codes outside 64..940 drive the normalised values below 0 and above 1, where the
    clamps and table indices have to agree.  generateGainMap over range, transfer, channels, scale and preset,
    and toneMap on the same HDR frames."""
    R, O = pair
    w, h = 1024, 256
    bad = []
    for dirty in (False, True):
        hb, sb = T.make_code_lattice(w, h, dirty)
        sdr, k2 = A.yuv420_image(sb, w, h, A.CG_BT709)
        for rng, ct in itertools.product([A.CR_LIMITED, A.CR_FULL], [A.CT_HLG, A.CT_PQ]):
            hdr, k1 = A.p010_image(hb, w, h, A.CG_BT2100, ct, rng)
            for multi, scale, preset in itertools.product([0, 1], [1, 4], [0, 1]):
                cfg = A.default_gm_config(scale_factor=scale, multichannel=multi, preset=preset)
                g1, m1 = R.generate(sdr, hdr, cfg)
                g2, m2 = O.generate(sdr, hdr, cfg)
                if not ((g1 == g2).all() and T.md_equal(m1, m2)):
                    bad.append(("generate", dirty, rng, ct, multi, scale, preset, int((g1 != g2).sum())))
            a, b = R.tonemap(hdr)[0], O.tonemap(hdr)[0]
            if not (a == b).all():
                bad.append(("tonemap", dirty, rng, ct, int((a != b).sum())))
    assert not bad, bad


def test_apply_matrix(pair):
    R, O = pair
    for multi, scale in ((1, 1), (0, 1), (1, 4), (0, 2)):
        hdr, sdr, keep = _inputs("noise", A.CT_HLG, 2, 0)
        g, m = R.generate(sdr, hdr, A.default_gm_config(scale_factor=scale, multichannel=multi))
        maps = [g] if not multi else [g, np.concatenate([g, np.full(g.shape[:2] + (1,), 255, np.uint8)], -1)]
        for gm in maps:
            gm = np.ascontiguousarray(gm)
            for gcg, ct, boost in itertools.product([-1, 0, 2], [A.CT_LINEAR, A.CT_HLG, A.CT_PQ], [A.FLT_MAX, 2.5]):
                gi = T.gm_image(gm, gcg)
                assert (R.apply(sdr, gi, m, ct, boost) == O.apply(sdr, gi, m, ct, boost)).all()
    # non-integer scale
    hdr, sdr, keep = _inputs("noise", A.CT_HLG, 2, 0)
    g, m = R.generate(sdr, hdr)
    for ch in (1, 3):
        crop = np.ascontiguousarray(g[:43, :64, :ch])  # keep alive: descriptors hold raw pointers
        gi = T.gm_image(crop, 2)
        assert (R.apply(sdr, gi, m, A.CT_LINEAR) == O.apply(sdr, gi, m, A.CT_LINEAR)).all()


def test_tonemap_and_convert(pair):
    R, O = pair
    for kind, hct, hcg in itertools.product(["noise", "white"], [A.CT_HLG, A.CT_PQ], [0, 1, 2]):
        hb = T.make_p010(W, H, kind)
        hdr, k = A.p010_image(hb, W, H, hcg, hct, A.CR_LIMITED)
        assert (R.tonemap(hdr)[0] == O.tonemap(hdr)[0]).all()
    hb = T.make_rgbaf16(W, H)
    hdr = A.raw_image(A.FMT_RGBAF16, 1, A.CT_LINEAR, A.CR_FULL, W, H, [hb], [W])
    assert (R.tonemap(hdr)[0] == O.tonemap(hdr)[0]).all()
    for s, d in itertools.permutations([0, 1, 2], 2):
        sb = T.make_yuv420(W, H, "noise")
        assert (R.convert_yuv(sb, W, H, s, d) == O.convert_yuv(sb, W, H, s, d)).all()
