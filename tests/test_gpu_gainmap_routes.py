"""Every generateGainMap route on the GPU against the CPU checker, bit exact (map bytes and metadata).

The library picks its kernels from the configuration (engine.cu, generate_gainmap_dev).  Each route below is
reached on purpose and the test asserts which kernels ran (per-kernel timers) and whether the quotient-screen
counter moved (uhdr_b200_generate_stats), as well as the result:

  A  scale 1, gamma 1, P010 + YUV420, w % 4 == 0, h even: statistics pass + code pass of k_gainmap_fast
  B  scale 2 / 4, gamma 1, map size % 4 == 0: k_gainmap_scaled with the quotient plane + k_affine_q
  C  scale 2 / 4 with a map size % 4 != 0: gains plane + k_gainmap_finalize + k_gainmap_affine
  D  gamma != 1 at scale 1, E  gamma != 1 at scale 2 / 4: gains plane + finalize + affine (double pow)
  F  P010 the fast kernels decline (w % 4 != 0, a source pitch that is not a multiple of 4): k_gainmap_pass1
  G  scales other than 1, 2, 4, and the reference's own scale when w / scale or h / scale is 0
  H  UHDR_B200_GAINS_PLANE=1 (read once per process: run in a child process): gains plane + k_affine_fast
  I  REALTIME preset: the one-pass kernels

Inputs that reach what noise does not: a lattice of every HDR and SDR luma code (incl. limited-range codes
outside 64..940 and dirty low bits of P010 words), and unique extremes planted into a constant frame at the
first / last pixel, in partial tiles and in the last warp of a middle tile, so that one CTA alone holds them.
"""
import ctypes as C
import itertools
import os
import subprocess
import sys
import tempfile
import threading

if __name__ == "__main__":   # child process of test_gains_plane_switch
    _ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [_ROOT, os.path.join(_ROOT, "tests")]

import numpy as np
import pytest

import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A

pytestmark = pytest.mark.gpu

P1, FIN, AFF, ONE = "gainmap_pass1", "gainmap_finalize", "gainmap_affine", "gainmap_onepass"
TWO_PASS_FAST = {P1, AFF}
GENERIC = {P1, FIN, AFF}


# ------------------------------------------------------------------------------------------------
# helpers
# ------------------------------------------------------------------------------------------------
def _map_geometry(w, h, scale):
    """the reference's map size (jpegr.cpp:692-706): with w / scale or h / scale == 0 it picks
    min(w, h) / 8 (or 1) as the scale"""
    mw, mh = w // scale, h // scale
    if mw == 0 or mh == 0:
        s = min(w, h)
        s = s // 8 if s >= 8 else 1
        mw, mh = w // s, h // s
    return mw, mh


def _generate(impl, sdr, hdr, cfg):
    """-> (map (mh, mw, c) u8, metadata); the map buffer is sized by the reference's rule"""
    mw, mh = _map_geometry(sdr.w, sdr.h, cfg.scale_factor)
    ch = 3 if cfg.multichannel else 1
    gm = np.zeros((mh, mw, ch), np.uint8)
    gmi = A.raw_image(A.FMT_RGB888 if ch == 3 else A.FMT_Y400, -1, -1, -1, mw, mh, [gm], [mw])
    md = A.GainmapMetadata()
    rc = impl.f("generate_gainmap")(C.byref(sdr), C.byref(hdr), C.byref(cfg), C.byref(md), C.byref(gmi))
    assert rc == 0, f"{impl.pfx}generate_gainmap rc={rc}"
    assert (gmi.w, gmi.h) == (mw, mh), (gmi.w, gmi.h, mw, mh)
    return gm, md


def _descs(p010, yuv, w, h, hcg=A.CG_BT2100, hct=A.CT_HLG, rng=A.CR_LIMITED, scg=A.CG_BT709):
    hdr, k1 = A.p010_image(p010, w, h, hcg, hct, rng)
    sdr, k2 = A.yuv420_image(yuv, w, h, scg)
    return hdr, sdr, (p010, yuv, k1, k2)


def _noise(w, h, seed=0):
    return T.make_p010(w, h, "noise", seed=T.SEED + 10 + seed), T.make_yuv420(w, h, "noise", seed=T.SEED + 20 + seed)


def _diff(g1, m1, g2, m2):
    """'' when map and metadata are identical, else a short description"""
    if g1.shape != g2.shape:
        return f"map shape {g1.shape} != {g2.shape}"
    out = []
    if not (g1 == g2).all():
        idx = np.argwhere(g1 != g2)
        out.append(f"{len(idx)} map bytes differ, first at {tuple(idx[0])}: {g1[tuple(idx[0])]} != {g2[tuple(idx[0])]}")
    if not T.md_equal(m1, m2):
        out.append(f"metadata {m1.as_dict()} != {m2.as_dict()}")
    return "; ".join(out)


def _stats(lib):
    st = (C.c_ulonglong * 2)()
    lib.uhdr_b200_generate_stats(st)
    return st[0], st[1]


def _timer_names(lib):
    buf = C.create_string_buffer(1 << 16)
    n = lib.uhdr_b200_kernel_timing_report(buf, C.c_size_t(len(buf)), 1)
    assert n >= 0, n
    return {line.split()[0] for line in buf.value.decode().splitlines() if line.strip()}


class Route:
    """Records what the generate calls inside the block ran: `kernels` (the gainmap_* timer names) and
    `values` / `exact` (growth of uhdr_b200_generate_stats: values quantised through the quotient screen and
    how many of them took the fp64 log2)."""

    def __init__(self, lib):
        self.lib = lib

    def __enter__(self):
        self.lib.uhdr_b200_set_kernel_timing(1)
        _timer_names(self.lib)   # drop what earlier calls left
        self.v0, self.e0 = _stats(self.lib)
        return self

    def __exit__(self, *exc):
        try:
            self.kernels = {n for n in _timer_names(self.lib) if n.startswith("gainmap_")}
            v1, e1 = _stats(self.lib)
            self.values, self.exact = v1 - self.v0, e1 - self.e0
        finally:
            self.lib.uhdr_b200_set_kernel_timing(0)
        return False


def _values(w, h, cfg):
    mw, mh = _map_geometry(w, h, cfg.scale_factor)
    return mw * mh * (3 if cfg.multichannel else 1)


# ------------------------------------------------------------------------------------------------
# 1. route table
# ------------------------------------------------------------------------------------------------
# route -> (cases, kernels expected, whether the quotient screen counts the values).  A case is
# (w, h, config keywords, input keywords).
_BQ = A.USAGE_BEST_QUALITY
ROUTES = {
    "A_scale1_statistics_and_code_pass": (
        [(1000, 722, {"multichannel": m}, {}) for m in (0, 1)] +
        [(1024, 256, {"multichannel": 1}, {"hct": A.CT_PQ, "rng": A.CR_FULL})],
        TWO_PASS_FAST, True),
    "B_scale2_4_quotient_plane": (
        [(1024, 512, {"scale_factor": s, "multichannel": m}, {}) for s in (2, 4) for m in (0, 1)],
        TWO_PASS_FAST, True),
    "C_scale4_gains_plane_generic_affine": (
        [(1284, 724, {"scale_factor": 4, "multichannel": 0}, {})], GENERIC, False),
    "D_gamma_scale1": (
        [(1000, 722, {"gamma": g, "multichannel": m}, {}) for g in (2.2, 0.7) for m in (0, 1)], GENERIC, False),
    "E_gamma_scale2_4": (
        [(1024, 512, {"gamma": g, "scale_factor": s, "multichannel": m}, {})
         for g in (2.2, 0.7) for s in (2, 4) for m in (0, 1)], GENERIC, False),
    "F_generic_p010": (
        [(998, 722, {"multichannel": m}, {}) for m in (0, 1)], GENERIC, False),
    "G_other_scales": (
        [(998, 722, {"scale_factor": 3}, {}), (1000, 722, {"scale_factor": 8, "multichannel": 0}, {}),
         (96, 64, {"scale_factor": 200}, {}), (96, 64, {"scale_factor": 200, "multichannel": 0}, {})],
        GENERIC, False),
    "I_onepass": (
        [(1000, 722, {"preset": A.USAGE_REALTIME, "multichannel": m}, {}) for m in (0, 1)] +
        [(998, 722, {"preset": A.USAGE_REALTIME}, {}),
         (1024, 512, {"preset": A.USAGE_REALTIME, "scale_factor": 4}, {})],
        {ONE}, False),
}


@pytest.mark.parametrize("route", sorted(ROUTES))
def test_route(gpu, checker, route):
    cases, kernels, screened = ROUTES[route]
    bad = []
    for i, (w, h, ckw, ikw) in enumerate(cases):
        p, y = _noise(w, h, i)
        hdr, sdr, keep = _descs(p, y, w, h, **ikw)
        cfg = A.default_gm_config(**ckw)
        with Route(gpu.lib) as r:
            g1, m1 = _generate(gpu, sdr, hdr, cfg)
        g2, m2 = _generate(checker, sdr, hdr, cfg)
        d = _diff(g1, m1, g2, m2)
        if d:
            bad.append((w, h, ckw, ikw, d))
        assert r.kernels == kernels, (w, h, ckw, r.kernels)
        assert r.values == (_values(w, h, cfg) if screened else 0), (w, h, ckw, r.values)
    assert not bad, bad


# ---- H: UHDR_B200_GAINS_PLANE=1, read once when the library loads: a child process ----------------
# (w, h, config keywords, kernels expected).  k_affine_fast needs tight map rows: the host-buffer API's map
# stride is the width rounded up to 64, so the generic affine pass runs where w / scale is not a multiple of 64.
GAINS_PLANE_CASES = [
    (3840, 2162, {"multichannel": 1}, TWO_PASS_FAST),
    (1024, 256, {"multichannel": 0}, TWO_PASS_FAST),
    (1000, 722, {"multichannel": 1}, GENERIC),
    (1024, 512, {"scale_factor": 4, "multichannel": 0}, TWO_PASS_FAST),
    (1024, 512, {"scale_factor": 4, "multichannel": 1}, TWO_PASS_FAST),
]


def _gains_plane_child(out_dir):
    gpu = T.Gpu()
    for i, (w, h, ckw, _k) in enumerate(GAINS_PLANE_CASES):
        p, y = _noise(w, h, i)
        hdr, sdr, keep = _descs(p, y, w, h)
        with Route(gpu.lib) as r:
            g, m = _generate(gpu, sdr, hdr, A.default_gm_config(**ckw))
        np.savez(os.path.join(out_dir, f"case{i}.npz"), map=g, md=np.frombuffer(bytes(m), np.uint8),
                 kernels=np.array(sorted(r.kernels)), values=r.values)


def test_gains_plane_switch(gpu, checker):
    """H: UHDR_B200_GAINS_PLANE=1 at scales 1 and 4, incl. 3840x2162 and 1000x722 (bottom partial tile row)."""
    with tempfile.TemporaryDirectory() as tmp:
        env = dict(os.environ, UHDR_B200_GAINS_PLANE="1")
        res = subprocess.run([sys.executable, "-s", os.path.abspath(__file__), "--gains-plane-child", tmp],
                             env=env, capture_output=True, text=True, timeout=600)
        assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
        bad = []
        for i, (w, h, ckw, kernels) in enumerate(GAINS_PLANE_CASES):
            got = np.load(os.path.join(tmp, f"case{i}.npz"))
            assert set(got["kernels"].tolist()) == kernels, (w, h, ckw, got["kernels"])
            assert int(got["values"]) == 0, (w, h, ckw, int(got["values"]))
            p, y = _noise(w, h, i)
            hdr, sdr, keep = _descs(p, y, w, h)
            g2, m2 = _generate(checker, sdr, hdr, A.default_gm_config(**ckw))
            m1 = A.GainmapMetadata.from_buffer_copy(got["md"].tobytes())
            d = _diff(got["map"], m1, g2, m2)
            if d:
                bad.append((w, h, ckw, d))
        assert not bad, bad


# ------------------------------------------------------------------------------------------------
# 2. exhaustive code lattice
# ------------------------------------------------------------------------------------------------
LW, LH = 1024, 256
# (hdr gamut, sdr gamut): no conversion, conversion on the SDR side, conversion on the HDR side
GAMUT_PAIRS = [(A.CG_P3, A.CG_P3), (A.CG_BT2100, A.CG_BT709), (A.CG_BT709, A.CG_BT2100)]
LATTICE_CONFIGS = list(itertools.product(
    [A.CR_LIMITED, A.CR_FULL], [A.CT_HLG, A.CT_PQ, A.CT_SRGB],
    [(1, 1), (0, 1), (0, 0)],   # (multichannel, use_luminance)
    GAMUT_PAIRS, [False, True]))
LATTICE_ROUTES = {
    # route -> (frame width, extra configs, kernels expected, screened)
    "A": (LW, [{}], TWO_PASS_FAST, True),
    "B": (LW, [{"scale_factor": 2}, {"scale_factor": 4}], TWO_PASS_FAST, True),
    "D": (LW, [{"gamma": 2.2}, {"gamma": 0.7}], GENERIC, False),
    "I": (LW, [{"preset": A.USAGE_REALTIME}], {ONE}, False),
    "F": (LW + 6, [{}], GENERIC, False),   # 1030 % 4 != 0: k_gainmap_pass1 on the same codes
}


@pytest.fixture(scope="module")
def lattices():
    return {(w, dirty): T.make_code_lattice(w, LH, dirty) for w in (LW, LW + 6) for dirty in (False, True)}


@pytest.mark.parametrize("route", sorted(LATTICE_ROUTES))
def test_code_lattice(gpu, checker, lattices, route):
    w, extras, kernels, screened = LATTICE_ROUTES[route]
    bad, n_values = [], 0
    with Route(gpu.lib) as r:
        for (rng, ct, (multi, lum), (hcg, scg), dirty), extra in itertools.product(LATTICE_CONFIGS, extras):
            p, y = lattices[(w, dirty)]
            hdr, sdr, keep = _descs(p, y, w, LH, hcg, ct, rng, scg)
            cfg = A.default_gm_config(multichannel=multi, use_luminance=lum, **extra)
            n_values += _values(w, LH, cfg)
            g1, m1 = _generate(gpu, sdr, hdr, cfg)
            g2, m2 = _generate(checker, sdr, hdr, cfg)
            d = _diff(g1, m1, g2, m2)
            if d:
                bad.append((rng, ct, multi, lum, hcg, scg, dirty, extra, d))
    assert not bad, (len(bad), bad[:6])
    assert r.kernels == kernels, r.kernels
    assert r.values == (n_values if screened else 0), (r.values, n_values)
    if route == "A":
        # the lattice puts many values next to a byte boundary: the lg2.approx screen must hand some over
        assert r.exact > 0, r.exact
        print(f"route A exact-path share on the lattice: {r.exact} / {r.values} = {r.exact / r.values:.5f}")


def test_tonemap_code_lattice(gpu, checker, lattices):
    """toneMap decodes P010 like generate and screens its powf: every code, clean and dirty low bits."""
    bad = []
    for (rng, ct, cg, dirty) in itertools.product([A.CR_LIMITED, A.CR_FULL], [A.CT_HLG, A.CT_PQ],
                                                  [A.CG_BT2100, A.CG_BT709], [False, True]):
        p, _y = lattices[(LW, dirty)]
        hdr, keep = A.p010_image(p, LW, LH, cg, ct, rng)
        g0 = _tonemap_groups(gpu.lib)
        a = gpu.tonemap(hdr)[0]
        assert _tonemap_groups(gpu.lib) - g0 == LW * LH // 4, "the fast tone-map kernel did not run"
        b = checker.tonemap(hdr)[0]
        if not (a == b).all():
            bad.append((rng, ct, cg, dirty, int((a != b).sum())))
    assert not bad, bad


def _tonemap_groups(lib):
    """2x2 pixel groups the fast tone-map kernel has processed since the library loaded"""
    st = (C.c_ulonglong * 2)()
    lib.uhdr_b200_tonemap_stats(st)
    return st[0]


# ------------------------------------------------------------------------------------------------
# 3. planted unique extremes
# ------------------------------------------------------------------------------------------------
# constant background: every pixel has the same quotient.  Codes: HDR (Y, U, V) 10 bit limited, SDR (Y, U, V).
BG_HDR, BG_SDR = (500, 512, 512), (128, 128, 128)
PLANTS = {
    # kind -> (hdr, sdr, metadata field it must move)
    "max": ((940, 512, 512), (2, 128, 128), "max_content_boost"),   # bright HDR over near-black (not dark) SDR
    "min": ((64, 512, 512), (255, 128, 128), "min_content_boost"),  # black HDR over white SDR
    "dark": ((940, 512, 512), (0, 128, 128), "max_content_boost"),  # SDR 0: dark, gain capped at 2.3 > background
}
# three channels: SDR pixels with one channel close to 0 (BT.709 coefficients): the gain of that channel alone peaks
CHANNEL_PLANTS = [(128, 128, 48), (86, 255, 255), (128, 60, 128)]   # R, G, B


def _positions(w, h, s):
    """top-left corners of the planted b x b block (b = 2 at scale 1, else the scale): first pixel, last pixel,
    last 4 columns of row 0, the bottom tile row, and the last warp of a middle tile (threads y = 3, x >= 32 of
    a CTA: the warp reduce_minmax folds last)"""
    b = max(2, s)
    if s == 1:   # k_gainmap_fast: 256 x 8 pixel tiles, a thread = 4 x 2 pixels
        mid = ((w // 512) * 256 + 200, (h // 16) * 8 + 6)
    else:        # k_gainmap_scaled: 64 x 4 map-pixel tiles, a thread = one map pixel
        mid = (((w // s) // 128 * 64 + 40) * s, ((h // s) // 8 * 4 + 3) * s)
    return {"first": (0, 0), "last": (w - b, h - b), "row0_right": (w - 4, 0),
            "bottom": ((w // 2) // b * b, h - b), "middle_last_warp": mid}


def _plant(p010, yuv, w, h, x, y, b, hv, sv):
    hy = p010[:w * h].reshape(h, w)
    huv = p010[w * h:].reshape(h // 2, w)
    hy[y:y + b, x:x + b] = hv[0] << 6
    huv[y // 2:(y + b) // 2, x:x + b:2] = hv[1] << 6
    huv[y // 2:(y + b) // 2, x + 1:x + b:2] = hv[2] << 6
    n, c = w * h, (w // 2) * (h // 2)
    sy = yuv[:n].reshape(h, w)
    su = yuv[n:n + c].reshape(h // 2, w // 2)
    sv_ = yuv[n + c:].reshape(h // 2, w // 2)
    sy[y:y + b, x:x + b] = sv[0]
    su[y // 2:(y + b) // 2, x // 2:(x + b) // 2] = sv[1]
    sv_[y // 2:(y + b) // 2, x // 2:(x + b) // 2] = sv[2]


def _background(w, h):
    p = np.empty(w * h * 3 // 2, np.uint16)
    p[:w * h] = BG_HDR[0] << 6
    p[w * h:] = np.tile(np.array([BG_HDR[1] << 6, BG_HDR[2] << 6], np.uint16), w * h // 4)
    y = np.empty(w * h * 3 // 2, np.uint8)
    y[:w * h] = BG_SDR[0]
    y[w * h:w * h + w * h // 4] = BG_SDR[1]
    y[w * h + w * h // 4:] = BG_SDR[2]
    return p, y


def planted_cases(w, h, scale):
    """-> list of (name, multichannel, plants [(x, y, hdr, sdr)], [(field, channel)] that each case must move
    relative to the same frame without its plants (the self-check))"""
    b = max(2, scale)
    pos = _positions(w, h, scale)
    cases = []
    for kind, (hv, sv, field) in PLANTS.items():
        for pname, (x, y) in pos.items():
            for multi in (0, 1):
                cases.append((f"{kind}@{pname}/{'3ch' if multi else '1ch'}", multi, [(x, y, hv, sv)],
                              [(field, c) for c in range(3 if multi else 1)]))
    # one extreme per channel, in three different tiles
    spots = [pos["middle_last_warp"], pos["last"], pos["first"]]
    cases.append(("per_channel_max", 1, [(x, y, BG_HDR, sv) for (x, y), sv in zip(spots, CHANNEL_PLANTS)],
                  [("max_content_boost", c) for c in range(3)]))
    return [(n, m, pl, sens, b) for n, m, pl, sens in cases]


def _planted_frame(w, h, plants, b):
    p, y = _background(w, h)
    for x, yy, hv, sv in plants:
        _plant(p, y, w, h, x, yy, b, hv, sv)
    return p, y


def _self_check(checker, w, h, scale, multi, plants, sens, b, md, cache):
    """the checker's metadata with the plants must differ, in every (field, channel) of sens, from its metadata
    for the frame without the plant of that channel (without any plant when there is one): else the case could
    not notice a kernel that loses the extreme"""
    cfg = A.default_gm_config(scale_factor=scale, multichannel=multi)
    for field, c in sens:
        rest = tuple((x, y, hv, sv) for i, (x, y, hv, sv) in enumerate(plants) if len(plants) > 1 and i != c)
        key = (multi, rest)
        if key not in cache:
            p, y = _planted_frame(w, h, rest, b)
            hdr, sdr, keep = _descs(p, y, w, h)
            cache[key] = _generate(checker, sdr, hdr, cfg)[1]
        a, z = getattr(md, field)[c], getattr(cache[key], field)[c]
        assert a != z, f"plant does not move {field}[{c}]: {a} == {z}"


PLANT_SIZES = [(3840, 2160, 1, TWO_PASS_FAST), (3840, 2160, 4, TWO_PASS_FAST), (1000, 722, 1, TWO_PASS_FAST),
               (998, 722, 1, GENERIC)]


@pytest.mark.parametrize("w,h,scale,kernels", PLANT_SIZES, ids=[f"{w}x{h}_s{s}" for w, h, s, _k in PLANT_SIZES])
def test_planted_extremes(gpu, checker, w, h, scale, kernels):
    bad, cache = [], {}
    for name, multi, plants, sens, b in planted_cases(w, h, scale):
        p, y = _planted_frame(w, h, plants, b)
        hdr, sdr, keep = _descs(p, y, w, h)
        cfg = A.default_gm_config(scale_factor=scale, multichannel=multi)
        g2, m2 = _generate(checker, sdr, hdr, cfg)
        _self_check(checker, w, h, scale, multi, plants, sens, b, m2, cache)
        with Route(gpu.lib) as r:
            g1, m1 = _generate(gpu, sdr, hdr, cfg)
        assert r.kernels == kernels, (name, r.kernels)
        d = _diff(g1, m1, g2, m2)
        if d:
            bad.append((name, d))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------
# 4. geometry and memory layout
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", [(1000, 722), (3840, 2162)])
def test_fast_modes_bottom_partial_tile(gpu, checker, w, h):
    """scale 1 with h % 8 == 2 (and 1000 % 256 != 0): statistics + code pass and one-pass on a bottom tile row
    of one pixel pair; the gains-plane mode at these sizes runs in test_gains_plane_switch"""
    p, y = _noise(w, h, 7)
    for ct, rng in ((A.CT_HLG, A.CR_LIMITED), (A.CT_PQ, A.CR_FULL)):
        hdr, sdr, keep = _descs(p, y, w, h, hct=ct, rng=rng)
        for kw, kernels in (({}, TWO_PASS_FAST), ({"preset": A.USAGE_REALTIME}, {ONE})):
            for multi in (0, 1):
                cfg = A.default_gm_config(multichannel=multi, **kw)
                with Route(gpu.lib) as r:
                    g1, m1 = _generate(gpu, sdr, hdr, cfg)
                g2, m2 = _generate(checker, sdr, hdr, cfg)
                assert r.kernels == kernels, (ct, rng, kw, multi, r.kernels)
                d = _diff(g1, m1, g2, m2)
                assert not d, (ct, rng, kw, multi, d)


def _dev_plane(torch, arr, h, w, pitch, fill):
    """(h, w) host plane -> device tensor with rows of `pitch` elements, the padding set to `fill`"""
    a = np.full((h, pitch), fill, arr.dtype)
    a[:, :w] = arr.reshape(h, w)
    if a.dtype == np.uint16:
        a = a.view(np.int16)
    return torch.from_numpy(a).cuda()


@pytest.mark.parametrize("pad,map_pad,kernels", [(64, 4, TWO_PASS_FAST), (2, 3, GENERIC)], ids=["fast", "generic"])
@pytest.mark.parametrize("multi", [0, 1])
def test_dev_api_pitched_planes(gpu, checker, pad, map_pad, kernels, multi):
    """uhdr_b200_generate_gainmap_dev with source rows of w + pad pixels (padding 0xFF..) and a map destination
    whose rows are longer than the map: equal to the reference's map, and not one padding byte written.  A
    pitch of w + 2 takes the generic kernels (F)."""
    import torch
    w, h = 640, 368
    p, y = _noise(w, h, 3)
    hdr_h, sdr_h, keep = _descs(p, y, w, h)
    cfg = A.default_gm_config(multichannel=multi)
    want, want_md = _generate(checker, sdr_h, hdr_h, cfg)
    P, Pc = w + pad, (w + pad) // 2
    n, c = w * h, (w // 2) * (h // 2)
    planes = [_dev_plane(torch, p[:n], h, w, P, 0xFFFF), _dev_plane(torch, p[n:], h // 2, w, P, 0xFFFF)]
    splanes = [_dev_plane(torch, y[:n], h, w, P, 0xFF), _dev_plane(torch, y[n:n + c], h // 2, w // 2, Pc, 0xFF),
               _dev_plane(torch, y[n + c:], h // 2, w // 2, Pc, 0xFF)]
    hdr_d = A.RawImage()
    hdr_d.fmt, hdr_d.cg, hdr_d.ct, hdr_d.range, hdr_d.w, hdr_d.h = A.FMT_P010, A.CG_BT2100, A.CT_HLG, A.CR_LIMITED, w, h
    hdr_d.planes[0], hdr_d.planes[1] = planes[0].data_ptr(), planes[1].data_ptr()
    hdr_d.stride[0], hdr_d.stride[1] = P, P
    sdr_d = A.RawImage()
    sdr_d.fmt, sdr_d.cg, sdr_d.ct, sdr_d.range, sdr_d.w, sdr_d.h = A.FMT_YUV420, A.CG_BT709, A.CT_SRGB, A.CR_FULL, w, h
    for i in range(3):
        sdr_d.planes[i] = splanes[i].data_ptr()
    sdr_d.stride[0], sdr_d.stride[1], sdr_d.stride[2] = P, Pc, Pc
    ch = 3 if multi else 1
    ms = w + map_pad
    sentinel = 0xA5
    gm_t = torch.full((h * ms * ch,), sentinel, dtype=torch.uint8, device="cuda")
    gm_d = A.RawImage()
    gm_d.fmt, gm_d.w, gm_d.h = A.FMT_RGB888 if multi else A.FMT_Y400, w, h
    gm_d.planes[0] = gm_t.data_ptr()
    gm_d.stride[0] = ms
    md = A.GainmapMetadata()
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    with Route(gpu.lib) as r:
        rc = gpu.lib.uhdr_b200_generate_gainmap_dev(C.byref(sdr_d), C.byref(hdr_d), C.byref(cfg), C.byref(md),
                                                    C.byref(gm_d), C.c_void_p(st.cuda_stream))
        assert rc == 0, T.gpu_err(gpu)
        st.synchronize()
    assert r.kernels == kernels, r.kernels
    got = gm_t.cpu().numpy().reshape(h, ms * ch)
    d = _diff(np.ascontiguousarray(got[:, :w * ch]).reshape(h, w, ch), md, want, want_md)
    assert not d, d
    assert (got[:, w * ch:] == sentinel).all(), "bytes past the map width were written"
    # the sources are read only
    assert (planes[0].cpu().numpy().view(np.uint16)[:, w:] == 0xFFFF).all()


# ------------------------------------------------------------------------------------------------
# 5. concurrent encoders
# ------------------------------------------------------------------------------------------------
def test_concurrent_encoders(gpu, oracle_libs):
    """Four host threads, each with its own encoder handle, encode four different 1920x1080 frames at the same
    time (twice, the second a re-armed encode of the resident inputs); every stream equals the reference's
    file of its frame."""
    if not oracle_libs.have_ref():
        pytest.skip("reference build not available")
    import bench
    w, h, n = 1920, 1080, 4
    ref = T.UhdrApi(oracle_libs.Ref().lib)
    frames, want = [], []
    for i in range(n):
        p, y = bench.make_frame(w, h, 20 + i)
        hdr, sdr, keep = bench.frame_descs(p, y, w, h)
        frames.append((hdr, sdr, keep, p, y))
        want.append(ref.encode(hdr, sdr))
    lib = gpu.lib
    T.UhdrApi(lib)   # restypes
    got = [[None, None] for _ in range(n)]
    errs = []
    gate = threading.Barrier(n)

    def work(i):
        hdr, sdr = frames[i][0], frames[i][1]
        enc = C.c_void_p(lib.uhdr_create_encoder())
        try:
            assert lib.uhdr_enc_set_raw_image(enc, C.byref(hdr), A.HDR_IMG).error_code == 0
            assert lib.uhdr_enc_set_raw_image(enc, C.byref(sdr), A.SDR_IMG).error_code == 0
            gate.wait()
            for it in range(2):
                e = lib.uhdr_encode(enc)
                assert e.error_code == 0, e.detail
                o = lib.uhdr_get_encoded_stream(enc).contents
                got[i][it] = C.string_at(o.data, o.data_sz)
                assert lib.uhdr_b200_enc_rearm(enc) == 0
        except BaseException as e:  # noqa: BLE001
            errs.append((i, repr(e)))
            gate.abort()
        finally:
            lib.uhdr_release_encoder(enc)

    th = [threading.Thread(target=work, args=(i,)) for i in range(n)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    for i in range(n):
        for it in range(2):
            assert got[i][it] == want[i], (i, it, len(got[i][it]), len(want[i]))


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "--gains-plane-child":
        _gains_plane_child(sys.argv[2])
