"""The encoder's JPEG block and entropy stage (k_fdct8_code, csrc/fdct8.cu, then k_huff_encode, csrc/huffman.cu) route by
route on the GPU: every uhdr_b200_jpeg_encode stream is compared whole, byte for byte, with the reference's own
JpegEncoderHelper on libjpeg-turbo (ref_jpeg_encode), or with the C restatement pinned to it (jo_encode) where that
build is absent.

Each case asserts its route from uhdr_b200_jpeg_encode_stats (the bpt of the launch, whether its grid exceeded one
wave; thresholds from the resident count the library reports, never a hard-coded one) and, from the scan model
(tests/jpeg_scan_model.py), that its input reaches the case it is there for.  A mismatch is reported as CTA / window /
scan block of the first differing byte.

  A  quality 1..100 x Y400, 4:2:0, 4:2:2, 4:4:4, RGB888 at ragged sizes (wblocks % 32 in {1, 31}, partial last warp
     item, dummy blocks, partial right RGB block); strides wider than the aligned width with bytes there; 4:4:0,
     4:1:1, 4:1:0 and layouts the helper refuses fail on the GPU with nothing written
  B  every bpt 1..8: blocks = k * 256 * R and just above, noise at q100 (several windows per CTA) and smooth at q95
  C  grids beyond one wave: RGB888 and 4:4:4 at 8192 x 8192
  D  a lone block in the last CTA inside one stream word and not, predecessors and a last segment ending on a word
  E  worst-case blocks: the longest AC strings 0/255 noise reaches, coefficient 63 alone, zero runs of 16 / 32 / 48,
     DC differences of category 11 in luma and chroma; binary RGB noise at q100 fits the device scan buffer
  F  0xFF bytes that take bits from two CTAs, sit at a window edge, or are the padded final byte
  G  output capacity: exactly the stream size succeeds, one byte less is UHDR_CODEC_MEM_ERROR with nothing written
"""
import ctypes as C
import os

import numpy as np
import pytest

import jpeg_scan_model as M
import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A

pytestmark = pytest.mark.gpu

E_MEM = 4   # UHDR_CODEC_MEM_ERROR
GUARD = 4096


# ------------------------------------------------------------------------------------------------
# checker, device call, route
# ------------------------------------------------------------------------------------------------
class Checker:
    """the reference's JpegEncoderHelper on libjpeg-turbo, else the C restatement pinned to it"""

    def __init__(self, oracle_libs):
        self.olib = oracle_libs.Oracle().lib
        self.turbo = C.CDLL(T.REF_TURBO_SO) if os.path.exists(T.REF_TURBO_SO) else None
        self.name = "JpegEncoderHelper/libjpeg-turbo" if self.turbo else "jo_encode"

    def encode(self, img, q):
        """-> stream bytes, or the error code"""
        if self.turbo is not None:
            cap = img.w * img.h * 8 + 65536
            out = np.zeros(cap, np.uint8)
            n = C.c_size_t()
            rc = self.turbo.ref_jpeg_encode(C.byref(img), q, None, C.c_size_t(0), out.ctypes.data_as(C.c_void_p),
                                            C.c_size_t(cap), C.byref(n))
            return rc if rc else bytes(out[:n.value])
        P, S = T._planes3(img)
        out, n = C.c_void_p(), C.c_size_t()
        gm = img.fmt in (A.FMT_RGB888, A.FMT_Y400)
        rc = self.olib.jo_encode(P, S, img.w, img.h, img.fmt, q, None, C.c_size_t(0), T.GM_COMMENT if gm else None,
                                 C.byref(out), C.byref(n))
        return rc if rc else C.string_at(out, n.value)


def gpu_encode(lib, img, q, cap=None):
    """-> (rc, bytes); checks that nothing past `cap` was written"""
    cap = cap if cap is not None else img.w * img.h * 6 + 65536
    out = np.full(cap + GUARD, 0xA5, np.uint8)
    n = C.c_size_t()
    rc = lib.uhdr_b200_jpeg_encode(C.byref(img), q, None, C.c_size_t(0), out.ctypes.data_as(C.c_void_p), C.c_size_t(cap),
                                   C.byref(n))
    assert (out[cap:] == 0xA5).all(), "bytes written past the capacity"
    if rc != 0:
        assert (out == 0xA5).all(), "a failing call wrote into the output"
    return rc, (bytes(out[:n.value]) if rc == 0 else None)


class Route:
    """growth of uhdr_b200_jpeg_encode_stats over the block: .bpt = launches by bpt 1..8, .beyond = launches beyond one wave"""

    def __init__(self, lib):
        self.lib = lib

    def __enter__(self):
        self.r0, self.b0, self.w0 = A.jpeg_encode_stats(self.lib)
        return self

    def __exit__(self, *exc):
        r, b, w = A.jpeg_encode_stats(self.lib)
        self.resident = r
        self.bpt = tuple(y - x for x, y in zip(self.b0, b))
        self.beyond = w - self.w0
        return False


def expected_bpt(nblocks, R):
    return min(8, max(1, -(-nblocks // (256 * R))))


@pytest.fixture(scope="module")
def env(gpu, oracle_libs):
    lib = A.declare_jpeg_encode_stats(gpu.lib)
    chk = Checker(oracle_libs)
    g = np.zeros((16, 16), np.uint8)
    rc, _ = gpu_encode(lib, A.raw_image(A.FMT_Y400, -1, -1, 1, 16, 16, [g], [16]), 90)
    assert rc == 0, T.gpu_err(gpu)
    R = A.jpeg_encode_stats(lib)[0]
    assert R > 0
    print(f"\nchecker: {chk.name}; k_huff_encode resident CTAs per wave: {R}")
    return lib, chk, R, gpu


def encode_and_compare(env, img, q, model=True, what=""):
    """GPU bytes == checker bytes at 0 tolerance, one k_huff_encode launch with the bpt the plan predicts.
    -> (scan model of the stream or None, Route)"""
    lib, chk, R, gpu = env
    want = chk.encode(img, q)
    assert not isinstance(want, int), f"checker refused {what}: {want}"
    with Route(lib) as rt:
        rc, got = gpu_encode(lib, img, q)
    assert rc == 0, (what, q, T.gpu_err(gpu))
    m = None
    if got != want or model:
        m = M.ScanModel(want, chk.olib)
    bpt = expected_bpt(m.nblocks, R) if m else None
    if got != want:
        k = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
        pytest.fail(f"{what} q{q}: {len(got)} vs {len(want)} bytes; first difference at {m.locate(k, bpt)}")
    assert sum(rt.bpt) == 1, rt.bpt
    if bpt:
        assert rt.bpt[bpt - 1] == 1, (what, q, bpt, rt.bpt)
    return m, rt


# ------------------------------------------------------------------------------------------------
# content
# ------------------------------------------------------------------------------------------------
def content(kind, h, w, ch=1, seed=0):
    rs = np.random.RandomState(T.SEED + 700 + seed)
    if kind == "noise":
        a = rs.randint(0, 256, (h, w, ch), dtype=np.uint8)
    elif kind == "binary":
        a = (rs.randint(0, 2, (h, w, ch), dtype=np.uint8) * np.uint8(255))
    elif kind == "smooth":
        x, y = np.arange(w, dtype=np.float32), np.arange(h, dtype=np.float32)[:, None]
        a = np.empty((h, w, ch), np.uint8)
        for k in range(ch):
            a[..., k] = 128 + 100 * np.sin(x / (37.0 + 11 * k)) * np.cos(y / (53.0 + 7 * k))
    elif kind == "flat":
        a = np.full((h, w, ch), 128, np.uint8)
    else:
        raise ValueError(kind)
    return np.ascontiguousarray(a)


def image(fmt, w, h, kind, seed=0):
    """-> (RawImage, arrays kept alive) in the layouts JpegEncoderHelper takes"""
    if fmt in (A.FMT_Y400, A.FMT_RGB888):
        a = content(kind, h, w, 1 if fmt == A.FMT_Y400 else 3, seed)
        return A.raw_image(fmt, -1, -1, 1, w, h, [a], [w]), a
    if fmt in (A.FMT_YUV420, A.FMT_YUV422, A.FMT_YUV444):
        cw = w if fmt == A.FMT_YUV444 else (w + 1) // 2
        chh = (h + 1) // 2 if fmt == A.FMT_YUV420 else h
        p = [content(kind, h, w, 1, seed)[..., 0].copy()] + [content(kind, chh, cw, 1, seed + k)[..., 0].copy() for k in (1, 2)]
        return A.raw_image(fmt, 1, 3, 1, w, h, p, [w, cw, cw]), p
    raise ValueError(fmt)


def y400(a):
    h, w = a.shape
    a = np.ascontiguousarray(a.astype(np.uint8))
    return A.raw_image(A.FMT_Y400, -1, -1, 1, w, h, [a], [w]), a


def tile_blocks(blocks, bw, bh):
    """(n, 8, 8) blocks -> a (bh*8, bw*8) plane, blocks repeated in raster order"""
    n = len(blocks)
    idx = np.arange(bw * bh) % n
    return blocks[idx].reshape(bh, bw, 8, 8).transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)


def basis_block(coefs):
    """{natural index: orthonormal DCT coefficient} -> an 8x8 block of samples (IDCT, +128, clamped)"""
    from scipy.fft import idctn
    X = np.zeros(64)
    for k, v in coefs.items():
        X[k] = v
    return np.clip(np.rint(idctn(X.reshape(8, 8), norm="ortho")) + 128, 0, 255).astype(np.uint8)


# ------------------------------------------------------------------------------------------------
# A: every quality x every layout at ragged sizes
# ------------------------------------------------------------------------------------------------
SIZES_A = {A.FMT_Y400: [(261, 37), (247, 19)], A.FMT_YUV420: [(264, 40), (246, 26)], A.FMT_YUV422: [(264, 36), (246, 19)],
           A.FMT_YUV444: [(261, 37), (247, 19)], A.FMT_RGB888: [(261, 37), (247, 19)]}


@pytest.mark.parametrize("fmt", list(SIZES_A))
def test_a_every_quality(env, fmt):
    for i, (w, h) in enumerate(SIZES_A[fmt]):
        img, keep = image(fmt, w, h, "noise" if i == 0 else "smooth", seed=i)
        for q in range(1, 101):
            m, rt = encode_and_compare(env, img, q, model=q in (1, 25, 100), what=f"fmt {fmt} {w}x{h}")
            if m is None:
                continue
            assert rt.bpt[0] == 1
            wb, hb = m.geom[0][2], m.geom[0][3]
            if fmt == A.FMT_RGB888:
                assert (wb * hb) % 8 and w % 8, "partial last warp item and right block"
            elif fmt == A.FMT_Y400:
                assert wb % 32 in (1, 31) and m.nblocks % 32
            else:   # dummy blocks: MCUs reach past a component's block grid
                assert (m.scan_blk < 0).any() or fmt == A.FMT_YUV444
        assert A.jpeg_encode_stats(env[0])[1][0] > 0


FMT_440, FMT_411, FMT_410 = 8, 9, 10   # UHDR_IMG_FMT_16bppYCbCr440, _12bppYCbCr411, _10bppYCbCr410


def test_a_refused_layouts(env):
    """4:4:0, 4:1:1 and 4:1:0, which the helper encodes, are not encoded on the GPU: a clean error, nothing written.
    What the helper refuses, the device call refuses too."""
    lib, chk, R, gpu = env
    p = np.full(64 * 48 * 4, 77, np.uint8)
    for fmt in (FMT_440, FMT_411, FMT_410):
        img = A.raw_image(fmt, 1, 3, 1, 64, 48, [p, p, p], [64, 64, 64])
        if chk.turbo is not None:
            assert not isinstance(chk.encode(img, 90), int), fmt
        with Route(lib) as rt:
            rc, _ = gpu_encode(lib, img, 90)
        assert rc != 0 and sum(rt.bpt) == 0, (fmt, rc)
    for fmt in (A.FMT_P010, A.FMT_RGBA8888, A.FMT_RGBA1010102, 99):
        img = A.raw_image(fmt, 1, 3, 1, 64, 48, [p, p, p], [64, 64, 64])
        if chk.turbo is not None:
            assert isinstance(chk.encode(img, 90), int), fmt
        rc, _ = gpu_encode(lib, img, 90)
        assert rc != 0, fmt


@pytest.mark.parametrize("fmt,w,h", [(A.FMT_Y400, 261, 37), (A.FMT_YUV420, 246, 26), (A.FMT_YUV422, 250, 19),
                                     (A.FMT_YUV444, 261, 37)])
def test_a_caller_bytes_past_the_width(env, fmt, w, h):
    """strides at least the 8-aligned width: the helper reads the caller's bytes between the width and the aligned
    width (noise here).  The stream and the forward stage's coefficients equal the checker's, and differ from those of
    the same image with zeros there (the case is reached)."""
    lib, chk, R, gpu = env
    rs = np.random.RandomState(w + h)
    cw = w if fmt in (A.FMT_Y400, A.FMT_YUV444) else (w + 1) // 2
    ch = (h + 1) // 2 if fmt == A.FMT_YUV420 else h
    dims = [(h, w, w + 11)] + ([] if fmt == A.FMT_Y400 else [(ch, cw, cw + 9)] * 2)
    noisy = [rs.randint(0, 256, (ph, st)).astype(np.uint8) for ph, pw, st in dims]
    clean = []
    for a, (ph, pw, st) in zip(noisy, dims):
        c = a.copy()
        c[:, pw:] = 0
        clean.append(c)
    strides = [st for _, _, st in dims]
    img = A.raw_image(fmt, 1, 3, 1, w, h, noisy, strides)
    img0 = A.raw_image(fmt, 1, 3, 1, w, h, clean, strides)
    for q in (100, 75):
        m, rt = encode_and_compare(env, img, q, what=f"fmt {fmt} {w}x{h} wide strides")
        assert rt.bpt[0] == 1
        assert chk.encode(img0, q) != chk.encode(img, q), "the bytes past the width must matter"
        f, want = T.oracle_forward(chk.olib, img, q)
        got = T.gpu_jpeg_forward(gpu, img, q, f)
        for c in range(f.ncomp):
            assert (got[c] == want[c]).all(), (fmt, q, c)


# ------------------------------------------------------------------------------------------------
# B: every bpt, both sides of each threshold
# ------------------------------------------------------------------------------------------------
def _factor(n, lim=8191):
    """n blocks as (wblocks, hblocks), both <= lim, the widest first; None if there is no such split"""
    for wb in range(min(lim, n), 0, -1):
        if n % wb == 0 and n // wb <= lim:
            return wb, n // wb
    return None


def threshold_sizes(R):
    """[(nblocks, wblocks, hblocks)]: k * 256 * R and the first block count above it that splits into a Y400 frame"""
    out = []
    for k in range(1, 9):
        n = k * 256 * R
        out.append((n,) + _factor(n))
        d = 1
        while _factor(n + d) is None:
            d += 1
        out.append((n + d,) + _factor(n + d))
    return out


@pytest.mark.parametrize("kind,q", [("noise", 100), ("smooth", 95)])
def test_b_every_bpt(env, kind, q):
    lib, chk, R, gpu = env
    seen = [0] * 8
    for n, wb, hb in threshold_sizes(R):
        img, keep = y400(content(kind, hb * 8, wb * 8, 1, seed=n % 97)[..., 0])
        m, rt = encode_and_compare(env, img, q, model=kind == "noise", what=f"Y400 {wb * 8}x{hb * 8} ({n} blocks)")
        bpt = expected_bpt(n, R)
        assert rt.bpt[bpt - 1] == 1 and rt.beyond == (1 if n > 8 * 256 * R else 0), (n, rt.bpt, rt.beyond)
        seen[bpt - 1] += 1
        if m is not None:
            assert m.nblocks == n
            P = m.plan(bpt)
            assert int(P["windows"].max()) >= 2, "noise at q100 must need several windows per CTA"
    assert all(seen), seen


# ------------------------------------------------------------------------------------------------
# C: beyond one wave
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt,kind,q", [(A.FMT_RGB888, "noise", 75), (A.FMT_YUV444, "smooth", 95)])
def test_c_beyond_one_wave(env, fmt, kind, q):
    lib, chk, R, gpu = env
    img, keep = image(fmt, 8192, 8192, kind, seed=3)
    m, rt = encode_and_compare(env, img, q, what=f"fmt {fmt} 8192x8192")
    assert m.nblocks == 3 * 1024 * 1024
    assert rt.bpt[7] == 1 and rt.beyond == 1, (rt.bpt, rt.beyond)
    assert m.plan(8)["ncta"] > R


# ------------------------------------------------------------------------------------------------
# D: short and aligned segment ends
# ------------------------------------------------------------------------------------------------
def test_d_short_and_aligned_segment_ends(env):
    """Y400 8 x 8 * (256 n + 1): a lone block in the last CTA at bpt 1.  Flat blocks of seeded levels give short
    blocks of varying length; the inputs below are chosen so the model shows the lone segment inside one stream
    word and not, a CTA whose predecessor ends on a word boundary, and a last segment that ends on one."""
    lib, chk, R, gpu = env
    want = {"one_word": 0, "not_one_word": 0, "pred_aligned": 0, "last_aligned": 0}
    for seed in range(64):
        n = 1 + seed % 24
        rs = np.random.RandomState(seed)
        nb = 256 * n + 1
        levels = rs.choice(np.array([128, 128, 128, 129, 120, 140, 0, 255]), nb)
        if seed % 4 == 3:
            levels[-1] = 255    # a long DC difference at the very end
        blocks = np.repeat(levels.astype(np.uint8), 64).reshape(nb, 8, 8)
        if seed % 8 == 5:
            blocks[-1] = content("noise", 8, 8, 1, seed)[..., 0]
        img, keep = y400(blocks.reshape(nb * 8, 8))
        ref = chk.encode(img, 90)
        P = M.ScanModel(ref, chk.olib).plan(1)
        hits = {"one_word": bool(P["one_word"][-1]), "not_one_word": not P["one_word"][-1],
                "pred_aligned": bool((P["sh"][1:] == 0).any()), "last_aligned": bool(P["ends_aligned"][-1])}
        if not any(hits[k] and want[k] < 2 for k in want):
            continue
        m, rt = encode_and_compare(env, img, 90, model=False, what=f"lone block, seed {seed}")
        assert rt.bpt[0] == 1
        for k in want:
            want[k] += hits[k]
        if all(v >= 2 for v in want.values()):
            break
    assert all(want.values()), want


# ------------------------------------------------------------------------------------------------
# E: worst-case blocks
# ------------------------------------------------------------------------------------------------
def test_e_ac_string_lengths(env):
    """AC strings of exactly 96 / 97 / 128 / 129 bits (the meta word is full / spills into the slot; the slot's
    first uint4 is full / not) and the longest ones 0/255 noise reaches at q100.  A block's AC string depends on
    that block alone, so blocks picked from seeded pools keep their lengths when tiled.  (8-bit samples bound the
    coefficient energy: with the Annex-K tables no block reaches much past 1100 bits.)"""
    lib, chk, R, gpu = env
    hit = {96: 0, 97: 0, 128: 0, 129: 0}
    for q, kind in ((100, "binary"), (100, "ramp"), (90, "ramp")):
        if kind == "ramp":   # noise whose amplitude grows from 1 to 32 over the block rows: every string length
            rs = np.random.RandomState(T.SEED + q)
            amp = (1 + np.arange(512) // 16)[:, None]
            a = 128 + np.rint((rs.rand(512, 512) * 2 - 1) * amp)
        else:
            a = content(kind, 512, 512, 1, seed=11)[..., 0]
        pool, keep = y400(a)
        pm = M.ScanModel(chk.encode(pool, q), chk.olib)
        blocks = keep.reshape(64, 8, 64, 8).transpose(0, 2, 1, 3).reshape(-1, 8, 8)
        pick = np.concatenate([np.nonzero(pm.acbits[0] == n)[0][:8] for n in hit] + [np.argsort(pm.acbits[0])[-32:]])
        img, k2 = y400(tile_blocks(blocks[pick], 37, 11))
        m, rt = encode_and_compare(env, img, q, what=f"AC string lengths, {kind} q{q}")
        cs = m.cases()
        for n in hit:
            hit[n] += cs[f"ac{n}"]
        if q == 100 and kind == "binary":
            assert cs["ac_max"] >= 960, cs
            print(f"longest AC string: {cs['ac_max']} bits")
    assert all(hit.values()), hit
    for fmt in (A.FMT_RGB888, A.FMT_YUV420):   # chroma strings, and the scan buffer bound of binary RGB noise
        img, keep = image(fmt, 1024 + 3, 512 + 5, "binary", seed=12)
        m, rt = encode_and_compare(env, img, 100, what=f"binary fmt {fmt}")
        assert m.cases()["ac_gt96"] > 0


def test_e_coefficient_63(env):
    blocks = np.stack([basis_block({63: a}) for a in (-300, -40, 40, 300)] + [basis_block({63: 200, 0: -500})])
    img, keep = y400(tile_blocks(blocks, 33, 9))
    for q in (50, 100):
        m, rt = encode_and_compare(env, img, q, what="coefficient 63")
        cs = m.cases()
        # at q100 the samples' rounding leaves small coefficients beside it; at q50 it stands alone (no EOB)
        assert cs["c63"] > 0 and (cs["c63_alone"] > 0 or q == 100), (q, cs)


def test_e_zero_runs(env):
    zz = M.NATURAL   # zigzag position -> natural index
    blocks = []
    for run in (16, 32, 48):
        for a in (200, -200):
            blocks.append(basis_block({int(zz[1]): a, int(zz[2 + run]): -a}))
            blocks.append(basis_block({int(zz[5]): a, int(zz[6 + run]): a}))
    img, keep = y400(tile_blocks(np.stack(blocks), 36, 7))
    for q in (50, 90):
        m, rt = encode_and_compare(env, img, q, what="zero runs")
        cs = m.cases()
        assert cs["zrl1"] > 0 and cs["zrl2"] > 0 and cs["zrl3"] > 0, (q, cs)


def test_e_dc_category_11(env):
    """0 / 255 blocks side by side: DC differences of +-2040 at q100 in Y (Y400, 4:2:0) and in Cb / Cr (RGB888
    blue / yellow, 4:4:4 and 4:2:0 chroma planes)"""
    lib, chk, R, gpu = env
    bw, bh = 19, 7
    yy, xx = np.mgrid[0:bh * 8, 0:bw * 8]
    chk_plane = (((yy // 8 + xx // 8) % 2) * 255).astype(np.uint8)
    img, keep = y400(chk_plane)
    m, _ = encode_and_compare(env, img, 100, what="Y400 DC swings")
    assert m.cases()["dc11_luma"] > 0
    rgb = np.where(chk_plane[..., None] > 0, np.uint8([0, 0, 255]), np.uint8([255, 255, 0])).astype(np.uint8)
    rgb = np.ascontiguousarray(rgb)
    img = A.raw_image(A.FMT_RGB888, -1, -1, 1, bw * 8, bh * 8, [rgb], [bw * 8])
    m, _ = encode_and_compare(env, img, 100, what="RGB888 DC swings")
    assert m.cases()["dc11_chroma"] > 0
    for fmt in (A.FMT_YUV444, A.FMT_YUV420):
        w, h = 16 * 9, 16 * 5
        yy, xx = np.mgrid[0:h, 0:w]
        y = (((yy // 8 + xx // 8) % 2) * 255).astype(np.uint8)
        cw, chh = (w, h) if fmt == A.FMT_YUV444 else (w // 2, h // 2)
        cy, cx = np.mgrid[0:chh, 0:cw]
        u = (((cy // 8 + cx // 8) % 2) * 255).astype(np.uint8)
        v = np.ascontiguousarray(255 - u)
        img = A.raw_image(fmt, 1, 3, 1, w, h, [y, u, v], [w, cw, cw])
        m, _ = encode_and_compare(env, img, 100, what=f"fmt {fmt} DC swings")
        cs = m.cases()
        assert cs["dc11_luma"] > 0 and cs["dc11_chroma"] > 0, cs


# ------------------------------------------------------------------------------------------------
# F: byte stuffing at CTA and window boundaries, padded final byte
# ------------------------------------------------------------------------------------------------
def test_f_stuffing_at_boundaries(env):
    lib, chk, R, gpu = env
    found = {"two_ctas": 0, "window_edge": 0, "padded_last": 0}
    # heavy segments (several windows per CTA) with many CTA boundaries
    for seed in range(6):
        img, keep = image(A.FMT_Y400, 2048, 1024, "binary", seed=40 + seed)
        m, rt = encode_and_compare(env, img, 100, what=f"stuffing seed {seed}")
        ff = m.ff_bytes(m.plan(expected_bpt(m.nblocks, R)))
        found["two_ctas"] += int(ff["two_ctas"].sum())
        found["window_edge"] += int(ff["window_edge"].sum())
        if found["two_ctas"] and found["window_edge"]:
            break
    # the padded final byte: a last block whose coefficient 63 ends in one bits, so the padded byte is all ones
    for seed in range(400):
        img, keep = image(A.FMT_Y400, 24, 16, "binary", seed=1000 + seed)
        ref = chk.encode(img, 100)
        mm = M.ScanModel(ref, chk.olib)
        if not mm.ff_bytes(mm.plan(1))["padded_last"].any():
            continue
        encode_and_compare(env, img, 100, model=False, what=f"padded 0xFF, seed {seed}")
        found["padded_last"] += 1
        if found["padded_last"] >= 2:
            break
    assert all(found.values()), found


# ------------------------------------------------------------------------------------------------
# G: output capacity
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt,w,h,kind", [(A.FMT_Y400, 261, 37, "noise"), (A.FMT_YUV420, 640, 480, "binary"),
                                          (A.FMT_RGB888, 250, 130, "smooth")])
def test_g_output_capacity(env, fmt, w, h, kind):
    lib, chk, R, gpu = env
    img, keep = image(fmt, w, h, kind, seed=5)
    want = chk.encode(img, 100)
    bpt = expected_bpt(M.ScanModel(want, chk.olib).nblocks, R)
    for cap in (len(want), len(want) - 1, len(want) // 2, 0):
        with Route(lib) as rt:
            rc, got = gpu_encode(lib, img, 100, cap=cap)
        assert sum(rt.bpt) == 1 and rt.bpt[bpt - 1] == 1 and rt.beyond == 0, (cap, rt.bpt)
        if cap == len(want):
            assert rc == 0 and got == want
        else:
            assert rc == E_MEM, (cap, rc)
