"""The GPU JPEG decoder route by route (huffdec.cu k_hd_layout / k_hd_sync / k_hd_scan / k_hd_write / k_dc_*, then
k_idct<8> and k_ycc_to_rgba) on streams other encoders write: optimised and hand-made Huffman tables, every table selector,
4:4:0 / 4:1:1 / 4:1:0 and 10-block MCUs, subsequence boundaries on every bit of a symbol, restart intervals of
n 1024 +- 1 bits, flat frames whose relaxation converges slowly or not at all, IDCT and colour-conversion edges.

Every case decodes through the single-JPEG stage API and must equal libjpeg-turbo (oracle/jpeg_scaled_ref.c) at 0
tolerance, planes and RGBA, and the host entropy decoder's output; the uhdr_b200_entropy_decoder_stats delta shows
the route (device done or handed back, and the relaxation rounds, against the lock-step model of
tests/jpeg_stream_writer.py).  The streams come from tests/jpeg_decode_cases.py."""
import ctypes as C
import math

import numpy as np
import pytest

import jpeg_decode_cases as D
import jpeg_stream_writer as W
import scaled_testlib as S
from libultrahdr_b200 import ctypes_api as A

pytestmark = pytest.mark.gpu
UNSUPPORTED = 6
SENTINEL = 0xA5


@pytest.fixture(scope="module")
def lib(gpu):
    L = gpu.lib
    L.uhdr_b200_entropy_decoder_stats.restype = None
    L.uhdr_b200_last_error.restype = C.c_char_p
    if not S.have_harness():
        pytest.skip("no libjpeg-turbo harness")
    return L


def _stats(L):
    st = (C.c_ulonglong * 3)()
    L.uhdr_b200_entropy_decoder_stats(st)
    return list(st)


def _decode(L, data, mode, entropy):
    """-> rc, out descriptor, buffer, stats delta (done, declined) and rounds after the decode"""
    cap = 4 * 8200 * 8200 if len(data) > 4000000 else 4 * (len(data) * 64 + (1 << 20))
    buf = np.full(cap, SENTINEL, np.uint8)
    out = A.raw_image(-1, -1, -1, -1, 0, 0, [buf], [0])
    src = np.frombuffer(data, np.uint8).copy()
    prev = L.uhdr_b200_set_entropy_decoder(entropy)
    try:
        s0 = _stats(L)
        rc = L.uhdr_b200_jpeg_decode(src.ctypes.data_as(C.c_void_p), C.c_size_t(src.size), mode, C.byref(out),
                                     C.c_size_t(cap))
        s1 = _stats(L)
    finally:
        L.uhdr_b200_set_entropy_decoder(prev)
    return rc, out, buf, (s1[0] - s0[0], s1[1] - s0[1], s1[2])


def _planes(out, buf, dims):
    res = []
    for c, (w, h) in enumerate(dims):
        off = out.planes[c] - buf.ctypes.data
        s = out.stride[c]
        res.append(buf[off:off + s * h].reshape(h, s)[:, :w])
    return res


def _first_diff(got, ref, c, name):
    ys, xs = np.nonzero(got != ref)
    y, x = int(ys[0]), int(xs[0])
    return "%s: component %d differs in %d samples, first at block (%d, %d) sample (%d, %d): %d != %d" % (
        name, c, len(ys), x // 8, y // 8, x, y, int(got[y, x]), int(ref[y, x]))


def _nseq(data):
    if isinstance(data, bytes):
        return None
    return len(W.subsequences(data))


def _rounds_ok(st, want, rounds):
    """the model runs every round in lock step; on the device a CTA that starts after the one before it wrote its
    states reads them in the same round, so the true states may cross a CTA boundary (128 subsequences) a round early"""
    return max(1, want - math.ceil(_nseq(st) / 128) - 1) <= rounds <= want


def check(L, name, st, expect, rgba=True):
    """planes (and RGBA) equal to libjpeg-turbo and to the host decoder; route from the stats delta -> device rounds"""
    data = st if isinstance(st, bytes) else st.data
    info, ref = S.harness_decode(data, 1)
    assert info[15] == 0, (name, "libjpeg-turbo warnings", info[15])
    dims = [(info[5 + 3 * c], info[6 + 3 * c]) for c in range(info[2])]
    rc, out, buf, (done, declined, rounds) = _decode(L, data, 0, 2)
    assert rc == 0, (name, L.uhdr_b200_last_error())
    want = expect["rounds"]
    if want is None:   # more than kMaxRounds: handed back to the host decoder
        assert (done, declined) == (0, 1), (name, done, declined, expect["why"])
    else:
        assert (done, declined) == (1, 0), (name, done, declined, expect["why"])
        if want == 0:
            assert rounds == 0, (name, rounds, expect["why"])
        elif want != "any":
            assert _rounds_ok(st, want, rounds), (name, "device rounds", rounds, "model", want, expect["why"])
    got = _planes(out, buf, dims)
    for c, (g, r) in enumerate(zip(got, ref)):
        if not (g == r).all():
            raise AssertionError(_first_diff(g, r, c, name))
    rc, out_h, buf_h, (hd, hdec, _r) = _decode(L, data, 0, 1)
    assert rc == 0 and (hd, hdec) == (0, 0), name
    for c, (g, h) in enumerate(zip(got, _planes(out_h, buf_h, dims))):
        if not (g == h).all():
            raise AssertionError("host decoder: " + _first_diff(g, h, c, name))
    if rgba and info[2] == 3:
        _i, ref_rgba = S.harness_decode(data, 1, 1)
        for entropy in (2, 1):
            rc, out, buf, _s = _decode(L, data, 1, entropy)
            assert rc == 0 and out.fmt == A.FMT_RGBA8888, (name, entropy, rc)
            g = buf[:info[0] * info[1] * 4].reshape(info[1], info[0], 4)
            bad = (g != ref_rgba).any(-1)
            assert not bad.any(), (name, entropy, "rgba differs at", int(bad.sum()), "pixels, first (y, x)",
                                   tuple(int(v) for v in np.argwhere(bad)[0]))
    return rounds


def _run(L, cases, **kw):
    seen = {}
    for name, st, expect in cases:
        seen[name] = (check(L, name, st, expect, **kw), expect["rounds"], expect["why"])
    print("\n".join("%s: device rounds %s, model %s (%s)" % (k, *v) for k, v in seen.items()))
    return seen


# ---- A, B: tables -------------------------------------------------------------------------------------------------
def test_A_table_shapes(lib):
    cases = D.cases_tables()
    why = {n: e["why"] for n, _s, e in cases}
    assert "1-bit" in why["A_dc_1bit"] and "12-bit" in why["A_dc_12bit"]
    assert why["A_ac_all_lut"].endswith("9 bits")
    ln = [int(x) for x in why["A_ac_long_common"].replace(",", " ").split() if x.isdigit()]
    assert all(14 <= v <= 16 for v in ln), why["A_ac_long_common"]
    _run(lib, cases)


def test_B_table_selectors(lib):
    _run(lib, D.cases_selectors())


# ---- C: samplings -------------------------------------------------------------------------------------------------
def test_C_samplings_planes(lib):
    _run(lib, D.cases_samplings(), rgba=False)


def test_C_rgba_of_440_411_410_is_unsupported(lib):
    """mode 1 of a sampling the colour conversion does not implement: UHDR_CODEC_UNSUPPORTED_FEATURE, nothing written"""
    for name, st, _e in D.cases_samplings():
        rc, out, buf, _s = _decode(lib, st.data, 1, 2)
        if name.startswith("C_422"):
            assert rc == 0, name
            continue
        assert rc == UNSUPPORTED, (name, rc)
        assert (buf == SENTINEL).all(), name


# ---- D: subsequence boundaries and interval lengths ----------------------------------------------------------------
def test_D_boundaries_on_every_bit_of_a_symbol(lib):
    cases = D.cases_boundaries()
    kinds = {n.rsplit("_bit", 1)[0] for n, _s, _e in cases}
    assert kinds == {"D_dc_code", "D_dc_mag", "D_ac_code", "D_ac_mag", "D_eob_code", "D_zrl_code", "D_mcu_last"}, kinds
    _run(lib, cases)


def test_D_interval_lengths(lib):
    seen = _run(lib, D.cases_interval_lengths())
    assert seen["D_every_interval_one_subsequence"][0] == 0


# ---- E: convergence -----------------------------------------------------------------------------------------------
def test_E_flat_frames_converge_as_the_model_predicts(lib):
    seen = _run(lib, D.cases_convergence())
    assert seen["E_flat_420_1920x1080_bad"][0] > 100 and seen["E_flat_420_1920x1080_good"][0] < 8, seen
    assert seen["E_flat_gray_1920x1080_bad"][0] > 100 and seen["E_flat_gray_1920x1080_good"][0] < 8, seen
    assert seen["E_black_420_3840x2160_bad"][1] is None and seen["E_black_420_3840x2160_good"][1] is not None


# ---- F: large scans -----------------------------------------------------------------------------------------------
def test_F_large_scans(lib):
    _run(lib, D.cases_large())


def test_F_8192_noise_q100(lib):
    """8192 x 8192 4:2:0 q100 noise: ~500k subsequences, so k_hd_scan carries over hundreds of its 1024-wide steps"""
    data = S.pil_jpeg(S.image(8192, 8192, "noise", seed=3), 100, "420")
    _run(lib, [("F_noise_420_8192x8192_q100", data, {"rounds": "any", "why": "%d bytes" % len(data)})], rgba=False)


# ---- G, H: IDCT and colour conversion -----------------------------------------------------------------------------
def test_G_idct_single_coefficients_and_checkerboards(lib):
    _run(lib, D.cases_idct())


def test_G_idct_wide_products_against_the_exact_islow(lib, oracle_libs):
    """|coefficient x quantiser| up to 32767 (single coefficients) and 2047 (checkerboards): libjpeg-turbo's SIMD
    IDCT wraps there, so the planes are compared with the C restatement's islow (jo_inverse) instead"""
    o = oracle_libs.Oracle().lib
    for name, st, expect in D.cases_idct(wide=True):
        rc, out, buf, (done, declined, rounds) = _decode(lib, st.data, 0, 2)
        assert rc == 0 and (done, declined) == (1, 0), (name, rc, done, declined)
        assert _rounds_ok(st, expect["rounds"], rounds), (name, rounds, expect["rounds"])
        f = st.frame
        dims = list(zip(f.dw, f.dh))
        _h, ref = oracle_libs.oracle_decode(o, st.data)
        for c, (g, r) in enumerate(zip(_planes(out, buf, dims), ref)):
            r = r[:dims[c][1], :dims[c][0]]
            if not (g == r).all():
                raise AssertionError(_first_diff(g, r, c, name))
            if c == 0:   # the two checkerboards, the last blocks of luma, overshoot [-128, 127] both ways
                n = len(D.idct_blocks(D.QUANTISERS[name.split("_")[3]][0], True))
                for i in (n - 2, n - 1):
                    by, bx = divmod(i, f.wb[0])
                    blk = r[by * 8:by * 8 + 8, bx * 8:bx * 8 + 8]
                    assert blk.min() == 0 and blk.max() == 255, (name, i)


def test_I_whole_file_from_writer_made_jpegs(lib, oracle_libs):
    """a JPEG/R assembled through API-4 from a writer-made 4:2:0 primary with optimal tables and a flat
    single-channel gain map: uhdr_decode equals the reference's, with both scans on the device"""
    if not oracle_libs.have_ref():
        pytest.skip("reference build not available")
    import uhdr_testlib as T
    from test_api4_cpu import _api4
    from test_probe_cpu import _probe
    base, gm, md = D.jpegr_parts(lib, 1280, 720)
    data = _api4(lib, base.data, gm.data, md, base_cg=A.CG_BT709)
    assert isinstance(data, bytes), data
    mine, ref = T.UhdrApi(lib), T.UhdrApi(oracle_libs.Ref().lib)
    s0 = _stats(lib)
    pa, ga, ma, cga = mine.decode(data)
    s1 = _stats(lib)
    assert (s1[0] - s0[0], s1[1] - s0[1]) == (2, 0), (s0, s1)
    pb, gb, mb, cgb = ref.decode(data)
    assert T.md_equal(ma, mb) and cga == cgb
    assert (ga == gb).all()
    assert (pa == pb).all(), int((pa != pb).sum())
    assert _probe(lib, data)["dims"] == (1280, 720, 320, 180)


def test_H_colour_conversion_tiny_frames(lib):
    cases = D.cases_colour()
    ref = np.concatenate([S.harness_decode(st.data, 1, 1)[1].reshape(-1, 4) for _n, st, _e in cases])
    for ch in range(3):   # every channel clamps both ways somewhere
        assert ref[:, ch].min() == 0 and ref[:, ch].max() == 255, ch
    _run(lib, cases)
