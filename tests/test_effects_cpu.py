"""The editor API's setters (uhdr_add_effect_mirror / _rotate / _crop / _resize) against the reference's state
machine, without a device: null handle, bad arguments, after uhdr_dec_probe, after the handle sailed, and a reset that
clears the list.  Also holds the helpers test_gpu_effects.py drives both libraries with."""
import ctypes as C

import numpy as np
import pytest

import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A

OK, INVALID_PARAM, INVALID_OPERATION = 0, 3, 5
MIRROR_VERTICAL, MIRROR_HORIZONTAL = 0, 1


def declare(lib):
    """restypes of the C API calls these tests make, on libuhdr_b200 or the reference build"""
    T.UhdrApi(lib)
    for f in ("uhdr_add_effect_mirror", "uhdr_add_effect_rotate", "uhdr_add_effect_crop", "uhdr_add_effect_resize",
              "uhdr_enc_set_compressed_image", "uhdr_enc_set_gainmap_image"):
        getattr(lib, f).restype = A.ErrorInfo
    lib.uhdr_add_effect_mirror.argtypes = [C.c_void_p, C.c_int]
    lib.uhdr_add_effect_rotate.argtypes = [C.c_void_p, C.c_int]
    lib.uhdr_add_effect_crop.argtypes = [C.c_void_p] + [C.c_int] * 4
    lib.uhdr_add_effect_resize.argtypes = [C.c_void_p] + [C.c_int] * 2
    return lib


def add(lib, handle, effect):
    """effect: ("mirror", direction) / ("rotate", degrees) / ("crop", left, right, top, bottom) / ("resize", w, h)"""
    return getattr(lib, "uhdr_add_effect_" + effect[0])(handle, *effect[1:]).error_code


def api4_inputs():
    """a small JPEG/R's base image, gain map and metadata, for host-only encodes (API-4)"""
    PIL = pytest.importorskip("PIL.Image")
    import io
    rng = np.random.default_rng(7)
    a = (rng.random((64, 96, 3)) * 255).astype(np.uint8)
    b, g = io.BytesIO(), io.BytesIO()
    PIL.fromarray(a).save(b, format="JPEG", quality=90)
    PIL.fromarray(a[::2, ::2, 0]).save(g, format="JPEG", quality=90)
    md = A.GainmapMetadata()
    for i in range(3):
        md.max_content_boost[i], md.min_content_boost[i], md.gamma[i] = 4.0, 1.0, 1.0
        md.offset_sdr[i] = md.offset_hdr[i] = 1.0 / 64
    md.hdr_capacity_min, md.hdr_capacity_max, md.use_base_cg = 1.0, 4.0, 1
    return b.getvalue(), g.getvalue(), md


def encode_api4(lib, enc, base, gm, md):
    bb, gb = np.frombuffer(base, np.uint8).copy(), np.frombuffer(gm, np.uint8).copy()
    bi = A.CompressedImage(bb.ctypes.data, len(base), len(base), A.CG_BT709, -1, -1)
    gi = A.CompressedImage(gb.ctypes.data, len(gm), len(gm), -1, -1, -1)
    assert lib.uhdr_enc_set_compressed_image(enc, C.byref(bi), A.BASE_IMG).error_code == OK
    assert lib.uhdr_enc_set_gainmap_image(enc, C.byref(gi), C.byref(md)).error_code == OK
    e = lib.uhdr_encode(enc)
    out = None
    if e.error_code == OK:
        o = lib.uhdr_get_encoded_stream(enc).contents
        out = C.string_at(o.data, o.data_sz)
    return e.error_code, out


@pytest.fixture(scope="module")
def libs(oracle_libs):
    if not oracle_libs.have_ref():
        pytest.skip("reference build not available")
    import __graft_entry__ as g
    g.build()
    return declare(C.CDLL(T.GPU_SO)), declare(C.CDLL(T.REF_SO))


BAD_AND_GOOD = [("mirror", MIRROR_VERTICAL), ("mirror", MIRROR_HORIZONTAL), ("mirror", 2), ("mirror", -1),
                ("rotate", 90), ("rotate", 180), ("rotate", 270), ("rotate", 0), ("rotate", 360), ("rotate", -90),
                ("rotate", 45), ("crop", 0, 0, 0, 0), ("crop", -5, -10, 7, 3), ("crop", 0, 100000, 0, 1),
                ("resize", 0, 0), ("resize", -1, 5), ("resize", 100000, 1), ("resize", 64, 48)]


@pytest.mark.parametrize("kind", ["encoder", "decoder"])
def test_setter_codes_equal_the_reference(libs, kind):
    codes = []
    for lib in libs:
        h = C.c_void_p(getattr(lib, f"uhdr_create_{kind}")())
        try:
            codes.append([add(lib, h, e) for e in BAD_AND_GOOD] + [add(lib, None, e) for e in BAD_AND_GOOD])
        finally:
            getattr(lib, f"uhdr_release_{kind}")(h)
    assert codes[0] == codes[1]
    assert codes[0][:len(BAD_AND_GOOD)].count(OK) == 12 and set(codes[0][len(BAD_AND_GOOD):]) == {INVALID_PARAM}


def test_encoder_effects_with_compressed_intent_then_after_sail(libs):
    base, gm, md = api4_inputs()
    for lib in libs:
        enc = C.c_void_p(lib.uhdr_create_encoder())
        try:
            assert add(lib, enc, ("rotate", 90)) == OK
            assert encode_api4(lib, enc, base, gm, md) == (INVALID_OPERATION, None)
            assert lib.uhdr_get_encoded_stream(enc) is None or not lib.uhdr_get_encoded_stream(enc)
            # sailed: every setter refuses, bad arguments first
            assert [add(lib, enc, e) for e in [("rotate", 90), ("rotate", 45), ("mirror", 7), ("crop", 0, 1, 0, 1),
                                               ("resize", 8, 8)]] == [INVALID_OPERATION, INVALID_PARAM, INVALID_PARAM,
                                                                      INVALID_OPERATION, INVALID_OPERATION]
            # a reset clears the list and the end state: the same inputs now encode, byte for byte as the reference
            lib.uhdr_reset_encoder(enc)
            rc, out = encode_api4(lib, enc, base, gm, md)
            assert rc == OK and out
            if lib is libs[1]:
                assert out == mine
            else:
                mine = out
        finally:
            lib.uhdr_release_encoder(enc)


def test_decoder_takes_effects_after_probe_and_not_after_sail(libs):
    base, gm, md = api4_inputs()
    ref = libs[1]
    enc = C.c_void_p(ref.uhdr_create_encoder())
    try:
        rc, data = encode_api4(ref, enc, base, gm, md)
    finally:
        ref.uhdr_release_encoder(enc)
    assert rc == OK
    buf = np.frombuffer(data, np.uint8).copy()
    ci = A.CompressedImage(buf.ctypes.data, len(data), len(data), -1, -1, -1)
    seen = []
    for lib in libs:
        dec = C.c_void_p(lib.uhdr_create_decoder())
        try:
            # an output pair uhdr_decode refuses before any decoding: it still sails the handle
            r = [lib.uhdr_dec_set_image(dec, C.byref(ci)).error_code,
                 lib.uhdr_dec_set_out_img_format(dec, A.FMT_RGBA8888).error_code,
                 lib.uhdr_dec_set_out_color_transfer(dec, A.CT_HLG).error_code, lib.uhdr_dec_probe(dec).error_code]
            # probed, not sailed: effects are still taken, other setters are not
            r += [add(lib, dec, ("mirror", MIRROR_HORIZONTAL)), lib.uhdr_dec_set_out_max_display_boost(dec, 2.0).error_code]
            r += [lib.uhdr_decode(dec).error_code, add(lib, dec, ("rotate", 90)), add(lib, dec, ("rotate", 1))]
            lib.uhdr_reset_decoder(dec)
            r += [add(lib, dec, ("rotate", 90))]
            seen.append(r)
        finally:
            lib.uhdr_release_decoder(dec)
    assert seen[0] == seen[1]
    assert seen[0] == [OK, OK, OK, OK, OK, INVALID_OPERATION, INVALID_PARAM, INVALID_OPERATION, INVALID_PARAM, OK]
