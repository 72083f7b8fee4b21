"""uhdr_add_effect_* chains through uhdr_decode and uhdr_encode on the GPU, against the reference's C API
(oracle/_ref/libuhdr_ref_turbo.so) byte for byte: decoded images and gain maps row by row with their w, h, fmt, cg and
ct; encoded JPEG/R files whole; error codes where the reference refuses, with nothing returned.  Also: one
k_effect_gather launch per plane whatever the chain's length, and no heap calls in steady state."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A
from test_effects_cpu import INVALID_OPERATION, INVALID_PARAM, MIRROR_HORIZONTAL as MH, MIRROR_VERTICAL as MV, OK, add, declare

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BPP = {A.FMT_RGBAF16: 8, A.FMT_RGBA1010102: 4, A.FMT_RGBA8888: 4, A.FMT_Y400: 1}


@pytest.fixture(scope="module")
def libs(gpu, oracle_libs):
    if not oracle_libs.have_ref():
        pytest.skip("reference build not available")
    gpu.lib.uhdr_b200_kernel_launches.restype = C.c_ulonglong
    return declare(gpu.lib), declare(C.CDLL(T.REF_SO))


def _rows(img):
    """((w, h, fmt, cg, ct, range), the w pixels of every row) of a returned packed image"""
    b = BPP[img.fmt]
    a = np.ctypeslib.as_array(C.cast(img.planes[0], C.POINTER(C.c_uint8)), (img.h, img.stride[0] * b))
    return (img.w, img.h, img.fmt, img.cg, img.ct, img.range), a[:, :img.w * b].copy()


def decode(lib, data, fmt, ct, effects):
    dec = C.c_void_p(lib.uhdr_create_decoder())
    try:
        buf = np.frombuffer(data, np.uint8).copy()
        ci = A.CompressedImage(buf.ctypes.data, len(data), len(data), -1, -1, -1)
        assert lib.uhdr_dec_set_image(dec, C.byref(ci)).error_code == OK
        assert lib.uhdr_dec_set_out_img_format(dec, fmt).error_code == OK
        assert lib.uhdr_dec_set_out_color_transfer(dec, ct).error_code == OK
        for e in effects:
            assert add(lib, dec, e) == OK
        rc = lib.uhdr_decode(dec).error_code
        if rc != OK:
            assert not lib.uhdr_get_decoded_image(dec) and not lib.uhdr_get_decoded_gainmap_image(dec)
            return rc, None, None
        return rc, _rows(lib.uhdr_get_decoded_image(dec).contents), _rows(lib.uhdr_get_decoded_gainmap_image(dec).contents)
    finally:
        lib.uhdr_release_decoder(dec)


def same_decode(libs, data, fmt, ct, effects):
    got, want = decode(libs[0], data, fmt, ct, effects), decode(libs[1], data, fmt, ct, effects)
    assert got[0] == want[0], (effects, got[0], want[0])
    for g, w in zip(got[1:], want[1:]):
        if w is None:
            continue
        # the descriptor's range is not compared: uhdr_decode reports UHDR_CR_FULL_RANGE where the reference leaves the
        # caller's UHDR_CR_UNSPECIFIED, with or without effects (the effects copy it unchanged in both libraries)
        assert g[0][:5] == w[0][:5], (effects, g[0], w[0])
        assert np.array_equal(g[1], w[1]), (effects, int((g[1] != w[1]).sum()))
    return want


# ---- decode -----------------------------------------------------------------------------------------------------
def _file(api, w, h, hdr_fmt, scale, multichannel):
    if hdr_fmt == A.FMT_P010:
        hb = T.make_p010(w, h, "smooth")
        hdr, k = A.p010_image(hb, w, h, A.CG_BT2100, A.CT_HLG, A.CR_LIMITED)
    else:
        hb = T.make_rgba1010102(w, h)
        hdr = A.raw_image(A.FMT_RGBA1010102, A.CG_BT2100, A.CT_PQ, A.CR_FULL, w, h, [hb], [w])
    return api.encode(hdr, None, scale=scale, multichannel=multichannel)


@pytest.fixture(scope="module")
def files(libs):
    mine = T.UhdrApi(libs[0])
    return {  # uhdr_encode's files equal the reference's (test_gpu_bench_geometry, test_gpu_stages)
        "998x722 1ch map/4": _file(mine, 998, 722, A.FMT_P010, 4, 0),         # map 250 x 181: ratios 3.992, 3.989
        "640x480 3ch map/1": _file(mine, 640, 480, A.FMT_RGBA1010102, 1, 1),
        "1001x723 3ch map/2": _file(mine, 1001, 723, A.FMT_RGBA1010102, 2, 1),  # odd image, odd map 501 x 362
    }


OUTPUTS = [(A.FMT_RGBAF16, A.CT_LINEAR), (A.FMT_RGBA1010102, A.CT_HLG), (A.FMT_RGBA1010102, A.CT_PQ),
           (A.FMT_RGBA8888, A.CT_SRGB)]
DECODE_CHAINS = [
    [("mirror", MH)], [("mirror", MV)], [("rotate", 90)], [("rotate", 180)], [("rotate", 270)],
    [("crop", 17, 611, 9, 333)], [("resize", 321, 205)],
    [("rotate", 90)] * 4, [("mirror", MH), ("mirror", MH)], [("mirror", MV), ("rotate", 90), ("mirror", MH)],
    [("crop", 10, 500, 7, 301), ("rotate", 270), ("resize", 100, 201)],
    [("resize", 333, 217)], [("resize", 1203, 901)],                     # down by non-dividing sizes, and up (ratio 0)
    [("crop", -20, 5000, -3, 100000)], [("crop", 3, 90, -7, 40), ("crop", 1, 50, 2, 30)],  # past the edges
    [("rotate", 270), ("crop", 5, 6, 11, 13), ("resize", 7, 3)],
]
DECODE_ERRORS = [
    [("crop", 50, 50, 0, 10)], [("crop", 0, 10, 60, 20)], [("crop", 5000, 6000, 0, 10)],   # empty on the image
    [("crop", 1, 3, 0, 100)], [("crop", 0, 100, 2, 3)],      # empty only on a scale-4 map: (int)(3 / 3.992) == 0
    [("resize", 8193, 10)], [("resize", 10, 0)], [("resize", -4, 9)], [("resize", 3, 3)],   # 3 / 3.992 -> 0 map columns
    [("rotate", 90), ("resize", 100, 100), ("crop", 100, 200, 0, 10)],
]


@pytest.mark.parametrize("name", ["998x722 1ch map/4", "640x480 3ch map/1", "1001x723 3ch map/2"])
@pytest.mark.parametrize("fmt,ct", OUTPUTS)
def test_decode_chains(libs, files, name, fmt, ct):
    codes = [same_decode(libs, files[name], fmt, ct, chain)[0] for chain in DECODE_CHAINS]
    # the last chain leaves a 1-pixel-wide image: its map rectangle is empty at map scales above 1
    assert codes[:-1] == [OK] * (len(codes) - 1) and codes[-1] in (OK, INVALID_PARAM), codes
    same_decode(libs, files[name], fmt, ct, [("resize", 8192, 4)])   # the largest size the reference takes


@pytest.mark.parametrize("name", ["998x722 1ch map/4", "1001x723 3ch map/2"])
def test_decode_errors(libs, files, name):
    seen = []
    for chain in DECODE_ERRORS:
        seen.append(same_decode(libs, files[name], A.FMT_RGBAF16, A.CT_LINEAR, chain)[0])
    assert seen.count(OK) <= 3 and INVALID_PARAM in seen, seen
    if name.startswith("998"):
        assert seen[3] == seen[4] == seen[8] == INVALID_PARAM


def test_decode_4080x3072_map_scale_4(libs):
    data = _file(T.UhdrApi(libs[0]), 4080, 3072, A.FMT_P010, 4, 0)
    for chain in ([("rotate", 90), ("crop", 3, 2001, 5, 3001)], [("crop", 1, 4079, 2, 3071), ("resize", 997, 733)],
                  [("mirror", MV), ("rotate", 270)]):
        same_decode(libs, data, A.FMT_RGBAF16, A.CT_LINEAR, chain)


def test_decode_8k_rotate_crop(libs):
    """bench.py's decode input through rotate 90 + crop: the swap-tile path on a grid of many waves"""
    import bench
    p, y = bench.make_frame(7680, 4320, 7)
    hdr, sdr, keep = bench.frame_descs(p, y, 7680, 4320)
    data = T.UhdrApi(libs[0]).encode(hdr, sdr)
    same_decode(libs, data, A.FMT_RGBAF16, A.CT_LINEAR, [("rotate", 90), ("crop", 8, 4312, 16, 7664)])


def test_decode_one_gather_per_image(libs, files):
    lib = libs[0]
    chain = [("mirror", MH), ("rotate", 90), ("mirror", MV), ("rotate", 270), ("rotate", 180)]
    counts = []
    for effects in ([], chain, []):
        n0 = lib.uhdr_b200_kernel_launches()
        decode(lib, files["640x480 3ch map/1"], A.FMT_RGBAF16, A.CT_LINEAR, effects)
        counts.append(lib.uhdr_b200_kernel_launches() - n0)
    assert counts[0] == counts[2] and counts[1] == counts[0] + 2, counts


# ---- encode -----------------------------------------------------------------------------------------------------
def _intents(hdr_fmt, sdr_fmt, w, h):
    keep = []
    if hdr_fmt == A.FMT_P010:
        hb = T.make_p010(w, h)
        hdr, _ = A.p010_image(hb, w, h, A.CG_BT2100, A.CT_PQ, A.CR_LIMITED)
    elif hdr_fmt == A.FMT_RGBA1010102:
        hb = T.make_rgba1010102(w, h)
        hdr = A.raw_image(A.FMT_RGBA1010102, A.CG_P3, A.CT_HLG, A.CR_FULL, w, h, [hb], [w])
    else:
        hb = T.make_rgbaf16(w, h)
        hdr = A.raw_image(A.FMT_RGBAF16, A.CG_BT2100, A.CT_LINEAR, A.CR_FULL, w, h, [hb], [w])
    keep.append(hb)
    sdr = None
    if sdr_fmt == A.FMT_YUV420:
        sb = T.make_yuv420(w, h)
        sdr, _ = A.yuv420_image(sb, w, h, A.CG_BT709)
        keep.append(sb)
    elif sdr_fmt == A.FMT_RGBA8888:
        sb = T.make_rgba8888(w, h)
        sdr = A.raw_image(A.FMT_RGBA8888, A.CG_P3, A.CT_SRGB, A.CR_FULL, w, h, [sb], [w])
        keep.append(sb)
    return hdr, sdr, keep


def encode(lib, hdr, sdr, effects, scale=4, compressed_sdr=None, rearm=0):
    enc = C.c_void_p(lib.uhdr_create_encoder())
    try:
        assert lib.uhdr_enc_set_raw_image(enc, C.byref(hdr), A.HDR_IMG).error_code == OK
        if sdr is not None:
            assert lib.uhdr_enc_set_raw_image(enc, C.byref(sdr), A.SDR_IMG).error_code == OK
        if compressed_sdr is not None:
            jb = np.frombuffer(compressed_sdr, np.uint8).copy()
            ci = A.CompressedImage(jb.ctypes.data, len(jb), len(jb), A.CG_BT709, -1, -1)
            assert lib.uhdr_enc_set_compressed_image(enc, C.byref(ci), A.SDR_IMG).error_code == OK
        assert lib.uhdr_enc_set_gainmap_scale_factor(enc, scale).error_code == OK
        for e in effects:
            assert add(lib, enc, e) == OK
        outs = []
        for it in range(1 + rearm):
            if it:
                assert lib.uhdr_b200_enc_rearm(enc) == 0
            rc = lib.uhdr_encode(enc).error_code
            if rc != OK:
                assert not lib.uhdr_get_encoded_stream(enc)
                return rc, None
            o = lib.uhdr_get_encoded_stream(enc).contents
            outs.append(C.string_at(o.data, o.data_sz))
        assert all(x == outs[0] for x in outs)
        return rc, outs[0]
    finally:
        lib.uhdr_release_encoder(enc)


def same_encode(libs, hdr, sdr, effects, **kw):
    got, want = encode(libs[0], hdr, sdr, effects, **kw), encode(libs[1], hdr, sdr, effects, **{k: v for k, v in kw.items() if k != "rearm"})
    assert got[0] == want[0], (effects, got[0], want[0])
    assert got[1] == want[1], (effects, None if got[1] is None else len(got[1]), None if want[1] is None else len(want[1]))
    return want[0]


ENCODE_CHAINS = [
    [("mirror", MH)], [("mirror", MV)], [("rotate", 90)], [("rotate", 180)], [("rotate", 270)],
    [("crop", 6, 206, 10, 150)], [("crop", 7, 201, 3, 151)],   # odd origin, even size: chroma from left / 2
    [("resize", 130, 94)], [("resize", 402, 300)],
    [("crop", 2, 300, 4, 200), ("rotate", 270), ("resize", 100, 140), ("mirror", MH)],
    [("rotate", 90)] * 4, [("crop", -10, 9999, -10, 9999)],
    [("crop", 100, 102, 50, 52)],                              # 2 x 2: the smallest P010 / 4:2:0 result
]
ODD = [[("crop", 0, 33, 0, 20)], [("crop", 0, 32, 0, 21)], [("resize", 33, 20)], [("resize", 32, 21)],
       [("crop", 5, 6, 9, 10)], [("crop", 0, 3, 0, 5)], [("crop", 0, 7, 0, 7)], [("resize", 1, 1)],
       [("rotate", 90), ("crop", 3, 12, 1, 10), ("resize", 5, 3)], [("crop", 0, 9, 0, 9)]]
ERRORS = [[("crop", 50, 50, 0, 10)], [("crop", 0, 10, 300, 400)], [("resize", 0, 8)], [("resize", 8194, 8)],
          [("resize", 8, -1)]]
PAIRS = [(A.FMT_P010, A.FMT_YUV420), (A.FMT_P010, A.FMT_RGBA8888), (A.FMT_P010, None), (A.FMT_RGBA1010102, A.FMT_YUV420),
         (A.FMT_RGBA1010102, A.FMT_RGBA8888), (A.FMT_RGBA1010102, None), (A.FMT_RGBAF16, A.FMT_RGBA8888),
         (A.FMT_RGBAF16, None)]


@pytest.mark.parametrize("hdr_fmt,sdr_fmt", PAIRS)
def test_encode_chains(libs, hdr_fmt, sdr_fmt):
    hdr, sdr, keep = _intents(hdr_fmt, sdr_fmt, 320, 240)
    codes = [same_encode(libs, hdr, sdr, chain, scale=(1, 2, 4)[i % 3], rearm=1 if i < 3 else 0)
             for i, chain in enumerate(ENCODE_CHAINS)]
    # noise content at map scale 1 can outgrow uhdr_encode's w * h * 6 byte output buffer: UHDR_CODEC_MEM_ERROR in both
    assert set(codes) <= {OK, 4} and codes.count(OK) >= len(codes) - 2, codes
    subsampled = hdr_fmt == A.FMT_P010 or sdr_fmt == A.FMT_YUV420
    for chain in ODD:   # refused with a 4:2:0 intent, encoded down to 1 x 1 otherwise
        for scale in (1, 4):
            rc = same_encode(libs, hdr, sdr, chain, scale=scale)
            assert (rc == INVALID_PARAM) if subsampled else (rc == OK), (chain, rc)
    for chain in ERRORS:
        assert same_encode(libs, hdr, sdr, chain) == INVALID_PARAM, chain


def test_encode_compressed_intents_refuse_effects(libs):
    hdr, sdr, keep = _intents(A.FMT_P010, A.FMT_YUV420, 320, 240)
    jpg = T.UhdrApi(libs[1]).encode(hdr, sdr)   # a JPEG/R is a JPEG: its primary image serves as the compressed SDR
    for lib in libs:
        assert encode(lib, hdr, sdr, [("rotate", 90)], compressed_sdr=jpg) == (INVALID_OPERATION, None)   # API-2
        assert encode(lib, hdr, None, [("mirror", MH)], compressed_sdr=jpg) == (INVALID_OPERATION, None)  # API-3
        assert encode(lib, hdr, None, [], compressed_sdr=jpg)[0] == OK


def test_encode_one_gather_per_plane(libs):
    lib = libs[0]
    hdr, sdr, keep = _intents(A.FMT_P010, A.FMT_YUV420, 256, 256)
    chain = [("mirror", MH), ("rotate", 90), ("mirror", MV), ("rotate", 270), ("rotate", 180)]
    counts = []
    for effects in ([], chain, []):
        n0 = lib.uhdr_b200_kernel_launches()
        assert encode(lib, hdr, sdr, effects)[0] == OK
        counts.append(lib.uhdr_b200_kernel_launches() - n0)
    assert counts[0] == counts[2] and counts[1] == counts[0] + 5, counts   # P010: Y, UV; 4:2:0: Y, U, V


def test_steady_state_effects_do_not_touch_the_heap(gpu, tmp_path):
    exe = str(tmp_path / "alloc_probe_effects")
    so = T.GPU_SO
    subprocess.run(["gcc", "-O1", "-g", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "tests", "cpp"),
                    os.path.join(ROOT, "tests", "cpp", "alloc_probe_effects.c"), "-o", exe, "-L", os.path.dirname(so),
                    "-l:" + os.path.basename(so), "-Wl,-rpath," + os.path.dirname(so), "-ldl", "-rdynamic"],
                   check=True, capture_output=True)
    r = subprocess.run([exe, "1280", "720"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout, r.stderr[-4000:])
    lines = [l for l in r.stdout.splitlines() if "ours=" in l]
    assert len(lines) == 2 and all("ours=0 " in l for l in lines), r.stdout
