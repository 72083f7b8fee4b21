"""Parity at the geometries the benchmark and the reference's own benchmark use (VERDICT r1, weak #3):
whole files at 3840x2160 on bench.py's frame generator (API-1 and API-0), re-armed encodes of resident
inputs, 7680x4320 uhdr_decode, 1920x1080 / 4080x3072 (benchmark/benchmark_test.cpp:55-72 of the
reference; both have MCU rows / columns that reach past the block grid), config 1 on the reference's
real 720p fixtures, and a 4:2:2 base image through applyGainMap."""
import ctypes as C
import io
import os

import numpy as np
import pytest

import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A

pytestmark = pytest.mark.gpu


def _bench_frame(w, h, idx):
    import bench
    p, y = bench.make_frame(w, h, idx)
    hdr, sdr, keep = bench.frame_descs(p, y, w, h)
    return hdr, sdr, (p, y, keep)


def _need_ref(oracle_libs):
    if not oracle_libs.have_ref():
        pytest.skip("reference build not available")
    return T.UhdrApi(oracle_libs.Ref().lib)


def test_4k_api1_file_and_rearmed_encodes(gpu, oracle_libs):
    """uhdr_encode at the headline geometry == the reference's file; encoding the same resident inputs
    again (uhdr_b200_enc_rearm, what bench.py's `value` arm does) returns the same bytes every time."""
    ref = _need_ref(oracle_libs)
    lib = gpu.lib
    T.UhdrApi(lib)
    hdr, sdr, keep = _bench_frame(3840, 2160, 3)
    want = ref.encode(hdr, sdr)
    enc = C.c_void_p(lib.uhdr_create_encoder())
    try:
        assert lib.uhdr_enc_set_raw_image(enc, C.byref(hdr), A.HDR_IMG).error_code == 0
        assert lib.uhdr_enc_set_raw_image(enc, C.byref(sdr), A.SDR_IMG).error_code == 0
        for it in range(3):
            e = lib.uhdr_encode(enc)
            assert e.error_code == 0, e.detail
            o = lib.uhdr_get_encoded_stream(enc).contents
            got = C.string_at(o.data, o.data_sz)
            assert len(got) == len(want), (it, len(got), len(want))
            assert got == want, it
            assert lib.uhdr_b200_enc_rearm(enc) == 0
    finally:
        lib.uhdr_release_encoder(enc)


def test_4k_api0_file(gpu, oracle_libs):
    ref = _need_ref(oracle_libs)
    mine = T.UhdrApi(gpu.lib)
    hdr, _sdr, keep = _bench_frame(3840, 2160, 5)
    assert mine.encode(hdr, None) == ref.encode(hdr, None)


@pytest.mark.parametrize("w,h", [(1920, 1080), (4080, 3072)])
def test_reference_benchmark_sizes(gpu, oracle_libs, w, h):
    """API-1 and API-0 files at the sizes of the reference's own benchmark.  1080 = 67.5 MCU rows and
    4080 = 255 MCU columns: libjpeg's dummy-block rule and the helper's chroma padding are in play."""
    ref = _need_ref(oracle_libs)
    mine = T.UhdrApi(gpu.lib)
    hdr, sdr, keep = _bench_frame(w, h, 9)
    a, b = mine.encode(hdr, sdr), ref.encode(hdr, sdr)
    assert len(a) == len(b) and a == b
    assert mine.encode(hdr, None, multichannel=0) == ref.encode(hdr, None, multichannel=0)
    pa, ga, ma, cga = mine.decode(b)
    pb, gb, mb, cgb = ref.decode(b)
    assert T.md_equal(ma, mb) and cga == cgb and (ga == gb).all() and (pa == pb).all()


def test_8k_uhdr_decode(gpu, oracle_libs):
    """config 3: uhdr_decode of a 7680x4320 JPEG/R to RGBA half float, device entropy decoder: pixels,
    gain map, metadata and gamut == the reference decoder's."""
    ref = _need_ref(oracle_libs)
    mine = T.UhdrApi(gpu.lib)
    hdr, sdr, keep = _bench_frame(7680, 4320, 7)
    A.declare_jpeg_encode_stats(gpu.lib)
    _, b0, _ = A.jpeg_encode_stats(gpu.lib)
    data = mine.encode(hdr, sdr)
    R, b1, _ = A.jpeg_encode_stats(gpu.lib)
    # the GPU-encoded file itself == the reference's.  Its two scans go through the entropy coder with the blocks per
    # thread of their sizes (4:2:0 base 777600 blocks, 3-channel map 1555200: bpt 4 and 8 at 792 resident CTAs)
    grew = [y - x for x, y in zip(b0, b1)]
    want_grew = [0] * 8
    for n in (777600, 1555200):
        want_grew[min(8, -(-n // (256 * R))) - 1] += 1
    assert grew == want_grew, (R, grew)
    want = ref.encode(hdr, sdr)
    assert len(data) == len(want) and data == want
    st0, st1 = (C.c_ulonglong * 3)(), (C.c_ulonglong * 3)()
    gpu.lib.uhdr_b200_entropy_decoder_stats.restype = None
    gpu.lib.uhdr_b200_entropy_decoder_stats(st0)
    pa, ga, ma, cga = mine.decode(data)
    gpu.lib.uhdr_b200_entropy_decoder_stats(st1)
    assert st1[0] - st0[0] == 2 and st1[1] == st0[1], "both scans must go through the device entropy decoder"
    pb, gb, mb, cgb = ref.decode(data)
    assert T.md_equal(ma, mb) and cga == cgb
    assert (ga == gb).all()
    assert (pa == pb).all(), int((pa != pb).sum())


def test_config1_real_fixtures(gpu, oracle_libs):
    """BASELINE config 1: the reference's own 1280x720 fixtures (copied next to oracle/_ref by its
    Makefile so they travel to the GPU box), ultrahdr_app's defaults: hdr P3 HLG limited, sdr BT.709."""
    ref = _need_ref(oracle_libs)
    mine = T.UhdrApi(gpu.lib)
    d = os.path.join(T.ROOT, "oracle", "_ref", "fixtures")
    pp, yp = os.path.join(d, "raw_p010_image.p010"), os.path.join(d, "raw_yuv420_image.yuv420")
    if not (os.path.exists(pp) and os.path.exists(yp)):
        pytest.skip("720p fixtures not present")
    w, h = 1280, 720
    p = np.fromfile(pp, np.uint16)[:w * h * 3 // 2].copy()
    y = np.fromfile(yp, np.uint8)[:w * h * 3 // 2].copy()
    hdr, k1 = A.p010_image(p, w, h, A.CG_P3, A.CT_HLG, A.CR_LIMITED)
    sdr, k2 = A.yuv420_image(y, w, h, A.CG_BT709)
    a, b = mine.encode(hdr, sdr), ref.encode(hdr, sdr)
    assert a == b
    assert mine.encode(hdr, None) == ref.encode(hdr, None)
    for fmt, ct in ((A.FMT_RGBAF16, A.CT_LINEAR), (A.FMT_RGBA1010102, A.CT_HLG), (A.FMT_RGBA1010102, A.CT_PQ)):
        pa, ga, ma, cga = mine.decode(b, fmt, ct)
        pb, gb, mb, cgb = ref.decode(b, fmt, ct)
        assert T.md_equal(ma, mb) and cga == cgb and (ga == gb).all() and (pa == pb).all(), (fmt, ct)


@pytest.mark.parametrize("subsampling,name", [(1, "4:2:2"), (0, "4:4:4"), (2, "4:2:0")])
def test_apply_on_subsampled_base(gpu, oracle_libs, subsampling, name):
    """applyGainMap with a 4:2:2 (and 4:4:4 / 4:2:0) base image: the base JPEG comes from a real
    libjpeg-turbo (Pillow), the stage result must equal the reference's applyGainMap on the same planes."""
    PIL = pytest.importorskip("PIL.Image")
    if not oracle_libs.have_ref():
        pytest.skip("reference build not available")
    chk = oracle_libs.Ref()
    w, h = 322, 182
    rs = np.random.RandomState(11)
    yy, xx = np.mgrid[0:h, 0:w]
    rgb = np.stack([(xx * 255 // w), (yy * 255 // h), ((xx + yy) % 256)], -1).astype(np.uint8)
    b = io.BytesIO()
    PIL.fromarray(rgb).save(b, "JPEG", quality=92, subsampling=subsampling)
    data = b.getvalue()
    # decode to raw planes with the product (uhdr_b200_jpeg_decode mode 0 = DECODE_TO_YCBCR_CS)
    buf = np.zeros(w * h * 4 + 65536, np.uint8)
    out = A.raw_image(-1, -1, -1, -1, 0, 0, [buf], [0])
    cbuf = (C.c_uint8 * len(data)).from_buffer_copy(data)
    assert gpu.lib.uhdr_b200_jpeg_decode(cbuf, C.c_size_t(len(data)), 0, C.byref(out), C.c_size_t(buf.size)) == 0, T.gpu_err(gpu)
    assert out.fmt == {1: A.FMT_YUV422, 0: A.FMT_YUV444, 2: A.FMT_YUV420}[subsampling]
    out.cg = A.CG_BT709
    out.ct = A.CT_SRGB
    out.range = A.CR_FULL
    gm = rs.randint(0, 256, (h // 2, w // 2, 3)).astype(np.uint8)
    gi = T.gm_image(gm, A.CG_P3)
    md = A.GainmapMetadata()
    for i in range(3):
        md.max_content_boost[i], md.min_content_boost[i], md.gamma[i] = 6.0 + i, 0.8, 1.0
        md.offset_sdr[i] = md.offset_hdr[i] = 1e-7
    md.hdr_capacity_min, md.hdr_capacity_max, md.use_base_cg = 1.0, 6.0, 1
    for ct in (A.CT_LINEAR, A.CT_PQ, A.CT_HLG):
        a = gpu.apply(out, gi, md, ct)
        bb = chk.apply(out, gi, md, ct)
        assert (a == bb).all(), (name, ct, int((a != bb).sum()))
