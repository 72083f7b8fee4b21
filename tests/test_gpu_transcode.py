"""uhdr_b200_transcode on the GPU: byte equality at 0 tolerance with the reference composition (transcode_testlib) for
every scale, base sampling choice and EXIF choice, over the library's own files, reference-made files, Pillow streams
with foreign Huffman tables and restart markers, the Apple fixtures, a map with its own ICC profile and bench.py's 8K
frame.  Each case also asserts its route: both scans entropy-decoded on the device, two device entropy-coder plans, and
the 4:2:0 input kernel exactly when a 4:4:4 base is written 4:2:0."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

import transcode_testlib as X
import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A

pytestmark = pytest.mark.gpu

EXIF = b"Exif\x00\x00MM\x00\x2a\x00\x00\x00\x08\x00\x00\x00\x00\x00\x00"
QUALITIES = [(1, 50), (50, 95), (75, 100), (95, 1), (100, 75)]


@pytest.fixture(scope="module")
def ref(oracle_libs):
    if not oracle_libs.ref_is_turbo() or X.turbo_lib() is None:
        pytest.skip("reference build on libjpeg-turbo not available")
    return oracle_libs.Ref().lib


@pytest.fixture(scope="module")
def lib(gpu):
    L = gpu.lib
    A.declare_transcode(L)
    A.declare_scaled_decode(L)
    A.declare_jpeg_encode_stats(L)
    L.uhdr_b200_last_error.restype = C.c_char_p
    L.uhdr_b200_kernel_timing_report.argtypes = [C.c_char_p, C.c_size_t, C.c_int]
    return L


def _own(gpu_lib, w, h, api0=False, **opts):
    api = T.UhdrApi(gpu_lib)
    if api0:
        buf = T.make_rgba1010102(w, h)
        return api.encode(A.raw_image(A.FMT_RGBA1010102, A.CG_P3, A.CT_PQ, A.CR_FULL, w, h, [buf], [w]), **opts)
    hb, sb = T.make_p010(w, h, "smooth"), T.make_yuv420(w, h, "smooth")
    hdr, _k1 = A.p010_image(hb, w, h, A.CG_BT2100, A.CT_HLG, A.CR_LIMITED)
    sdr, _k2 = A.yuv420_image(sb, w, h, A.CG_BT709)
    return api.encode(hdr, sdr, **opts)


@pytest.fixture(scope="module")
def files(ref, lib):
    md = X.metadata()
    out = {
        "own_api1_420_rgbmap": _own(lib, 256, 192),
        "own_api1_graymap_s4": _own(lib, 320, 240, multichannel=0, scale=4),
        "own_api0_444": _own(lib, 264, 136, api0=True, scale=2),
        "ref_api1": T.UhdrApi(ref).encode(*_ref_intents(256, 128), scale=2),
        "p420_gray_ragged": X.api4_file(ref, md, 457, 331, "420", "gray", 1, exif=EXIF),
        "p444_444map_s4": X.api4_file(ref, md, 455, 333, "444", "444", 4, exif=EXIF),
        "p444_tiny": X.api4_file(ref, md, 8, 8, "444", "gray", 1),
        "p444_w63x8": X.api4_file(ref, md, 504, 87, "444", "gray", 4),
        "pgray": X.api4_file(ref, md, 201, 99, "gray", "gray", 1),
        "foreign_tables_restart": X.api4_file(ref, md, 390, 261, "420", "gray", 1, optimize=True,
                                              restart_marker_blocks=5),
        "map_icc_alt_space": X.api4_file(ref, X.metadata(use_base_cg=0), 300, 200, "444", "gray", 2,
                                         map_icc_cg=A.CG_BT2100),
    }
    for name in ("apple_gainmap_new.jpg", "apple_gainmap_old.jpg"):
        out[name] = open(os.path.join(T.ROOT, "tests", "golden", name), "rb").read()
    return out


def _ref_intents(w, h):
    hb, sb = T.make_p010(w, h, "smooth", seed=5), T.make_yuv420(w, h, "smooth", seed=6)
    _ref_intents.keep = (hb, sb)
    hdr, _ = A.p010_image(hb, w, h, A.CG_BT2100, A.CT_PQ, A.CR_LIMITED)
    sdr, _ = A.yuv420_image(sb, w, h, A.CG_P3)
    return hdr, sdr


def _kernel_counts(lib):
    buf = C.create_string_buffer(1 << 16)
    lib.uhdr_b200_kernel_timing_report(buf, len(buf), 1)
    counts = {}
    for line in buf.value.decode().splitlines():
        f = line.split()
        if len(f) >= 2 and f[1].isdigit():
            counts[f[0]] = int(f[1])
    return counts


def _stats(lib):
    e = (C.c_ulonglong * 3)()
    lib.uhdr_b200_entropy_decoder_stats(e)
    _, bpt, _ = A.jpeg_encode_stats(lib)
    return e[0], e[1], sum(bpt)


def _base_is_444(ref, data, k):
    base = X._probe(ref, data)["base_image"]
    _, planes = X.S.harness_decode(base, k, 0)
    return X.planes_format(planes) == A.FMT_YUV444


def _check(ref, lib, data, k, bq, gq, b420, exif):
    want = X.composition(ref, data, k, bq, gq, b420, exif)
    d0, h0, p0 = _stats(lib)
    lib.uhdr_b200_set_kernel_timing(1)
    _kernel_counts(lib)
    try:
        rc, got, _ = X.transcode(lib, data, k, bq, gq, b420, exif)
        kc = _kernel_counts(lib)
    finally:
        lib.uhdr_b200_set_kernel_timing(0)
    if not isinstance(want, bytes):
        assert rc == want[1], (rc, want, lib.uhdr_b200_last_error())
        return None
    assert rc == 0, lib.uhdr_b200_last_error()
    assert got == want
    d1, h1, p1 = _stats(lib)
    assert (d1 - d0, h1 - h0, p1 - p0) == (2, 0, 2)   # both scans on the device, two device entropy-coder plans
    assert kc.get("ycc444_to_420", 0) == (1 if b420 and _base_is_444(ref, data, k) else 0)
    return got


def _settings(name):
    for k in (1, 2, 4, 8):
        for b420 in (0, 1):
            for exif in (0, 1):
                yield k, b420, exif


@pytest.mark.parametrize("name", ["own_api1_420_rgbmap", "own_api1_graymap_s4", "own_api0_444", "ref_api1", "p420_gray_ragged",
                                  "p444_444map_s4", "p444_tiny", "p444_w63x8", "pgray", "foreign_tables_restart",
                                  "map_icc_alt_space", "apple_gainmap_new.jpg", "apple_gainmap_old.jpg"])
def test_equals_composition(ref, lib, files, name):
    data = files[name]
    for i, (k, b420, exif) in enumerate(_settings(name)):
        bq, gq = QUALITIES[i % len(QUALITIES)]
        got = _check(ref, lib, data, k, bq, gq, b420, exif)
        if b420 and got is not None and _base_is_444(ref, data, k):
            # the 4:2:0 route is taken: the file differs from the one that keeps the 4:4:4 base
            rc, keep, _ = X.transcode(lib, data, k, bq, gq, 0, exif)
            assert rc == 0 and keep != got


@pytest.mark.parametrize("layout", ["422", "444_420map"])
def test_full_size_only_samplings(ref, lib, layout):
    """4:2:2 primary and a 3-channel 4:2:0 map: k = 1 re-encodes them as they are; 4:2:2 at k > 1 and a 4:2:2 base
    written 4:2:0 are UHDR_CODEC_UNSUPPORTED_FEATURE, as uhdr_b200_decode_scaled_dev refuses them"""
    md = X.metadata()
    data = X.api4_file(ref, md, 131, 67, "422", "gray", 1, exif=EXIF) if layout == "422" else \
        X.api4_file(ref, md, 129, 65, "444", "420", 1)
    for i, (bq, gq) in enumerate(QUALITIES):
        _check(ref, lib, data, 1, bq, gq, i % 2, 1)
    for k in (2, 4, 8):
        if layout == "422":
            rc, out, _ = X.transcode(lib, data, k, 75, 75)
            assert rc == A.CODEC_UNSUPPORTED and out is None
        else:   # the 4:2:0 map comes out of the scaled decode 4:4:4
            _check(ref, lib, data, k, 75, 60, 1, 0)
    if layout == "422":
        assert X.transcode(lib, data, 1, 75, 75, base_420=1)[0] == A.CODEC_UNSUPPORTED


def test_errors(ref, lib, files):
    data = files["p420_gray_ragged"]
    rc, full, n = X.transcode(lib, data, 2, 75, 75)
    assert rc == 0
    rc, out, need = X.transcode(lib, data, 2, 75, 75, cap=n - 1)
    assert rc == A.CODEC_MEM_ERROR and out is None and need == n
    assert X.transcode(lib, data, 2, 75, 75, cap=n)[1] == full
    # a progressive primary image: refused by the probe, as uhdr_b200_decode_scaled_dev refuses it; nothing written
    import io
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(X.S.image(64, 48, "smooth")).save(b, "JPEG", quality=80, progressive=True)
    gm = X._probe(ref, data)["gainmap_image"]
    prog = X._api4(ref, b.getvalue(), gm, X.metadata(), A.CG_BT709)
    assert isinstance(prog, bytes)
    u = C.c_uint()
    buf = np.frombuffer(prog, np.uint8).copy()
    want = lib.uhdr_b200_scaled_dims(buf.ctypes.data, buf.size, 2, C.byref(u), C.byref(u), C.byref(u), C.byref(u))
    rc, out, _ = X.transcode(lib, prog, 2, 75, 75)
    assert rc == want != 0 and out is None


def _decode_dev(torch, lib, data, k):
    from test_gpu_scaled_decode import ScaledDecode
    d = ScaledDecode(torch, lib, data, k, A.FMT_RGBAF16, A.CT_LINEAR)
    assert d.run(lib) == 0, lib.uhdr_b200_last_error()
    torch.cuda.synchronize()
    return d.pixels()[0]


def test_interleaved_with_decode_and_threads(ref, lib, files):
    import torch
    names = ["own_api1_420_rgbmap", "p444_444map_s4", "foreign_tables_restart", "p420_gray_ragged"]
    want = {n: X.transcode(lib, files[n], 2, 80, 70, 1, 1)[1] for n in names}
    pix = {n: _decode_dev(torch, lib, files[n], 2) for n in names}
    for n in names:   # same thread: decode, transcode, decode
        assert (_decode_dev(torch, lib, files[n], 4) is not None)
        assert X.transcode(lib, files[n], 2, 80, 70, 1, 1)[1] == want[n]
        assert (_decode_dev(torch, lib, files[n], 2) == pix[n]).all()
    errors = []

    def worker(t):
        try:
            for r in range(3):
                n = names[(t + r) % len(names)]
                if X.transcode(lib, files[n], 2, 80, 70, 1, 1)[1] != want[n]:
                    errors.append((t, r, n, "transcode"))
                if not (_decode_dev(torch, lib, files[n], 2) == pix[n]).all():
                    errors.append((t, r, n, "decode"))
        except Exception as e:  # noqa: BLE001
            errors.append((t, repr(e)))
    th = [threading.Thread(target=worker, args=(t,)) for t in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors


@pytest.mark.parametrize("k", [8, 1])
def test_bench_8k_file(ref, lib, k):
    import bench
    p010, yuv = bench.make_frame(bench.W8K, bench.H8K, 0)
    hdr, sdr, _keep = bench.frame_descs(p010, yuv, bench.W8K, bench.H8K)
    data = T.UhdrApi(lib).encode(hdr, sdr)
    _check(ref, lib, data, k, 75, 75, 1, 1)
