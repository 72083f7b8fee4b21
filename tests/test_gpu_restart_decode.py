"""Restart-interval JPEG (DRI marker, RSTn markers in the entropy-coded data) on the device entropy
decoder: planes equal to the host decoder's and the CPU checker's across layouts, sizes, intervals,
qualities and content; whole JPEG/R files (Apple's gain-map photos, an API-4 assembly, an API-3
encode) equal to the reference's; irregular marker sequences handed to the host decoder with the
same result; and no heap calls in steady state."""
import os
import subprocess

import numpy as np
import pytest

import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A
from test_api4_cpu import _api4
from test_gpu_huffdec import _decode, _stats
from test_gpu_jpeg_api import _frames
from test_oracle_restart_cpu import image, pil_jpeg
from test_xmp_cpu import _vals

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
APPLE = ["apple_gainmap_new.jpg", "apple_gainmap_old.jpg"]
MCU = {"gray": (8, 8), "444": (8, 8), "422": (16, 8), "420": (16, 16)}


def _planes(out, buf, ncomp, widths, heights):
    """the decoded component planes of a mode-0 uhdr_b200_jpeg_decode, cropped to each component's size"""
    res = []
    for k in range(ncomp):
        off = out.planes[k] - buf.ctypes.data
        s = out.stride[k]
        res.append(buf[off:off + s * heights[k]].reshape(heights[k], s)[:, :widths[k]])
    return res


def _both(lib, data, w, h):
    """mode 0 decode with the host decoder, then with the device decoder; -> (rc, buf) pairs and stats delta"""
    prev = lib.uhdr_b200_set_entropy_decoder(1)
    try:
        rh, oh, bh = _decode(lib, data, 0, w, h)
        s0 = _stats(lib)
        lib.uhdr_b200_set_entropy_decoder(2)
        rd, od, bd = _decode(lib, data, 0, w, h)
        s1 = _stats(lib)
    finally:
        lib.uhdr_b200_set_entropy_decoder(prev)
    return (rh, oh, bh), (rd, od, bd), [b - a for a, b in zip(s0, s1)]


@pytest.fixture(scope="module")
def lib(gpu):
    gpu.lib.uhdr_b200_entropy_decoder_stats.restype = None
    return gpu.lib


@pytest.mark.parametrize("w,h", [(72, 34), (1000, 562), (1280, 720), (3840, 2160)])
@pytest.mark.parametrize("layout", ["gray", "420", "422", "444"])
def test_restart_streams_decode_on_device(lib, oracle_libs, layout, w, h):
    o = oracle_libs.Oracle().lib
    mw, mh = MCU[layout]
    per_row = -(-w // mw)
    total = per_row * -(-h // mh)
    intervals = [1, 3, 24, per_row, min(total + 1, 65535)]
    combos = [(100, "noise"), (20, "smooth")]
    if w * h <= 1280 * 720:
        combos += [(100, "smooth"), (20, "noise")]
    for q, kind in combos:
        a = image(w, h, kind, seed=w + h + q)
        for ri in intervals:
            data = pil_jpeg(a, q, layout, restart_marker_blocks=ri)
            (rh, oh, bh), (rd, od, bd), ds = _both(lib, data, w, h)
            case = (layout, w, h, q, kind, ri)
            assert rh == 0 and rd == 0, case
            assert ds[0] == 1 and ds[1] == 0, ("device decoder did not run", case, ds)
            assert (bd == bh).all(), (case, int((bd != bh).sum()))
            hd, ref = T.oracle_decode(o, data)
            f = hd.frame
            widths = [f.comp[c].width for c in range(f.ncomp)]
            heights = [f.comp[c].height for c in range(f.ncomp)]
            for c, (p, r) in enumerate(zip(_planes(od, bd, f.ncomp, widths, heights), ref)):
                assert (p == r[:heights[c], :widths[c]]).all(), (case, c)


OUTPUTS = [(A.FMT_RGBAF16, A.CT_LINEAR), (A.FMT_RGBA1010102, A.CT_HLG), (A.FMT_RGBA1010102, A.CT_PQ),
           (A.FMT_RGBA8888, A.CT_SRGB)]


def _same_decodes(lib, ref_lib, data, xmp=False):
    mine, ref = T.UhdrApi(lib), T.UhdrApi(ref_lib)
    for fmt, ct in OUTPUTS:
        s0 = _stats(lib)
        pa, ga, ma, cga = mine.decode(data, fmt, ct)
        s1 = _stats(lib)
        assert s1[0] == s0[0] + 2 and s1[1] == s0[1], ("both scans must decode on the device", fmt, ct, s0, s1)
        pb, gb, mb, cgb = ref.decode(data, fmt, ct)
        # the reference never initialises use_base_cg on its XMP (Apple) branch: compare the other fields there
        assert (_vals(ma, False) == _vals(mb, False) if xmp else T.md_equal(ma, mb)) and cga == cgb, (fmt, ct)
        assert (ga == gb).all(), (fmt, ct)
        assert (pa == pb).all(), (fmt, ct, int((pa != pb).sum()))


@pytest.mark.parametrize("name", APPLE)
def test_apple_gainmap_files_decode_on_device(lib, oracle_libs, name):
    if not oracle_libs.have_ref():
        pytest.skip("reference build not available")
    data = open(os.path.join(GOLDEN, name), "rb").read()
    assert data.count(b"\xff\xdd") == 2   # a DRI marker in the primary image and in the gain map
    _same_decodes(lib, oracle_libs.Ref().lib, data, xmp=True)


def _dri_jpegr(lib):
    """a JPEG/R assembled (API-4) from a DRI base image (4:2:0, Ri = 24 MCUs) and a DRI gain map (Ri = one MCU row)"""
    w, h = 1000, 562
    md = A.GainmapMetadata()
    for i in range(3):
        md.max_content_boost[i], md.min_content_boost[i], md.gamma[i] = 4.0, 1.0, 1.0
        md.offset_sdr[i] = md.offset_hdr[i] = 1.0 / 64
    md.hdr_capacity_min, md.hdr_capacity_max, md.use_base_cg = 1.0, 4.0, 1
    a = image(w, h, "smooth", seed=11)
    base = pil_jpeg(a, 90, "420", restart_marker_blocks=24)
    gm = pil_jpeg(a[::2, ::2], 90, "gray", restart_marker_rows=1)
    data = _api4(lib, base, gm, md, A.CG_BT709)
    assert isinstance(data, bytes), data
    return data, (base, gm, md)


def test_api4_file_with_restart_intervals(lib, oracle_libs):
    if not oracle_libs.have_ref():
        pytest.skip("reference build not available")
    ref_lib = oracle_libs.Ref().lib
    data, (base, gm, md) = _dri_jpegr(lib)
    assert data == _api4(ref_lib, base, gm, md, A.CG_BT709)
    _same_decodes(lib, ref_lib, data)


def test_api3_with_restart_interval_sdr_intent(lib, oracle_libs):
    """API-3 (raw hdr + compressed sdr): the DRI sdr JPEG is decoded on the device; the file equals the reference's"""
    if not oracle_libs.have_ref():
        pytest.skip("reference build not available")
    w, h = 648, 364
    hdr, _sdr, keep = _frames(w, h, "smooth")
    jpg = pil_jpeg(image(w, h, "noise", seed=5), 90, "420", restart_marker_blocks=24)
    s0 = _stats(lib)
    a = T.UhdrApi(lib).encode_with_compressed_sdr(hdr, jpg, None, A.CG_BT709)
    s1 = _stats(lib)
    b = T.UhdrApi(oracle_libs.Ref().lib).encode_with_compressed_sdr(hdr, jpg, None, A.CG_BT709)
    assert isinstance(a, bytes) and isinstance(b, bytes), (a, b)
    assert a == b
    assert s1[0] >= s0[0] + 1 and s1[1] == s0[1], (s0, s1)


def _scan(data):
    """-> (offset of the entropy-coded data, offsets of its RSTn markers)"""
    s = data.index(b"\xff\xda")
    s += 2 + ((data[s + 2] << 8) | data[s + 3])
    return s, [i for i in range(s, len(data) - 1) if data[i] == 0xFF and 0xD0 <= data[i + 1] <= 0xD7]


def _code_positions(data, lo, hi):
    """offsets in [lo, hi) whose byte may be replaced, or before which bytes may be cut or inserted, without
    touching the marker / stuffing structure"""
    return [i for i in range(lo, hi) if data[i] != 0xFF and data[i - 1] != 0xFF]


def test_irregular_restart_streams_agree_with_host_decoder(lib):
    w, h = 320, 240
    good = pil_jpeg(image(w, h, "noise", seed=3), 90, "420", restart_marker_blocks=3)
    start, rst = _scan(good)
    assert len(rst) == -(-(20 * 15) // 3) - 1
    rs = np.random.RandomState(17)
    m = rst[5]
    dri = good.index(b"\xff\xdd")
    ins = _code_positions(good, rst[7] - 40, rst[7])[0]
    cut = _code_positions(good, m - 16, m - 8)[0]
    cases = {  # name -> (stream, whether the device must decline it)
        "deleted_rst": (good[:m] + good[m + 2:], True),
        "renumbered_rst": (good[:m + 1] + bytes([0xD0 + (good[m + 1] - 0xD0 + 3) % 8]) + good[m + 2:], True),
        "extra_rst": (good[:ins] + b"\xff" + bytes([good[rst[7] + 1]]) + good[ins:], True),
        "rst_without_dri": (good[:dri] + good[dri + 6:], True),
        "other_marker_in_scan": (good[:ins] + b"\xff\xc8" + good[ins:], True),
        "truncated_interval": (good[:cut] + good[m:], False),
        "truncated_file": (good[:rst[40]], False),
    }
    junk = bytearray(good)
    for i in _code_positions(good, rst[8] + 2, rst[9])[:24:3]:
        junk[i] = int(rs.randint(0, 255))
    cases["junk_in_interval"] = (bytes(junk), False)
    for t in range(24):
        bad = bytearray(good)
        pos = _code_positions(good, start + 1, len(good) - 2)
        for _ in range(1 + t % 3):
            bad[pos[int(rs.randint(0, len(pos)))]] = int(rs.randint(0, 255)) & 0xFE   # never 0xFF
        cases["flip_%d" % t] = (bytes(bad), False)
    for name, (data, declines) in cases.items():
        (rh, oh, bh), (rd, od, bd), ds = _both(lib, data, w, h)
        assert rh == rd, (name, rh, rd)
        if rh == 0:
            assert (bh == bd).all(), name
        if declines:
            assert ds[0] == 0 and ds[1] == 1, (name, ds)


def test_restart_decode_steady_state_does_not_touch_the_heap(lib, tmp_path):
    exe = str(tmp_path / "alloc_probe_decode")
    so = T.GPU_SO
    cmd = ["gcc", "-O1", "-g", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "alloc_probe_decode.c"),
           "-o", exe, "-L", os.path.dirname(so), "-l:" + os.path.basename(so), "-Wl,-rpath," + os.path.dirname(so), "-ldl",
           "-rdynamic"]
    subprocess.run(cmd, check=True, capture_output=True)
    # Apple's files are left out: their XMP metadata parse allocates, entropy decoding or not
    path = str(tmp_path / "dri_jpegr.jpg")
    with open(path, "wb") as f:
        f.write(_dri_jpegr(lib)[0])
    r = subprocess.run([exe, path], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout, r.stderr[-4000:])
    assert "ours=0 " in r.stdout and "device_scans=6 handed_back=0" in r.stdout, r.stdout
