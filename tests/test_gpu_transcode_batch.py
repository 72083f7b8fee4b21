"""uhdr_b200_transcode_batch on the GPU, at 0 tolerance: every item of a mixed batch equals uhdr_b200_transcode of that
file alone (bytes, out_size, status) for every k x base_420 x keep_exif at two quality pairs, and the reference
composition (transcode_testlib) for one setting per file; the route (one staging, block-stage and entropy-coding launch
per group, launch counts that do not grow with the batch); per-item errors that write nothing; a scan handed back to
the host decoder; groups; 300 small files; interleaving with other calls; two threads; the heap probe."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

import transcode_testlib as X
import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A
from test_gpu_transcode import EXIF, _kernel_counts, _own, _ref_intents

pytestmark = pytest.mark.gpu

QUALITY_PAIRS = [(75, 60), (95, 100)]


@pytest.fixture(scope="module")
def ref(oracle_libs):
    if not oracle_libs.ref_is_turbo() or X.turbo_lib() is None:
        pytest.skip("reference build on libjpeg-turbo not available")
    return oracle_libs.Ref().lib


@pytest.fixture(scope="module")
def lib(gpu):
    L = gpu.lib
    A.declare_transcode(L)
    A.declare_transcode_batch(L)
    A.declare_scaled_decode(L)
    L.uhdr_b200_last_error.restype = C.c_char_p
    L.uhdr_b200_kernel_launches.restype = C.c_ulonglong
    L.uhdr_b200_kernel_timing_report.argtypes = [C.c_char_p, C.c_size_t, C.c_int]
    L.uhdr_b200_entropy_decoder_stats.argtypes = [C.POINTER(C.c_ulonglong)]
    L.uhdr_b200_entropy_decoder_stats.restype = None
    return L


@pytest.fixture(scope="module")
def corpus(ref, lib):
    """the kinds of file test_gpu_transcode covers, in one list"""
    md = X.metadata()
    out = {
        "own_api1_420_rgbmap": _own(lib, 256, 192),
        "own_api1_graymap_s4": _own(lib, 320, 240, multichannel=0, scale=4),
        "own_api0_444": _own(lib, 264, 136, api0=True, scale=2),
        "ref_api1": T.UhdrApi(ref).encode(*_ref_intents(256, 128), scale=2),
        "p420_gray_ragged": X.api4_file(ref, md, 457, 331, "420", "gray", 1, exif=EXIF),
        "p444_444map_s4": X.api4_file(ref, md, 455, 333, "444", "444", 4, exif=EXIF),
        "p420_420map_s2": X.api4_file(ref, md, 203, 117, "420", "420", 2),
        "p444_tiny": X.api4_file(ref, md, 8, 8, "444", "gray", 1),
        "p420_tiny": X.api4_file(ref, md, 8, 8, "420", "444", 1),
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


def batch(lib, datas, k, bq, gq, b420=0, exif=0, caps=None):
    """uhdr_b200_transcode_batch -> (rc, [(status, bytes or None, out_size)]); failing items' buffers are checked
    untouched"""
    n = len(datas)
    cfg = A.TranscodeConfig(k, bq, gq, b420, exif)
    srcs = [np.frombuffer(d, np.uint8).copy() for d in datas]
    caps = caps or [len(d) * 2 + (1 << 20) for d in datas]
    outs = [np.full(max(c, 1), 0xA5, np.uint8) for c in caps]
    items = (A.TranscodeItem * n)()
    for i in range(n):
        items[i] = A.TranscodeItem(srcs[i].ctypes.data, srcs[i].size, outs[i].ctypes.data, caps[i], 0, -1)
    rc = lib.uhdr_b200_transcode_batch(items, n, C.byref(cfg))
    res = []
    for i in range(n):
        st, m = items[i].status, items[i].out_size
        if st:
            assert (outs[i] == 0xA5).all(), ("a failing item wrote into out", i)
            res.append((st, None, m))
        else:
            res.append((0, bytes(outs[i][:m]), m))
    return rc, res


def singles(lib, datas, k, bq, gq, b420=0, exif=0, caps=None):
    caps = caps or [None] * len(datas)
    return [X.transcode(lib, d, k, bq, gq, b420, exif, cap=c) for d, c in zip(datas, caps)]


def _dec_stats(lib):
    e = (C.c_ulonglong * 3)()
    lib.uhdr_b200_entropy_decoder_stats(e)
    return e[0], e[1]


def _check_batch(lib, datas, k, bq, gq, b420=0, exif=0, caps=None):
    want = singles(lib, datas, k, bq, gq, b420, exif, caps)
    rc, got = batch(lib, datas, k, bq, gq, b420, exif, caps)
    assert got == [tuple(w) for w in want], [(i, g[0], w[0], g[2], w[2]) for i, (g, w) in enumerate(zip(got, want))
                                             if tuple(w) != g]
    first = next((i for i, g in enumerate(got) if g[0]), None)
    assert rc == (0 if first is None else got[first][0])
    if first is not None:
        assert lib.uhdr_b200_last_error().startswith(b"item %d: " % first), lib.uhdr_b200_last_error()
    return got


def test_equals_single_calls(lib, corpus):
    datas = list(corpus.values())
    for k in (1, 2, 4, 8):
        for b420 in (0, 1):
            for exif in (0, 1):
                for bq, gq in QUALITY_PAIRS:
                    got = _check_batch(lib, datas, k, bq, gq, b420, exif)
                    assert all(g[0] == 0 for g in got), (k, b420, exif, [g[0] for g in got])


def test_equals_the_reference_composition(ref, lib, corpus):
    names = list(corpus)
    settings = [(k, b420) for k in (1, 2, 4, 8) for b420 in (0, 1)]
    for r in range(2):   # every file at two of the eight k x base_420 settings
        per = {}
        for i, name in enumerate(names):
            per.setdefault(settings[(i + 3 * r) % len(settings)], []).append(name)
        for (k, b420), ns in per.items():
            rc, got = batch(lib, [corpus[n] for n in ns], k, 80, 70, b420, 1)
            assert rc == 0, lib.uhdr_b200_last_error()
            for n, g in zip(ns, got):
                want = X.composition(ref, corpus[n], k, 80, 70, b420, 1)
                assert g[1] == want, (n, k, b420)


def test_route_one_launch_per_stage_and_counts_that_do_not_grow(lib, corpus):
    data = corpus["p420_gray_ragged"]
    launches = []
    for n in (1, 4, 32):
        d0, h0 = _dec_stats(lib)
        b0 = A.jpeg_encode_batch_stats(lib)
        lib.uhdr_b200_set_kernel_timing(1)
        _kernel_counts(lib)
        try:
            l0 = lib.uhdr_b200_kernel_launches()
            rc, got = batch(lib, [data] * n, 2, 75, 75, 1, 1)
            launches.append(lib.uhdr_b200_kernel_launches() - l0)
            kc = _kernel_counts(lib)
        finally:
            lib.uhdr_b200_set_kernel_timing(0)
        assert rc == 0 and len(set(g[1] for g in got)) == 1
        d1, h1 = _dec_stats(lib)
        b1 = A.jpeg_encode_batch_stats(lib)
        assert (d1 - d0, h1 - h0) == (2 * n, 0)              # every scan entropy-decoded on the device
        assert (b1[0] - b0[0], b1[1] - b0[1]) == (1, 2 * n)  # one batched entropy-coder plan for the group
        assert (kc.get("stage_batch"), kc.get("fdct_code_batch"), kc.get("huff_encode_batch"), kc.get("pack_scans")) == \
            (1, 1, 1, 1), kc
        assert "huff_encode" not in kc and "fdct_quant" not in kc and "ycc444_to_420" not in kc, kc
    assert launches[0] == launches[1] == launches[2], launches


def _progressive(ref, good):
    import io
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(X.S.image(64, 48, "smooth")).save(b, "JPEG", quality=80, progressive=True)
    gm = X._probe(ref, good)["gainmap_image"]
    out = X._api4(ref, b.getvalue(), gm, X.metadata(), A.CG_BT709)
    assert isinstance(out, bytes)
    return out


def test_per_item_errors(ref, lib, corpus):
    good = [corpus["own_api1_420_rgbmap"], corpus["p420_gray_ragged"], corpus["p444_444map_s4"], corpus["pgray"]]
    s422 = X.api4_file(ref, X.metadata(), 131, 67, "422", "gray", 1, exif=EXIF)
    prog = _progressive(ref, good[1])
    garbage = b"\xff\xd8\xff\xe0" + bytes(range(200)) + b"\xff\xd9"
    _rc, full, n_ok = X.transcode(lib, good[1], 2, 75, 75, 0, 1)
    datas = [good[0], s422, good[1], prog, good[2], garbage, good[1], good[3]]
    caps = [None, None, n_ok - 1, None, None, None, n_ok, None]
    caps = [c if c is not None else len(d) * 2 + (1 << 20) for c, d in zip(caps, datas)]
    for k, b420 in ((2, 0), (1, 1), (4, 1)):
        got = _check_batch(lib, datas, k, 75, 75, b420, 1, caps)
        st = [g[0] for g in got]
        assert st[1] == A.CODEC_UNSUPPORTED and st[3] != 0 and st[5] != 0 and [st[i] for i in (0, 4, 7)] == [0, 0, 0]
        if (k, b420) == (2, 0):   # the size the caps were made for: one byte short, then exactly enough
            assert st[2] == A.CODEC_MEM_ERROR and got[2][2] == n_ok and got[6][1] == full, (got[2], got[6][0])


def test_scan_handed_back_to_the_host(lib, corpus):
    from test_gpu_decode_batch import flat_file
    flat = flat_file(lib)
    datas = [corpus["own_api1_420_rgbmap"], flat, corpus["p444_444map_s4"]]
    d0, h0 = _dec_stats(lib)
    rc, _got = batch(lib, datas, 1, 75, 75)
    d1, h1 = _dec_stats(lib)
    assert rc == 0 and (d1 - d0, h1 - h0) == (5, 1)   # exactly the flat primary's scan on the host
    _check_batch(lib, datas, 1, 75, 75)
    _check_batch(lib, datas, 2, 60, 90, 1, 1)



def test_host_decoder_switch_applies_to_batches(lib, corpus):
    """uhdr_b200_set_entropy_decoder(1) sends every scan of a batch to the host decoder: the same bytes, sizes and
    codes as the device decoder gives, and the device decoder's counts do not move"""
    garbage = b"\xff\xd8\xff\xe0" + bytes(range(200)) + b"\xff\xd9"
    datas = [corpus["own_api1_420_rgbmap"], corpus["foreign_tables_restart"], garbage, corpus["pgray"],
             corpus["apple_gainmap_new.jpg"]]
    runs = {}
    for mode in (2, 1):
        prev = lib.uhdr_b200_set_entropy_decoder(mode)
        try:
            s0 = _dec_stats(lib)
            rc, got = batch(lib, datas, 2, 75, 60, 1, 1)
            s1 = _dec_stats(lib)
        finally:
            lib.uhdr_b200_set_entropy_decoder(prev)
        runs[mode] = (rc, got, lib.uhdr_b200_last_error(), (s1[0] - s0[0], s1[1] - s0[1]))
    assert [g[0] for g in runs[2][1]] == [0, 0, runs[2][0], 0, 0] and runs[2][0] != 0, runs[2][:3]
    assert runs[1][:3] == runs[2][:3]
    assert runs[2][3][0] > 0 and runs[1][3] == (0, 0), (runs[2][3], runs[1][3])

def test_groups_give_the_same_bytes(lib, corpus, monkeypatch):
    datas = list(corpus.values())
    _rc, whole = batch(lib, datas, 2, 75, 75, 1, 1)
    monkeypatch.setenv("UHDR_B200_BATCH_GROUP_BYTES", str(1 << 20))   # about one file per group
    b0 = A.jpeg_encode_batch_stats(lib)
    rc, grouped = batch(lib, datas, 2, 75, 75, 1, 1)
    b1 = A.jpeg_encode_batch_stats(lib)
    assert rc == 0 and grouped == whole and b1[0] - b0[0] > 3
    monkeypatch.delenv("UHDR_B200_BATCH_GROUP_BYTES")
    import bench
    p010, yuv = bench.make_frame(bench.W8K, bench.H8K, 0)
    hdr, sdr, _keep = bench.frame_descs(p010, yuv, bench.W8K, bench.H8K)
    big = T.UhdrApi(lib).encode(hdr, sdr)
    got = _check_batch(lib, [corpus["p420_gray_ragged"], big, corpus["pgray"], big, corpus["p444_tiny"]], 1, 75, 75, 1, 1)
    assert all(g[0] == 0 for g in got)


def test_three_hundred_small_files(ref, lib):
    md = X.metadata()
    lay = ["420", "444", "gray"]
    datas = [X.api4_file(ref, md, 8 + i % 41, 8 + i % 29, lay[i % 3], lay[(i // 3) % 3], 1 + i % 2, seed=i)
             for i in range(300)]
    got = _check_batch(lib, datas, 2, 80, 70, 1, 1)
    assert all(g[0] == 0 for g in got)


def test_interleaved_with_single_calls_and_decodes(lib, corpus):
    import torch
    from test_gpu_transcode import _decode_dev
    names = ["own_api1_420_rgbmap", "p444_444map_s4", "foreign_tables_restart", "p420_gray_ragged"]
    datas = [corpus[n] for n in names]
    want = singles(lib, datas, 2, 80, 70, 1, 1)
    pix = [_decode_dev(torch, lib, d, 2) for d in datas]
    for r in range(3):
        rc, got = batch(lib, datas, 2, 80, 70, 1, 1)
        assert rc == 0 and got == [tuple(w) for w in want]
        assert X.transcode(lib, datas[r], 2, 80, 70, 1, 1) == want[r]
        assert (_decode_dev(torch, lib, datas[r], 2) == pix[r]).all()


def test_two_threads_batching_at_once(lib, corpus):
    datas = list(corpus.values())
    want = [tuple(w) for w in singles(lib, datas, 4, 80, 70, 1, 0)]
    errors = []

    def run(t):
        try:
            for _rep in range(3):
                rc, got = batch(lib, datas[t::2] + datas, 4, 80, 70, 1, 0)
                if rc != 0 or got != want[t::2] + want:
                    errors.append((t, rc))
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    th = [threading.Thread(target=run, args=(t,)) for t in range(2)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors


def test_steady_state_does_not_touch_the_heap(lib, corpus, tmp_path):
    import subprocess
    exe = str(tmp_path / "alloc_probe_transcode_batch")
    so = T.GPU_SO
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    cmd = ["gcc", "-O1", "-g", "-I", os.path.join(T.ROOT, "include"), "-I", os.path.join(cuda, "include"),
           os.path.join(T.ROOT, "tests", "cpp", "alloc_probe_transcode_batch.c"), "-o", exe, "-L", os.path.dirname(so),
           "-l:" + os.path.basename(so), "-Wl,-rpath," + os.path.dirname(so), "-L", os.path.join(cuda, "lib64"),
           "-lcudart", "-Wl,-rpath," + os.path.join(cuda, "lib64"), "-ldl", "-rdynamic"]
    subprocess.run(cmd, check=True, capture_output=True)
    path = str(tmp_path / "file.jpg")
    with open(path, "wb") as f:
        f.write(corpus["p444_444map_s4"])
    r = subprocess.run([exe, path], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout, r.stderr[-4000:])
    assert "ours=0 " in r.stdout, r.stdout
