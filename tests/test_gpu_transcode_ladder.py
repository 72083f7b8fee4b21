"""uhdr_b200_transcode_ladder on the GPU, at 0 tolerance: every rung of several ladders equals uhdr_b200_transcode with
that rung's config alone (bytes, out_size, status) for every file of the batch test's corpus, and the reference
composition for one ladder per file; the route (two scans entropy-decoded, one k_idct<0>, one staging launch, one
block-stage launch per quality pair, launch counts that do not grow with the rungs); IDCT extremes at every size;
per-rung and file-level errors that write nothing; a scan handed back to the host decoder; interleaving with other
calls; two threads; the heap probe."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

import jpeg_decode_cases as D
import jpeg_stream_writer as W
import transcode_testlib as X
import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A
from test_gpu_transcode import EXIF, _kernel_counts
from test_gpu_transcode_batch import _progressive, batch, corpus, ref  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

LADDERS = {
    "all_k": [(k, 80, 70, 0, 0) for k in (1, 2, 4, 8)],
    "k1_two_qualities": [(1, 85, 85, 0, 0), (1, 60, 90, 0, 1), (2, 80, 70, 0, 0), (4, 80, 70, 0, 0), (8, 80, 70, 0, 0)],
    "mixed_420_exif": [(1, 75, 75, 1, 0), (2, 75, 75, 0, 1), (2, 75, 75, 1, 1), (4, 75, 75, 1, 1), (8, 75, 75, 0, 0)],
    "duplicated": [(2, 80, 70, 1, 1), (4, 95, 100, 0, 0), (2, 80, 70, 1, 1)],
}
LADDERS["reversed"] = LADDERS["k1_two_qualities"][::-1]


@pytest.fixture(scope="module")
def lib(gpu):
    L = gpu.lib
    A.declare_transcode(L)
    A.declare_transcode_batch(L)
    A.declare_transcode_ladder(L)
    A.declare_scaled_decode(L)
    L.uhdr_b200_last_error.restype = C.c_char_p
    L.uhdr_b200_kernel_launches.restype = C.c_ulonglong
    L.uhdr_b200_kernel_timing_report.argtypes = [C.c_char_p, C.c_size_t, C.c_int]
    L.uhdr_b200_entropy_decoder_stats.argtypes = [C.POINTER(C.c_ulonglong)]
    L.uhdr_b200_entropy_decoder_stats.restype = None
    return L


def ladder(lib, data, cfgs, caps=None):
    """uhdr_b200_transcode_ladder -> (rc, [(status, bytes or None, out_size)]); failing rungs' buffers are checked
    untouched"""
    n = len(cfgs)
    src = np.frombuffer(data, np.uint8).copy()
    caps = caps or [len(data) * 2 + (1 << 20)] * n
    outs = [np.full(max(c, 1), 0xA5, np.uint8) for c in caps]
    rungs = (A.TranscodeRung * n)()
    for i in range(n):
        rungs[i] = A.TranscodeRung(A.TranscodeConfig(*cfgs[i]), outs[i].ctypes.data, caps[i], 0, -1)
    rc = lib.uhdr_b200_transcode_ladder(src.ctypes.data, src.size, rungs, n)
    res = []
    for i in range(n):
        st, m = rungs[i].status, rungs[i].out_size
        if st:
            assert (outs[i] == 0xA5).all(), ("a failing rung wrote into out", i)
            res.append((st, None, m))
        else:
            res.append((0, bytes(outs[i][:m]), m))
    return rc, res


def singles(lib, data, cfgs, caps=None):
    caps = caps or [None] * len(cfgs)
    return [tuple(X.transcode(lib, data, *c, cap=cap)) for c, cap in zip(cfgs, caps)]


def _check(lib, data, cfgs, caps=None):
    want = singles(lib, data, cfgs, caps)
    rc, got = ladder(lib, data, cfgs, caps)
    assert got == want, [(i, g[0], w[0], g[2], w[2]) for i, (g, w) in enumerate(zip(got, want)) if w != g]
    first = next((i for i, g in enumerate(got) if g[0]), None)
    assert rc == (0 if first is None else got[first][0])
    if first is not None:
        assert lib.uhdr_b200_last_error().startswith(b"rung %d: " % first), lib.uhdr_b200_last_error()
    return got


def _dec_stats(lib):
    e = (C.c_ulonglong * 3)()
    lib.uhdr_b200_entropy_decoder_stats(e)
    return e[0], e[1]


def test_equals_single_calls(lib, corpus):
    for name, data in corpus.items():
        for lname, cfgs in LADDERS.items():
            got = _check(lib, data, cfgs)
            assert all(g[0] == 0 for g in got), (name, lname, [g[0] for g in got])


def test_equals_the_reference_composition(ref, lib, corpus):
    for i, (name, data) in enumerate(corpus.items()):
        cfgs = list(LADDERS.values())[i % len(LADDERS)]
        rc, got = ladder(lib, data, cfgs)
        assert rc == 0, lib.uhdr_b200_last_error()
        for c, g in zip(cfgs, got):
            assert g[1] == X.composition(ref, data, *c), (name, c)


def _route(lib, data, cfgs):
    d0, h0 = _dec_stats(lib)
    lib.uhdr_b200_set_kernel_timing(1)
    _kernel_counts(lib)
    try:
        l0 = lib.uhdr_b200_kernel_launches()
        rc, got = ladder(lib, data, cfgs)
        launches = lib.uhdr_b200_kernel_launches() - l0
        kc = _kernel_counts(lib)
    finally:
        lib.uhdr_b200_set_kernel_timing(0)
    assert rc == 0, lib.uhdr_b200_last_error()
    d1, h1 = _dec_stats(lib)
    assert (d1 - d0, h1 - h0) == (2, 0)   # each scan entropy-decoded once, on the device
    assert not [n for n in kc if n.startswith("idct_dequant") or n.startswith("idct_scaled")], kc
    return kc, launches


def test_route(lib, corpus):
    data = corpus["p420_gray_ragged"]
    for cfgs in LADDERS.values():
        kc, _ = _route(lib, data, cfgs)
        pairs = len(set((c[1], c[2]) for c in cfgs))
        assert (kc.get("idct_multi"), kc.get("stage_batch"), kc.get("fdct_code_batch"), kc.get("huff_encode_batch"),
                kc.get("pack_scans")) == (1, 1, pairs, 1, 1), kc
    launches = [_route(lib, data, [(k, 75, 75, 1, 1) for k in ks])[1] for ks in ((2,), (2, 4), (1, 2, 4, 8))]
    assert launches[0] == launches[1] == launches[2], launches


def _extreme_file(lib, layout, w, h, q, seed):
    """a writer-made primary whose blocks saturate 0 / 255 at S = 8 and 4 (single coefficients at the category
    limits, checkerboards) and whose DC wraps modulo 1024 at S = 1, with a Pillow gray map, wrapped by API-4"""
    samp = {"gray": D.GRAY, "444": D.S444, "420": D.S420}[layout]
    b = D.idct_blocks(q)
    dc = np.zeros((8, 64), np.int64)
    dc[:, 0] = [1023, -1023, 700, -700, 300, -300, 129, -129]   # x q up to 255: (dc q + 4) >> 3 past +-512
    b = np.concatenate([dc, b])
    fr = W.Frame(w, h, samp)
    co = [np.resize(np.roll(b, c * 17 + seed, axis=0), (fr.blocks(c), 64)) for c in range(fr.ncomp)]
    sel = [(0, 0)] + [(1, 1)] * (fr.ncomp - 1)
    st = W.write_jpeg(w, h, samp, co, W.optimal_tables(fr, co, sel), sel, qt={0: q, 1: q})
    gm = X.pil_bytes(X.S.image(max(1, w // 2), max(1, h // 2), "smooth", seed), "gray", 85)
    out = X._api4(lib, st.data, gm, X.metadata(), A.CG_BT709)
    assert isinstance(out, bytes), out
    return out


def test_idct_extremes(lib):
    cfgs = [(1, 75, 75, 0, 0), (2, 75, 75, 0, 0), (4, 90, 60, 1, 0), (8, 75, 75, 0, 0), (1, 75, 75, 1, 0)]
    for i, (layout, w, h) in enumerate((("444", 317, 123), ("420", 325, 251), ("gray", 301, 117), ("420", 9, 7))):
        for qn, q in (("q1", [1] * 64), ("q255", [255] * 64), ("ramp", list(range(1, 65)))):
            data = _extreme_file(lib, layout, w, h, q, i)
            got = _check(lib, data, cfgs)
            assert all(g[0] == 0 for g in got), (layout, qn, [g[0] for g in got])


def test_per_rung_and_file_errors(ref, lib, corpus):
    s422 = X.api4_file(ref, X.metadata(), 131, 67, "422", "gray", 1, exif=EXIF)
    got = _check(lib, s422, [(1, 75, 75, 0, 0), (2, 75, 75, 0, 0), (1, 75, 75, 1, 0)])
    assert [g[0] for g in got] == [0, A.CODEC_UNSUPPORTED, A.CODEC_UNSUPPORTED]
    data = corpus["p420_gray_ragged"]
    _rc, full, n_ok = X.transcode(lib, data, 2, 75, 75, 0, 1)
    cfgs = [(2, 75, 75, 0, 1), (4, 75, 75, 1, 1), (2, 75, 75, 0, 1)]
    got = _check(lib, data, cfgs, [n_ok - 1, len(data) * 2, n_ok])
    assert got[0] == (A.CODEC_MEM_ERROR, None, n_ok) and got[1][0] == 0 and got[2][1] == full
    garbage = b"\xff\xd8\xff\xe0" + bytes(range(200)) + b"\xff\xd9"
    for bad in (garbage, _progressive(ref, data)):
        got = _check(lib, bad, [(1, 75, 75, 0, 0), (3, 75, 75, 0, 0), (4, 80, 70, 1, 1), (2, 75, 75, 0, 0)])
        st = [g[0] for g in got]
        assert st[1] == A.CODEC_INVALID_PARAM and st[0] == st[2] == st[3] != 0, st


def test_scan_handed_back_to_the_host(lib, corpus):
    from test_gpu_decode_batch import flat_file
    flat = flat_file(lib)
    d0, h0 = _dec_stats(lib)
    rc, _got = ladder(lib, flat, LADDERS["all_k"])
    d1, h1 = _dec_stats(lib)
    assert rc == 0 and (d1 - d0, h1 - h0) == (1, 1)   # the flat primary's scan on the host, the map's on the device
    for cfgs in LADDERS.values():
        _check(lib, flat, cfgs)


def test_interleaved_with_other_calls(lib, corpus):
    import torch
    from test_gpu_transcode import _decode_dev
    names = ["own_api1_420_rgbmap", "p444_444map_s4", "foreign_tables_restart", "p420_gray_ragged"]
    datas = [corpus[n] for n in names]
    cfgs = LADDERS["mixed_420_exif"]
    want = [singles(lib, d, cfgs) for d in datas]
    bwant = [tuple(X.transcode(lib, d, 2, 80, 70, 1, 1)) for d in datas]
    pix = [_decode_dev(torch, lib, d, 2) for d in datas]
    for r in range(3):
        for i, d in enumerate(datas):
            rc, got = ladder(lib, d, cfgs)
            assert rc == 0 and got == want[i]
        assert X.transcode(lib, datas[r], *cfgs[r]) == want[r][r]
        rc, got = batch(lib, datas, 2, 80, 70, 1, 1)
        assert rc == 0 and got == bwant
        assert (_decode_dev(torch, lib, datas[r], 2) == pix[r]).all()


def test_two_threads_at_once(lib, corpus):
    datas = list(corpus.values())
    cfgs = LADDERS["k1_two_qualities"]
    want = [singles(lib, d, cfgs) for d in datas]
    errors = []

    def run(t):
        try:
            for _rep in range(2):
                for i in (range(len(datas)) if t == 0 else reversed(range(len(datas)))):
                    rc, got = ladder(lib, datas[i], cfgs)
                    if rc != 0 or got != want[i]:
                        errors.append((t, i, rc))
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
    exe = str(tmp_path / "alloc_probe_transcode_ladder")
    so = T.GPU_SO
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    cmd = ["gcc", "-O1", "-g", "-I", os.path.join(T.ROOT, "include"), "-I", os.path.join(cuda, "include"),
           os.path.join(T.ROOT, "tests", "cpp", "alloc_probe_transcode_ladder.c"), "-o", exe, "-L", os.path.dirname(so),
           "-l:" + os.path.basename(so), "-Wl,-rpath," + os.path.dirname(so), "-L", os.path.join(cuda, "lib64"),
           "-lcudart", "-Wl,-rpath," + os.path.join(cuda, "lib64"), "-ldl", "-rdynamic"]
    subprocess.run(cmd, check=True, capture_output=True)
    path = str(tmp_path / "file.jpg")
    with open(path, "wb") as f:
        f.write(corpus["p444_444map_s4"])
    r = subprocess.run([exe, path], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout, r.stderr[-4000:])
    assert "ours=0 " in r.stdout, r.stdout
