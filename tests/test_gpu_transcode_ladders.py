"""uhdr_b200_transcode_ladders on the GPU, at 0 tolerance: every file of the batch test's corpus, each with its own ladder,
equals uhdr_b200_transcode_ladder on that file alone (bytes, out_size, every status and the file's status), and a subset
of rungs equals the reference composition; the route of one group (two scans per file entropy-decoded on the device, one
k_idct<0>, one staging launch, one block-stage launch per quality pair, one entropy coding, launch counts that do not
grow with the files); file, rung and call errors in one call; groups formed on scratch and on quality pairs; the host
entropy decoder; interleaving with the other calls; two threads; the heap probe."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

import transcode_testlib as X
import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A
from test_gpu_transcode import EXIF, _kernel_counts
from test_gpu_transcode_batch import _progressive, batch, corpus, ref  # noqa: F401  (fixtures)
from test_gpu_transcode_ladder import LADDERS, ladder

pytestmark = pytest.mark.gpu

LADDER_LIST = list(LADDERS.values())


@pytest.fixture(scope="module")
def lib(gpu):
    L = gpu.lib
    A.declare_transcode(L)
    A.declare_transcode_batch(L)
    A.declare_transcode_ladder(L)
    A.declare_transcode_ladders(L)
    A.declare_scaled_decode(L)
    L.uhdr_b200_last_error.restype = C.c_char_p
    L.uhdr_b200_kernel_launches.restype = C.c_ulonglong
    L.uhdr_b200_kernel_timing_report.argtypes = [C.c_char_p, C.c_size_t, C.c_int]
    L.uhdr_b200_entropy_decoder_stats.argtypes = [C.POINTER(C.c_ulonglong)]
    L.uhdr_b200_entropy_decoder_stats.restype = None
    return L


def ladders(lib, entries):
    """uhdr_b200_transcode_ladders over entries [(data or None, cfgs or None, caps or None, n or None)] -> (rc,
    [(file status, [(status, bytes or None, out_size)] or None)]); a file's rungs are None when its status is an argument
    error of the file, and its buffers are then checked untouched, as those of every failing rung"""
    keep, outs = [], []
    files = (A.TranscodeFile * len(entries))()
    for i, (data, cfgs, caps, n) in enumerate(entries):
        src = None if data is None else np.frombuffer(data, np.uint8).copy()
        rungs, o = None, []
        if cfgs is not None:
            caps = caps or [len(data or b"") * 2 + (1 << 20)] * len(cfgs)
            o = [np.full(max(c, 1), 0xA5, np.uint8) for c in caps]
            rungs = (A.TranscodeRung * max(len(cfgs), 1))()
            for j, c in enumerate(cfgs):
                rungs[j] = A.TranscodeRung(A.TranscodeConfig(*c), o[j].ctypes.data, caps[j], 0, -1)
        keep.append((src, rungs))
        outs.append(o)
        files[i] = A.TranscodeFile(None if src is None else src.ctypes.data, 0 if src is None else src.size, rungs,
                                   len(cfgs or []) if n is None else n, -1)
    rc = lib.uhdr_b200_transcode_ladders(files, len(entries))
    res = []
    for i, (data, cfgs, caps, n) in enumerate(entries):
        rungs = keep[i][1]
        if cfgs is None or (n is not None and not 1 <= n <= 16) or data is None:
            assert all((b == 0xA5).all() for b in outs[i]), ("a file with an argument error wrote into out", i)
            assert all(rungs[j].status == -1 for j in range(len(cfgs or []))), i
            res.append((files[i].status, None))
            continue
        got = []
        for j in range(len(cfgs)):
            st, m = rungs[j].status, rungs[j].out_size
            if st:
                assert (outs[i][j] == 0xA5).all(), ("a failing rung wrote into out", i, j)
                got.append((st, None, m))
            else:
                got.append((0, bytes(outs[i][j][:m]), m))
        res.append((files[i].status, got))
    return rc, res


def per_file(lib, entries):
    """what uhdr_b200_transcode_ladder gives each entry alone, in ladders()'s form, and its message"""
    want = []
    for data, cfgs, caps, n in entries:
        if cfgs is None or data is None or (n is not None and not 1 <= n <= 16):
            src = np.frombuffer(data or b"\xff", np.uint8).copy()
            rungs = (A.TranscodeRung * max(len(cfgs or []), 1))()
            rc = lib.uhdr_b200_transcode_ladder(src.ctypes.data if data else None, src.size,
                                                rungs if cfgs is not None else None,
                                                len(cfgs or []) if n is None else n)
            want.append(((rc, None), lib.uhdr_b200_last_error()))
            continue
        rc, got = ladder(lib, data, cfgs, caps)
        want.append(((rc, got), lib.uhdr_b200_last_error()))
    return want


def _check(lib, entries):
    want = per_file(lib, entries)
    rc, got = ladders(lib, entries)
    assert got == [w[0] for w in want], [(i, g[0], w[0][0]) for i, (g, w) in enumerate(zip(got, want)) if g != w[0]]
    first = next((i for i, g in enumerate(got) if g[0]), None)
    assert rc == (0 if first is None else got[first][0])
    if first is not None:
        assert lib.uhdr_b200_last_error() == b"file %d: " % first + want[first][1], lib.uhdr_b200_last_error()
    return got


def _dec_stats(lib):
    e = (C.c_ulonglong * 3)()
    lib.uhdr_b200_entropy_decoder_stats(e)
    return e[0], e[1]


def _entries(corpus, shift=0):
    return [(d, LADDER_LIST[(i + shift) % len(LADDER_LIST)], None, None) for i, d in enumerate(corpus.values())]


def test_equals_per_file_ladders(lib, corpus):
    for shift in range(len(LADDER_LIST)):
        got = _check(lib, _entries(corpus, shift))
        assert all(g[0] == 0 for g in got), (shift, [g[0] for g in got])


def test_equals_the_reference_composition(ref, lib, corpus):
    entries = _entries(corpus, 2)
    rc, got = ladders(lib, entries)
    assert rc == 0, lib.uhdr_b200_last_error()
    for (data, cfgs, _c, _n), (_st, rungs) in zip(entries, got):
        for j in (0, len(cfgs) - 1):
            assert rungs[j][1] == X.composition(ref, data, *cfgs[j]), cfgs[j]


def _route(lib, entries):
    d0, h0 = _dec_stats(lib)
    b0 = A.jpeg_encode_batch_stats(lib)
    lib.uhdr_b200_set_kernel_timing(1)
    _kernel_counts(lib)
    try:
        l0 = lib.uhdr_b200_kernel_launches()
        rc, got = ladders(lib, entries)
        launches = lib.uhdr_b200_kernel_launches() - l0
        kc = _kernel_counts(lib)
    finally:
        lib.uhdr_b200_set_kernel_timing(0)
    assert rc == 0, lib.uhdr_b200_last_error()
    d1, h1 = _dec_stats(lib)
    b1 = A.jpeg_encode_batch_stats(lib)
    assert (d1 - d0, h1 - h0) == (2 * len(entries), 0)   # both scans of every file once, on the device
    assert b1[0] - b0[0] == 1                              # one group
    pairs = len(set((c[1], c[2]) for e in entries for c in e[1]))
    assert (kc.get("idct_multi"), kc.get("stage_batch"), kc.get("fdct_code_batch"), kc.get("huff_encode_batch"),
            kc.get("pack_scans")) == (1, 1, pairs, 1, 1), kc
    for name in ("idct_dequant", "idct_scaled", "huff_encode", "fdct_quant", "ycc444_to_420"):
        assert name not in kc, kc
    return got, launches


def test_route(lib, corpus):
    names = ["own_api1_420_rgbmap", "own_api1_graymap_s4", "p420_gray_ragged", "p444_444map_s4", "pgray",
             "foreign_tables_restart"]
    _route(lib, [(corpus[n], LADDER_LIST[i % len(LADDER_LIST)], None, None) for i, n in enumerate(names)])
    data = corpus["p420_gray_ragged"]
    launches = []
    for n in (1, 4, 32):
        got, nl = _route(lib, [(data, LADDERS["mixed_420_exif"], None, None)] * n)
        assert len(set(str(g) for g in got)) == 1
        launches.append(nl)
    assert launches[0] == launches[1] == launches[2], launches


def test_errors_in_one_call(ref, lib, corpus):
    from test_gpu_decode_batch import flat_file
    good = corpus["p420_gray_ragged"]
    s422 = X.api4_file(ref, X.metadata(), 131, 67, "422", "gray", 1, exif=EXIF)
    garbage = b"\xff\xd8\xff\xe0" + bytes(range(200)) + b"\xff\xd9"
    _rc, full, n_ok = X.transcode(lib, good, 2, 75, 75, 0, 1)
    short = [(2, 75, 75, 0, 1), (4, 75, 75, 1, 1), (2, 75, 75, 0, 1)]
    d0, h0 = _dec_stats(lib)
    entries = [
        (corpus["own_api1_420_rgbmap"], LADDERS["all_k"], None, None),
        (garbage, LADDERS["mixed_420_exif"], None, None),
        (_progressive(ref, good), LADDERS["duplicated"], None, None),
        (corpus["pgray"], LADDERS["reversed"], None, None),
        (good, None, None, 1),                               # null rungs
        (good, LADDERS["all_k"], None, 0),
        (good, [(1, 75, 75, 0, 0)] * 16, None, 17),
        (None, LADDERS["all_k"], None, None),                # null data
        (s422, [(1, 75, 75, 0, 0), (2, 75, 75, 0, 0), (1, 75, 75, 1, 0)], None, None),
        (good, short, [n_ok - 1, len(good) * 2, n_ok], None),
        (flat_file(lib), LADDERS["all_k"], None, None),      # its primary's scan goes to the host decoder
        (corpus["p444_444map_s4"], LADDERS["k1_two_qualities"] + [(3, 75, 75, 0, 0), (2, 75, 75, 0, 0)], None, None),
    ]
    got = _check(lib, entries)
    st = [g[0] for g in got]
    assert st[0] == st[3] == st[10] == 0 and all(s != 0 for s in st[1:3]), st
    assert st[4:8] == [A.CODEC_INVALID_PARAM] * 4 and st[11] == A.CODEC_INVALID_PARAM, st
    assert [r[0] for r in got[8][1]] == [0, A.CODEC_UNSUPPORTED, A.CODEC_UNSUPPORTED]
    assert got[9][1][0] == (A.CODEC_MEM_ERROR, None, n_ok) and got[9][1][1][0] == 0 and got[9][1][2][1] == full
    assert [r[0] for r in got[11][1]][-2:] == [A.CODEC_INVALID_PARAM, 0]
    assert lib.uhdr_b200_last_error().startswith(b"file 1: ")
    d1, h1 = _dec_stats(lib)
    assert h1 - h0 >= 2   # the flat primary, in the per-file ladder and in the call


def test_groups_give_the_same_results(lib, corpus, monkeypatch):
    entries = _entries(corpus, 1)
    _rc, whole = ladders(lib, entries)
    monkeypatch.setenv("UHDR_B200_BATCH_GROUP_BYTES", "1")   # one file per group
    b0 = A.jpeg_encode_batch_stats(lib)
    rc, grouped = ladders(lib, entries)
    b1 = A.jpeg_encode_batch_stats(lib)
    assert rc == 0 and grouped == whole and b1[0] - b0[0] == len(entries)
    # files with argument errors after a file over the budget: a group with no rung
    bad = [(entries[0][0], None, None, 1), (None, LADDERS["all_k"], None, None)]
    rc, got = ladders(lib, entries[:2] + bad)
    assert rc == A.CODEC_INVALID_PARAM and got == whole[:2] + [(A.CODEC_INVALID_PARAM, None)] * 2
    assert lib.uhdr_b200_last_error().startswith(b"file 2: ")
    monkeypatch.delenv("UHDR_B200_BATCH_GROUP_BYTES")
    # 6 files x 4 distinct quality pairs: groups of 16 pairs, then 8
    names = ["own_api1_420_rgbmap", "p420_gray_ragged", "p444_444map_s4", "pgray", "p420_420map_s2", "p444_w63x8"]
    entries = [(corpus[n], [(k, 50 + 4 * i + j, 60 + j, j & 1, 1) for j, k in enumerate((1, 2, 4, 8))], None, None)
               for i, n in enumerate(names)]
    b0 = A.jpeg_encode_batch_stats(lib)
    got = _check(lib, entries)
    b1 = A.jpeg_encode_batch_stats(lib)
    assert all(g[0] == 0 for g in got) and b1[0] - b0[0] == 2 + len(entries), b1[0] - b0[0]


def test_host_decoder_switch(lib, corpus):
    garbage = b"\xff\xd8\xff\xe0" + bytes(range(200)) + b"\xff\xd9"
    entries = _entries(corpus, 3) + [(garbage, LADDERS["all_k"], None, None)]
    runs = {}
    for mode in (2, 1):
        prev = lib.uhdr_b200_set_entropy_decoder(mode)
        try:
            s0 = _dec_stats(lib)
            rc, got = ladders(lib, entries)
            s1 = _dec_stats(lib)
        finally:
            lib.uhdr_b200_set_entropy_decoder(prev)
        runs[mode] = (rc, got, lib.uhdr_b200_last_error(), (s1[0] - s0[0], s1[1] - s0[1]))
    assert runs[2][0] != 0 and all(g[0] == 0 for g in runs[2][1][:-1]), runs[2][0]
    assert runs[1][:3] == runs[2][:3]
    assert runs[2][3][0] > 0 and runs[1][3] == (0, 0), (runs[2][3], runs[1][3])


def test_interleaved_with_other_calls(lib, corpus):
    import torch
    from test_gpu_transcode import _decode_dev
    names = ["own_api1_420_rgbmap", "p444_444map_s4", "foreign_tables_restart", "p420_gray_ragged"]
    datas = [corpus[n] for n in names]
    entries = [(d, LADDER_LIST[i], None, None) for i, d in enumerate(datas)]
    want = per_file(lib, entries)
    bwant = [tuple(X.transcode(lib, d, 2, 80, 70, 1, 1)) for d in datas]
    pix = [_decode_dev(torch, lib, d, 2) for d in datas]
    for r in range(3):
        rc, got = ladders(lib, entries)
        assert rc == 0 and got == [w[0] for w in want]
        assert X.transcode(lib, datas[r], 2, 80, 70, 1, 1) == bwant[r]
        rc, got = batch(lib, datas, 2, 80, 70, 1, 1)
        assert rc == 0 and got == bwant
        assert ladder(lib, datas[r], LADDER_LIST[r]) == want[r][0]
        assert (_decode_dev(torch, lib, datas[r], 2) == pix[r]).all()


def test_two_threads_at_once(lib, corpus):
    entries = _entries(corpus)
    want = [w[0] for w in per_file(lib, entries)]
    errors = []

    def run(t):
        try:
            for _rep in range(2):
                e = entries if t == 0 else entries[::-1]
                rc, got = ladders(lib, e)
                if rc != 0 or got != (want if t == 0 else want[::-1]):
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
    exe = str(tmp_path / "alloc_probe_transcode_ladders")
    so = T.GPU_SO
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    cmd = ["gcc", "-O1", "-g", "-I", os.path.join(T.ROOT, "include"), "-I", os.path.join(cuda, "include"),
           os.path.join(T.ROOT, "tests", "cpp", "alloc_probe_transcode_ladders.c"), "-o", exe, "-L", os.path.dirname(so),
           "-l:" + os.path.basename(so), "-Wl,-rpath," + os.path.dirname(so), "-L", os.path.join(cuda, "lib64"),
           "-lcudart", "-Wl,-rpath," + os.path.join(cuda, "lib64"), "-ldl", "-rdynamic"]
    subprocess.run(cmd, check=True, capture_output=True)
    paths = []
    for n in ("p444_444map_s4", "p420_gray_ragged"):
        p = str(tmp_path / (n + ".jpg"))
        with open(p, "wb") as f:
            f.write(corpus[n])
        paths.append(p)
    r = subprocess.run([exe] + paths, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout, r.stderr[-4000:])
    assert "ours=0 " in r.stdout, r.stdout
