"""uhdr_b200_decode_batch_dev on the GPU, at 0 tolerance: every item of a batch equals uhdr_b200_decode_scaled_dev of
that file alone (pixels, map, metadata, descriptor fields), for every k and output, over a batch that mixes sizes,
samplings, map channels and scales, ISO and XMP-only metadata, restart intervals, a resized map and a scan handed to
the host decoder; per-item errors that write nothing; groups; the launch count; stream order and threads."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

import scaled_testlib as S
import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A
from test_api4_cpu import _api4
from test_gpu_dev_codec import BPP, OUTPUTS, _sleep_cycles
from test_gpu_resident_render import encoded, golden, resize_file, restart_file

pytestmark = pytest.mark.gpu

GUARD = 0x5A
INVALID, UNSUPPORTED = 3, 6


@pytest.fixture(scope="module")
def lib(gpu):
    L = A.declare_decode_batch(A.declare_scaled_decode(gpu.lib))
    L.uhdr_b200_last_error.restype = C.c_char_p
    L.uhdr_b200_kernel_launches.restype = C.c_ulonglong
    L.uhdr_b200_entropy_decoder_stats.argtypes = [C.POINTER(C.c_ulonglong)]
    L.uhdr_b200_entropy_decoder_stats.restype = None
    return L


def torch():
    import torch as t
    return t


def _md(boost=4.0):
    md = A.GainmapMetadata()
    for i in range(3):
        md.max_content_boost[i], md.min_content_boost[i], md.gamma[i] = boost, 1.0, 1.0
        md.offset_sdr[i] = md.offset_hdr[i] = 1.0 / 64
    md.hdr_capacity_min, md.hdr_capacity_max, md.use_base_cg = 1.0, boost, 1
    return md


def api4_file(lib, w, h, layout, gw, gh, glayout, seed=1):
    data = _api4(lib, S.pil_jpeg(S.image(w, h, "smooth", seed=seed), 90, layout),
                 S.pil_jpeg(S.image(gw, gh, "noise", seed=seed + 1), 90, glayout), _md(), A.CG_BT709)
    assert isinstance(data, bytes), data
    return data


def flat_file(lib):
    """a black 3840x2160 primary whose flat run never falls back into step: its scan goes to the host decoder"""
    import jpeg_decode_cases as D
    lead, _ph = D.lead_for_phase(D.S420, True, 32, dc=-128)
    st = D.flat_frame(3840, 2160, D.S420, lead, dc=-128)
    data = _api4(lib, st.data, S.pil_jpeg(S.image(96, 54, "noise", seed=4), 90, "gray"), _md(), A.CG_BT709)
    assert isinstance(data, bytes), data
    return data


_cache = {}


def files(lib, k):
    """the mixed batch for k: library-encoded files (map scales 1 / 2 / 4, one- and three-channel maps), odd and
    minimum sizes of 4:2:0 / 4:4:4 primaries (4:2:2 at k = 1 only), the Apple files (ISO and XMP-only metadata), a
    restart-interval file and a map that needs a resize"""
    if "base" not in _cache:
        _cache["base"] = [encoded(lib, 998, 722, 1, 1), encoded(lib, 1920, 1080, 2, 0), encoded(lib, 998, 722, 4, 1),
                          api4_file(lib, 1, 1, "444", 1, 1, "gray"), api4_file(lib, 17, 9, "420", 5, 3, "444"),
                          api4_file(lib, 33, 21, "444", 9, 6, "gray"),
                          golden("apple_gainmap_old.jpg"), golden("apple_gainmap_new.jpg"), restart_file(lib),
                          resize_file(lib)]
        _cache["422"] = api4_file(lib, 64, 48, "422", 32, 24, "gray")
    return _cache["base"] + ([_cache["422"]] if k == 1 else [])


class Item:
    """one file with guarded device destinations of its 1/k sizes"""

    def __init__(self, lib, data, k, fmt, want_map=True, want_md=True):
        t = torch()
        self.src = np.frombuffer(data, np.uint8).copy()
        d = [C.c_uint() for _ in range(4)]
        assert lib.uhdr_b200_scaled_dims(self.src.ctypes.data, self.src.size, k, *[C.byref(x) for x in d]) == 0
        w, h, gw, gh = [x.value for x in d]
        self.buf = t.full((h * w * BPP[fmt],), GUARD, dtype=t.uint8, device="cuda")
        self.dest = A.raw_image(fmt, -1, -1, -1, w, h, [], [])
        self.dest.planes[0], self.dest.stride[0] = self.buf.data_ptr(), w
        self.gbuf = self.gdesc = None
        if want_map:
            self.gbuf = t.full((gh * gw * 4,), GUARD, dtype=t.uint8, device="cuda")
            self.gdesc = A.raw_image(-1, -1, -1, -1, gw, gh, [], [])
            self.gdesc.planes[0], self.gdesc.stride[0] = self.gbuf.data_ptr(), gw
        self.md = A.GainmapMetadata() if want_md else None

    def item(self):
        return A.DecodeItem(self.src.ctypes.data, self.src.size, C.pointer(self.dest),
                            C.pointer(self.gdesc) if self.gdesc is not None else None,
                            C.pointer(self.md) if self.md is not None else None, -1)

    def single(self, lib, k, ct, boost, stream=None):
        return lib.uhdr_b200_decode_scaled_dev(self.src.ctypes.data, self.src.size, k, ct, boost, C.byref(self.dest),
                                               C.byref(self.gdesc) if self.gdesc is not None else None,
                                               C.byref(self.md) if self.md is not None else None, stream)

    def result(self):
        return (self.buf.clone(), None if self.gbuf is None else self.gbuf.clone(),
                None if self.md is None else bytes(self.md),
                (self.dest.cg, self.dest.ct, self.dest.range),
                None if self.gdesc is None else (self.gdesc.fmt, self.gdesc.cg, self.gdesc.ct, self.gdesc.range))

    def untouched(self):
        return bool((self.buf == GUARD).all()) and (self.gbuf is None or bool((self.gbuf == GUARD).all()))


def batch(lib, items, k, ct, boost, stream=None):
    arr = (A.DecodeItem * len(items))(*[it.item() for it in items])
    rc = lib.uhdr_b200_decode_batch_dev(arr, len(items), k, ct, boost, stream)
    return rc, [arr[i].status for i in range(len(items))]


def singles(lib, datas, k, fmt, ct, boost, **kw):
    out = []
    for d in datas:
        it = Item(lib, d, k, fmt, **kw)
        rc = it.single(lib, k, ct, boost)
        torch().cuda.synchronize()
        out.append((rc, it.result() if rc == 0 else None, it))
    return out


def same(a, b):
    t = torch()
    return all((x is None and y is None) or (isinstance(x, t.Tensor) and t.equal(x, y)) or
               (not isinstance(x, t.Tensor) and x == y) for x, y in zip(a, b))


@pytest.mark.parametrize("k", [1, 2, 4, 8])
def test_mixed_batch_equals_single_decodes(lib, k):
    datas = files(lib, k)
    for fmt, ct in OUTPUTS:
        for boost in ([3.0, A.FLT_MAX] if ct != A.CT_SRGB else [A.FLT_MAX]):
            want = singles(lib, datas, k, fmt, ct, boost)
            assert all(rc == 0 for rc, _r, _i in want), [(rc, lib.uhdr_b200_last_error()) for rc, _r, _i in want]
            items = [Item(lib, d, k, fmt) for d in datas]
            rc, st = batch(lib, items, k, ct, boost)
            assert rc == 0 and st == [0] * len(items), (rc, st, lib.uhdr_b200_last_error())
            torch().cuda.synchronize()
            for i, (it, (_rc, w, _x)) in enumerate(zip(items, want)):
                assert same(it.result(), w), (k, fmt, ct, boost, i)


def test_items_without_map_or_metadata(lib):
    datas = files(lib, 2)[:6]
    for ct in (A.CT_HLG, A.CT_PQ, A.CT_SRGB):
        fmt = A.FMT_RGBA8888 if ct == A.CT_SRGB else A.FMT_RGBA1010102
        kw = [dict(want_map=i % 2 == 0, want_md=i % 3 == 0) for i in range(len(datas))]
        if ct == A.CT_SRGB:   # metadata without a map is an error of the single call there: keep those apart
            kw = [dict(want_map=i % 2 == 0, want_md=i % 2 == 0 and i % 3 == 0) for i in range(len(datas))]
        items = [Item(lib, d, 2, fmt, **kw[i]) for i, d in enumerate(datas)]
        rc, st = batch(lib, items, 2, ct, 5.0)
        assert rc == 0 and st == [0] * len(items), (rc, st, lib.uhdr_b200_last_error())
        torch().cuda.synchronize()
        for i, d in enumerate(datas):
            w = Item(lib, d, 2, fmt, **kw[i])
            assert w.single(lib, 2, ct, 5.0) == 0
            torch().cuda.synchronize()
            assert same(items[i].result(), w.result()), (ct, i)


def _stats(lib):
    st = (C.c_ulonglong * 3)()
    lib.uhdr_b200_entropy_decoder_stats(st)
    return list(st)


def test_flat_scan_goes_to_the_host_decoder_alone(lib):
    datas = [encoded(lib, 998, 722, 1, 1), flat_file(lib), golden("apple_gainmap_new.jpg")]
    want = singles(lib, datas, 1, A.FMT_RGBAF16, A.CT_LINEAR, 4.0)
    assert all(rc == 0 for rc, _r, _i in want)
    items = [Item(lib, d, 1, A.FMT_RGBAF16) for d in datas]
    s0 = _stats(lib)
    rc, st = batch(lib, items, 1, A.CT_LINEAR, 4.0)
    torch().cuda.synchronize()
    s1 = _stats(lib)
    assert rc == 0 and st == [0, 0, 0], (rc, st)
    assert s1[1] - s0[1] == 1, (s0, s1)          # exactly the flat primary was handed back
    assert s1[0] - s0[0] == 5, (s0, s1)          # the other five scans were decoded on the device
    for it, (_rc, w, _x) in zip(items, want):
        assert same(it.result(), w)



def test_host_decoder_switch_applies_to_batches(lib):
    """uhdr_b200_set_entropy_decoder(1) sends every scan of a batch to the host decoder: the same pixels and codes as
    the device decoder gives, and the device decoder's counts do not move"""
    good = files(lib, 1)
    datas = [good[0], corrupt_file(lib, good[0]), good[6], good[8], good[9]]
    runs = {}
    for mode in (2, 1):
        prev = lib.uhdr_b200_set_entropy_decoder(mode)
        try:
            items = [Item(lib, d, 1, A.FMT_RGBAF16) for d in datas]
            s0 = _stats(lib)
            rc, st = batch(lib, items, 1, A.CT_LINEAR, 4.0)
            torch().cuda.synchronize()
            s1 = _stats(lib)
        finally:
            lib.uhdr_b200_set_entropy_decoder(prev)
        runs[mode] = (rc, st, lib.uhdr_b200_last_error(), items, (s1[0] - s0[0], s1[1] - s0[1]))
    rc, st, err, items, dev = runs[2]
    assert st == [0, rc, 0, 0, 0] and rc != 0, (rc, st, err)
    assert runs[1][:3] == (rc, st, err)
    assert items[1].untouched() and runs[1][3][1].untouched()
    for a, b in zip(items, runs[1][3]):
        assert same(a.result(), b.result())
    assert dev[0] > 0 and runs[1][4] == (0, 0), (dev, runs[1][4])

def corrupt_file(lib, data):
    """data with bytes of the primary image's entropy-coded segment overwritten so that decoding it fails (not every
    damage does: some decode to other pixels), found by trying seeded damages"""
    sos = data.index(b"\xff\xda")
    end = data.index(b"\xff\xd9", sos)   # the primary's EOI: the headers of both JPEGs stay intact
    rs = np.random.RandomState(5)
    for _t in range(32):
        bad = bytearray(data)
        for _ in range(4):   # no 0xFF: the container's marker scan must still find both images
            pos = int(rs.randint(sos + 16, end - 64))
            bad[pos:pos + 48] = rs.randint(0, 255, 48).astype(np.uint8).tobytes()
        it = Item(lib, data, 1, A.FMT_RGBAF16)
        it.src = np.frombuffer(bytes(bad), np.uint8).copy()
        rc = it.single(lib, 1, A.CT_LINEAR, 4.0)
        torch().cuda.synchronize()
        if rc != 0:
            return bytes(bad)
    raise AssertionError("no damage made the file fail to decode")


def test_per_item_errors(lib):
    good = files(lib, 1)
    corrupt = corrupt_file(lib, good[0])
    no_md = S.pil_jpeg(S.image(64, 48, "smooth"), 90, "420")          # a plain JPEG: no gain map, no metadata
    s422 = api4_file(lib, 64, 48, "422", 32, 24, "gray")
    for k, datas in ((1, [good[1], bytes(corrupt), good[3], no_md, good[6]]),
                     (2, [good[1], s422, good[3], bytes(corrupt), good[6]])):
        want = []
        for d in datas:
            it = Item(lib, d, k, A.FMT_RGBAF16) if d is not no_md else None
            if it is None:
                src = np.frombuffer(d, np.uint8).copy()
                dims = [C.c_uint() for _ in range(4)]
                want.append((lib.uhdr_b200_scaled_dims(src.ctypes.data, src.size, k, *[C.byref(x) for x in dims]), None))
                continue
            rc = it.single(lib, k, A.CT_LINEAR, 4.0)
            torch().cuda.synchronize()
            want.append((rc, it.result() if rc == 0 else None))
        assert [rc != 0 for rc, _ in want] == [False, True, False, True, False]
        items = []
        for d in datas:
            if d is no_md:  # destinations sized like a good item: the probe fails before sizes matter
                it = Item(lib, good[3], k, A.FMT_RGBAF16)
                it.src = np.frombuffer(d, np.uint8).copy()
            else:
                it = Item(lib, d, k, A.FMT_RGBAF16)
            items.append(it)
        rc, st = batch(lib, items, k, A.CT_LINEAR, 4.0)
        torch().cuda.synchronize()
        assert st == [w[0] for w in want], (k, st, want)
        first = next(i for i, s in enumerate(st) if s)
        assert rc == st[first] and lib.uhdr_b200_last_error().startswith(b"item %d: " % first), lib.uhdr_b200_last_error()
        for it, (wrc, w) in zip(items, want):
            if wrc:
                assert it.untouched()
            else:
                assert same(it.result(), w)


def test_call_level_errors_decode_nothing(lib):
    it = Item(lib, files(lib, 1)[3], 1, A.FMT_RGBAF16)
    for args in ((1, 3), (1, 0), (0, 1)):
        n, k = args
        arr = (A.DecodeItem * 1)(it.item())
        assert lib.uhdr_b200_decode_batch_dev(arr, n, k, A.CT_LINEAR, 4.0, None) == INVALID
        assert arr[0].status == -1
    assert lib.uhdr_b200_decode_batch_dev(None, 1, 1, A.CT_LINEAR, 4.0, None) == INVALID
    torch().cuda.synchronize()
    assert it.untouched()


def test_groups_give_the_same_bytes(lib, monkeypatch):
    datas = files(lib, 4)
    ref = [Item(lib, d, 4, A.FMT_RGBA1010102) for d in datas]
    assert batch(lib, ref, 4, A.CT_PQ, 6.0)[0] == 0
    torch().cuda.synchronize()
    monkeypatch.setenv("UHDR_B200_BATCH_GROUP_BYTES", str(1 << 20))   # about one file per group
    items = [Item(lib, d, 4, A.FMT_RGBA1010102) for d in datas]
    rc, st = batch(lib, items, 4, A.CT_PQ, 6.0)
    torch().cuda.synchronize()
    assert rc == 0 and st == [0] * len(items)
    for a, b in zip(items, ref):
        assert same(a.result(), b.result())
    # n = 1 equals the single call
    one = Item(lib, datas[0], 4, A.FMT_RGBA1010102)
    assert batch(lib, [one], 4, A.CT_PQ, 6.0)[0] == 0
    w = Item(lib, datas[0], 4, A.FMT_RGBA1010102)
    assert w.single(lib, 4, A.CT_PQ, 6.0) == 0
    torch().cuda.synchronize()
    assert same(one.result(), w.result())


def test_three_hundred_small_files(lib):
    datas = [api4_file(lib, 40 + i % 23, 24 + i % 17, "420" if i % 2 else "444", 10 + i % 5, 6 + i % 3,
                       "gray" if i % 3 else "444", seed=i) for i in range(300)]
    items = [Item(lib, d, 1, A.FMT_RGBAF16) for d in datas]
    rc, st = batch(lib, items, 1, A.CT_LINEAR, 4.0)
    torch().cuda.synchronize()
    assert rc == 0 and st == [0] * 300, (rc, lib.uhdr_b200_last_error())
    for i in range(0, 300, 7):
        w = Item(lib, datas[i], 1, A.FMT_RGBAF16)
        assert w.single(lib, 1, A.CT_LINEAR, 4.0) == 0
        torch().cuda.synchronize()
        assert same(items[i].result(), w.result()), i


def test_launches_do_not_grow_with_per_file_stages(lib):
    """32 and 64 copies of one file: the difference is the per-file writes only (one apply kernel each for a gray map
    at linear output), no entropy, DC or IDCT launch per file"""
    data = encoded(lib, 998, 722, 1, 0)
    counts = []
    for n in (32, 64):
        items = [Item(lib, data, 2, A.FMT_RGBAF16) for _ in range(n)]
        l0 = lib.uhdr_b200_kernel_launches()
        rc, _st = batch(lib, items, 2, A.CT_LINEAR, 4.0)
        counts.append(lib.uhdr_b200_kernel_launches() - l0)
        torch().cuda.synchronize()
        assert rc == 0
    one = Item(lib, data, 2, A.FMT_RGBAF16)
    l0 = lib.uhdr_b200_kernel_launches()
    assert one.single(lib, 2, A.CT_LINEAR, 4.0) == 0
    single = lib.uhdr_b200_kernel_launches() - l0
    torch().cuda.synchronize()
    per_file = (counts[1] - counts[0]) / 32
    assert per_file == 1, (counts, single)
    # the shared stages: what one file's decode launches, give or take the IDCT planes' and DC plans' launches
    assert counts[0] - 32 <= single, (counts, single)


def test_stream_order_without_host_sync(lib):
    t = torch()
    datas = files(lib, 8)
    want = singles(lib, datas, 8, A.FMT_RGBAF16, A.CT_LINEAR, 4.0)
    s = t.cuda.Stream()
    items = [Item(lib, d, 8, A.FMT_RGBAF16) for d in datas]
    with t.cuda.stream(s):
        t.cuda._sleep(_sleep_cycles(20))
        rc, st = batch(lib, items, 8, A.CT_LINEAR, 4.0, stream=s.cuda_stream)
        sums = [it.buf.sum() for it in items]     # enqueued after the call, on the same stream
    assert rc == 0
    s.synchronize()
    for it, sm, (_rc, w, _x) in zip(items, sums, want):
        assert int(sm) == int(w[0].sum())


def test_two_threads_with_their_own_streams(lib):
    t = torch()
    datas = files(lib, 2)
    want = singles(lib, datas, 2, A.FMT_RGBA1010102, A.CT_HLG, 4.0)
    errors = []

    def run():
        try:
            s = t.cuda.Stream()
            for _rep in range(3):
                items = [Item(lib, d, 2, A.FMT_RGBA1010102) for d in datas]
                with t.cuda.stream(s):
                    rc, _st = batch(lib, items, 2, A.CT_HLG, 4.0, stream=s.cuda_stream)
                s.synchronize()
                if rc != 0 or not all(same(it.result(), w[1]) for it, w in zip(items, want)):
                    errors.append(rc)
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    th = [threading.Thread(target=run) for _ in range(2)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors


def test_steady_state_does_not_touch_the_heap(lib, tmp_path):
    import subprocess
    exe = str(tmp_path / "alloc_probe_decode_batch")
    so = T.GPU_SO
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    cmd = ["gcc", "-O1", "-g", "-I", os.path.join(T.ROOT, "include"), "-I", os.path.join(cuda, "include"),
           os.path.join(T.ROOT, "tests", "cpp", "alloc_probe_decode_batch.c"), "-o", exe, "-L", os.path.dirname(so),
           "-l:" + os.path.basename(so), "-Wl,-rpath," + os.path.dirname(so), "-L", os.path.join(cuda, "lib64"),
           "-lcudart", "-Wl,-rpath," + os.path.join(cuda, "lib64"), "-ldl", "-rdynamic"]
    subprocess.run(cmd, check=True, capture_output=True)
    path = str(tmp_path / "file.jpg")
    with open(path, "wb") as f:
        f.write(encoded(lib, 998, 722, 1, 1))
    r = subprocess.run([exe, path], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout, r.stderr[-4000:])
    assert "ours=0 " in r.stdout, r.stdout
