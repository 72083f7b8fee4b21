"""Per-device kernel state (the constant tables in device memory and the wave sizes of the persistent kernels) is made
once per device and afterwards only looked up.  After one warm-up of every kind of call that keeps such state, the
same calls from 8 new host threads and a uhdr_b200_encode_batch call (whose workers are new threads too) leave
uhdr_b200_device_state_stats unchanged and give the warm-up's bytes.  With two visible GPUs, the second device gets
its own state on its first use, gives device 0's bytes, and makes nothing more when the work alternates between them."""
import ctypes as C
import threading

import numpy as np
import pytest

import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A

pytestmark = pytest.mark.gpu

W, H = 1920, 1080
BATCH = 4   # frames (and streams) of the uhdr_b200_encode_batch call


@pytest.fixture(scope="module")
def lib(gpu):
    L = gpu.lib
    T.UhdrApi(L)   # result types of the uhdr_* calls
    A.declare_transcode_batch(L)
    L.uhdr_b200_device_state_stats.argtypes = [C.POINTER(C.c_ulonglong)]
    L.uhdr_b200_device_state_stats.restype = None
    L.uhdr_b200_jpeg_encode_dev.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                            C.c_void_p, C.c_void_p]
    L.uhdr_b200_last_error.restype = C.c_char_p
    L.uhdr_reset_decoder.restype = None
    return L


def _stats(lib):
    st = (C.c_ulonglong * 2)()
    lib.uhdr_b200_device_state_stats(st)
    return st[0], st[1]


def _ck(e):
    assert e.error_code == 0, (e.error_code, e.detail)


class DeviceWork:
    """Every kind of call that keeps per-device state, on device `dev`: an API-1 (map scale 1) and an API-0 (map
    scale 4) uhdr_encode handle and a half-float uhdr_decode handle, made on that device and driven from any thread;
    a uhdr_b200_transcode_batch of the API-1 file; a uhdr_b200_jpeg_encode_dev of an RGB888 image; and a
    uhdr_b200_encode_batch of the API-1 frame on 4 streams."""

    def __init__(self, lib, torch, dev):
        self.lib, self.torch, self.dev = lib, torch, dev
        torch.cuda.set_device(dev)
        hb, sb = T.make_p010(W, H, "smooth"), T.make_yuv420(W, H, "smooth")
        self.hdr, k1 = A.p010_image(hb, W, H, A.CG_BT2100, A.CT_HLG, A.CR_LIMITED)
        self.sdr, k2 = A.yuv420_image(sb, W, H, A.CG_BT709)
        self.keep = (hb, sb, k1, k2)
        self.enc1 = self._encoder(with_sdr=True, scale=1)
        self.enc0 = self._encoder(with_sdr=False, scale=4)
        self.dec = C.c_void_p(lib.uhdr_create_decoder())
        self.locks = {h: threading.Lock() for h in ("enc1", "enc0", "dec")}   # a handle serves one call at a time
        rgb = np.random.RandomState(T.SEED).randint(0, 256, (H, W * 3)).astype(np.uint8)
        self.rgb = torch.from_numpy(rgb).to(f"cuda:{dev}")
        torch.cuda.synchronize(dev)
        self.rgb_img = A.raw_image(A.FMT_RGB888, A.CG_BT709, A.CT_SRGB, A.CR_FULL, W, H, [], [])
        self.rgb_img.planes[0], self.rgb_img.stride[0] = self.rgb.data_ptr(), W
        with self.locks["enc1"]:
            self.file = self._encode(self.enc1)

    def _encoder(self, with_sdr, scale):
        L = self.lib
        enc = C.c_void_p(L.uhdr_create_encoder())
        _ck(L.uhdr_enc_set_raw_image(enc, C.byref(self.hdr), A.HDR_IMG))
        if with_sdr:
            _ck(L.uhdr_enc_set_raw_image(enc, C.byref(self.sdr), A.SDR_IMG))
        _ck(L.uhdr_enc_set_quality(enc, 95, A.BASE_IMG))
        _ck(L.uhdr_enc_set_quality(enc, 95, A.GAIN_MAP_IMG))
        _ck(L.uhdr_enc_set_gainmap_scale_factor(enc, scale))
        _ck(L.uhdr_enc_set_using_multi_channel_gainmap(enc, 1))
        return enc

    def close(self):
        self.lib.uhdr_release_encoder(self.enc1)
        self.lib.uhdr_release_encoder(self.enc0)
        self.lib.uhdr_release_decoder(self.dec)

    def _encode(self, enc):
        L = self.lib
        assert L.uhdr_b200_enc_rearm(enc) == 0
        _ck(L.uhdr_encode(enc))
        o = L.uhdr_get_encoded_stream(enc).contents
        return C.string_at(o.data, o.data_sz)

    def _decode(self):
        L = self.lib
        buf = np.frombuffer(self.file, np.uint8).copy()
        ci = A.CompressedImage(buf.ctypes.data, buf.size, buf.size, -1, -1, -1)
        L.uhdr_reset_decoder(self.dec)
        _ck(L.uhdr_dec_set_image(self.dec, C.byref(ci)))
        _ck(L.uhdr_dec_set_out_img_format(self.dec, A.FMT_RGBAF16))
        _ck(L.uhdr_dec_set_out_color_transfer(self.dec, A.CT_LINEAR))
        _ck(L.uhdr_decode(self.dec))
        d = L.uhdr_get_decoded_image(self.dec).contents
        return C.string_at(d.planes[0], d.h * d.stride[0] * 8)

    def _transcode_batch(self):
        L = self.lib
        data = np.frombuffer(self.file, np.uint8).copy()
        cap = data.size + (1 << 20)
        out = np.zeros(cap, np.uint8)
        items = (A.TranscodeItem * 1)(A.TranscodeItem(data.ctypes.data, data.size, out.ctypes.data, cap, 0, -1))
        rc = L.uhdr_b200_transcode_batch(items, 1, C.byref(A.TranscodeConfig(2, 90, 85, 0, 0)))
        assert rc == 0 and items[0].status == 0, L.uhdr_b200_last_error()
        return bytes(out[:items[0].out_size])

    def _jpeg_encode_dev(self):
        L = self.lib
        cap = W * H * 6 + (1 << 16)
        out = np.zeros(cap, np.uint8)
        n = C.c_size_t()
        rc = L.uhdr_b200_jpeg_encode_dev(C.byref(self.rgb_img), 90, None, 0, out.ctypes.data, cap, C.byref(n), None)
        assert rc == 0, L.uhdr_b200_last_error()
        return bytes(out[:n.value])

    def _encode_batch(self):
        L = self.lib
        hdrs, sdrs = (A.RawImage * BATCH)(*[self.hdr] * BATCH), (A.RawImage * BATCH)(*[self.sdr] * BATCH)
        cap = W * H * 6 + (1 << 16)
        bufs = [np.zeros(cap, np.uint8) for _ in range(BATCH)]
        outs = (A.CompressedImage * BATCH)(*[A.CompressedImage(b.ctypes.data, 0, cap, -1, -1, -1) for b in bufs])
        rc = L.uhdr_b200_encode_batch(BATCH, hdrs, sdrs, C.byref(A.default_gm_config()), 95, outs, BATCH)
        assert rc == 0, L.uhdr_b200_last_error()
        return [bytes(bufs[i][:outs[i].data_sz]) for i in range(BATCH)]

    def run(self, batch=True):
        """every call once on this device, from the calling thread -> {call: output bytes}"""
        self.torch.cuda.set_device(self.dev)
        out = {}
        with self.locks["enc1"]:
            out["api1"] = self._encode(self.enc1)
        with self.locks["enc0"]:
            out["api0"] = self._encode(self.enc0)
        with self.locks["dec"]:
            out["decode"] = self._decode()
        out["transcode_batch"] = self._transcode_batch()
        out["jpeg_encode_dev"] = self._jpeg_encode_dev()
        if batch:
            out["encode_batch"] = self._encode_batch()
        return out


def from_new_threads(work, n=8):
    """work.run() from n new host threads at once, the encode_batch call from one of them"""
    results, errors = [None] * n, []

    def body(i):
        try:
            results[i] = work.run(batch=i == 0)
        except BaseException as e:   # re-raised on the main thread
            errors.append(e)

    threads = [threading.Thread(target=body, args=(i,)) for i in range(n)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise errors[0]
    return results


def assert_same(got, want, what):
    for k, v in got.items():
        assert v == want[k], (what, k)


def test_state_is_made_once_per_device(lib):
    import torch
    work = DeviceWork(lib, torch, 0)
    try:
        warm = work.run()
        assert warm["encode_batch"] == [warm["api1"]] * BATCH
        s = _stats(lib)
        assert s[0] > 0 and s[1] > 0, s
        for i, r in enumerate(from_new_threads(work)):
            assert_same(r, warm, f"thread {i}")
        assert _stats(lib) == s
    finally:
        work.close()


def test_second_device_gets_its_own_state(lib):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    works = [DeviceWork(lib, torch, 0)]
    try:
        warm = works[0].run()
        s0 = _stats(lib)
        works.append(DeviceWork(lib, torch, 1))
        assert_same(works[1].run(), warm, "device 1")
        s1 = _stats(lib)
        assert s1[0] > s0[0] and s1[1] > s0[1], (s0, s1)   # device 1's own tables and wave sizes
        for i, r in enumerate(from_new_threads(works[1])):
            assert_same(r, warm, f"device 1, thread {i}")
        for _ in range(4):
            for w in works:
                assert_same(w.run(), warm, f"device {w.dev}")
        assert _stats(lib) == s1
    finally:
        for w in works:
            w.close()
