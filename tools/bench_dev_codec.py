"""Host-buffer codec calls against their device-memory forms, on one GPU.

  8K JPEG/R -> RGBA half float: uhdr_decode (pixels land in host memory) against uhdr_b200_decode_dev into a torch
  tensor.  One host thread, a stream synchronise after every call, the two alternating.
  4K API-1 encode: uhdr_encode from pinned host intents against uhdr_b200_encode_dev from torch tensors, at 1 and 8
  host threads (one stream each).
  Block-stage staging: 4K API-1 encode_dev with a Display-P3 SDR intent (no colour conversion), its planes read in
  place (8-byte aligned rows) against the same planes with a 4-pixel pitch tail (copied into a padded workspace image
  first); the gain-map kernels are the same in both.

Prints the GPU name and power limit first, then one JSON line.  Usage:
  python tools/bench_dev_codec.py [--repeats 5] [--frames 16]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from libultrahdr_b200 import ctypes_api as A  # noqa: E402

SO = os.path.join(ROOT, "libultrahdr_b200", "libuhdr_b200.so")


def gpu_card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def load():
    L = C.CDLL(SO)
    L.uhdr_create_encoder.restype = C.c_void_p
    L.uhdr_create_decoder.restype = C.c_void_p
    for f in ("uhdr_enc_set_raw_image", "uhdr_encode", "uhdr_dec_set_image", "uhdr_decode", "uhdr_dec_set_out_img_format",
              "uhdr_dec_set_out_color_transfer", "uhdr_enc_set_quality"):
        getattr(L, f).restype = A.ErrorInfo
    L.uhdr_get_encoded_stream.restype = C.POINTER(A.CompressedImage)
    L.uhdr_get_decoded_image.restype = C.POINTER(A.RawImage)
    L.uhdr_b200_last_error.restype = C.c_char_p
    L.uhdr_b200_decode_dev.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p]
    L.uhdr_b200_encode_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p,
                                       C.c_size_t, C.c_void_p, C.c_void_p]
    return L


def ok(e):
    assert e.error_code == 0, (e.error_code, e.detail)


def frames(w, h, pinned):
    """smooth P010 (HLG, BT.2100) and YUV420 (BT.709) intents as uint8 tensors: pinned host or device memory"""
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    luma = (0.5 + 0.4 * np.sin(xx / 97.0) * np.cos(yy / 61.0))
    p010 = np.concatenate([(64 + luma * 876).astype(np.uint16).ravel(),
                           np.full(w * h // 2, 512, np.uint16)]) << 6
    yuv = np.concatenate([(16 + luma * 219).astype(np.uint8).ravel(), np.full(w * h // 2, 128, np.uint8)])
    th, ts = torch.from_numpy(p010.view(np.uint8).copy()), torch.from_numpy(yuv.copy())
    if pinned:
        return th.pin_memory(), ts.pin_memory()
    return th.cuda(), ts.cuda()


def descs(th, ts, w, h):
    hdr = A.raw_image(A.FMT_P010, A.CG_BT2100, A.CT_HLG, A.CR_LIMITED, w, h, [], [])
    hdr.planes[0], hdr.planes[1] = th.data_ptr(), th.data_ptr() + w * h * 2
    hdr.stride[0] = hdr.stride[1] = w
    sdr = A.raw_image(A.FMT_YUV420, A.CG_BT709, A.CT_SRGB, A.CR_FULL, w, h, [], [])
    sdr.planes[0], sdr.planes[1], sdr.planes[2] = ts.data_ptr(), ts.data_ptr() + w * h, ts.data_ptr() + w * h * 5 // 4
    sdr.stride[0], sdr.stride[1], sdr.stride[2] = w, w // 2, w // 2
    return hdr, sdr


def host_encode(L, hdr, sdr):
    enc = C.c_void_p(L.uhdr_create_encoder())
    try:
        ok(L.uhdr_enc_set_raw_image(enc, C.byref(hdr), A.HDR_IMG))
        ok(L.uhdr_enc_set_raw_image(enc, C.byref(sdr), A.SDR_IMG))
        ok(L.uhdr_encode(enc))
        o = L.uhdr_get_encoded_stream(enc).contents
        return C.string_at(o.data, o.data_sz)
    finally:
        L.uhdr_release_encoder(enc)


def dev_encode(L, hdr, sdr, out, stream):
    n = C.c_size_t()
    cfg = A.default_gm_config()
    rc = L.uhdr_b200_encode_dev(C.byref(hdr), C.byref(sdr), C.byref(cfg), 95, None, 0, out.ctypes.data, out.size,
                                C.byref(n), stream)
    assert rc == 0, L.uhdr_b200_last_error()
    return n.value


def bench_decode(L, repeats):
    w, h = 7680, 4320
    th, ts = frames(w, h, pinned=True)
    hdr, sdr = descs(th, ts, w, h)
    data = host_encode(L, hdr, sdr)
    buf = np.frombuffer(data, np.uint8).copy()
    dest_t = torch.empty(w * h * 8, dtype=torch.uint8, device="cuda")
    dest = A.raw_image(A.FMT_RGBAF16, -1, -1, -1, w, h, [], [])
    dest.planes[0], dest.stride[0] = dest_t.data_ptr(), w
    st = torch.cuda.Stream()
    dec = C.c_void_p(L.uhdr_create_decoder())

    def host_call():
        L.uhdr_reset_decoder(dec)
        ci = A.CompressedImage(buf.ctypes.data, buf.size, buf.size, -1, -1, -1)
        ok(L.uhdr_dec_set_image(dec, C.byref(ci)))
        ok(L.uhdr_dec_set_out_img_format(dec, A.FMT_RGBAF16))
        ok(L.uhdr_dec_set_out_color_transfer(dec, A.CT_LINEAR))
        t0 = time.perf_counter()
        ok(L.uhdr_decode(dec))
        assert L.uhdr_get_decoded_image(dec)
        return time.perf_counter() - t0

    def dev_call():
        t0 = time.perf_counter()
        rc = L.uhdr_b200_decode_dev(buf.ctypes.data, buf.size, A.CT_LINEAR, A.FLT_MAX, C.byref(dest), None, None,
                                    st.cuda_stream)
        st.synchronize()
        assert rc == 0, L.uhdr_b200_last_error()
        return time.perf_counter() - t0

    for _ in range(2):
        host_call(), dev_call()
    per = {"host": [], "dev": []}
    for _ in range(repeats):
        for _ in range(5):
            per["host"].append(host_call())
            per["dev"].append(dev_call())
    L.uhdr_release_decoder(dec)
    return {k: {"median_ms": round(float(np.median(v)) * 1e3, 3), "min_ms": round(min(v) * 1e3, 3),
                "max_ms": round(max(v) * 1e3, 3)} for k, v in per.items()}


def bench_encode(L, threads, frames_per_thread):
    w, h = 3840, 2160
    res = {}
    for kind in ("host", "dev"):
        bufs = [frames(w, h, pinned=(kind == "host")) for _ in range(threads)]
        outs = [np.zeros(w * h * 6, np.uint8) for _ in range(threads)]
        sizes = [[] for _ in range(threads)]
        barrier = threading.Barrier(threads + 1)

        def work(i):
            torch.cuda.set_device(0)
            hdr, sdr = descs(*bufs[i], w, h)
            st = torch.cuda.Stream()
            run = (lambda: len(host_encode(L, hdr, sdr))) if kind == "host" else \
                (lambda: dev_encode(L, hdr, sdr, outs[i], st.cuda_stream))
            run()     # warm-up: per-thread workspaces
            barrier.wait()
            for _ in range(frames_per_thread):
                sizes[i].append(run())
            barrier.wait()

        th = [threading.Thread(target=work, args=(i,)) for i in range(threads)]
        for t in th:
            t.start()
        barrier.wait()
        t0 = time.perf_counter()
        barrier.wait()
        dt = time.perf_counter() - t0
        for t in th:
            t.join()
        res[kind] = round(threads * frames_per_thread * w * h / dt / 1e9, 2)
    return res


def bench_staging(L, frames_per_arm, repeats):
    """Display-P3 SDR planes read in place vs staged; one thread, alternating arms -> GPix/s per arm (median).
    Both arms keep every plane 16-byte aligned with strides a multiple of 4 pixels, so the gain-map kernels are the
    same; only the staged arm's 4-pixel pitch tail (rows not 8-byte multiples) sends its planes through the copy."""
    w, h = 3840, 2160
    th, ts = frames(w, h, pinned=False)
    out = np.zeros(w * h * 6, np.uint8)
    st = torch.cuda.Stream()
    arms, keep = {}, []
    for name, pad in (("in_place", 0), ("staged", 4)):
        hdr, sdr = descs(th, ts, w, h)
        sdr.cg = A.CG_P3
        for i, (pw, ph, off) in enumerate(((w, h, 0), (w // 2, h // 2, w * h), (w // 2, h // 2, w * h * 5 // 4))):
            t = torch.zeros(ph, pw + pad, dtype=torch.uint8, device="cuda")
            t[:, :pw] = ts[off:off + pw * ph].view(ph, pw)
            keep.append(t)
            sdr.planes[i], sdr.stride[i] = t.data_ptr(), pw + pad
        arms[name] = (hdr, sdr)
    torch.cuda.synchronize()
    sizes = {k: dev_encode(L, *v, out, st.cuda_stream) for k, v in arms.items()}
    assert sizes["in_place"] == sizes["staged"]
    rates = {k: [] for k in arms}
    for _ in range(repeats):
        for k, (hdr, sdr) in arms.items():
            t0 = time.perf_counter()
            for _ in range(frames_per_arm):
                dev_encode(L, hdr, sdr, out, st.cuda_stream)
            rates[k].append(frames_per_arm * w * h / (time.perf_counter() - t0) / 1e9)
    return {k: round(float(np.median(v)), 2) for k, v in rates.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--frames", type=int, default=16)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_dev_codec: no CUDA device")
    name, power = gpu_card()
    print(f"gpu: {name}, power limit {power}", flush=True)
    L = load()
    out = {"gpu": name, "power_limit": power, "decode_8k_f16": bench_decode(L, args.repeats)}
    for n in (1, 8):
        out[f"encode_4k_api1_gpix_s_{n}t"] = bench_encode(L, n, args.frames)
    out["encode_4k_p3_sdr_gpix_s_1t"] = bench_staging(L, args.frames, args.repeats)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
