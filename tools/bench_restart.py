"""uhdr_decode of an 8K JPEG/R whose primary and gain-map JPEGs carry restart intervals, with the device and the host
entropy decoder and with the reference's CPU decode; prints one JSON line.

  python tools/bench_restart.py

The file is bench.py's 8K decode input (frame 7, API-1 defaults) with both JPEGs re-encoded by Pillow's libjpeg-turbo
(same quantisation tables, sampling and ICC profile) plus restart markers, reassembled through API-4.  Two intervals:
24 MCUs, what Apple's gain-map photos use, and one MCU row, the other common choice of camera encoders.  The card's
name and power limit are read in the same run."""
import ctypes as C
import io
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
from PIL.JpegImagePlugin import JpegImageFile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import uhdr_testlib as T  # noqa: E402
from libultrahdr_b200 import ctypes_api as A  # noqa: E402

W, H = bench.W8K, bench.H8K


def card_info():
    try:
        o = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=10).stdout.strip().splitlines()
        name, limit = [x.strip() for x in o[0].split(",")]
        return {"name": name, "power_limit": limit}
    except Exception as e:  # noqa: BLE001
        return {"error": repr(e)}


def jpegr_parts(lib, data):
    """-> (primary JPEG, gain-map JPEG, GainmapMetadata) of a JPEG/R, through uhdr_dec_probe"""
    lib.uhdr_dec_probe.restype = A.ErrorInfo
    for f in ("uhdr_dec_get_base_image", "uhdr_dec_get_gainmap_image"):
        getattr(lib, f).restype = C.POINTER(A.MemBlock)
    buf = np.frombuffer(data, np.uint8).copy()
    ci = A.CompressedImage(buf.ctypes.data, len(data), len(data), -1, -1, -1)
    dec = C.c_void_p(lib.uhdr_create_decoder())
    try:
        assert lib.uhdr_dec_set_image(dec, C.byref(ci)).error_code == 0
        e = lib.uhdr_dec_probe(dec)
        assert e.error_code == 0, e.detail
        parts = [C.string_at(b.contents.data, b.contents.data_sz)
                 for b in (lib.uhdr_dec_get_base_image(dec), lib.uhdr_dec_get_gainmap_image(dec))]
        md = A.GainmapMetadata.from_buffer_copy(bytes(lib.uhdr_dec_get_gainmap_metadata(dec).contents))
        return parts[0], parts[1], md
    finally:
        lib.uhdr_release_decoder(dec)


def assemble_api4(lib, base, gm, md):
    """uhdr_encode API-4: compressed base (BT.709) + compressed gain map + metadata -> JPEG/R"""
    lib.uhdr_enc_set_compressed_image.restype = A.ErrorInfo
    lib.uhdr_enc_set_gainmap_image.restype = A.ErrorInfo
    bb, gb = np.frombuffer(base, np.uint8).copy(), np.frombuffer(gm, np.uint8).copy()
    bi = A.CompressedImage(bb.ctypes.data, len(base), len(base), A.CG_BT709, -1, -1)
    gi = A.CompressedImage(gb.ctypes.data, len(gm), len(gm), -1, -1, -1)
    enc = C.c_void_p(lib.uhdr_create_encoder())
    try:
        assert lib.uhdr_enc_set_compressed_image(enc, C.byref(bi), A.BASE_IMG).error_code == 0
        assert lib.uhdr_enc_set_gainmap_image(enc, C.byref(gi), C.byref(md)).error_code == 0
        e = lib.uhdr_encode(enc)
        assert e.error_code == 0, e.detail
        o = lib.uhdr_get_encoded_stream(enc).contents
        return C.string_at(o.data, o.data_sz)
    finally:
        lib.uhdr_release_encoder(enc)


def with_restarts(jpg, restart):
    src, b = JpegImageFile(io.BytesIO(jpg)), io.BytesIO()
    src.save(b, "JPEG", quality="keep", subsampling="keep", icc_profile=src.info.get("icc_profile"), **restart)
    return b.getvalue()


def timed_decode(lib, data, n):
    """uhdr_dec_set_image + uhdr_decode + uhdr_get_decoded_image -> 64bppRGBAHalfFloat, a new handle per call;
    -> (best, median) seconds"""
    buf = np.frombuffer(data, np.uint8).copy()
    ci = A.CompressedImage(buf.ctypes.data, len(data), len(data), -1, -1, -1)
    ts = []
    for _ in range(n):
        dec = C.c_void_p(lib.uhdr_create_decoder())
        t0 = time.perf_counter()
        assert lib.uhdr_dec_set_image(dec, C.byref(ci)).error_code == 0
        e = lib.uhdr_decode(dec)
        assert e.error_code == 0, e.detail
        assert lib.uhdr_get_decoded_image(dec).contents.w == W
        ts.append(time.perf_counter() - t0)
        lib.uhdr_release_decoder(dec)
    return min(ts), sorted(ts)[len(ts) // 2]


def ms(t):
    return {"ms": round(t[0] * 1e3, 2), "ms_median": round(t[1] * 1e3, 2), "mpix_s": round(W * H / 1e6 / t[0], 1)}


def main():
    api, lib = bench.load_api(T.GPU_SO)
    lib.uhdr_b200_entropy_decoder_stats.restype = None
    ref = bench.load_api(T.REF_SO)[1] if T.have_ref() else None
    p, y = bench.make_frame(W, H, 7)
    hdr, sdr, _keep = bench.frame_descs(p, y, W, H)
    plain = api.encode(hdr, sdr)
    base, gm, md = jpegr_parts(lib, plain)
    res = {"card": card_info(), "image": "%dx%d" % (W, H)}
    timed_decode(lib, plain, 2)   # warm-up: module load, arena growth
    res["no_restart_markers"] = {"device_decoder": ms(timed_decode(lib, plain, 6))}
    if ref is not None:
        res["no_restart_markers"]["cpu_reference_ms"] = round(timed_decode(ref, plain, 1)[0] * 1e3, 1)
    for name, restart in (("ri_24_mcus", {"restart_marker_blocks": 24}), ("ri_1_mcu_row", {"restart_marker_rows": 1})):
        data = assemble_api4(lib, with_restarts(base, restart), with_restarts(gm, restart), md)
        st0, st1 = (C.c_ulonglong * 3)(), (C.c_ulonglong * 3)()
        prev = lib.uhdr_b200_set_entropy_decoder(2)
        try:
            timed_decode(lib, data, 1)
            lib.uhdr_b200_entropy_decoder_stats(st0)
            dev = timed_decode(lib, data, 6)
            lib.uhdr_b200_entropy_decoder_stats(st1)
            px_dev = api.decode(data)
            lib.uhdr_b200_set_entropy_decoder(1)
            host = timed_decode(lib, data, 3)
            px_host = api.decode(data)
        finally:
            lib.uhdr_b200_set_entropy_decoder(prev)
        r = {"stream_bytes": len(data), "rst_markers": len(re.findall(rb"\xff[\xd0-\xd7]", data)),
             "device_decoder": ms(dev), "host_decoder": ms(host),
             "entropy_decoder": {"device_scans": int(st1[0] - st0[0]), "handed_to_host": int(st1[1] - st0[1])},
             "device_equals_host_pixels": bool(np.array_equal(px_dev[0], px_host[0]) and np.array_equal(px_dev[1], px_host[1]))}
        del px_dev, px_host
        if ref is not None:
            r["cpu_reference_ms"] = round(timed_decode(ref, data, 1)[0] * 1e3, 1)
        res[name] = r
    res["how"] = ("best / median of 6 calls (device entropy decoder), 3 (host, uhdr_b200_set_entropy_decoder(1)), 1 (reference "
                  "on the host); compressed stream and pixels in host memory, one handle at a time")
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
