"""Resident rendering against a decode per frame, on bench.py's 8K JPEG/R (7680x4320, map scale 1, multichannel):
    python tools/bench_render.py [--iters N]

Median call times, each call followed by a stream synchronise, of
  * uhdr_b200_decode_dev to RGBA half float (what a viewer pays today for every re-render),
  * uhdr_b200_image_render_dev of the full frame, of a 1920x1080 viewport, and of the full frame at k = 4,
and their kernel times (CUDA events around each call on its stream, median).  Every render is checked equal to the
matching crop of a decode first.  The card's name and power limit are read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import uhdr_testlib as T  # noqa: E402
from libultrahdr_b200 import ctypes_api as A  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception as e:  # noqa: BLE001
        return repr(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_render needs a CUDA device")
    gpu = T.Gpu()
    lib = A.declare_resident_image(A.declare_scaled_decode(gpu.lib))
    lib.uhdr_b200_decode_dev.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_float] + [C.c_void_p] * 4
    lib.uhdr_b200_last_error.restype = C.c_char_p
    p8, y8 = bench.make_frame(bench.W8K, bench.H8K, 7)
    h8, s8, _k = bench.frame_descs(p8, y8, bench.W8K, bench.H8K)
    data = np.frombuffer(T.UhdrApi(gpu.lib).encode(h8, s8), np.uint8).copy()
    del p8, y8, h8, s8
    W, H = bench.W8K, bench.H8K
    st = torch.cuda.Stream()
    sp = st.cuda_stream

    def dest(w, h):
        buf = torch.empty((h, w * 8), dtype=torch.uint8, device="cuda")
        d = A.raw_image(A.FMT_RGBAF16, -1, -1, -1, w, h, [], [])
        d.planes[0], d.stride[0] = buf.data_ptr(), w
        return buf, d

    full, dfull = dest(W, H)
    boost = 4.0

    def decode():
        rc = lib.uhdr_b200_decode_dev(data.ctypes.data, data.size, A.CT_LINEAR, boost, C.byref(dfull), None, None, sp)
        assert rc == 0, lib.uhdr_b200_last_error()

    images = {}
    for k in (1, 4):
        h = C.c_void_p()
        assert lib.uhdr_b200_image_open_dev(data.ctypes.data, data.size, k, C.byref(h)) == 0, lib.uhdr_b200_last_error()
        images[k] = h
    nbytes = C.c_size_t()
    lib.uhdr_b200_image_info(images[1], None, None, None, None, None, C.byref(nbytes))
    vp_x, vp_y = 2880, 1620
    cases = {"decode_dev_full": (None, (W, H), (0, 0), 1), "render_full": (images[1], (W, H), (0, 0), 1),
             "render_1920x1080": (images[1], (1920, 1080), (vp_x, vp_y), 1),
             "render_full_k4": (images[4], (W // 4, H // 4), (0, 0), 4)}
    # correctness of what is timed: each render equals the crop of a decode at the same k
    decode()
    st.synchronize()
    ref1 = full.clone()
    q = torch.empty((H // 4, W // 4 * 8), dtype=torch.uint8, device="cuda")
    dq = A.raw_image(A.FMT_RGBAF16, -1, -1, -1, W // 4, H // 4, [], [])
    dq.planes[0], dq.stride[0] = q.data_ptr(), W // 4
    assert lib.uhdr_b200_decode_scaled_dev(data.ctypes.data, data.size, 4, A.CT_LINEAR, boost, C.byref(dq), None, None,
                                           sp) == 0
    st.synchronize()
    outs = {}
    for name, (img, (w, h), (x, y), k) in cases.items():
        if img is None:
            continue
        buf, d = dest(w, h)
        outs[name] = (buf, d)
        assert lib.uhdr_b200_image_render_dev(img, A.CT_LINEAR, boost, x, y, C.byref(d), sp) == 0
        st.synchronize()
        want = (q if k == 4 else ref1)[y:y + h, x * 8:(x + w) * 8]
        assert torch.equal(buf, want), name

    def call(name):
        img, _wh, (x, y), _k = cases[name]
        if img is None:
            return decode()
        _buf, d = outs[name]
        assert lib.uhdr_b200_image_render_dev(img, A.CT_LINEAR, boost, x, y, C.byref(d), sp) == 0

    res = {}
    for name in cases:
        for _ in range(5):
            call(name)
        st.synchronize()
        wall, dev = [], []
        for _ in range(args.iters):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record(st)
            call(name)
            e1.record(st)
            st.synchronize()
            wall.append((time.perf_counter() - t0) * 1e3)
            dev.append(e0.elapsed_time(e1))
        res[name] = {"call_ms_median": round(float(np.median(wall)), 4), "call_ms_min": round(float(np.min(wall)), 4),
                     "stream_ms_median": round(float(np.median(dev)), 4)}
    # kernel time of the resident renders alone: the profiler's device-side record of the apply kernel
    from torch.profiler import ProfilerActivity, profile
    kern = {}
    for name in ("render_full", "render_1920x1080", "render_full_k4"):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                call(name)
            st.synchronize()
        ev = [e for e in prof.events() if e.device_type.name == "CUDA" and "apply" in e.name]
        kern[name] = {"kernel": ev[0].name.split("<")[0] if ev else None,
                      "kernel_ms_median": round(float(np.median([getattr(e, "device_time", None) or e.cuda_time for e in ev])) / 1e3, 4) if ev else None}
    for k, h in images.items():
        assert lib.uhdr_b200_image_release(h) == 0
    base = res["decode_dev_full"]["call_ms_median"]
    print(json.dumps({
        "card": card(), "file": "bench.py 8K JPEG/R, %d bytes" % data.size, "output": "RGBA half float, linear, boost 4",
        "resident_device_bytes": nbytes.value, "calls": res, "kernels": kern,
        "speedup_full_render_vs_decode_dev": round(base / res["render_full"]["call_ms_median"], 2),
        "speedup_viewport_vs_decode_dev": round(base / res["render_1920x1080"]["call_ms_median"], 2),
    }, indent=1))


if __name__ == "__main__":
    main()
