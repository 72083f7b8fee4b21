"""Reduced-size decoding: uhdr_b200_decode_scaled_dev at k = 1, 2, 4, 8 into device memory (RGBA half float), on
bench.py's 8K input (frame 7, API-1 defaults) and on a 4080x3072 file (map scale 4, a non-integer map ratio after
scaling).  Per k: median and best of >= 20 calls, each followed by a stream synchronise; then the block-stage kernel
times from the library's kernel-timing report (CUDA events): k_idct<8> ("idct_dequant") against the reduced
IDCT k_idct<4 / 2 / 1> ("idct_scaled"), and the colour conversion and apply kernels.  On this device-output path the report holds the
gain-map JPEG's kernels, which run on the codec's second stream; the primary JPEG's are not collected.  The card's name and power limit are read
in the same run.  Prints one JSON line.

  python tools/bench_scaled_decode.py [--calls 20]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import uhdr_testlib as T  # noqa: E402
from bench_restart import card_info  # noqa: E402
from libultrahdr_b200 import ctypes_api as A  # noqa: E402


def make_file(api, w, h, frame, scale):
    p, y = bench.make_frame(w, h, frame)
    hdr, sdr, _keep = bench.frame_descs(p, y, w, h)
    return api.encode(hdr, sdr, scale=scale)


def dims(lib, buf, k):
    d = [C.c_uint() for _ in range(4)]
    assert lib.uhdr_b200_scaled_dims(buf.ctypes.data, buf.size, k, *[C.byref(x) for x in d]) == 0
    return [x.value for x in d]


def run(lib, data, k, calls):
    buf = np.frombuffer(data, np.uint8).copy()
    w, h, gw, gh = dims(lib, buf, k)
    dst = torch.empty(w * h * 8, dtype=torch.uint8, device="cuda")
    desc = A.raw_image(A.FMT_RGBAF16, -1, -1, -1, w, h, [], [])
    desc.planes[0], desc.stride[0] = dst.data_ptr(), w
    st = torch.cuda.Stream()

    def call():
        rc = lib.uhdr_b200_decode_scaled_dev(buf.ctypes.data, buf.size, k, A.CT_LINEAR, A.FLT_MAX, C.byref(desc), None,
                                             None, st.cuda_stream)
        assert rc == 0, lib.uhdr_b200_last_error()
        st.synchronize()

    for _ in range(3):
        call()
    ts = []
    for _ in range(calls):
        t0 = time.perf_counter()
        call()
        ts.append(time.perf_counter() - t0)
    ts.sort()
    # kernel times on a separate set of calls: the event pairs around every launch change the timing above
    lib.uhdr_b200_set_kernel_timing(1)
    bench.kernel_report(lib)
    n = 5
    for _ in range(n):
        call()
    rep = bench.kernel_report(lib)
    lib.uhdr_b200_set_kernel_timing(0)
    kern = {name: round(v[1] / n, 4) for name, v in rep.items()
            if name.startswith(("idct", "huff_dec", "ycc", "apply"))}
    return {"out": "%dx%d" % (w, h), "map": "%dx%d" % (gw, gh), "ms_median": round(ts[len(ts) // 2] * 1e3, 3),
            "ms_best": round(ts[0] * 1e3, 3), "kernel_ms_per_call": kern}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    api, lib = bench.load_api(T.GPU_SO)
    A.declare_scaled_decode(lib)
    lib.uhdr_b200_last_error.restype = C.c_char_p
    res = {"card": card_info()}
    files = {"8k_bench_input": make_file(api, bench.W8K, bench.H8K, 7, 1), "4080x3072_map_scale_4": make_file(api, 4080, 3072, 3, 4)}
    for name, data in files.items():
        res[name] = {"k%d" % k: run(lib, data, k, max(20, args.calls)) for k in A.SCALE_DENOMS}
    res["how"] = ("uhdr_b200_decode_scaled_dev -> RGBA half float in device memory on a torch stream, median / best of the "
                  "timed calls, each followed by a stream synchronise (compressed file in host memory); kernel times: "
                  "CUDA-event totals per call over 5 further calls with kernel timing on")
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
