"""Batched decoding: uhdr_b200_decode_batch_dev against a loop of uhdr_b200_decode_scaled_dev over the same files,
into device memory (RGBA half float, linear), on one host thread and on eight (each thread with its own stream and
1/8 of the files).  Workloads: 256 copies of a 4080x3072 file (bench.py's frame 3, map scale 4) at k = 8 and k = 1,
and 32 of bench.py's 8K files at k = 1.  Per arm: files/s from the median of 5 timed repetitions (host clock around
work that ends in a stream synchronise, after 2 warm-up repetitions), and the library's kernel launches per file.
Host waits are structural: the loop waits 2 per JPEG plus 1 per 16 relaxation rounds (4+ per file); a batch waits
1 per 16 rounds for all its scans plus 1.  The card's name and power limit are read in the same run.  One JSON line.

  python tools/bench_decode_batch.py [--reps 5]
"""
import argparse
import ctypes as C
import json
import os
import sys
import threading
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


class Files:
    """n files with their device destinations at 1/k"""

    def __init__(self, lib, datas, k):
        self.k, self.bufs = k, [np.frombuffer(d, np.uint8).copy() for d in datas]
        self.descs, self.keep = [], []
        for b in self.bufs:
            d = [C.c_uint() for _ in range(4)]
            assert lib.uhdr_b200_scaled_dims(b.ctypes.data, b.size, k, *[C.byref(x) for x in d]) == 0
            w, h = d[0].value, d[1].value
            t = torch.empty(w * h * 8, dtype=torch.uint8, device="cuda")
            desc = A.raw_image(A.FMT_RGBAF16, -1, -1, -1, w, h, [], [])
            desc.planes[0], desc.stride[0] = t.data_ptr(), w
            self.descs.append(desc)
            self.keep.append(t)
        self.items = (A.DecodeItem * len(self.bufs))(*[A.DecodeItem(b.ctypes.data, b.size, C.pointer(d), None, None, 0)
                                                       for b, d in zip(self.bufs, self.descs)])


def arm_loop(lib, f, lo, hi, st):
    for i in range(lo, hi):
        b = f.bufs[i]
        rc = lib.uhdr_b200_decode_scaled_dev(b.ctypes.data, b.size, f.k, A.CT_LINEAR, A.FLT_MAX, C.byref(f.descs[i]), None,
                                             None, st.cuda_stream)
        assert rc == 0, lib.uhdr_b200_last_error()
    st.synchronize()


def arm_batch(lib, f, lo, hi, st):
    items = C.cast(C.byref(f.items, lo * C.sizeof(A.DecodeItem)), C.POINTER(A.DecodeItem))
    rc = lib.uhdr_b200_decode_batch_dev(items, hi - lo, f.k, A.CT_LINEAR, A.FLT_MAX, st.cuda_stream)
    assert rc == 0, lib.uhdr_b200_last_error()
    st.synchronize()


def timed(lib, f, arm, threads, reps):
    n = len(f.bufs)
    streams = [torch.cuda.Stream() for _ in range(threads)]
    parts = [(n * t // threads, n * (t + 1) // threads) for t in range(threads)]

    def once():
        if threads == 1:
            arm(lib, f, 0, n, streams[0])
            return
        th = [threading.Thread(target=arm, args=(lib, f, lo, hi, s)) for (lo, hi), s in zip(parts, streams)]
        for x in th:
            x.start()
        for x in th:
            x.join()

    for _ in range(2):
        once()
    torch.cuda.synchronize()
    l0 = lib.uhdr_b200_kernel_launches()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        once()
        ts.append(time.perf_counter() - t0)
    launches = (lib.uhdr_b200_kernel_launches() - l0) / (reps * n)
    med = float(np.median(ts))
    return {"files_per_s": round(n / med, 1), "ms_per_call": round(med * 1e3, 3), "launches_per_file": round(launches, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    gpu = T.Gpu()
    lib = A.declare_decode_batch(A.declare_scaled_decode(gpu.lib))
    lib.uhdr_b200_last_error.restype = C.c_char_p
    lib.uhdr_b200_kernel_launches.restype = C.c_ulonglong
    api = T.UhdrApi(lib)
    f4k = make_file(api, 4080, 3072, 3, 4)
    f8k = make_file(api, bench.W8K, bench.H8K, 7, 1)
    res = {"card": card_info()}
    for name, data, n, k in (("4080x3072_k8", f4k, 256, 8), ("4080x3072_k1", f4k, 256, 1), ("8k_k1", f8k, 32, 1)):
        f = Files(lib, [data] * n, k)
        row = {}
        for threads in (1, 8):
            for arm_name, arm in (("loop", arm_loop), ("batch", arm_batch)):
                row["%s_%dt" % (arm_name, threads)] = timed(lib, f, arm, threads, a.reps)
        res[name] = row
        del f
        torch.cuda.empty_cache()
    res["how"] = ("uhdr_b200_decode_batch_dev vs a loop of uhdr_b200_decode_scaled_dev, RGBA half float in device memory, "
                  "median of %d repetitions after 2 warm-ups, each ending in a stream synchronise" % a.reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
