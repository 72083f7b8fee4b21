"""Batched transcoding: uhdr_b200_transcode_batch against a loop of uhdr_b200_transcode over the same files, host bytes in
and out, on one host thread and on eight (each thread transcodes its own 1/8 of the files, the batch arm in one call per
thread).  Workloads: 256 copies of a 4080x3072 file (bench.py's frame 3, map scale 4) at k = 8 and at k = 4, 64 of a
1920x1080 file at k = 1, and 16 of bench.py's 8K files at k = 2; base_420 and keep_exif on, qualities 85 / 85.  Every
arm's output is checked equal to the single call's before it is timed.  Per arm: files/s from the median of 5 timed
repetitions after 2 warm-up repetitions, and the library's kernel launches per file.  The card's name and power limit
are read in the same run.  One JSON line.

  python tools/bench_transcode_batch.py [--reps 5]
"""
import argparse
import ctypes as C
import json
import os
import sys
import threading
import time

import numpy as np

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
    """n copies of one file with an output buffer each"""

    def __init__(self, data, n, cfg):
        self.cfg = cfg
        self.src = np.frombuffer(data, np.uint8).copy()
        self.cap = self.src.size * 2 + (1 << 20)
        self.outs = [np.zeros(self.cap, np.uint8) for _ in range(n)]
        self.sizes = (C.c_size_t * n)()
        self.items = (A.TranscodeItem * n)(*[A.TranscodeItem(self.src.ctypes.data, self.src.size, o.ctypes.data, self.cap,
                                                             0, -1) for o in self.outs])

    def result(self, i, batch):
        m = self.items[i].out_size if batch else self.sizes[i]
        return bytes(self.outs[i][:m])


def arm_loop(lib, f, lo, hi):
    for i in range(lo, hi):
        rc = lib.uhdr_b200_transcode(f.src.ctypes.data, f.src.size, C.byref(f.cfg), f.outs[i].ctypes.data, f.cap,
                                     C.cast(C.byref(f.sizes, i * C.sizeof(C.c_size_t)), C.POINTER(C.c_size_t)))
        assert rc == 0, lib.uhdr_b200_last_error()


def arm_batch(lib, f, lo, hi):
    items = C.cast(C.byref(f.items, lo * C.sizeof(A.TranscodeItem)), C.POINTER(A.TranscodeItem))
    rc = lib.uhdr_b200_transcode_batch(items, hi - lo, C.byref(f.cfg))
    assert rc == 0, lib.uhdr_b200_last_error()


def run(lib, f, arm, threads):
    n = len(f.outs)
    if threads == 1:
        arm(lib, f, 0, n)
        return
    th = [threading.Thread(target=arm, args=(lib, f, n * t // threads, n * (t + 1) // threads)) for t in range(threads)]
    for x in th:
        x.start()
    for x in th:
        x.join()


def timed(lib, f, arm, threads, reps, want):
    n = len(f.outs)
    for o in f.outs:
        o[:] = 0
    run(lib, f, arm, threads)
    batch = arm is arm_batch
    assert all(f.result(i, batch) == want for i in range(n)), "output differs from the single call's"
    run(lib, f, arm, threads)
    l0 = lib.uhdr_b200_kernel_launches()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        run(lib, f, arm, threads)
        ts.append(time.perf_counter() - t0)
    launches = (lib.uhdr_b200_kernel_launches() - l0) / (reps * n)
    med = float(np.median(ts))
    return {"files_per_s": round(n / med, 1), "ms_per_file": round(med * 1e3 / n, 3), "launches_per_file": round(launches, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    gpu = T.Gpu()
    lib = A.declare_transcode_batch(A.declare_transcode(gpu.lib))
    lib.uhdr_b200_last_error.restype = C.c_char_p
    lib.uhdr_b200_kernel_launches.restype = C.c_ulonglong
    api = T.UhdrApi(lib)
    f4k = make_file(api, 4080, 3072, 3, 4)
    fhd = make_file(api, 1920, 1080, 1, 1)
    f8k = make_file(api, bench.W8K, bench.H8K, 7, 1)
    res = {"card": card_info()}
    for name, data, n, k in (("4080x3072_k8", f4k, 256, 8), ("4080x3072_k4", f4k, 256, 4), ("1920x1080_k1", fhd, 64, 1),
                             ("8k_k2", f8k, 16, 2)):
        cfg = A.TranscodeConfig(k, 85, 85, 1, 1)
        one = Files(data, 1, cfg)
        arm_loop(lib, one, 0, 1)
        want = one.result(0, False)
        f = Files(data, n, cfg)
        row = {}
        for threads in (1, 8):
            for arm_name, arm in (("loop", arm_loop), ("batch", arm_batch)):
                row["%s_%dt" % (arm_name, threads)] = timed(lib, f, arm, threads, a.reps, want)
        for threads in (1, 8):
            row["speedup_%dt" % threads] = round(row["batch_%dt" % threads]["files_per_s"] /
                                                 row["loop_%dt" % threads]["files_per_s"], 2)
        res[name] = row
        del f
    res["how"] = ("uhdr_b200_transcode_batch vs a loop of uhdr_b200_transcode, host bytes in and out, base_420 and "
                  "keep_exif on, q 85 / 85, median of %d repetitions after 2 warm-ups (the first checked equal to the "
                  "single call)" % a.reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
