"""Ladder transcoding: one uhdr_b200_transcode_ladder call against a loop of uhdr_b200_transcode over the same rungs, host
bytes in and out, on one host thread.

Files: bench.py's 8K API-1 file (q95, map scale 1), a 4080x3072 file with map scale 4 and a 1920x1080 file.  Ladders:
"full+3" = k = 1 at quality 85 / 85 plus k = 2, 4, 8 at 80 / 70 (a recompressed copy, a preview and two thumbnails), and
"3 sizes" = k = 2, 4, 8 at 80 / 70; base_420 and keep_exif on in every rung.  Both arms' outputs are checked equal
before timing.  Per arm: the median wall clock per ladder over --iters iterations after 3 warm-ups, the two arms
alternated within each iteration, and the library's kernel launches per ladder.  Then, in a separate pass with kernel
timing on: k_idct<0>'s time per ladder ("idct_multi") against the summed k_idct<S> times ("idct_dequant", "idct_scaled") of the loop arm.  The
card's name and power limit are read in the same run.  One JSON line.

  python tools/bench_transcode_ladder.py [--iters 15]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import bench  # noqa: E402
import uhdr_testlib as T  # noqa: E402
from bench_restart import card_info  # noqa: E402
from libultrahdr_b200 import ctypes_api as A  # noqa: E402

LADDERS = {"full+3": [(1, 85, 85, 1, 1)] + [(k, 80, 70, 1, 1) for k in (2, 4, 8)],
           "3 sizes": [(k, 80, 70, 1, 1) for k in (2, 4, 8)]}


def make_file(lib, w, h, scale):
    p010, yuv = bench.make_frame(w, h, 0)
    hdr, sdr, _keep = bench.frame_descs(p010, yuv, w, h)
    return T.UhdrApi(lib).encode(hdr, sdr, quality=95, gm_quality=95, scale=scale)


class Ladder:
    """one file, its rungs, an output buffer per rung for each arm"""

    def __init__(self, data, cfgs):
        n = len(cfgs)
        self.src = np.frombuffer(data, np.uint8).copy()
        self.cap = self.src.size * 2 + (1 << 20)
        self.cfgs = [A.TranscodeConfig(*c) for c in cfgs]
        self.loop_out = [np.zeros(self.cap, np.uint8) for _ in range(n)]
        self.sizes = (C.c_size_t * n)()
        self.lad_out = [np.zeros(self.cap, np.uint8) for _ in range(n)]
        self.rungs = (A.TranscodeRung * n)(*[A.TranscodeRung(c, o.ctypes.data, self.cap, 0, -1)
                                             for c, o in zip(self.cfgs, self.lad_out)])

    def loop(self, lib):
        for i, cfg in enumerate(self.cfgs):
            rc = lib.uhdr_b200_transcode(self.src.ctypes.data, self.src.size, C.byref(cfg), self.loop_out[i].ctypes.data,
                                         self.cap, C.cast(C.byref(self.sizes, i * C.sizeof(C.c_size_t)),
                                                          C.POINTER(C.c_size_t)))
            assert rc == 0, lib.uhdr_b200_last_error()

    def ladder(self, lib):
        rc = lib.uhdr_b200_transcode_ladder(self.src.ctypes.data, self.src.size, self.rungs, len(self.cfgs))
        assert rc == 0, lib.uhdr_b200_last_error()

    def equal(self):
        return all(bytes(self.loop_out[i][:self.sizes[i]]) == bytes(self.lad_out[i][:self.rungs[i].out_size])
                   for i in range(len(self.cfgs)))


def kernel_ms(lib, fn, reps):
    """per call: {kernel name: total ms} from the library's kernel timing over reps calls"""
    buf = C.create_string_buffer(1 << 16)
    lib.uhdr_b200_set_kernel_timing(1)
    lib.uhdr_b200_kernel_timing_report(buf, len(buf), 1)
    try:
        for _ in range(reps):
            fn(lib)
        lib.uhdr_b200_kernel_timing_report(buf, len(buf), 1)
    finally:
        lib.uhdr_b200_set_kernel_timing(0)
    out = {}
    for line in buf.value.decode().splitlines():
        f = line.split()
        if len(f) >= 3 and f[1].isdigit():
            out[f[0]] = float(f[2]) / reps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=15)
    a = ap.parse_args()
    gpu = T.Gpu()
    lib = A.declare_transcode_ladder(A.declare_transcode(gpu.lib))
    lib.uhdr_b200_last_error.restype = C.c_char_p
    lib.uhdr_b200_kernel_launches.restype = C.c_ulonglong
    lib.uhdr_b200_kernel_timing_report.argtypes = [C.c_char_p, C.c_size_t, C.c_int]
    files = {"8K 7680x4320 s1": make_file(lib, bench.W8K, bench.H8K, 1),
             "4080x3072 s4": make_file(lib, 4080, 3072, 4),
             "1920x1080 s1": make_file(lib, 1920, 1080, 1)}
    res = {"card": card_info(), "iters": a.iters}
    for fname, data in files.items():
        for lname, cfgs in LADDERS.items():
            L = Ladder(data, cfgs)
            L.loop(lib)
            L.ladder(lib)
            assert L.equal(), ("ladder output differs from the single calls'", fname, lname)
            for _ in range(2):
                L.loop(lib)
                L.ladder(lib)
            ts = {"loop": [], "ladder": []}
            launches = {"loop": 0, "ladder": 0}
            for it in range(a.iters):
                order = (("loop", L.loop), ("ladder", L.ladder)) if it % 2 == 0 else (("ladder", L.ladder), ("loop", L.loop))
                for arm, fn in order:
                    l0 = lib.uhdr_b200_kernel_launches()
                    t0 = time.perf_counter()
                    fn(lib)
                    ts[arm].append(time.perf_counter() - t0)
                    launches[arm] += lib.uhdr_b200_kernel_launches() - l0
            assert L.equal()
            kl = kernel_ms(lib, L.ladder, 5)
            kp = kernel_ms(lib, L.loop, 5)
            idct_loop = sum(v for k, v in kp.items() if k.startswith("idct_dequant") or k.startswith("idct_scaled"))
            loop_ms, lad_ms = float(np.median(ts["loop"])) * 1e3, float(np.median(ts["ladder"])) * 1e3
            res["%s, %s" % (fname, lname)] = {
                "rungs": len(cfgs), "bytes": [int(L.sizes[i]) for i in range(len(cfgs))],
                "loop_ms": round(loop_ms, 3), "ladder_ms": round(lad_ms, 3), "speedup": round(loop_ms / lad_ms, 2),
                "loop_spread_ms": [round(min(ts["loop"]) * 1e3, 3), round(max(ts["loop"]) * 1e3, 3)],
                "ladder_spread_ms": [round(min(ts["ladder"]) * 1e3, 3), round(max(ts["ladder"]) * 1e3, 3)],
                "launches_loop": launches["loop"] / a.iters, "launches_ladder": launches["ladder"] / a.iters,
                "idct_multi_ms": round(kl.get("idct_multi", 0.0), 4), "idct_loop_ms": round(idct_loop, 4),
            }
            del L
    res["how"] = ("uhdr_b200_transcode_ladder vs a loop of uhdr_b200_transcode over the same rungs, one host thread, host "
                  "bytes in and out, base_420 and keep_exif on; median wall clock of %d alternated iterations after 3 "
                  "warm-ups; kernel times from the library's CUDA-event kernel timing over 5 further calls per arm"
                  % a.iters)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
