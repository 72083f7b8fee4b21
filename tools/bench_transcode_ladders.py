"""Ladders over many files: one uhdr_b200_transcode_ladders call against a loop of uhdr_b200_transcode_ladder calls over
the same files and rungs, host bytes in and out, on 1 and on 8 host threads (each thread its share of the files, its
own outputs and the library's per-thread codec).

Workloads: 256 4080x3072 files (map scale 4) with the "3 sizes" ladder, 64 1920x1080 files with "full+3", and 16 of
bench.py's 8K API-1 file (q95, map scale 1) with "3 sizes".  Ladders as in bench_transcode_ladder.py: "full+3" = k = 1
at quality 85 / 85 plus k = 2, 4, 8 at 80 / 70, "3 sizes" = k = 2, 4, 8 at 80 / 70; base_420 and keep_exif on in every
rung.  The files of a workload cycle through four seeds.  Both arms' outputs are checked byte-equal before timing.  Per
arm and thread count: files per second from the median of --reps repetitions (after one warm-up), the two arms
alternated within each repetition, and on one thread the library's kernel launches per file.  The card's name and
power limit are read in the same run.  One JSON line.

  python tools/bench_transcode_ladders.py [--reps 5]
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
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

import bench  # noqa: E402
import uhdr_testlib as T  # noqa: E402
from bench_restart import card_info  # noqa: E402
from libultrahdr_b200 import ctypes_api as A  # noqa: E402

LADDERS = {"full+3": [(1, 85, 85, 1, 1)] + [(k, 80, 70, 1, 1) for k in (2, 4, 8)],
           "3 sizes": [(k, 80, 70, 1, 1) for k in (2, 4, 8)]}
WORKLOADS = [("4080x3072 s4", 4080, 3072, 4, 256, "3 sizes"),
             ("1920x1080 s1", 1920, 1080, 1, 64, "full+3"),
             ("8K 7680x4320 s1", bench.W8K, bench.H8K, 1, 16, "3 sizes")]
SEEDS = 4


def make_file(lib, w, h, scale, seed):
    p010, yuv = bench.make_frame(w, h, seed)
    hdr, sdr, _keep = bench.frame_descs(p010, yuv, w, h)
    return T.UhdrApi(lib).encode(hdr, sdr, quality=95, gm_quality=95, scale=scale)


class Share:
    """one thread's files: per arm its own rung array and outputs; `files` for the one call"""

    def __init__(self, datas, cfgs):
        self.srcs = [np.frombuffer(d, np.uint8).copy() for d in datas]
        n = len(cfgs)
        self.out, self.rungs = {}, {}
        for arm in ("loop", "ladders"):
            outs, rungs = [], []
            for s in self.srcs:
                caps = [s.size * 2 // (c[0] * c[0]) + (1 << 20) for c in cfgs]
                o = [np.zeros(cap, np.uint8) for cap in caps]
                outs.append(o)
                rungs.append((A.TranscodeRung * n)(*[A.TranscodeRung(A.TranscodeConfig(*c), b.ctypes.data, cap, 0, -1)
                                                     for c, b, cap in zip(cfgs, o, caps)]))
            self.out[arm], self.rungs[arm] = outs, rungs
        self.n = n
        self.files = (A.TranscodeFile * len(self.srcs))(*[A.TranscodeFile(s.ctypes.data, s.size, r, n, -1)
                                                          for s, r in zip(self.srcs, self.rungs["ladders"])])

    def loop(self, lib):
        for s, r in zip(self.srcs, self.rungs["loop"]):
            rc = lib.uhdr_b200_transcode_ladder(s.ctypes.data, s.size, r, self.n)
            assert rc == 0, lib.uhdr_b200_last_error()

    def ladders(self, lib):
        rc = lib.uhdr_b200_transcode_ladders(self.files, len(self.srcs))
        assert rc == 0, lib.uhdr_b200_last_error()

    def equal(self):
        a, b = self.rungs["loop"], self.rungs["ladders"]
        return all(bytes(self.out["loop"][f][j][:a[f][j].out_size]) == bytes(self.out["ladders"][f][j][:b[f][j].out_size])
                   for f in range(len(self.srcs)) for j in range(self.n))


def run_threads(lib, shares, arm):
    """wall clock of every share's arm, one thread each (inline for one share)"""
    if len(shares) == 1:
        t0 = time.perf_counter()
        getattr(shares[0], arm)(lib)
        return time.perf_counter() - t0
    errors = []

    def body(s):
        try:
            getattr(s, arm)(lib)
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    th = [threading.Thread(target=body, args=(s,)) for s in shares]
    t0 = time.perf_counter()
    for x in th:
        x.start()
    for x in th:
        x.join()
    dt = time.perf_counter() - t0
    assert not errors, errors
    return dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    gpu = T.Gpu()
    lib = A.declare_transcode_ladders(A.declare_transcode_ladder(gpu.lib))
    lib.uhdr_b200_last_error.restype = C.c_char_p
    lib.uhdr_b200_kernel_launches.restype = C.c_ulonglong
    res = {"card": card_info(), "reps": a.reps}
    for wname, w, h, scale, nfiles, lname in WORKLOADS:
        seeds = [make_file(lib, w, h, scale, s) for s in range(SEEDS)]
        datas = [seeds[i % SEEDS] for i in range(nfiles)]
        cfgs = LADDERS[lname]
        for threads in (1, 8):
            shares = [Share(datas[t::threads], cfgs) for t in range(threads)]
            for arm in ("loop", "ladders"):   # warm-up, and the outputs compared
                run_threads(lib, shares, arm)
            assert all(s.equal() for s in shares), ("ladders output differs from the per-file ladders'", wname, threads)
            ts = {"loop": [], "ladders": []}
            launches = {"loop": 0, "ladders": 0}
            for rep in range(a.reps):
                for arm in (("loop", "ladders") if rep % 2 == 0 else ("ladders", "loop")):
                    l0 = lib.uhdr_b200_kernel_launches()
                    ts[arm].append(run_threads(lib, shares, arm))
                    launches[arm] += lib.uhdr_b200_kernel_launches() - l0
            assert all(s.equal() for s in shares)
            loop_fps, lad_fps = nfiles / float(np.median(ts["loop"])), nfiles / float(np.median(ts["ladders"]))
            r = {"files": nfiles, "ladder": lname, "bytes_in": len(datas[0]),
                 "loop_files_per_s": round(loop_fps, 1), "ladders_files_per_s": round(lad_fps, 1),
                 "speedup": round(lad_fps / loop_fps, 2),
                 "loop_spread_s": [round(min(ts["loop"]), 4), round(max(ts["loop"]), 4)],
                 "ladders_spread_s": [round(min(ts["ladders"]), 4), round(max(ts["ladders"]), 4)]}
            if threads == 1:
                r["launches_per_file_loop"] = launches["loop"] / a.reps / nfiles
                r["launches_per_file_ladders"] = launches["ladders"] / a.reps / nfiles
            res["%s, %d thread%s" % (wname, threads, "s" if threads > 1 else "")] = r
            del shares
    res["how"] = ("uhdr_b200_transcode_ladders vs a loop of uhdr_b200_transcode_ladder over the same files and rungs, host "
                  "bytes in and out, base_420 and keep_exif on; files/s from the median wall clock of %d alternated "
                  "repetitions after one warm-up; launches from the library's counter on one thread" % a.reps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
