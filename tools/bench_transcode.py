"""Time uhdr_b200_transcode against the same composition through the existing host-buffer entry points and against the
reference composition on the CPU (one thread).

Files: bench.py's 8K API-1 file, a 4080x3072 file with map scale 4 and a 1920x1080 file.  Settings: k = 2, 4, 8 and
k = 1, all at quality 75 for both JPEGs, the base kept in its decoded sampling.  Every arm's output is first checked
against the reference composition.  Reports the median call time, the output bytes and the kernel launches per call,
with the GPU's name and power limit, as one JSON line per (file, k) and a table on stderr.

  python tools/bench_transcode.py [--iters 20] [--out results/bench_transcode.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import bench  # noqa: E402
import transcode_testlib as X  # noqa: E402
import uhdr_testlib as T  # noqa: E402
from libultrahdr_b200 import ctypes_api as A  # noqa: E402

Q = 75


def gpu_info():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def make_file(lib, w, h, scale):
    p010, yuv = bench.make_frame(w, h, 0)
    hdr, sdr, _keep = bench.frame_descs(p010, yuv, w, h)
    return T.UhdrApi(lib).encode(hdr, sdr, quality=95, gm_quality=95, scale=scale)


def host_chain(lib, ref, data, k):
    """the composition through the existing host-buffer entry points: uhdr_b200_jpeg_decode_scaled of both JPEGs,
    uhdr_b200_jpeg_encode of both, API-4 uhdr_encode"""
    p = X._probe(lib, data)
    jpgs = []
    for jpg in (p["base_image"], p["gainmap_image"]):
        buf = np.frombuffer(jpg, np.uint8).copy()
        cap = len(jpg) * 64 + (1 << 20)
        out = np.zeros(cap, np.uint8)
        img = A.RawImage()
        img.planes[0] = out.ctypes.data
        rc = lib.uhdr_b200_jpeg_decode_scaled(buf.ctypes.data, buf.size, 0, k, C.byref(img), C.c_size_t(cap))
        assert rc == 0, T.gpu_err(T.Gpu())
        w, h = img.w, img.h
        dims = {A.FMT_Y400: [(w, h)], A.FMT_YUV444: [(w, h)] * 3,
                A.FMT_YUV420: [(w, h)] + [((w + 1) // 2, (h + 1) // 2)] * 2}[img.fmt]
        planes, o = [], 0
        for pw, ph in dims:
            planes.append(out[o:o + pw * ph])
            o += pw * ph
        enc = A.raw_image(img.fmt, -1, -1, -1, w, h, planes, [pw for pw, _ in dims])
        jpgs.append(T.gpu_jpeg_encode(T.Gpu(), enc, Q, X.icc_of(jpg) or None))
    bicc = X.icc_of(p["base_image"])
    return X._api4(lib, jpgs[0], jpgs[1], p["md"], ref.ref_icc_gamut(C.c_char_p(bicc), C.c_size_t(len(bicc))))


def timed(fn, iters, sync=None):
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        if sync:
            sync()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--cpu-iters", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_transcode: no CUDA device")
    import __graft_entry__ as g
    g.build()
    lib = T.Gpu().lib
    A.declare_transcode(lib)
    A.declare_scaled_decode(lib)
    ref = T.Ref().lib
    dev = gpu_info()
    files = {"8K 7680x4320 s1": make_file(lib, bench.W8K, bench.H8K, 1),
             "4080x3072 s4": make_file(lib, 4080, 3072, 4),
             "1920x1080 s1": make_file(lib, 1920, 1080, 1)}
    rows = []
    for name, data in files.items():
        for k in (2, 4, 8, 1):
            want = X.composition(ref, data, k, Q, Q)
            rc, got, _ = X.transcode(lib, data, k, Q, Q)
            assert rc == 0 and got == want, (name, k, rc)
            chain_same = host_chain(lib, ref, data, k) == want
            for _ in range(3):
                X.transcode(lib, data, k, Q, Q)
                host_chain(lib, ref, data, k)
            l0 = lib.uhdr_b200_kernel_launches()
            t_gpu = timed(lambda: X.transcode(lib, data, k, Q, Q), a.iters)
            l_gpu = (lib.uhdr_b200_kernel_launches() - l0) / a.iters
            l0 = lib.uhdr_b200_kernel_launches()
            t_chain = timed(lambda: host_chain(lib, ref, data, k), a.iters)
            l_chain = (lib.uhdr_b200_kernel_launches() - l0) / a.iters
            t_cpu = timed(lambda: X.composition(ref, data, k, Q, Q), a.cpu_iters)
            r = {"file": name, "k": k, "quality": Q, "gpu": dev, "bytes_in": len(data), "bytes_out": len(got),
                 "transcode_ms": round(t_gpu, 3), "transcode_launches": l_gpu,
                 "host_chain_ms": round(t_chain, 3), "host_chain_launches": l_chain, "host_chain_same_bytes": chain_same,
                 "reference_cpu_1thread_ms": round(t_cpu, 2)}
            rows.append(r)
            print(json.dumps(r), flush=True)
    sys.stderr.write(f"GPU: {dev}\n{'file':<18} {'k':>2} {'out B':>9} {'transcode ms':>13} {'launch':>6} "
                     f"{'host chain ms':>14} {'launch':>6} {'ref CPU ms':>11}\n")
    for r in rows:
        sys.stderr.write(f"{r['file']:<18} {r['k']:>2} {r['bytes_out']:>9} {r['transcode_ms']:>13.3f} "
                         f"{r['transcode_launches']:>6.0f} {r['host_chain_ms']:>14.3f} {r['host_chain_launches']:>6.0f} "
                         f"{r['reference_cpu_1thread_ms']:>11.1f}\n")
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
