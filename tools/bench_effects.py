"""Image effects (uhdr_add_effect_*) on bench.py's inputs:
    python tools/bench_effects.py [--iters N] [--ref-iters M]

Median wall time of
  * uhdr_decode of the 8K JPEG/R (7680x4320, map scale 1, multichannel) to RGBA half float, with no effect, mirror,
    rotate 90 and crop + rotate 90 + resize, on warmed handles (create, set image, effects, decode, release);
  * k_effect_gather's kernel time in those decodes (CUDA events, uhdr_b200_kernel_timing_report), and the bytes it
    moves over that time against the H100 SXM's 3.35 TB/s;
  * a 4K (3840x2160) API-1 uhdr_encode with and without rotate 90;
  * the reference's uhdr_decode of the same chains, for context.
Every GPU result is checked equal to the reference's first.  The card's name and power limit are read in the same run."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402
import uhdr_testlib as T  # noqa: E402
from libultrahdr_b200 import ctypes_api as A  # noqa: E402
from test_effects_cpu import MIRROR_HORIZONTAL, declare  # noqa: E402
from test_gpu_effects import decode, encode  # noqa: E402

HBM_TBPS = 3.35
CHAINS = {"none": [], "mirror": [("mirror", MIRROR_HORIZONTAL)], "rotate90": [("rotate", 90)],
          "crop+rotate90+resize": [("crop", 0, 7680, 540, 3780), ("rotate", 90), ("resize", 1620, 3840)]}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception as e:  # noqa: BLE001
        return repr(e)


def gather_ms(lib):
    buf = C.create_string_buffer(1 << 16)
    lib.uhdr_b200_kernel_timing_report(buf, len(buf), 1)
    for line in buf.value.decode().splitlines():
        f = line.split()
        if f and f[0] == "effect_gather":
            return int(f[1]), float(f[2])
    return 0, 0.0


def timed(fn, iters):
    fn()
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--ref-iters", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_effects needs a CUDA device")
    gpu = T.Gpu()
    lib = declare(gpu.lib)
    ref = declare(C.CDLL(T.REF_SO)) if T.have_ref() else None
    p8, y8 = bench.make_frame(bench.W8K, bench.H8K, 7)
    h8, s8, _k = bench.frame_descs(p8, y8, bench.W8K, bench.H8K)
    data = T.UhdrApi(lib).encode(h8, s8)
    out = {"card": card(), "decode_8k_f16": {}, "encode_4k_api1": {}}
    for name, chain in CHAINS.items():
        rc, img, gm = decode(lib, data, A.FMT_RGBAF16, A.CT_LINEAR, chain)
        assert rc == 0, (name, rc)
        row = {"size": [img[0][0], img[0][1]]}
        if ref is not None:
            t0 = time.perf_counter()
            want = decode(ref, data, A.FMT_RGBAF16, A.CT_LINEAR, chain)
            row["ref_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
            assert want[1][0][:5] == img[0][:5] and (want[1][1] == img[1]).all() and (want[2][1] == gm[1]).all(), name
        row["ms"] = round(timed(lambda: decode(lib, data, A.FMT_RGBAF16, A.CT_LINEAR, chain), args.iters), 3)
        if chain:
            lib.uhdr_b200_set_kernel_timing(1)
            gather_ms(lib)
            for _ in range(args.iters):
                decode(lib, data, A.FMT_RGBAF16, A.CT_LINEAR, chain)
            n, total = gather_ms(lib)
            lib.uhdr_b200_set_kernel_timing(0)
            # per decode: the output image (8 B/px read and written) and the RGBA8888 map (4 B/px); the launch count
            # is checked to be two gathers per decode
            w, h = img[0][0], img[0][1]
            gw, gh = gm[0][0], gm[0][1]
            nbytes = 2 * (w * h * 8 + gw * gh * 4)
            per = total / max(1, n // 2)
            row.update(gather_launches=n, gather_ms_per_decode=round(per, 4), gather_bytes=nbytes,
                       gather_tbps=round(nbytes / (per * 1e-3) / 1e12, 3),
                       bound_ms=round(nbytes / (HBM_TBPS * 1e12) * 1e3, 4))
        out["decode_8k_f16"][name] = row
    p4, y4 = bench.make_frame(3840, 2160, 3)
    h4, s4, _k4 = bench.frame_descs(p4, y4, 3840, 2160)
    for name, chain in (("none", []), ("rotate90", [("rotate", 90)])):
        rc, mine = encode(lib, h4, s4, chain, scale=1)
        assert rc == 0
        if ref is not None:
            assert encode(ref, h4, s4, chain, scale=1) == (0, mine), name
        out["encode_4k_api1"][name] = {"ms": round(timed(lambda: encode(lib, h4, s4, chain, scale=1), args.iters), 3)}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
