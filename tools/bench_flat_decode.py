"""uhdr_decode of 3840x2160 JPEG/R files whose primary image has flat runs: a black frame whose run sits at a bit phase
that falls back into step, the same frame at one that does not (more than kMaxRounds relaxation rounds, so the host
entropy decoder takes the scan), and a letterbox (flat bars around content).  For each: the route and rounds of the
primary's scan (stage API), and the best uhdr_decode time on the default route and with the host entropy decoder.

    python tools/bench_flat_decode.py [--reps 5]

The files are made by tests/jpeg_stream_writer.py and assembled with API-4 (flat single-channel map, w/4 x h/4)."""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

import jpeg_decode_cases as D  # noqa: E402
import uhdr_testlib as T  # noqa: E402
from libultrahdr_b200 import ctypes_api as A  # noqa: E402
from test_api4_cpu import _api4  # noqa: E402


def stats(L):
    st = (C.c_ulonglong * 3)()
    L.uhdr_b200_entropy_decoder_stats(st)
    return list(st)


def stage_route(L, data):
    cap = 3840 * 2160 * 4
    buf = np.zeros(cap, np.uint8)
    out = A.raw_image(-1, -1, -1, -1, 0, 0, [buf], [0])
    s0 = stats(L)
    assert L.uhdr_b200_jpeg_decode(data, C.c_size_t(len(data)), 0, C.byref(out), C.c_size_t(cap)) == 0
    s1 = stats(L)
    return {"device": s1[0] - s0[0], "handed_to_host": s1[1] - s0[1], "rounds": s1[2] if s1[0] > s0[0] else None}


def best_decode_ms(L, api, data, reps, entropy):
    prev = L.uhdr_b200_set_entropy_decoder(entropy)
    try:
        api.decode(data)
        best = 1e9
        for _ in range(reps):
            t = time.perf_counter()
            api.decode(data)
            best = min(best, (time.perf_counter() - t) * 1e3)
    finally:
        L.uhdr_b200_set_entropy_decoder(prev)
    return round(best, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    L = T.Gpu().lib
    L.uhdr_b200_entropy_decoder_stats.restype = None
    api = T.UhdrApi(L)
    w, h = 3840, 2160
    files = {
        "black_good_phase": D.flat_frame(w, h, D.S420, D.lead_for_phase(D.S420, False, 32, dc=-128)[0], dc=-128),
        "black_bad_phase": D.flat_frame(w, h, D.S420, D.lead_for_phase(D.S420, True, 32, dc=-128)[0], dc=-128),
        "letterbox": D.flat_frame(w, h, D.S420, 0, bars=(17, 17)),
    }
    res = {}
    for name, st in files.items():
        _p, gm, md = D.jpegr_parts(L, w, h, primary=st)
        data = _api4(L, st.data, gm.data, md, base_cg=A.CG_BT709)
        assert isinstance(data, bytes), data
        r = stage_route(L, st.data)
        r["uhdr_decode_ms_default"] = best_decode_ms(L, api, data, a.reps, 0)
        r["uhdr_decode_ms_host_entropy"] = best_decode_ms(L, api, data, a.reps, 1)
        r["bytes"] = len(data)
        res[name] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
