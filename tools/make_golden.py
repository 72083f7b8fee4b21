"""Generates tests/golden/uhdr_golden_320x192.npz: a 320x192 crop of the reference's own 1280x720
fixtures (tests/data/raw_p010_image.p010 + raw_yuv420_image.yuv420, the config-1 inputs) together with
the outputs of the reference's own code (oracle/_ref) for every stage of the hot path, so that the tests
need neither the reference checkout nor its fixtures.
    python tools/make_golden.py /path/to/libultrahdr"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import uhdr_testlib as T  # noqa: E402
from libultrahdr_b200 import ctypes_api as A  # noqa: E402

W, H, X0, Y0, CW, CH = 1280, 720, 864, 312, 320, 192  # most varied 320x192 window of the colour-bar fixture
p010 = np.fromfile(os.path.join(sys.argv[1], "tests", "data", "raw_p010_image.p010"), dtype=np.uint16)
yuv = np.fromfile(os.path.join(sys.argv[1], "tests", "data", "raw_yuv420_image.yuv420"), dtype=np.uint8)
Y = p010[:W * H].reshape(H, W)[Y0:Y0 + CH, X0:X0 + CW]
UV = p010[W * H:].reshape(H // 2, W)[Y0 // 2:(Y0 + CH) // 2, X0:X0 + CW]
hb = np.concatenate([Y.ravel(), UV.ravel()]).astype(np.uint16)
y8 = yuv[:W * H].reshape(H, W)[Y0:Y0 + CH, X0:X0 + CW]
u8 = yuv[W * H:W * H * 5 // 4].reshape(H // 2, W // 2)[Y0 // 2:(Y0 + CH) // 2, X0 // 2:(X0 + CW) // 2]
v8 = yuv[W * H * 5 // 4:].reshape(H // 2, W // 2)[Y0 // 2:(Y0 + CH) // 2, X0 // 2:(X0 + CW) // 2]
sb = np.concatenate([y8.ravel(), u8.ravel(), v8.ravel()]).astype(np.uint8)

R = T.Ref()
hdr, k1 = A.p010_image(hb, CW, CH, A.CG_BT2100, A.CT_HLG, A.CR_LIMITED)
sdr, k2 = A.yuv420_image(sb, CW, CH, A.CG_BT709)
out = {"p010": hb, "yuv420": sb}
for name, kw in (("default", {}), ("s4_single", {"scale_factor": 4, "multichannel": 0}),
                 ("onepass", {"preset": A.USAGE_REALTIME})):
    g, m = R.generate(sdr, hdr, A.default_gm_config(**kw))
    out["gm_" + name] = g
    out["md_" + name] = np.frombuffer(bytes(m), np.uint8).copy()
    gi = T.gm_image(g, A.CG_BT2100)
    out["apply_f16_" + name] = R.apply(sdr, gi, m, A.CT_LINEAR)
    out["apply_pq_" + name] = R.apply(sdr, gi, m, A.CT_PQ)
out["tonemap"] = R.tonemap(hdr)[0]
out["convert_709_601"] = R.convert_yuv(sb, CW, CH, 0, 1)
api = T.UhdrApi(R.lib)
out["file_api1"] = np.frombuffer(api.encode(hdr, sdr), np.uint8).copy()
px, gm, md, cg = api.decode(bytes(out["file_api1"]))
out["decoded_f16"] = px
dst = os.path.join(ROOT, "tests", "golden", "uhdr_golden_320x192.npz")
np.savez_compressed(dst, **out)
print("wrote", dst, os.path.getsize(dst), "bytes")
