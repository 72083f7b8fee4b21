"""Generates the Apple gain-map vectors of tests/test_xmp_cpu.py from the reference's own fixtures
(tests/data/apple_gainmap_{new,old}.jpg of a libultrahdr checkout):

  tests/golden/apple_gainmap_{new,old}_headers.jpg : the fixture with the entropy-coded data of both
      JPEGs cut to 64 bytes.  Every marker segment (EXIF with the maker notes, ICC, MPF, XMP, tables,
      frame and scan headers) is the fixture's own; the MPF entries are rewritten to the new image sizes
      (keeping the file's 70-byte overstatement of the primary image's size).  Metadata parsing reads
      none of the removed bytes: the reference's probe returns the same dimensions, EXIF, ICC and
      gain-map metadata for the cut file as for the original.
  tests/golden/apple_gainmap_probe.json : the reference's uhdr_dec_probe of each cut file (oracle/_ref).

    python tools/make_apple_golden.py /path/to/libultrahdr
"""
import hashlib
import json
import os
import struct
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import uhdr_testlib as T  # noqa: E402
from test_probe_cpu import _probe  # noqa: E402
from test_xmp_cpu import _vals, probe_record  # noqa: E402


def scan_span(d, p):
    """(first entropy-coded byte, EOI offset) of the JPEG starting at p"""
    i = p + 2
    while True:
        assert d[i] == 0xFF, i
        mk, seg = d[i + 1], (d[i + 2] << 8) | d[i + 3]
        if mk == 0xDA:
            j = s = i + 2 + seg
            while not (d[j] == 0xFF and d[j + 1] != 0 and not 0xD0 <= d[j + 1] <= 0xD7):
                j += 1
            assert d[j + 1] == 0xD9
            return s, j
        i += 2 + seg


def cut_scans(d, keep=64):
    s0, e0 = scan_span(d, 0)
    g = e0 + 2   # the gain-map JPEG follows the primary's EOI
    s1, e1 = scan_span(d, g)
    assert e1 + 2 == len(d)

    def head(a):
        k = keep
        while d[a + k - 1] == 0xFF:   # never end inside a stuffed 0xFF 0x00 pair
            k += 1
        return d[a:a + k]
    prim = bytearray(d[:s0] + head(s0) + b"\xff\xd9")
    gm = d[g:s1] + head(s1) + b"\xff\xd9"
    t = prim.index(b"MPF\x00") + 4   # MPF TIFF header
    bo = ">" if prim[t:t + 2] == b"MM" else "<"
    ifd = t + struct.unpack(bo + "I", prim[t + 4:t + 8])[0]
    ent = None
    for k in range(struct.unpack(bo + "H", prim[ifd:ifd + 2])[0]):
        tag, _typ, _cnt, val = struct.unpack(bo + "HHII", prim[ifd + 2 + 12 * k:ifd + 14 + 12 * k])
        if tag == 0xB002:   # MP entries
            ent = t + val
    sz0 = struct.unpack(bo + "I", prim[ent + 4:ent + 8])[0]
    off1 = struct.unpack(bo + "I", prim[ent + 24:ent + 28])[0]
    assert off1 + t == g
    prim[ent + 4:ent + 8] = struct.pack(bo + "I", len(prim) + sz0 - g)
    prim[ent + 20:ent + 28] = struct.pack(bo + "II", len(gm), len(prim) - t)
    return bytes(prim) + gm


ref = T.Ref().lib
golden = {}
for name in ("apple_gainmap_new", "apple_gainmap_old"):
    full = open(os.path.join(sys.argv[1], "tests", "data", name + ".jpg"), "rb").read()
    cut = cut_scans(full)
    a, b = _probe(ref, full), _probe(ref, cut)
    assert a["dims"] == b["dims"] and a["exif"] == b["exif"] and a["icc"] == b["icc"]
    assert _vals(a["md"], False) == _vals(b["md"], False)
    with open(os.path.join(ROOT, "tests", "golden", name + "_headers.jpg"), "wb") as f:
        f.write(cut)
    golden[name] = probe_record(b)
    print(name, len(full), "->", len(cut), "bytes", hashlib.sha256(cut).hexdigest()[:16])
with open(os.path.join(ROOT, "tests", "golden", "apple_gainmap_probe.json"), "w") as f:
    json.dump(golden, f, sort_keys=True)
    f.write("\n")
