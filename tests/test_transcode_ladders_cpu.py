"""uhdr_b200_transcode_ladders without a device: the symbol is exported, the ctypes mirror of uhdr_b200_transcode_file_t
has the C layout (the header compiled with gcc), the call-level argument errors touch no file and no rung, a file's own
argument errors and a rung's own argument errors come before any device work and stay on that file or rung, and valid
rungs without a device get UHDR_CODEC_ERROR."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A

INVALID, ERROR = 3, 1


def test_symbol_exported():
    out = subprocess.run(["nm", "-D", "--defined-only", T.GPU_SO], capture_output=True, text=True, check=True).stdout
    assert " T uhdr_b200_transcode_ladders" in out


def test_file_layout_matches_the_header(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text("""
#include <stddef.h>
#include <stdio.h>
#include "uhdr_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(uhdr_b200_transcode_file_t), offsetof(uhdr_b200_transcode_file_t, data),
         offsetof(uhdr_b200_transcode_file_t, size), offsetof(uhdr_b200_transcode_file_t, rungs),
         offsetof(uhdr_b200_transcode_file_t, n), offsetof(uhdr_b200_transcode_file_t, status));
  return 0;
}
""")
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(T.ROOT, "include"), str(src), "-o", exe], check=True)
    got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    D = A.TranscodeFile
    assert got == [C.sizeof(D)] + [getattr(D, f).offset for f, _t in D._fields_], got


@pytest.fixture(scope="module")
def lib():
    L = A.declare_transcode_ladders(A.declare_transcode_ladder(C.CDLL(T.GPU_SO)))
    L.uhdr_b200_last_error.restype = C.c_char_p
    return L


class Files:
    """files[i] = (data bytes or None, [rung cfgs] or None, n or None); every rung's buffer and fields are sentinels"""

    def __init__(self, specs):
        self.keep, self.bufs, self.rungs = [], [], []
        self.files = (A.TranscodeFile * len(specs))()
        for i, (data, cfgs, n) in enumerate(specs):
            src = None if data is None else np.frombuffer(data, np.uint8).copy()
            self.keep.append(src)
            rungs = None
            if cfgs is not None:
                rungs = (A.TranscodeRung * max(len(cfgs), 1))()
                for j, c in enumerate(cfgs):
                    buf = np.full(64, 0xA5, np.uint8)
                    self.bufs.append(buf)
                    rungs[j] = A.TranscodeRung(A.TranscodeConfig(*c), buf.ctypes.data, 64, 7, -7)
            self.rungs.append(rungs)
            self.files[i] = A.TranscodeFile(None if src is None else src.ctypes.data, 0 if src is None else src.size,
                                            rungs, len(cfgs or []) if n is None else n, -9)

    def status(self, i):
        return self.files[i].status

    def rung_status(self, i):
        r = self.rungs[i]
        return [] if r is None else [r[j].status for j in range(len(r))]

    def untouched(self):
        return all((b == 0xA5).all() for b in self.bufs)


EOI = b"\xff\xd8\xff\xd9"


def test_call_level_errors_touch_no_file(lib):
    f = Files([(EOI, [(1, 75, 75, 0, 0)] * 2, None)] * 3)
    assert lib.uhdr_b200_transcode_ladders(None, 3) == INVALID
    assert b"files" in lib.uhdr_b200_last_error()
    for n in (0, -1):
        assert lib.uhdr_b200_transcode_ladders(f.files, n) == INVALID
        assert b"files" in lib.uhdr_b200_last_error()
    assert [f.status(i) for i in range(3)] == [-9] * 3
    assert all(f.rung_status(i) == [-7, -7] for i in range(3)) and f.untouched()


def test_file_and_rung_argument_errors_stay_on_their_file_and_rung(lib):
    bad = [(0, 75, 75, 0, 0), (3, 75, 75, 0, 0), (2, -1, 75, 0, 0), (2, 75, 101, 0, 0)]
    f = Files([(EOI, bad, None),                    # every rung invalid: the file's status is its first rung's
               (None, [(1, 75, 75, 0, 0)], None),   # null data
               (EOI, None, 1),                      # null rungs
               (EOI, [(1, 75, 75, 0, 0)], 0),       # n = 0
               (EOI, [(1, 75, 75, 0, 0)] * 16, 17),  # n = 17
               (EOI, bad[:2] + [(2, 75, 75, 0, 0)], None)])   # a valid rung meets the probe's error
    rc = lib.uhdr_b200_transcode_ladders(f.files, 6)
    assert rc == INVALID and lib.uhdr_b200_last_error().startswith(b"file 0: rung 0: scale denominator")
    assert [f.status(i) for i in range(5)] == [INVALID] * 5
    assert f.rung_status(0) == [INVALID] * 4
    assert f.rung_status(1) == [-7] and f.rung_status(3) == [-7] and f.rung_status(4) == [-7] * 16
    # the last file: its own rung errors first, its valid rung the probe's error, what the ladder alone gives
    st = f.rung_status(5)
    assert st[:2] == [INVALID, INVALID] and st[2] not in (0, -7, ERROR), st
    g = Files([(EOI, bad[:2] + [(2, 75, 75, 0, 0)], None)])
    want = lib.uhdr_b200_transcode_ladder(g.keep[0].ctypes.data, 4, g.rungs[0], 3)
    assert f.status(5) == want == INVALID and f.rung_status(5) == g.rung_status(0)
    assert f.untouched()
    # a file's own error named in the message
    f = Files([(None, [(1, 75, 75, 0, 0)], None), (EOI, [(1, 75, 75, 0, 0)], 17)])
    assert lib.uhdr_b200_transcode_ladders(f.files, 2) == INVALID
    assert lib.uhdr_b200_last_error().startswith(b"file 0: received nullptr for compressed")


def test_without_a_device_every_valid_rung_gets_the_cuda_error(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is present")
    data = open(os.path.join(T.ROOT, "tests", "golden", "apple_gainmap_new.jpg"), "rb").read()
    f = Files([(data, [(4, 101, 70, 0, 0)], None),
               (data, [(1, 85, 85, 0, 0), (2, 80, 70, 1, 1), (4, 101, 70, 0, 0)], None),
               (None, [(1, 75, 75, 0, 0)], None)])
    rc = lib.uhdr_b200_transcode_ladders(f.files, 3)
    assert rc == INVALID and lib.uhdr_b200_last_error().startswith(b"file 0: rung 0: invalid quality")
    assert [f.status(i) for i in range(3)] == [INVALID, ERROR, INVALID]
    assert f.rung_status(0) == [INVALID] and f.rung_status(1) == [ERROR, ERROR, INVALID] and f.rung_status(2) == [-7]
    assert f.untouched()
    f = Files([(data, [(1, 85, 85, 0, 0)], None), (data, [(8, 80, 70, 0, 0)], None)])
    assert lib.uhdr_b200_transcode_ladders(f.files, 2) == ERROR
    msg = lib.uhdr_b200_last_error()
    assert msg.startswith(b"file 0: rung 0: ") and b"CUDA" in msg, msg
    assert [f.status(i) for i in range(2)] == [ERROR, ERROR] and f.untouched()
