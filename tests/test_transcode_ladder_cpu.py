"""uhdr_b200_transcode_ladder without a device: the symbol is exported, the ctypes mirror of uhdr_b200_transcode_rung_t
has the C layout (the header compiled with gcc), the call-level argument errors touch no rung, a rung's own argument
errors come before any device work and only on that rung, and valid rungs without a device get UHDR_CODEC_ERROR."""
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
    assert " T uhdr_b200_transcode_ladder" in out


def test_rung_layout_matches_the_header(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text("""
#include <stddef.h>
#include <stdio.h>
#include "uhdr_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu\\n", sizeof(uhdr_b200_transcode_rung_t), offsetof(uhdr_b200_transcode_rung_t, cfg),
         offsetof(uhdr_b200_transcode_rung_t, out), offsetof(uhdr_b200_transcode_rung_t, cap),
         offsetof(uhdr_b200_transcode_rung_t, out_size), offsetof(uhdr_b200_transcode_rung_t, status),
         sizeof(uhdr_b200_transcode_config_t));
  return 0;
}
""")
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(T.ROOT, "include"), str(src), "-o", exe], check=True)
    got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    D = A.TranscodeRung
    want = [C.sizeof(D)] + [getattr(D, f).offset for f, _t in D._fields_] + [C.sizeof(A.TranscodeConfig)]
    assert got == want, (got, want)


@pytest.fixture(scope="module")
def lib():
    L = A.declare_transcode_ladder(C.CDLL(T.GPU_SO))
    L.uhdr_b200_last_error.restype = C.c_char_p
    return L


def _rungs(cfgs):
    n = len(cfgs)
    keep = [np.full(64, 0xA5, np.uint8) for _ in range(n)]
    rungs = (A.TranscodeRung * n)()
    for i, c in enumerate(cfgs):
        rungs[i] = A.TranscodeRung(A.TranscodeConfig(*c), keep[i].ctypes.data, 64, 7, -7)
    return rungs, keep


def test_call_level_errors_touch_no_rung(lib):
    data = np.frombuffer(b"\xff\xd8\xff\xd9", np.uint8).copy()
    rungs, keep = _rungs([(1, 75, 75, 0, 0)] * 17)
    assert lib.uhdr_b200_transcode_ladder(None, 4, rungs, 2) == INVALID
    assert lib.uhdr_b200_transcode_ladder(data.ctypes.data, 4, None, 2) == INVALID
    for n in (0, -1, 17):
        assert lib.uhdr_b200_transcode_ladder(data.ctypes.data, 4, rungs, n) == INVALID
        assert b"rungs" in lib.uhdr_b200_last_error()
    assert all((rungs[i].status, rungs[i].out_size) == (-7, 7) for i in range(17))
    assert all((b == 0xA5).all() for b in keep)


def test_rung_argument_errors_only_on_those_rungs(lib):
    data = np.frombuffer(b"\xff\xd8\xff\xd9", np.uint8).copy()   # a valid rung meets the probe's error
    bad = [(0, 75, 75, 0, 0), (3, 75, 75, 0, 0), (16, 75, 75, 0, 0), (2, -1, 75, 0, 0), (2, 101, 75, 0, 0),
           (2, 75, -1, 0, 0), (2, 75, 101, 0, 0)]
    rungs, keep = _rungs(bad + [(2, 75, 75, 0, 0)] * 2)
    rungs[len(bad) + 1].out = None   # a null out
    rc = lib.uhdr_b200_transcode_ladder(data.ctypes.data, data.size, rungs, len(bad) + 2)
    st = [rungs[i].status for i in range(len(bad) + 2)]
    assert st[:len(bad)] == [INVALID] * len(bad) and st[len(bad) + 1] == INVALID
    assert rc == INVALID and lib.uhdr_b200_last_error().startswith(b"rung 0: scale denominator")
    # the valid rung gets the file's probe error, what the single call gives
    A.declare_transcode(lib)
    n = C.c_size_t(0)
    want = lib.uhdr_b200_transcode(data.ctypes.data, data.size, C.byref(A.TranscodeConfig(2, 75, 75, 0, 0)),
                                   keep[0].ctypes.data, 64, C.byref(n))
    assert st[len(bad)] == want != 0, (st, want)
    assert all((b == 0xA5).all() for b in keep)
    # all rungs invalid: nothing of the file is looked at
    rungs, keep = _rungs(bad)
    assert lib.uhdr_b200_transcode_ladder(data.ctypes.data, data.size, rungs, len(bad)) == INVALID
    assert [rungs[i].status for i in range(len(bad))] == [INVALID] * len(bad)


def test_without_a_device_every_valid_rung_gets_the_cuda_error(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is present")
    data = np.frombuffer(open(os.path.join(T.ROOT, "tests", "golden", "apple_gainmap_new.jpg"), "rb").read(),
                         np.uint8).copy()
    rungs, keep = _rungs([(1, 85, 85, 0, 0), (2, 80, 70, 1, 1), (4, 101, 70, 0, 0), (8, 80, 70, 0, 0)])
    rc = lib.uhdr_b200_transcode_ladder(data.ctypes.data, data.size, rungs, 4)
    assert rc == ERROR, lib.uhdr_b200_last_error()
    assert lib.uhdr_b200_last_error().startswith(b"rung 0: ") and b"CUDA" in lib.uhdr_b200_last_error()
    assert [rungs[i].status for i in range(4)] == [ERROR, ERROR, INVALID, ERROR]
    assert all((b == 0xA5).all() for b in keep)
