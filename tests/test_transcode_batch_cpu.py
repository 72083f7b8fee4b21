"""uhdr_b200_transcode_batch without a device: the symbol is exported, the ctypes mirror of uhdr_b200_transcode_item_t has
the C layout (the header compiled with gcc), the call-level argument errors come before any device work, and valid
arguments without a device give UHDR_CODEC_ERROR on the call and on every item."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A

INVALID, ERROR = 3, 1


def test_symbols_exported():
    out = subprocess.run(["nm", "-D", "--defined-only", T.GPU_SO], capture_output=True, text=True, check=True).stdout
    assert " T uhdr_b200_transcode_batch" in out
    assert " T uhdr_b200_jpeg_encode_batch_stats" in out


def test_item_layout_matches_the_header(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text("""
#include <stddef.h>
#include <stdio.h>
#include "uhdr_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu\\n", sizeof(uhdr_b200_transcode_item_t), offsetof(uhdr_b200_transcode_item_t, data),
         offsetof(uhdr_b200_transcode_item_t, size), offsetof(uhdr_b200_transcode_item_t, out),
         offsetof(uhdr_b200_transcode_item_t, cap), offsetof(uhdr_b200_transcode_item_t, out_size),
         offsetof(uhdr_b200_transcode_item_t, status));
  return 0;
}
""")
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(T.ROOT, "include"), str(src), "-o", exe], check=True)
    got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    D = A.TranscodeItem
    want = [C.sizeof(D)] + [getattr(D, f).offset for f, _t in D._fields_]
    assert got == want, (got, want)


@pytest.fixture(scope="module")
def lib():
    L = A.declare_transcode_batch(C.CDLL(T.GPU_SO))
    L.uhdr_b200_last_error.restype = C.c_char_p
    return L


def _items(n, data=b"\xff\xd8\xff\xd9"):
    keep = [np.frombuffer(data, np.uint8).copy() for _ in range(n)] + [np.full(64, 0xA5, np.uint8) for _ in range(n)]
    items = (A.TranscodeItem * n)()
    for i in range(n):
        items[i] = A.TranscodeItem(keep[i].ctypes.data, keep[i].size, keep[n + i].ctypes.data, 64, 7, -7)
    return items, keep


def test_call_level_errors_need_no_device(lib):
    items, keep = _items(2)
    cfg = A.TranscodeConfig(2, 75, 75, 0, 0)
    assert lib.uhdr_b200_transcode_batch(None, 1, C.byref(cfg)) == INVALID
    assert lib.uhdr_b200_transcode_batch(items, 1, None) == INVALID
    assert lib.uhdr_b200_transcode_batch(items, 0, C.byref(cfg)) == INVALID
    assert lib.uhdr_b200_transcode_batch(items, -3, C.byref(cfg)) == INVALID
    for k in (0, 3, 16):
        assert lib.uhdr_b200_transcode_batch(items, 2, C.byref(A.TranscodeConfig(k, 75, 75, 0, 0))) == INVALID
        assert b"scale denominator" in lib.uhdr_b200_last_error()
    for bq, gq in ((-1, 75), (101, 75), (75, -1), (75, 101)):
        assert lib.uhdr_b200_transcode_batch(items, 2, C.byref(A.TranscodeConfig(1, bq, gq, 0, 0))) == INVALID
        assert b"quality" in lib.uhdr_b200_last_error()
    assert [(items[i].status, items[i].out_size) for i in range(2)] == [(-7, 7), (-7, 7)]
    assert all((b == 0xA5).all() for b in keep[2:])


def test_without_a_device_every_item_gets_the_cuda_error(lib, monkeypatch):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is present")
    data = open(os.path.join(T.ROOT, "tests", "golden", "apple_gainmap_new.jpg"), "rb").read()
    items, keep = _items(3, data)
    rc = lib.uhdr_b200_transcode_batch(items, 3, C.byref(A.TranscodeConfig(2, 75, 75, 0, 0)))
    assert rc == ERROR, lib.uhdr_b200_last_error()
    assert b"CUDA" in lib.uhdr_b200_last_error() and lib.uhdr_b200_last_error().startswith(b"item 0: ")
    assert [items[i].status for i in range(3)] == [ERROR] * 3
    assert all((b == 0xA5).all() for b in keep[3:])
