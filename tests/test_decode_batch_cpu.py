"""uhdr_b200_decode_batch_dev without a device: the symbol is exported, the ctypes mirror of uhdr_b200_decode_item_t has
the C layout (the header compiled with gcc), and the call-level argument errors come before any device work."""
import ctypes as C
import os
import subprocess

import pytest

import uhdr_testlib as T
from libultrahdr_b200 import ctypes_api as A

INVALID = 3


def test_symbol_exported():
    out = subprocess.run(["nm", "-D", "--defined-only", T.GPU_SO], capture_output=True, text=True, check=True).stdout
    assert " T uhdr_b200_decode_batch_dev" in out


def test_item_layout_matches_the_header(tmp_path):
    src = tmp_path / "layout.c"
    src.write_text("""
#include <stddef.h>
#include <stdio.h>
#include "uhdr_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu\\n", sizeof(uhdr_b200_decode_item_t), offsetof(uhdr_b200_decode_item_t, data),
         offsetof(uhdr_b200_decode_item_t, size), offsetof(uhdr_b200_decode_item_t, dest_dev),
         offsetof(uhdr_b200_decode_item_t, gainmap_dev), offsetof(uhdr_b200_decode_item_t, metadata_out),
         offsetof(uhdr_b200_decode_item_t, status));
  return 0;
}
""")
    exe = str(tmp_path / "layout")
    subprocess.run(["gcc", "-I", os.path.join(T.ROOT, "include"), str(src), "-o", exe], check=True)
    got = [int(x) for x in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    D = A.DecodeItem
    want = [C.sizeof(D)] + [getattr(D, f).offset for f, _t in D._fields_]
    assert got == want, (got, want)


@pytest.fixture(scope="module")
def lib():
    L = A.declare_decode_batch(C.CDLL(T.GPU_SO))
    L.uhdr_b200_last_error.restype = C.c_char_p
    return L


def test_call_level_errors_need_no_device(lib):
    items = (A.DecodeItem * 2)()
    for i in range(2):
        items[i].status = -7
    assert lib.uhdr_b200_decode_batch_dev(None, 1, 1, A.CT_LINEAR, 4.0, None) == INVALID
    assert lib.uhdr_b200_decode_batch_dev(items, 0, 1, A.CT_LINEAR, 4.0, None) == INVALID
    assert lib.uhdr_b200_decode_batch_dev(items, -3, 1, A.CT_LINEAR, 4.0, None) == INVALID
    for k in (0, 3, 16):
        assert lib.uhdr_b200_decode_batch_dev(items, 2, k, A.CT_LINEAR, 4.0, None) == INVALID
        assert b"scale denominator" in lib.uhdr_b200_last_error()
    assert [items[i].status for i in range(2)] == [-7, -7]
