"""uhdr_b200_device_state_stats without a device: the symbol is exported, declared in uhdr_b200.h (a C program that
includes the header calls it), and reads two zeros in a process that made no per-device kernel state."""
import os
import subprocess

import uhdr_testlib as T


def test_exported():
    out = subprocess.run(["nm", "-D", "--defined-only", T.GPU_SO], capture_output=True, text=True, check=True).stdout
    assert " T uhdr_b200_device_state_stats" in out


def test_declared_and_callable_without_a_device(tmp_path):
    src = tmp_path / "stats.c"
    src.write_text("""
#include <stdio.h>
#include "uhdr_b200.h"
int main(void) {
  unsigned long long s[2] = {7, 7};
  uhdr_b200_device_state_stats(NULL);
  uhdr_b200_device_state_stats(s);
  printf("%llu %llu\\n", s[0], s[1]);
  return 0;
}
""")
    exe = str(tmp_path / "stats")
    so = T.GPU_SO
    subprocess.run(["gcc", "-Werror=implicit-function-declaration", "-I", os.path.join(T.ROOT, "include"), str(src),
                    "-o", exe, "-L", os.path.dirname(so), "-l:" + os.path.basename(so),
                    "-Wl,-rpath," + os.path.dirname(so)], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.split() == ["0", "0"]
