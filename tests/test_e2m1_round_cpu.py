"""The branch-free E2M1 rounding of the NVFP4 / MXFP4 fake-quant kernels (e2m1_round_mag in csrc/common.cuh) gives
the same bits as the reference's compare chain (e2m1_round_mag_ref) for every non-negative fp32 bit pattern: all
finite values, +inf and the NaNs.  Both functions are compiled from the header as host code, so no GPU is needed;
tests/test_gpu_e2m1_round.py runs the same comparison with the device build."""

import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r"""
#include <cstdio>
#include "common.cuh"

int main() {
  unsigned long long checked = 0, bad = 0;
  for (unsigned long long u = 0; u < (1ull << 31); ++u) {
    const uint32_t b = (uint32_t)u;
    float a;
    memcpy(&a, &b, 4);
    const float x = b200q::e2m1_round_mag(a), y = b200q::e2m1_round_mag_ref(a);
    uint32_t bx, by;
    memcpy(&bx, &x, 4);
    memcpy(&by, &y, 4);
    if (bx != by && bad++ < 4) printf("mismatch %08x: %a vs %a\n", b, x, y);
    ++checked;
  }
  printf("checked %llu mismatches %llu\n", checked, bad);
  return 0;
}
"""


def test_e2m1_round_mag_matches_compare_chain_on_every_non_negative_float(tmp_path):
    import __graft_entry__ as g

    src = tmp_path / "e2m1_check.cu"
    exe = tmp_path / "e2m1_check"
    src.write_text(SRC)
    subprocess.run([g._nvcc(), *g.NVCC_FLAGS, "-Xcompiler", "-O3", "-I", os.path.join(ROOT, "include"),
                    "-I", g.CSRC, str(src), "-o", str(exe)], check=True, capture_output=True, text=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    assert out.strip().splitlines()[-1] == f"checked {1 << 31} mismatches 0", out
