"""GEMM tile-schedule coverage on the GPU (-m gpu): runs the native tests/native/test_gemm_sched binary, which checks
vj_gemm against a double-precision host reference on shapes that exercise the persistent tile schedule (many and odd
tile counts per CTA, ragged M, 1 / 7 / 131-CTA grids, every epilogue, K-major and MN-major B)."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_native_gemm_schedule():
    exe = os.path.join(ROOT, "tests", "native", "test_gemm_sched")
    assert os.path.exists(exe), "run __graft_entry__.build() first"
    out = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "ALL PASSED" in out.stdout, out.stdout[-4000:] + out.stderr[-1000:]
