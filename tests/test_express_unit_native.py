"""The express lane's page sum in 4 KB units (skywalking-banyandb_b200/csrc/scan_kernels.cu: scan_sum_express_kernel) compiles for
the host over the lane words of lane_decode.cuh: tests/native/express_unit_test.cc emulates whole pages with the unit geometry,
the zeroed bytes around the body, the carried rank base and the two- to three-class redo, against a byte-at-a-time page sum, for
every body start 0..15, body lengths around the piece, window, half and unit edges, 3-byte varints at every half and unit edge,
4-byte varints after the switch, windows of 64 terminators and stale stage bytes.  No GPU."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_express_units_equal_the_plain_page_sum(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    cuda_inc = next((p for p in ("/usr/local/cuda/include", "/usr/local/cuda/targets/x86_64-linux/include") if os.path.exists(os.path.join(p, "vector_types.h"))), None)
    if cuda_inc is None:
        pytest.skip("no CUDA headers (vector_types.h)")
    exe = tmp_path / "express_unit_test"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "skywalking-banyandb_b200", "csrc"), "-I", cuda_inc, "-o", str(exe),
                           os.path.join(ROOT, "tests", "native", "express_unit_test.cc")])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout[-2000:] + out.stderr[-2000:]
