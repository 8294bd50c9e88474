"""The dense page form (skywalking-banyandb_b200/csrc/dense_page.cuh) is a set of plain per-lane functions that compile for the host:
tests/native/dense_page_test.cc encodes pages with the write pass's word encoder and sums them with the express lane's per-piece
sum, walking 4 KB units with stale bytes past the stream, against the exact 128-bit sum -- every bit length 0..32, 1..8448 rows,
m at both ends of int64.  No GPU."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_dense_pages_sum_to_the_exact_value_sum(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    cuda_inc = next((p for p in ("/usr/local/cuda/include", "/usr/local/cuda/targets/x86_64-linux/include") if os.path.exists(os.path.join(p, "vector_types.h"))), None)
    if cuda_inc is None:
        pytest.skip("no CUDA headers (vector_types.h)")
    exe = tmp_path / "dense_page_test"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "skywalking-banyandb_b200", "csrc"), "-I", cuda_inc, "-o", str(exe),
                           os.path.join(ROOT, "tests", "native", "dense_page_test.cc")])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout[-2000:] + out.stderr[-2000:]
