"""The two-class SWAR word of the express lane (skywalking-banyandb_b200/csrc/lane_decode.cuh: swar_word2) and its switch to the
three-class word compile for the host: tests/native/lane_switch_test.cc emulates whole pages with 3-byte varints placed across
lane and chunk edges, in the first and last chunk, and 4-byte varints after the switch, against the plain page sum.  No GPU."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_two_class_switch_equals_the_plain_page_sum(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    cuda_inc = next((p for p in ("/usr/local/cuda/include", "/usr/local/cuda/targets/x86_64-linux/include") if os.path.exists(os.path.join(p, "vector_types.h"))), None)
    if cuda_inc is None:
        pytest.skip("no CUDA headers (vector_types.h)")
    exe = tmp_path / "lane_switch_test"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "skywalking-banyandb_b200", "csrc"), "-I", cuda_inc, "-o", str(exe),
                           os.path.join(ROOT, "tests", "native", "lane_switch_test.cc")])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout[-2000:] + out.stderr[-2000:]
