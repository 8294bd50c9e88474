"""The per-lane fast decoders of the scan kernel (skywalking-banyandb_b200/csrc/lane_decode.cuh) are plain functions of one lane's
registers and compile for the host: tests/native/lane_decode_test.cc runs them (multiply-add formulation, masked chunks, the
head correction) against a byte-at-a-time reference on 200k random windows, and the SWAR sum decoders (all rows, row mask) over
whole emulated pages against the plain sum.  No GPU."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_lane_decoders_equal_the_bytewise_reference(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    cuda_inc = next((p for p in ("/usr/local/cuda/include", "/usr/local/cuda/targets/x86_64-linux/include") if os.path.exists(os.path.join(p, "vector_types.h"))), None)
    if cuda_inc is None:
        pytest.skip("no CUDA headers (vector_types.h)")
    exe = tmp_path / "lane_decode_test"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-I", os.path.join(ROOT, "skywalking-banyandb_b200", "csrc"), "-I", cuda_inc, "-o", str(exe),
                           os.path.join(ROOT, "tests", "native", "lane_decode_test.cc")])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout[-2000:] + out.stderr[-2000:]
