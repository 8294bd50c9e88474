"""The fast lane's delta-of-delta page decoder (skywalking-banyandb_b200/csrc/scan_kernels.cu: dod_page_fast) compiles for the host
over the lane functions of lane_decode.cuh: tests/native/dod_lane_test.cc emulates whole pages with the kernel's geometry -- the
first difference read alone, the second differences from the unaligned byte after it, 32 B lanes, 1 KB chunks, 2 KB stages --
with pass 1, the head fix, the (n, q, r) warp scan, pass 2 and the carries, against a byte-at-a-time decode: every body start
0..15, first differences of 1..10 bytes (alone too: a 2-row page), 3-byte second differences across every lane and chunk edge, the wide check and the
stage accounting of the bail-out for 4-byte ones, and int32 P / sumP on the widest lanes the wide check admits.  No GPU."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_dod_pages_equal_the_plain_decode(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    cuda_inc = next((p for p in ("/usr/local/cuda/include", "/usr/local/cuda/targets/x86_64-linux/include") if os.path.exists(os.path.join(p, "vector_types.h"))), None)
    if cuda_inc is None:
        pytest.skip("no CUDA headers (vector_types.h)")
    exe = tmp_path / "dod_lane_test"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "skywalking-banyandb_b200", "csrc"), "-I", cuda_inc, "-o", str(exe),
                           os.path.join(ROOT, "tests", "native", "dod_lane_test.cc")])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout[-2000:] + out.stderr[-2000:]
