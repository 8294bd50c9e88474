"""The C++ operator (include/bydb_operator.hpp) with two to four stored-tag GroupBy keys, driven by
tests/native/operator_keys_wide_test.cc.  Without a GPU the program checks the output schema and the error contract; with one
(pytest -m gpu) MaxKeyValues = 1000 routes the stored keys to bydb_scan_agg_keys_wide, each row checked against that call made
directly, and a fifth stored key, two stored keys at MaxKeyValues 256 and OrderDesc are refused with BYDB_ENOTSUP."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(tmp_path, bydb):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    lib_dir = os.path.dirname(bydb.library_path())
    exe = tmp_path / "operator_keys_wide_test"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", str(exe),
                           os.path.join(ROOT, "tests", "native", "operator_keys_wide_test.cc"), "-L", lib_dir, "-lbydbgpu",
                           "-Wl,-rpath," + lib_dir])
    return exe


def test_operator_keys_wide_contract_without_a_device(tmp_path, bydb):
    out = subprocess.run([str(_build(tmp_path, bydb))], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and ("OK host-only" in out.stdout or "OK full" in out.stdout), out.stdout + out.stderr


@pytest.mark.gpu
def test_operator_keys_wide_on_the_device(tmp_path, bydb):
    out = subprocess.run([str(_build(tmp_path, bydb))], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "OK full" in out.stdout, out.stdout + out.stderr
