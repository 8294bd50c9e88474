"""The C++ operator (include/bydb_operator.hpp) with a stored-tag GroupBy key above 256 values, driven by
tests/native/operator_keyed_wide_test.cc.  Without a GPU the program checks the output schema and the error contract; with one
(pytest -m gpu) MaxKeyValues = 1000 runs through the one-pass form, each row checked against bydb_scan_agg_keyed_wide called
directly, and MaxKeyValues = 256 stays on the per-value passes."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(tmp_path, bydb):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    lib_dir = os.path.dirname(bydb.library_path())
    exe = tmp_path / "operator_keyed_wide_test"
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", str(exe),
                           os.path.join(ROOT, "tests", "native", "operator_keyed_wide_test.cc"), "-L", lib_dir, "-lbydbgpu",
                           "-Wl,-rpath," + lib_dir])
    return exe


def test_operator_keyed_wide_contract_without_a_device(tmp_path, bydb):
    out = subprocess.run([str(_build(tmp_path, bydb))], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and ("OK host-only" in out.stdout or "OK full" in out.stdout), out.stdout + out.stderr


@pytest.mark.gpu
def test_operator_keyed_wide_on_the_device(tmp_path, bydb):
    out = subprocess.run([str(_build(tmp_path, bydb))], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "OK full" in out.stdout, out.stdout + out.stderr
