"""The prepared tuple group-by from plain C99 (tests/native/keys_wide_prepared_caller.c): the three prototypes include/bydb_gpu.h
declares link against libbydbgpu.so, and a NULL context or out pointer is refused with BYDB_EINVAL on a machine without a GPU."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_prepare_keys_wide_links_and_refuses_null(tmp_path, bydb):
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    lib_dir = os.path.dirname(bydb.library_path())
    exe = tmp_path / "keys_wide_prepared_caller"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", str(exe),
                           os.path.join(ROOT, "tests", "native", "keys_wide_prepared_caller.c"), "-L", lib_dir, "-lbydbgpu",
                           "-Wl,-rpath," + lib_dir])
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.strip() == "OK", out.stdout + out.stderr
