"""bydb_scan_agg_keys_wide / bydb_scan_partials_keys_wide from plain C99 (tests/native/keys_wide_caller.c): the prototypes
include/bydb_gpu.h declares compile with -std=c99 -Wall -Wextra -Werror and link against libbydbgpu.so; the argument refusals that
need no device run without a GPU, and on a GPU the caller also runs every refusal through a context and one two-tag query."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import oracle as O
from tests.helpers import build_part, grid

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _caller(tmp_path, bydb):
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    lib_dir = os.path.dirname(bydb.library_path())
    exe = tmp_path / "keys_wide_caller"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", str(exe),
                           os.path.join(ROOT, "tests", "native", "keys_wide_caller.c"), "-L", lib_dir, "-lbydbgpu",
                           "-Wl,-rpath," + lib_dir])
    return exe


def test_keys_wide_links_and_refuses_bad_arguments(tmp_path, bydb):
    out = subprocess.run([str(_caller(tmp_path, bydb))], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.strip() == "OK", out.stdout + out.stderr


@pytest.mark.gpu
def test_keys_wide_two_tags_from_c(tmp_path, bydb):
    """two series of 6 rows; a = x/y alternating in pairs, b = row % 3 (int64): the (a, b) tuples in insertion order"""
    sids, ts, _ = grid(2, 6)
    n = sids.size
    r = np.arange(n) % 6
    a = [b"x" if (i // 2) % 2 == 0 else b"y" for i in r.tolist()]
    b = (r % 3).astype(np.int64)
    part = build_part(sids, ts, np.ones(n, np.int64), [("v", O.VT_INT64, np.arange(n, dtype=np.int64), None)],
                      [("default", [("a", O.VT_STR, a, None), ("b", O.VT_INT64, b, None)])])
    args = []
    for name, data in part.files().items():
        p = tmp_path / name
        p.write_bytes(bytes(data))
        args.append(f"{name}={p}")
    out = subprocess.run([str(_caller(tmp_path, bydb))] + args, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.strip().splitlines()
    assert lines[-1] == "OK" and lines[-2] == "tuples 5 tags 2", out.stdout
    # rows 0..5 of a series: (x,0) (x,1) (y,2) (y,0) (x,1) (x,2); both series fold into group 0
    assert lines[:-2] == ["0 x 0 2", "0 x 1 4", "0 y 2 2", "0 y 0 2", "0 x 2 2"], out.stdout
