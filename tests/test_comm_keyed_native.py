"""tests/native/comm_keyed_ranks.c: the keyed collective (bydb_scan_reduce_keyed) from plain C, one process per rank, mailbox
handles over a pipe, checked against bydb_scan_agg_keyed on one context over all shards."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(tmp_path, bydb):
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    lib_dir = os.path.dirname(bydb.library_path())
    exe = tmp_path / "comm_keyed_ranks"
    subprocess.check_call(["gcc", "-std=c99", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"), "-o", str(exe),
                           os.path.join(ROOT, "tests", "native", "comm_keyed_ranks.c"), "-L", lib_dir, "-lbydbgpu", "-lm",
                           "-Wl,-rpath," + lib_dir])
    return exe


def test_keyed_ranks_program_compiles(tmp_path, bydb):
    """the program builds against the declared prototypes with -Werror (no GPU needed)"""
    assert _build(tmp_path, bydb).exists()


@pytest.mark.gpu
def test_multi_process_keyed_reduce(tmp_path, bydb):
    """One device: the ranks share it (CUDA IPC works within a device); more: round-robin."""
    import torch
    exe = _build(tmp_path, bydb)
    ndev = max(1, torch.cuda.device_count())
    for nranks in sorted({3, min(4, max(3, ndev))}):
        out = subprocess.run([str(exe), str(nranks), str(ndev)], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
