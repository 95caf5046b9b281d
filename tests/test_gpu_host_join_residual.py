"""Runs the C++ parity binary of the join node's residual filter and null-equal keys (arrow_b200/cpp/b200_join_host_test.cc):
the stock "hashjoin" and "b200_hashjoin" over the same tables and options; rows and refusals must match."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "arrow_b200", "lib", "b200_join_host_test")


@pytest.mark.gpu
def test_join_residual_and_null_equal_parity():
    assert os.path.exists(EXE), "run __graft_entry__.build() first"
    p = subprocess.run([EXE], capture_output=True, text=True, timeout=900)
    tail = "\n".join(p.stdout.splitlines()[-15:])
    assert p.returncode == 0, tail + p.stderr[-2000:]
    assert "PASS" in p.stdout and "FAIL" not in p.stdout, tail


def test_join_parity_binary_is_built():
    assert os.path.exists(EXE), "run __graft_entry__.build() first"
