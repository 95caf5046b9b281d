"""Runs the C++ parity binary of the cumulative functions (arrow_b200/cpp/b200_cumulative_host_test.cc): the plug-in's
seven cumulative functions against the stock registry for every type, start and skip_nulls, over device arrays and device
ChunkedArrays, with the reference's error codes and texts for overflow, a start that fails its cast and a type without a
kernel."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "arrow_b200", "lib", "b200_cumulative_host_test")


@pytest.mark.gpu
def test_cumulative_plugin_parity():
    assert os.path.exists(EXE), "run __graft_entry__.build() first"
    p = subprocess.run([EXE], capture_output=True, text=True, timeout=900)
    tail = "\n".join(p.stdout.splitlines()[-15:])
    assert p.returncode == 0, tail + p.stderr[-2000:]
    assert "PASS" in p.stdout and "FAIL" not in p.stdout, tail


def test_cumulative_parity_binary_is_built():
    assert os.path.exists(EXE), "run __graft_entry__.build() first"
