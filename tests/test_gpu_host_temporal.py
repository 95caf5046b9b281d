"""Runs the C++ parity binary of the temporal functions (arrow_b200/cpp/b200_temporal_host_test.cc): the plug-in's casts,
compares (implicit unit casts and the naive / zoned refusal included) and calendar / clock fields against the stock
registry, a named zone refused on the device, and a b200_filter -> b200_project -> b200_aggregate plan over dates and
timestamps against its stock equivalent."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "arrow_b200", "lib", "b200_temporal_host_test")


@pytest.mark.gpu
def test_temporal_plugin_parity():
    assert os.path.exists(EXE), "run __graft_entry__.build() first"
    p = subprocess.run([EXE], capture_output=True, text=True, timeout=900)
    tail = "\n".join(p.stdout.splitlines()[-15:])
    assert p.returncode == 0, tail + p.stderr[-2000:]
    assert "PASS" in p.stdout and "FAIL" not in p.stdout, tail


def test_temporal_parity_binary_is_built():
    assert os.path.exists(EXE), "run __graft_entry__.build() first"
