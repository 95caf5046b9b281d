"""Runs the C++ parity binary of the numeric math functions (arrow_b200/cpp/b200_math_host_test.cc): the plug-in's abs ...
trunc, round / round_to_multiple / round_binary, power, the bit-wise ops and the shifts against the stock registry for every
type and option case, the calls the device refuses, and two b200_ plans (a filter feeding a project, and a project feeding an
aggregate's key) against their stock equivalents."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "arrow_b200", "lib", "b200_math_host_test")


@pytest.mark.gpu
def test_math_plugin_parity():
    assert os.path.exists(EXE), "run __graft_entry__.build() first"
    p = subprocess.run([EXE], capture_output=True, text=True, timeout=900)
    tail = "\n".join(p.stdout.splitlines()[-15:])
    assert p.returncode == 0, tail + p.stderr[-2000:]
    assert "PASS" in p.stdout and "FAIL" not in p.stdout, tail


def test_math_parity_binary_is_built():
    assert os.path.exists(EXE), "run __graft_entry__.build() first"
