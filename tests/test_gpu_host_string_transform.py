"""Runs the C++ parity binary of the string transforms (arrow_b200/cpp/b200_string_transform_host_test.cc): the
plug-in's binary_length, utf8_length, ascii_upper / ascii_lower, utf8_slice_codeunits, binary_slice and
binary_join_element_wise against the stock registry for every type and option case, the calls the device refuses, and
three b200_ plans (a filter, a project, and a project feeding an aggregate's key) against their stock equivalents."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "arrow_b200", "lib", "b200_string_transform_host_test")


@pytest.mark.gpu
def test_string_transform_plugin_parity():
    assert os.path.exists(EXE), "run __graft_entry__.build() first"
    p = subprocess.run([EXE], capture_output=True, text=True, timeout=900)
    tail = "\n".join(p.stdout.splitlines()[-15:])
    assert p.returncode == 0, tail + p.stderr[-2000:]
    assert "PASS" in p.stdout and "FAIL" not in p.stdout, tail


def test_string_transform_parity_binary_is_built():
    assert os.path.exists(EXE), "run __graft_entry__.build() first"
