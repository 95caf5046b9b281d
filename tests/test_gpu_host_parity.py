"""Runs the C++ parity binaries (arrow_b200/cpp/*_host_test.cc, built into arrow_b200/lib/): each sends the same inputs
through arrow::compute::CallFunction / Acero with the stock CPU registry of the installed reference binary and with the
plug-in's nested GPU registry on device copies, and requires equal results, or the same error codes and texts."""
import glob
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "arrow_b200", "lib")
BINARIES = sorted(os.path.basename(p)[:-len(".cc")] for p in glob.glob(os.path.join(ROOT, "arrow_b200", "cpp", "*_host_test.cc")))


@pytest.mark.gpu
@pytest.mark.parametrize("name", BINARIES)
def test_plugin_parity(name):
    exe = os.path.join(LIB, name)
    assert os.path.exists(exe), "run __graft_entry__.build() first"
    p = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    tail = "\n".join(p.stdout.splitlines()[-15:])
    assert p.returncode == 0, tail + p.stderr[-2000:]
    assert "PASS" in p.stdout and "FAIL" not in p.stdout, tail


@pytest.mark.parametrize("name", BINARIES)
def test_parity_binary_is_built(name):
    assert os.path.exists(os.path.join(LIB, name)), "run __graft_entry__.build() first"


def test_cpp_dropin_built_and_links_reference_binaries():
    """CPU: the plugin is built, links the installed reference libraries and exports its entry points."""
    so = os.path.join(ROOT, "arrow_b200", "lib", "libarrow_b200_compute.so")
    assert os.path.exists(so), "run __graft_entry__.build() first"
    ldd = subprocess.run(["ldd", so], capture_output=True, text=True).stdout
    assert "libarrow.so.2400" in ldd and "libarrow_compute.so.2400" in ldd and "libarrow_b200.so" in ldd
    assert "not found" not in ldd, ldd
    nm = subprocess.run(["nm", "-D", "--defined-only", "-C", so], capture_output=True, text=True).stdout
    for sym in ("arrow_b200::Runtime::Get", "arrow_b200::RegisterFunctions", "arrow_b200::MakeGrouper",
                "arrow_b200::RegisterAceroNodes", "arrow_b200::ToDevice"):
        assert sym in nm, sym
