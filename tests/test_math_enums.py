"""The math op-code tables of the Python binding (UNARY_OPS, ROUND_MODES) against the enums of include/arrow_b200.h, as
the C compiler sees them, and ROUND_MODES against the values of pyarrow's RoundMode."""
import shutil
import subprocess

import pyarrow.compute as pc
import pytest

from arrow_b200 import _cabi as cabi
from tests.test_cabi_enums import ROOT, header_enumerators

TABLES = {
    "UNARY_OPS": (cabi.UNARY_OPS, "B2UnaryOp", lambda k: "B2_" + k.upper()),
    "ROUND_MODES": (cabi.ROUND_MODES, "B2RoundMode", lambda k: "B2_ROUND_" + k.upper()),
}


def test_math_tables_match_the_header_enums(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    enums = header_enumerators()
    members = [e for name in ("B2UnaryOp", "B2RoundMode") for e in enums[name]]
    src = tmp_path / "enums.c"
    src.write_text('#include <stdio.h>\n#include "arrow_b200.h"\nint main(void) {\n'
                   + "\n".join(f'printf("{e} %lld\\n", (long long){e});' for e in members) + "\nreturn 0; }\n")
    exe = tmp_path / "enums"
    subprocess.check_call(["gcc", "-std=c11", "-I", f"{ROOT}/include", str(src), "-o", str(exe)])
    got = {k: int(v) for k, v in (l.split() for l in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())}
    for table_name, (table, enum, enumerator) in TABLES.items():
        want = {e: got[e] for e in enums[enum]}
        assert {enumerator(k): v for k, v in table.items()} == want, f"{table_name} differs from {enum}"


def test_round_modes_follow_pyarrow_order():
    # RoundOptions' repr names the mode; its position in the reference's enum is the code
    for name, code in cabi.ROUND_MODES.items():
        assert f"round_mode={name.upper()}" in str(pc.RoundOptions(0, name))
    assert list(cabi.ROUND_MODES.values()) == list(range(10))
