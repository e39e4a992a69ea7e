"""Every operator kind of include/cds.h is registered wherever the tests judge operators: cabi's OP_* constants, the
interpreter (tests/emulator.py) and the program audit (tests/program_audit.py), so that no kind is half registered."""
import os
import re

import emulator
import program_audit as pa
from cleandiffuser_b200.engine import cabi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_every_operator_kind_is_interpreted_and_audited():
    with open(os.path.join(ROOT, "include", "cds.h")) as f:
        enum = re.search(r"typedef enum cds_op_kind \{(.*?)\} cds_op_kind;", f.read(), re.S).group(1)
    header = {n: int(v) for n, v in re.findall(r"CDS_(OP_\w+) = (\d+)", re.sub(r"/\*.*?\*/", "", enum, flags=re.S))}
    assert {n: getattr(cabi, n) for n in dir(cabi) if n.startswith("OP_")} == header
    kinds = set(header.values())
    assert set(emulator.OPS) == set(pa.KIND_NAME) == set(pa.Auditor.REFERENCE) == kinds
    assert all(hasattr(cabi.Op().u, field) for field, _ in emulator.OPS.values())
