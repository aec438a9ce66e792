"""ops.py guards memory with LavbError only (python -O strips asserts), and its host record dtypes match the header's records."""
import ast
import os

import pytest

from lav_b200 import ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_ops_has_no_assert():
    tree = ast.parse(open(os.path.join(ROOT, "lav_b200", "ops.py")).read())
    lines = [node.lineno for node in ast.walk(tree) if isinstance(node, ast.Assert)]
    assert not lines, f"assert statements at ops.py lines {lines}"


@pytest.mark.parametrize("name,nbytes", [("STACK_JOB_DTYPE", 72), ("BEV_JOB_DTYPE", 128), ("PNG_JOB_DTYPE", 32),
                                         ("LIDAR_SWEEP_DTYPE", 88), ("PLAN_SAFETY_ACTOR_DTYPE", 56), ("NAV_STATE_DTYPE", 128)])
def test_record_dtypes_have_the_header_sizes(name, nbytes):
    assert getattr(ops, name).itemsize == nbytes
