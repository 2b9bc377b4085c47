"""The normalisation case table (tests/norm_cases.py) against the kernels csrc/norm.cu declares and launches."""
import os
import re

import norm_cases as nc
from conformance import CSRC, declared, source

NORM_CU = os.path.join(CSRC, "norm.cu")


def test_norm_cu_declares_one_kernel_per_pass():
    assert declared(NORM_CU) == nc.KERNELS


def test_table_covers_every_instance_and_the_sliced_grid():
    src = source(NORM_CU)
    launched = set(re.findall(r"\b(norm_\w+_kernel<\d+>)", src))
    assert launched, "no templated launch found in norm.cu"
    covered = {k for c in nc.CASES for k in c.kernels if "<" in k}
    assert covered == launched, f"instances without a case: {sorted(launched - covered)}; " \
                                f"the table names instances norm.cu does not launch: {sorted(covered - launched)}"
    for vec in (1, 4):
        assert any(g.vec == vec and g.slices > 1 for g in nc.GEOMS), f"no case with channel slices at VEC {vec}"


def test_table_is_well_formed():
    ids = [c.id for c in nc.CASES]
    assert len(ids) == len(set(ids))
    for g in nc.GEOMS:
        assert g.why, f"{g.name}: every geometry names the edge it exists for"
        assert all(any(c.geom == g and c.act == a for c in nc.CASES) for a in nc.ACTS)
    for a in nc.ACTS:
        assert {c.rtf for c in nc.CASES if c.act == a} == {False, True}, f"{a}: round_tf32 on and off"
