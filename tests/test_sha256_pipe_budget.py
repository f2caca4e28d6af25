"""CPU: the SHA-256 TMR kernel keeps its additions on the IMAD pipe (DESIGN.md §5.0), and the identity that rests on holds.

The segmented kernel is bound by ALU-pipe issue.  Its round and schedule additions are issued as IMAD x * 1 + y with the 1
in the constant bank; a ptxas upgrade or a source change that folds them back into IADD3 would quietly give that back, so
the SASS of the embedded cubin is held to a budget here."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import sha_pipe_rates as spr  # noqa: E402
from mock_run import CUBIN, res_usage  # noqa: E402

# whole-function SASS counts (the tile loop is nearly all of them): ALU-pipe instructions at most, IMAD-pipe at least.
# With every addition on the ALU pipe the fault-free kernel issued 2235 ALU and 234 IMAD instructions, the injecting one
# 6136 and 349.
BUDGET = {"xmr_sha256_b64_seg_nc3_inj0": (1900, 950), "xmr_sha256_b64_seg_nc3_inj1": (5750, 1050)}
MAX_REGS_INJ0 = 56     # 3 CTAs of 384 threads per SM: 65536 / 1152 registers per thread


def _pipes(fun):
    counts = {"alu": 0, "imad": 0, "other": 0}
    for op, n in spr.histogram(spr.sass_ops(CUBIN, fun)).items():
        counts[spr.pipe_of(op)] += n
    return counts


@pytest.mark.parametrize("fun", sorted(BUDGET))
def test_segmented_kernel_keeps_its_pipe_split(built_lib, fun):
    alu_max, imad_min = BUDGET[fun]
    p = _pipes(fun)
    assert p["alu"] <= alu_max and p["imad"] >= imad_min, (fun, p)


@pytest.mark.parametrize("fun", sorted(BUDGET))
def test_segmented_kernel_has_no_local_memory(built_lib, fun):
    fields = res_usage()[fun]
    assert fields["STACK"] == 0 and fields["LOCAL"] == 0, fields
    if fun.endswith("inj0"):
        assert fields["REG"] <= MAX_REGS_INJ0, fields
    assert not [op for _, op, _ in spr.sass_ops(CUBIN, fun) if op.startswith(("LDL", "STL"))]


@pytest.fixture(scope="module")
def words():
    rng = np.random.default_rng(2026)
    special = np.array([0, 0xFFFFFFFF] + [1 << k for k in range(32)], dtype=np.uint64)
    return np.concatenate([special, rng.integers(0, 1 << 32, size=1 << 20, dtype=np.uint64)])


def test_addition_is_multiply_by_one_add(words):
    m32 = np.uint64(0xFFFFFFFF)
    for b in (np.roll(words, 1), words[::-1].copy()):
        assert np.array_equal((words * np.uint64(1) + b) & m32, (words + b) & m32)
