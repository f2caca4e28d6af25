"""The CPU reference of scaled GEMM_FP8 (tests/gemm_fp8_scaled_ref.py).  Pinned here: at scales of 1 it is GEMM_FP8's reference
(tests/gemm_fp8_ref.py, the oracle's GEMM_TF32 element on widened operands) on outputs and all five counters, at NC 1-3, without
a plan, with a Bernoulli plan whose units cross 2^32, with a TABLE plan and with the majority voter; and, by hand, what a scale
does to a flip: a zero scale hides it, a NaN scale makes every vote of its row or column disagree, and a scale that rounds two
accumulators to one value hides it too."""
import numpy as np
import pytest

import gemm_fp8_ref as ref8
import gemm_fp8_scaled_ref as sref

STAT_KEYS = ("errors_corrected", "dwc_detected", "syncs", "injected", "first_fault_unit")
M, N, K = 24, 40, 128


def operands(seed):
    return ref8.int_operands(np.random.default_rng(seed), M, N, K, 4)


def table(oracle, seed, nc):
    rng = np.random.default_rng(seed)
    tab = np.zeros(M * N, dtype=np.uint32)
    for u in rng.choice(M * N, size=200, replace=False):
        site = 0 if rng.random() < 0.8 else 1                    # site 1 does not exist: ignored
        tab[u] = oracle.fault_entry(int(rng.integers(0, 4)), site, int(rng.integers(0, 32)))   # replica >= NC: ignored
    return tab


@pytest.mark.parametrize("plan", ["none", "bernoulli", "table", "majority"])
@pytest.mark.parametrize("nc", [1, 2, 3])
def test_scale_one_is_gemm_fp8s_reference(oracle, nc, plan):
    A, B = operands(nc)
    flags, base, pl = 3, 0, None
    if plan in ("bernoulli", "majority"):
        base = 2 ** 32 - M * N // 2                              # the global units cross 2^32
        pl = oracle.make_plan(oracle.PLAN_BERNOULLI, seed=11 + nc, p=0.3)
        flags |= sref.F_MAJORITY_VOTER if plan == "majority" else 0
    if plan == "table":
        pl = oracle.make_plan(oracle.PLAN_TABLE, table=table(oracle, nc, nc))
    want, ws = ref8.run(oracle, nc, A, B, flags=flags, plan=pl, unit_base=base)
    for sa, sb in ((np.float32(1), np.float32(1)), (np.ones(M, np.float32), np.ones(N, np.float32))):
        got, gs, status = sref.run(oracle, nc, A, B, sa, sb, flags=flags, plan=pl, unit_base=base)
        f = want.view(np.float32)
        same = (got == want) | (np.isnan(f) & np.isnan(got.view(np.float32)))    # x 1.0 keeps every value but a NaN's payload
        assert same.all()
        assert {k: gs[k] for k in STAT_KEYS} == {k: ws[k] for k in STAT_KEYS}
        if plan != "none":
            assert gs["injected"] > 0
        assert int(status.sum()) == (gs["errors_corrected"] if nc == 3 else gs["dwc_detected"] if nc == 2 else 0)


def test_scales_apply_in_order_to_the_accumulator(oracle):
    """(acc x sa_i) x sb_j in float32, against the same two roundings done with numpy scalars"""
    A, B = operands(5)
    rng = np.random.default_rng(5)
    sa = (rng.standard_normal(M) * 2.0 ** rng.integers(-20, 20, M)).astype(np.float32)
    sb = (rng.standard_normal(N) * 2.0 ** rng.integers(-20, 20, N)).astype(np.float32)
    got, st, _ = sref.run(oracle, 3, A, B, sa, sb)
    acc = sref.exact_acc(A, B)
    for i, j in ((0, 0), (3, 17), (M - 1, N - 1)):
        assert got[i * N + j] == np.float32(np.float32(acc[i, j] * sa[i]) * sb[j]).view(np.uint32)
    assert st["errors_corrected"] == 0 and st["syncs"] == M * N


def one_flip(oracle, nc, u, replica, bit):
    tab = np.zeros(M * N, dtype=np.uint32)
    tab[u] = oracle.fault_entry(replica, 0, bit)
    return oracle.make_plan(oracle.PLAN_TABLE, table=tab)


@pytest.mark.parametrize("nc", [2, 3])
def test_a_zero_scale_hides_a_flip_that_leaves_the_accumulator_finite(oracle, nc):
    A, B = operands(7)
    sa = np.ones(M, np.float32)
    sa[5] = 0.0
    u = 5 * N + 9
    for bit in (0, 22, 31):
        _, st, status = sref.run(oracle, nc, A, B, sa, np.float32(1), plan=one_flip(oracle, nc, u, 1, bit))
        assert st["injected"] == 1 and st["errors_corrected"] == st["dwc_detected"] == 0 and not status.any(), bit
    # the same flip where the scale is 1 is seen
    _, st, status = sref.run(oracle, nc, A, B, sa, np.float32(1), plan=one_flip(oracle, nc, 6 * N + 9, 1, 22))
    assert (st["errors_corrected"] if nc == 3 else st["dwc_detected"]) == 1 and status[6 * N + 9] == 1


@pytest.mark.parametrize("nc", [1, 2, 3])
def test_a_nan_scale_makes_every_vote_of_its_row_or_column_disagree(oracle, nc):
    A, B = operands(8)
    sa, sb = np.ones(M, np.float32), np.ones(N, np.float32)
    sa[3], sb[11] = np.nan, np.nan
    got, st, status = sref.run(oracle, nc, A, B, sa, sb)
    nan = np.zeros((M, N), dtype=bool)
    nan[3, :], nan[:, 11] = True, True
    assert np.array_equal(np.isnan(got.view(np.float32)).reshape(M, N), nan)
    want = int(nan.sum()) if nc > 1 else 0
    assert (st["errors_corrected"] if nc == 3 else st["dwc_detected"] if nc == 2 else 0) == want
    assert int(status.sum()) == want and st["first_fault_unit"] == (11 if nc > 1 else sref.NO_FAULT_UNIT)


@pytest.mark.parametrize("nc", [2, 3])
def test_a_scale_that_rounds_two_accumulators_together_hides_the_flip(oracle, nc):
    """acc 3.0 and acc 3.0 with its lowest mantissa bit flipped differ by 2^-22; times 2^-140 both land on the same subnormal"""
    A = np.zeros((M, K), dtype=np.uint8)
    B = np.zeros((K, N), dtype=np.uint8)
    A[:, 0], B[0, :] = ref8.bits(np.float32(3.0)), ref8.bits(np.float32(1.0))
    sa = np.full(M, 2.0 ** -140, dtype=np.float32)
    u = 2 * N + 4
    assert np.float32(3.0) * sa[0] == np.float32(np.nextafter(np.float32(3.0), np.float32(4.0))) * sa[0]
    _, st, status = sref.run(oracle, nc, A, B, sa, np.float32(1), plan=one_flip(oracle, nc, u, 0, 0))
    assert st["injected"] == 1 and st["errors_corrected"] == st["dwc_detected"] == 0 and not status.any()
    _, st, _ = sref.run(oracle, nc, A, B, np.float32(1), np.float32(1), plan=one_flip(oracle, nc, u, 0, 0))
    assert (st["errors_corrected"] if nc == 3 else st["dwc_detected"]) == 1
