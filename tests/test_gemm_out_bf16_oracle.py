"""The CPU reference of BF16 output (tests/gemm_out_bf16_ref.py).  Pinned here: its round-to-nearest-even conversion equals
torch's CPU .to(torch.bfloat16) on every non-NaN fp32 whose low 16 bits are one of the patterns that decide a rounding (ties to
even at every exponent, carries into the next binade, the overflow to infinity, subnormals, +-0), and maps every NaN to one
pattern; its vote equals the rounded vote of the fp32-output references under Bernoulli and TABLE plans at NC 1-3 with both
voters (the output identity of DESIGN.md §3.13); and, by hand, the flips the rounding absorbs, the flips it does not, the
signed zeros, NaN operands and the one exception to the identity, the sign of a zero."""
import numpy as np
import pytest
import torch

import gemm_bf16_ref as ref16
import gemm_fp8_ref as ref8
import gemm_out_bf16_ref as oref

STAT_KEYS = ("errors_corrected", "dwc_detected", "syncs", "injected", "first_fault_unit")
M, N, K = 24, 40, 128
LOW = np.array([0x0000, 0x0001, 0x7FFF, 0x8000, 0x8001, 0xC000, 0xFFFF], dtype=np.uint32)   # below, at and above the tie


def torch_bf16(w):
    return torch.from_numpy(w.view(np.float32).copy()).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)


def test_rne_equals_torch_on_every_upper_half_and_the_tie_bits():
    hi = np.arange(1 << 16, dtype=np.uint32) << 16
    w = (hi[:, None] | LOW[None, :]).ravel()
    nan = (w & 0x7FFFFFFF) > 0x7F800000
    got, want = oref.rne(w), torch_bf16(w)
    assert np.array_equal(got[~nan], want[~nan]), w[~nan][got[~nan] != want[~nan]][:8]
    assert (got[nan] == oref.NAN_BF16).all() and nan.sum() > 0


@pytest.mark.parametrize("w, want", [
    (0x3F808000, 0x3F80),              # tie, even below: stays
    (0x3F818000, 0x3F82),              # tie, odd below: up to even
    (0x3FFF8000, 0x4000),              # tie that carries into the next binade
    (0x3FFFFFFF, 0x4000),              # above the tie, into the next binade
    (0x7F7F7FFF, 0x7F7F),              # below the tie at the largest finite: stays finite
    (0x7F7F8000, 0x7F80),              # the tie at the largest finite rounds to infinity
    (0xFF7FFFFF, 0xFF80),              # and to -infinity
    (0x00008000, 0x0000),              # the smallest subnormal tie: to even zero
    (0x00018000, 0x0002),              # subnormal tie, odd below
    (0x007FFFFF, 0x0080),              # the largest subnormal rounds up to the smallest normal
    (0x80000000, 0x8000),              # -0 stays -0
    (0x7F800000, 0x7F80),              # infinity
    (0x7FC00000, oref.NAN_BF16), (0xFFFFFFFF, oref.NAN_BF16), (0x7F800001, oref.NAN_BF16),
])
def test_rne_by_hand(w, want):
    assert int(oref.rne(np.array([w], np.uint32))[0]) == want


def table(oracle, seed):
    rng = np.random.default_rng(seed)
    tab = np.zeros(M * N, dtype=np.uint32)
    for u in rng.choice(M * N, size=300, replace=False):
        tab[u] = oracle.fault_entry(int(rng.integers(0, 4)), 0, int(rng.integers(0, 32)))
    return tab


def operands(kind, seed):
    rng = np.random.default_rng(seed)
    if kind == "bf16":                   # sums above 256: the fp32 values have more than 8 significant bits
        return (ref16.bits(rng.integers(-64, 65, (M, K)).astype(np.float32)),
                ref16.bits(rng.integers(-64, 65, (K, N)).astype(np.float32)))
    return ref8.int_operands(rng, M, N, K, 4)


@pytest.mark.parametrize("kind", ["bf16", "fp8"])
@pytest.mark.parametrize("plan", ["none", "bernoulli", "table", "majority"])
@pytest.mark.parametrize("nc", [1, 2, 3])
def test_vote_on_bf16_is_the_rounded_fp32_vote(oracle, kind, nc, plan):
    """at most one flip per unit: the bf16 output is RNE of the fp32 output of the same plan, for both voters"""
    A, B = operands(kind, nc)
    flags, base, pl = 3, 0, None
    if plan in ("bernoulli", "majority"):
        base = 2 ** 32 - M * N // 2
        pl = oracle.make_plan(oracle.PLAN_BERNOULLI, seed=5 + nc, p=0.4)
        flags |= oref.F_MAJORITY_VOTER if plan == "majority" else 0
    if plan == "table":
        pl = oracle.make_plan(oracle.PLAN_TABLE, table=table(oracle, nc))
    kw = dict(flags=flags, plan=pl, unit_base=base)
    if kind == "bf16":
        want, ws = ref16.run(oracle, nc, A, B, **kw)
        got, gs, status = oref.run_bf16(oracle, nc, A, B, **kw)
    else:
        want, ws = ref8.run(oracle, nc, A, B, **kw)
        got, gs, status = oref.run_fp8(oracle, nc, A, B, **kw)
    assert np.array_equal(got, oref.rne(want))
    assert gs["injected"] == ws["injected"] and gs["syncs"] == ws["syncs"]
    # a unit the fp32 vote counts and the rounding makes agree is the only difference in the counts
    key = "errors_corrected" if nc == 3 else "dwc_detected"
    assert gs[key] <= ws[key]
    assert int(status.sum()) == (gs[key] if nc > 1 else 0)
    if plan != "none":
        assert gs["injected"] > 0 and (nc == 1 or gs[key] > 0)


def one_flip(oracle, u, replica, bit):
    tab = np.zeros(M * N, dtype=np.uint32)
    tab[u] = oracle.fault_entry(replica, 0, bit)
    return oracle.make_plan(oracle.PLAN_TABLE, table=tab)


def constant(value):
    """every accumulator `value`: A[:, 0] = value, B[0, :] = 1, the rest zero (GEMM_FP8 operands)"""
    A, B = np.zeros((M, K), dtype=np.uint8), np.zeros((K, N), dtype=np.uint8)
    A[:, 0], B[0, :] = ref8.bits(np.float32(value)), ref8.bits(np.float32(1.0))
    return A, B


@pytest.mark.parametrize("nc", [2, 3])
def test_a_flip_below_bf16_precision_is_injected_but_not_counted(oracle, nc):
    A, B = constant(3.0)
    u = 4 * N + 7
    for bit in (0, 7, 15):                                         # 3.0 + 2^-22 .. 2^-8 rounds back to 3.0
        out, st, status = oref.run_fp8(oracle, nc, A, B, plan=one_flip(oracle, u, 1, bit))
        assert st["injected"] == 1 and st["errors_corrected"] == st["dwc_detected"] == 0 and not status.any(), bit
        assert (out == 0x4040).all() and st["first_fault_unit"] == oref.NO_FAULT_UNIT


@pytest.mark.parametrize("nc", [2, 3])
@pytest.mark.parametrize("bit", [16, 22, 30])
def test_a_flip_that_changes_the_rounded_value_is_counted(oracle, nc, bit):
    A, B = constant(3.0)
    u = 4 * N + 7
    out, st, status = oref.run_fp8(oracle, nc, A, B, plan=one_flip(oracle, u, 1, bit))
    assert st["injected"] == 1 and (st["errors_corrected"] if nc == 3 else st["dwc_detected"]) == 1
    assert status[u] == 1 and status.sum() == 1 and st["first_fault_unit"] == u
    assert (out == 0x4040).all()                                   # replica 0 wins under DWC and TMR


@pytest.mark.parametrize("voter", [0, oref.F_MAJORITY_VOTER])
@pytest.mark.parametrize("replica", [0, 1, 2])
def test_signed_zeros_agree(oracle, replica, voter):
    A, B = constant(0.0)
    u = 9
    out, st, status = oref.run_fp8(oracle, 3, A, B, flags=3 | voter, plan=one_flip(oracle, u, replica, 31))
    assert st["injected"] == 1 and st["errors_corrected"] == 0 and not status.any()
    # the select voter keeps r0 (a -0 from replica 0 is stored), the majority voter the two +0
    assert out[u] == (0x8000 if replica == 0 and not voter else 0x0000) and (np.delete(out, u) == 0).all()


@pytest.mark.parametrize("nc", [1, 2, 3])
def test_a_nan_operand_rounds_to_the_canonical_nan_and_disagrees(oracle, nc):
    A, B = operands("fp8", 3)
    A[2, 5] = 0xFF                                                 # E4M3 NaN, negative sign: row 2 of C is NaN
    out, st, status = oref.run_fp8(oracle, nc, A, B)
    nan = np.zeros((M, N), dtype=bool)
    nan[2, :] = True
    assert np.array_equal(out.reshape(M, N) == oref.NAN_BF16, nan)
    want = N if nc > 1 else 0
    assert (st["errors_corrected"] if nc == 3 else st["dwc_detected"] if nc == 2 else 0) == want
    assert int(status.sum()) == want and st["first_fault_unit"] == (2 * N if nc > 1 else oref.NO_FAULT_UNIT)


def test_the_one_exception_to_the_identity_is_the_sign_of_a_zero(oracle):
    """TMR select: replica 0's sign flipped on a value that rounds to zero.  fp32 compares x with -x, disagrees and stores r2 = x;
    bf16 compares -0 with +0, agrees and stores r0 = -0 (DESIGN.md §3.13)"""
    A, B = np.zeros((M, K), dtype=np.uint16), np.zeros((K, N), dtype=np.uint16)
    A[:, 0] = B[0, :] = ref16.bits(np.float32(2.0 ** -70))         # accumulators 2^-140: below half the smallest bf16 subnormal
    u = 3 * N + 2
    pl = one_flip(oracle, u, 0, 31)
    want, ws = ref16.run(oracle, 3, A, B, plan=pl)
    got, gs, status = oref.run_bf16(oracle, 3, A, B, plan=pl)
    assert ws["errors_corrected"] == 1 and gs["errors_corrected"] == 0 and not status.any()
    assert np.array_equal(np.delete(got, u), np.delete(oref.rne(want), u)) and (np.delete(got, u) == 0).all()
    assert got[u] == 0x8000 and oref.rne(want)[u] == 0x0000
    got_m, _, _ = oref.run_bf16(oracle, 3, A, B, plan=pl, flags=3 | oref.F_MAJORITY_VOTER)
    assert got_m[u] == 0x0000                                      # the majority voter has no such case
