"""The CPU reference of COAST_K_GEMM_F16 and COAST_MM_OUT_F16 (tests/gemm_f16_ref.py).  Pinned here: the runtime's per-unit
numbers for the new id equal the oracle's GEMM_TF32 numbers, with ids 9, 11 and 13 still unassigned; the fp32 reference equals
GEMM_TF32 on the widened operands and an exact float64 sum on integer data; the f16 conversion equals torch's CPU
.to(torch.float16) on every non-NaN fp32 whose low 13 bits decide a rounding, and maps every NaN to one pattern; the f16 vote
equals the rounded fp32 vote under Bernoulli and TABLE plans at NC 1-3 with both voters (the output identity of DESIGN.md §3.15);
and, by hand, ties, the overflow at 65520, subnormal results, the flips the rounding absorbs, the sign flip of a value that
rounds to zero under each voter, and the majority voter on 16-bit patterns."""
import numpy as np
import pytest
import torch

import gemm_f16_ref as ref

K_GEMM_F16 = 14
M, N, K = 24, 40, 128


def test_per_unit_numbers_equal_gemm_tf32s_and_ids_9_11_13_are_unassigned(oracle, built_lib):
    """the runtime's numbers for the new id against the oracle's for GEMM_TF32 (no driver is needed to ask)"""
    from coast_b200 import runtime as R
    L, t = R.load_library(), oracle.K_GEMM_TF32
    assert R.K_GEMM_F16 == K_GEMM_F16 and R.OUT_BYTES[K_GEMM_F16] == 4 and R.MM_ELEM_BYTES[K_GEMM_F16] == 2
    assert R.out_bytes(K_GEMM_F16) == 4 and R.out_bytes(K_GEMM_F16, 0, R.MM_OUT_F16) == 2
    assert R.out_bytes(K_GEMM_F16, 0, R.MM_OUT_BF16) == 4 and R.out_bytes(R.K_GEMM_BF16, 0, R.MM_OUT_F16) == 4
    assert L.coast_fault_sites(K_GEMM_F16, 0, 128) == oracle.fault_sites(t, 0, 128) == 1
    assert L.coast_fault_site_bits(K_GEMM_F16, 0, 128, 0) == oracle.fault_site_bits(t, 0, 128, 0) == 32
    assert L.coast_out_bytes_per_unit(K_GEMM_F16) == oracle.out_bytes_per_unit(t) == 4
    assert L.coast_votes_per_unit(K_GEMM_F16) == oracle.votes_per_unit(t) == 1
    assert L.coast_flags_honoured(K_GEMM_F16, 3, 0x200 | 0x4) == 0 and L.coast_flags_honoured(K_GEMM_F16, 3, 0x400 | 0x1) == 0x401
    for k in (9, 11, 13, 15):
        assert L.coast_out_bytes_per_unit(k) == L.coast_votes_per_unit(k) == L.coast_fault_sites(k, 0, 128) == 0


# ------------------------------------------------------------------------------------------ fp32 C
@pytest.mark.parametrize("nc", [1, 2, 3])
def test_fp32_reference_is_gemm_tf32_on_the_widened_operands_and_exact_on_integers(oracle, nc):
    rng = np.random.default_rng(nc)
    A, B = ref.int_operands(rng, M, N, K)
    got, st = ref.run(oracle, nc, A, B)
    want, wst = oracle.run(oracle.K_GEMM_TF32, nc, ref.value(A), M * N, M=M, N=N, K=K, aux=ref.value(B), flags=3)
    assert np.array_equal(got, want.view(np.uint32)) and st == wst
    exact = ref.value(A).astype(np.float64) @ ref.value(B).astype(np.float64)
    assert np.array_equal(got.view(np.float32), exact.astype(np.float32).ravel())


def test_every_float16_widens_exactly_and_back():
    h = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    v = ref.value(h)
    nan = np.isnan(v)
    assert nan.sum() == 2 * 1023
    assert np.array_equal(ref.bits(v[~nan]), h[~nan])
    assert np.array_equal(ref.rne(ref.widen(h[~nan])), h[~nan])
    # a TF32 operand (top 19 bits) holds every float16 exactly: the low 13 bits of every widened pattern are zero
    assert not (ref.widen(h[~nan]) & 0x1FFF).any()


# ------------------------------------------------------------------------------------------ the f16 conversion
LOW = np.array([0x0000, 0x0001, 0x0FFF, 0x1000, 0x1001, 0x17FF, 0x1FFF], dtype=np.uint32)   # below, at and above the tie


def torch_f16(w):
    return torch.from_numpy(w.view(np.float32).copy()).to(torch.float16).view(torch.int16).numpy().view(np.uint16)


def test_rne_equals_torch_on_every_upper_part_and_the_tie_bits():
    hi = np.arange(1 << 19, dtype=np.uint32) << 13
    w = (hi[:, None] | LOW[None, :]).ravel()
    nan = (w & 0x7FFFFFFF) > 0x7F800000
    got, want = ref.rne(w), torch_f16(w)
    assert np.array_equal(got[~nan], want[~nan]), w[~nan][got[~nan] != want[~nan]][:8]
    assert (got[nan] == ref.NAN_F16).all() and nan.sum() > 0


def f32(x):
    return int(np.array([x], np.float32).view(np.uint32)[0])


@pytest.mark.parametrize("w, want", [
    (f32(1 + 2 ** -11), 0x3C00),                   # tie, even below: stays
    (f32(1 + 3 * 2 ** -11), 0x3C02),               # tie, odd below: up to even
    (f32(2 - 2 ** -11), 0x4000),                   # tie that carries into the next binade
    (f32(65504.0), 0x7BFF),                        # the largest finite float16
    (f32(65519.996), 0x7BFF),                      # below the tie at the largest finite: stays finite
    (f32(65520.0), 0x7C00),                        # the tie at the largest finite rounds to infinity
    (f32(-65520.0), 0xFC00),                       # and to -infinity
    (f32(1e30), 0x7C00),                           # far past it
    (f32(2.0 ** -24), 0x0001),                     # the smallest subnormal
    (f32(2.0 ** -25), 0x0000),                     # half of it, a tie: to even zero
    (f32(3 * 2.0 ** -25), 0x0002),                 # subnormal tie, odd below: up
    (f32(2.0 ** -25 + 2.0 ** -40), 0x0001),        # just above half: up
    (f32(2.0 ** -14 - 2.0 ** -25), 0x0400),        # the largest subnormal's tie rounds up to the smallest normal
    (f32(-2.0 ** -30), 0x8000),                    # rounds to -0
    (0x80000000, 0x8000),                          # -0 stays -0
    (0x7F800000, 0x7C00), (0xFF800000, 0xFC00),    # infinities
    (0x7FC00000, ref.NAN_F16), (0xFFFFFFFF, ref.NAN_F16), (0x7F800001, ref.NAN_F16),
])
def test_rne_by_hand(w, want):
    assert int(ref.rne(np.array([w], np.uint32))[0]) == want


# ------------------------------------------------------------------------------------------ the output identity
def table(oracle, seed):
    rng = np.random.default_rng(seed)
    tab = np.zeros(M * N, dtype=np.uint32)
    for u in rng.choice(M * N, size=300, replace=False):
        tab[u] = oracle.fault_entry(int(rng.integers(0, 4)), 0, int(rng.integers(0, 32)))
    return tab


@pytest.mark.parametrize("plan", ["none", "bernoulli", "table", "majority"])
@pytest.mark.parametrize("nc", [1, 2, 3])
def test_vote_on_f16_is_the_rounded_fp32_vote(oracle, nc, plan):
    """at most one flip per unit: the f16 output is RNE of the fp32 output of the same plan, for both voters (sums up to 2^21
    have more than 11 significant bits, so the rounding is not trivial)"""
    A, B = ref.int_operands(np.random.default_rng(nc), M, N, K, 128)
    flags, base, pl = 3, 0, None
    if plan in ("bernoulli", "majority"):
        base = 2 ** 32 - M * N // 2
        pl = oracle.make_plan(oracle.PLAN_BERNOULLI, seed=5 + nc, p=0.4)
        flags |= ref.F_MAJORITY_VOTER if plan == "majority" else 0
    if plan == "table":
        pl = oracle.make_plan(oracle.PLAN_TABLE, table=table(oracle, nc))
    kw = dict(flags=flags, plan=pl, unit_base=base)
    want, ws = ref.run(oracle, nc, A, B, **kw)
    got, gs, status = ref.run_f16(oracle, nc, A, B, **kw)
    exc = exceptions(oracle, nc, A, B, kw)
    assert np.array_equal(np.delete(got, exc), np.delete(ref.rne(want), exc))
    assert np.array_equal(got[exc], ref.rne(want)[exc] ^ 0x8000) and (ref.rne(want)[exc] & 0x7FFF == 0).all()
    assert gs["injected"] == ws["injected"] and gs["syncs"] == ws["syncs"]
    key = "errors_corrected" if nc == 3 else "dwc_detected"
    assert gs[key] <= ws[key]
    assert int(status.sum()) == (gs[key] if nc > 1 else 0)
    if plan != "none":
        assert gs["injected"] > 0 and (nc == 1 or gs[key] > 0)


def exceptions(oracle, nc, A, B, kw):
    """the units of the documented exception: TMR's select voter, a bit-31 flip on replica 0 of a nonzero value that rounds to
    zero (a flipped zero is -0, which `fcmp oeq` takes for +0 in fp32 too)"""
    if nc != 3 or kw["flags"] & ref.F_MAJORITY_VOTER or kw["plan"] is None:
        return np.zeros(0, dtype=np.int64)
    acc = ref.clean_acc(oracle, A, B).ravel()
    fl = ref.sref.faults(oracle, kw["plan"], 3, K, M * N, kw["unit_base"])
    w = acc.view(np.uint32)
    return np.array([u for u, r, bit in fl if r == 0 and bit == 31 and w[u] & 0x7FFFFFFF and ref.rne(w[u:u + 1])[0] & 0x7FFF == 0],
                    dtype=np.int64)


# ------------------------------------------------------------------------------------------ by hand
def one_flip(oracle, u, replica, bit):
    tab = np.zeros(M * N, dtype=np.uint32)
    tab[u] = oracle.fault_entry(replica, 0, bit)
    return oracle.make_plan(oracle.PLAN_TABLE, table=tab)


def constant(a, b=1.0):
    """every accumulator a * b: A[:, 0] = a, B[0, :] = b, the rest zero"""
    A, B = np.zeros((M, K), dtype=np.uint16), np.zeros((K, N), dtype=np.uint16)
    A[:, 0], B[0, :] = ref.bits(np.float32(a)), ref.bits(np.float32(b))
    return A, B


def test_ties_round_to_even():
    """sums of exact float16 values that land on ties: 2049 = 2048 + 1 (even below), 2051 (odd below) and 4097 + 2"""
    A = np.zeros((M, K), dtype=np.uint16)
    B = np.zeros((K, N), dtype=np.uint16)
    A[0, :3] = ref.bits(np.float32([2048, 1, 0]))
    A[1, :3] = ref.bits(np.float32([2048, 2, 1]))
    A[2, :3] = ref.bits(np.float32([4096, 4, 2]))
    B[:3, 0] = ref.bits(np.float32([1, 1, 1]))
    acc = (ref.value(A).astype(np.float64) @ ref.value(B).astype(np.float64)).astype(np.float32)
    assert acc[0, 0] == 2049 and acc[1, 0] == 2051 and acc[2, 0] == 4102
    got = ref.rne(acc.ravel().view(np.uint32)).reshape(M, N)[:3, 0]
    assert list(got) == [int(ref.bits(np.float32(x))) for x in (2048, 2052, 4104)]


@pytest.mark.parametrize("nc", [1, 2, 3])
def test_65504_stays_finite_and_65520_overflows_to_infinity(oracle, nc):
    A, B = constant(32752.0, 2.0)                                   # 65504: the largest finite float16
    out, st, status = ref.run_f16(oracle, nc, A, B)
    assert (out.reshape(M, N)[:, 0] == 0x7BFF).all() and not status.any()
    A[:, 1] = ref.bits(np.float32(8.0))                             # + 8 * 2 = 65520: the tie above it, to infinity
    B[1, :] = ref.bits(np.float32(2.0))
    out, st, status = ref.run_f16(oracle, nc, A, B)
    assert (out == 0x7C00).all() and not status.any() and st["errors_corrected"] == st["dwc_detected"] == 0
    A[:, 0] = ref.bits(np.float32(-32752.0))                         # -65504 - (-16) is -65520: -infinity
    A[:, 1] = ref.bits(np.float32(-8.0))
    out, _, _ = ref.run_f16(oracle, nc, A, B)
    assert (out == 0xFC00).all()


def test_subnormal_results_are_kept(oracle):
    """2^-12 x 2^-12 = 2^-24, the smallest float16 subnormal; 3 x 2^-25 rounds up to 2^-23; 2^-26 rounds to zero"""
    A, B = constant(2.0 ** -12, 2.0 ** -12)
    out, _, _ = ref.run_f16(oracle, 3, A, B)
    assert (out == 0x0001).all()
    A, B = constant(3 * 2.0 ** -13, 2.0 ** -12)
    out, _, _ = ref.run_f16(oracle, 3, A, B)
    assert (out == 0x0002).all()
    A, B = constant(2.0 ** -13, -(2.0 ** -13))
    out, _, _ = ref.run_f16(oracle, 3, A, B)
    assert (out == 0x8000).all()


@pytest.mark.parametrize("nc", [2, 3])
def test_a_flip_below_f16_precision_is_injected_but_not_counted(oracle, nc):
    A, B = constant(3.0)
    u = 4 * N + 7
    for bit in (0, 7, 12):                                          # 3.0 + 2^-22 .. 2^-10 (a tie, to even) rounds back to 3.0
        out, st, status = ref.run_f16(oracle, nc, A, B, plan=one_flip(oracle, u, 1, bit))
        assert st["injected"] == 1 and st["errors_corrected"] == st["dwc_detected"] == 0 and not status.any(), bit
        assert (out == 0x4200).all() and st["first_fault_unit"] == ref.NO_FAULT_UNIT


@pytest.mark.parametrize("nc", [2, 3])
@pytest.mark.parametrize("bit", [13, 22, 30])
def test_a_flip_that_changes_the_rounded_value_is_counted(oracle, nc, bit):
    A, B = constant(3.0)
    u = 4 * N + 7
    out, st, status = ref.run_f16(oracle, nc, A, B, plan=one_flip(oracle, u, 1, bit))
    assert st["injected"] == 1 and (st["errors_corrected"] if nc == 3 else st["dwc_detected"]) == 1
    assert status[u] == 1 and status.sum() == 1 and st["first_fault_unit"] == u
    assert (out == 0x4200).all()                                    # replica 0 wins under DWC and TMR


@pytest.mark.parametrize("voter", [0, ref.F_MAJORITY_VOTER])
@pytest.mark.parametrize("replica", [0, 1, 2])
def test_a_sign_flip_of_a_value_that_rounds_to_zero(oracle, replica, voter):
    """accumulators 2^-30: below half the smallest float16 subnormal.  The sign flip makes -2^-30, which rounds to -0; -0 and +0
    agree, so nothing is counted, and the select voter stores replica 0's zero -- the exception to the identity when replica 0
    is flipped -- while the majority voter stores the two +0"""
    A, B = constant(2.0 ** -15, 2.0 ** -15)
    u = 3 * N + 2
    pl = one_flip(oracle, u, replica, 31)
    want, ws = ref.run(oracle, 3, A, B, plan=pl, flags=3 | voter)
    got, gs, status = ref.run_f16(oracle, 3, A, B, plan=pl, flags=3 | voter)
    assert ws["errors_corrected"] == 1 and gs["errors_corrected"] == 0 and gs["injected"] == 1 and not status.any()
    assert (np.delete(got, u) == 0).all() and ref.rne(want)[u] == 0x0000
    assert got[u] == (0x8000 if replica == 0 and not voter else 0x0000)


def test_the_majority_voter_works_on_the_16_bit_patterns(oracle):
    """a flip the rounding keeps on a subnormal result: replica 1's 2^-24 becomes 2^-24 + 2^-40 (bit 16 of the fp32 word
    0x33800000 is a mantissa bit), which rounds back to 0x0001; a flip of bit 28 makes 2^-56, which rounds to +0 and which the
    two agreeing replicas outvote bit by bit on the 16-bit patterns"""
    A, B = constant(2.0 ** -12, 2.0 ** -12)
    u = 5
    for bit, counted in ((16, 0), (28, 1)):
        got, gs, status = ref.run_f16(oracle, 3, A, B, plan=one_flip(oracle, u, 1, bit), flags=3 | ref.F_MAJORITY_VOTER)
        assert (got == 0x0001).all() and gs["errors_corrected"] == counted and int(status.sum()) == counted
