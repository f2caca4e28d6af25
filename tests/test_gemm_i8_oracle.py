"""The CPU reference of COAST_K_GEMM_I8 (tests/gemm_i8_ref.py).  Pinned here: the fault-free reference equals the oracle's
MM_U32 element (matrix_multiply, exact mod 2^32) on the sign-extended operands, including sums that wrap past 2^31 and 2^32; the
integer vote by hand on the words where an fp32 vote goes wrong -- a bit-31 flip of a zero C (0x80000000 is -0.0) and flips of
C = -1 and other NaN patterns -- under DWC and TMR with both voters, every store and counter written out; and the runtime's
per-unit numbers for the new id, with ids 9 and 11 still unassigned."""
import numpy as np
import pytest

import gemm_fp8_scaled_ref
import gemm_i8_ref as ref

K_GEMM_I8 = 12
NO_FAULT = 2 ** 64 - 1


def mm_u32(oracle, A, B):
    """the oracle's MM_U32 on A and B sign-extended to 32 bits -> C as uint32, flat"""
    M, K = A.shape
    N = B.shape[1]
    a, b = A.astype(np.int32).view(np.uint32), B.astype(np.int32).view(np.uint32)
    out, st = oracle.run(oracle.K_MM_U32, 1, a, M * N, M=M, N=N, K=K, aux=b)
    return out.view(np.uint32)


@pytest.mark.parametrize("M,N,K", [(5, 7, 128), (3, 9, 2048), (16, 4, 31), (1, 1, 1)])
def test_fault_free_reference_equals_mm_u32_on_sign_extended_operands(oracle, M, N, K):
    rng = np.random.default_rng(K)
    A = rng.integers(-128, 128, size=(M, K)).astype(np.int8)
    B = rng.integers(-128, 128, size=(K, N)).astype(np.int8)
    want = mm_u32(oracle, A, B)
    assert np.array_equal(ref.exact(A, B).ravel(), want)
    for nc in (1, 2, 3):
        out, st, status = ref.run(oracle, nc, A, B)
        assert np.array_equal(out, want) and not status.any()
        assert st == dict(errors_corrected=0, dwc_detected=0, syncs=M * N if nc == 3 else 0, injected=0, first_fault_unit=NO_FAULT)


@pytest.mark.parametrize("K,want", [(2 ** 17, -2 ** 31), (2 ** 17 + 128, -2 ** 31 + 2 ** 21), (2 ** 18 + 64, 2 ** 20),
                                    (130688, 2141192192)])
def test_sums_past_two_to_the_31_wrap_like_mm_u32(oracle, K, want):
    """all -128: every product is 2^14 and the sum 2^14 K, which passes 2^31 from K = 2^17 and 2^32 from K = 2^18"""
    A = np.full((2, K), -128, dtype=np.int8)
    B = np.full((K, 3), -128, dtype=np.int8)
    c = ref.exact(A, B).ravel()
    assert (c.view(np.int32) == want).all()
    assert np.array_equal(c, mm_u32(oracle, A, B))
    # mixed signs: the sums wrap in both directions
    rng = np.random.default_rng(1)
    A = np.where(rng.random((2, 2 ** 17 + 256)) < 0.9, -128, 127).astype(np.int8)
    B = np.where(rng.random((2 ** 17 + 256, 3)) < 0.5, -128, 127).astype(np.int8)
    assert np.array_equal(ref.exact(A, B).ravel(), mm_u32(oracle, A, B))


def one(oracle, nc, word, replica, bit, flags=3):
    """a 1 x 2 C of the given word in both elements, a TABLE flip of `bit` on `replica` of element 0 -> (stores, stats, status)"""
    A, B = np.zeros((1, 128), dtype=np.int8), np.zeros((128, 2), dtype=np.int8)
    table = np.array([oracle.fault_entry(replica, 0, bit), 0], dtype=np.uint32)
    plan = oracle.make_plan(oracle.PLAN_TABLE, table=table)
    out, st, status = ref.run(oracle, nc, A, B, flags=flags, plan=plan, table=table, unit_base=40,
                              acc=np.array([word, word], dtype=np.uint32))
    return out.tolist(), st, status.tolist()


def stats(**kw):
    return {**dict(errors_corrected=0, dwc_detected=0, syncs=0, injected=1, first_fault_unit=NO_FAULT), **kw}


MAJ = 3 | ref.F_MAJORITY_VOTER


def test_bit_31_flip_of_a_zero_c_by_hand(oracle):
    """0x80000000 is -0.0 to fp32 and equals +0.0 under `fcmp oeq`; the integer vote sees two different words"""
    INT_MIN = 0x80000000
    # DWC stores replica 0 and detects the flip, wherever it lands
    assert one(oracle, 2, 0, 0, 31) == ([INT_MIN, 0], stats(dwc_detected=1, first_fault_unit=40), [1, 0])
    assert one(oracle, 2, 0, 1, 31) == ([0, 0], stats(dwc_detected=1, first_fault_unit=40), [1, 0])
    # TMR, select voter: r0 != r1 stores r2; r0 == r1 stores r0; counted either way
    for r in (0, 1, 2):
        assert one(oracle, 3, 0, r, 31) == ([0, 0], stats(errors_corrected=1, syncs=2, first_fault_unit=40), [1, 0]), r
        assert one(oracle, 3, 0, r, 31, MAJ) == ([0, 0], stats(errors_corrected=1, syncs=2, first_fault_unit=40), [1, 0]), r
    # unprotected: the flip is stored and nothing is counted
    assert one(oracle, 1, 0, 0, 31) == ([INT_MIN, 0], stats(), [0, 0])
    # what the fp32 vote would have done: no disagreement, and TMR's select voter keeps replica 0's INT_MIN
    v = np.array([[INT_MIN], [0], [0]], dtype=np.uint32)
    out, bad, _ = gemm_fp8_scaled_ref.vote(v, 3, 3, 0)
    assert out.tolist() == [INT_MIN] and not bad.any()
    _, bad, _ = gemm_fp8_scaled_ref.vote(v[:2], 2, 3, 0)
    assert not bad.any()


@pytest.mark.parametrize("word", [0xFFFFFFFF, 0xFF800001, 0xFFC00000, 0x7F800001, 0x7FA00000, 0x7FFFFFFF])
def test_flips_of_nan_pattern_words_by_hand(oracle, word):
    """C = -1, -8388607, -4194304, 2139095041, 2141192192 and 2147483647: NaN patterns to fp32, plain integers here"""
    for bit in (0, 22, 31):
        x = word ^ (1 << bit)
        assert one(oracle, 2, word, 0, bit) == ([x, word], stats(dwc_detected=1, first_fault_unit=40), [1, 0])
        assert one(oracle, 2, word, 1, bit) == ([word, word], stats(dwc_detected=1, first_fault_unit=40), [1, 0])
        for r in (0, 1, 2):
            for flags in (3, MAJ):
                assert one(oracle, 3, word, r, bit, flags) == ([word, word], stats(errors_corrected=1, syncs=2, first_fault_unit=40),
                                                               [1, 0]), (r, bit, flags)
    # without a fault the replicas agree: nothing is counted (the fp32 vote would count every NaN pattern as a disagreement)
    A, B = np.zeros((1, 128), dtype=np.int8), np.zeros((128, 2), dtype=np.int8)
    for nc in (2, 3):
        out, st, status = ref.run(oracle, nc, A, B, acc=np.array([word, word], dtype=np.uint32))
        assert out.tolist() == [word, word] and not status.any()
        assert st == stats(injected=0, syncs=2 if nc == 3 else 0)
    _, bad, _ = gemm_fp8_scaled_ref.vote(np.array([[word], [word], [word]], dtype=np.uint32), 3, 3, 0)
    assert bad.all()


def test_per_unit_numbers_equal_gemm_tf32s_and_ids_9_and_11_are_unassigned(oracle, built_lib):
    """the runtime's numbers for the new id against the oracle's for GEMM_TF32 (no driver is needed to ask)"""
    from coast_b200 import runtime as R
    L, t = R.load_library(), oracle.K_GEMM_TF32
    assert R.K_GEMM_I8 == K_GEMM_I8 and R.OUT_BYTES[K_GEMM_I8] == 4 and R.MM_ELEM_BYTES[K_GEMM_I8] == 1
    assert L.coast_fault_sites(K_GEMM_I8, 0, 128) == oracle.fault_sites(t, 0, 128) == 1
    assert L.coast_fault_site_bits(K_GEMM_I8, 0, 128, 0) == oracle.fault_site_bits(t, 0, 128, 0) == 32
    assert L.coast_out_bytes_per_unit(K_GEMM_I8) == oracle.out_bytes_per_unit(t) == 4
    assert L.coast_votes_per_unit(K_GEMM_I8) == oracle.votes_per_unit(t) == 1
    assert L.coast_flags_honoured(K_GEMM_I8, 3, 0x200 | 0x4) == 0 and L.coast_flags_honoured(K_GEMM_I8, 3, 0x400 | 0x1) == 0x401
    for k in (9, 11, 13):
        assert L.coast_out_bytes_per_unit(k) == L.coast_votes_per_unit(k) == L.coast_fault_sites(k, 0, 128) == 0


def test_python_refuses_scales_and_bf16_output_before_the_library():
    from coast_b200 import runtime as R
    for mode, sa in ((R.MM_SCALE_TENSOR, None), (R.MM_SCALE_ROWWISE, None), (R.MM_OUT_BF16, None), (0, 1)):
        with pytest.raises(R.CoastError) as e:
            R.Runtime._check_i8(R.K_GEMM_I8, mode, sa, None)
        assert e.value.code == R.ERR_BAD_ARG and "K_GEMM_I8" in str(e.value)
    R.Runtime._check_i8(R.K_GEMM_I8, R.MM_BATCHED | R.MM_B_TRANSPOSED, None, None)
    R.Runtime._check_i8(R.K_GEMM_FP8, R.MM_SCALE_TENSOR, 1, 1)
