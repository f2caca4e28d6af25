"""The CPU reference of COAST_K_GEMM_FP8 (tests/gemm_fp8_ref.py): E4M3 operands as uint8 bit patterns, widened exactly to fp32
and run through the oracle's GEMM_TF32 element, whose TF32 truncation leaves a widened E4M3 value unchanged.  Pinned here: the
decode table against torch.float8_e4m3fn on all 256 patterns; that widening and truncation are exact; the reference against a
float64 numpy matmul on integer-valued operands of the exact domain; NaN operands reaching the element; the runtime's per-unit
numbers for the new id, and that id 9 stays unassigned."""
import numpy as np
import pytest

import gemm_fp8_ref as ref8
from gemm_fp8_ref import bits, value

K_GEMM_FP8 = 10


def test_decode_table_equals_torch_float8_e4m3fn_on_every_pattern():
    import torch
    t = torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn).float().numpy()
    nan = np.isnan(t)
    assert np.flatnonzero(nan).tolist() == [0x7F, 0xFF] and np.array_equal(np.isnan(ref8.TABLE), nan)
    assert np.array_equal(t[~nan].view(np.uint32), ref8.TABLE[~nan].view(np.uint32))      # signed zeros and subnormals included
    assert ref8.TABLE[0x7E] == 448 and ref8.TABLE[0x01] == 2.0 ** -9 and ref8.TABLE[0x08] == 2.0 ** -6
    assert str(ref8.TABLE[0x80]) == "-0.0"
    # torch's own rounding lands on the same patterns
    x = ref8.TABLE[~nan]
    assert np.array_equal(torch.from_numpy(x).to(torch.float8_e4m3fn).view(torch.uint8).numpy(), np.arange(256)[~nan])
    assert np.array_equal(bits(x), np.arange(256)[~nan].astype(np.uint8))


def test_widening_is_exact_and_survives_tf32_truncation():
    """at most 4 significant bits: nothing below the 19 bits TF32 reads, and every integer |x| <= 16 is an E4M3 value"""
    w = ref8.TABLE.view(np.uint32)
    assert not (w & 0x1FFF).any() and not (w & 0xFFFFF).any()
    ints = np.arange(-16, 17, dtype=np.float32)
    assert np.array_equal(value(bits(ints)), ints)


@pytest.mark.parametrize("M,N,K,amax", [(5, 7, 128, 4), (3, 130, 2048, 1), (17, 9, 512, 2), (2, 2, 8, 16)])
def test_elements_equal_the_float64_matmul_on_integer_valued_operands(oracle, M, N, K, amax):
    A, B = ref8.int_operands(np.random.default_rng(K), M, N, K, amax)
    ref = value(A).astype(np.float64) @ value(B).astype(np.float64)
    assert (np.abs(value(A)).astype(np.float64) @ np.abs(value(B)).astype(np.float64)).max() <= ref8.EXACT_SUM
    out, st = ref8.run(oracle, 1, A, B)
    assert np.array_equal(out.view(np.float32).reshape(M, N).astype(np.float64), ref)
    assert st == dict(errors_corrected=0, dwc_detected=0, syncs=0, injected=0, first_fault_unit=oracle.NO_FAULT_UNIT)


def test_nan_operands_reach_the_element(oracle):
    A = np.array([[0x7F, 0x38], [0x38, 0x00]], dtype=np.uint8)            # NaN, 1 / 1, 0
    B = np.array([[0x38, 0x00], [0x38, 0x38]], dtype=np.uint8)
    c = ref8.run(oracle, 1, A, B)[0].view(np.float32)
    assert np.isnan(c[0]) and np.isnan(c[1]) and c[2] == 1.0 and c[3] == 0.0


def test_per_unit_numbers_equal_gemm_tf32s_and_id_9_is_unassigned(oracle, built_lib):
    """the runtime's numbers for the new id against the oracle's for GEMM_TF32 (no driver is needed to ask)"""
    from coast_b200 import runtime as R
    L, t = R.load_library(), oracle.K_GEMM_TF32
    assert R.K_GEMM_FP8 == K_GEMM_FP8 and R.OUT_BYTES[K_GEMM_FP8] == 4
    assert L.coast_fault_sites(K_GEMM_FP8, 0, 128) == oracle.fault_sites(t, 0, 128) == 1
    assert L.coast_fault_site_bits(K_GEMM_FP8, 0, 128, 0) == oracle.fault_site_bits(t, 0, 128, 0) == 32
    assert L.coast_out_bytes_per_unit(K_GEMM_FP8) == oracle.out_bytes_per_unit(t) == 4
    assert L.coast_votes_per_unit(K_GEMM_FP8) == oracle.votes_per_unit(t) == 1
    assert L.coast_flags_honoured(K_GEMM_FP8, 3, 0x200 | 0x4) == 0 and L.coast_flags_honoured(K_GEMM_FP8, 3, 0x400 | 0x1) == 0x401
    assert L.coast_out_bytes_per_unit(9) == L.coast_votes_per_unit(9) == L.coast_fault_sites(9, 0, 128) == 0
    assert L.coast_out_bytes_per_unit(11) == 0
