"""The CPU reference of COAST_K_GEMM_FP8, shared by tests/test_gemm_fp8_oracle.py and tests/test_gpu_gemm_fp8.py.

numpy has no FP8: operands are uint8 bit patterns of E4M3, the OCP encoding torch.float8_e4m3fn uses (sign, 4 exponent bits
with bias 7, 3 mantissa bits; exponent 0 is subnormal, S.1111.111 is NaN and there are no infinities).  Every E4M3 value is an
fp32 with at most 4 significant bits and an exponent in [-9, 8], so widening is exact, and the TF32 truncation of the oracle's
GEMM_TF32 element (the top 19 bits of each operand) leaves it as it is.  GEMM_FP8's definition -- exact products, one fault
site of width 32 on the final accumulator, one fp32 vote per element -- is therefore GEMM_TF32's on the widened operands, and
that is the reference: oracle.run(K_GEMM_TF32) sums the exact products in double and rounds once.  The device sums in the
tensor core's FP8 accumulator, which keeps fewer bits than fp32 (DESIGN.md §6), so the reference is bit-exact only where every
partial sum is a small integer: integer-valued operands with sum_k |a_ik b_kj| <= 2^11."""
import numpy as np


def _decode(p):
    s = -1.0 if p & 0x80 else 1.0
    e, m = (p >> 3) & 0xF, p & 7
    if e == 15 and m == 7:
        return np.float32(np.nan)
    if e == 0:
        return np.float32(s * m * 2.0 ** -9)
    return np.float32(s * (8 + m) * 2.0 ** (e - 10))


# the fp32 value of every E4M3 pattern, bit for bit (both NaN patterns: a quiet NaN)
TABLE = np.array([_decode(p) for p in range(256)], dtype=np.float32)
TABLE[0x80] = np.float32(-0.0)
EXACT_SUM = 2 ** 11      # the largest sum_k |a_ik b_kj| of integer operands at which the device is held bit-exact


def value(b):
    """E4M3 bit patterns (uint8) -> the fp32 values they stand for"""
    return TABLE[np.asarray(b, dtype=np.uint8)]


def bits(x):
    """float32 array -> E4M3 bit patterns; only for values E4M3 holds exactly (no NaN)"""
    x = np.asarray(x, dtype=np.float32)
    order = np.argsort(TABLE[:0x7F])                      # the finite non-negative patterns 0x00..0x7E, ascending
    pos = TABLE[:0x7F][order]
    i = np.searchsorted(pos, np.abs(x))
    assert (i < len(pos)).all() and (pos[np.minimum(i, len(pos) - 1)] == np.abs(x)).all(), "not an E4M3 value"
    return (order[i].astype(np.uint8) | np.where(np.signbit(x), 0x80, 0).astype(np.uint8)).astype(np.uint8)


def int_operands(rng, M, N, K, amax, *, rows_a=None):
    """integer operands in [-amax, amax] with K amax^2 <= EXACT_SUM: every partial sum is an integer the device keeps exactly"""
    assert amax <= 16 and K * amax * amax <= EXACT_SUM
    return (bits(rng.integers(-amax, amax + 1, (rows_a or M, K)).astype(np.float32)),
            bits(rng.integers(-amax, amax + 1, (K, N)).astype(np.float32)))


def run(oracle, nc, A, B, *, flags=3, plan=None, unit_base=0, threads=1):
    """A: (M x K) uint8, B: (K x N) uint8 -> (C bits as uint32, flat; stats dict)"""
    assert A.dtype == np.uint8 and B.dtype == np.uint8
    M, K = A.shape
    N = B.shape[1]
    o, st = oracle.run(oracle.K_GEMM_TF32, nc, value(A), M * N, M=M, N=N, K=K, aux=value(B), flags=flags, plan=plan,
                       unit_base=unit_base, threads=threads)
    return o.view(np.uint32), st
