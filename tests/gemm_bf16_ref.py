"""The CPU reference of COAST_K_GEMM_BF16, shared by tests/test_gemm_bf16_oracle.py and tests/test_gpu_gemm_bf16.py.

numpy has no bfloat16: operands are uint16 bit patterns.  A bfloat16 is an fp32 whose low 16 bits are zero, so widening is a
shift and exact for every pattern (zeros, denormals, infinities, NaNs), and the TF32 truncation of the oracle's GEMM_TF32
element (the top 19 bits of each operand) leaves a widened bfloat16 as it is.  GEMM_BF16's definition -- exact products of the
operands, accumulated in fp32 on the device, one fault site of width 32 on the final accumulator, one fp32 vote per element --
is therefore GEMM_TF32's on the widened operands, and that is the reference: oracle.run(K_GEMM_TF32) sums the exact products in
double and rounds once, which is bit-exact against the device wherever every partial sum is exactly representable in fp32
(integer-valued operands with K amax^2 < 2^24) and a tolerance reference otherwise."""
import numpy as np


def bits(x):
    """float32 array -> bfloat16 bit patterns (uint16); only for values a bfloat16 holds (8 significant bits)"""
    w = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    assert not (w & 0xFFFF).any()
    return (w >> 16).astype(np.uint16)


def value(b):
    """bfloat16 bit patterns -> the fp32 values they stand for, bit for bit"""
    return (np.asarray(b).astype(np.uint32) << 16).view(np.float32)


def run(oracle, nc, A, B, *, flags=3, plan=None, unit_base=0, threads=1):
    """A: (M x K) uint16, B: (K x N) uint16 -> (C bits as uint32, flat; stats dict)"""
    assert A.dtype == np.uint16 and B.dtype == np.uint16
    M, K = A.shape
    N = B.shape[1]
    o, st = oracle.run(oracle.K_GEMM_TF32, nc, value(A), M * N, M=M, N=N, K=K, aux=value(B), flags=flags, plan=plan,
                       unit_base=unit_base, threads=threads)
    return o.view(np.uint32), st
