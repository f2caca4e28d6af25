"""The CPU reference of COAST_K_GEMM_F16 and of its FP16 output (COAST_MM_OUT_F16), shared by tests/test_gemm_f16_oracle.py and
tests/test_gpu_gemm_f16.py.

Operands are uint16 bit patterns of IEEE binary16, which numpy calls float16.  Every float16 -- subnormals, infinities and NaNs
included -- widens exactly to an fp32 with at most 11 significant bits, and the TF32 truncation of the oracle's GEMM_TF32
element (the top 19 bits: sign, 8 exponent and 10 mantissa bits) leaves it as it is.  GEMM_F16's definition -- exact products,
fp32 accumulation, one fault site of width 32 on the final accumulator, one fp32 vote per element -- is therefore GEMM_TF32's on
the widened operands, exactly as for GEMM_BF16 (tests/gemm_bf16_ref.py): oracle.run(K_GEMM_TF32) sums the exact products in
double and rounds once, bit-exact against the device wherever every partial sum is exactly representable in fp32
(integer-valued operands with K amax^2 < 2^24) and a tolerance reference otherwise.

FP16 output (include/coast_rt.h, DESIGN.md §3.15) is the BF16-output reference (tests/gemm_out_bf16_ref.py) with f16 for bf16:
each replica's accumulator after the fault hook is rounded to nearest even by numpy's float32 -> float16 conversion (subnormals
kept, finite values of 65520 or more in magnitude to infinities) and every NaN becomes NAN_F16.  The compares and counters are
tests/gemm_fp8_scaled_ref.py's voter run on the widened values (`fcmp oeq`); the majority voter works on the 16-bit patterns,
which for f16, unlike bf16, is not the same as on the widened fp32 patterns (a subnormal's exponent field changes on widening)."""
import numpy as np

import gemm_fp8_scaled_ref as sref

F_COUNT_ERRORS, F_COUNT_SYNCS, F_MAJORITY_VOTER = sref.F_COUNT_ERRORS, sref.F_COUNT_SYNCS, sref.F_MAJORITY_VOTER
NO_FAULT_UNIT = sref.NO_FAULT_UNIT
NAN_F16 = 0x7FFF           # the canonical NaN of the device's cvt.rn.f16x2.f32 (measured on an H100, DESIGN.md §3.15)


def bits(x):
    """float32 array -> float16 bit patterns (uint16); only for values a float16 holds exactly"""
    x = np.asarray(x, dtype=np.float32)
    h = x.astype(np.float16)
    assert np.array_equal(h.astype(np.float32), x, equal_nan=True), "not a float16 value"
    return h.view(np.uint16)


def value(h):
    """float16 bit patterns -> the fp32 values they stand for, bit for bit"""
    return np.asarray(h, dtype=np.uint16).view(np.float16).astype(np.float32)


def int_operands(rng, M, N, K, amax=16, *, rows_a=None):
    """integer operands in [-amax, amax] with K amax^2 < 2^24: every partial sum is an integer fp32 holds exactly"""
    assert K * amax * amax < 2 ** 24
    return (bits(rng.integers(-amax, amax + 1, (rows_a or M, K)).astype(np.float32)),
            bits(rng.integers(-amax, amax + 1, (K, N)).astype(np.float32)))


def run(oracle, nc, A, B, *, flags=3, plan=None, unit_base=0, threads=1):
    """fp32 C: A (M x K) and B (K x N) uint16 -> (C bits as uint32, flat; stats dict)"""
    assert A.dtype == np.uint16 and B.dtype == np.uint16
    M, K = A.shape
    N = B.shape[1]
    o, st = oracle.run(oracle.K_GEMM_TF32, nc, value(A), M * N, M=M, N=N, K=K, aux=value(B), flags=flags, plan=plan,
                       unit_base=unit_base, threads=threads)
    return o.view(np.uint32), st


def rne(w):
    """fp32 bit patterns (uint32) -> float16 bit patterns (uint16), round to nearest, ties to even; every NaN becomes NAN_F16"""
    w = np.asarray(w, dtype=np.uint32)
    with np.errstate(all="ignore"):
        r = w.view(np.float32).astype(np.float16).view(np.uint16)
    nan = (w & 0x7FFFFFFF) > 0x7F800000
    return np.where(nan, np.uint16(NAN_F16), r).astype(np.uint16)


def widen(h):
    """float16 bit patterns -> the fp32 bit patterns of the same values (exact)"""
    return value(h).view(np.uint32)


def run_acc(oracle, nc, acc, K, *, flags=3, plan=None, unit_base=0):
    """f16 C: acc, the clean fp32 accumulators of one product (M x N) -> (C as float16 bit patterns, uint16, flat; stats dict;
    d_status bytes as uint8)"""
    acc = np.ascontiguousarray(acc, dtype=np.float32)
    n = acc.size
    x = np.repeat(acc.reshape(1, n).view(np.uint32), nc, axis=0)
    fl = sref.faults(oracle, plan, nc, K, n, unit_base)
    for u, r, bit in fl:
        x[r, u] ^= np.uint32(1 << bit)
    v = rne(x)                                                  # every replica rounds its own value
    _, bad, st = sref.vote(widen(v), nc, flags, unit_base)      # compares and counters on the widened values
    out = v[0]
    if nc == 3:
        f = value(v)
        out = (v[0] & v[1]) | (v[0] & v[2]) | (v[1] & v[2]) if flags & F_MAJORITY_VOTER else np.where(f[0] == f[1], v[0], v[2])
    st["injected"] = len(fl)
    status = (bad if nc > 1 else np.zeros(n, dtype=bool)).astype(np.uint8)
    return out.astype(np.uint16), st, status


def clean_acc(oracle, A, B):
    """the fault-free fp32 C of GEMM_F16, as float32 (M x N)"""
    c, _ = run(oracle, 1, A, B, flags=0)
    return c.view(np.float32).reshape(A.shape[0], B.shape[1])


def run_f16(oracle, nc, A, B, **kw):
    """GEMM_F16 with COAST_MM_OUT_F16: A (M x K) and B (K x N) float16 bit patterns"""
    return run_acc(oracle, nc, clean_acc(oracle, A, B), A.shape[1], **kw)
