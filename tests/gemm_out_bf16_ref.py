"""The CPU reference of matmuls with BF16 output (COAST_MM_OUT_BF16), built on tests/gemm_bf16_ref.py, tests/gemm_fp8_ref.py
and the fault plan and voter of tests/gemm_fp8_scaled_ref.py.

Definition (include/coast_rt.h, DESIGN.md §3.13): element (i, j) of replica r is x_r, the accumulator after the fault hook;
the replica rounds it to bfloat16, round to nearest even, v_r = bf16(x_r).  The
vote, the counters and d_status work on v_0 .. v_{NC-1} as the fp32-output launch's do on x_r.  This restates it step by step:
  * the clean accumulators are the fp32-output references' (GEMM_BF16 and GEMM_FP8 at NC 1 without a plan), so this
    reference is bit-exact where they are;
  * each unit's fault (active, replica, bit) is the oracle's own fault_for_unit for a one-site, 32-bit kernel, so Bernoulli and
    TABLE plans draw the faults of the fp32-output launch;
  * the flip lands on the accumulator, then `rne` rounds each replica's value;
  * the select or bitwise majority voter with `fcmp oeq` on the widened values (NaN disagrees with everything, +0 and -0 agree),
    and the five counters: the fp32 reference's voter run on the widened bfloat16 values.
A NaN rounds to NAN_BF16, the one pattern the device's cvt.rn.bf16x2.f32 writes for every NaN input."""
import numpy as np

import gemm_bf16_ref
import gemm_fp8_ref
import gemm_fp8_scaled_ref as sref

F_COUNT_ERRORS, F_COUNT_SYNCS, F_MAJORITY_VOTER = sref.F_COUNT_ERRORS, sref.F_COUNT_SYNCS, sref.F_MAJORITY_VOTER
NO_FAULT_UNIT = sref.NO_FAULT_UNIT
NAN_BF16 = 0x7FFF          # the canonical NaN of the device's conversion (measured on an H100, DESIGN.md §3.13)


def rne(w):
    """fp32 bit patterns (uint32) -> bfloat16 bit patterns (uint16), round to nearest, ties to even.  Subnormals are kept, a
    value that rounds past the largest finite bfloat16 becomes an infinity, and every NaN becomes NAN_BF16."""
    w = np.asarray(w, dtype=np.uint32).astype(np.uint64)
    r = ((w + 0x7FFF + ((w >> 16) & 1)) >> 16).astype(np.uint16)
    nan = (w & 0x7FFFFFFF) > 0x7F800000
    return np.where(nan, np.uint16(NAN_BF16), r).astype(np.uint16)


def widen(h):
    """bfloat16 bit patterns -> the fp32 bit patterns of the same values (exact)"""
    return np.asarray(h, dtype=np.uint16).astype(np.uint32) << 16


def run_acc(oracle, nc, acc, K, *, flags=3, plan=None, unit_base=0):
    """acc: the clean fp32 accumulators of one product (M x N).  Returns (C as bfloat16 bit patterns, uint16, flat; stats dict;
    d_status bytes as uint8)."""
    acc = np.ascontiguousarray(acc, dtype=np.float32)
    M, N = acc.shape
    n = M * N
    x = np.repeat(acc.reshape(1, n).view(np.uint32), nc, axis=0)
    fl = sref.faults(oracle, plan, nc, K, n, unit_base)
    for u, r, bit in fl:
        x[r, u] ^= np.uint32(1 << bit)
    v = rne(x)                                                  # every replica rounds its own value
    out, bad, st = sref.vote(widen(v), nc, flags, unit_base)
    st["injected"] = len(fl)
    status = (bad if nc > 1 else np.zeros(n, dtype=bool)).astype(np.uint8)
    return (out >> 16).astype(np.uint16), st, status


def clean_acc(ref, oracle, A, B):
    """the fault-free fp32 C of gemm_bf16_ref or gemm_fp8_ref, as float32 (M x N)"""
    c, _ = ref.run(oracle, 1, A, B, flags=0)
    return c.view(np.float32).reshape(A.shape[0], B.shape[1])


def run_bf16(oracle, nc, A, B, **kw):
    """GEMM_BF16: A (M x K) and B (K x N) bfloat16 bit patterns"""
    return run_acc(oracle, nc, clean_acc(gemm_bf16_ref, oracle, A, B), A.shape[1], **kw)


def run_fp8(oracle, nc, A, B, **kw):
    """GEMM_FP8: A (M x K) and B (K x N) E4M3 bit patterns"""
    return run_acc(oracle, nc, clean_acc(gemm_fp8_ref, oracle, A, B), A.shape[1], **kw)
