"""The CPU reference of scaled GEMM_FP8 (COAST_MM_SCALE_TENSOR / COAST_MM_SCALE_ROWWISE), built on tests/gemm_fp8_ref.py.

Definition (include/coast_rt.h): element (i, j) of replica r is v_r = (acc_r * sa_i) * sb_j, two fp32 multiplies rounded to
nearest, where acc_r is the replica's accumulator after the fault hook; the vote, the counters and d_status work on
v_0 .. v_{NC-1} as GEMM_FP8's do on acc_r.  This restates it step by step:
  * the accumulators are exact: integer-valued operands with sum_k |a_ik b_kj| <= gemm_fp8_ref.EXACT_SUM, summed in float64;
  * each unit's fault (active, replica, bit) is the oracle's own fault_for_unit for a one-site, 32-bit kernel (GEMM_TF32's
    geometry, which GEMM_FP8 shares), so Bernoulli and TABLE plans are the oracle's;
  * the flip lands on acc_r, then numpy multiplies in float32 (IEEE, round to nearest, subnormals kept);
  * the select voter or the bitwise majority voter, with `fcmp oeq` (NaN disagrees with everything), and the five counters."""
import numpy as np

import gemm_fp8_ref

F_COUNT_ERRORS, F_COUNT_SYNCS, F_MAJORITY_VOTER = 0x1, 0x2, 0x100
NO_FAULT_UNIT = 2 ** 64 - 1


def exact_acc(A, B):
    """A: (M x K), B: (K x N) E4M3 bit patterns in the exact domain -> the accumulators, float32 (M x N)"""
    a, b = gemm_fp8_ref.value(A).astype(np.float64), gemm_fp8_ref.value(B).astype(np.float64)
    assert (np.abs(a) @ np.abs(b)).max(initial=0) <= gemm_fp8_ref.EXACT_SUM, "outside the exact domain"
    return (a @ b).astype(np.float32)


def faults(oracle, plan, nc, K, n, unit_base):
    """(local unit, replica, bit) of every active fault of the plan over units [unit_base, unit_base + n)"""
    if plan is None:
        return []
    out = []
    for u in range(n):
        f = oracle.fault_for_unit(plan, oracle.K_GEMM_TF32, nc, 0, K, unit_base + u, u)
        if f is not None:
            out.append((u, f[0], f[2]))
    return out


def vote(v, nc, flags, unit_base):
    """v: (NC, n) scaled replica values as uint32 -> (voted uint32 (n,), per-unit disagreement (n,) bool, stats)"""
    f = v.view(np.float32)
    n = v.shape[1]
    bad = np.zeros(n, dtype=bool)
    out = v[0].copy()
    if nc == 2:
        bad = ~(f[0] == f[1])
    if nc == 3:
        c01, c02 = f[0] == f[1], f[0] == f[2]
        out = (v[0] & v[1]) | (v[0] & v[2]) | (v[1] & v[2]) if flags & F_MAJORITY_VOTER else np.where(c01, v[0], v[2])
        bad = ~(c01 & c02)
    st = dict(errors_corrected=0, dwc_detected=0, syncs=0, injected=0, first_fault_unit=NO_FAULT_UNIT)
    if nc == 3 and flags & F_COUNT_ERRORS:
        st["errors_corrected"] = int(bad.sum())
        if flags & F_COUNT_SYNCS:
            st["syncs"] = n
    if nc == 2:
        st["dwc_detected"] = int(bad.sum())
    if nc > 1 and bad.any():
        st["first_fault_unit"] = unit_base + int(np.flatnonzero(bad)[0])
    return out, bad, st


def run(oracle, nc, A, B, sa, sb, *, flags=3, plan=None, unit_base=0, acc=None):
    """one product: A (M x K) and B (K x N) E4M3 bit patterns, sa (M,) and sb (N,) float32 scales (np.broadcast_to a scalar for
    tensorwise).  acc: the accumulators, when the caller has them exactly (default: exact_acc).  Returns (C bits as uint32, flat;
    stats dict; d_status bytes as uint8)."""
    M, K = A.shape
    N = B.shape[1]
    acc = exact_acc(A, B) if acc is None else np.asarray(acc, dtype=np.float32)
    n = M * N
    v = np.repeat(acc.reshape(1, n).view(np.uint32), nc, axis=0)
    fl = faults(oracle, plan, nc, K, n, unit_base)
    for u, r, bit in fl:
        v[r, u] ^= np.uint32(1 << bit)
    sa = np.broadcast_to(np.asarray(sa, dtype=np.float32), (M,))
    sb = np.broadcast_to(np.asarray(sb, dtype=np.float32), (N,))
    with np.errstate(all="ignore"):
        scaled = (v.view(np.float32).reshape(nc, M, N) * sa[None, :, None]) * sb[None, None, :]
    out, bad, st = vote(scaled.astype(np.float32).reshape(nc, n).view(np.uint32), nc, flags, unit_base)
    st["injected"] = len(fl)
    status = (bad if nc > 1 else np.zeros(n, dtype=bool)).astype(np.uint8)
    return out, st, status
