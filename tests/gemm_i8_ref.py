"""The CPU reference of COAST_K_GEMM_I8: int8 A and B, int32 C, exact mod 2^32, integer vote.

Definition (include/coast_rt.h): element (i, j) of replica r is acc_r = sum_k a_ik b_kj mod 2^32 after the fault hook; the vote is
integer equality on the 32-bit words, with the select voter r0 == r1 ? r0 : r2 or the bitwise majority, and the five counters and
d_status follow it as for the other GEMMs.  This restates it step by step:
  * the product is exact: the sum is formed in float64, exact because |sum| <= 2^14 K < 2^53, taken to int64 and reduced mod 2^32;
  * each unit's fault (active, replica, bit) is the oracle's own fault_for_unit for a one-site, 32-bit kernel (GEMM_TF32's
    geometry, which GEMM_I8 shares), so Bernoulli and TABLE plans are the oracle's;
  * the flip lands on the replica's word, then the integer vote and the counters."""
import numpy as np

F_COUNT_ERRORS, F_COUNT_SYNCS, F_MAJORITY_VOTER = 0x1, 0x2, 0x100
NO_FAULT_UNIT = 2 ** 64 - 1


def exact(A, B):
    """A: (M x K) int8, B: (K x N) int8 -> C (M x N) as uint32, the two's-complement words of sum_k a_ik b_kj mod 2^32"""
    assert A.dtype == np.int8 and B.dtype == np.int8 and A.shape[1] < 2 ** 39
    s = A.astype(np.float64) @ B.astype(np.float64)
    return (s.astype(np.int64) & 0xFFFFFFFF).astype(np.uint32)


def faults(oracle, plan, nc, K, n, unit_base, table=None):
    """(local unit, replica, bit) of every active fault of the plan over units [unit_base, unit_base + n); with the TABLE plan's
    own table given, only its nonzero entries are asked about"""
    if plan is None:
        return []
    units = range(n) if table is None else np.flatnonzero(table[:n]).tolist()
    out = []
    for u in units:
        f = oracle.fault_for_unit(plan, oracle.K_GEMM_TF32, nc, 0, K, unit_base + u, u)
        if f is not None:
            out.append((u, f[0], f[2]))
    return out


def vote(v, nc, flags, unit_base):
    """v: (NC, n) replica words as uint32 -> (voted uint32 (n,), per-unit disagreement (n,) bool, stats).  `icmp eq`."""
    n = v.shape[1]
    bad = np.zeros(n, dtype=bool)
    out = v[0].copy()
    if nc == 2:
        bad = v[0] != v[1]
    if nc == 3:
        c01, c02 = v[0] == v[1], v[0] == v[2]
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


def run(oracle, nc, A, B, *, flags=3, plan=None, table=None, unit_base=0, acc=None):
    """one product: A (M x K) and B (K x N) int8.  acc: C's words when the caller has them (default: exact(A, B)); table: the
    TABLE plan's entries, to skip its empty ones.  Returns (C as uint32, flat; stats dict; d_status bytes as uint8)."""
    M, K = A.shape
    N = B.shape[1]
    acc = exact(A, B) if acc is None else np.asarray(acc, dtype=np.uint32)
    n = M * N
    v = np.repeat(acc.reshape(1, n), nc, axis=0)
    fl = faults(oracle, plan, nc, K, n, unit_base, table)
    for u, r, bit in fl:
        v[r, u] ^= np.uint32(1 << bit)
    out, bad, st = vote(v, nc, flags, unit_base)
    st["injected"] = len(fl)
    status = (bad if nc > 1 else np.zeros(n, dtype=bool)).astype(np.uint8)
    return out, st, status
