"""The CPU reference of a grouped matmul (COAST_MM_GROUPED): one oracle run per product, product g with M = ro[g+1] - ro[g],
its A rows, its own B and unit_base + (ro[g] - ro[0]) * N, concatenated over the products.  This is the definition the GPU
kernels are held to (include/coast_rt.h).  Pinned here against numpy: the u32 products exactly mod 2^32, the TF32 products on
integer-valued fp32 operands (exact in float64 and fp32), the summed counters, and the fault plan keyed by the global unit
index, so a product's faults do not depend on which other products share its launch."""
import numpy as np
import pytest

M32 = 0xFFFFFFFF


def grouped_oracle(oracle, kernel, nc, A, B, ro, N, K, *, flags=3, plan=None, base=0):
    """C rows [ro[0], ro[G]) and the summed stats of G single oracle runs"""
    outs, total = [], dict(errors_corrected=0, dwc_detected=0, syncs=0, injected=0, first_fault_unit=oracle.NO_FAULT_UNIT)
    for g in range(len(ro) - 1):
        m = ro[g + 1] - ro[g]
        if m == 0:
            continue
        out, st = oracle.run(kernel, nc, A[ro[g] * K:ro[g + 1] * K], m * N, flags=flags, M=m, N=N, K=K,
                             aux=B[g * K * N:(g + 1) * K * N], plan=plan, unit_base=base + (ro[g] - ro[0]) * N)
        outs.append(out)
        for k in ("errors_corrected", "dwc_detected", "syncs", "injected"):
            total[k] += st[k]
        total["first_fault_unit"] = min(total["first_fault_unit"], st["first_fault_unit"])
    return np.concatenate(outs), total


def u32_ref(A, B, ro, N, K):
    rows = []
    for g in range(len(ro) - 1):
        a = A[ro[g] * K:ro[g + 1] * K].reshape(-1, K).astype(np.uint64)
        b = B[g * K * N:(g + 1) * K * N].reshape(K, N).astype(np.uint64)
        c = np.zeros((a.shape[0], N), dtype=np.uint64)
        for k in range(K):                                   # mod 2^64 sums; the low 32 bits are the mod-2^32 product
            c += np.outer(a[:, k], b[k])
        rows.append((c & M32).astype(np.uint32))
    return np.concatenate(rows).reshape(-1)


RO = [4, 4, 9, 10, 10, 30, 31]


@pytest.mark.parametrize("nc", [1, 2, 3])
def test_u32_grouped_reference_is_the_exact_product(oracle, nc):
    N, K = 7, 5
    rng = np.random.default_rng(nc)
    A = rng.integers(0, 2 ** 32, RO[-1] * K, dtype=np.uint64).astype(np.uint32)
    B = rng.integers(0, 2 ** 32, (len(RO) - 1) * K * N, dtype=np.uint64).astype(np.uint32)
    out, st = grouped_oracle(oracle, oracle.K_MM_U32, nc, A, B, RO, N, K)
    assert np.array_equal(out.view(np.uint32), u32_ref(A, B, RO, N, K))
    n = (RO[-1] - RO[0]) * N
    assert st["injected"] == 0 and st["first_fault_unit"] == oracle.NO_FAULT_UNIT and st["syncs"] == (n if nc == 3 else 0)


@pytest.mark.parametrize("nc", [1, 3])
def test_tf32_grouped_reference_on_integer_valued_operands(oracle, nc):
    N, K = 6, 8
    rng = np.random.default_rng(10 + nc)
    A = rng.integers(-8, 9, RO[-1] * K).astype(np.float32)
    B = rng.integers(-8, 9, (len(RO) - 1) * K * N).astype(np.float32)
    out, _ = grouped_oracle(oracle, oracle.K_GEMM_TF32, nc, A, B, RO, N, K)
    ref = np.concatenate([A[RO[g] * K:RO[g + 1] * K].reshape(-1, K).astype(np.float64) @ B[g * K * N:(g + 1) * K * N].reshape(K, N)
                          for g in range(len(RO) - 1)]).reshape(-1)
    assert np.array_equal(out.view(np.float32).astype(np.float64), ref)


def test_a_products_faults_do_not_depend_on_its_neighbours(oracle):
    """Bernoulli plans are keyed by the global unit: running the last two products alone, with their own unit_base, gives
    the same bytes as the whole launch's tail"""
    N, K = 7, 5
    rng = np.random.default_rng(3)
    A = rng.integers(0, 2 ** 32, RO[-1] * K, dtype=np.uint64).astype(np.uint32)
    B = rng.integers(0, 2 ** 32, (len(RO) - 1) * K * N, dtype=np.uint64).astype(np.uint32)
    plan = oracle.make_plan(oracle.PLAN_BERNOULLI, seed=9, p=0.4)
    base = (1 << 32) - 50
    whole, st = grouped_oracle(oracle, oracle.K_MM_U32, 2, A, B, RO, N, K, plan=plan, base=base)
    lo = 4
    tail, _ = grouped_oracle(oracle, oracle.K_MM_U32, 2, A, B[lo * K * N:], RO[lo:], N, K, plan=plan,
                             base=base + (RO[lo] - RO[0]) * N)
    assert st["injected"] > 0 and st["dwc_detected"] > 0
    assert np.array_equal(whole[-len(tail):], tail)
