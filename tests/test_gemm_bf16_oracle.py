"""The CPU reference of COAST_K_GEMM_BF16 (tests/gemm_bf16_ref.py): bfloat16 operands as uint16 bit patterns, widened exactly to
fp32 and run through the oracle's GEMM_TF32 element, whose TF32 truncation leaves a widened bfloat16 unchanged.  Pinned here:
that widening and truncation are exact for all 65536 patterns; the reference against a float64 numpy matmul on integer-valued
operands, where every partial sum is an exact fp32 integer (|a| <= 256 and amax^2 K < 2^24) and equality is bit for bit;
infinities and NaNs reaching the element; that the runtime's per-unit numbers for the new kernel id equal the oracle's for
GEMM_TF32; the one fault site; and the batched / grouped references, single runs per product as for the other matmuls."""
import numpy as np
import pytest

import gemm_bf16_ref as ref16
from gemm_bf16_ref import bits, value

K_GEMM_BF16 = 8


def int_operands(rng, M, N, K, amax):
    assert amax <= 256 and amax * amax * K < 2 ** 24
    return (bits(rng.integers(-amax, amax + 1, (M, K)).astype(np.float32)), bits(rng.integers(-amax, amax + 1, (K, N)).astype(np.float32)))


@pytest.mark.parametrize("M,N,K,amax", [(5, 7, 64, 8), (3, 130, 255, 256), (17, 9, 1024, 100), (2, 2, 1, 256)])
def test_elements_equal_the_float64_matmul_on_integer_valued_operands(oracle, M, N, K, amax):
    A, B = int_operands(np.random.default_rng(K), M, N, K, amax)
    ref = value(A).astype(np.float64) @ value(B).astype(np.float64)
    out, st = ref16.run(oracle, 1, A, B)
    assert np.array_equal(out.view(np.float32).reshape(M, N).astype(np.float64), ref)
    assert st == dict(errors_corrected=0, dwc_detected=0, syncs=0, injected=0, first_fault_unit=oracle.NO_FAULT_UNIT)


def test_every_bf16_pattern_widens_exactly_and_survives_tf32_truncation(oracle):
    """a bfloat16 is the top half of an fp32: zeros keep their sign, denormals, infinities and NaNs keep their bits; none of
    them has a bit below the 19 that TF32 reads"""
    pat = np.arange(65536, dtype=np.uint32).astype(np.uint16)
    w = value(pat).view(np.uint32)
    assert np.array_equal(w, pat.astype(np.uint32) << 16) and not (w & 0x1FFF).any()
    assert np.array_equal(bits(value(pat)), pat)
    v = value(np.array([0x0000, 0x8000, 0x0001, 0x3F80, 0xBF80, 0x7F80, 0xFF80, 0x7FC0], dtype=np.uint16))
    assert str(v[1]) == "-0.0" and v[2] == 2.0 ** -133 and v[3] == 1.0 and v[4] == -1.0 and v[5] == np.inf and v[6] == -np.inf
    assert np.isnan(v[7]) and not np.signbit(v[0])
    # inf and NaN operands reach the element: inf * 1 = inf, inf * 0 = NaN
    A = np.array([[0x7F80, 0x3F80], [0x7F80, 0x0000]], dtype=np.uint16)
    B = np.array([[0x3F80, 0x0000], [0x3F80, 0x3F80]], dtype=np.uint16)
    c = ref16.run(oracle, 1, A, B)[0].view(np.float32)
    assert c[0] == np.inf and np.isnan(c[1]) and c[2] == np.inf and np.isnan(c[3])


def test_per_unit_numbers_equal_gemm_tf32s(oracle, built_lib):
    """the runtime's numbers for the new id against the oracle's for GEMM_TF32 (no driver is needed to ask)"""
    from coast_b200 import runtime as R
    L, t = R.load_library(), oracle.K_GEMM_TF32
    assert R.K_GEMM_BF16 == K_GEMM_BF16 and R.OUT_BYTES[K_GEMM_BF16] == 4
    assert L.coast_fault_sites(K_GEMM_BF16, 0, 64) == oracle.fault_sites(t, 0, 64) == 1
    assert L.coast_fault_site_bits(K_GEMM_BF16, 0, 64, 0) == oracle.fault_site_bits(t, 0, 64, 0) == 32
    assert L.coast_out_bytes_per_unit(K_GEMM_BF16) == oracle.out_bytes_per_unit(t) == 4
    assert L.coast_votes_per_unit(K_GEMM_BF16) == oracle.votes_per_unit(t) == 1
    # in-loop store votes are not built: asking for them is not honoured, asking for none is
    assert L.coast_flags_honoured(K_GEMM_BF16, 3, 0x200 | 0x4) == L.coast_flags_honoured(t, 3, 0x200 | 0x4) == 0
    assert L.coast_flags_honoured(K_GEMM_BF16, 3, 0x400 | 0x1) == 0x400 | 0x1


@pytest.mark.parametrize("nc", [1, 2, 3])
def test_fault_plan_on_site_zero(oracle, nc):
    """TABLE entries on site 0 flip one bit of one replica's final accumulator: voted out under TMR (counted), stored under DWC
    when replica 0 was hit (detected), applied as is unprotected; other sites and replicas >= NC are ignored"""
    M, N, K = 4, 8, 64
    A, B = int_operands(np.random.default_rng(2), M, N, K, 8)
    A[1] = 0                                                  # a +0.0 row: a flipped sign there compares equal
    clean, _ = ref16.run(oracle, 1, A, B)
    tab = np.zeros(M * N, dtype=np.uint32)
    picks = {0: (0, 0, 5), 3: (1, 0, 30), 9: (0, 0, 31), 17: (2, 0, 1), 20: (0, 1, 4), 25: (3, 0, 4)}
    for u, (r, s, b) in picks.items():
        tab[u] = oracle.fault_entry(r, s, b)
    out, st = ref16.run(oracle, nc, A, B, plan=oracle.make_plan(oracle.PLAN_TABLE, table=tab))
    live = {u: (r, b) for u, (r, s, b) in picks.items() if s == 0 and r < nc}
    assert st["injected"] == len(live)
    counted = sorted(u for u in live if u != 9)               # unit 9 lies in the zero row: -0.0 == +0.0
    want = clean.copy()
    for u, (r, b) in live.items():
        if r == 0 and (nc < 3 or u == 9):                     # the select voter stores r0 when it compares equal to r1: r0's -0.0
            want[u] ^= np.uint32(1 << b)
    assert np.array_equal(out, want)
    if nc == 3:
        assert st["errors_corrected"] == len(counted) and st["syncs"] == M * N and st["first_fault_unit"] == counted[0]
    elif nc == 2:
        assert st["dwc_detected"] == len(counted) and st["first_fault_unit"] == counted[0]
    else:
        assert st["first_fault_unit"] == oracle.NO_FAULT_UNIT


RO = [4, 4, 9, 10, 10, 30, 31]


def grouped_ref(oracle, nc, A, B, ro, *, plan=None, base=0):
    """C rows [ro[0], ro[G]) and the summed stats of G single reference runs: product g with its rows of A (rows x K), its own
    B (of the G stacked K x N) and unit_base + (ro[g] - ro[0]) N"""
    K, N = A.shape[1], B.shape[1]
    outs, total = [], dict(errors_corrected=0, dwc_detected=0, syncs=0, injected=0, first_fault_unit=oracle.NO_FAULT_UNIT)
    for g in range(len(ro) - 1):
        if ro[g + 1] == ro[g]:
            continue
        out, st = ref16.run(oracle, nc, A[ro[g]:ro[g + 1]], B[g * K:(g + 1) * K], plan=plan, unit_base=base + (ro[g] - ro[0]) * N)
        outs.append(out)
        for k in ("errors_corrected", "dwc_detected", "syncs", "injected"):
            total[k] += st[k]
        total["first_fault_unit"] = min(total["first_fault_unit"], st["first_fault_unit"])
    return np.concatenate(outs), total


@pytest.mark.parametrize("nc", [1, 3])
def test_grouped_and_batched_references(oracle, nc):
    N, K = 6, 64
    rng = np.random.default_rng(10 + nc)
    G = len(RO) - 1
    A = bits(rng.integers(-8, 9, (RO[-1], K)).astype(np.float32))
    B = bits(rng.integers(-8, 9, (G * K, N)).astype(np.float32))
    plan = oracle.make_plan(oracle.PLAN_BERNOULLI, seed=4, p=0.3)
    out, st = grouped_ref(oracle, nc, A, B, RO, plan=plan, base=(1 << 32) - 40)
    ref = np.concatenate([value(A[RO[g]:RO[g + 1]]).astype(np.float64) @ value(B[g * K:(g + 1) * K]).astype(np.float64)
                          for g in range(G)]).reshape(-1)
    assert st["injected"] > 0 and st["syncs"] == ((RO[-1] - RO[0]) * N if nc == 3 else 0)
    if nc == 3:
        assert np.array_equal(out.view(np.float32).astype(np.float64), ref) and st["errors_corrected"] > 0
    # a product's faults depend on its global units only: the last two products alone give the launch's tail
    lo = 4
    tail, _ = grouped_ref(oracle, nc, A, B[lo * K:], RO[lo:], plan=plan, base=(1 << 32) - 40 + (RO[lo] - RO[0]) * N)
    assert np.array_equal(out[-len(tail):], tail)
    # a batch is a group of equal row counts from row 0
    M, batch = 5, 4
    outb, _ = grouped_ref(oracle, nc, A, B, [b * M for b in range(batch + 1)], plan=plan, base=7)
    for b in range(batch):
        o, _ = ref16.run(oracle, nc, A[b * M:(b + 1) * M], B[b * K:(b + 1) * K], plan=plan, unit_base=7 + b * M * N)
        assert np.array_equal(outb[b * M * N:(b + 1) * M * N], o)
