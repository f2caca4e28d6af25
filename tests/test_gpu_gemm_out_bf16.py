"""GPU (H100): matmuls with BF16 output (COAST_MM_OUT_BF16, the xmr_o16_* kernels).

Every replica rounds its value -- the accumulator after the fault hook -- to bfloat16 with round to nearest even, and the vote
is on the rounded values.  Pinned here:
  * bit-exact against the CPU reference (tests/gemm_out_bf16_ref.py) on integer operands whose fp32 sums are exact and exceed
    bfloat16's 8 significant bits (so ties and roundings happen), for every variant (wide, narrow, pair, single-CTA, B^T), at
    NC 1-3, with and without a plan and with both voters;
  * the output identity of DESIGN.md §3.13 on the device: for the same operands and plan, the bf16 output equals the fp32
    launch's output converted by torch, on uniform(-1, 1) operands, every layout, batched and grouped launches; `injected` is
    equal and the counted units are exactly the faulted units whose flipped value rounds to a different bfloat16;
  * unprotected torch bit for bit on integer operands: torch.matmul in bfloat16, and torch._scaled_mm at scale 1 with bf16
    output;
  * shards over rows, products and groups, and the host call;
  * the NaN pattern the conversion writes.
Output buffers start as POISON16, a NaN pattern the conversion never writes, so a skipped element fails."""
import numpy as np
import pytest

import gemm_fp8_ref as ref8
import gemm_out_bf16_ref as oref
from mm_gpu import STAT_KEYS, Bf16, Fp8, dev, env, transposed
from coast_b200.runtime import F_MAJORITY_VOTER, MM_B_TRANSPOSED as MM_BT, MM_BATCHED, MM_GROUPED, MM_OUT_BF16

pytestmark = pytest.mark.gpu

POISON16 = 0x7FA5                                  # a NaN; every NaN the conversion writes is oref.NAN_BF16
RO = [3, 3, 100, 101, 101, 500, 700, 828]          # from row 3: empty products, a one-row product, a 128-row product


def poisoned(n):
    import torch
    return torch.full((n,), POISON16, dtype=torch.int16, device="cuda").view(torch.bfloat16)


def launch(rt, t, nc, A, B, *, o16=True, flags=3, plan=None, table=None, unit_base=0, mode=0, M=None, n=None, rows=None, out=None,
           bt=False, status=None):
    """A: (rows x K), B: (P K x N) bit patterns of t -> (C as uint16 bf16 patterns, or uint32 fp32 patterns; stats dict)"""
    import torch
    import coast_b200 as cb
    K, N = A.shape[1], B.shape[1]
    M = A.shape[0] if M is None else M
    n = A.shape[0] * N if n is None else n
    if table is not None:
        plan = cb.FaultPlan(mode=cb.PLAN_TABLE, table=torch.from_numpy(table.view(np.int32).copy()).cuda())
    if out is None:
        out = poisoned(A.shape[0] * N) if o16 else torch.full((A.shape[0] * N,), float("nan"), dtype=torch.float32, device="cuda")
    aux = dev(t, transposed(B, K)) if bt else dev(t, B)
    _, st = rt.run(t.kernel, nc, dev(t, A), n, M=M, N=N, K=K, aux=aux, flags=flags, plan=plan, unit_base=unit_base, status=status,
                   mode=mode | (MM_BT if bt else 0) | (MM_OUT_BF16 if o16 else 0), rows=rows, out=out)
    c = out.cpu()
    return (c.view(torch.int16).numpy().view(np.uint16) if o16 else c.numpy().view(np.uint32)), st.as_dict()


def torch_rne(c32):
    """fp32 bit patterns -> bf16 patterns, converted by torch on the device"""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(c32).view(np.float32)).cuda()
    return t.to(torch.bfloat16).view(torch.int16).cpu().numpy().view(np.uint16)


def int_operands(t, M, N, K, seed):
    """integer operands with exact fp32 sums above 256: BF16 in [-16, 16], FP8 in [-2, 2] (K 4 <= 2^11)"""
    if t is Bf16:
        return Bf16.int_operands(M, N, K, seed, amax=16)
    return Fp8.int_operands(M, N, K, seed, amax=2 if 4 * K <= ref8.EXACT_SUM else 1)


def cpu(oracle, t, nc, A, B, *, flags=3, plan_kw=None, unit_base=0):
    plan = oracle.make_plan(oracle.PLAN_BERNOULLI, **plan_kw) if plan_kw else None
    return (oref.run_bf16 if t is Bf16 else oref.run_fp8)(oracle, nc, A, B, flags=flags, plan=plan, unit_base=unit_base)


TYPES = [Bf16, Fp8]
# (id, M, N, K, environment): wide (nc 1, N % 256 == 0), narrow (nc 1), pair, single CTA
VARIANTS = [("wide", 384, 512, 512, {}), ("narrow", 384, 384, 512, {}), ("pair", 512, 256, 512, {"COAST_GEMM_PAIR": "1"}),
            ("single", 384, 256, 512, {"COAST_GEMM_PAIR": "0"})]


@pytest.mark.parametrize("bt", [False, True], ids=["B", "Bt"])
@pytest.mark.parametrize("variant", VARIANTS, ids=[v[0] for v in VARIANTS])
@pytest.mark.parametrize("nc", [1, 2, 3])
@pytest.mark.parametrize("t", TYPES, ids=["bf16", "fp8"])
def test_integer_operands_bit_exact(rt, oracle, monkeypatch, t, nc, variant, bt):
    _, M, N, K, e = variant
    env(monkeypatch, **e)
    A, B = int_operands(t, M, N, K, 10 * nc + len(variant[0]))
    for flags, plan_kw, base in ((3, None, 0), (3, dict(seed=3 + nc, p=0.2), 2 ** 32 - M * N // 2),
                                 (3 | F_MAJORITY_VOTER, dict(seed=9, p=0.2), 77)):
        import coast_b200 as cb
        plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, **plan_kw) if plan_kw else None
        g, gs = launch(rt, t, nc, A, B, flags=flags, plan=plan, unit_base=base, bt=bt)
        o, os_, _ = cpu(oracle, t, nc, A, B, flags=flags, plan_kw=plan_kw, unit_base=base)
        assert np.array_equal(g, o), (np.flatnonzero(g != o)[:8], g[g != o][:4], o[g != o][:4])
        assert {k: gs[k] for k in STAT_KEYS} == {k: os_[k] for k in STAT_KEYS}
        if plan_kw:
            assert gs["injected"] > 0 and (nc == 1 or gs["errors_corrected"] + gs["dwc_detected"] > 0)


def test_nan_pattern_of_the_conversion(rt, oracle, monkeypatch):
    """NaN accumulators of either sign (E4M3 NaN operands 0x7F and 0xFF; BF16 NaN operands 0x7FC1 and 0xFFFF, payloads
    included): the device writes one pattern, the reference's"""
    env(monkeypatch)
    M, N, K = 128, 128, 128
    seen, runs = set(), []
    for t, nans in ((Fp8, (0x7F, 0xFF)), (Bf16, (0x7FC1, 0xFFFF))):
        A, B = int_operands(t, M, N, K, 1)
        A[3, 0], A[4, 5] = nans
        B[9, 6] = nans[1]
        g, _ = launch(rt, t, 3, A, B)
        nan = (g & 0x7FFF) > 0x7F80
        assert nan.sum() > 0
        seen |= {int(x) for x in np.unique(g[nan])}
        runs.append((g, cpu(oracle, t, 3, A, B)[0]))
    assert seen == {oref.NAN_BF16}, sorted(hex(x) for x in seen)
    for g, o in runs:
        assert np.array_equal(g, o)


# ------------------------------------------------------------------------------------------ the identity on the device
def faulted_units(oracle, nc, K, n, unit_base, plan_kw):
    plan = oracle.make_plan(oracle.PLAN_BERNOULLI, **plan_kw)
    import gemm_fp8_scaled_ref as sref
    return sref.faults(oracle, plan, nc, K, n, unit_base)


def counted(clean32, faults):
    """faulted units whose flipped value rounds to a bfloat16 that `fcmp oeq` tells from the clean one's"""
    c = 0
    for u, _, bit in faults:
        a = oref.widen(oref.rne(np.array([clean32[u]], np.uint32))).view(np.float32)[0]
        b = oref.widen(oref.rne(np.array([clean32[u] ^ (1 << bit)], np.uint32))).view(np.float32)[0]
        c += not (a == b)
    return c


LAYOUTS = [("single", None), ("batched", 3), ("grouped", RO)]


@pytest.mark.parametrize("voter", [0, F_MAJORITY_VOTER], ids=["select", "majority"])
@pytest.mark.parametrize("bt", [False, True], ids=["B", "Bt"])
@pytest.mark.parametrize("layout", LAYOUTS, ids=[c[0] for c in LAYOUTS])
@pytest.mark.parametrize("t", TYPES, ids=["bf16", "fp8"])
def test_bf16_output_is_the_fp32_output_rounded(rt, oracle, monkeypatch, t, layout, bt, voter):
    import torch
    env(monkeypatch)
    name, extra = layout
    N, K = 256, 512
    if name == "single":
        A, B = t.uniform_operands(512, N, K, 1)
        kw = dict()
    elif name == "batched":
        A, B = t.uniform_operands(extra * 256, N, K * extra, 2)
        A = np.ascontiguousarray(A[:, :K])
        kw = dict(M=256, mode=MM_BATCHED)
    else:
        G = len(extra) - 1
        A, B = t.uniform_operands(extra[-1], N, K * G, 3)
        A = np.ascontiguousarray(A[:, :K])
        kw = dict(M=G, mode=MM_GROUPED, n=(extra[-1] - extra[0]) * N,
                  rows=torch.tensor(extra, dtype=torch.int64, device="cuda"))
    rows = A.shape[0]
    first = extra[0] if name == "grouped" else 0
    n = (rows - first) * N
    import coast_b200 as cb
    for nc in (1, 2, 3):
        flags = 3 | voter
        for plan_kw, base in ((None, 0), (dict(seed=4 + nc, p=0.3), 2 ** 32 - 1000)):
            plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, **plan_kw) if plan_kw else None
            g32, s32 = launch(rt, t, nc, A, B, o16=False, flags=flags, plan=plan, unit_base=base, bt=bt, **kw)
            g16, s16 = launch(rt, t, nc, A, B, flags=flags, plan=plan, unit_base=base, bt=bt, **kw)
            assert np.array_equal(g16[first * N:], torch_rne(g32[first * N:]))
            if name == "grouped":
                assert (g16[:first * N] == POISON16).all()
            assert s16["injected"] == s32["injected"] and s16["syncs"] == s32["syncs"]
            key = "errors_corrected" if nc == 3 else "dwc_detected"
            if plan_kw and nc > 1:
                clean, _ = launch(rt, t, 3, A, B, o16=False, flags=flags, bt=bt, **kw)
                fl = faulted_units(oracle, nc, K, n, base, plan_kw)
                assert len(fl) == s16["injected"] > 0
                assert s16[key] == counted(clean[first * N:], fl) and s16[key] <= s32[key]
            elif nc > 1:
                assert s16[key] == s32[key] == 0


# ------------------------------------------------------------------------------------------ unprotected torch
def test_gemm_bf16_equals_torch_matmul_on_integer_operands(rt, monkeypatch):
    import torch
    env(monkeypatch)
    saved = torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction
    torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = False
    try:
        for M, N, K in ((512, 512, 1024), (384, 384, 512)):
            A, B = int_operands(Bf16, M, N, K, M)
            want = torch.matmul(dev(Bf16, A), dev(Bf16, B)).view(torch.int16).cpu().numpy().view(np.uint16).ravel()
            for nc in (1, 3):
                for bt in (False, True):
                    g, _ = launch(rt, Bf16, nc, A, B, bt=bt)
                    assert np.array_equal(g, want), (nc, bt)
    finally:
        torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = saved


def test_gemm_fp8_equals_torch_scaled_mm_at_scale_one(rt, monkeypatch):
    """torch._scaled_mm(a, b, 1, 1, out_dtype=torch.bfloat16), A row-major and B column-major, on integer operands"""
    import torch
    env(monkeypatch)
    one = torch.ones((), device="cuda")
    for M, N, K in ((512, 512, 512), (384, 256, 1024)):
        A, B = int_operands(Fp8, M, N, K, M)
        want = torch._scaled_mm(dev(Fp8, A), dev(Fp8, np.ascontiguousarray(B.T)).t(), scale_a=one, scale_b=one,
                                out_dtype=torch.bfloat16).view(torch.int16).cpu().numpy().view(np.uint16).ravel()
        for nc in (1, 3):
            for bt in (False, True):
                g, _ = launch(rt, Fp8, nc, A, B, bt=bt)
                assert np.array_equal(g, want), (nc, bt)


# ------------------------------------------------------------------------------------------ shards and the host call
@pytest.mark.parametrize("t", TYPES, ids=["bf16", "fp8"])
def test_shards_over_rows_products_and_groups(rt, monkeypatch, t):
    import torch
    import coast_b200 as cb
    env(monkeypatch)
    N, K = 256, 256
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=3, p=0.2)
    # rows: two launches of 256 and 256 rows of one 512-row product
    A, B = int_operands(t, 512, N, K, 1)
    full, fs = launch(rt, t, 3, A, B, plan=plan, unit_base=10)
    out = poisoned(512 * N)
    tot = dict.fromkeys(STAT_KEYS[:4], 0)
    for lo in (0, 256):
        _, st = rt.run(t.kernel, 3, dev(t, A[lo:lo + 256]), 256 * N, M=256, N=N, K=K, aux=dev(t, B), flags=3, plan=plan,
                       unit_base=10 + lo * N, mode=MM_OUT_BF16, out=out[lo * N:])
        for k in tot:
            tot[k] += st.as_dict()[k]
    assert np.array_equal(out.cpu().view(torch.int16).numpy().view(np.uint16), full)
    assert tot == {k: fs[k] for k in tot}
    # products: a batch of 4 as 1 + 3
    A, B = int_operands(t, 4 * 128, N, 4 * K, 2)
    A = np.ascontiguousarray(A[:, :K])
    full, _ = launch(rt, t, 2, A, B, plan=plan, M=128, mode=MM_BATCHED)
    out = poisoned(4 * 128 * N)
    for lo, hi in ((0, 1), (1, 4)):
        rt.run(t.kernel, 2, dev(t, A[lo * 128:hi * 128]), (hi - lo) * 128 * N, M=128, N=N, K=K, aux=dev(t, B[lo * K:hi * K]),
               flags=3, plan=plan, unit_base=lo * 128 * N, mode=MM_BATCHED | MM_OUT_BF16, out=out[lo * 128 * N:])
    assert np.array_equal(out.cpu().view(torch.int16).numpy().view(np.uint16), full)
    # groups: products [0, 3) and [3, 7) of RO, the same d_in and d_out
    G = len(RO) - 1
    A, B = int_operands(t, RO[-1], N, G * K, 3)
    A = np.ascontiguousarray(A[:, :K])
    ro = torch.tensor(RO, dtype=torch.int64, device="cuda")
    full, _ = launch(rt, t, 3, A, B, plan=plan, M=G, mode=MM_GROUPED, n=(RO[-1] - RO[0]) * N, rows=ro)
    out = poisoned(RO[-1] * N)
    d_a = dev(t, A)
    for lo, hi in ((0, 3), (3, G)):
        rt.run(t.kernel, 3, d_a, (RO[hi] - RO[lo]) * N, M=hi - lo, N=N, K=K, aux=dev(t, B[lo * K:hi * K]), flags=3, plan=plan,
               unit_base=(RO[lo] - RO[0]) * N, mode=MM_GROUPED | MM_OUT_BF16, rows=ro[lo:], out=out)
    assert np.array_equal(out.cpu().view(torch.int16).numpy().view(np.uint16)[RO[0] * N:], full[RO[0] * N:])


@pytest.mark.parametrize("case", ["row_blocks", "products", "groups"])
def test_host_call(rt, monkeypatch, case):
    import torch
    import coast_b200 as cb
    env(monkeypatch, COAST_HOST_CHUNK_BYTES="400000")
    t = Fp8 if case == "groups" else Bf16
    N, K = 256, 256
    kw = {}
    if case == "row_blocks":
        A, B = int_operands(t, 1024, N, K, 4)
        M, n = 1024, 1024 * N
    elif case == "products":
        A, B = int_operands(t, 5 * 128, N, 5 * K, 5)
        A = np.ascontiguousarray(A[:, :K])
        M, n, kw = 128, 5 * 128 * N, dict(mode=MM_BATCHED)
    else:
        G = len(RO) - 1
        A, B = int_operands(t, RO[-1], N, G * K, 6)
        A = np.ascontiguousarray(A[:, :K])
        M, n = G, (RO[-1] - RO[0]) * N
    rows_d = torch.tensor(RO, dtype=torch.int64, device="cuda") if case == "groups" else None
    mode = kw.get("mode", 0) | (MM_GROUPED if case == "groups" else 0)
    dev_out, ds = launch(rt, t, 3, A, B, M=M, n=n, mode=mode, rows=rows_d)
    h_out = np.full(A.shape[0] * N, POISON16, dtype=np.uint16)
    st = rt.run_host(t.kernel, 3, t.tensor(A), h_out, n, M=M, N=N, K=K, h_aux=t.tensor(B), flags=3, mode=mode | MM_OUT_BF16,
                     h_rows=np.array(RO, dtype=np.uint64) if case == "groups" else None)
    first = RO[0] if case == "groups" else 0
    assert np.array_equal(h_out[first * N:], dev_out[first * N:]) and (h_out[:first * N] == POISON16).all()
    assert st.syncs == ds["syncs"] == n
    assert rt.last_host_path == {"row_blocks": "row-blocks", "products": "staged", "groups": "groups"}[case]
