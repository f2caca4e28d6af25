"""GPU (H100): scaled GEMM_FP8 (COAST_MM_SCALE_TENSOR / COAST_MM_SCALE_ROWWISE, the xmr_scaled_fp8* kernels).

Every replica multiplies its accumulator by the row's A scale and then the column's B scale, two fp32 multiplies rounded to
nearest, after the fault hook and before the vote.  Bit-exact where arithmetic allows it: integer-valued E4M3 operands in
GEMM_FP8's exact domain (tests/gemm_fp8_ref.py) make the accumulators exact, so every output bit, all five counters and
d_status must equal the CPU reference (tests/gemm_fp8_scaled_ref.py) whatever the scales -- random signs and magnitudes, powers
of two, scales whose products are subnormal, a zero row and a NaN column.  A NaN's payload is not pinned: the device's multiply
returns the canonical NaN.  General operands are held to bit-equality between scale layouts, variants and replica counts, to
the unscaled launch at scale 1, to float64 within GEMM_FP8's bound times the scales, and to unprotected torch._scaled_mm."""
import numpy as np
import pytest

import gemm_fp8_scaled_ref as sref
from mm_gpu import POISON, STAT_KEYS, Fp8, add_stats, dev, env, no_stats, transposed
from coast_b200.runtime import MM_B_TRANSPOSED as MM_BT, MM_BATCHED, MM_GROUPED, MM_SCALE_ROWWISE, MM_SCALE_TENSOR

pytestmark = pytest.mark.gpu

RO = [3, 3, 100, 101, 101, 500, 700, 828]          # from row 3: empty products, a one-row product, a 128-row product


def zipf_offsets(G, R, start, seed):
    """a mixture-of-experts routing: Zipf-like expert loads, some experts empty, rows from `start`"""
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, G + 1) ** 1.1
    rng.shuffle(w)
    rows = np.floor(R * w / w.sum()).astype(int)
    rows[rng.choice(G, size=G // 5, replace=False)] = 0
    rows[np.argmax(rows)] += R - rows.sum()
    return [int(start)] + [int(start + x) for x in np.cumsum(rows)]


def row_col_scales(M, N, seed, *, nan_col=None, zero_row=None):
    """fp32 scales with random signs and magnitudes 2^-12 .. 2^12, every fourth a power of two, a few pairs whose product with an
    accumulator is subnormal (2^-70 x 2^-70), an optional zero row and NaN column"""
    rng = np.random.default_rng(seed)

    def one(n):
        s = rng.choice([-1.0, 1.0], n) * 2.0 ** rng.uniform(-12, 12, n)
        s[::4] = np.rint(np.log2(np.abs(s[::4])))
        s[::4] = np.where(rng.random(len(s[::4])) < 0.5, -1, 1) * 2.0 ** s[::4]
        return s.astype(np.float32)
    sa, sb = one(M), one(N)
    sa[1::17], sb[2::19] = np.float32(2.0 ** -70), np.float32(2.0 ** -70)
    if zero_row is not None:
        sa[zero_row] = 0.0
    if nan_col is not None:
        sb[nan_col] = np.nan
    return sa, sb


def same(g, o):
    """bit-equal except that two NaNs are equal whatever their payloads"""
    gf, of = g.view(np.float32), o.view(np.float32)
    return (g == o) | (np.isnan(gf) & np.isnan(of))


def scaled(rt, nc, A, B, sa, sb, *, rowwise=True, flags=3, plan=None, table=None, unit_base=0, status=None, mode=0, M=None, n=None,
           rows=None, out=None, bt=False):
    """A: (rows x K), B: (P K x N) E4M3 bit patterns, sa / sb float32 (rowwise) or one float each -> (C bits, stats dict)"""
    import torch
    import coast_b200 as cb
    K, N = A.shape[1], B.shape[1]
    M = A.shape[0] if M is None else M
    n = A.shape[0] * N if n is None else n
    if table is not None:
        plan = cb.FaultPlan(mode=cb.PLAN_TABLE, table=torch.from_numpy(table.view(np.int32).copy()).cuda())
    if out is None:
        out = torch.full((A.shape[0] * N,), POISON, dtype=torch.int32, device="cuda").view(torch.float32)
    aux = dev(Fp8, transposed(B, K)) if bt else dev(Fp8, B)
    d_sa = torch.from_numpy(np.atleast_1d(np.asarray(sa, dtype=np.float32)).copy()).cuda()
    d_sb = torch.from_numpy(np.atleast_1d(np.asarray(sb, dtype=np.float32)).copy()).cuda()
    _, st = rt.run(cb.K_GEMM_FP8, nc, dev(Fp8, A), n, M=M, N=N, K=K, aux=aux, flags=flags, plan=plan, unit_base=unit_base, status=status,
                   mode=mode | (MM_BT if bt else 0) | (MM_SCALE_ROWWISE if rowwise else MM_SCALE_TENSOR), rows=rows, out=out,
                   scale_a=d_sa, scale_b=d_sb)
    return out.cpu().numpy().view(np.uint32), st.as_dict()


def ref(oracle, nc, A, B, sa, sb, *, flags=3, plan_kw=None, table=None, unit_base=0):
    plan = None
    if table is not None:
        plan = oracle.make_plan(oracle.PLAN_TABLE, table=table)
    elif plan_kw:
        plan = oracle.make_plan(oracle.PLAN_BERNOULLI, **plan_kw)
    return sref.run(oracle, nc, A, B, sa, sb, flags=flags, plan=plan, unit_base=unit_base)


# (id, environment, NC, M, N, the kernel the launcher must pick)
VARIANTS = [
    ("narrow_nc1", {}, 1, 256, 384, "xmr_scaled_fp8n_inj0_nc1"),
    ("wide_nc1", {"COAST_GEMM_PAIR": "0"}, 1, 256, 256, "xmr_scaled_fp8_inj0_nc1"),
    ("pair_nc1", {}, 1, 256, 256, "xmr_scaled_fp8p_inj0_nc1"),
    ("pair_nc2", {}, 2, 256, 128, "xmr_scaled_fp8p_inj0_nc2"),
    ("single_nc2", {"COAST_GEMM_PAIR": "0"}, 2, 256, 128, "xmr_scaled_fp8_inj0_nc2"),
    ("single_nc3", {}, 3, 256, 128, "xmr_scaled_fp8_inj0_nc3"),
    ("pair_nc3", {"COAST_GEMM_PAIR": "1"}, 3, 256, 256, "xmr_scaled_fp8p_inj0_nc3"),
]


@pytest.mark.parametrize("K", [128, 896])
@pytest.mark.parametrize("variant", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_integer_operands_any_scales_bit_exact_with_the_reference(rt, oracle, variant, K, monkeypatch, capfd):
    """every output bit, the five counters and d_status, with B and B^T, without a plan, Bernoulli across 2^32, TABLE, majority"""
    import torch
    import coast_b200 as cb
    _, e, nc, M, N, kname = variant
    env(monkeypatch, **e)
    A, B = Fp8.int_operands(M, N, K, seed=K + nc, amax=1)
    sa, sb = row_col_scales(M, N, seed=K + nc, zero_row=5, nan_col=77)
    n = M * N
    capfd.readouterr()
    scaled(rt, nc, A, B, sa, sb, flags=cb.F_VERBOSE)
    assert f"{kname} " in capfd.readouterr().err
    base = 2 ** 32 - n // 2
    rng = np.random.default_rng(K + nc)
    tab = np.zeros(n, dtype=np.uint32)
    for u in rng.choice(n, size=300, replace=False):
        tab[u] = oracle.fault_entry(int(rng.integers(0, 4)), 0 if rng.random() < 0.8 else 1, int(rng.integers(0, 32)))
    cases = [dict(), dict(plan_kw=dict(seed=K, p=0.3), unit_base=base), dict(table=tab, unit_base=base),
             dict(flags=3 | cb.F_MAJORITY_VOTER, plan_kw=dict(seed=K + 1, p=0.3))]
    for bt in (False, True):
        for c in cases:
            plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, **c["plan_kw"]) if "plan_kw" in c else None
            status = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
            g, gs = scaled(rt, nc, A, B, sa, sb, flags=c.get("flags", 3), plan=plan, table=c.get("table"),
                           unit_base=c.get("unit_base", 0), status=status, bt=bt)
            o, os_, ostat = ref(oracle, nc, A, B, sa, sb, **c)
            assert same(g, o).all(), (bt, c.keys(), np.flatnonzero(~same(g, o))[:8])
            assert {k: gs[k] for k in STAT_KEYS} == {k: os_[k] for k in STAT_KEYS}, (bt, c.keys())
            assert np.array_equal(status.cpu().numpy(), ostat), (bt, c.keys())
            if c:
                assert gs["injected"] > 0
    # the NaN column disagrees in every row under DWC and TMR, and the zero row hides every flip there
    if nc > 1:
        assert (gs["errors_corrected"] if nc == 3 else gs["dwc_detected"]) >= M


@pytest.mark.parametrize("bt", [False, True])
@pytest.mark.parametrize("nc", [1, 2, 3])
def test_batched_and_grouped_equal_the_reference_per_product(rt, oracle, nc, bt):
    """a batch (B per product, sa per stacked row, sb per product column) and groups with empty experts: per product, the
    reference with the product's unit_base; d_out rows outside the groups keep their poison"""
    import torch
    import coast_b200 as cb
    N, K = 256, 256
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=3, p=0.2)
    base = 2 ** 32 - 5000
    # batched
    M, batch = 128, 5
    A, B = Fp8.stacked_operands(batch * M, N, K, batch, seed=nc)
    sa, sb = row_col_scales(batch * M, batch * N, seed=nc, zero_row=130, nan_col=300)
    g, st = scaled(rt, nc, A, B, sa, sb, M=M, mode=MM_BATCHED, plan=plan, unit_base=base, bt=bt)
    tot = no_stats()
    for b in range(batch):
        o, s, _ = ref(oracle, nc, A[b * M:(b + 1) * M], B[b * K:(b + 1) * K], sa[b * M:(b + 1) * M], sb[b * N:(b + 1) * N],
                      plan_kw=dict(seed=3, p=0.2), unit_base=base + b * M * N)
        assert same(g[b * M * N:(b + 1) * M * N], o).all(), b
        add_stats(tot, s)
    assert st == tot and st["injected"] > 0
    # grouped
    G, R, rows_alloc = len(RO) - 1, RO[-1] - RO[0], RO[-1] + 40
    A, B = Fp8.stacked_operands(rows_alloc, N, K, G, seed=nc + 10)
    sa, sb = row_col_scales(rows_alloc, G * N, seed=nc + 10, zero_row=200, nan_col=G * N - 3)
    sa[:RO[0]], sa[RO[-1]:] = np.nan, np.nan                        # rows outside the table: never read
    out = torch.full((rows_alloc * N,), POISON, dtype=torch.int32, device="cuda").view(torch.float32)
    d_ro = torch.tensor(RO, dtype=torch.int64, device="cuda")
    g, st = scaled(rt, nc, A, B, sa, sb, M=G, n=R * N, mode=MM_GROUPED, rows=d_ro, plan=plan, unit_base=base, out=out, bt=bt)
    g = g.reshape(rows_alloc, N)
    assert (g[:RO[0]] == POISON).all() and (g[RO[-1]:] == POISON).all()
    tot = no_stats()
    for i in range(G):
        if RO[i + 1] == RO[i]:
            continue
        o, s, _ = ref(oracle, nc, A[RO[i]:RO[i + 1]], B[i * K:(i + 1) * K], sa[RO[i]:RO[i + 1]], sb[i * N:(i + 1) * N],
                      plan_kw=dict(seed=3, p=0.2), unit_base=base + (RO[i] - RO[0]) * N)
        assert same(g[RO[i]:RO[i + 1]].ravel(), o).all(), i
        add_stats(tot, s)
    assert st == tot and st["injected"] > 0


def test_three_or_more_tiles_per_persistent_cta_equal_the_reference(rt, oracle, monkeypatch):
    """4096 x 2048 on 128-row tiles: 512 or 256 tiles on 132 CTAs, every variant; row-wise and tensorwise"""
    M, N, K = 4096, 2048, 128
    A, B = Fp8.int_operands(M, N, K, seed=41, amax=2)
    sa, sb = row_col_scales(M, N, seed=41, zero_row=4000, nan_col=1000)
    acc = sref.exact_acc(A, B)
    for e, nc in [({"COAST_GEMM_PAIR": "0"}, 3), ({"COAST_GEMM_PAIR": "1"}, 3), ({}, 2), ({"COAST_GEMM_PAIR": "0"}, 1), ({}, 1)]:
        env(monkeypatch, **e)
        for rowwise in (True, False):
            a, b = (sa, sb) if rowwise else (sa[7], sb[9])
            g, st = scaled(rt, nc, A, B, a, b, rowwise=rowwise, bt=nc == 2)
            o, os_, _ = sref.run(oracle, nc, A, B, a, b, acc=acc)
            assert same(g, o).all() and {k: st[k] for k in STAT_KEYS} == {k: os_[k] for k in STAT_KEYS}, (e, nc, rowwise)


RUNS = [({"COAST_GEMM_PAIR": p}, nc) for nc in (1, 2, 3) for p in ("0", "1")] + [
    ({"COAST_GEMM_TAIL_SPLIT": "0"}, 1), ({"COAST_GEMM_GROUP_M": "3"}, 3), ({"COAST_GEMM_L2_HINTS": "0"}, 3)]


@pytest.mark.parametrize("M,N,K", [(512, 768, 384), (384, 256, 2048)])
def test_general_operands_scale_one_layouts_and_variants(rt, M, N, K, monkeypatch):
    """uniform(-1, 1) operands: scale 1.0 tensorwise and row-wise equals the unscaled GEMM_FP8 launch (outputs, counters and
    d_status, with the same fault plan); tensorwise equals row-wise with constant vectors bit for bit; every variant, NC and B
    layout gives the same bits"""
    import torch
    import coast_b200 as cb
    from mm_gpu import gpu
    A, B = Fp8.uniform_operands(M, N, K, seed=K)
    ones_a, ones_b = np.ones(M, np.float32), np.ones(N, np.float32)
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=K, p=0.2)
    for nc in (1, 2, 3):
        s0 = torch.full((M * N,), 0xEE, dtype=torch.uint8, device="cuda")
        g0, st0 = gpu(rt, Fp8, nc, A, B, plan=plan, status=s0, unit_base=2 ** 32 - 99)
        for rowwise, a, b in ((True, ones_a, ones_b), (False, 1.0, 1.0)):
            s1 = torch.full((M * N,), 0xEE, dtype=torch.uint8, device="cuda")
            g1, st1 = scaled(rt, nc, A, B, a, b, rowwise=rowwise, plan=plan, status=s1, unit_base=2 ** 32 - 99)
            assert same(g1, g0).all() and st1 == st0 and torch.equal(s1, s0), (nc, rowwise)
        c = np.float32(-0.3715)
        d = np.float32(2.0 ** -5 * 1.37)
        gt, stt = scaled(rt, nc, A, B, c, d, rowwise=False, plan=plan)
        gr, str_ = scaled(rt, nc, A, B, np.full(M, c), np.full(N, d), plan=plan)
        assert (gt == gr).all() and stt == str_, nc
    sa, sb = row_col_scales(M, N, seed=K)
    first = None
    for e, nc in RUNS:
        env(monkeypatch, **e)
        for bt in (False, True):
            g, st = scaled(rt, nc, A, B, sa, sb, bt=bt)
            assert st["errors_corrected"] == 0 and st["dwc_detected"] == 0, (e, nc, bt)
            first = g if first is None else first
            assert (g == first).all(), (e, nc, bt)


def bound(A, B, sa, sb):
    """GEMM_FP8's bound on the accumulator, times the scales, plus two fp32 roundings of the scaled float64 value"""
    c64 = Fp8.value(A).astype(np.float64) @ Fp8.value(B).astype(np.float64)
    s = np.abs(sa.astype(np.float64))[:, None] * np.abs(sb.astype(np.float64))[None, :]
    want = c64 * sa.astype(np.float64)[:, None] * sb.astype(np.float64)[None, :]
    return want, Fp8.bound(A, B) * s + 2.0 ** -23 * np.abs(want) + 2.0 ** -148


def test_uniform_operands_stay_within_the_bound(rt):
    M, N, K = 512, 512, 4096
    A, B = Fp8.uniform_operands(M, N, K, seed=5)
    sa, sb = row_col_scales(M, N, seed=5)
    want, tol = bound(A, B, sa, sb)
    for nc in (1, 3):
        g, _ = scaled(rt, nc, A, B, sa, sb)
        err = np.abs(g.view(np.float32).reshape(M, N).astype(np.float64) - want)
        assert (err <= tol).all(), (nc, (err - tol).max())


def test_against_unprotected_torch_scaled_mm(rt):
    """integer operands: bit-equal at power-of-two tensorwise scales; within 2 ulp at general tensorwise scales (cuBLAS multiplies
    by sa * sb once, the kernels by sa and then sb).  Row-wise: against torch._scaled_mm where the installed torch takes (M, 1)
    and (1, N) fp32 scales with fp32 output, else against float64 only, with a warning that says so.  torch 2.11 refuses it
    ("Only bf16 and fp16 high precision output types are supported for row-wise scaling")."""
    import torch
    import coast_b200 as cb
    M, N, K = 1024, 768, 2048
    A, B = Fp8.int_operands(M, N, K, seed=31)
    dA, dBt = dev(Fp8, A), dev(Fp8, transposed(B, K))

    def mine(nc, sa, sb, rowwise):
        g, _ = scaled(rt, nc, A, B, sa, sb, rowwise=rowwise, bt=True)
        return torch.from_numpy(g.view(np.float32).reshape(M, N).copy())

    def ulps(m, t):
        """distance in units in the last place, +0 and -0 equal (cuBLAS's epilogue may turn a -0 product into +0)"""
        d = torch.abs(m.view(torch.int32).long() - t.view(torch.int32).long())
        return torch.where(m == t, torch.zeros_like(d), d)

    def theirs(sa, sb):
        return torch._scaled_mm(dA, dBt.t(), scale_a=sa.cuda(), scale_b=sb.cuda(), out_dtype=torch.float32).cpu()
    for nc in (1, 3):
        for a, b in ((2.0 ** -3, 2.0 ** 5), (0.5, 0.25), (2.0 ** -20, 2.0 ** -9)):
            assert torch.equal(mine(nc, a, b, False), theirs(torch.tensor(a), torch.tensor(b))), (nc, a, b)
        for a, b in ((0.3, 1.7), (-3.1e-3, 0.0123)):
            m, t = mine(nc, a, b, False), theirs(torch.tensor(a), torch.tensor(b))
            assert int(ulps(m, t).max()) <= 2, (nc, a, b, int(ulps(m, t).max()))
    sa, sb = row_col_scales(M, N, seed=8)
    m = mine(3, sa, sb, True)
    try:
        t = theirs(torch.from_numpy(sa).view(M, 1), torch.from_numpy(sb).view(1, N))
    except (RuntimeError, ValueError) as e:                        # torch 2.11 takes row-wise scales with bf16 / fp16 output only
        import warnings
        warnings.warn(f"torch._scaled_mm refused row-wise scales with fp32 output; row-wise checked against float64 only: {e}")
        want = (Fp8.value(A).astype(np.float64) @ Fp8.value(B).astype(np.float64)) * sa[:, None].astype(np.float64) * sb[None, :]
        err = np.abs(m.numpy().astype(np.float64) - want)
        assert (err <= 2.0 ** -23 * np.abs(want) + 2.0 ** -148).all(), f"float64 only ({e}): {err.max()}"
        return
    assert int(ulps(m, t).max()) <= 2


# ------------------------------------------------------------------------------------------ shards and the host call
def test_shards_over_rows_products_and_groups(rt):
    """row and product shards pass d_scale_a + their first row and d_scale_b + p_lo N; group shards the same d_scale_a and
    d_scale_b + g_lo N"""
    import torch
    import coast_b200 as cb
    from coast_b200.shard import shard_groups
    N, K = 256, 256
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=2, p=0.1)

    def t32(x):
        return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()
    # rows of one product: 128-row shards
    M = 768
    A, B = Fp8.int_operands(M, N, K, seed=1, amax=1)
    sa, sb = row_col_scales(M, N, seed=1)
    whole, sw = scaled(rt, 3, A, B, sa, sb, plan=plan, unit_base=50)
    dA, dB, dsa, dsb = dev(Fp8, A), dev(Fp8, B), t32(sa), t32(sb)
    out, tot = torch.zeros(M * N, dtype=torch.float32, device="cuda"), no_stats()
    for lo, hi in ((0, 256), (256, 384), (384, 768)):
        _, s = rt.run(cb.K_GEMM_FP8, 3, dA.view(-1)[lo * K:], (hi - lo) * N, M=hi - lo, N=N, K=K, aux=dB, flags=3, plan=plan,
                      unit_base=50 + lo * N, out=out[lo * N:hi * N], mode=MM_SCALE_ROWWISE, scale_a=dsa[lo:hi], scale_b=dsb)
        add_stats(tot, s.as_dict())
    assert (out.cpu().numpy().view(np.uint32) == whole).all() and tot == sw
    # products of a batch
    M, batch = 128, 6
    A, B = Fp8.stacked_operands(batch * M, N, K, batch, seed=2)
    sa, sb = row_col_scales(batch * M, batch * N, seed=2)
    whole, sw = scaled(rt, 2, A, B, sa, sb, M=M, mode=MM_BATCHED, plan=plan, unit_base=50)
    dA, dB, dsa, dsb = dev(Fp8, A), dev(Fp8, B), t32(sa), t32(sb)
    out, tot = torch.zeros(batch * M * N, dtype=torch.float32, device="cuda"), no_stats()
    for lo, hi in ((0, 1), (1, 4), (4, 6)):
        _, s = rt.run(cb.K_GEMM_FP8, 2, dA.view(-1)[lo * M * K:], (hi - lo) * M * N, M=M, N=N, K=K, aux=dB.view(-1)[lo * K * N:], flags=3, plan=plan,
                      unit_base=50 + lo * M * N, out=out[lo * M * N:hi * M * N], mode=MM_BATCHED | MM_SCALE_ROWWISE,
                      scale_a=dsa[lo * M:hi * M], scale_b=dsb[lo * N:hi * N])
        add_stats(tot, s.as_dict())
    assert (out.cpu().numpy().view(np.uint32) == whole).all() and tot == sw
    # groups
    ro = zipf_offsets(12, 900, start=3, seed=5)
    G, R = len(ro) - 1, ro[-1] - ro[0]
    A, B = Fp8.stacked_operands(ro[-1], N, K, G, seed=13)
    sa, sb = row_col_scales(ro[-1], G * N, seed=13)
    d_ro = torch.tensor(ro, dtype=torch.int64, device="cuda")
    whole, sw = scaled(rt, 3, A, B, sa, sb, M=G, n=R * N, mode=MM_GROUPED, rows=d_ro, plan=plan, unit_base=50,
                       out=torch.zeros(ro[-1] * N, dtype=torch.float32, device="cuda"))
    for bt in (False, True):
        out, tot = torch.zeros(ro[-1] * N, dtype=torch.float32, device="cuda"), no_stats()
        dA, dB, dsa, dsb = dev(Fp8, A), dev(Fp8, transposed(B, K) if bt else B), t32(sa), t32(sb)
        for r in range(3):
            lo, hi = shard_groups(ro, r, 3)
            if hi == lo or ro[hi] == ro[lo]:
                continue
            _, s = rt.run(cb.K_GEMM_FP8, 3, dA, (ro[hi] - ro[lo]) * N, M=hi - lo, N=N, K=K, aux=dB.view(-1)[lo * K * N:], flags=3,
                          mode=MM_GROUPED | MM_SCALE_ROWWISE | (MM_BT if bt else 0), rows=d_ro[lo:], plan=plan,
                          unit_base=50 + (ro[lo] - ro[0]) * N, out=out, scale_a=dsa, scale_b=dsb[lo * N:hi * N])
            add_stats(tot, s.as_dict())
        assert (out.cpu().numpy().view(np.uint32) == whole).all() and tot == sw, bt


@pytest.mark.parametrize("pinned", [False, True])
def test_host_call_row_blocks_products_and_groups(rt, pinned, monkeypatch):
    """coast_run_host with tensorwise and row-wise scales, cut into many chunks, against the device launch"""
    import torch
    import coast_b200 as cb
    env(monkeypatch, COAST_HOST_CHUNK_BYTES=str(300000))

    def host(x, dtype=None):
        x = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)) if dtype else Fp8.tensor(x)
        return x.pin_memory() if pinned else x
    N, K = 128, 256
    for rowwise in (False, True):
        bit = MM_SCALE_ROWWISE if rowwise else MM_SCALE_TENSOR
        # row blocks
        M = 1024
        A, B = Fp8.int_operands(M, N, K, seed=3)
        sa, sb = row_col_scales(M, N, seed=3)
        sa, sb = (sa, sb) if rowwise else (sa[:1], sb[:1])
        want, sw = scaled(rt, 3, A, B, sa, sb, rowwise=rowwise)
        for bt in (False, True):
            h_out = host(np.full(M * N, np.nan), float)
            st = rt.run_host(cb.K_GEMM_FP8, 3, host(A), h_out, M * N, M=M, N=N, K=K, h_aux=host(transposed(B, K) if bt else B), flags=3,
                             mode=bit | (MM_BT if bt else 0), scale_a=host(sa, float), scale_b=host(sb, float))
            assert rt.last_host_path == "row-blocks" and (h_out.numpy().view(np.uint32) == want).all() and st.as_dict() == sw
        # whole products
        M, batch = 128, 9
        A, B = Fp8.stacked_operands(batch * M, N, K, batch, seed=4)
        sa, sb = row_col_scales(batch * M, batch * N, seed=4)
        sa, sb = (sa, sb) if rowwise else (sa[:1], sb[:1])
        want, sw = scaled(rt, 2, A, B, sa, sb, rowwise=rowwise, M=M, mode=MM_BATCHED)
        h_out = host(np.full(batch * M * N, np.nan), float)
        st = rt.run_host(cb.K_GEMM_FP8, 2, host(A), h_out, batch * M * N, M=M, N=N, K=K, h_aux=host(B), flags=3, mode=MM_BATCHED | bit,
                         scale_a=host(sa, float), scale_b=host(sb, float))
        assert (h_out.numpy().view(np.uint32) == want).all() and st.as_dict() == sw
        # groups
        ro = zipf_offsets(10, 700, start=3, seed=9)
        G, R = len(ro) - 1, ro[-1] - ro[0]
        A, B = Fp8.stacked_operands(ro[-1], N, K, G, seed=5)
        sa, sb = row_col_scales(ro[-1], G * N, seed=5)
        sa, sb = (sa, sb) if rowwise else (sa[:1], sb[:1])
        h_ro = torch.tensor(ro, dtype=torch.int64)
        want, sw = scaled(rt, 3, A, B, sa, sb, rowwise=rowwise, M=G, n=R * N, mode=MM_GROUPED, rows=h_ro.cuda(), unit_base=9,
                          out=torch.zeros(ro[-1] * N, dtype=torch.float32, device="cuda"))
        h_out = host(np.zeros(ro[-1] * N), float)
        st = rt.run_host(cb.K_GEMM_FP8, 3, host(A), h_out, R * N, M=G, N=N, K=K, h_aux=host(B), flags=3, mode=MM_GROUPED | bit, h_rows=h_ro,
                         unit_base=9, scale_a=host(sa, float), scale_b=host(sb, float))
        assert rt.last_host_path == "groups" and (h_out.numpy().view(np.uint32) == want).all() and st.as_dict() == sw


def test_run_refuses_scales_of_the_wrong_kind_or_length(rt):
    import torch
    import coast_b200 as cb
    M = N = K = 128
    A, B = Fp8.int_operands(M, N, K, seed=1)
    dA, dB = dev(Fp8, A), dev(Fp8, B)
    ok_a, ok_b = torch.ones(M, device="cuda"), torch.ones(N, device="cuda")
    bad = [(MM_SCALE_ROWWISE, ok_a[:-1], ok_b), (MM_SCALE_ROWWISE, ok_a, torch.ones(2 * N, device="cuda")),
           (MM_SCALE_ROWWISE, ok_a.double(), ok_b), (MM_SCALE_ROWWISE, ok_a.cpu(), ok_b), (MM_SCALE_TENSOR, ok_a, ok_b[:1]),
           (MM_SCALE_TENSOR, None, ok_b[:1]), (MM_SCALE_ROWWISE, torch.ones(2 * M, device="cuda")[::2], ok_b)]
    for mode, a, b in bad:
        with pytest.raises(cb.CoastError) as e:
            rt.run(cb.K_GEMM_FP8, 3, dA, M * N, M=M, N=N, K=K, aux=dB, mode=mode, scale_a=a, scale_b=b)
        assert e.value.code == cb.runtime.ERR_BAD_ARG


def test_8192_cubed_tmr_rowwise_against_float64_on_the_device(rt):
    import torch
    import coast_b200 as cb
    M = N = K = 8192
    g = torch.Generator(device="cuda").manual_seed(8192)
    dA = (torch.rand(M, K, device="cuda", generator=g) * 2 - 1).to(torch.float8_e4m3fn)
    dBt = (torch.rand(N, K, device="cuda", generator=g) * 2 - 1).to(torch.float8_e4m3fn)
    sa = (2.0 ** (torch.rand(M, device="cuda", generator=g) * 16 - 8)).float()
    sb = -(2.0 ** (torch.rand(N, device="cuda", generator=g) * 16 - 8)).float()
    out, st = rt.run(cb.K_GEMM_FP8, 3, dA, M * N, M=M, N=N, K=K, aux=dBt, mode=MM_BT | MM_SCALE_ROWWISE, flags=3, scale_a=sa, scale_b=sb)
    assert st.errors_corrected == 0 and st.syncs == M * N
    a64, b64 = dA.double(), dBt.double()
    c64 = a64 @ b64.t()
    s = sa.double()[:, None] * sb.double()[None, :]
    want = c64 * s
    tol = 2.0 ** -10 * (a64.abs() @ b64.abs().t()) * s.abs() + 2.0 ** -23 * want.abs() + 2.0 ** -148
    err = (out.view(torch.float32).view(M, N).double() - want).abs()
    assert bool((err <= tol).all()), float((err - tol).max())
