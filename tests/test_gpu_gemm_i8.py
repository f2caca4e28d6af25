"""GPU (H100): GEMM_I8 (COAST_K_GEMM_I8, the xmr_gemm_i8* kernels): int8 A and B, int32 C = A . B mod 2^32, integer vote.

The product is exact for any operands and any K, so every test is bit for bit: uniform random int8 data against the CPU reference
(tests/gemm_i8_ref.py) with every output word, all five counters and d_status, without a plan, with Bernoulli plans across 2^32
and TABLE plans, for both voters, with B and B^T; batches and Zipf-routed groups with empty experts; multi-wave shapes, a shard
with a nonzero unit_base and the host call; sums that wrap past 2^31; unprotected torch._int_mm and a MM_U32 launch on the
sign-extended operands; and TABLE plans that flip bit 31 of zero elements and flip elements whose words are fp32 NaN patterns, where
an fp32 vote would go wrong."""
import numpy as np
import pytest

import gemm_i8_ref as ref
from mm_gpu import POISON, STAT_KEYS, add_stats, env, no_stats, transposed
from coast_b200.runtime import K_GEMM_I8, K_MM_U32, MM_B_TRANSPOSED as MM_BT, MM_BATCHED, MM_GROUPED

pytestmark = pytest.mark.gpu

RO = [3, 3, 100, 101, 101, 500, 700, 828]          # from row 3: empty products, a one-row product, a 128-row product


def operands(rows, N, K, seed, P=1):
    """uniform int8: rows x K of A and P stacked K x N matrices B"""
    rng = np.random.default_rng(seed)
    return (rng.integers(-128, 128, size=(rows, K)).astype(np.int8), rng.integers(-128, 128, size=(P * K, N)).astype(np.int8))


def zipf_offsets(G, R, start, seed):
    """a mixture-of-experts routing: Zipf-like expert loads, some experts empty, rows from `start`"""
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, G + 1) ** 1.1
    rng.shuffle(w)
    rows = np.floor(R * w / w.sum()).astype(int)
    rows[rng.choice(G, size=G // 5, replace=False)] = 0
    rows[np.argmax(rows)] += R - rows.sum()
    return [int(start)] + [int(start + x) for x in np.cumsum(rows)]


def dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def gpu(rt, nc, A, B, *, flags=3, plan=None, table=None, unit_base=0, status=None, mode=0, M=None, n=None, rows=None, out=None,
        bt=False):
    """A: (rows x K), B: (P K x N) int8 -> (C words as uint32, flat; stats dict); bt: launch with B^T"""
    import torch
    import coast_b200 as cb
    K, N = A.shape[1], B.shape[1]
    M = A.shape[0] if M is None else M
    n = A.shape[0] * N if n is None else n
    if table is not None:
        plan = cb.FaultPlan(mode=cb.PLAN_TABLE, table=dev(table.view(np.int32)))
    if out is None:
        out = torch.full((A.shape[0] * N,), POISON, dtype=torch.int32, device="cuda")
    aux = dev(transposed(B, K)) if bt else dev(B)
    _, st = rt.run(K_GEMM_I8, nc, dev(A), n, M=M, N=N, K=K, aux=aux, flags=flags, plan=plan, unit_base=unit_base, status=status,
                   mode=mode | (MM_BT if bt else 0), rows=rows, out=out)
    return out.cpu().numpy().view(np.uint32), st.as_dict()


def cpu(oracle, nc, A, B, *, flags=3, plan_kw=None, table=None, unit_base=0, acc=None):
    plan = None
    if table is not None:
        plan = oracle.make_plan(oracle.PLAN_TABLE, table=table)
    elif plan_kw:
        plan = oracle.make_plan(oracle.PLAN_BERNOULLI, **plan_kw)
    return ref.run(oracle, nc, A, B, flags=flags, plan=plan, table=table, unit_base=unit_base, acc=acc)


def check(rt, oracle, nc, A, B, c, *, bt=False, acc=None):
    """one launch of case c (flags, plan_kw or table, unit_base) against the reference: words, counters and d_status"""
    import torch
    import coast_b200 as cb
    n = A.shape[0] * B.shape[1]
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, **c["plan_kw"]) if "plan_kw" in c else None
    status = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    g, gs = gpu(rt, nc, A, B, flags=c.get("flags", 3), plan=plan, table=c.get("table"), unit_base=c.get("unit_base", 0),
                status=status, bt=bt)
    o, os_, ostat = cpu(oracle, nc, A, B, acc=acc, **c)
    assert (g == o).all(), (nc, bt, sorted(c), np.flatnonzero(g != o)[:8])
    assert {k: gs[k] for k in STAT_KEYS} == {k: os_[k] for k in STAT_KEYS}, (nc, bt, sorted(c))
    assert np.array_equal(status.cpu().numpy(), ostat), (nc, bt, sorted(c))
    return g, gs


def random_table(oracle, n, count, seed):
    """count random entries, a fifth of them inert (site 1, or replica 3 on every NC)"""
    rng = np.random.default_rng(seed)
    tab = np.zeros(n, dtype=np.uint32)
    for u in rng.choice(n, size=count, replace=False):
        tab[u] = oracle.fault_entry(int(rng.integers(0, 4)), 0 if rng.random() < 0.8 else 1, int(rng.integers(0, 32)))
    return tab


# (id, environment, NC, M, N, the kernel the launcher must pick)
VARIANTS = [
    ("narrow_nc1", {}, 1, 256, 384, "xmr_gemm_i8n_inj0_nc1"),
    ("wide_nc1", {"COAST_GEMM_PAIR": "0"}, 1, 256, 256, "xmr_gemm_i8_inj0_nc1"),
    ("pair_nc1", {}, 1, 256, 256, "xmr_gemm_i8p_inj0_nc1"),
    ("pair_nc2", {}, 2, 256, 128, "xmr_gemm_i8p_inj0_nc2"),
    ("single_nc2", {"COAST_GEMM_PAIR": "0"}, 2, 256, 128, "xmr_gemm_i8_inj0_nc2"),
    ("single_nc3", {}, 3, 256, 128, "xmr_gemm_i8_inj0_nc3"),
    ("pair_nc3", {"COAST_GEMM_PAIR": "1"}, 3, 256, 256, "xmr_gemm_i8p_inj0_nc3"),
]


@pytest.mark.parametrize("K", [128, 1152])
@pytest.mark.parametrize("variant", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_uniform_int8_bit_exact_with_the_reference(rt, oracle, variant, K, monkeypatch, capfd):
    """every word, the five counters and d_status, with B and B^T: no plan, Bernoulli across 2^32, TABLE, majority voter"""
    import coast_b200 as cb
    _, e, nc, M, N, kname = variant
    env(monkeypatch, **e)
    A, B = operands(M, N, K, seed=K + nc)
    n = M * N
    capfd.readouterr()
    gpu(rt, nc, A, B, flags=cb.F_VERBOSE)
    assert f"{kname} " in capfd.readouterr().err
    base = 2 ** 32 - n // 2
    acc = ref.exact(A, B)
    cases = [dict(), dict(plan_kw=dict(seed=K, p=0.3), unit_base=base), dict(table=random_table(oracle, n, 300, K + nc), unit_base=base),
             dict(flags=3 | cb.F_MAJORITY_VOTER, plan_kw=dict(seed=K + 1, p=0.3))]
    for bt in (False, True):
        for c in cases:
            _, gs = check(rt, oracle, nc, A, B, c, bt=bt, acc=acc)
            if c:
                assert gs["injected"] > 0


@pytest.mark.parametrize("bt", [False, True])
@pytest.mark.parametrize("nc", [1, 2, 3])
def test_batched_and_grouped_equal_the_reference_per_product(rt, oracle, nc, bt):
    """a batch, fixed groups with empty products, and Zipf-routed groups: per product, the reference with the product's
    unit_base; d_out rows outside the groups keep their poison"""
    import torch
    import coast_b200 as cb
    N, K = 256, 384
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=3, p=0.2)
    base = 2 ** 32 - 5000
    M, batch = 128, 5
    A, B = operands(batch * M, N, K, seed=nc, P=batch)
    g, st = gpu(rt, nc, A, B, M=M, mode=MM_BATCHED, plan=plan, unit_base=base, bt=bt)
    tot = no_stats()
    for b in range(batch):
        o, s, _ = cpu(oracle, nc, A[b * M:(b + 1) * M], B[b * K:(b + 1) * K], plan_kw=dict(seed=3, p=0.2), unit_base=base + b * M * N)
        assert (g[b * M * N:(b + 1) * M * N] == o).all(), b
        add_stats(tot, s)
    assert st == tot and st["injected"] > 0
    for ro in (RO, zipf_offsets(16, 1500, 40, seed=nc)):
        G, R, rows_alloc = len(ro) - 1, ro[-1] - ro[0], ro[-1] + 40
        assert any(ro[i + 1] == ro[i] for i in range(G))                 # at least one empty product
        A, B = operands(rows_alloc, N, K, seed=nc + 10, P=G)
        out = torch.full((rows_alloc * N,), POISON, dtype=torch.int32, device="cuda")
        g, st = gpu(rt, nc, A, B, M=G, n=R * N, mode=MM_GROUPED, rows=dev(np.array(ro, dtype=np.int64)), plan=plan, unit_base=base,
                    out=out, bt=bt)
        g = g.reshape(rows_alloc, N)
        assert (g[:ro[0]] == POISON).all() and (g[ro[-1]:] == POISON).all()
        tot = no_stats()
        for i in range(G):
            if ro[i + 1] == ro[i]:
                continue
            o, s, _ = cpu(oracle, nc, A[ro[i]:ro[i + 1]], B[i * K:(i + 1) * K], plan_kw=dict(seed=3, p=0.2),
                          unit_base=base + (ro[i] - ro[0]) * N)
            assert (g[ro[i]:ro[i + 1]].ravel() == o).all(), (G, i)
            add_stats(tot, s)
        assert st == tot and st["injected"] > 0


RUNS = [({"COAST_GEMM_PAIR": p}, nc) for nc in (1, 2, 3) for p in ("0", "1")] + [
    ({"COAST_GEMM_TAIL_SPLIT": "0"}, 1), ({"COAST_GEMM_GROUP_M": "3"}, 3), ({"COAST_GEMM_L2_HINTS": "0"}, 3)]


def test_multi_wave_shapes_equal_the_exact_product(rt, oracle, monkeypatch):
    """4096 x 2048 on 128-row tiles: 256 to 512 tiles on 132 CTAs, every variant and switch, B and B^T, with a sparse TABLE
    plan; and 4096 x 2304 unprotected on 128 x 256 tiles: 288 tiles, whose last 24 are split in halves"""
    M, N, K = 4096, 2048, 256
    A, B = operands(M, N, K, seed=41)
    acc = ref.exact(A, B)
    n = M * N
    tab = random_table(oracle, n, 2000, 41)
    for e, nc in RUNS:
        env(monkeypatch, **e)
        for bt in (False, True):
            g, st = gpu(rt, nc, A, B, bt=bt)
            assert (g == acc.ravel()).all() and st["errors_corrected"] == st["dwc_detected"] == 0, (e, nc, bt)
        check(rt, oracle, nc, A, B, dict(table=tab, unit_base=7), acc=acc)
    env(monkeypatch, COAST_GEMM_PAIR="0")
    A, B = operands(4096, 2304, 128, seed=42)
    g, _ = gpu(rt, 1, A, B)
    assert (g == ref.exact(A, B).ravel()).all()


def test_a_shard_with_a_nonzero_unit_base_equals_its_rows_of_the_whole(rt, oracle):
    """rows [256, 640) of a 1024-row product, launched alone with unit_base = 256 N + base: the whole launch's words, counters
    restricted to the shard, and the reference with the shard's unit_base"""
    import torch
    import coast_b200 as cb
    M, N, K = 1024, 256, 512
    A, B = operands(M, N, K, seed=5)
    base, lo, hi = 2 ** 32 - 70000, 256, 640
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=9, p=0.05)
    whole, _ = gpu(rt, 3, A, B, plan=plan, unit_base=base)
    out = torch.full(((hi - lo) * N,), POISON, dtype=torch.int32, device="cuda")
    part, st = gpu(rt, 3, A[lo:hi], B, plan=plan, unit_base=base + lo * N, out=out)
    assert (part == whole[lo * N:hi * N]).all()
    o, os_, _ = cpu(oracle, 3, A[lo:hi], B, plan_kw=dict(seed=9, p=0.05), unit_base=base + lo * N)
    assert (part == o).all() and st == os_ and st["injected"] > 0


@pytest.mark.parametrize("pinned", [False, True])
def test_host_call_equals_the_reference(rt, oracle, pinned, monkeypatch):
    """coast_run_host: row blocks of one product, and a batch in whole-product chunks with B^T, from host int8 buffers"""
    import torch
    import coast_b200 as cb
    plan_kw = dict(seed=4, p=0.1)
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, **plan_kw)
    env(monkeypatch)

    def host(x):
        t = torch.from_numpy(np.ascontiguousarray(x))
        return t.pin_memory() if pinned else t
    M, N, K = 1024, 256, 256
    A, B = operands(M, N, K, seed=6)
    h_out = host(np.full(M * N, POISON, dtype=np.int32))
    st = rt.run_host(K_GEMM_I8, 3, host(A), h_out, M * N, M=M, N=N, K=K, h_aux=host(B), flags=3, plan=plan, unit_base=11)
    o, os_, _ = cpu(oracle, 3, A, B, plan_kw=plan_kw, unit_base=11)
    assert (h_out.numpy().view(np.uint32) == o).all() and st.as_dict() == os_ and rt.last_host_path == "row-blocks"
    M, batch = 128, 5
    A, B = operands(batch * M, N, K, seed=7, P=batch)
    h_out = host(np.full(batch * M * N, POISON, dtype=np.int32))
    env(monkeypatch, COAST_HOST_CHUNK_BYTES=str(2 * (M * K + K * N + 4 * M * N) + 100))
    st = rt.run_host(K_GEMM_I8, 2, host(A), h_out, batch * M * N, M=M, N=N, K=K, h_aux=host(transposed(B, K)), flags=3, plan=plan,
                     mode=MM_BATCHED | MM_BT, unit_base=11)
    tot = no_stats()
    for b in range(batch):
        o, s, _ = cpu(oracle, 2, A[b * M:(b + 1) * M], B[b * K:(b + 1) * K], plan_kw=plan_kw, unit_base=11 + b * M * N)
        assert (h_out.numpy().view(np.uint32)[b * M * N:(b + 1) * M * N] == o).all(), b
        add_stats(tot, s)
    assert st.as_dict() == tot and rt.last_host_path == "staged"


@pytest.mark.parametrize("K,want", [(2 ** 17, -2 ** 31), (2 ** 17 + 128, -2 ** 31 + 2 ** 21), (130688, 2141192192)])
def test_sums_past_two_to_the_31_wrap(rt, oracle, K, want):
    """all -128: every sum is 2^14 K; from K = 2^17 it wraps to INT_MIN and on (130688: the fp32 NaN pattern 0x7FA00000)"""
    M = N = 128
    A, B = np.full((M, K), -128, dtype=np.int8), np.full((K, N), -128, dtype=np.int8)
    for nc in (1, 2, 3):
        for bt in (False, True):
            g, st = gpu(rt, nc, A, B, bt=bt)
            assert (g.view(np.int32) == want).all() and st["errors_corrected"] == st["dwc_detected"] == 0, (nc, bt)
    A[5, :] = 127                                                        # row 5: -2^14 + 2^7 per k
    acc = ref.exact(A, B)
    check(rt, oracle, 3, A, B, dict(table=random_table(oracle, M * N, 500, K), unit_base=0), acc=acc)


def test_equals_torch_int_mm_and_mm_u32_on_sign_extended_operands(rt):
    """unprotected torch._int_mm (K < 2^17, so no sum leaves int32) and the protected MM_U32 path on the operands widened to 32
    bits, at NC 1 and 3, with B and B^T"""
    import torch
    for M, N, K in ((512, 384, 1024), (1024, 1024, 4096), (128, 256, 16384)):
        A, B = operands(M, N, K, seed=M + K)
        want = torch._int_mm(dev(A), dev(B)).cpu().numpy().ravel().view(np.uint32)
        mm = torch.empty(M * N, dtype=torch.int32, device="cuda")
        rt.run(K_MM_U32, 3, dev(A.astype(np.int32)), M * N, M=M, N=N, K=K, aux=dev(B.astype(np.int32)), flags=3, out=mm)
        assert (mm.cpu().numpy().view(np.uint32) == want).all(), (M, N, K)
        for nc in (1, 3):
            for bt in (False, True):
                g, _ = gpu(rt, nc, A, B, bt=bt)
                assert (g == want).all(), (M, N, K, nc, bt)


def test_integer_vote_on_zero_and_nan_pattern_words(rt, oracle):
    """TABLE plans on chosen elements: bit 31 of zero elements on every replica, and flips of every bit position on elements
    whose words are fp32 NaN patterns -- negative C in [-8388607, -1] and, at K = 130688, C = 0x7FA00000 -- for DWC and TMR
    with both voters.  An fp32 vote would take 0x80000000 for +0.0 (a silent INT_MIN under TMR's select voter, a missed flip
    under DWC) and count every NaN-pattern element as a disagreement."""
    import coast_b200 as cb
    M, N = 256, 256
    rng = np.random.default_rng(77)
    for K in (256, 130688):
        if K == 256:
            A, B = operands(M, N, K, seed=78)
            A[:64] = 0                                                   # rows 0-63: C = 0
        else:
            A, B = np.full((M, K), -128, dtype=np.int8), np.full((K, N), -128, dtype=np.int8)
            A[:64] = 0
        acc = ref.exact(A, B).ravel()
        zero = np.flatnonzero(acc == 0)
        nan = np.flatnonzero(np.isnan(acc.view(np.float32)))
        assert len(zero) >= 64 * N and len(nan) > 1000
        if K == 256:
            assert (acc.view(np.int32)[nan] < 0).all() and (acc.view(np.int32)[nan] >= -8388607).all()
        else:
            assert (acc[nan] == 0x7FA00000).all()
        for nc in (2, 3):
            tab = np.zeros(M * N, dtype=np.uint32)
            zs = rng.choice(zero, size=600, replace=False)
            for i, u in enumerate(zs):
                tab[u] = oracle.fault_entry(i % nc, 0, 31)
            for i, u in enumerate(rng.choice(nan, size=600, replace=False)):
                tab[u] = oracle.fault_entry(i % nc, 0, i % 32)
            for flags in ((3,) if nc == 2 else (3, 3 | cb.F_MAJORITY_VOTER)):
                g, gs = check(rt, oracle, nc, A, B, dict(table=tab, flags=flags, unit_base=0), acc=acc)
                assert gs["injected"] == 1200 and (gs["dwc_detected"] if nc == 2 else gs["errors_corrected"]) == 1200, (K, nc, flags)
                if nc == 3:
                    assert (g[zs] == 0).all()                            # never INT_MIN
                    assert (g == acc).all()
                else:                                                    # DWC stores replica 0: its bit-31 flips are stored
                    r0 = zs[np.arange(len(zs)) % nc == 0]
                    assert (g[r0] == 0x80000000).all()
