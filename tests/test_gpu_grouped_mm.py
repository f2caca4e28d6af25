"""GPU (H100): grouped matmuls (COAST_MM_GROUPED) -- G products that share N and K, each with its own row count, in one launch,
on every matmul path: the u8-limb tensor-core kernel, the register-tiled kernel, the plain kernel and the TF32 GEMM (128 x 128
tiles on single CTAs, unprotected and protected).

A grouped launch must equal G single launches (include/coast_rt.h), product g with M = ro[g+1] - ro[g], d_in + ro[g]*K,
d_aux + g*K*N, d_out + ro[g]*N and unit_base + (ro[g] - ro[0])*N: every output element, the five counters and the status bytes,
bit for bit.  The u32 products are compared with single launches on the plain kernel; TF32 on integer-valued operands (exact in
fp32 whatever the order of the additions) with a float64 reference, on general operands with single launches whose A is
zero-padded to 128 rows.  Row tables start past row 0 (the TF32 A map is rebased on the device), include empty products, one-row
products and one large product, and the output buffers start poisoned: rows outside [ro[0], ro[G]) must keep the poison."""
import pytest

from test_gpu_stream_exact import GiB, _free, _room

pytestmark = pytest.mark.gpu

POISON = 0x5A5A5A5A
M32 = 0xFFFFFFFF
KNOBS = ("COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT", "COAST_MM_PATH",
         "COAST_HOST_CHUNK_BYTES", "COAST_HOST_PATH")


def _env(monkeypatch, **env):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def row_table(G, total, seed, first=5):
    """G + 1 offsets from row `first`: about a quarter of the products empty, some with one row, one with a third of the rows"""
    import random
    rnd = random.Random(seed)
    w = [0 if rnd.random() < 0.25 else (1 if rnd.random() < 0.2 else rnd.randint(1, 100)) for _ in range(G)]
    w[rnd.randrange(G)] = sum(w) // 2 + 1
    rows = [x * total // max(sum(w), 1) for x in w]
    rows[max(range(G), key=lambda g: w[g])] += total - sum(rows)
    ro = [first]
    for r in rows:
        ro.append(ro[-1] + r)
    return ro


def operands(rt, kernel, rows, G, N, K, seed, integer=True):
    import torch
    import coast_b200 as cb
    if kernel == cb.K_MM_U32:
        A = torch.empty(rows * K, dtype=torch.int32, device="cuda")
        B = torch.empty(G * K * N, dtype=torch.int32, device="cuda")
        rt.fill_philox(A, seed=seed)
        rt.fill_philox(B, seed=seed + 1)
        return A, B
    g = torch.Generator(device="cuda").manual_seed(seed)
    if integer:
        return (torch.randint(-8, 9, (rows * K,), dtype=torch.float32, device="cuda", generator=g),
                torch.randint(-8, 9, (G * K * N,), dtype=torch.float32, device="cuda", generator=g))
    return (torch.randn(rows * K, device="cuda", generator=g), torch.randn(G * K * N, device="cuda", generator=g))


def poisoned(n, kernel):
    import torch
    import coast_b200 as cb
    out = torch.full((n,), POISON, dtype=torch.int32, device="cuda")
    return out if kernel == cb.K_MM_U32 else out.view(torch.float32)


def table(n, nc, n_sites, seed):
    import torch
    import coast_b200 as cb
    g = torch.Generator(device="cuda").manual_seed(seed)
    hit = torch.rand(n, device="cuda", generator=g) < 0.3
    rep = torch.randint(0, 4, (n,), device="cuda", generator=g)
    site = torch.randint(0, n_sites + 1, (n,), device="cuda", generator=g)
    bit = torch.randint(0, 32, (n,), device="cuda", generator=g)
    e = cb.fault_entry(0, 0, 0) | (rep << 29) | (site << 5) | bit
    e = torch.where(hit, e, torch.zeros_like(e))
    return ((e + 2 ** 31) % 2 ** 32 - 2 ** 31).to(torch.int32)


def grouped(rt, kernel, nc, A, B, out, ro, N, K, *, flags=3, plan=None, base=0, status=None, lo=0, hi=None):
    """one grouped launch over products [lo, hi) of the table (a shard when not all of them)"""
    import torch
    import coast_b200 as cb
    hi = len(ro) - 1 if hi is None else hi
    rows = torch.tensor(ro, dtype=torch.int64, device="cuda")
    d = rt.make_desc(kernel, nc, A, out, (ro[hi] - ro[lo]) * N, flags=flags, mode=cb.MM_GROUPED, M=hi - lo, N=N, K=K,
                     d_aux=B.data_ptr() + 4 * lo * K * N, plan=plan, unit_base=base + (ro[lo] - ro[0]) * N, d_status=status,
                     d_rows=rows.data_ptr() + 8 * lo)
    rt.launch(d)
    torch.cuda.synchronize()
    return rows


def singles(rt, kernel, nc, A, B, out, ro, N, K, *, flags=3, plan=None, tab=None, base=0, status=None):
    """the same products as G single launches; a TABLE plan is sliced per product, status bytes per product"""
    import coast_b200 as cb
    for g in range(len(ro) - 1):
        m = ro[g + 1] - ro[g]
        if m == 0:
            continue
        u0 = (ro[g] - ro[0]) * N
        pg = cb.FaultPlan(mode=cb.PLAN_TABLE, table=tab[u0:u0 + m * N]) if tab is not None else plan
        d = rt.make_desc(kernel, nc, A[ro[g] * K:ro[g + 1] * K], out[ro[g] * N:ro[g + 1] * N], m * N, flags=flags, M=m, N=N, K=K,
                         d_aux=B[g * K * N:(g + 1) * K * N], plan=pg, unit_base=base + u0,
                         d_status=status[u0:u0 + m * N] if status is not None else None)
        rt.launch(d)


def _plan(kind, n, nc, sites, seed):
    import coast_b200 as cb
    if kind == "table":
        tab = table(n, nc, sites, seed)
        return cb.FaultPlan(mode=cb.PLAN_TABLE, table=tab), tab
    if kind in ("bernoulli", "majority"):
        return cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=seed, p=0.3), None
    return None, None


def _poison_kept(C, ro, N):
    import torch
    v = C.view(torch.int32)
    return bool((v[:ro[0] * N] == POISON).all()) and bool((v[ro[-1] * N:] == POISON).all())


# (id, N, K, G, total rows, COAST_MM_PATH of the grouped launch, the kernel it must pick)
U32_PATHS = [
    ("tc", 64, 128, 37, 30000, None, "xmr_mm_u32_tc_grp"),        # 235+ row tiles x 2 (NC 2/3) columns: >= 3 tiles per CTA
    ("tiled", 128, 32, 23, 3000, None, "xmr_mm_u32_tiled_grp"),
    ("plain", 9, 9, 41, 700, None, "xmr_mm_u32_grp"),
]


@pytest.mark.parametrize("plan_kind", ["none", "bernoulli", "table", "majority"])
@pytest.mark.parametrize("nc", [1, 2, 3])
@pytest.mark.parametrize("path", U32_PATHS, ids=[p[0] for p in U32_PATHS])
def test_grouped_u32_equals_single_launches_on_the_plain_kernel(rt, monkeypatch, capfd, path, nc, plan_kind):
    """every path at NC 1/2/3 under every plan, global units crossing 2^32: outputs, counters and status bytes equal G single
    launches on the plain kernel, and the rows outside the table keep their poison"""
    import torch
    import coast_b200 as cb
    pid, N, K, G, total, mm_path, name = path
    _env(monkeypatch)
    ro = row_table(G, total, seed=nc + len(pid))
    n = (ro[-1] - ro[0]) * N
    base = (1 << 32) - n // 2 - 7
    flags = 3 | (cb.F_MAJORITY_VOTER if plan_kind == "majority" else 0)
    A, B = operands(rt, cb.K_MM_U32, ro[-1] + 3, G, N, K, seed=17 * nc)
    plan, tab = _plan(plan_kind, n, nc, K, seed=nc)
    rt.sync()
    one, s1 = poisoned((ro[-1] + 3) * N, cb.K_MM_U32), torch.zeros(n, dtype=torch.uint8, device="cuda")
    capfd.readouterr()
    grouped(rt, cb.K_MM_U32, nc, A, B, one, ro, N, K, flags=flags | cb.F_VERBOSE, plan=plan, base=base, status=s1)
    st1 = rt.sync()
    err = capfd.readouterr().err
    assert f"{name}_inj{0 if plan_kind == 'none' else 1}_nc{nc} " in err, err
    monkeypatch.setenv("COAST_MM_PATH", "naive")
    many, sn = poisoned((ro[-1] + 3) * N, cb.K_MM_U32), torch.zeros(n, dtype=torch.uint8, device="cuda")
    singles(rt, cb.K_MM_U32, nc, A, B, many, ro, N, K, flags=flags, plan=plan, tab=tab, base=base, status=sn)
    stn = rt.sync()
    assert torch.equal(one.view(torch.int32), many.view(torch.int32))
    assert st1 == stn, (st1, stn)
    assert torch.equal(s1, sn)
    assert _poison_kept(one, ro, N)
    if plan_kind == "none":
        assert st1.injected == 0 and (nc < 3 or st1.syncs == n)
    else:
        assert st1.injected > 0


@pytest.mark.parametrize("nc", [2, 3])
def test_no_mem_replication_votes_every_k_step_of_every_product(rt, monkeypatch, capfd, nc):
    """-noMemReplication: the plain kernel with K + 1 votes per unit, grouped as single"""
    import coast_b200 as cb
    _env(monkeypatch)
    N, K, G = 128, 32, 11
    ro = row_table(G, 400, seed=3)
    n = (ro[-1] - ro[0]) * N
    flags = 3 | cb.F_NO_MEM_REPLICATION
    A, B = operands(rt, cb.K_MM_U32, ro[-1], G, N, K, seed=9)
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=5, p=0.3)
    rt.sync()
    one = poisoned(ro[-1] * N, cb.K_MM_U32)
    capfd.readouterr()
    grouped(rt, cb.K_MM_U32, nc, A, B, one, ro, N, K, flags=flags | cb.F_VERBOSE, plan=plan, base=1 << 33)
    st1 = rt.sync()
    assert f"xmr_mm_u32_grp_inj1_nc{nc} " in capfd.readouterr().err
    many = poisoned(ro[-1] * N, cb.K_MM_U32)
    singles(rt, cb.K_MM_U32, nc, A, B, many, ro, N, K, flags=flags, plan=plan, base=1 << 33)
    stn = rt.sync()
    assert (one.view(-1) == many.view(-1)).all() and st1 == stn
    if nc == 3:
        assert st1.syncs == n * (K + 1)


def tf32_ref(A, B, ro, N, K):
    """float64 C rows [ro[0], ro[G]) of the grouped product"""
    import torch
    outs = []
    for g in range(len(ro) - 1):
        a = A[ro[g] * K:ro[g + 1] * K].view(-1, K).double()
        outs.append(a @ B[g * K * N:(g + 1) * K * N].view(K, N).double())
    return torch.cat(outs).view(-1)


# (nc, N, the kernel)
TF32_CASES = [(1, 256, "xmr_gemm_tf32n_grp_inj0_nc1"), (1, 128, "xmr_gemm_tf32n_grp_inj0_nc1"), (2, 128, "xmr_gemm_tf32_grp_inj0_nc2"),
              (3, 128, "xmr_gemm_tf32_grp_inj0_nc3"), (3, 384, "xmr_gemm_tf32_grp_inj0_nc3")]


@pytest.mark.parametrize("nc,N,name", TF32_CASES)
def test_tf32_integer_valued_is_exact(rt, monkeypatch, capfd, nc, N, name):
    """integer-valued operands: every output equals the float64 product, the counters are the clean ones; with enough rows for
    three tiles per persistent CTA"""
    import coast_b200 as cb
    _env(monkeypatch)
    K, G = 64, 29
    ro = row_table(G, 400 * 128, seed=N + nc)              # >= 400 row tiles: >= 3 tiles per CTA
    n = (ro[-1] - ro[0]) * N
    A, B = operands(rt, cb.K_GEMM_TF32, ro[-1] + 2, G, N, K, seed=nc)
    rt.sync()
    C = poisoned((ro[-1] + 2) * N, cb.K_GEMM_TF32)
    capfd.readouterr()
    grouped(rt, cb.K_GEMM_TF32, nc, A, B, C, ro, N, K, flags=3 | cb.F_VERBOSE, base=(1 << 32) - n // 3)
    st = rt.sync()
    assert name + " " in capfd.readouterr().err
    assert (C[ro[0] * N:ro[-1] * N].double() == tf32_ref(A, B, ro, N, K)).all()
    assert _poison_kept(C, ro, N)
    assert st.injected == st.errors_corrected == st.dwc_detected == 0 and (nc < 3 or st.syncs == n)


@pytest.mark.parametrize("nc", [1, 3])
def test_tf32_general_operands_equal_padded_single_launches(rt, monkeypatch, nc):
    """general fp32 operands: each product's rows equal a single launch of its A zero-padded to a multiple of 128 rows"""
    import torch
    import coast_b200 as cb
    _env(monkeypatch)
    N, K, G = 128, 96, 13
    ro = row_table(G, 3000, seed=nc)
    A, B = operands(rt, cb.K_GEMM_TF32, ro[-1], G, N, K, seed=4, integer=False)
    C = poisoned(ro[-1] * N, cb.K_GEMM_TF32)
    grouped(rt, cb.K_GEMM_TF32, nc, A, B, C, ro, N, K)
    rt.sync()
    for g in range(G):
        m = ro[g + 1] - ro[g]
        if not m:
            continue
        mp = -(-m // 128) * 128
        a = torch.zeros(mp * K, device="cuda")
        a[:m * K] = A[ro[g] * K:ro[g + 1] * K]
        c = torch.empty(mp * N, device="cuda")
        rt.run(cb.K_GEMM_TF32, nc, a, mp * N, flags=3, M=mp, N=N, K=K, aux=B[g * K * N:(g + 1) * K * N], out=c)
        assert torch.equal(C[ro[g] * N:ro[g + 1] * N].view(torch.int32), c[:m * N].view(torch.int32)), g


@pytest.mark.parametrize("kernel,nc,N,K", [(4, 3, 128, 64), (4, 1, 256, 32), (3, 3, 64, 128), (3, 2, 128, 32)])
def test_equal_tile_multiples_are_the_batched_launch(rt, monkeypatch, kernel, nc, N, K):
    """products of 128 rows each: bit-identical outputs and counters to a COAST_MM_BATCHED launch"""
    import torch
    import coast_b200 as cb
    _env(monkeypatch, COAST_GEMM_PAIR="0")
    G, M = 20, 128
    ro = [M * g for g in range(G + 1)]
    A, B = operands(rt, kernel, G * M, G, N, K, seed=2)
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=8, p=0.2)
    rt.sync()
    one = poisoned(G * M * N, kernel)
    grouped(rt, kernel, nc, A, B, one, ro, N, K, plan=plan, base=99)
    st1 = rt.sync()
    two = poisoned(G * M * N, kernel)
    rt.launch(rt.make_desc(kernel, nc, A, two, G * M * N, flags=3, mode=cb.MM_BATCHED, M=M, N=N, K=K, d_aux=B, plan=plan, unit_base=99))
    st2 = rt.sync()
    assert torch.equal(one.view(torch.int32), two.view(torch.int32)) and st1 == st2


@pytest.mark.parametrize("kernel", [3, 4])
def test_shards_over_groups_equal_one_launch(rt, monkeypatch, kernel):
    """three shards from shard_groups (d_rows + g_lo, the same d_in and d_out) equal the whole launch"""
    import torch
    import coast_b200 as cb
    from coast_b200.shard import shard_groups
    _env(monkeypatch)
    N, K, G = 128, 128, 31
    ro = row_table(G, 5000, seed=kernel)
    A, B = operands(rt, kernel, ro[-1], G, N, K, seed=kernel)
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=1, p=0.1)
    rt.sync()
    one = poisoned(ro[-1] * N, kernel)
    grouped(rt, kernel, 3, A, B, one, ro, N, K, plan=plan, base=1 << 40)
    st1 = rt.sync()
    many = poisoned(ro[-1] * N, kernel)
    cuts = [shard_groups(ro, r, 3) for r in range(3)]
    assert cuts[0][0] == 0 and cuts[-1][1] == G and all(a[1] == b[0] for a, b in zip(cuts, cuts[1:]))
    for lo, hi in cuts:
        if hi > lo:
            grouped(rt, kernel, 3, A, B, many, ro, N, K, plan=plan, base=1 << 40, lo=lo, hi=hi)
    stn = rt.sync()
    assert torch.equal(one.view(torch.int32), many.view(torch.int32)) and st1 == stn


@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("kernel,N,K", [(3, 64, 128), (4, 128, 64)])
def test_host_call_in_many_chunks_equals_the_device_launch(rt, monkeypatch, kernel, N, K, pinned):
    """coast_run_host with a small chunk budget (many chunks of whole products): outputs and counters of the device launch"""
    import numpy as np
    import torch
    import coast_b200 as cb
    _env(monkeypatch)
    G = 40
    ro = row_table(G, 6000, seed=7)
    A, B = operands(rt, kernel, ro[-1], G, N, K, seed=3)
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=6, p=0.2)
    rt.sync()
    C = poisoned(ro[-1] * N, kernel)
    grouped(rt, kernel, 3, A, B, C, ro, N, K, plan=plan, base=12345)
    st1 = rt.sync()
    monkeypatch.setenv("COAST_HOST_CHUNK_BYTES", str(300000))
    hA, hB = A.cpu(), B.cpu()
    hC = torch.full((ro[-1] * N,), POISON, dtype=torch.int32)
    if pinned:
        hA, hB, hC = hA.pin_memory(), hB.pin_memory(), hC.pin_memory()
    h_rows = np.array(ro, dtype=np.uint64)
    st2 = rt.run_host(kernel, 3, hA, hC, (ro[-1] - ro[0]) * N, flags=3, mode=cb.MM_GROUPED, M=G, N=N, K=K, h_aux=hB, plan=plan,
                      unit_base=12345, h_rows=h_rows)
    assert rt.last_host_path == "groups"
    assert torch.equal(hC, C.view(torch.int32).cpu()) and st1 == st2


@pytest.mark.parametrize("kernel,N,K", [(4, 128, 32), (3, 64, 128), (3, 128, 32), (3, 9, 9)], ids=["tf32", "tc", "tiled", "plain"])
def test_a_malformed_table_is_clamped_inside_the_buffers(rt, monkeypatch, kernel, N, K):
    """a launched table that decreases and overshoots R: nothing outside rows [ro[0], ro[0] + R) is written, and the rows only
    the well-formed first product covers are its single launch's"""
    import torch
    import coast_b200 as cb
    _env(monkeypatch)
    R, first = 700, 40
    ro = [first, first + 300, first + 300, first + 200, first + 5000]     # product 2 decreases: no rows; product 3 clamps at R
    A, B = operands(rt, kernel, first + R + 40, 4, N, K, seed=5)
    C = poisoned((first + R + 40) * N, kernel)
    rows = torch.tensor(ro, dtype=torch.int64, device="cuda")
    rt.launch(rt.make_desc(kernel, 3, A, C, R * N, flags=3, mode=cb.MM_GROUPED, M=4, N=N, K=K, d_aux=B, d_rows=rows))
    rt.sync()
    v = C.view(torch.int32)
    assert (v[:first * N] == POISON).all() and (v[(first + R) * N:] == POISON).all()
    ok = poisoned((first + R + 40) * N, kernel)
    good = [first, first + 300]
    grouped(rt, kernel, 3, A, B, ok, good, N, K)
    rt.sync()
    assert torch.equal(v[first * N:(first + 200) * N], ok.view(torch.int32)[first * N:(first + 200) * N])   # product 3 restarts at 200


def test_runtime_run_refuses_a_malformed_table(rt):
    import torch
    import coast_b200 as cb
    A = torch.zeros(100 * 32, device="cuda")
    B = torch.zeros(2 * 32 * 128, device="cuda")
    for ro in ([0, 50, 40], [0, 50, 90]):                    # decreasing; not spanning n_units / N rows
        with pytest.raises(cb.CoastError):
            rt.run(cb.K_GEMM_TF32, 3, A, 100 * 128, flags=3, mode=cb.MM_GROUPED, M=2, N=128, K=32, aux=B,
                   rows=torch.tensor(ro, dtype=torch.int64, device="cuda"))


def test_tmr_launch_past_2p32_units_against_float64(rt, monkeypatch):
    """one TF32 TMR launch of 2^32 + 2^21 units (integer-valued operands): every output row block against float64 on the device"""
    import torch
    import coast_b200 as cb
    _env(monkeypatch)
    N, K = 256, 32
    R = (1 << 24) + (1 << 13)
    _room(R * (K + N) * 4 + 4 * GiB)
    ro = [0, 1000, 1000 + (1 << 23), R - 77, R]
    G = len(ro) - 1
    A, B = operands(rt, cb.K_GEMM_TF32, R, G, N, K, seed=1)
    C = torch.empty(R * N, device="cuda")
    grouped(rt, cb.K_GEMM_TF32, 3, A, B, C, ro, N, K, base=5)
    st = rt.sync()
    assert st.syncs == R * N and st.errors_corrected == 0
    step = 1 << 20
    for g in range(G):
        Bg = B[g * K * N:(g + 1) * K * N].view(K, N).double()
        for r in range(ro[g], ro[g + 1], step):
            e = min(r + step, ro[g + 1])
            ref = A[r * K:e * K].view(-1, K).double() @ Bg
            assert (C[r * N:e * N].view(-1, N).double() == ref).all(), (g, r)
    del A, B, C
    _free()
