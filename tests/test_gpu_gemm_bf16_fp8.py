"""GPU (H100): the BF16 and FP8 GEMMs, one suite run for each operand type (tests/mm_gpu.py holds a record per type).

COAST_K_GEMM_BF16: bfloat16 A and B, fp32 accumulators and C, wgmma m64n128k16, B read in place (MN-major) from the caller's
row-major buffer, or B^T K-major with COAST_MM_B_TRANSPOSED.  COAST_K_GEMM_FP8: E4M3 A and B, wgmma m64n128k32 into the tensor
core's accumulator, fp32 C, B^T read K-major (from the byte-transposing pre-pass, or the caller's with COAST_MM_B_TRANSPOSED).
Both keep NC register accumulator replicas and the voting epilogue of GEMM_TF32.

Exact wherever arithmetic allows it: BF16 integer-valued operands with K amax^2 < 2^24 make every partial sum an exact fp32
integer; FP8 integer-valued operands whose sum_k |a_ik b_kj| is at most 2^11 (gemm_fp8_ref.EXACT_SUM) make every partial sum a
small integer the narrower FP8 accumulator keeps.  There, outputs equal the CPU reference (tests/gemm_bf16_ref.py,
tests/gemm_fp8_ref.py) and a float64 matmul bit for bit, whatever order the tensor core adds in; the FP8 accumulator's width is
measured here and must cover that domain.  General operands are held to each type's bound (mm_gpu.Bf16.bound, Fp8.bound) and to
bit-equality between every kernel variant, replica count and B layout."""
import numpy as np
import pytest

from mm_gpu import POISON, STAT_KEYS, Bf16, Fp8, add_stats, both, cpu, dev, env, gpu, no_stats, transposed
from coast_b200.runtime import MM_B_TRANSPOSED as MM_BT, MM_BATCHED, MM_GROUPED

pytestmark = pytest.mark.gpu


def per_type(cases, ids=lambda c: "-".join(map(str, c))):
    """one pytest parameter set per (type, case) of {type: [case tuple, ...]}: each type keeps its own cases"""
    return [pytest.param(t, *c, id=f"{t.name}-{ids(c)}") for t, cs in cases.items() for c in cs]


def zipf_offsets(G, R, start, seed=3):
    """a mixture-of-experts routing: Zipf-like expert loads, some experts empty, rows from `start`"""
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, G + 1) ** 1.1
    rng.shuffle(w)
    rows = np.floor(R * w / w.sum()).astype(int)
    rows[rng.choice(G, size=G // 5, replace=False)] = 0
    rows[np.argmax(rows)] += R - rows.sum()
    return [int(start)] + [int(start + x) for x in np.cumsum(rows)]


RO = [3, 3, 100, 101, 101, 500, 700, 828]          # from row 3: empty products, a one-row product, a 128-row product

# (id, environment, NC, M, N, the kernel the launcher must pick)
VARIANTS = {t: [
    ("narrow_nc1", {}, 1, 256, 384, f"xmr_gemm_{t.name}n_inj0_nc1"),                  # N % 256 != 0: 128 x 128 tiles
    ("wide_nc1", {"COAST_GEMM_PAIR": "0"}, 1, 256, 256, f"xmr_gemm_{t.name}_inj0_nc1"),  # 128 x 256 tiles
    ("pair_nc1", {}, 1, 256, 256, f"xmr_gemm_{t.name}p_inj0_nc1"),
    ("pair_nc2", {}, 2, 256, 128, f"xmr_gemm_{t.name}p_inj0_nc2"),                    # one 64-wide B box per CTA of the pair
    ("single_nc2", {"COAST_GEMM_PAIR": "0"}, 2, 256, 128, f"xmr_gemm_{t.name}_inj0_nc2"),
    ("single_nc3", {}, 3, 256, 128, f"xmr_gemm_{t.name}_inj0_nc3"),
    ("pair_nc3", {"COAST_GEMM_PAIR": "1"}, 3, 256, 256, f"xmr_gemm_{t.name}p_inj0_nc3"),
] for t in (Bf16, Fp8)}
# one k-block; one 6-stage ring exactly; one wrap; many wraps
K_RING = {Bf16: [64, 384, 448, 1088], Fp8: [128, 768, 896, 2048]}


@pytest.mark.parametrize("t,variant,K", per_type({t: [(v, K) for v in VARIANTS[t] for K in K_RING[t]] for t in VARIANTS},
                                                 ids=lambda c: f"{c[0][0]}-{c[1]}"))
def test_integer_operands_bit_exact_with_the_oracle(rt, oracle, t, variant, K, monkeypatch, capfd):
    import torch
    import coast_b200 as cb
    _, e, nc, M, N, kname = variant
    env(monkeypatch, **e)
    A, B = t.int_operands(M, N, K, seed=K + 10 * nc)
    n = M * N
    capfd.readouterr()
    gpu(rt, t, nc, A, B, flags=cb.F_VERBOSE)
    assert f"{kname} " in capfd.readouterr().err
    g, st = both(rt, oracle, t, nc, A, B)
    assert (g.view(np.float32).reshape(M, N).astype(np.float64) == t.value(A).astype(np.float64) @ t.value(B).astype(np.float64)).all()
    assert st["errors_corrected"] == st["dwc_detected"] == 0 and st["syncs"] == (n if nc == 3 else 0)
    for bt in (False, True):
        _, st = both(rt, oracle, t, nc, A, B, plan_kw=dict(seed=K, p=0.3), bt=bt)
        assert st["injected"] > n // 5
    both(rt, oracle, t, nc, A, B, flags=3 | cb.F_MAJORITY_VOTER, plan_kw=dict(seed=K + 1, p=0.3))
    rng = np.random.default_rng(K + nc)
    tab = np.zeros(n, dtype=np.uint32)
    for u in rng.choice(n, size=300, replace=False):
        site = 0 if rng.random() < 0.8 else 1                      # site 1 does not exist: ignored
        tab[u] = oracle.fault_entry(int(rng.integers(0, 4)), site, int(rng.integers(0, 32)))   # replica >= NC: ignored
    base = 2 ** 32 - n // 2                                        # the global units cross 2^32
    both(rt, oracle, t, nc, A, B, flags=1, plan_kw=dict(seed=K + 2, threshold=1 << 30), unit_base=base)
    status = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    g, gs = gpu(rt, t, nc, A, B, table=tab, unit_base=base, status=status)
    o, os_ = cpu(oracle, t, nc, A, B, table=tab, unit_base=base)
    assert (g == o).all() and {k: gs[k] for k in STAT_KEYS} == {k: os_[k] for k in STAT_KEYS} and gs["injected"] > 0
    s = status.cpu().numpy()
    assert set(np.unique(s)) <= {0, 1}
    assert int(s.sum()) == (gs["errors_corrected"] if nc == 3 else gs["dwc_detected"] if nc == 2 else 0)


RUNS = [({"COAST_GEMM_PAIR": p}, nc) for nc in (1, 2, 3) for p in ("0", "1")] + [
    ({"COAST_GEMM_TAIL_SPLIT": "0"}, 1), ({"COAST_GEMM_TAIL_SPLIT": "0", "COAST_GEMM_PAIR": "0"}, 1),
    ({"COAST_GEMM_GROUP_M": "3"}, 1), ({"COAST_GEMM_GROUP_M": "3"}, 3), ({"COAST_GEMM_L2_HINTS": "0"}, 3)]


@pytest.mark.parametrize("t,M,N,K", per_type({Bf16: [(512, 768, 320), (256, 384, 64), (384, 256, 2048)],
                                              Fp8: [(512, 768, 384), (256, 384, 128), (384, 256, 2048)]}))
def test_general_operands_every_variant_and_layout_same_bits_and_within_bound(rt, t, M, N, K, monkeypatch):
    """uniform(-1, 1) operands: every variant, replica count and B layout adds in the same order and gives the same bits, and
    the float64 reference is held to the type's bound"""
    A, B = t.uniform_operands(M, N, K, seed=K)
    ref = t.value(A).astype(np.float64) @ t.value(B).astype(np.float64)
    bound = t.bound(A, B)
    first = None
    for e, nc in RUNS:
        env(monkeypatch, **e)
        for bt in (False, True):
            g, st = gpu(rt, t, nc, A, B, bt=bt)
            assert st["errors_corrected"] == 0 and st["dwc_detected"] == 0, (e, nc, bt)
            if first is None:
                first = g
                err = np.abs(g.view(np.float32).reshape(M, N).astype(np.float64) - ref)
                assert (err <= bound).all(), err.max()
            assert (g == first).all(), (e, nc, bt)


def position_b(t, K, N):
    """B[k][n] that tells its position apart from its neighbours', in every column box and every k group, in t's values"""
    k_idx, n_idx = np.arange(K)[:, None], np.arange(N)[None, :]
    if t is Bf16:                                                  # exact in bfloat16 (8 significant bits)
        return ((k_idx % 16) * 8 + (n_idx % 8) - 64 + ((k_idx // 16 + n_idx // 8) % 3 - 1) * 0.5).astype(np.float32)
    return (((k_idx % 8) + 1) * np.where((n_idx // 8 + k_idx // 8) % 2, 1.0, -1.0) * 2.0 ** ((n_idx % 8) - 4)).astype(np.float32)


@pytest.mark.parametrize("nc", [1, 3])
@pytest.mark.parametrize("t,M,N,K", per_type({Bf16: [(128, 256, 64), (256, 128, 192), (128, 384, 128), (384, 128, 1024)],
                                              Fp8: [(128, 256, 128), (256, 128, 384), (128, 384, 256), (384, 128, 1024)]}))
def test_b_entries_that_encode_their_position(rt, t, nc, M, N, K, monkeypatch):
    """position_b with N != K and one-hot rows of A: C[i] is row k_i of B, so a transposed, mis-strided or mis-swizzled B or
    B^T shows at once"""
    env(monkeypatch, COAST_GEMM_PAIR="0")
    Bv = position_b(t, K, N)
    hot = (np.arange(M) * 7 + 3) % K
    Av = np.zeros((M, K), dtype=np.float32)
    Av[np.arange(M), hot] = 1.0
    for bt in (False, True):
        g, _ = gpu(rt, t, nc, t.bits(Av), t.bits(Bv), bt=bt)
        assert (g.view(np.float32).reshape(M, N) == Bv[hot]).all(), bt


@pytest.mark.parametrize("t,M,N,K,amax", per_type({Bf16: [(4096, 4096, 4096, 8), (2560, 2048, 256, 8), (2432, 2048, 320, 8)],
                                                   Fp8: [(4096, 4096, 2048, 1), (2560, 2048, 256, 2), (2432, 2048, 512, 2)]}))
def test_multi_wave_every_variant_equals_fp64(rt, t, M, N, K, amax, monkeypatch):
    """several tiles per persistent CTA (the ring phase carries from tile to tile); 2560 / 2432 rows leave a short last round
    that the unprotected kernels split into half tiles.  Every run, with B and with B^T, equals the float64 matmul on the device."""
    import torch
    A, B = t.int_operands(M, N, K, seed=7, amax=amax)
    dA, dB, dBt = dev(t, A), dev(t, B), dev(t, transposed(B, K))
    ref = dA.float().double() @ dB.float().double()
    for e, nc in RUNS:
        env(monkeypatch, **e)
        for aux, mode in ((dB, 0), (dBt, MM_BT)):
            out = torch.full((M * N,), float("nan"), dtype=torch.float32, device="cuda")
            _, st = rt.run(t.kernel, nc, dA, M * N, M=M, N=N, K=K, aux=aux, flags=3, out=out, mode=mode)
            assert st.errors_corrected == 0 and st.dwc_detected == 0, (e, nc)
            assert torch.equal(out.view(M, N).to(torch.float64), ref), (e, nc, mode)


def test_integer_operands_equal_torch_scaled_mm(rt):
    """unprotected torch._scaled_mm (scales 1.0, fp32 out, B^T layout) with fast accumulation on and off: the same bits"""
    import torch
    import coast_b200 as cb
    M, N, K = 1024, 768, 2048
    A, B = Fp8.int_operands(M, N, K, seed=31)
    dA, dBt = dev(Fp8, A), dev(Fp8, transposed(B, K))
    one = torch.ones((), device="cuda")
    for nc in (1, 3):
        out, _ = rt.run(cb.K_GEMM_FP8, nc, dA, M * N, M=M, N=N, K=K, aux=dBt, mode=MM_BT, flags=3)
        mine = out.view(torch.float32).view(M, N)
        for fast in (True, False):
            ref = torch._scaled_mm(dA, dBt.t(), scale_a=one, scale_b=one, out_dtype=torch.float32, use_fast_accum=fast)
            assert torch.equal(mine, ref), (nc, fast)


def test_accumulator_keeps_the_exact_domain(rt):
    """one product of 2^16 and K - 1 products of 2^(16 - d) per element, against the exact sum: the accumulator keeps every
    small product at d <= 11 (the exact domain's ratio of largest partial sum to smallest product) for K = 128 (one k-block) up to
    4096.  The width it does keep is recorded in DESIGN.md §6 (tools/bench_gemm_fp8.py --numerics)."""
    import torch
    import coast_b200 as cb
    M = N = 128
    ea = 8 - (np.arange(M) % 18)
    eb = np.where(np.arange(N) % 2 == 0, 8, 0)
    ratio = 16 - ea[:, None] - eb[None, :]
    small = 2.0 ** (ea[:, None] + eb[None, :])
    for K in (128, 1024, 4096):
        Av = np.empty((M, K), dtype=np.float32)
        Btv = np.empty((N, K), dtype=np.float32)
        Av[:, 0], Btv[:, 0] = 256, 256
        Av[:, 1:], Btv[:, 1:] = (2.0 ** ea)[:, None], (2.0 ** eb)[:, None]
        out, _ = rt.run(cb.K_GEMM_FP8, 1, dev(Fp8, Fp8.bits(Av)), M * N, M=M, N=N, K=K, aux=dev(Fp8, Fp8.bits(Btv)), mode=MM_BT,
                        flags=3)
        c = out.view(torch.float32).cpu().numpy().reshape(M, N).astype(np.float64)
        exact = 65536.0 + (K - 1) * small
        assert (c[ratio <= 11] == exact[ratio <= 11]).all(), K
        assert (c[ratio <= 13] == exact[ratio <= 13]).all() and (c[ratio >= 14] == 65536.0).all(), K   # measured: 14 bits
        assert (c <= exact).all() and (c >= 65536.0).all(), K     # what is lost is lost toward the large product


# ------------------------------------------------------------------------------------------ batched and grouped launches
@pytest.mark.parametrize("bt", [False, True])
@pytest.mark.parametrize("t,nc,M,N,K,batch,e", per_type(
    {Bf16: [(1, 128, 256, 128, 5, {"COAST_GEMM_PAIR": "0"}), (1, 256, 256, 64, 3, {}), (1, 128, 128, 192, 4, {}),
            (2, 256, 128, 64, 3, {}), (3, 128, 128, 128, 7, {})],
     Fp8: [(1, 128, 256, 128, 5, {"COAST_GEMM_PAIR": "0"}), (1, 256, 256, 128, 3, {}), (1, 128, 128, 384, 4, {}),
           (2, 256, 128, 128, 3, {}), (3, 128, 128, 256, 7, {})]}, ids=lambda c: "-".join(map(str, c[:5]))))
def test_batched_equals_single_launches(rt, t, nc, M, N, K, batch, e, bt, monkeypatch):
    import coast_b200 as cb
    env(monkeypatch, **e)
    A, B = t.stacked_operands(batch * M, N, K, batch, seed=batch)  # batch stacked A (M x K each), batch stacked B (K x N each)
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=9, p=0.2)
    base = 2 ** 32 - M * N
    g, st = gpu(rt, t, nc, A, B, M=M, mode=MM_BATCHED, plan=plan, unit_base=base, bt=bt)
    want, tot = [], no_stats()
    for b in range(batch):
        o, s = gpu(rt, t, nc, A[b * M:(b + 1) * M], B[b * K:(b + 1) * K], plan=plan, unit_base=base + b * M * N)
        want.append(o)
        add_stats(tot, s)
    assert (g == np.concatenate(want)).all() and st == tot
    if nc == 3:                                                    # TMR votes every fault out
        clean = t.value(A).astype(np.float64).reshape(batch, M, K) @ t.value(B).astype(np.float64).reshape(batch, K, N)
        assert (g.view(np.float32).astype(np.float64) == clean.ravel()).all()


@pytest.mark.parametrize("bt", [False, True])
@pytest.mark.parametrize("nc", [1, 2, 3])
@pytest.mark.parametrize("t,N,K,ro", per_type({Bf16: [(128, 64, RO), (384, 192, RO)], Fp8: [(256, 256, zipf_offsets(16, 1500, start=3))]},
                                              ids=lambda c: f"{c[0]}-{c[1]}-G{len(c[2]) - 1}"))
def test_grouped_equals_single_launches_and_keeps_rows_outside_the_table(rt, oracle, t, N, K, ro, nc, bt):
    import torch
    import coast_b200 as cb
    assert 0 in np.diff(ro) and max(np.diff(ro)) > 128            # empty products, and one product taller than a tile
    G, R = len(ro) - 1, ro[-1] - ro[0]
    rows_alloc = ro[-1] + 40
    A, B = t.stacked_operands(rows_alloc, N, K, G, seed=nc)
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=5, p=0.2)
    base = 2 ** 32 - 1000
    out = torch.full((rows_alloc * N,), POISON, dtype=torch.int32, device="cuda").view(torch.float32)
    d_ro = torch.tensor(ro, dtype=torch.int64, device="cuda")
    g, st = gpu(rt, t, nc, A, B, M=G, n=R * N, mode=MM_GROUPED, rows=d_ro, plan=plan, unit_base=base, out=out, bt=bt)
    g = g.reshape(rows_alloc, N)
    assert (g[:ro[0]] == POISON).all() and (g[ro[-1]:] == POISON).all()
    tot = no_stats()
    for i in range(G):
        m = ro[i + 1] - ro[i]
        if not m:
            continue
        Ai, Bi, ub = A[ro[i]:ro[i + 1]], B[i * K:(i + 1) * K], base + (ro[i] - ro[0]) * N
        o, s = cpu(oracle, t, nc, Ai, Bi, plan_kw=dict(seed=5, p=0.2), unit_base=ub)      # the oracle takes any row count
        assert (g[ro[i]:ro[i + 1]].ravel() == o).all(), i
        add_stats(tot, s)
        if m % 128 == 0:                                           # and the device's own single launch where its shape rule allows
            o1, _ = gpu(rt, t, nc, Ai, Bi, plan=plan, unit_base=ub)
            assert (o1 == o).all(), i
    assert st == tot and st["injected"] > 0


@pytest.mark.parametrize("t", [Bf16, Fp8], ids=lambda t: t.name)
def test_equal_groups_equal_the_batched_launch(rt, t):
    import torch
    M, N, K, batch = 128, 256, 128, 6
    A, B = t.stacked_operands(batch * M, N, K, batch, seed=77)
    for nc in (1, 3):
        gb, sb = gpu(rt, t, nc, A, B, M=M, mode=MM_BATCHED, unit_base=11)
        ro = torch.arange(0, (batch + 1) * M, M, dtype=torch.int64, device="cuda")
        gg, sg = gpu(rt, t, nc, A, B, M=batch, mode=MM_GROUPED, rows=ro, unit_base=11)
        assert (gb == gg).all() and sb == sg


@pytest.mark.parametrize("t,N,K,ro", per_type({Bf16: [(128, 128, RO)], Fp8: [(128, 256, zipf_offsets(12, 900, start=3, seed=5))]},
                                              ids=lambda c: f"{c[0]}-{c[1]}"))
def test_sharding_over_products(rt, t, N, K, ro):
    """whole products [g_lo, g_hi) per shard: same d_in / d_out, d_aux + g_lo K N, d_rows + g_lo, unit_base by rows"""
    import torch
    import coast_b200 as cb
    from coast_b200.shard import shard_groups
    G, R = len(ro) - 1, ro[-1] - ro[0]
    A, B = t.stacked_operands(ro[-1], N, K, G, seed=13)
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=2, p=0.1)
    d_ro = torch.tensor(ro, dtype=torch.int64, device="cuda")
    whole, sw = gpu(rt, t, 3, A, B, M=G, n=R * N, mode=MM_GROUPED, rows=d_ro, plan=plan, unit_base=50,
                    out=torch.zeros(ro[-1] * N, dtype=torch.float32, device="cuda"))
    for bt in (False, True):
        out = torch.zeros(ro[-1] * N, dtype=torch.float32, device="cuda")
        dA, dB = dev(t, A), dev(t, transposed(B, K) if bt else B)
        tot = no_stats()
        for r in range(3):
            lo, hi = shard_groups(ro, r, 3)
            if hi == lo or ro[hi] == ro[lo]:
                continue
            _, s = rt.run(t.kernel, 3, dA, (ro[hi] - ro[lo]) * N, M=hi - lo, N=N, K=K, aux=dB.view(-1)[lo * K * N:], flags=3,
                          mode=MM_GROUPED | (MM_BT if bt else 0), rows=d_ro[lo:], plan=plan, unit_base=50 + (ro[lo] - ro[0]) * N, out=out)
            add_stats(tot, s.as_dict())
        assert (out.cpu().numpy().view(np.uint32) == whole).all() and tot == sw, bt


@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("t,K,ro", per_type({Bf16: [(128, RO)], Fp8: [(256, zipf_offsets(10, 700, start=3, seed=9))]},
                                            ids=lambda c: str(c[0])))
def test_host_call_row_blocks_products_and_groups(rt, t, K, ro, pinned, monkeypatch):
    """coast_run_host with t's A and B and 4-byte C: row blocks (B once, or B^T once), whole products per chunk, groups per
    chunk, each cut into many chunks, against the device launch"""
    import torch
    import coast_b200 as cb
    env(monkeypatch, COAST_HOST_CHUNK_BYTES=str(300000))

    def host(x):
        x = t.tensor(x) if isinstance(x, np.ndarray) else x
        return x.pin_memory() if pinned else x
    # row blocks
    M, N = 1024, 128
    A, B = t.int_operands(M, N, K, seed=3)
    want, _ = gpu(rt, t, 3, A, B)
    h_out = host(torch.full((M * N,), float("nan"), dtype=torch.float32))
    st = rt.run_host(t.kernel, 3, host(A), h_out, M * N, M=M, N=N, K=K, h_aux=host(B), flags=3)
    assert rt.last_host_path == "row-blocks" and (h_out.numpy().view(np.uint32) == want).all() and st.syncs == M * N
    h_out = host(torch.full((M * N,), float("nan"), dtype=torch.float32))
    rt.run_host(t.kernel, 3, host(A), h_out, M * N, M=M, N=N, K=K, h_aux=host(transposed(B, K)), flags=3, mode=MM_BT)
    assert (h_out.numpy().view(np.uint32) == want).all()
    # whole products
    M, batch = 128, 9
    A, B = t.stacked_operands(batch * M, N, K, batch, seed=4)
    want, _ = gpu(rt, t, 2, A, B, M=M, mode=MM_BATCHED)
    h_out = host(torch.full((batch * M * N,), float("nan"), dtype=torch.float32))
    rt.run_host(t.kernel, 2, host(A), h_out, batch * M * N, M=M, N=N, K=K, h_aux=host(B), flags=3, mode=MM_BATCHED)
    assert (h_out.numpy().view(np.uint32) == want).all()
    # groups
    G, R = len(ro) - 1, ro[-1] - ro[0]
    A, B = t.stacked_operands(ro[-1], N, K, G, seed=5)
    h_ro = torch.tensor(ro, dtype=torch.int64)
    want, sw = gpu(rt, t, 3, A, B, M=G, n=R * N, mode=MM_GROUPED, rows=h_ro.cuda(), unit_base=9,
                   out=torch.zeros(ro[-1] * N, dtype=torch.float32, device="cuda"))
    h_out = host(torch.zeros(ro[-1] * N, dtype=torch.float32))
    st = rt.run_host(t.kernel, 3, host(A), h_out, R * N, M=G, N=N, K=K, h_aux=host(B), flags=3, mode=MM_GROUPED, h_rows=h_ro,
                     unit_base=9)
    assert rt.last_host_path == "groups" and (h_out.numpy().view(np.uint32) == want).all() and st.as_dict() == sw


# ------------------------------------------------------------------------------------------ operand edges through the fp32 vote
def test_subnormal_operands_are_exact(rt, oracle):
    """subnormal E4M3 (m 2^-9) against integers in [-1, 1]: the sums are multiples of 2^-9 below 2^11 of them, so exact"""
    M, N, K = 256, 256, 256
    rng = np.random.default_rng(23)
    A = (rng.integers(1, 8, (M, K)) | np.where(rng.random((M, K)) < 0.5, 0x80, 0)).astype(np.uint8)
    _, B = Fp8.int_operands(M, N, K, seed=24)
    for nc in (1, 3):
        g, _ = both(rt, oracle, Fp8, nc, A, B)
        assert (g.view(np.float32).reshape(M, N).astype(np.float64) == Fp8.value(A).astype(np.float64) @ Fp8.value(B).astype(np.float64)).all()


@pytest.mark.parametrize("t,K", per_type({Bf16: [(64,)], Fp8: [(128,)]}))
def test_vote_is_ordered_equal_on_signed_zeros(rt, oracle, t, K):
    """a row of negative-zero operands in A against B >= 0 gives a +0.0 row of C; a flip of bit 31 there makes -0.0, equal to
    +0.0 under `fcmp oeq`: not counted, and r0's value is stored.  A flip of bit 0 makes a denormal: counted."""
    M, N = 256, 256
    A, B = t.int_operands(M, N, K, seed=3)
    B = t.bits(np.abs(t.value(B)))
    z = 77
    A[z] = t.neg_zero
    tab = np.zeros(M * N, dtype=np.uint32)
    signs = [(z * N + 7 * c, c % 3) for c in range(30)]
    for u, r in signs:
        tab[u] = oracle.fault_entry(r, 0, 31)
    denormals = [(z * N + 250, 1), (z * N + 251, 0), (z * N + 252, 2)]
    for u, r in denormals:
        tab[u] = oracle.fault_entry(r, 0, 0)
    clean, _ = gpu(rt, t, 1, A, B)
    assert (clean.reshape(M, N)[z] == 0).all()                     # -0 x b summed from +0: +0.0
    for nc in (2, 3):
        g, st = both(rt, oracle, t, nc, A, B, table=tab)
        row = g.reshape(M, N)[z]
        counted = [u for u, r in denormals if r < nc]
        assert st["injected"] == sum(r < nc for _, r in signs + denormals)
        assert (st["errors_corrected"] if nc == 3 else st["dwc_detected"]) == len(counted)
        for u, r in signs:
            assert row[u - z * N] == (0x80000000 if r == 0 else 0), (nc, u, r)


@pytest.mark.parametrize("nc", [1, 2, 3])
@pytest.mark.parametrize("t", [Bf16, Fp8], ids=lambda t: t.name)
def test_nan_operand_disagrees_in_every_element_of_its_row(rt, oracle, t, nc):
    """a NaN operand (bfloat16 0x7FC0, E4M3 0x7F) in one row of A makes that C row NaN in every replica; NaN != NaN under
    `fcmp oeq`, so TMR -countErrors counts N disagreements and DWC N detections, as the oracle does.  The payload is not pinned."""
    M, N, K = 256, 128, 128
    A, B = t.int_operands(M, N, K, seed=19)
    z = 130
    A[z, 9] = t.nan
    o, os_ = cpu(oracle, t, nc, A, B)
    g, gs = gpu(rt, t, nc, A, B)
    nan = np.isnan(o.view(np.float32)).reshape(M, N)
    assert nan[z].all() and nan.sum() == N
    assert (np.isnan(g.view(np.float32)).reshape(M, N) == nan).all()
    assert (g.reshape(M, N)[~nan] == o.reshape(M, N)[~nan]).all()
    assert {k: gs[k] for k in STAT_KEYS} == {k: os_[k] for k in STAT_KEYS}
    if nc > 1:
        assert (gs["errors_corrected"] if nc == 3 else gs["dwc_detected"]) == N and gs["first_fault_unit"] == z * N
