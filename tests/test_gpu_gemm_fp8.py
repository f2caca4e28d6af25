"""GPU (H100): the FP8 GEMM (COAST_K_GEMM_FP8): E4M3 A and B, wgmma m64n128k32 into the tensor core's accumulator, fp32 C,
B^T read K-major (from the byte-transposing pre-pass, or the caller's with COAST_MM_B_TRANSPOSED), NC register accumulator
replicas and the voting epilogue of GEMM_TF32.

Exact where the accumulator's width cannot matter: integer-valued operands whose sum_k |a_ik b_kj| is at most 2^11 (gemm_fp8_ref.
EXACT_SUM) make every partial sum a small integer, so outputs equal the CPU reference (tests/gemm_fp8_ref.py), a float64 matmul
and torch._scaled_mm bit for bit.  The accumulator's width is measured here and must cover that domain.  General operands are
held to a bound relative to sum_k |a_ik b_kj| and to bit-equality between every kernel variant, replica count and B layout.
numpy has no FP8: operands are uint8 bit patterns on the host."""
import numpy as np
import pytest

import gemm_fp8_ref as ref8
from gemm_fp8_ref import bits, value

pytestmark = pytest.mark.gpu

KNOBS = ("COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT", "COAST_HOST_CHUNK_BYTES", "COAST_HOST_PATH")
STAT_KEYS = ("errors_corrected", "dwc_detected", "syncs", "injected", "first_fault_unit")
MM_BATCHED, MM_GROUPED, MM_BT = 0x20000, 0x40000, 0x80000
# max |C - C64| / sum_k |a_ik b_kj| on uniform(-1, 1) E4M3 operands: measured at most 3.7e-4 (2^-11.4) on an H100 up to K = 8192
# (DESIGN.md §6); the bound leaves a factor of 2.6
GENERAL_BOUND = 2.0 ** -10


def int_operands(M, N, K, seed, amax=1):
    return ref8.int_operands(np.random.default_rng(seed), M, N, K, amax)


def stacked_operands(rows, N, K, P, seed):
    """rows x K of A and P stacked K x N matrices B, integers in [-1, 1]: each product stays in the exact domain"""
    rng = np.random.default_rng(seed)
    A, _ = ref8.int_operands(rng, rows, N, K, 1)
    return A, np.concatenate([ref8.int_operands(rng, 1, N, K, 1)[1] for _ in range(P)])


def uniform_operands(M, N, K, seed):
    """uniform(-1, 1) rounded to E4M3 by torch (round to nearest even)"""
    import torch
    g = torch.Generator().manual_seed(seed)

    def one(r, c):
        return (torch.rand(r, c, generator=g) * 2 - 1).to(torch.float8_e4m3fn).view(torch.uint8).numpy().copy()
    return one(M, K), one(K, N)


def dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda().view(torch.float8_e4m3fn)


def transposed(B, K):
    """the products' B (P K x N, stacked) as their B^T (P N x K, stacked)"""
    N = B.shape[1]
    return np.ascontiguousarray(B.reshape(-1, K, N).transpose(0, 2, 1).reshape(-1, K))


def env(monkeypatch, **kv):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in kv.items():
        monkeypatch.setenv(k, v)


def gpu(rt, nc, A, B, *, flags=3, plan=None, table=None, unit_base=0, status=None, mode=0, M=None, n=None, rows=None, out=None, bt=False):
    """A: (rows x K) uint8, B: (P K x N) uint8 -> (C bits as uint32, flat; stats dict); bt: launch with B^T"""
    import torch
    import coast_b200 as cb
    K, N = A.shape[1], B.shape[1]
    M = A.shape[0] if M is None else M
    n = A.shape[0] * N if n is None else n
    if table is not None:
        plan = cb.FaultPlan(mode=cb.PLAN_TABLE, table=torch.from_numpy(table.view(np.int32).copy()).cuda())
    if out is None:
        out = torch.full((A.shape[0] * N,), float("nan"), dtype=torch.float32, device="cuda")    # poison: every element is written
    aux = dev(transposed(B, K)) if bt else dev(B)
    _, st = rt.run(cb.K_GEMM_FP8, nc, dev(A), n, M=M, N=N, K=K, aux=aux, flags=flags, plan=plan, unit_base=unit_base,
                   status=status, mode=mode | (MM_BT if bt else 0), rows=rows, out=out)
    return out.cpu().numpy().view(np.uint32), st.as_dict()


def cpu(oracle, nc, A, B, *, flags=3, plan_kw=None, table=None, unit_base=0):
    plan = None
    if table is not None:
        plan = oracle.make_plan(oracle.PLAN_TABLE, table=table)
    elif plan_kw:
        plan = oracle.make_plan(oracle.PLAN_BERNOULLI, **plan_kw)
    return ref8.run(oracle, nc, A, B, flags=flags, plan=plan, unit_base=unit_base, threads=8)


def both(rt, oracle, nc, A, B, *, flags=3, plan_kw=None, table=None, unit_base=0, bt=False):
    import coast_b200 as cb
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, **plan_kw) if plan_kw else None
    g, gs = gpu(rt, nc, A, B, flags=flags, plan=plan, table=table, unit_base=unit_base, bt=bt)
    o, os_ = cpu(oracle, nc, A, B, flags=flags, plan_kw=plan_kw, table=table, unit_base=unit_base)
    assert (g == o).all(), (nc, flags, np.flatnonzero(g != o)[:8])
    assert {k: gs[k] for k in STAT_KEYS} == {k: os_[k] for k in STAT_KEYS}
    return g, gs


# (id, environment, NC, M, N, the kernel the launcher must pick)
VARIANTS = [
    ("narrow_nc1", {}, 1, 256, 384, "xmr_gemm_fp8n_inj0_nc1"),                   # N % 256 != 0: 128 x 128 tiles
    ("wide_nc1", {"COAST_GEMM_PAIR": "0"}, 1, 256, 256, "xmr_gemm_fp8_inj0_nc1"),   # 128 x 256 tiles: two B^T boxes per stage
    ("pair_nc1", {}, 1, 256, 256, "xmr_gemm_fp8p_inj0_nc1"),
    ("pair_nc2", {}, 2, 256, 128, "xmr_gemm_fp8p_inj0_nc2"),                     # one 64-row B^T box per CTA of the pair
    ("single_nc2", {"COAST_GEMM_PAIR": "0"}, 2, 256, 128, "xmr_gemm_fp8_inj0_nc2"),
    ("single_nc3", {}, 3, 256, 128, "xmr_gemm_fp8_inj0_nc3"),
    ("pair_nc3", {"COAST_GEMM_PAIR": "1"}, 3, 256, 256, "xmr_gemm_fp8p_inj0_nc3"),
]


@pytest.mark.parametrize("K", [128, 768, 896, 2048])     # one k-block; one 6-stage ring exactly; one wrap; many wraps
@pytest.mark.parametrize("variant", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_integer_operands_bit_exact_with_the_oracle(rt, oracle, variant, K, monkeypatch, capfd):
    import torch
    import coast_b200 as cb
    _, e, nc, M, N, kname = variant
    env(monkeypatch, **e)
    A, B = int_operands(M, N, K, seed=K + 10 * nc)
    n = M * N
    capfd.readouterr()
    gpu(rt, nc, A, B, flags=cb.F_VERBOSE)
    assert f"{kname} " in capfd.readouterr().err
    g, st = both(rt, oracle, nc, A, B)
    assert (g.view(np.float32).reshape(M, N).astype(np.float64) == value(A).astype(np.float64) @ value(B).astype(np.float64)).all()
    assert st["errors_corrected"] == st["dwc_detected"] == 0 and st["syncs"] == (n if nc == 3 else 0)
    _, st = both(rt, oracle, nc, A, B, plan_kw=dict(seed=K, p=0.3), bt=True)
    assert st["injected"] > n // 5
    both(rt, oracle, nc, A, B, flags=3 | cb.F_MAJORITY_VOTER, plan_kw=dict(seed=K + 1, p=0.3))
    rng = np.random.default_rng(K + nc)
    tab = np.zeros(n, dtype=np.uint32)
    for u in rng.choice(n, size=300, replace=False):
        site = 0 if rng.random() < 0.8 else 1                      # site 1 does not exist: ignored
        tab[u] = oracle.fault_entry(int(rng.integers(0, 4)), site, int(rng.integers(0, 32)))   # replica >= NC: ignored
    base = 2 ** 32 - n // 2                                        # the global units cross 2^32
    status = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    g, gs = gpu(rt, nc, A, B, table=tab, unit_base=base, status=status)
    o, os_ = cpu(oracle, nc, A, B, table=tab, unit_base=base)
    assert (g == o).all() and {k: gs[k] for k in STAT_KEYS} == {k: os_[k] for k in STAT_KEYS} and gs["injected"] > 0
    s = status.cpu().numpy()
    assert set(np.unique(s)) <= {0, 1}
    assert int(s.sum()) == (gs["errors_corrected"] if nc == 3 else gs["dwc_detected"] if nc == 2 else 0)


RUNS = [({"COAST_GEMM_PAIR": p}, nc) for nc in (1, 2, 3) for p in ("0", "1")] + [
    ({"COAST_GEMM_TAIL_SPLIT": "0"}, 1), ({"COAST_GEMM_TAIL_SPLIT": "0", "COAST_GEMM_PAIR": "0"}, 1),
    ({"COAST_GEMM_GROUP_M": "3"}, 1), ({"COAST_GEMM_GROUP_M": "3"}, 3), ({"COAST_GEMM_L2_HINTS": "0"}, 3)]


@pytest.mark.parametrize("M,N,K", [(512, 768, 384), (256, 384, 128), (384, 256, 2048)])
def test_general_operands_every_variant_and_layout_same_bits_and_within_bound(rt, M, N, K, monkeypatch):
    """uniform(-1, 1) E4M3 operands: every variant, replica count and B layout runs the same m64n128k32 steps in the same order
    and gives the same bits, and the float64 reference is held to |C - C64| <= GENERAL_BOUND * sum_k |a_ik b_kj|"""
    A, B = uniform_operands(M, N, K, seed=K)
    ref = value(A).astype(np.float64) @ value(B).astype(np.float64)
    mag = np.abs(value(A)).astype(np.float64) @ np.abs(value(B)).astype(np.float64)
    first = None
    for e, nc in RUNS:
        env(monkeypatch, **e)
        for bt in (False, True):
            g, st = gpu(rt, nc, A, B, bt=bt)
            assert st["errors_corrected"] == 0 and st["dwc_detected"] == 0, (e, nc, bt)
            if first is None:
                first = g
                ratio = (np.abs(g.view(np.float32).reshape(M, N).astype(np.float64) - ref) / mag).max()
                assert ratio <= GENERAL_BOUND, ratio
            assert (g == first).all(), (e, nc, bt)


@pytest.mark.parametrize("nc", [1, 3])
@pytest.mark.parametrize("M,N,K", [(128, 256, 128), (256, 128, 384), (128, 384, 256), (384, 128, 1024)])
def test_b_entries_that_encode_their_position(rt, nc, M, N, K, monkeypatch):
    """B[k][n] = ((k % 8) + 1) * (1 if (n // 8 + k // 8) % 2 else -1) * 2^((n % 8) - 4), all E4M3 values, with N != K and
    one-hot rows of A: C[i] is row k_i of B, so a transposed, mis-strided or mis-swizzled B^T shows at once"""
    env(monkeypatch, COAST_GEMM_PAIR="0")
    k_idx, n_idx = np.arange(K)[:, None], np.arange(N)[None, :]
    Bv = ((k_idx % 8) + 1) * np.where((n_idx // 8 + k_idx // 8) % 2, 1.0, -1.0) * 2.0 ** ((n_idx % 8) - 4)
    Bv = Bv.astype(np.float32)
    hot = (np.arange(M) * 7 + 3) % K
    Av = np.zeros((M, K), dtype=np.float32)
    Av[np.arange(M), hot] = 1.0
    for bt in (False, True):
        g, _ = gpu(rt, nc, bits(Av), bits(Bv), bt=bt)
        assert (g.view(np.float32).reshape(M, N) == Bv[hot]).all(), bt


@pytest.mark.parametrize("M,N,K,amax", [(4096, 4096, 2048, 1), (2560, 2048, 256, 2), (2432, 2048, 512, 2)])
def test_multi_wave_every_variant_equals_fp64(rt, M, N, K, amax, monkeypatch):
    """several tiles per persistent CTA (the ring phase carries from tile to tile: 4096 x 4096 is 1024 tiles, 7.8 per CTA for
    TMR); 2560 / 2432 rows leave a short last round that the unprotected kernels split into half tiles.  Every run equals the
    float64 matmul on the device."""
    import torch
    import coast_b200 as cb
    A, B = int_operands(M, N, K, seed=7, amax=amax)
    dA, dB, dBt = dev(A), dev(B), dev(transposed(B, K))
    ref = dA.float().double() @ dB.float().double()
    for e, nc in RUNS:
        env(monkeypatch, **e)
        for aux, mode in ((dB, 0), (dBt, MM_BT)):
            out = torch.full((M * N,), float("nan"), dtype=torch.float32, device="cuda")
            _, st = rt.run(cb.K_GEMM_FP8, nc, dA, M * N, M=M, N=N, K=K, aux=aux, flags=3, out=out, mode=mode)
            assert st.errors_corrected == 0 and st.dwc_detected == 0, (e, nc)
            assert torch.equal(out.view(M, N).to(torch.float64), ref), (e, nc, mode)


def test_integer_operands_equal_torch_scaled_mm(rt):
    """unprotected torch._scaled_mm (scales 1.0, fp32 out, B^T layout) with fast accumulation on and off: the same bits"""
    import torch
    import coast_b200 as cb
    M, N, K = 1024, 768, 2048
    A, B = int_operands(M, N, K, seed=31)
    dA, dBt = dev(A), dev(transposed(B, K))
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
        out, _ = rt.run(cb.K_GEMM_FP8, 1, dev(bits(Av)), M * N, M=M, N=N, K=K, aux=dev(bits(Btv)), mode=MM_BT, flags=3)
        c = out.view(torch.float32).cpu().numpy().reshape(M, N).astype(np.float64)
        exact = 65536.0 + (K - 1) * small
        assert (c[ratio <= 11] == exact[ratio <= 11]).all(), K
        assert (c[ratio <= 13] == exact[ratio <= 13]).all() and (c[ratio >= 14] == 65536.0).all(), K   # measured: 14 bits
        assert (c <= exact).all() and (c >= 65536.0).all(), K     # what is lost is lost toward the large product


# ------------------------------------------------------------------------------------------ batched and grouped launches
BATCH_CASES = [(1, 128, 256, 128, 5, {"COAST_GEMM_PAIR": "0"}), (1, 256, 256, 128, 3, {}), (1, 128, 128, 384, 4, {}),
               (2, 256, 128, 128, 3, {}), (3, 128, 128, 256, 7, {})]


@pytest.mark.parametrize("bt", [False, True])
@pytest.mark.parametrize("nc,M,N,K,batch,e", BATCH_CASES)
def test_batched_equals_single_launches(rt, nc, M, N, K, batch, e, bt, monkeypatch):
    import coast_b200 as cb
    env(monkeypatch, **e)
    A, B = stacked_operands(batch * M, N, K, batch, seed=batch)    # batch stacked A (M x K each), batch stacked B (K x N each)
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=9, p=0.2)
    base = 2 ** 32 - M * N
    g, st = gpu(rt, nc, A, B, M=M, mode=MM_BATCHED, plan=plan, unit_base=base, bt=bt)
    want, tot = [], dict(errors_corrected=0, dwc_detected=0, syncs=0, injected=0, first_fault_unit=2 ** 64 - 1)
    for b in range(batch):
        o, s = gpu(rt, nc, A[b * M:(b + 1) * M], B[b * K:(b + 1) * K], plan=plan, unit_base=base + b * M * N)
        want.append(o)
        for k in STAT_KEYS[:4]:
            tot[k] += s[k]
        tot["first_fault_unit"] = min(tot["first_fault_unit"], s["first_fault_unit"])
    assert (g == np.concatenate(want)).all() and st == tot
    if nc == 3:                                                    # TMR votes every fault out
        clean = value(A).astype(np.float64).reshape(batch, M, K) @ value(B).astype(np.float64).reshape(batch, K, N)
        assert (g.view(np.float32).astype(np.float64) == clean.ravel()).all()


def zipf_offsets(G, R, start, seed=3):
    """a mixture-of-experts routing: Zipf-like expert loads, some experts empty, rows from `start`"""
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, G + 1) ** 1.1
    rng.shuffle(w)
    rows = np.floor(R * w / w.sum()).astype(int)
    rows[rng.choice(G, size=G // 5, replace=False)] = 0
    rows[np.argmax(rows)] += R - rows.sum()
    return [int(start)] + [int(start + x) for x in np.cumsum(rows)]


@pytest.mark.parametrize("bt", [False, True])
@pytest.mark.parametrize("nc", [1, 2, 3])
def test_grouped_moe_equals_single_launches_and_keeps_rows_outside_the_table(rt, oracle, nc, bt):
    import torch
    import coast_b200 as cb
    N, K, G = 256, 256, 16
    RO = zipf_offsets(G, 1500, start=3)
    assert 0 in np.diff(RO) and max(np.diff(RO)) > 128
    R = RO[-1] - RO[0]
    rows_alloc = RO[-1] + 40
    A, B = stacked_operands(rows_alloc, N, K, G, seed=nc)
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=5, p=0.2)
    base = 2 ** 32 - 1000
    POISON = 0x7FC00BAD
    out = torch.full((rows_alloc * N,), POISON, dtype=torch.int32, device="cuda").view(torch.float32)
    ro = torch.tensor(RO, dtype=torch.int64, device="cuda")
    g, st = gpu(rt, nc, A, B, M=G, n=R * N, mode=MM_GROUPED, rows=ro, plan=plan, unit_base=base, out=out, bt=bt)
    g = g.reshape(rows_alloc, N)
    assert (g[:RO[0]] == POISON).all() and (g[RO[-1]:] == POISON).all()
    tot = dict(errors_corrected=0, dwc_detected=0, syncs=0, injected=0, first_fault_unit=2 ** 64 - 1)
    for i in range(G):
        m = RO[i + 1] - RO[i]
        if not m:
            continue
        Ai, Bi, ub = A[RO[i]:RO[i + 1]], B[i * K:(i + 1) * K], base + (RO[i] - RO[0]) * N
        o, s = cpu(oracle, nc, Ai, Bi, plan_kw=dict(seed=5, p=0.2), unit_base=ub)      # the oracle takes any row count
        assert (g[RO[i]:RO[i + 1]].ravel() == o).all(), i
        for k in STAT_KEYS[:4]:
            tot[k] += s[k]
        tot["first_fault_unit"] = min(tot["first_fault_unit"], s["first_fault_unit"])
        if m % 128 == 0:                                           # and the device's own single launch where its shape rule allows
            o1, _ = gpu(rt, nc, Ai, Bi, plan=plan, unit_base=ub)
            assert (o1 == o).all(), i
    assert st == tot and st["injected"] > 0


def test_sharding_over_products(rt):
    """whole products [g_lo, g_hi) per shard: same d_in / d_out, d_aux + g_lo K N, d_rows + g_lo, unit_base by rows"""
    import torch
    import coast_b200 as cb
    from coast_b200.shard import shard_groups
    N, K = 128, 256
    RO = zipf_offsets(12, 900, start=3, seed=5)
    G, R = len(RO) - 1, RO[-1] - RO[0]
    A, B = stacked_operands(RO[-1], N, K, G, seed=13)
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=2, p=0.1)
    ro = torch.tensor(RO, dtype=torch.int64, device="cuda")
    whole, sw = gpu(rt, 3, A, B, M=G, n=R * N, mode=MM_GROUPED, rows=ro, plan=plan, unit_base=50,
                    out=torch.zeros(RO[-1] * N, dtype=torch.float32, device="cuda"))
    for bt in (False, True):
        out = torch.zeros(RO[-1] * N, dtype=torch.float32, device="cuda")
        dA, dB = dev(A), dev(transposed(B, K) if bt else B)
        tot = dict(errors_corrected=0, dwc_detected=0, syncs=0, injected=0, first_fault_unit=2 ** 64 - 1)
        for r in range(3):
            lo, hi = shard_groups(RO, r, 3)
            if hi == lo or RO[hi] == RO[lo]:
                continue
            _, s = rt.run(cb.K_GEMM_FP8, 3, dA, (RO[hi] - RO[lo]) * N, M=hi - lo, N=N, K=K, aux=dB.view(-1)[lo * K * N:], flags=3,
                          mode=MM_GROUPED | (MM_BT if bt else 0), rows=ro[lo:], plan=plan, unit_base=50 + (RO[lo] - RO[0]) * N, out=out)
            s = s.as_dict()
            for k in STAT_KEYS[:4]:
                tot[k] += s[k]
            tot["first_fault_unit"] = min(tot["first_fault_unit"], s["first_fault_unit"])
        assert (out.cpu().numpy().view(np.uint32) == whole).all() and tot == sw, bt


@pytest.mark.parametrize("pinned", [False, True])
def test_host_call_row_blocks_products_and_groups(rt, pinned, monkeypatch):
    """coast_run_host with 1-byte A and B and 4-byte C: row blocks (B once), whole products per chunk, groups per chunk, each
    cut into many chunks, against the device launch"""
    import torch
    import coast_b200 as cb
    env(monkeypatch, COAST_HOST_CHUNK_BYTES=str(300000))

    def host(t):
        return t.pin_memory() if pinned else t

    def h8(x):
        return host(torch.from_numpy(np.ascontiguousarray(x)))
    # row blocks
    M, N, K = 1024, 128, 256
    A, B = int_operands(M, N, K, seed=3)
    want, _ = gpu(rt, 3, A, B)
    h_out = host(torch.full((M * N,), float("nan"), dtype=torch.float32))
    st = rt.run_host(cb.K_GEMM_FP8, 3, h8(A), h_out, M * N, M=M, N=N, K=K, h_aux=h8(B), flags=3)
    assert rt.last_host_path == "row-blocks" and (h_out.numpy().view(np.uint32) == want).all() and st.syncs == M * N
    h_out = host(torch.full((M * N,), float("nan"), dtype=torch.float32))
    rt.run_host(cb.K_GEMM_FP8, 3, h8(A), h_out, M * N, M=M, N=N, K=K, h_aux=h8(transposed(B, K)), flags=3, mode=MM_BT)
    assert (h_out.numpy().view(np.uint32) == want).all()
    # whole products
    M, batch = 128, 9
    A, B = stacked_operands(batch * M, N, K, batch, seed=4)
    want, _ = gpu(rt, 2, A, B, M=M, mode=MM_BATCHED)
    h_out = host(torch.full((batch * M * N,), float("nan"), dtype=torch.float32))
    rt.run_host(cb.K_GEMM_FP8, 2, h8(A), h_out, batch * M * N, M=M, N=N, K=K, h_aux=h8(B), flags=3, mode=MM_BATCHED)
    assert (h_out.numpy().view(np.uint32) == want).all()
    # groups
    RO = zipf_offsets(10, 700, start=3, seed=9)
    G, R = len(RO) - 1, RO[-1] - RO[0]
    A, B = stacked_operands(RO[-1], N, K, G, seed=5)
    ro = torch.tensor(RO, dtype=torch.int64)
    want, sw = gpu(rt, 3, A, B, M=G, n=R * N, mode=MM_GROUPED, rows=ro.cuda(), unit_base=9,
                   out=torch.zeros(RO[-1] * N, dtype=torch.float32, device="cuda"))
    h_out = host(torch.zeros(RO[-1] * N, dtype=torch.float32))
    st = rt.run_host(cb.K_GEMM_FP8, 3, h8(A), h_out, R * N, M=G, N=N, K=K, h_aux=h8(B), flags=3, mode=MM_GROUPED, h_rows=ro,
                     unit_base=9)
    assert rt.last_host_path == "groups" and (h_out.numpy().view(np.uint32) == want).all() and st.as_dict() == sw


# ------------------------------------------------------------------------------------------ E4M3 edges through the vote
def test_subnormal_operands_are_exact(rt, oracle):
    """subnormal E4M3 (m 2^-9) against integers in [-1, 1]: the sums are multiples of 2^-9 below 2^11 of them, so exact"""
    M, N, K = 256, 256, 256
    rng = np.random.default_rng(23)
    A = (rng.integers(1, 8, (M, K)) | np.where(rng.random((M, K)) < 0.5, 0x80, 0)).astype(np.uint8)
    _, B = int_operands(M, N, K, seed=24)
    for nc in (1, 3):
        g, _ = both(rt, oracle, nc, A, B)
        assert (g.view(np.float32).reshape(M, N).astype(np.float64) == value(A).astype(np.float64) @ value(B).astype(np.float64)).all()


def test_vote_is_ordered_equal_on_signed_zeros(rt, oracle):
    """a zero row of A against B >= 0 gives a +0.0 row of C, and so do negative-zero operands (0x80); a flip of bit 31 there
    makes -0.0, equal to +0.0 under `fcmp oeq`: not counted, and r0's value is stored.  A flip of bit 0 makes a denormal: counted."""
    M, N, K = 256, 256, 128
    A, B = int_operands(M, N, K, seed=3)
    B = bits(np.abs(value(B)))
    z = 77
    A[z] = 0x80
    tab = np.zeros(M * N, dtype=np.uint32)
    signs = [(z * N + 7 * c, c % 3) for c in range(30)]
    for u, r in signs:
        tab[u] = oracle.fault_entry(r, 0, 31)
    denormals = [(z * N + 250, 1), (z * N + 251, 0), (z * N + 252, 2)]
    for u, r in denormals:
        tab[u] = oracle.fault_entry(r, 0, 0)
    clean, _ = gpu(rt, 1, A, B)
    assert (clean.reshape(M, N)[z] == 0).all()                     # -0 x b summed from +0: +0.0
    for nc in (2, 3):
        g, st = both(rt, oracle, nc, A, B, table=tab)
        row = g.reshape(M, N)[z]
        counted = [u for u, r in denormals if r < nc]
        assert st["injected"] == sum(r < nc for _, r in signs + denormals)
        assert (st["errors_corrected"] if nc == 3 else st["dwc_detected"]) == len(counted)
        for u, r in signs:
            assert row[u - z * N] == (0x80000000 if r == 0 else 0), (nc, u, r)


@pytest.mark.parametrize("nc", [1, 2, 3])
def test_nan_operand_disagrees_in_every_element_of_its_row(rt, oracle, nc):
    """the E4M3 NaN (0x7F) in one row of A makes that C row NaN in every replica; NaN != NaN under `fcmp oeq`, so TMR
    -countErrors counts N disagreements and DWC N detections, as the oracle does.  The payload is not pinned."""
    M, N, K = 256, 128, 128
    A, B = int_operands(M, N, K, seed=19)
    z = 130
    A[z, 9] = 0x7F
    o, os_ = cpu(oracle, nc, A, B)
    g, gs = gpu(rt, nc, A, B)
    nan = np.isnan(o.view(np.float32)).reshape(M, N)
    assert nan[z].all() and nan.sum() == N
    assert (np.isnan(g.view(np.float32)).reshape(M, N) == nan).all()
    assert (g.reshape(M, N)[~nan] == o.reshape(M, N)[~nan]).all()
    assert {k: gs[k] for k in STAT_KEYS} == {k: os_[k] for k in STAT_KEYS}
    if nc > 1:
        assert (gs["errors_corrected"] if nc == 3 else gs["dwc_detected"]) == N and gs["first_fault_unit"] == z * N
