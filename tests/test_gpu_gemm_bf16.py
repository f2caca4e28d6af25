"""GPU (H100): the BF16 GEMM (COAST_K_GEMM_BF16): bfloat16 A and B, fp32 accumulators and C, wgmma m64n128k16, B read in
place (MN-major) from the caller's row-major buffer, NC register accumulator replicas and the voting epilogue of GEMM_TF32.

Exact wherever arithmetic allows it: integer-valued operands with K amax^2 < 2^24 make every partial sum an exact fp32
integer, so outputs equal the CPU reference (tests/gemm_bf16_ref.py) and a float64 matmul bit for bit, whatever
order the tensor core adds in.  General operands are held to a stated absolute bound, and to bit-equality between every
kernel variant and replica count.  numpy has no bfloat16: operands are uint16 bit patterns on the host."""
import numpy as np
import pytest

import gemm_bf16_ref as ref16
from gemm_bf16_ref import bits, value

pytestmark = pytest.mark.gpu

KNOBS = ("COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT", "COAST_HOST_CHUNK_BYTES", "COAST_HOST_PATH")
STAT_KEYS = ("errors_corrected", "dwc_detected", "syncs", "injected", "first_fault_unit")
MM_BATCHED, MM_GROUPED = 0x20000, 0x40000


def int_operands(M, N, K, seed, amax=8):
    rng = np.random.default_rng(seed)
    assert amax <= 256 and amax * amax * K < 2 ** 24
    A = rng.integers(-amax, amax + 1, size=(M, K)).astype(np.float32)
    B = rng.integers(-amax, amax + 1, size=(K, N)).astype(np.float32)
    return bits(A), bits(B)


def uniform_operands(M, N, K, seed):
    """uniform(-1, 1) rounded to bfloat16 by torch (round to nearest even)"""
    import torch
    g = torch.Generator().manual_seed(seed)
    def one(r, c):
        t = (torch.rand(r, c, generator=g) * 2 - 1).to(torch.bfloat16)
        return t.view(torch.int16).numpy().view(np.uint16).copy()
    return one(M, K), one(K, N)


def dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x).view(np.int16)).cuda().view(torch.bfloat16)


def env(monkeypatch, **kv):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in kv.items():
        monkeypatch.setenv(k, v)


def gpu(rt, nc, A, B, *, flags=3, plan=None, table=None, unit_base=0, status=None, mode=0, M=None, n=None, rows=None, out=None):
    """A: (rows x K) uint16, B: (.. x N) uint16 -> (C bits as uint32, flat; stats dict)"""
    import torch
    import coast_b200 as cb
    K, N = A.shape[1], B.shape[1]
    M = A.shape[0] if M is None else M
    n = A.shape[0] * N if n is None else n
    if table is not None:
        plan = cb.FaultPlan(mode=cb.PLAN_TABLE, table=torch.from_numpy(table.view(np.int32).copy()).cuda())
    if out is None:
        out = torch.full((A.shape[0] * N,), float("nan"), dtype=torch.float32, device="cuda")    # poison: every element is written
    _, st = rt.run(cb.K_GEMM_BF16, nc, dev(A), n, M=M, N=N, K=K, aux=dev(B), flags=flags, plan=plan, unit_base=unit_base,
                   status=status, mode=mode, rows=rows, out=out)
    return out.cpu().numpy().view(np.uint32), st.as_dict()


def cpu(oracle, nc, A, B, *, flags=3, plan_kw=None, table=None, unit_base=0):
    plan = None
    if table is not None:
        plan = oracle.make_plan(oracle.PLAN_TABLE, table=table)
    elif plan_kw:
        plan = oracle.make_plan(oracle.PLAN_BERNOULLI, **plan_kw)
    return ref16.run(oracle, nc, A, B, flags=flags, plan=plan, unit_base=unit_base, threads=8)


def both(rt, oracle, nc, A, B, *, flags=3, plan_kw=None, table=None, unit_base=0):
    import coast_b200 as cb
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, **plan_kw) if plan_kw else None
    g, gs = gpu(rt, nc, A, B, flags=flags, plan=plan, table=table, unit_base=unit_base)
    o, os_ = cpu(oracle, nc, A, B, flags=flags, plan_kw=plan_kw, table=table, unit_base=unit_base)
    assert (g == o).all(), (nc, flags, np.flatnonzero(g != o)[:8])
    assert {k: gs[k] for k in STAT_KEYS} == {k: os_[k] for k in STAT_KEYS}
    return g, gs


# (id, environment, NC, M, N, the kernel the launcher must pick)
VARIANTS = [
    ("narrow_nc1", {}, 1, 256, 384, "xmr_gemm_bf16n_inj0_nc1"),                  # N % 256 != 0: 128 x 128 tiles
    ("wide_nc1", {"COAST_GEMM_PAIR": "0"}, 1, 256, 256, "xmr_gemm_bf16_inj0_nc1"),  # 128 x 256 tiles: four B boxes per stage
    ("pair_nc1", {}, 1, 256, 256, "xmr_gemm_bf16p_inj0_nc1"),
    ("pair_nc2", {}, 2, 256, 128, "xmr_gemm_bf16p_inj0_nc2"),                    # one 64-column box per CTA of the pair
    ("single_nc2", {"COAST_GEMM_PAIR": "0"}, 2, 256, 128, "xmr_gemm_bf16_inj0_nc2"),
    ("single_nc3", {}, 3, 256, 128, "xmr_gemm_bf16_inj0_nc3"),
    ("pair_nc3", {"COAST_GEMM_PAIR": "1"}, 3, 256, 256, "xmr_gemm_bf16p_inj0_nc3"),
]


@pytest.mark.parametrize("K", [64, 384, 448, 1088])      # one k-block; one 6-stage ring exactly; one wrap; many wraps
@pytest.mark.parametrize("variant", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_integer_operands_bit_exact_with_the_oracle(rt, oracle, variant, K, monkeypatch, capfd):
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
    _, st = both(rt, oracle, nc, A, B, plan_kw=dict(seed=K, p=0.3))
    assert st["injected"] > n // 5
    both(rt, oracle, nc, A, B, flags=3 | cb.F_MAJORITY_VOTER, plan_kw=dict(seed=K + 1, p=0.3))
    rng = np.random.default_rng(K + nc)
    tab = np.zeros(n, dtype=np.uint32)
    for u in rng.choice(n, size=300, replace=False):
        site = 0 if rng.random() < 0.8 else 1                      # site 1 does not exist: ignored
        tab[u] = oracle.fault_entry(int(rng.integers(0, 4)), site, int(rng.integers(0, 32)))   # replica >= NC: ignored
    base = 2 ** 32 - n // 2                                        # the global units cross 2^32
    both(rt, oracle, nc, A, B, flags=1, plan_kw=dict(seed=K + 2, threshold=1 << 30), unit_base=base)
    import torch
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


@pytest.mark.parametrize("M,N,K", [(512, 768, 320), (256, 384, 64), (384, 256, 2048)])
def test_general_operands_every_variant_same_bits_and_within_bound(rt, M, N, K, monkeypatch):
    """uniform(-1, 1) bfloat16 operands: the products are exact in fp32, the fp32 accumulation order is the tensor core's, so the
    float64 reference is held to the absolute bound 2e-6 K that GEMM_TF32 is held to; every variant and replica count adds in
    the same order and gives the same bits"""
    A, B = uniform_operands(M, N, K, seed=K)
    ref = value(A).astype(np.float64) @ value(B).astype(np.float64)
    first = None
    for e, nc in RUNS:
        env(monkeypatch, **e)
        g, st = gpu(rt, nc, A, B)
        assert st["errors_corrected"] == 0 and st["dwc_detected"] == 0, (e, nc)
        if first is None:
            first = g
            err = np.abs(g.view(np.float32).reshape(M, N).astype(np.float64) - ref).max()
            assert err <= 2e-6 * K, err
        assert (g == first).all(), (e, nc)


@pytest.mark.parametrize("nc", [1, 3])
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 128, 192), (128, 384, 128), (384, 128, 1024)])
def test_b_entries_that_encode_their_position(rt, nc, M, N, K, monkeypatch):
    """B[k][n] = (k % 16) * 8 + (n % 8) - 64, plus a half that tells neighbouring blocks apart, with N != K and one-hot rows of A:
    C[i] is row k_i of B, so a transposed, mis-strided or mis-swizzled B shows at once, in every column box and every k group"""
    env(monkeypatch, COAST_GEMM_PAIR="0")
    k_idx, n_idx = np.arange(K)[:, None], np.arange(N)[None, :]
    Bv = ((k_idx % 16) * 8 + (n_idx % 8) - 64).astype(np.float32)
    Bv += ((k_idx // 16 + n_idx // 8) % 3 - 1) * 0.5              # still exact in bfloat16 (8 significant bits)
    hot = (np.arange(M) * 7 + 3) % K
    Av = np.zeros((M, K), dtype=np.float32)
    Av[np.arange(M), hot] = 1.0
    g, _ = gpu(rt, nc, bits(Av), bits(Bv))
    assert (g.view(np.float32).reshape(M, N) == Bv[hot]).all()


@pytest.mark.parametrize("M,N,K", [(4096, 4096, 4096), (2560, 2048, 256), (2432, 2048, 320)])
def test_multi_wave_every_variant_equals_fp64(rt, M, N, K, monkeypatch):
    """several tiles per persistent CTA (the ring phase carries from tile to tile); 2560 / 2432 rows leave a short last round that
    the unprotected kernels split into half tiles.  Every run is bit-identical and equals the float64 matmul on the device."""
    import torch
    import coast_b200 as cb
    A, B = int_operands(M, N, K, seed=7, amax=8)
    dA, dB = dev(A), dev(B)
    ref = dA.to(torch.float64) @ dB.to(torch.float64)
    for e, nc in RUNS:
        env(monkeypatch, **e)
        out = torch.full((M * N,), float("nan"), dtype=torch.float32, device="cuda")
        _, st = rt.run(cb.K_GEMM_BF16, nc, dA, M * N, M=M, N=N, K=K, aux=dB, flags=3, out=out)
        assert st.errors_corrected == 0 and st.dwc_detected == 0, (e, nc)
        assert torch.equal(out.view(M, N).to(torch.float64), ref), (e, nc)


# ------------------------------------------------------------------------------------------ batched and grouped launches
BATCH_CASES = [(1, 128, 256, 128, 5, {"COAST_GEMM_PAIR": "0"}), (1, 256, 256, 64, 3, {}), (1, 128, 128, 192, 4, {}),
               (2, 256, 128, 64, 3, {}), (3, 128, 128, 128, 7, {})]


@pytest.mark.parametrize("nc,M,N,K,batch,e", BATCH_CASES)
def test_batched_equals_single_launches(rt, nc, M, N, K, batch, e, monkeypatch):
    import coast_b200 as cb
    env(monkeypatch, **e)
    A, B = int_operands(batch * M, N, batch * K, seed=batch)
    A = A[:, :K].copy()                                            # batch stacked A (M x K each), batch stacked B (K x N each)
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=9, p=0.2)
    base = 2 ** 32 - M * N
    g, st = gpu(rt, nc, A, B, M=M, mode=MM_BATCHED, plan=plan, unit_base=base)
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


RO = [3, 3, 100, 101, 101, 500, 700, 828]          # from row 3: empty products, a one-row product, a 128-row product


@pytest.mark.parametrize("nc", [1, 2, 3])
@pytest.mark.parametrize("N,K", [(128, 64), (384, 192)])
def test_grouped_equals_single_launches_and_keeps_rows_outside_the_table(rt, oracle, nc, N, K):
    import torch
    import coast_b200 as cb
    G, R = len(RO) - 1, RO[-1] - RO[0]
    rows_alloc = RO[-1] + 40
    A, B = int_operands(rows_alloc, N, G * K, seed=nc)
    A = A[:, :K].copy()
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=5, p=0.2)
    base = 2 ** 32 - 1000
    POISON = 0x7FC00BAD
    out = torch.full((rows_alloc * N,), POISON, dtype=torch.int32, device="cuda").view(torch.float32)
    ro = torch.tensor(RO, dtype=torch.int64, device="cuda")
    g, st = gpu(rt, nc, A, B, M=G, n=R * N, mode=MM_GROUPED, rows=ro, plan=plan, unit_base=base, out=out)
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


def test_equal_groups_equal_the_batched_launch(rt):
    import torch
    M, N, K, batch = 128, 256, 128, 6
    A, B = int_operands(batch * M, N, batch * K, seed=77)
    A = A[:, :K].copy()
    for nc in (1, 3):
        gb, sb = gpu(rt, nc, A, B, M=M, mode=MM_BATCHED, unit_base=11)
        ro = torch.arange(0, (batch + 1) * M, M, dtype=torch.int64, device="cuda")
        gg, sg = gpu(rt, nc, A, B, M=batch, mode=MM_GROUPED, rows=ro, unit_base=11)
        assert (gb == gg).all() and sb == sg


def test_sharding_over_products(rt):
    """whole products [g_lo, g_hi) per shard: same d_in / d_out, d_aux + g_lo K N, d_rows + g_lo, unit_base by rows"""
    import torch
    import coast_b200 as cb
    from coast_b200.shard import shard_groups
    N, K = 128, 128
    G, R = len(RO) - 1, RO[-1] - RO[0]
    A, B = int_operands(RO[-1], N, G * K, seed=13)
    A = A[:, :K].copy()
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=2, p=0.1)
    ro = torch.tensor(RO, dtype=torch.int64, device="cuda")
    whole, sw = gpu(rt, 3, A, B, M=G, n=R * N, mode=MM_GROUPED, rows=ro, plan=plan, unit_base=50,
                    out=torch.zeros(RO[-1] * N, dtype=torch.float32, device="cuda"))
    out = torch.zeros(RO[-1] * N, dtype=torch.float32, device="cuda")
    dA, dB = dev(A), dev(B)
    tot = dict(errors_corrected=0, dwc_detected=0, syncs=0, injected=0, first_fault_unit=2 ** 64 - 1)
    for r in range(3):
        lo, hi = shard_groups(RO, r, 3)
        if hi == lo or RO[hi] == RO[lo]:
            continue
        _, s = rt.run(cb.K_GEMM_BF16, 3, dA, (RO[hi] - RO[lo]) * N, M=hi - lo, N=N, K=K, aux=dB.view(-1)[lo * K * N:], flags=3,
                      mode=MM_GROUPED, rows=ro[lo:], plan=plan, unit_base=50 + (RO[lo] - RO[0]) * N, out=out)
        s = s.as_dict()
        for k in STAT_KEYS[:4]:
            tot[k] += s[k]
        tot["first_fault_unit"] = min(tot["first_fault_unit"], s["first_fault_unit"])
    assert (out.cpu().numpy().view(np.uint32) == whole).all() and tot == sw


@pytest.mark.parametrize("pinned", [False, True])
def test_host_call_row_blocks_products_and_groups(rt, pinned, monkeypatch):
    """coast_run_host with 2-byte A and B and 4-byte C: row blocks (B once), whole products per chunk, groups per chunk, each
    cut into many chunks, against the device launch"""
    import torch
    import coast_b200 as cb
    env(monkeypatch, COAST_HOST_CHUNK_BYTES=str(300000))

    def host(t):
        return t.pin_memory() if pinned else t

    def h16(x):
        return host(torch.from_numpy(np.ascontiguousarray(x).view(np.int16)))
    # row blocks
    M, N, K = 1024, 128, 128
    A, B = int_operands(M, N, K, seed=3)
    want, _ = gpu(rt, 3, A, B)
    h_out = host(torch.full((M * N,), float("nan"), dtype=torch.float32))
    st = rt.run_host(cb.K_GEMM_BF16, 3, h16(A), h_out, M * N, M=M, N=N, K=K, h_aux=h16(B), flags=3)
    assert rt.last_host_path == "row-blocks" and (h_out.numpy().view(np.uint32) == want).all() and st.syncs == M * N
    # whole products
    M, batch = 128, 9
    A, B = int_operands(batch * M, N, batch * K, seed=4)
    A = A[:, :K].copy()
    want, _ = gpu(rt, 2, A, B, M=M, mode=MM_BATCHED)
    h_out = host(torch.full((batch * M * N,), float("nan"), dtype=torch.float32))
    rt.run_host(cb.K_GEMM_BF16, 2, h16(A), h_out, batch * M * N, M=M, N=N, K=K, h_aux=h16(B), flags=3, mode=MM_BATCHED)
    assert (h_out.numpy().view(np.uint32) == want).all()
    # groups
    G, R = len(RO) - 1, RO[-1] - RO[0]
    A, B = int_operands(RO[-1], N, G * K, seed=5)
    A = A[:, :K].copy()
    ro = torch.tensor(RO, dtype=torch.int64)
    want, sw = gpu(rt, 3, A, B, M=G, n=R * N, mode=MM_GROUPED, rows=ro.cuda(), unit_base=9,
                   out=torch.zeros(RO[-1] * N, dtype=torch.float32, device="cuda"))
    h_out = host(torch.zeros(RO[-1] * N, dtype=torch.float32))
    st = rt.run_host(cb.K_GEMM_BF16, 3, h16(A), h_out, R * N, M=G, N=N, K=K, h_aux=h16(B), flags=3, mode=MM_GROUPED, h_rows=ro,
                     unit_base=9)
    assert rt.last_host_path == "groups" and (h_out.numpy().view(np.uint32) == want).all() and st.as_dict() == sw


# ------------------------------------------------------------------------------------------ fp32 voter edges through BF16 operands
def test_vote_is_ordered_equal_on_signed_zeros(rt, oracle):
    """a zero row of A against B >= 0 gives a +0.0 row of C; a flip of bit 31 there makes -0.0, equal to +0.0 under `fcmp oeq`:
    not counted, and r0's value is stored.  A flip of bit 0 makes a denormal: counted."""
    M, N, K = 256, 256, 64
    A, B = int_operands(M, N, K, seed=3)
    B = bits(np.abs(value(B)))
    z = 77
    A[z] = 0
    tab = np.zeros(M * N, dtype=np.uint32)
    signs = [(z * N + 7 * c, c % 3) for c in range(30)]
    for u, r in signs:
        tab[u] = oracle.fault_entry(r, 0, 31)
    denormals = [(z * N + 250, 1), (z * N + 251, 0), (z * N + 252, 2)]
    for u, r in denormals:
        tab[u] = oracle.fault_entry(r, 0, 0)
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
    """a quiet NaN bfloat16 (0x7FC0) in one row of A makes that C row NaN in every replica; NaN != NaN under `fcmp oeq`, so
    TMR -countErrors counts N disagreements and DWC N detections, as the oracle does.  The payload is not pinned."""
    M, N, K = 256, 128, 128
    A, B = int_operands(M, N, K, seed=19)
    z = 130
    A[z, 9] = 0x7FC0
    o, os_ = cpu(oracle, nc, A, B)
    g, gs = gpu(rt, nc, A, B)
    nan = np.isnan(o.view(np.float32)).reshape(M, N)
    assert nan[z].all() and nan.sum() == N
    assert (np.isnan(g.view(np.float32)).reshape(M, N) == nan).all()
    assert (g.reshape(M, N)[~nan] == o.reshape(M, N)[~nan]).all()
    assert {k: gs[k] for k in STAT_KEYS} == {k: os_[k] for k in STAT_KEYS}
    if nc > 1:
        assert (gs["errors_corrected"] if nc == 3 else gs["dwc_detected"]) == N and gs["first_fault_unit"] == z * N
