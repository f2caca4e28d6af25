"""GPU (H100): matmuls with B stored transposed (COAST_MM_B_TRANSPOSED: d_aux holds B^T, N rows of K per product).

The definition is checked bit for bit: a launch with the bit equals the same launch without it whose d_aux holds B = (B^T)^T --
every output element on poisoned buffers, all five counters and d_status -- on every path (MM_U32 limbs, register-tiled and
plain; GEMM_TF32 and GEMM_BF16 wide, narrow, pair, single and grouped), NC 1/2/3, every fault plan kind and every launch form,
with global units crossing 2^32.  Integer-valued TF32 / BF16 operands are also held to a float64 A @ B^T.T exactly, and a B^T
whose entries encode their own position shows a mis-strided or mis-swizzled K-major box at once."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KNOBS = ("COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT", "COAST_HOST_CHUNK_BYTES",
         "COAST_HOST_PATH", "COAST_MM_PATH")
MM_BATCHED, MM_GROUPED, BT = 0x20000, 0x40000, 0x80000
K_MM_U32, K_GEMM_TF32, K_GEMM_BF16 = 3, 4, 8
STAT_KEYS = ("errors_corrected", "dwc_detected", "syncs", "injected", "first_fault_unit")
POISON = 0x7FC00BAD
RO = [3, 3, 100, 101, 101, 500, 700, 828]          # from row 3: empty products, a one-row product, a 128-row product


def env(monkeypatch, **kv):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in kv.items():
        monkeypatch.setenv(k, v)


def operands(kernel, rows, batch, N, K, seed, integer=True, amax=8):
    """A (rows x K) and B^T (batch x N x K) on the device in the kernel's element type; TF32 / BF16 integer-valued with
    K amax^2 < 2^24 (exact in fp32), or uniform(-1, 1)"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kernel == K_MM_U32:
        def one(*s):
            return torch.randint(-2 ** 31, 2 ** 31, s, generator=g, device="cuda", dtype=torch.int64).to(torch.int32)
    else:
        dt = torch.bfloat16 if kernel == K_GEMM_BF16 else torch.float32
        assert not integer or amax * amax * K < 2 ** 24

        def one(*s):
            if integer:
                return torch.randint(-amax, amax + 1, s, generator=g, device="cuda").to(dt)
            return (torch.rand(s, generator=g, device="cuda") * 2 - 1).to(dt)
    return one(rows, K), one(batch, N, K)


def untransposed(Bt):
    return Bt.transpose(1, 2).contiguous()


def plan_of(kind, n, nc, n_sites, seed):
    import torch
    import coast_b200 as cb
    if kind == "none":
        return None, 3
    if kind in ("bernoulli", "majority"):
        return cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=seed, p=0.3), 3 | (cb.F_MAJORITY_VOTER if kind == "majority" else 0)
    rng = np.random.default_rng(seed)
    tab = np.zeros(n, dtype=np.uint32)
    for u in rng.choice(n, size=min(n, 400), replace=False):
        tab[u] = cb.fault_entry(int(rng.integers(0, nc + 1)), int(rng.integers(0, n_sites + 1)), int(rng.integers(0, 32)))
    return cb.FaultPlan(mode=cb.PLAN_TABLE, table=torch.from_numpy(tab.view(np.int32)).cuda()), 3


def launch(rt, kernel, nc, A, B, *, M, N, K, mode=0, rows=None, out_rows=None, n=None, flags=3, plan=None, unit_base=0):
    """one launch on poisoned C and status: (C bits, stats, status bytes)"""
    import torch
    out_rows = A.shape[0] if out_rows is None else out_rows
    n = out_rows * N if n is None else n
    out = torch.full((out_rows * N,), POISON, dtype=torch.int32, device="cuda")
    status = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    if kernel != K_MM_U32:
        out = out.view(torch.float32)
    _, st = rt.run(kernel, nc, A, n, M=M, N=N, K=K, aux=B, flags=flags, plan=plan, unit_base=unit_base, status=status,
                   mode=mode, rows=rows, out=out)
    return out.view(torch.int32).cpu().numpy(), st.as_dict(), status.cpu().numpy()


def same(rt, kernel, nc, A, Bt, *, form, M=None, N, K, **kw):
    """the launch with the bit on B^T equals the launch without it on B = (B^T)^T; returns its record"""
    mode = {"single": 0, "batched": MM_BATCHED, "grouped": MM_GROUPED}[form]
    b = untransposed(Bt)
    Bflat = b.reshape(-1, N) if form != "single" else b[0]
    with_bit = launch(rt, kernel, nc, A, Bt.reshape(-1, K), M=M, N=N, K=K, mode=mode | BT, **kw)
    without = launch(rt, kernel, nc, A, Bflat, M=M, N=N, K=K, mode=mode, **kw)
    assert (with_bit[0] == without[0]).all(), np.flatnonzero(with_bit[0] != without[0])[:8]
    assert with_bit[1] == without[1]
    assert (with_bit[2] == without[2]).all()
    return with_bit


def form_shapes(form, kernel, M, N, K, seed, integer=True):
    """(A, B^T, launch keywords) of a single, batched or grouped launch"""
    import torch
    if form == "single":
        A, Bt = operands(kernel, M, 1, N, K, seed, integer)
        return A, Bt, dict(M=M)
    if form == "batched":
        batch = 3
        A, Bt = operands(kernel, batch * M, batch, N, K, seed, integer)
        return A, Bt, dict(M=M)
    G = len(RO) - 1
    A, Bt = operands(kernel, RO[-1] + 40, G, N, K, seed, integer)
    ro = torch.tensor(RO, dtype=torch.int64, device="cuda")
    return A, Bt, dict(M=G, rows=ro, n=(RO[-1] - RO[0]) * N)


def poison_kept(C, N, grouped):
    if grouped:
        C = C.reshape(-1, N)
        assert (C[:RO[0]] == POISON).all() and (C[RO[-1]:] == POISON).all()
    else:
        assert not (C == POISON).any()


# ------------------------------------------------------------------------------------------ MM_U32, every path
@pytest.mark.parametrize("form", ["single", "batched", "grouped"])
@pytest.mark.parametrize("plan_kind", ["none", "bernoulli", "table", "majority"])
@pytest.mark.parametrize("nc", [1, 2, 3])
@pytest.mark.parametrize("path", ["tc", "tiled", "naive"])
def test_mm_u32_every_path_equals_the_b_launch(rt, monkeypatch, capfd, path, nc, plan_kind, form):
    import coast_b200 as cb
    env(monkeypatch, COAST_MM_PATH=path)
    M, N, K = 256, 128, 128
    A, Bt, kw = form_shapes(form, K_MM_U32, M, N, K, seed=nc + 10 * len(path))
    n = kw.get("n", A.shape[0] * N)
    plan, flags = plan_of(plan_kind, n, nc, K, seed=nc)
    base = 2 ** 32 - n // 2                                        # the global units cross 2^32
    capfd.readouterr()
    C, st, _ = same(rt, K_MM_U32, nc, A, Bt, form=form, N=N, K=K, plan=plan, flags=flags | cb.F_VERBOSE, unit_base=base, **kw)
    names = [ln.split()[1] for ln in capfd.readouterr().err.splitlines() if ln.startswith("coast_rt: xmr_mm_u32")]
    stem = {"tc": "xmr_mm_u32_tc_", "tiled": "xmr_mm_u32_tiled_", "naive": "xmr_mm_u32_"}[path]
    assert len(names) == 2 and all(x.startswith(stem) for x in names), names
    assert ("_bt_" in names[0]) == (path != "tc" or plan is not None), names  # the limb inj0 kernels never read B
    poison_kept(C, N, form == "grouped")
    if plan_kind != "none":
        assert st["injected"] > 0


@pytest.mark.parametrize("form", ["single", "batched", "grouped"])
@pytest.mark.parametrize("nc", [2, 3])
def test_mm_u32_no_mem_replication_votes_every_k_step(rt, monkeypatch, nc, form):
    """-countErrors -countSyncs -noMemReplication on the plain kernel: K + 1 votes per unit, with and without the bit"""
    import coast_b200 as cb
    env(monkeypatch)
    M, N, K = 128, 128, 96
    A, Bt, kw = form_shapes(form, K_MM_U32, M, N, K, seed=5)
    n = kw.get("n", A.shape[0] * N)
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=3, p=0.2)
    _, st, _ = same(rt, K_MM_U32, nc, A, Bt, form=form, N=N, K=K, plan=plan, flags=3 | cb.F_NO_MEM_REPLICATION, **kw)
    assert st["syncs"] == (n * (K + 1) if nc == 3 else 0) and st["injected"] > 0


# ------------------------------------------------------------------------------------------ TF32 and BF16, every variant
# (id, environment, NC, M, N): multi-wave, at least 3 tiles per persistent CTA
VARIANTS = [
    ("wide_nc1", {"COAST_GEMM_PAIR": "0"}, 1, 4096, 4096),
    ("wide_nc1_no_tail_split", {"COAST_GEMM_PAIR": "0", "COAST_GEMM_TAIL_SPLIT": "0"}, 1, 2560, 4096),
    ("wide_nc1_tail_split", {"COAST_GEMM_PAIR": "0"}, 1, 2560, 4096),
    ("narrow_nc1", {}, 1, 4096, 3968),
    ("pair_nc1", {"COAST_GEMM_PAIR": "1"}, 1, 4096, 4096),
    ("pair_nc2", {"COAST_GEMM_PAIR": "1"}, 2, 2048, 3072),
    ("pair_nc3", {"COAST_GEMM_PAIR": "1"}, 3, 2048, 3072),
    ("single_nc2", {"COAST_GEMM_PAIR": "0"}, 2, 2048, 3072),
    ("single_nc3", {"COAST_GEMM_PAIR": "0"}, 3, 2048, 3072),
]


@pytest.mark.parametrize("plan_kind", ["none", "bernoulli", "table"])
@pytest.mark.parametrize("variant", VARIANTS, ids=[v[0] for v in VARIANTS])
@pytest.mark.parametrize("kernel", [K_GEMM_TF32, K_GEMM_BF16], ids=["tf32", "bf16"])
def test_gemm_every_variant_equals_the_b_launch(rt, monkeypatch, kernel, variant, plan_kind):
    _, e, nc, M, N = variant
    env(monkeypatch, **e)
    K = 256
    A, Bt = operands(kernel, M, 1, N, K, seed=nc + M, integer=False)
    plan, flags = plan_of(plan_kind, M * N, nc, 1, seed=nc)
    _, st, _ = same(rt, kernel, nc, A, Bt, form="single", M=M, N=N, K=K, plan=plan, flags=flags, unit_base=2 ** 32 - 12345)
    assert (st["injected"] > 0) == (plan is not None)


@pytest.mark.parametrize("form", ["batched", "grouped"])
@pytest.mark.parametrize("plan_kind", ["none", "bernoulli", "table"])
@pytest.mark.parametrize("nc", [1, 2, 3])
@pytest.mark.parametrize("kernel", [K_GEMM_TF32, K_GEMM_BF16], ids=["tf32", "bf16"])
def test_gemm_batched_and_grouped_equal_the_b_launch(rt, monkeypatch, kernel, nc, plan_kind, form):
    env(monkeypatch)
    M, N, K = 256, 256, 192
    A, Bt, kw = form_shapes(form, kernel, M, N, K, seed=nc, integer=False)
    n = kw.get("n", A.shape[0] * N)
    plan, flags = plan_of(plan_kind, n, nc, 1, seed=nc + 1)
    C, _, _ = same(rt, kernel, nc, A, Bt, form=form, N=N, K=K, plan=plan, flags=flags, unit_base=2 ** 32 - 999, **kw)
    poison_kept(C, N, form == "grouped")


@pytest.mark.parametrize("kernel", [K_GEMM_TF32, K_GEMM_BF16], ids=["tf32", "bf16"])
def test_integer_operands_at_4096_cubed_equal_float64(rt, monkeypatch, kernel):
    import torch
    M = N = K = 4096
    A, Bt = operands(kernel, M, 1, N, K, seed=7, amax=8)
    ref = A.to(torch.float64) @ Bt[0].to(torch.float64).T
    for e, nc in [({"COAST_GEMM_PAIR": "0"}, 1), ({}, 1), ({}, 2), ({}, 3)]:
        env(monkeypatch, **e)
        out = torch.full((M * N,), float("nan"), dtype=torch.float32, device="cuda")
        _, st = rt.run(kernel, nc, A, M * N, M=M, N=N, K=K, aux=Bt[0], flags=3, mode=BT, out=out)
        assert st.errors_corrected == 0 and st.dwc_detected == 0
        assert torch.equal(out.view(M, N).to(torch.float64), ref), (e, nc)


@pytest.mark.parametrize("kernel", [K_GEMM_TF32, K_GEMM_BF16], ids=["tf32", "bf16"])
def test_moe_shapes_with_empty_experts_equal_float64(rt, monkeypatch, kernel):
    """a batched and a grouped mixture-of-experts shape (experts 3 and 6 get no rows), integer-valued, against float64"""
    import torch
    env(monkeypatch)
    N, K, E = 512, 1024, 8
    counts = [300, 0, 129, 1, 640, 17, 0, 256]
    ro = np.concatenate([[0], np.cumsum(counts)]).tolist()
    A, Bt = operands(kernel, ro[-1], E, N, K, seed=11, amax=4)
    out = torch.full((ro[-1] * N,), float("nan"), dtype=torch.float32, device="cuda")
    rows = torch.tensor(ro, dtype=torch.int64, device="cuda")
    rt.run(kernel, 3, A, ro[-1] * N, M=E, N=N, K=K, aux=Bt, flags=3, mode=MM_GROUPED | BT, rows=rows, out=out)
    ref = torch.cat([A[ro[g]:ro[g + 1]].to(torch.float64) @ Bt[g].to(torch.float64).T for g in range(E)])
    assert torch.equal(out.view(-1, N).to(torch.float64), ref)
    M = 256
    A, Bt = operands(kernel, E * M, E, N, K, seed=12, amax=4)
    out = torch.full((E * M * N,), float("nan"), dtype=torch.float32, device="cuda")
    rt.run(kernel, 2, A, E * M * N, M=M, N=N, K=K, aux=Bt, flags=3, mode=MM_BATCHED | BT, out=out)
    ref = torch.bmm(A.view(E, M, K).to(torch.float64), Bt.to(torch.float64).transpose(1, 2))
    assert torch.equal(out.view(E, M, N).to(torch.float64), ref)


@pytest.mark.parametrize("nc", [1, 3])
@pytest.mark.parametrize("pair", ["0", "1"])
@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (256, 128, 192), (256, 384, 128), (512, 256, 1024)])
@pytest.mark.parametrize("kernel", [K_GEMM_TF32, K_GEMM_BF16], ids=["tf32", "bf16"])
def test_b_transposed_entries_that_encode_their_position(rt, monkeypatch, kernel, M, N, K, pair, nc):
    """B^T[n][k] = (n % 16) * 8 + (k % 8) - 64, plus a half that tells neighbouring blocks apart, with one-hot rows of A:
    C[i] is column k_i of B^T, so a mis-strided or mis-swizzled K-major B box shows in every row box and every k group"""
    import torch
    env(monkeypatch, COAST_GEMM_PAIR=pair)
    dt = torch.bfloat16 if kernel == K_GEMM_BF16 else torch.float32
    n_idx, k_idx = torch.arange(N, device="cuda")[:, None], torch.arange(K, device="cuda")[None, :]
    Btv = ((n_idx % 16) * 8 + (k_idx % 8) - 64).float() + ((n_idx // 16 + k_idx // 8) % 3 - 1).float() * 0.5
    hot = (torch.arange(M, device="cuda") * 7 + 3) % K
    A = torch.zeros(M, K, device="cuda")
    A[torch.arange(M, device="cuda"), hot] = 1.0
    out = torch.full((M * N,), float("nan"), dtype=torch.float32, device="cuda")
    rt.run(kernel, nc, A.to(dt), M * N, M=M, N=N, K=K, aux=Btv.to(dt), flags=3, mode=BT, out=out)
    assert torch.equal(out.view(M, N), Btv.T[hot])


@pytest.mark.parametrize("kernel", [K_GEMM_TF32, K_GEMM_BF16], ids=["tf32", "bf16"])
def test_general_operands_within_the_bound_of_float64(rt, monkeypatch, kernel):
    import torch
    env(monkeypatch)
    M, N, K = 1024, 1024, 2048
    A, Bt = operands(kernel, M, 1, N, K, seed=3, integer=False)
    C, _, _ = same(rt, kernel, 3, A, Bt, form="single", M=M, N=N, K=K)
    ref = A.to(torch.float64) @ Bt[0].to(torch.float64).T
    err = (torch.from_numpy(C.view(np.float32)).cuda().view(M, N).to(torch.float64) - ref).abs().max().item()
    assert err <= (2e-6 if kernel == K_GEMM_BF16 else 2e-3) * K, err


# ------------------------------------------------------------------------------------------ shards and the host call
@pytest.mark.parametrize("kernel", [K_MM_U32, K_GEMM_TF32, K_GEMM_BF16], ids=["mm_u32", "tf32", "bf16"])
def test_shards_sum_to_the_whole_launch(rt, monkeypatch, kernel):
    import torch
    import coast_b200 as cb
    from coast_b200.shard import shard_groups
    env(monkeypatch)
    N, K = 128, 128
    G, R = len(RO) - 1, RO[-1] - RO[0]
    A, Bt = operands(kernel, RO[-1], G, N, K, seed=13)
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=2, p=0.1)
    ro = torch.tensor(RO, dtype=torch.int64, device="cuda")
    dt = torch.int32 if kernel == K_MM_U32 else torch.float32

    def fold(tot, s):
        for k in STAT_KEYS[:4]:
            tot[k] += s[k]
        tot["first_fault_unit"] = min(tot["first_fault_unit"], s["first_fault_unit"])
    whole, sw = rt.run(kernel, 3, A, R * N, M=G, N=N, K=K, aux=Bt, flags=3, mode=MM_GROUPED | BT, rows=ro, plan=plan, unit_base=50,
                       out=torch.zeros(RO[-1] * N, dtype=dt, device="cuda"))
    out = torch.zeros(RO[-1] * N, dtype=dt, device="cuda")
    tot = dict(errors_corrected=0, dwc_detected=0, syncs=0, injected=0, first_fault_unit=2 ** 64 - 1)
    for r in range(3):
        lo, hi = shard_groups(RO, r, 3)
        if hi == lo or RO[hi] == RO[lo]:
            continue
        _, s = rt.run(kernel, 3, A, (RO[hi] - RO[lo]) * N, M=hi - lo, N=N, K=K, aux=Bt[lo:], flags=3, mode=MM_GROUPED | BT,
                      rows=ro[lo:], plan=plan, unit_base=50 + (RO[lo] - RO[0]) * N, out=out)
        fold(tot, s.as_dict())
    assert torch.equal(out, whole) and tot == sw.as_dict()
    # batched: whole matrices per shard
    M, batch = 128, 5
    A, Bt = operands(kernel, batch * M, batch, N, K, seed=14)
    whole, sw = rt.run(kernel, 2, A, batch * M * N, M=M, N=N, K=K, aux=Bt, flags=3, mode=MM_BATCHED | BT, plan=plan, unit_base=7)
    parts, tot = [], dict(errors_corrected=0, dwc_detected=0, syncs=0, injected=0, first_fault_unit=2 ** 64 - 1)
    for lo, hi in ((0, 2), (2, 3), (3, 5)):
        o, s = rt.run(kernel, 2, A[lo * M:hi * M], (hi - lo) * M * N, M=M, N=N, K=K, aux=Bt[lo:hi], flags=3, mode=MM_BATCHED | BT,
                      plan=plan, unit_base=7 + lo * M * N)
        parts.append(o)
        fold(tot, s.as_dict())
    assert torch.equal(torch.cat(parts), whole) and tot == sw.as_dict()


@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("kernel", [K_MM_U32, K_GEMM_TF32, K_GEMM_BF16], ids=["mm_u32", "tf32", "bf16"])
def test_host_call_in_many_chunks_equals_the_device_launch(rt, monkeypatch, kernel, pinned):
    """coast_run_host with B^T: row blocks (B^T once), whole products per chunk and groups per chunk, against the device launch"""
    import torch
    env(monkeypatch, COAST_HOST_CHUNK_BYTES=str(300000))

    def host(t):
        t = t.cpu()
        return t.pin_memory() if pinned else t

    def hout(n):
        return host(torch.zeros(n, dtype=torch.int32 if kernel == K_MM_U32 else torch.float32))

    def same_bytes(h, want):                                       # Runtime.run returns its own outputs as bytes
        return torch.equal(h.view(torch.uint8), want.cpu().contiguous().view(torch.uint8))
    N, K = 128, 128
    # row blocks
    M = 1024
    A, Bt = operands(kernel, M, 1, N, K, seed=3)
    want, sw = rt.run(kernel, 3, A, M * N, M=M, N=N, K=K, aux=Bt[0], flags=3, mode=BT)
    h = hout(M * N)
    st = rt.run_host(kernel, 3, host(A), h, M * N, M=M, N=N, K=K, h_aux=host(Bt[0]), flags=3, mode=BT)
    assert rt.last_host_path == "row-blocks" and same_bytes(h, want) and st.as_dict() == sw.as_dict()
    # whole products
    M, batch = 128, 9
    A, Bt = operands(kernel, batch * M, batch, N, K, seed=4)
    want, sw = rt.run(kernel, 2, A, batch * M * N, M=M, N=N, K=K, aux=Bt, flags=3, mode=MM_BATCHED | BT)
    h = hout(batch * M * N)
    st = rt.run_host(kernel, 2, host(A), h, batch * M * N, M=M, N=N, K=K, h_aux=host(Bt), flags=3, mode=MM_BATCHED | BT)
    assert same_bytes(h, want) and st.as_dict() == sw.as_dict()
    # groups
    G, R = len(RO) - 1, RO[-1] - RO[0]
    A, Bt = operands(kernel, RO[-1], G, N, K, seed=5)
    ro = torch.tensor(RO, dtype=torch.int64)
    dt = torch.int32 if kernel == K_MM_U32 else torch.float32
    want, sw = rt.run(kernel, 3, A, R * N, M=G, N=N, K=K, aux=Bt, flags=3, mode=MM_GROUPED | BT, rows=ro.cuda(), unit_base=9,
                      out=torch.zeros(RO[-1] * N, dtype=dt, device="cuda"))
    h = hout(RO[-1] * N)
    st = rt.run_host(kernel, 3, host(A), h, R * N, M=G, N=N, K=K, h_aux=host(Bt), flags=3, mode=MM_GROUPED | BT, h_rows=ro,
                     unit_base=9)
    assert rt.last_host_path == "groups" and same_bytes(h, want) and st.as_dict() == sw.as_dict()
