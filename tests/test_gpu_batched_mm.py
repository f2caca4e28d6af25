"""GPU (H100): batched matmuls (COAST_MM_BATCHED) -- `batch` independent products of one shape in one launch, on every matmul
path: the u8-limb tensor-core kernel, the register-tiled kernel, the plain kernel and the TF32 GEMM (single CTA, CTA pair, wide
128 x 256 with the tail split, narrow 128 x 128).

A batched launch must equal `batch` single launches (include/coast_rt.h), product b with d_in + b*M*K, d_aux + b*K*N,
d_out + b*M*N and unit_base + b*M*N: every output element and all five counters, bit for bit, with output buffers that start
poisoned.  The batched outputs are also checked against exact references: the u32 products against an exact mod-2^32 batched
matmul on 16-bit limbs in float64 (the limb scheme of test_gpu_wgmma_exact.mm_u32_ref), the TF32 products on integer-valued
operands (exact in fp32 whatever the order of the additions) against a float64 batched matmul.  The multi-wave sizes make
every persistent CTA run at least 3 tiles, with tiles of different products in one wave."""
import pytest

from test_gpu_stream_exact import GiB, _free, _room

pytestmark = pytest.mark.gpu

POISON = 0x5A5A5A5A
M32 = 0xFFFFFFFF
SMS = 132
GEMM_KNOBS = ("COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT", "COAST_MM_PATH",
              "COAST_HOST_CHUNK_BYTES", "COAST_HOST_PATH")


# ------------------------------------------------------------------------------------------ references (on the device)
def bmm_u32_ref(A, B):
    """exact C = A . B mod 2^32 per product of int32 tensors (batch x M x K, batch x K x N) holding u32 bits: 16-bit limbs,
    float64 batched matmuls, each limb-product sum below 2^32 * K < 2^53.  Returns int64 values in [0, 2^32)."""
    import torch
    assert A.shape[2] == B.shape[1] and A.shape[2] < 2 ** 21
    a, b = A.to(torch.int64) & M32, B.to(torch.int64) & M32
    a0, a1, b0, b1 = (a & 0xFFFF).double(), (a >> 16).double(), (b & 0xFFFF).double(), (b >> 16).double()
    lo = torch.bmm(a0, b0).to(torch.int64)
    mid = torch.bmm(a0, b1).to(torch.int64) + torch.bmm(a1, b0).to(torch.int64)
    return (lo + ((mid & 0xFFFF) << 16)) & M32


def u32(x):
    import torch
    return x.to(torch.int64) & M32


def operands(rt, kernel, M, N, K, batch, seed):
    """u32: Philox words; TF32: integers in [-8, 8], so |C| <= 64 K < 2^24 and every partial sum is exact in fp32"""
    import torch
    import coast_b200 as cb
    if kernel == cb.K_MM_U32:
        A = torch.empty(batch * M * K, dtype=torch.int32, device="cuda")
        B = torch.empty(batch * K * N, dtype=torch.int32, device="cuda")
        rt.fill_philox(A, seed=seed)
        rt.fill_philox(B, seed=seed + 1)
        return A, B
    assert 64 * K < 2 ** 24
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randint(-8, 9, (batch * M * K,), dtype=torch.float32, device="cuda", generator=g)
    B = torch.randint(-8, 9, (batch * K * N,), dtype=torch.float32, device="cuda", generator=g)
    return A, B


def reference(kernel, A, B, M, N, K, batch):
    """the exact products, as int64 u32 bits (MM_U32) or as float64 values (GEMM_TF32)"""
    import torch
    import coast_b200 as cb
    if kernel == cb.K_MM_U32:
        return bmm_u32_ref(A.view(batch, M, K), B.view(batch, K, N)).view(-1)
    return torch.bmm(A.view(batch, M, K).double(), B.view(batch, K, N).double()).view(-1)


def as_ref(kernel, C):
    import coast_b200 as cb
    return u32(C) if kernel == cb.K_MM_U32 else C.double()


def poisoned(n, kernel):
    import torch
    import coast_b200 as cb
    out = torch.full((n,), POISON, dtype=torch.int32, device="cuda")
    return out if kernel == cb.K_MM_U32 else out.view(torch.float32)


def table(n, nc, n_sites, seed):
    """a TABLE plan: about a third of the units get an entry; some name a replica or a site that does not exist (ignored)"""
    import torch
    import coast_b200 as cb
    g = torch.Generator(device="cuda").manual_seed(seed)
    hit = torch.rand(n, device="cuda", generator=g) < 0.3
    rep = torch.randint(0, 4, (n,), device="cuda", generator=g)
    site = torch.randint(0, n_sites + 1, (n,), device="cuda", generator=g)
    bit = torch.randint(0, 32, (n,), device="cuda", generator=g)
    e = cb.fault_entry(0, 0, 0) | (rep << 29) | (site << 5) | bit
    e = torch.where(hit, e, torch.zeros_like(e))
    return ((e + 2 ** 31) % 2 ** 32 - 2 ** 31).to(torch.int32)            # the u32 entries' bits


def launch(rt, kernel, nc, A, B, out, M, N, K, n, *, flags, plan, base, batched=True):
    import coast_b200 as cb
    d = rt.make_desc(kernel, nc, A, out, n, flags=flags, mode=cb.MM_BATCHED if batched else 0, M=M, N=N, K=K, d_aux=B, plan=plan,
                     unit_base=base)
    rt.launch(d)


def batched_vs_singles(rt, kernel, nc, M, N, K, batch, *, flags, plan_kind, seed, base):
    """one batched launch and `batch` single launches of the same operands: outputs and counters must be identical"""
    import torch
    import coast_b200 as cb
    A, B = operands(rt, kernel, M, N, K, batch, seed)
    n, mn = batch * M * N, M * N
    tab = None
    if plan_kind == "table":
        tab = table(n, nc, rt.fault_sites(kernel, 0, K), seed)
        plan = cb.FaultPlan(mode=cb.PLAN_TABLE, table=tab)
    elif plan_kind == "bernoulli":
        plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=seed, p=0.3)
    else:
        plan = None
    rt.sync()
    one = poisoned(n, kernel)
    launch(rt, kernel, nc, A, B, one, M, N, K, n, flags=flags, plan=plan, base=base)
    st1 = rt.sync()
    many = poisoned(n, kernel)
    for b in range(batch):
        pb = plan
        if tab is not None:
            pb = cb.FaultPlan(mode=cb.PLAN_TABLE, table=tab[b * mn:(b + 1) * mn])
        launch(rt, kernel, nc, A[b * M * K:(b + 1) * M * K], B[b * K * N:(b + 1) * K * N], many[b * mn:(b + 1) * mn], M, N, K, mn,
               flags=flags, plan=pb, base=base + b * mn, batched=False)
    stn = rt.sync()
    assert torch.equal(one.view(torch.int32), many.view(torch.int32))
    assert st1 == stn, (st1, stn)
    return A, B, one, st1


# (id, kernel id (3 MM_U32, 4 GEMM_TF32), M, N, K, batch, COAST_GEMM_PAIR, the kernel the launcher must pick)
PATHS = [
    ("tc", 3, 128, 64, 128, 400, None, "xmr_mm_u32_tc_nc{nc}"),                 # >= 3 tiles per persistent CTA
    ("tiled", 3, 64, 128, 32, 64, None, "xmr_mm_u32_tiled_nc{nc}"),
    ("plain", 3, 9, 9, 9, 300, None, "xmr_mm_u32_nc{nc}"),
    ("tf32_single", 4, 128, 128, 64, 400, "0", "xmr_gemm_tf32_nc{nc}"),         # NC 1: N % 256 != 0, the narrow kernel
    ("tf32_pair", 4, 256, 256, 64, 200, "1", "xmr_gemm_tf32p_nc{nc}"),
    ("tf32_wide", 4, 128, 256, 32, 446, "0", "xmr_gemm_tf32_nc{nc}"),
    ("tf32_narrow", 4, 128, 128, 32, 400, None, "xmr_gemm_tf32n_nc{nc}"),
]
PLANS = ["none", "bernoulli", "table", "majority"]


def _env(monkeypatch, **env):
    for k in GEMM_KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _expected_name(path, nc):
    pid, _, M, N, _, _, _, name = path
    if pid == "tf32_single" and nc == 1:
        return "xmr_gemm_tf32n_nc1"
    if pid in ("tf32_wide", "tf32_narrow") and nc > 1:
        return f"xmr_gemm_tf32_nc{nc}"
    return name.format(nc=nc)


@pytest.mark.parametrize("plan_kind", PLANS)
@pytest.mark.parametrize("nc", [1, 2, 3])
@pytest.mark.parametrize("path", PATHS, ids=[p[0] for p in PATHS])
def test_batched_launch_equals_single_launches(rt, monkeypatch, capfd, path, nc, plan_kind):
    """every path at NC 1/2/3 under every plan, global units crossing 2^32: bit-identical to the single launches; with no
    plan also equal to the exact reference"""
    import coast_b200 as cb
    pid, kernel, M, N, K, batch, pair, _ = path
    _env(monkeypatch, **({"COAST_GEMM_PAIR": pair} if pair else {}))
    n = batch * M * N
    base = (1 << 32) - n // 2 - 7
    flags = 3 | (cb.F_MAJORITY_VOTER if plan_kind == "majority" else 0)
    capfd.readouterr()
    A, B, C, st = batched_vs_singles(rt, kernel, nc, M, N, K, batch, flags=flags | cb.F_VERBOSE,
                                     plan_kind="table" if plan_kind == "table" else "none" if plan_kind == "none" else "bernoulli",
                                     seed=11 * nc + len(pid), base=base)
    first = capfd.readouterr().err.splitlines()[0]
    assert f"{_expected_name(path, nc)}_inj{0 if plan_kind == 'none' else 1} " in first and f"units={n}" in first, first
    if plan_kind == "none":
        assert (as_ref(kernel, C) == reference(kernel, A, B, M, N, K, batch)).all()
        assert st.injected == st.errors_corrected == st.dwc_detected == 0 and (nc < 3 or st.syncs == n)
    else:
        assert st.injected > 0
        if nc == 3:                                              # single flips are out-voted
            assert (as_ref(kernel, C) == reference(kernel, A, B, M, N, K, batch)).all()


@pytest.mark.parametrize("nc", [2, 3])
@pytest.mark.parametrize("shape", [(9, 9, 9, 300), (128, 64, 128, 40), (64, 128, 32, 24)], ids=["plain", "tc", "tiled"])
def test_no_mem_replication_votes_every_k_step_of_every_product(rt, monkeypatch, capfd, nc, shape):
    """-noMemReplication: every product runs on the plain kernel with K + 1 votes per unit, batched as single"""
    import coast_b200 as cb
    _env(monkeypatch)
    M, N, K, batch = shape
    n = batch * M * N
    capfd.readouterr()
    A, B, C, st = batched_vs_singles(rt, cb.K_MM_U32, nc, M, N, K, batch, flags=3 | cb.F_NO_MEM_REPLICATION | cb.F_VERBOSE,
                                     plan_kind="bernoulli", seed=5 + nc, base=(1 << 32) - 1000)
    assert f"xmr_mm_u32_nc{nc}_inj1 " in capfd.readouterr().err.splitlines()[0]
    if nc == 3:                                                  # syncs are counted under TMR
        assert st.syncs == (K + 1) * n
        assert (u32(C) == reference(cb.K_MM_U32, A, B, M, N, K, batch)).all()


def _grid(capfd):
    line = capfd.readouterr().err.splitlines()[0]
    return int(line.split("grid=")[1].split()[0]), line


@pytest.mark.parametrize("nc", [1, 3])
def test_multi_wave_batches_of_the_reference_size_on_the_plain_kernel(rt, monkeypatch, capfd, nc):
    """the reference's 9 x 9 products, enough of them for every warp of the grid-stride grid to take 3 warp-tiles"""
    import coast_b200 as cb
    _env(monkeypatch)
    batch = 40100
    n = batch * 81
    A, B = operands(rt, cb.K_MM_U32, 9, 9, 9, batch, seed=3)
    C = poisoned(n, cb.K_MM_U32)
    capfd.readouterr()
    launch(rt, cb.K_MM_U32, nc, A, B, C, 9, 9, 9, n, flags=3 | cb.F_VERBOSE, plan=None, base=0)
    st = rt.sync()
    grid, line = _grid(capfd)
    assert "xmr_mm_u32_nc" in line and n >= 3 * grid * 8 * (32 // nc), (n, grid)
    assert (u32(C) == reference(cb.K_MM_U32, A, B, 9, 9, 9, batch)).all()
    assert st.syncs == (n if nc == 3 else 0)


@pytest.mark.parametrize("case", [
    ("tc_nc3", 3, 128, 64, 256, 200, {}, "xmr_mm_u32_tc_nc3"),         # BN 32: 2 tiles per product
    ("tc_nc1", 1, 128, 64, 256, 400, {}, "xmr_mm_u32_tc_nc1"),
    ("tf32_tmr", 3, 128, 128, 96, 400, {}, "xmr_gemm_tf32_nc3"),
    ("tf32_pair_dwc", 2, 256, 128, 64, 200, {}, "xmr_gemm_tf32p_nc2"),
    ("tf32_wide_tail", 1, 128, 256, 64, 3 * SMS + 50, {"COAST_GEMM_PAIR": "0"}, "xmr_gemm_tf32_nc1"),
], ids=lambda c: c[0])
def test_multi_wave_batches_on_the_persistent_kernels(rt, monkeypatch, capfd, case):
    """at least 3 tiles per persistent CTA, products of different matrices in one wave; the unprotected wide batch leaves a
    short last round (50 tiles on 132 CTAs) that the kernel splits into halves"""
    import coast_b200 as cb
    cid, nc, M, N, K, batch, env, name = case
    kernel = cb.K_GEMM_TF32 if cid.startswith("tf32") else cb.K_MM_U32
    _env(monkeypatch, **env)
    n = batch * M * N
    A, B = operands(rt, kernel, M, N, K, batch, seed=len(cid))
    C = poisoned(n, kernel)
    capfd.readouterr()
    launch(rt, kernel, nc, A, B, C, M, N, K, n, flags=3 | cb.F_VERBOSE, plan=None, base=0)
    rt.sync()
    grid, line = _grid(capfd)
    assert f"{name}_inj0 " in line
    bn = {"tc_nc3": 32, "tc_nc1": 64}.get(cid, N)
    tiles = batch * (M // 128) * (N // bn) // (2 if "pair" in cid else 1)
    workers = grid // (2 if "pair" in cid else 1)
    assert tiles >= 3 * workers and (M // 128) * (N // bn) < workers, (tiles, workers)
    if cid == "tf32_wide_tail":
        assert grid == SMS and 0 < tiles % workers and 2 * (tiles % workers) <= workers
    assert (as_ref(kernel, C) == reference(kernel, A, B, M, N, K, batch)).all()


@pytest.mark.parametrize("kernel", ["mm_u32", "gemm_tf32"])
def test_shards_over_products_equal_one_launch(rt, monkeypatch, kernel):
    import torch
    import coast_b200 as cb
    _env(monkeypatch)
    k = cb.K_MM_U32 if kernel == "mm_u32" else cb.K_GEMM_TF32
    M, N, K, batch, lo = 128, 128, 128, 41, 17
    A, B = operands(rt, k, M, N, K, batch, seed=9)
    n, mn = batch * M * N, M * N
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=77, p=0.25)
    one, two = poisoned(n, k), poisoned(n, k)
    rt.sync()
    launch(rt, k, 3, A, B, one, M, N, K, n, flags=3, plan=plan, base=1 << 32)
    st1 = rt.sync()
    launch(rt, k, 3, A[: lo * M * K], B[: lo * K * N], two[: lo * mn], M, N, K, lo * mn, flags=3, plan=plan, base=1 << 32)
    sa = rt.sync()
    launch(rt, k, 3, A[lo * M * K:], B[lo * K * N:], two[lo * mn:], M, N, K, (batch - lo) * mn, flags=3, plan=plan,
           base=(1 << 32) + lo * mn)
    sb = rt.sync()
    assert torch.equal(one.view(torch.int32), two.view(torch.int32))
    assert st1.injected == sa.injected + sb.injected > 0
    assert st1.errors_corrected == sa.errors_corrected + sb.errors_corrected
    assert st1.syncs == sa.syncs + sb.syncs
    assert st1.first_fault_unit == min(sa.first_fault_unit, sb.first_fault_unit)


@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("kernel,M,N,K,batch", [("mm_u32", 128, 64, 128, 37), ("mm_u32", 9, 9, 9, 1000), ("gemm_tf32", 128, 128, 64, 29)])
def test_host_call_in_chunks_of_products_equals_the_device_launch(rt, monkeypatch, kernel, M, N, K, batch, pinned):
    import torch
    import coast_b200 as cb
    _env(monkeypatch)
    k = cb.K_MM_U32 if kernel == "mm_u32" else cb.K_GEMM_TF32
    A, B = operands(rt, k, M, N, K, batch, seed=21)
    n = batch * M * N
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=8, p=0.3)
    d_out = poisoned(n, k)
    launch(rt, k, 3, A, B, d_out, M, N, K, n, flags=3, plan=plan, base=1 << 33)
    d_st = rt.sync()
    h_in, h_aux, h_out = A.cpu(), B.cpu(), poisoned(n, k).cpu()
    if pinned:
        h_in, h_aux, h_out = h_in.pin_memory(), h_aux.pin_memory(), h_out.pin_memory()
    per = 4 * (M * K + K * N + M * N)
    monkeypatch.setenv("COAST_HOST_CHUNK_BYTES", str(5 * per + per // 2))          # 5 products per chunk
    h_st = rt.run_host(k, 3, h_in, h_out, n, mode=cb.MM_BATCHED, M=M, N=N, K=K, h_aux=h_aux, flags=3, plan=plan, unit_base=1 << 33)
    assert rt.last_host_path == "staged"
    assert torch.equal(h_out.view(torch.int32), d_out.view(torch.int32).cpu()) and h_st == d_st and d_st.injected > 0


def test_tf32_tmr_batch_past_4gib(rt, monkeypatch):
    """2^18 products of 128 x 128 x 32: 2^32 units, 16 GiB of C, 4 GiB each of A, B and the B^T scratch, TMR with a Bernoulli
    plan.  Every element equals the float64 reference (single flips are out-voted; each one is a counted disagreement),
    checked on the device a group of products at a time."""
    import torch
    import coast_b200 as cb
    _env(monkeypatch)
    M, N, K, batch = 128, 128, 32, 1 << 18
    n = batch * M * N
    assert n == 1 << 32
    _room(28 * GiB + 2 * GiB)
    A, B = operands(rt, cb.K_GEMM_TF32, M, N, K, batch, seed=31)
    C = torch.empty(n, dtype=torch.float32, device="cuda")
    rt.sync()
    launch(rt, cb.K_GEMM_TF32, 3, A, B, C, M, N, K, n, flags=3, plan=cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=5, threshold=1 << 20),
           base=0)
    st = rt.sync()
    assert st.injected > 0 and 0 < st.errors_corrected <= st.injected and st.syncs == n   # a flipped sign of 0.0 still compares equal
    g = 4096
    for b0 in range(0, batch, g):
        a = A[b0 * M * K:(b0 + g) * M * K].view(g, M, K).double()
        b = B[b0 * K * N:(b0 + g) * K * N].view(g, K, N).double()
        assert torch.equal(C[b0 * M * N:(b0 + g) * M * N].view(g, M, N).double(), torch.bmm(a, b)), b0
    del A, B, C
    _free()


def test_bad_batches_are_refused(rt):
    import torch
    import coast_b200 as cb
    buf = torch.zeros(1 << 16, dtype=torch.int32, device="cuda")
    for kernel, n, M, N, K in ((cb.K_MM_U32, 64 * 3 + 1, 8, 8, 8), (cb.K_MM_U32, 0, 8, 8, 8), (cb.K_CRC16, 64, 8, 8, 8)):
        with pytest.raises(cb.CoastError) as e:
            rt.launch(rt.make_desc(kernel, 3, buf, buf, n, mode=cb.MM_BATCHED, M=M, N=N, K=K, d_aux=buf, unit_bytes=8))
        assert e.value.code == cb.runtime.ERR_BAD_ARG and "COAST_MM_BATCHED" in str(e.value)
