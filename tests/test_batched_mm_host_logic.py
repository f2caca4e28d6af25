"""Host logic of batched matmuls (COAST_MM_BATCHED with COAST_K_MM_U32 and COAST_K_GEMM_TF32) on a GPU-less box, against the
mock driver (tests/mock_cuda/mock_cuda.c) through tests/mock_cuda/mm_child.py.  A batch is `batch` products of one shape: the stacked A and C are one (batch*M)-row
matrix, and the B matrices become one stacked (batch*N) x K operand in the pre-pass.  Pinned here: the kernel and pre-passes
each path selects, the tensor maps of the stacked operands, the scratch and the grid; the TF32 CTA pair's need for a per-product
M that is a multiple of 256; every refusal; a batch of one being the unbatched launch, event for event; and the chunks of whole
products of the host call."""
import pytest

from mock_run import (BAD_ARG, K_CRC16, K_GEMM_TF32, K_MM_U32, MM_BATCHED, SMS, UNSUPPORTED, args_of, mock_dir,  # noqa: F401
                      run, spans, work)


# (id, kernel, nc, M, N, K, batch, env, launches in order, grid, scratch bytes or None)
PATHS = [
    ("tc_nc3", K_MM_U32, 3, 128, 64, 128, 5, {}, ["xmr_mm_split_a", "xmr_mm_split_bt", "xmr_mm_u32_tc_nc3_inj0"], 10,
     (5 * 128 * 128 + 5 * 128 * 64) * 4),
    ("tc_nc1_capped", K_MM_U32, 1, 128, 64, 128, 300, {}, ["xmr_mm_split_a", "xmr_mm_split_bt", "xmr_mm_u32_tc_nc1_inj0"], SMS,
     (300 * 128 * 128 + 300 * 128 * 64) * 4),
    ("tiled_nc2", K_MM_U32, 2, 64, 128, 16, 7, {}, ["xmr_mm_u32_tiled_nc2_inj0"], 7, None),
    ("plain_nc3", K_MM_U32, 3, 9, 9, 9, 100, {}, ["xmr_mm_u32_nc3_inj0"], -(-(-(-8100 // 10)) // 8), None),
    ("tf32_single_nc3", K_GEMM_TF32, 3, 128, 128, 64, 300, {}, ["xmr_gemm_bt", "xmr_gemm_tf32_nc3_inj0"], SMS, 300 * 64 * 128 * 4),
    ("tf32_pair_nc2", K_GEMM_TF32, 2, 256, 128, 64, 3, {}, ["xmr_gemm_bt", "xmr_gemm_tf32p_nc2_inj0"], 6, 3 * 64 * 128 * 4),
    ("tf32_pair_nc1", K_GEMM_TF32, 1, 256, 256, 32, 70, {}, ["xmr_gemm_bt", "xmr_gemm_tf32p_nc1_inj0"], SMS, 70 * 32 * 256 * 4),
    ("tf32_wide_nc1", K_GEMM_TF32, 1, 128, 256, 64, 5, {"COAST_GEMM_PAIR": "0"}, ["xmr_gemm_bt", "xmr_gemm_tf32_nc1_inj0"], 5,
     5 * 64 * 256 * 4),
    ("tf32_narrow_nc1", K_GEMM_TF32, 1, 128, 128, 64, 5, {}, ["xmr_gemm_bt", "xmr_gemm_tf32n_nc1_inj0"], 5, 5 * 64 * 128 * 4),
]


@pytest.mark.parametrize("case", PATHS, ids=[c[0] for c in PATHS])
def test_each_path_runs_its_prepasses_and_kernel_on_the_stacked_operands(mock_dir, tmp_path, case):
    _, kernel, nc, M, N, K, batch, env, want, grid, scratch = case
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="launch", kernel=kernel, nc=nc, M=M, N=N, K=K, batch=batch, unit_base=1 << 32,
                                               flags=3)], env_extra=env)
    r = res["ops"][0]
    assert r["rc"] == 0, r["err"]
    la = work(ev)
    assert [e["name"] for e in la] == want and len({e["stream"] for e in la}) == 1
    k = la[-1]
    assert k["grid"] == grid
    a = args_of(k)
    assert (a.n_units, a.M, a.N, a.K, a.unit_base) == (batch * M * N, M, N, K, 1 << 32)
    assert a.mode & MM_BATCHED == 0                                   # the kernels find the batch from n_units / N and M
    assert a.inp == r["in"] and a.out == r["out"] and a.aux == r["aux"]
    tm = [e for e in ev if e["op"] == "tmap"]
    allocs = [e for e in ev if e["op"] == "alloc"]
    if scratch is None:
        assert not tm and allocs[-1]["ptr"] == r["out"]             # the caller's C buffer was the last allocation
        return
    assert [(t["dim0"], t["dim1"]) for t in tm] == [(K, batch * M), (K, batch * N)]   # A: batch*M rows; B^T: batch*N rows
    assert allocs[-1]["bytes"] == scratch                             # the launch's one scratch allocation
    assert {"op": "free", "id": allocs[-1]["id"]} in ev[ev.index(k):]


@pytest.mark.parametrize("nc,M,N,env,want", [
    (1, 128, 256, {}, "xmr_gemm_tf32_nc1_inj0"),                     # 512 stacked rows, but a pair tile would straddle products
    (2, 128, 128, {}, "xmr_gemm_tf32_nc2_inj0"),
    (3, 128, 128, {"COAST_GEMM_PAIR": "1"}, "xmr_gemm_tf32_nc3_inj0"),
    (2, 256, 128, {}, "xmr_gemm_tf32p_nc2_inj0"),                    # M = 256 per product: pairs
])
def test_a_cta_pair_needs_the_per_product_rows(mock_dir, tmp_path, nc, M, N, env, want):
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="launch", kernel=K_GEMM_TF32, nc=nc, M=M, N=N, K=32, batch=4)], env_extra=env)
    assert res["ops"][0]["rc"] == 0
    assert work(ev)[-1]["name"] == want


TINY = [16, 16, 16]                                   # element counts of A, B and C: a refusal needs no memory
REFUSALS = [
    ("other_kernel", dict(kernel=K_CRC16, M=8, N=8, K=8, batch=2), BAD_ARG, "COAST_MM_BATCHED"),
    ("zero_units", dict(M=8, N=8, K=8, batch=0, alloc=TINY), BAD_ARG, "COAST_MM_BATCHED"),
    ("not_a_multiple", dict(M=8, N=8, K=8, n=2 * 64 + 1, batch=3), BAD_ARG, "multiple of M*N"),
    ("zero_M", dict(M=0, N=8, K=8, n=64, batch=1, alloc=TINY), BAD_ARG, "COAST_MM_BATCHED"),
    ("batch_M_2p31", dict(M=1 << 16, N=1, K=1, batch=1 << 15, alloc=TINY), BAD_ARG, "below 2^31"),
    ("batch_N_2p31", dict(M=1, N=1 << 16, K=1, batch=1 << 15, alloc=TINY), BAD_ARG, "below 2^31"),
    ("tf32_batch_M_2p31", dict(kernel=K_GEMM_TF32, M=128, N=128, K=32, batch=1 << 24, alloc=TINY), BAD_ARG, "below 2^31"),
    ("tf32_shape", dict(kernel=K_GEMM_TF32, M=100, N=128, K=64, batch=4), UNSUPPORTED, "multiples of 128"),
    ("unbatched_n", dict(M=8, N=8, K=8, n=2 * 64, batch=2, mode=0), BAD_ARG, "n_units must be M*N"),
    ("unbatched_tf32_n", dict(kernel=K_GEMM_TF32, M=128, N=128, K=32, n=2 * 128 * 128, batch=2, mode=0), BAD_ARG,
     "n_units must be M*N"),
]


# the unbatched host call blocks rows itself (each row block is a valid launch): its n_units refusals are launch-only
CALLS = [(call, c) for call in ("launch", "run_host") for c in REFUSALS if call == "launch" or c[1].get("mode") != 0]


@pytest.mark.parametrize("call,case", CALLS, ids=[f"{call}-{c[0]}" for call, c in CALLS])
def test_refusals_fail_loudly_before_any_work(mock_dir, tmp_path, call, case):
    _, op, code, needle = case
    res, ev, _ = run(mock_dir, tmp_path, [{"op": call, "kernel": K_MM_U32, **op}])
    r = res["ops"][0]
    assert r["rc"] == code and needle in r["err"], r
    assert not work(ev)
    if code == BAD_ARG:                    # the batch checks come before any copy; a path's shape rule at the first chunk's launch
        assert not [e for e in ev if e["op"] in ("h2d", "d2h")]


@pytest.mark.parametrize("kernel,nc,M,N,K,env", [
    (K_MM_U32, 3, 128, 64, 128, {}),
    (K_MM_U32, 2, 64, 128, 16, {}),
    (K_MM_U32, 3, 9, 9, 9, {}),
    (K_GEMM_TF32, 3, 128, 128, 64, {}),
    (K_GEMM_TF32, 1, 256, 256, 64, {}),
    (K_GEMM_TF32, 1, 128, 256, 64, {"COAST_GEMM_PAIR": "0"}),
    (K_GEMM_TF32, 1, 128, 128, 64, {}),
])
def test_a_batch_of_one_is_the_unbatched_launch(mock_dir, tmp_path, kernel, nc, M, N, K, env):
    """the same buffers launched with and without the bit: the same kernels, grids, argument blocks, tensor maps and scratch"""
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="launch", kernel=kernel, nc=nc, M=M, N=N, K=K, batch=1, twice=True, p=0.5,
                                               unit_base=77, flags=3)], env_extra=env)
    assert [r["rc"] for r in res["ops"]] == [0, 0]
    start = [i for i, e in enumerate(ev) if e["op"] == "alloc"][4] + 1          # after the counters and the caller's three buffers
    # each launch allocates its own scratch: its address, and the maps' on it, may differ
    seen = [{k: v for k, v in e.items() if k not in ("id", "ptr", "addr")} for e in ev[start:] if e["op"] in ("launch", "tmap", "alloc")]
    assert len(seen) % 2 == 0 and len(seen) >= 2
    assert seen[: len(seen) // 2] == seen[len(seen) // 2:]
    assert sum(e["op"] == "launch" for e in seen) >= 2


@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("kernel,M,N,K,batch,budget,per", [
    (K_MM_U32, 64, 64, 64, 10, 100000, 2),           # 48 KiB per product: two per chunk
    (K_MM_U32, 64, 64, 64, 10, 30000, 1),            # a product larger than the budget is a chunk of its own
    (K_MM_U32, 128, 64, 128, 7, 0, 7),               # default 16 MiB: one chunk (the limb kernel)
    (K_GEMM_TF32, 128, 128, 32, 9, 200000, 2),
])
def test_host_call_chunks_are_whole_products(mock_dir, tmp_path, kernel, M, N, K, batch, budget, per, pinned):
    env = {"COAST_HOST_CHUNK_BYTES": str(budget)} if budget else {}
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", kernel=kernel, nc=3, M=M, N=N, K=K, batch=batch, unit_base=1000,
                                               pinned=pinned)], env_extra=env)
    r = res["ops"][0]
    assert r["rc"] == 0 and r["path"] == "staged", r
    ab, bb, cb = 4 * M * K, 4 * K * N, 4 * M * N
    ups_a, ups_b = spans(ev, "h2d", r["host_in"], batch * ab), spans(ev, "h2d", r["host_aux"], batch * bb)
    downs = spans(ev, "d2h", r["host_out"], batch * cb)
    la = [e for e in work(ev) if "_nc" in e["name"]]
    chunks = [(f, min(per, batch - f)) for f in range(0, batch, per)]
    assert len(ups_a) == len(ups_b) == len(downs) == len(la) == len(chunks)
    for i, ((f, cnt), ua, ub, dc, k) in enumerate(zip(chunks, ups_a, ups_b, downs, la)):
        assert ua[:2] == (f * ab, cnt * ab) and ub[:2] == (f * bb, cnt * bb) and dc[:2] == (f * cb, cnt * cb)
        assert ua[2] == ub[2] == dc[2] == k["stream"]                  # one stream per chunk ...
        a = args_of(k)
        assert (a.n_units, a.unit_base, a.M, a.N, a.K) == (cnt * M * N, 1000 + f * M * N, M, N, K)
    assert len({k["stream"] for k in la}) == min(3, len(chunks))       # ... round-robin over the three host streams
