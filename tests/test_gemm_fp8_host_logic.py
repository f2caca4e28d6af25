"""Host logic of COAST_K_GEMM_FP8 on a GPU-less box, against the mock driver (tests/mock_cuda/mock_cuda.c) through
tests/mock_cuda/mm_child.py, whose A and B buffers hold 1-byte elements.  Pinned here: the kernel each shape gets (single CTA
wide / narrow, CTA pair, grouped), grid and shared memory, both UINT8 tensor maps (A rows x K and B^T (P N) rows x K, boxes of
128 bytes), the byte-transposing pre-pass and its P K N bytes of scratch without COAST_MM_B_TRANSPOSED and neither with it,
every refusal with its message, that a batch of one is the unbatched launch, the bytes the host call copies per chunk (1-byte A
and B, 4-byte C), that every xmr_gemm_fp8 function of the cubin runs the E4M3 wgmma, and that none keeps more stack than its
TF32 or BF16 twin.  tests/test_mm_plan_sweep.py shows that each is reached."""
import re

import pytest

from mock_run import (BAD_ARG, GRP_BYTES, K_CRC16, K_GEMM_FP8, MM_B_TRANSPOSED as MM_BT, MM_BATCHED, MM_GROUPED, SMS,  # noqa: F401
                      UNSUPPORTED, arg0_ptr, args_of, maps, mock_dir, res_usage, run, sass_by_function, spans, work)

SMEM = 6 * (128 * 128 + 128 * 128) + 1024 + 256          # xmr_gemm_smem: the same bytes wide and narrow


# (id, nc, M, N, K, batch or None, environment, kernel, grid)
LAUNCHES = [
    ("single_nc3", 3, 512, 512, 128, None, {}, "xmr_gemm_fp8_inj0_nc3", 16),
    ("narrow_nc1", 1, 512, 384, 128, None, {}, "xmr_gemm_fp8n_inj0_nc1", 12),         # N % 256 != 0
    ("wide_nc1", 1, 384, 512, 256, None, {}, "xmr_gemm_fp8_inj0_nc1", 6),             # M % 256 != 0: no pair tile
    ("pair_nc1", 1, 512, 512, 128, None, {}, "xmr_gemm_fp8p_inj0_nc1", 8),            # 256 x 256 pair tiles: 4 pairs
    ("pair_nc2", 2, 512, 384, 128, None, {}, "xmr_gemm_fp8p_inj0_nc2", 12),
    ("pair_nc3", 3, 512, 512, 128, None, {"COAST_GEMM_PAIR": "1"}, "xmr_gemm_fp8p_inj0_nc3", 16),
    ("single_nc2", 2, 512, 512, 128, None, {"COAST_GEMM_PAIR": "0"}, "xmr_gemm_fp8_inj0_nc2", 16),
    ("batched_nc3", 3, 128, 128, 128, 300, {}, "xmr_gemm_fp8_inj0_nc3", SMS),
    ("batched_pair_nc2", 2, 256, 128, 384, 3, {}, "xmr_gemm_fp8p_inj0_nc2", 6),
    ("batched_wide_nc1", 1, 128, 256, 128, 5, {}, "xmr_gemm_fp8_inj0_nc1", 5),        # a pair tile would straddle two products
]


@pytest.mark.parametrize("bt", [False, True], ids=["B", "Bt"])
@pytest.mark.parametrize("case", LAUNCHES, ids=[c[0] for c in LAUNCHES])
def test_launch_records(mock_dir, tmp_path, case, bt):
    _, nc, M, N, K, batch, env, name, grid = case
    op = dict(op="launch", kernel=K_GEMM_FP8, nc=nc, M=M, N=N, K=K, unit_base=1 << 32, flags=3, bt=bt)
    if batch:
        op["batch"] = batch
    b = batch or 1
    res, ev, _ = run(mock_dir, tmp_path, [op], env_extra=env)
    r = res["ops"][0]
    assert r["rc"] == 0, r["err"]
    la = work(ev)
    k = la[-1]
    assert (k["name"], k["grid"], k["block"], k["smem"]) == (name, grid, 384, SMEM) and (grid % 2 == 0 or "fp8p" not in name)
    a = args_of(k)
    assert (a.n_units, a.M, a.N, a.K, a.unit_base, a.n_sites) == (b * M * N, M, N, K, 1 << 32, 1)
    assert a.mode & (MM_GROUPED | MM_BATCHED | MM_BT) == 0 and (a.inp, a.aux, a.out) == (r["in"], r["aux"], r["out"])
    allocs = [e for e in ev if e["op"] == "alloc" and not e["host"]]
    caller = allocs.index([e for e in allocs if e["ptr"] == r["out"]][0])
    scratch = allocs[caller + 1:]
    if bt:                                                         # the caller's B^T in place: no pre-pass, no scratch
        assert [e["name"] for e in la] == [name] and scratch == []
        b_at = r["aux"]
    else:                                                          # B^T of every product into P K N bytes of scratch first
        assert [e["name"] for e in la] == ["xmr_gemm_bt_u8", name] and [e["bytes"] for e in scratch] == [b * K * N]
        assert arg0_ptr(la[0]) == r["aux"] and la[0]["stream"] == k["stream"]
        b_at = scratch[0]["ptr"]
        assert {"op": "free", "id": scratch[0]["id"]} in ev[ev.index(k):]
    # A: (batch M) rows of K bytes, boxes of one 128-byte k-block x 128 rows; B^T: (batch N) rows of K, 128 bytes x 128 (pairs: 64)
    assert maps(ev) == [(r["in"], 1, K, b * M, 128, 128), (b_at, 1, K, b * N, 128, 64 if "fp8p" in name else 128)]


RO = [3, 3, 100, 101, 101, 500, 700]
R, G = RO[-1] - RO[0], len(RO) - 1


@pytest.mark.parametrize("bt", [False, True], ids=["B", "Bt"])
@pytest.mark.parametrize("nc,N,K", [(3, 128, 128), (2, 256, 256), (1, 256, 128)])
def test_grouped_launch(mock_dir, tmp_path, nc, N, K, bt):
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="launch", kernel=K_GEMM_FP8, nc=nc, N=N, K=K, ro=RO, unit_base=1 << 32, flags=3, bt=bt)],
                     env_extra={"COAST_GEMM_PAIR": "1"})
    r = res["ops"][0]
    assert r["rc"] == 0, r["err"]
    name = f"xmr_gemm_fp8_grp_inj0_nc{nc}"
    la = work(ev)
    assert [e["name"] for e in la] == ([] if bt else ["xmr_gemm_bt_u8"]) + ["xmr_mm_group_scan", name]
    assert len({e["stream"] for e in la}) == 1
    k = la[-1]
    a = args_of(k)
    assert (a.n_units, a.M, a.N, a.K, a.unit_base) == (R * N, G, N, K, 1 << 32)
    assert k["grid"] == min((R // 128 + G) * (N // 128), SMS) and (k["block"], k["smem"]) == (384, SMEM)
    allocs = [e for e in ev if e["op"] == "alloc"]
    # B^T scratch (G K N bytes) then the group block; with the caller's B^T the group block alone
    assert [e["bytes"] for e in allocs[-1:]] == [(0 if bt else G * K * N) + GRP_BYTES(G)]
    base = r["aux"] if bt else allocs[-1]["ptr"]
    # A is a 128-row placeholder over B^T that the scan rebases; B^T is the G stacked N x K matrices
    assert maps(ev) == [(base, 1, K, 128, 128, 128), (base, 1, K, G * N, 128, 128)]


OK = dict(kernel=K_GEMM_FP8, M=128, N=128, K=128)
REFUSALS = [
    ("k_64", dict(OK, K=64), UNSUPPORTED, "GEMM_FP8 tiles are 128x128x128: M,N must be multiples of 128 and K of 128"),
    ("n_64", dict(OK, N=64), UNSUPPORTED, "multiples of 128"),
    ("m_100", dict(OK, M=100), UNSUPPORTED, "multiples of 128"),
    ("grouped_k_192", dict(N=128, K=192, ro=[0, 128]), UNSUPPORTED, "GEMM_FP8 grouped tiles are 128 x 128 x 128"),
    ("grouped_n_100", dict(N=100, K=128, ro=[0, 128]), UNSUPPORTED, "multiple of 128"),
    ("misaligned_in", dict(OK, shift=[8, 0, 0]), BAD_ARG, "16-byte aligned"),
    ("misaligned_aux", dict(OK, shift=[0, 1, 0]), BAD_ARG, "16-byte aligned"),
    ("misaligned_out", dict(OK, shift=[0, 0, 4]), BAD_ARG, "16-byte aligned"),
    ("n_units", dict(OK, n=128 * 128 * 2), BAD_ARG, "n_units must be M*N"),
    ("no_b", dict(OK, K=0), BAD_ARG, "GEMM needs A (d_in), B (d_aux) and M,N,K"),
    ("batch_rows_2p31", dict(OK, batch=1 << 24, alloc=[16, 16, 16]), BAD_ARG, "batch*M and batch*N must be below 2^31"),
    ("batch_n_2p31", dict(M=256, N=2048, K=128, batch=1 << 20, alloc=[16, 16, 16]), BAD_ARG, "batch*M and batch*N must be below 2^31"),
    ("batch_n_2p31_bt", dict(M=256, N=2048, K=128, batch=1 << 20, alloc=[16, 16, 16], bt=True), BAD_ARG, "batch*N must be below 2^31"),
    ("groups_n_2p31", dict(N=2048, K=128, ro=[0, 128], M=1 << 20), BAD_ARG, "G*N must be below 2^31"),
    ("batched_on_crc16", dict(OK, kernel=K_CRC16, batch=2), BAD_ARG,
     "COAST_MM_BATCHED: batched products exist for MM_U32, GEMM_TF32 and GEMM_BF16 only, plus GEMM_FP8"),
    ("grouped_on_crc16", dict(N=128, K=128, ro=[0, 128], kernel=K_CRC16), BAD_ARG,
     "COAST_MM_GROUPED: grouped products exist for MM_U32, GEMM_TF32 and GEMM_BF16 only, plus GEMM_FP8"),
    ("bt_on_crc16", dict(OK, kernel=K_CRC16, bt=True), BAD_ARG, "a transposed B exists for MM_U32, GEMM_TF32 and GEMM_BF16 only, plus GEMM_FP8"),
    ("batched_and_grouped", dict(N=128, K=128, ro=[0, 128], mode=MM_GROUPED | MM_BATCHED), BAD_ARG, "COAST_MM_BATCHED"),
    ("id_9", dict(OK, kernel=9), BAD_ARG, "unknown kernel id 9"),
    ("id_11", dict(OK, kernel=11), BAD_ARG, "unknown kernel id 11"),
]


@pytest.mark.parametrize("case", REFUSALS, ids=[c[0] for c in REFUSALS])
def test_refusals_name_their_rule_and_launch_nothing(mock_dir, tmp_path, case):
    _, op, code, needle = case
    res, ev, _ = run(mock_dir, tmp_path, [{"op": "launch", "kernel": K_GEMM_FP8, **op}])
    r = res["ops"][0]
    assert r["rc"] == code and needle in r["err"], r
    assert not work(ev)


def test_unassigned_id_9_is_refused_by_the_host_call(mock_dir, tmp_path):
    res, ev, _ = run(mock_dir, tmp_path, [dict(OK, op="run_host", kernel=9)])
    assert res["ops"][0]["rc"] == UNSUPPORTED and not work(ev)


def test_store_vote_flags_warn_or_refuse(mock_dir, tmp_path):
    op = dict(op="launch", nc=3, flags=0x200, **OK)              # -storeDataSync
    res, ev, err = run(mock_dir, tmp_path, [op])
    assert res["ops"][0]["rc"] == 0 and "NOT honoured by the gemm_fp8 kernel" in err and len(work(ev)) == 2
    res, ev, _ = run(mock_dir, tmp_path, [op], env_extra={"COAST_STRICT_FLAGS": "1"})
    assert res["ops"][0]["rc"] == UNSUPPORTED and "gemm_fp8" in res["ops"][0]["err"] and not work(ev)


@pytest.mark.parametrize("bt", [False, True])
@pytest.mark.parametrize("nc,M,N,env", [(3, 128, 128, {}), (1, 256, 256, {}), (1, 128, 256, {"COAST_GEMM_PAIR": "0"}), (2, 256, 128, {})])
def test_a_batch_of_one_is_the_unbatched_launch(mock_dir, tmp_path, nc, M, N, env, bt):
    recs = []
    for extra in (dict(batch=1), {}):
        res, ev, _ = run(mock_dir, tmp_path, [dict(op="launch", kernel=K_GEMM_FP8, nc=nc, M=M, N=N, K=256, unit_base=77, flags=3, bt=bt, **extra)], env_extra=env)
        assert res["ops"][0]["rc"] == 0
        la = work(ev)
        a = args_of(la[-1])
        recs.append(([(e["name"], e["grid"], e["block"], e["smem"]) for e in la], [m[1:] for m in maps(ev)],
                     (a.n_units, a.unit_base, a.M, a.N, a.K, a.mode, a.flags, a.n_sites), [e["bytes"] for e in ev if e["op"] == "alloc"]))
    assert recs[0] == recs[1]


@pytest.mark.parametrize("pinned", [False, True])
def test_host_call_row_blocks_copy_one_byte_operands(mock_dir, tmp_path, pinned):
    M, N, K = 1024, 128, 128
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", kernel=K_GEMM_FP8, nc=3, M=M, N=N, K=K, pinned=pinned, unit_base=5)])
    r = res["ops"][0]
    assert r["rc"] == 0 and r["path"] == "row-blocks", r
    ups_a, ups_b = spans(ev, "h2d", r["host_in"], M * K), spans(ev, "h2d", r["host_aux"], K * N)
    downs = spans(ev, "d2h", r["host_out"], 4 * M * N)
    assert [u[:2] for u in ups_a] == [(i * 128 * K, 128 * K) for i in range(8)]
    assert [u[:2] for u in ups_b] == [(0, K * N)]                   # B goes up once
    assert [d[:2] for d in downs] == [(i * 128 * N * 4, 128 * N * 4) for i in range(8)]
    la = work(ev)
    assert [e["name"] for e in la] == ["xmr_gemm_bt_u8", "xmr_gemm_fp8_inj0_nc3"] * 8
    assert [(args_of(e).M, args_of(e).unit_base) for e in la[1::2]] == [(128, 5 + i * 128 * N) for i in range(8)]


@pytest.mark.parametrize("bt", [False, True])
@pytest.mark.parametrize("pinned", [False, True])
def test_host_call_whole_products_per_chunk(mock_dir, tmp_path, pinned, bt):
    M, N, K, batch = 128, 128, 256, 5
    ab, bb, cb = M * K, K * N, M * N * 4
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", kernel=K_GEMM_FP8, nc=2, M=M, N=N, K=K, batch=batch, pinned=pinned, bt=bt)],
                     env_extra={"COAST_HOST_CHUNK_BYTES": str(2 * (ab + bb + cb) + 100)})
    r = res["ops"][0]
    assert r["rc"] == 0, r
    chunks = [(0, 2), (2, 2), (4, 1)]
    assert [u[:2] for u in spans(ev, "h2d", r["host_in"], batch * ab)] == [(f * ab, n * ab) for f, n in chunks]
    assert [u[:2] for u in spans(ev, "h2d", r["host_aux"], batch * bb)] == [(f * bb, n * bb) for f, n in chunks]
    assert [d[:2] for d in spans(ev, "d2h", r["host_out"], batch * cb)] == [(f * cb, n * cb) for f, n in chunks]
    la = [e for e in work(ev) if e["name"] != "xmr_gemm_bt_u8"]
    assert [args_of(e).n_units for e in la] == [n * M * N for _, n in chunks]
    assert len(work(ev)) == len(chunks) * (1 if bt else 2)


@pytest.mark.parametrize("pinned", [False, True])
def test_host_call_groups_per_chunk(mock_dir, tmp_path, pinned):
    N, K, ro, budget = 128, 128, [7, 100, 228, 228, 500, 501], 90000
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", kernel=K_GEMM_FP8, nc=3, N=N, K=K, ro=ro, unit_base=1000, pinned=pinned)],
                     env_extra={"COAST_HOST_CHUNK_BYTES": str(budget)})
    r = res["ops"][0]
    assert r["rc"] == 0 and r["path"] == "groups", r
    chunks, f, G = [], 0, len(ro) - 1
    while f < G:                                                   # the schedule's rule with 1-byte A and B, 4-byte C
        e = f + 1
        while e < G and (ro[e + 1] - ro[f]) * (K + N * 4) + (e + 1 - f) * (K * N + 8) + 8 <= budget:
            e += 1
        chunks.append((f, e))
        f = e
    assert len(chunks) > 2
    ups_b, ups_r = spans(ev, "h2d", r["host_aux"], G * K * N), spans(ev, "h2d", r["host_rows"], 8 * (G + 1))
    assert [u[:2] for u in ups_b] == [(f * K * N, (e - f) * K * N) for f, e in chunks]
    assert [u[:2] for u in ups_r] == [(8 * f, 8 * (e - f + 1)) for f, e in chunks]
    with_rows = [(f, e) for f, e in chunks if ro[e] > ro[f]]
    assert [u[:2] for u in spans(ev, "h2d", r["host_in"], ro[-1] * K)] == [(ro[f] * K, (ro[e] - ro[f]) * K) for f, e in with_rows]
    assert [d[:2] for d in spans(ev, "d2h", r["host_out"], 4 * ro[-1] * N)] == [(4 * ro[f] * N, 4 * (ro[e] - ro[f]) * N) for f, e in with_rows]
    la = [e for e in work(ev) if "_grp_inj" in e["name"]]
    assert [(args_of(k).n_units, args_of(k).unit_base, args_of(k).M) for k in la] == \
        [((ro[e] - ro[f]) * N, 1000 + (ro[f] - ro[0]) * N, e - f) for f, e in with_rows]
    assert [e["name"] for e in work(ev) if "_grp_inj" not in e["name"]] == ["xmr_gemm_bt_u8", "xmr_mm_group_scan"] * len(with_rows)


# ------------------------------------------------------------------------------------------ the cubin's FP8 functions
def test_fp8_functions_run_the_e4m3_wgmma_and_the_pre_pass_none(built_lib):
    sass = sass_by_function()
    fns = sorted(f for f in sass if f.startswith("xmr_gemm_fp8"))
    assert len(fns) == 20
    for f in fns:
        assert re.search(r"QGMMA\.64x128x32\.F32\.E4M3\.E4M3", sass[f]), f
    assert "GMMA" not in sass["xmr_gemm_bt_u8"]


def twins(f):
    """the TF32 and BF16 kernels of the same variant, NC and injection"""
    m = re.fullmatch(r"xmr_gemm_fp8(p|n|)(_grp|)_inj(\d)_nc(\d)", f)
    v, grp, inj, nc = m.groups()
    if grp:
        v = "n" if nc == "1" else ""
        return f"xmr_gemm_tf32{v}_grp_inj{inj}_nc{nc}", f"xmr_gemm_bf16{v}_grp_inj{inj}_nc{nc}"
    return f"xmr_gemm_tf32{v}_nc{nc}_inj{inj}", f"xmr_gemm_bf16{v}_inj{inj}_nc{nc}"


def test_no_fp8_function_keeps_more_stack_than_its_twins(built_lib):
    """spills show as stack: an FP8 kernel holds the same 64-register accumulator fragments as BF16, so it may keep no more
    local memory than the TF32 or BF16 kernel of its variant"""
    res = res_usage()
    fns = sorted(f for f in res if f.startswith("xmr_gemm_fp8"))
    assert len(fns) == 20
    for f in fns:
        tf, bf = twins(f)
        assert res[f]["STACK"] <= max(res[tf]["STACK"], res[bf]["STACK"]), (f, res[f], res[tf], res[bf])
        assert res[f]["LOCAL"] <= max(res[tf]["LOCAL"], res[bf]["LOCAL"]), (f, res[f], res[tf], res[bf])
