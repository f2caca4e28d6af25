"""Host logic of grouped matmuls (COAST_MM_GROUPED with COAST_K_MM_U32 and COAST_K_GEMM_TF32) on a GPU-less box, against the
mock driver (tests/mock_cuda/mock_cuda.c) through tests/mock_cuda/mm_child.py.  A grouped launch is G products sharing N and K with a row count each, given by
G + 1 row offsets (d_rows).  Pinned here: the pre-passes and kernel each path selects, that the shape rules apply to N and K
only, the tensor maps (R rows of A limb planes, G*N rows of B^T, TF32's A map encoded over 128 rows for the device to rebase),
the scratch bytes (operands, then the group block), the grid bound (R / tile height + G) * column tiles, that an empty product
adds no tiles to the bound's rows, every refusal, and the host call's chunks of whole products: an oversized product alone,
empty products, the offset slices uploaded unchanged, d_in / d_out biases and unit_base per chunk."""
import pytest

from mock_run import (BAD_ARG, GRP_BYTES, K_CRC16, K_GEMM_TF32, K_MM_U32, MM_BATCHED, MM_GROUPED, SMS, UNIT_OFFSETS,  # noqa: F401
                      UNSUPPORTED, arg0_ptr, args_of, mock_dir, run, spans, work)

RO = [3, 3, 100, 101, 101, 500, 700]             # from row 3; empty products, a one-row product
R, G = RO[-1] - RO[0], len(RO) - 1

# (id, kernel, nc, N, K, env, launches in order, kernel TM (0: plain), column tiles, tensor maps (dim0, dim1), scratch bytes)
PATHS = [
    ("tc_nc3", K_MM_U32, 3, 64, 128, {}, ["xmr_mm_grp_split_a", "xmr_mm_split_bt", "xmr_mm_group_scan", "xmr_mm_u32_tc_grp_inj0_nc3"],
     128, 2, [(128, R), (128, G * 64)], (R * 128 + G * 128 * 64) * 4 + GRP_BYTES(G)),
    ("tc_nc1", K_MM_U32, 1, 64, 128, {}, ["xmr_mm_grp_split_a", "xmr_mm_split_bt", "xmr_mm_group_scan", "xmr_mm_u32_tc_grp_inj0_nc1"],
     128, 1, [(128, R), (128, G * 64)], (R * 128 + G * 128 * 64) * 4 + GRP_BYTES(G)),
    ("tiled_nc2", K_MM_U32, 2, 128, 16, {}, ["xmr_mm_group_scan", "xmr_mm_u32_tiled_grp_inj0_nc2"], 64, 1, [], GRP_BYTES(G)),
    ("plain_nc3", K_MM_U32, 3, 9, 9, {}, ["xmr_mm_u32_grp_inj0_nc3"], 0, 0, [], None),
    ("forced_naive", K_MM_U32, 2, 128, 128, {"COAST_MM_PATH": "naive"}, ["xmr_mm_u32_grp_inj0_nc2"], 0, 0, [], None),
    ("tf32_nc3", K_GEMM_TF32, 3, 128, 64, {}, ["xmr_gemm_bt", "xmr_mm_group_scan", "xmr_gemm_tf32_grp_inj0_nc3"], 128, 1,
     [(64, 128), (64, G * 128)], G * 64 * 128 * 4 + GRP_BYTES(G)),
    ("tf32_nc2", K_GEMM_TF32, 2, 256, 32, {"COAST_GEMM_PAIR": "1"}, ["xmr_gemm_bt", "xmr_mm_group_scan", "xmr_gemm_tf32_grp_inj0_nc2"],
     128, 2, [(32, 128), (32, G * 256)], G * 32 * 256 * 4 + GRP_BYTES(G)),
    ("tf32_nc1", K_GEMM_TF32, 1, 256, 32, {}, ["xmr_gemm_bt", "xmr_mm_group_scan", "xmr_gemm_tf32n_grp_inj0_nc1"], 128, 2,
     [(32, 128), (32, G * 256)], G * 32 * 256 * 4 + GRP_BYTES(G)),
]


@pytest.mark.parametrize("case", PATHS, ids=[c[0] for c in PATHS])
def test_each_path_runs_its_prepasses_and_kernel(mock_dir, tmp_path, case):
    """rows of any count on every path: pre-passes, kernel, maps, scratch and the grid bound; the argument block carries
    M = G and n_units = R*N without the mode bit"""
    _, kernel, nc, N, K, env, want, tm, tiles_n, maps, scratch = case
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="launch", kernel=kernel, nc=nc, N=N, K=K, ro=RO, unit_base=1 << 32, flags=3)],
                     env_extra=env)
    r = res["ops"][0]
    assert r["rc"] == 0, r["err"]
    la = work(ev)
    assert [e["name"] for e in la] == want and len({e["stream"] for e in la}) == 1
    k = la[-1]
    a = args_of(k)
    assert (a.n_units, a.M, a.N, a.K, a.unit_base) == (R * N, G, N, K, 1 << 32)
    assert a.mode & (MM_GROUPED | MM_BATCHED) == 0
    assert a.inp == r["in"] and a.out == r["out"] and a.aux == r["aux"]
    for e in la[:-1]:
        if e["name"] in ("xmr_mm_grp_split_a", "xmr_mm_group_scan"):
            assert arg0_ptr(e) == r["rows"]                             # the caller's table, read on the device
    if tm:
        bound = (R // tm + G) * tiles_n
        assert k["grid"] == (min(bound, SMS) if k["block"] == 384 else bound)
    assert [(t["dim0"], t["dim1"]) for t in ev if t["op"] == "tmap"] == maps
    allocs = [e for e in ev if e["op"] == "alloc"]
    if scratch is None:
        assert allocs[-1]["bytes"] == 8 * len(RO)                     # the caller's offsets were the last allocation
    else:
        assert allocs[-1]["bytes"] == scratch
        assert {"op": "free", "id": allocs[-1]["id"]} in ev[ev.index(k):]


def test_empty_products_add_no_rows_to_the_grid_bound(mock_dir, tmp_path):
    """the grid bound counts R / TM + G row tiles: the same rows with or without empty products around them differ by G only"""
    ro1, ro2 = [0, 640], [0, 0, 0, 640, 640]
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="launch", kernel=K_MM_U32, nc=2, N=128, K=16, ro=ro) for ro in (ro1, ro2)])
    assert [o["rc"] for o in res["ops"]] == [0, 0]
    grids = [e["grid"] for e in work(ev) if e["name"].startswith("xmr_mm_u32_tiled_grp")]
    assert grids == [640 // 64 + 1, 640 // 64 + 4]


REFUSALS = [
    ("other_kernel", dict(kernel=K_CRC16, N=8, K=8, ro=[0, 8]), BAD_ARG, "COAST_MM_GROUPED"),
    ("with_batched", dict(N=8, K=8, ro=[0, 8], mode=MM_GROUPED | MM_BATCHED), BAD_ARG, "COAST_MM_BATCHED"),
    ("with_offsets", dict(N=8, K=8, ro=[0, 8], mode=MM_GROUPED | UNIT_OFFSETS), BAD_ARG, "COAST_UNIT_OFFSETS"),
    ("zero_groups", dict(N=8, K=8, ro=[0, 8], M=0), BAD_ARG, "product count"),
    ("too_many_groups", dict(N=8, K=8, ro=[0, 8], M=(1 << 20) + 1), BAD_ARG, "product count"),
    ("not_a_multiple", dict(N=8, K=8, ro=[0, 8], n=8 * 8 + 3), BAD_ARG, "multiple of N"),
    ("rows_2p31", dict(N=1, K=1, ro=[0, 8], n=1 << 31), BAD_ARG, "below 2^31"),
    ("gn_2p31", dict(N=1 << 16, K=1, ro=[0, 1], M=1 << 15, n=1 << 16), BAD_ARG, "below 2^31"),
    ("null_rows", dict(N=8, K=8, M=1, n=64, mode=MM_GROUPED), BAD_ARG, "d_rows"),        # no ro: d_rows stays null
]
# the host call's shape rule is its first chunk's launch: after that chunk's uploads
LAUNCH_ONLY = [("tf32_shape", dict(kernel=K_GEMM_TF32, N=100, K=64, ro=[0, 128]), UNSUPPORTED, "multiple of 128"),
               ("misaligned_rows", dict(N=8, K=8, ro=[0, 8, 8], rows_shift=4), BAD_ARG, "d_rows")]
HOST_ONLY = [("decreasing", dict(N=8, K=8, ro=[0, 8, 4, 12]), BAD_ARG, "must not decrease"),
             ("short_span", dict(N=8, K=8, ro=[0, 8, 12], n=8 * 16), BAD_ARG, "n_units / N")]
CALLS = [("launch", c) for c in REFUSALS + LAUNCH_ONLY] + [("run_host", c) for c in REFUSALS + HOST_ONLY]


@pytest.mark.parametrize("call,case", CALLS, ids=[f"{call}-{c[0]}" for call, c in CALLS])
def test_refusals_fail_loudly_before_any_work(mock_dir, tmp_path, call, case):
    _, op, code, needle = case
    res, ev, _ = run(mock_dir, tmp_path, [{"op": call, "kernel": K_MM_U32, **op}])
    r = res["ops"][0]
    assert r["rc"] == code and needle in r["err"], r
    assert not work(ev)
    if call == "run_host":
        assert not [e for e in ev if e["op"] in ("h2d", "d2h")]


def chunks_of(ro, N, K, budget):
    """the schedule's rule: the longest run of whole products whose A rows, B, C rows and offsets fit the budget, at least one"""
    out, f, G = [], 0, len(ro) - 1
    while f < G:
        e = f + 1
        while e < G and (ro[e + 1] - ro[f]) * (K + N) * 4 + (e + 1 - f) * (K * N * 4 + 8) + 8 <= budget:
            e += 1
        out.append((f, e))
        f = e
    return out


@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("kernel,N,K,ro,budget", [
    (K_MM_U32, 64, 128, [2, 2, 40, 41, 300, 300, 330, 800, 805, 805], 120000),    # an oversized product alone, empty products
    (K_MM_U32, 9, 9, [0, 5, 5, 17, 30], 0),                                        # default budget: one chunk
    (K_GEMM_TF32, 128, 32, [7, 100, 228, 228, 500, 501], 70000),
])
def test_host_call_chunks_are_whole_products(mock_dir, tmp_path, kernel, N, K, ro, budget, pinned):
    env = {"COAST_HOST_CHUNK_BYTES": str(budget)} if budget else {}
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", kernel=kernel, nc=3, N=N, K=K, ro=ro, unit_base=1000, pinned=pinned)],
                     env_extra=env)
    r = res["ops"][0]
    assert r["rc"] == 0 and r["path"] == "groups", r
    G = len(ro) - 1
    chunks = chunks_of(ro, N, K, budget or 16 << 20)
    assert len(chunks) > (2 if budget else 0) or not budget
    ups_a = spans(ev, "h2d", r["host_in"], 4 * ro[-1] * K)
    ups_b = spans(ev, "h2d", r["host_aux"], 4 * G * K * N)
    ups_r = spans(ev, "h2d", r["host_rows"], 8 * (G + 1))
    downs = spans(ev, "d2h", r["host_out"], 4 * ro[-1] * N)
    la = [e for e in work(ev) if "_grp_inj" in e["name"]]
    assert len(ups_r) == len(ups_b) == len(chunks)
    rows_chunks = [(f, e) for f, e in chunks if ro[e] > ro[f]]
    assert len(ups_a) == len(downs) == len(rows_chunks) == len(la)       # a chunk of empty products launches nothing
    for (f, e), ur, ub in zip(chunks, ups_r, ups_b):
        assert ur[:2] == (8 * f, 8 * (e - f + 1)) and ub[:2] == (4 * f * K * N, 4 * (e - f) * K * N)   # offsets unchanged
    slots = {}
    for (f, e), ua, dc, k in zip(rows_chunks, ups_a, downs, la):
        rows = ro[e] - ro[f]
        assert ua[:2] == (4 * ro[f] * K, 4 * rows * K) and dc[:2] == (4 * ro[f] * N, 4 * rows * N)
        a = args_of(k)
        assert (a.n_units, a.unit_base, a.M, a.N, a.K) == (rows * N, 1000 + (ro[f] - ro[0]) * N, e - f, N, K)
        assert ua[2] == dc[2] == k["stream"] and ua[3] == dc[3] == 0
        # d_in / d_out are the slot buffers biased by ro[first] rows: un-biased, every chunk of a stream sees the same slot
        slots.setdefault(k["stream"], set()).add(((a.inp + 4 * ro[f] * K) % (1 << 64), (a.out + 4 * ro[f] * N) % (1 << 64)))
    assert all(len(v) == 1 for v in slots.values()), slots
