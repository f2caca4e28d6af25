"""Host logic of COAST_K_GEMM_BF16 on a GPU-less box, against the mock driver (tests/mock_cuda/mock_cuda_bf16.c:
mock_cuda.c with 2-byte tensor-map elements).  Pinned here: the
kernel each shape gets (single CTA wide / narrow, CTA pair, grouped), grid and shared memory, both tensor maps (2-byte
elements; A rows x K in boxes of 64 k x 128 rows; B read in place as (batch K) rows x N in boxes of 64 columns x 64 k-rows,
for pairs too), that a single or batched launch allocates nothing and runs no pre-pass while a grouped launch allocates the
group block alone and runs the scan alone, every refusal with its message, that a batch of one is the unbatched launch, and
the bytes the host call copies per chunk (2-byte A and B, 4-byte C) for row blocks, whole products and groups."""
import json
import os
import subprocess
import sys

import pytest

from test_host_logic import ROOT, args_of

MM_GROUPED, MM_BATCHED = 0x40000, 0x20000
K_CRC16, K_GEMM_BF16 = 0, 8
BAD_ARG, UNSUPPORTED = -100003, -100004
SMS = 132
SMEM = 6 * (128 * 128 + 128 * 128) + 1024 + 256          # xmr_gemm_smem: the same bytes wide (4 stages of 48 KiB) and narrow
GRP_BYTES = lambda G: 128 + 4 * (G + 1)                  # noqa: E731  (xmr_mm_grp_bytes)


@pytest.fixture(scope="session")
def mock_dir(tmp_path_factory, built_lib):
    """the mock driver with bfloat16 tensor maps (mock_cuda_bf16.c includes mock_cuda.c)"""
    d = tmp_path_factory.mktemp("mockcuda_bf16")
    subprocess.run(["gcc", "-O1", "-shared", "-fPIC", "-Wall", "-I/usr/local/cuda/include", "-o", str(d / "libcuda.so.1"),
                    os.path.join(ROOT, "tests", "mock_cuda", "mock_cuda_bf16.c")], check=True)
    return d


def run(mock_dir, tmp_path, ops, env_extra=None):
    log = tmp_path / "mock.log"
    if log.exists():
        log.unlink()
    env = dict(os.environ, LD_LIBRARY_PATH=f"{mock_dir}:" + os.environ.get("LD_LIBRARY_PATH", ""), MOCK_CUDA_LOG=str(log))
    for k in ("COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT", "COAST_HOST_CHUNK_BYTES",
              "COAST_HOST_PATH", "COAST_STRICT_FLAGS"):
        env.pop(k, None)
    env.update(env_extra or {})
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "mock_cuda", "gemm_bf16_child.py"), json.dumps({"ops": ops})],
                         capture_output=True, text=True, env=env, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    events = [json.loads(ln) for ln in open(log)] if log.exists() else []
    assert not [e for e in events if e["op"] == "error"], [e for e in events if e["op"] == "error"]
    assert events[-1] == {"op": "exit", "live_allocations": 0}
    return json.loads(res.stdout.strip().splitlines()[-1]), events, res.stderr


def work(ev):
    return [e for e in ev if e["op"] == "launch" and e["name"] != "xmr_counters_reset"]


def tmaps(ev):
    return [(t["elem"], t["dim0"], t["dim1"], t["box0"], t["box1"], t["box_bytes"]) for t in ev if t["op"] == "tmap16"]


# (id, nc, M, N, K, batch or None, environment, kernel, grid)
LAUNCHES = [
    ("single_nc3", 3, 512, 512, 128, None, {}, "xmr_gemm_bf16_inj0_nc3", 16),
    ("narrow_nc1", 1, 512, 384, 64, None, {}, "xmr_gemm_bf16n_inj0_nc1", 12),          # N % 256 != 0
    ("wide_nc1", 1, 384, 512, 64, None, {}, "xmr_gemm_bf16_inj0_nc1", 6),              # M % 256 != 0: no pair tile
    ("pair_nc1", 1, 512, 512, 64, None, {}, "xmr_gemm_bf16p_inj0_nc1", 8),             # 256 x 256 pair tiles: 4 pairs
    ("pair_nc2", 2, 512, 384, 64, None, {}, "xmr_gemm_bf16p_inj0_nc2", 12),
    ("pair_nc3", 3, 512, 512, 64, None, {"COAST_GEMM_PAIR": "1"}, "xmr_gemm_bf16p_inj0_nc3", 16),
    ("single_nc2", 2, 512, 512, 64, None, {"COAST_GEMM_PAIR": "0"}, "xmr_gemm_bf16_inj0_nc2", 16),
    ("batched_nc3", 3, 128, 128, 64, 300, {}, "xmr_gemm_bf16_inj0_nc3", SMS),
    ("batched_pair_nc2", 2, 256, 128, 192, 3, {}, "xmr_gemm_bf16p_inj0_nc2", 6),
    ("batched_wide_nc1", 1, 128, 256, 64, 5, {}, "xmr_gemm_bf16_inj0_nc1", 5),         # a pair tile would straddle two products
]


@pytest.mark.parametrize("case", LAUNCHES, ids=[c[0] for c in LAUNCHES])
def test_launch_records(mock_dir, tmp_path, case):
    _, nc, M, N, K, batch, env, name, grid = case
    op = dict(op="launch", nc=nc, M=M, N=N, K=K, unit_base=1 << 32, flags=3)
    if batch:
        op["batch"] = batch
    b = batch or 1
    res, ev, _ = run(mock_dir, tmp_path, [op], env_extra=env)
    r = res["ops"][0]
    assert r["rc"] == 0, r["err"]
    la = work(ev)
    assert [e["name"] for e in la] == [name]                       # no pre-pass of any kind
    k = la[0]
    assert (k["grid"], k["block"], k["smem"]) == (grid, 384, SMEM) and (grid % 2 == 0 or "bf16p" not in name)
    a = args_of(k)
    assert (a.n_units, a.M, a.N, a.K, a.unit_base, a.n_sites) == (b * M * N, M, N, K, 1 << 32, 1)
    assert a.mode & (MM_GROUPED | MM_BATCHED) == 0 and (a.inp, a.aux, a.out) == (r["in"], r["aux"], r["out"])
    # A: (batch M) rows of K, boxes of one 128-byte k-block x 128 rows; B in place: (batch K) rows of N, boxes of 64 columns x 64 k-rows
    assert tmaps(ev) == [(2, K, b * M, 64, 128, 16384), (2, N, b * K, 64, 64, 8192)]
    allocs = [e for e in ev if e["op"] == "alloc"]
    # nothing is allocated between the caller's three buffers and the launch: no scratch
    three = [e for e in allocs if not e["host"]][-3:]
    assert ev.index(three[-1]) < ev.index(k) and not [e for e in ev[ev.index(three[-1]) + 1:ev.index(k)] if e["op"] == "alloc"]


RO = [3, 3, 100, 101, 101, 500, 700]
R, G = RO[-1] - RO[0], len(RO) - 1


@pytest.mark.parametrize("nc,N,K,name", [(3, 128, 64, "xmr_gemm_bf16_grp_inj0_nc3"), (2, 256, 128, "xmr_gemm_bf16_grp_inj0_nc2"),
                                         (1, 256, 64, "xmr_gemm_bf16n_grp_inj0_nc1")])
def test_grouped_launch_runs_the_scan_alone_over_the_group_block_alone(mock_dir, tmp_path, nc, N, K, name):
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="launch", nc=nc, N=N, K=K, ro=RO, unit_base=1 << 32, flags=3)],
                     env_extra={"COAST_GEMM_PAIR": "1"})
    r = res["ops"][0]
    assert r["rc"] == 0, r["err"]
    la = work(ev)
    assert [e["name"] for e in la] == ["xmr_mm_group_scan", name] and len({e["stream"] for e in la}) == 1
    assert int.from_bytes(bytes.fromhex(la[0]["arg0"]), "little") == r["rows"]      # the caller's table, read on the device
    k = la[-1]
    a = args_of(k)
    assert (a.n_units, a.M, a.N, a.K, a.unit_base) == (R * N, G, N, K, 1 << 32)
    assert k["grid"] == min((R // 128 + G) * (N // 128), SMS) and (k["block"], k["smem"]) == (384, SMEM)
    # A's map is a 128-row placeholder the scan rebases; B is the G stacked matrices in place
    assert tmaps(ev) == [(2, K, 128, 64, 128, 16384), (2, N, G * K, 64, 64, 8192)]
    allocs = [e for e in ev if e["op"] == "alloc"]
    assert [e["bytes"] for e in allocs[-2:]] == [8 * len(RO), GRP_BYTES(G)]
    assert {"op": "free", "id": allocs[-1]["id"]} in ev[ev.index(k):]


OK = dict(M=128, N=128, K=64)
REFUSALS = [
    ("k_32", dict(OK, K=32), UNSUPPORTED, "K of 64"),
    ("n_64", dict(OK, N=64), UNSUPPORTED, "multiples of 128"),
    ("m_100", dict(OK, M=100), UNSUPPORTED, "multiples of 128"),
    ("grouped_k_96", dict(N=128, K=96, ro=[0, 128]), UNSUPPORTED, "K of 64"),
    ("grouped_n_100", dict(N=100, K=64, ro=[0, 128]), UNSUPPORTED, "multiple of 128"),
    ("misaligned_in", dict(OK, shift=[8, 0, 0]), BAD_ARG, "16-byte aligned"),
    ("misaligned_aux", dict(OK, shift=[0, 2, 0]), BAD_ARG, "16-byte aligned"),
    ("misaligned_out", dict(OK, shift=[0, 0, 4]), BAD_ARG, "16-byte aligned"),
    ("n_units", dict(OK, n=128 * 128 * 2), BAD_ARG, "n_units must be M*N"),
    ("batch_rows_2p31", dict(OK, batch=1 << 24, alloc=[16, 16, 16]), BAD_ARG, "batch*M and batch*K must be below 2^31"),
    ("batch_k_2p31", dict(M=128, N=128, K=256, batch=1 << 23, alloc=[16, 16, 16]), BAD_ARG, "batch*M and batch*K must be below 2^31"),
    ("groups_k_2p31", dict(N=128, K=2048, ro=[0, 128], M=1 << 20), BAD_ARG, "G*K must be below 2^31"),
    ("batched_on_crc16", dict(OK, kernel=K_CRC16, batch=2), BAD_ARG, "COAST_MM_BATCHED: batched products exist for MM_U32, GEMM_TF32 and GEMM_BF16"),
    ("grouped_on_crc16", dict(N=128, K=64, ro=[0, 128], kernel=K_CRC16), BAD_ARG, "COAST_MM_GROUPED: grouped products exist for MM_U32, GEMM_TF32 and GEMM_BF16"),
    ("batched_and_grouped", dict(N=128, K=64, ro=[0, 128], mode=MM_GROUPED | MM_BATCHED), BAD_ARG, "COAST_MM_BATCHED"),
]


@pytest.mark.parametrize("case", REFUSALS, ids=[c[0] for c in REFUSALS])
def test_refusals_name_their_rule_and_launch_nothing(mock_dir, tmp_path, case):
    _, op, code, needle = case
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="launch", **op)])
    r = res["ops"][0]
    assert r["rc"] == code and needle in r["err"], r
    assert not work(ev)


def test_store_vote_flags_warn_or_refuse(mock_dir, tmp_path):
    """in-loop store votes are not built for the GEMMs: a warning names the kernel, COAST_STRICT_FLAGS=1 makes it an error"""
    op = dict(op="launch", nc=3, flags=0x200, **OK)              # -storeDataSync
    res, ev, err = run(mock_dir, tmp_path, [op])
    assert res["ops"][0]["rc"] == 0 and "NOT honoured by the gemm_bf16 kernel" in err and len(work(ev)) == 1
    res, ev, _ = run(mock_dir, tmp_path, [op], env_extra={"COAST_STRICT_FLAGS": "1"})
    assert res["ops"][0]["rc"] == UNSUPPORTED and "gemm_bf16" in res["ops"][0]["err"] and not work(ev)


@pytest.mark.parametrize("nc,M,N,env", [(3, 128, 128, {}), (1, 256, 256, {}), (1, 128, 256, {"COAST_GEMM_PAIR": "0"}), (2, 256, 128, {})])
def test_a_batch_of_one_is_the_unbatched_launch(mock_dir, tmp_path, nc, M, N, env):
    recs = []
    for extra in (dict(batch=1), {}):
        res, ev, _ = run(mock_dir, tmp_path, [dict(op="launch", nc=nc, M=M, N=N, K=128, unit_base=77, flags=3, **extra)], env_extra=env)
        assert res["ops"][0]["rc"] == 0
        la = work(ev)
        a = args_of(la[0])
        recs.append(([(e["name"], e["grid"], e["block"], e["smem"]) for e in la], tmaps(ev),
                     (a.n_units, a.unit_base, a.M, a.N, a.K, a.mode, a.flags, a.n_sites), [e["bytes"] for e in ev if e["op"] == "alloc"]))
    assert recs[0] == recs[1]


def spans(ev, op, base, size):
    return [(e["host"] - base, e["bytes"], e["stream"]) for e in ev if e["op"] == op and base <= e["host"] < base + size]


@pytest.mark.parametrize("pinned", [False, True])
def test_host_call_row_blocks_copy_two_byte_operands(mock_dir, tmp_path, pinned):
    M, N, K = 1024, 128, 64
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", nc=3, M=M, N=N, K=K, pinned=pinned, unit_base=5)])
    r = res["ops"][0]
    assert r["rc"] == 0 and r["path"] == "row-blocks", r
    ups_a, ups_b = spans(ev, "h2d", r["host_in"], 2 * M * K), spans(ev, "h2d", r["host_aux"], 2 * K * N)
    downs = spans(ev, "d2h", r["host_out"], 4 * M * N)
    assert [u[:2] for u in ups_a] == [(i * 128 * K * 2, 128 * K * 2) for i in range(8)]
    assert [u[:2] for u in ups_b] == [(0, K * N * 2)]               # B goes up once
    assert [d[:2] for d in downs] == [(i * 128 * N * 4, 128 * N * 4) for i in range(8)]
    la = work(ev)
    assert [e["name"] for e in la] == ["xmr_gemm_bf16_inj0_nc3"] * 8
    assert [(args_of(e).M, args_of(e).unit_base) for e in la] == [(128, 5 + i * 128 * N) for i in range(8)]


@pytest.mark.parametrize("pinned", [False, True])
def test_host_call_whole_products_per_chunk(mock_dir, tmp_path, pinned):
    M, N, K, batch = 128, 128, 64, 5
    ab, bb, cb = M * K * 2, K * N * 2, M * N * 4
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", nc=2, M=M, N=N, K=K, batch=batch, pinned=pinned)],
                     env_extra={"COAST_HOST_CHUNK_BYTES": str(2 * (ab + bb + cb) + 100)})
    r = res["ops"][0]
    assert r["rc"] == 0, r
    chunks = [(0, 2), (2, 2), (4, 1)]
    assert [u[:2] for u in spans(ev, "h2d", r["host_in"], batch * ab)] == [(f * ab, n * ab) for f, n in chunks]
    assert [u[:2] for u in spans(ev, "h2d", r["host_aux"], batch * bb)] == [(f * bb, n * bb) for f, n in chunks]
    assert [d[:2] for d in spans(ev, "d2h", r["host_out"], batch * cb)] == [(f * cb, n * cb) for f, n in chunks]
    assert [args_of(e).n_units for e in work(ev)] == [n * M * N for _, n in chunks]


@pytest.mark.parametrize("pinned", [False, True])
def test_host_call_groups_per_chunk(mock_dir, tmp_path, pinned):
    N, K, ro, budget = 128, 64, [7, 100, 228, 228, 500, 501], 70000
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", nc=3, N=N, K=K, ro=ro, unit_base=1000, pinned=pinned)],
                     env_extra={"COAST_HOST_CHUNK_BYTES": str(budget)})
    r = res["ops"][0]
    assert r["rc"] == 0 and r["path"] == "groups", r
    chunks, f, G = [], 0, len(ro) - 1
    while f < G:                                                   # the schedule's rule with 2-byte A and B, 4-byte C
        e = f + 1
        while e < G and (ro[e + 1] - ro[f]) * (K * 2 + N * 4) + (e + 1 - f) * (K * N * 2 + 8) + 8 <= budget:
            e += 1
        chunks.append((f, e))
        f = e
    assert len(chunks) > 2
    ups_b, ups_r = spans(ev, "h2d", r["host_aux"], 2 * G * K * N), spans(ev, "h2d", r["host_rows"], 8 * (G + 1))
    assert [u[:2] for u in ups_b] == [(2 * f * K * N, 2 * (e - f) * K * N) for f, e in chunks]
    assert [u[:2] for u in ups_r] == [(8 * f, 8 * (e - f + 1)) for f, e in chunks]
    with_rows = [(f, e) for f, e in chunks if ro[e] > ro[f]]
    assert [u[:2] for u in spans(ev, "h2d", r["host_in"], 2 * ro[-1] * K)] == [(2 * ro[f] * K, 2 * (ro[e] - ro[f]) * K) for f, e in with_rows]
    assert [d[:2] for d in spans(ev, "d2h", r["host_out"], 4 * ro[-1] * N)] == [(4 * ro[f] * N, 4 * (ro[e] - ro[f]) * N) for f, e in with_rows]
    la = [e for e in work(ev) if "_grp_inj" in e["name"]]
    assert [(args_of(k).n_units, args_of(k).unit_base, args_of(k).M) for k in la] == \
        [((ro[e] - ro[f]) * N, 1000 + (ro[f] - ro[0]) * N, e - f) for f, e in with_rows]
    assert [e["name"] for e in work(ev) if "_grp_inj" not in e["name"]] == ["xmr_mm_group_scan"] * len(with_rows)
