"""Host logic of COAST_MM_B_TRANSPOSED on a GPU-less box, against the mock driver (tests/mock_cuda/mock_cuda_bt.c: mock_cuda.c
with 2-byte tensor-map elements and the start of every map logged).  Every launch form of every matmul path is run with and
without the bit and the two records are compared.  Pinned here: the kernel the bit selects, with the grid, block and shared
memory of the B launch; that GEMM_TF32 runs no transposing pre-pass and allocates no B^T scratch (grouped: the group block and
the scan alone); that the limb path splits B^T with the streaming split of A into the same planes; that B's map lies on the
caller's d_aux as (batch N) or (G N) rows of K with the per-kernel box; every refusal; and the bytes a host call copies."""
import json
import os
import subprocess
import sys

import pytest

from test_host_logic import ROOT, args_of

MM_GROUPED, MM_BATCHED, BT = 0x40000, 0x20000, 0x80000
K_CRC16, K_SHA256, K_AES128, K_MM_U32, K_GEMM_TF32, K_QSORT, K_CHSTONE_SHA, K_CHSTONE_AES, K_GEMM_BF16 = range(9)
BAD_ARG = -100003
PREPASSES = ("xmr_gemm_bt", "xmr_mm_split_a", "xmr_mm_split_bt", "xmr_mm_grp_split_a", "xmr_mm_group_scan")
GRP_BYTES = lambda G: 128 + 4 * (G + 1)                  # noqa: E731  (xmr_mm_grp_bytes)
KNOBS = ("COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT", "COAST_HOST_CHUNK_BYTES",
         "COAST_HOST_PATH", "COAST_STRICT_FLAGS", "COAST_MM_PATH")


@pytest.fixture(scope="session")
def mock_dir(tmp_path_factory, built_lib):
    d = tmp_path_factory.mktemp("mockcuda_bt")
    subprocess.run(["gcc", "-O1", "-shared", "-fPIC", "-Wall", "-I/usr/local/cuda/include", "-o", str(d / "libcuda.so.1"),
                    os.path.join(ROOT, "tests", "mock_cuda", "mock_cuda_bt.c")], check=True)
    return d


def run(mock_dir, tmp_path, ops, env_extra=None, driver_errors=False):
    log = tmp_path / "mock.log"
    if log.exists():
        log.unlink()
    env = dict(os.environ, LD_LIBRARY_PATH=f"{mock_dir}:" + os.environ.get("LD_LIBRARY_PATH", ""), MOCK_CUDA_LOG=str(log))
    for k in KNOBS:
        env.pop(k, None)
    env.update(env_extra or {})
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "mock_cuda", "mm_bt_child.py"), json.dumps({"ops": ops})],
                         capture_output=True, text=True, env=env, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    events = [json.loads(ln) for ln in open(log)] if log.exists() else []
    if not driver_errors:
        assert not [e for e in events if e["op"] == "error"], [e for e in events if e["op"] == "error"]
    assert events[-1] == {"op": "exit", "live_allocations": 0}
    return json.loads(res.stdout.strip().splitlines()[-1]), events


def work(ev):
    return [e for e in ev if e["op"] == "launch" and e["name"] != "xmr_counters_reset"]


def maps(ev):
    """(start, element bytes, dim0, dim1, box0, box1) of every tensor map, in encoding order"""
    out = []
    for i, e in enumerate(ev):
        if e["op"] == "tmap_at":
            t = ev[i + 1]
            assert t["op"] in ("tmap", "tmap16")
            out.append((e["addr"], t["elem"], t["dim0"], t["dim1"], t["box0"], t["box1"]))
    return out


def scratch(ev, sizes):
    """bytes of every allocation after the caller's buffers (sizes, in order) and before the matmul kernel"""
    allocs = [(i, e["bytes"]) for i, e in enumerate(ev) if e["op"] == "alloc" and not e["host"]]
    for j in range(len(allocs) - len(sizes) + 1):
        if [b for _, b in allocs[j:j + len(sizes)]] == sizes:
            k = ev.index(work(ev)[-1])
            return [b for i, b in allocs[j + len(sizes):] if i < k]
    raise AssertionError("the caller's buffers are not in the log")


def arg0_ptr(launch):
    return int.from_bytes(bytes.fromhex(launch["arg0"]), "little")


RO = [3, 3, 100, 101, 101, 500, 700]
G, R = len(RO) - 1, RO[-1] - RO[0]

# (id, op, environment, the kernel with the bit)
LAUNCHES = [
    ("limb_single_nc3", dict(kernel=K_MM_U32, nc=3, M=256, N=64, K=256), {}, "xmr_mm_u32_tc_nc3_inj0"),
    ("limb_single_inj1_nc1", dict(kernel=K_MM_U32, nc=1, M=128, N=128, K=128, p=0.3), {}, "xmr_mm_u32_tc_bt_inj1_nc1"),
    ("limb_batched_inj1_nc2", dict(kernel=K_MM_U32, nc=2, M=128, N=64, K=128, batch=3, p=0.3), {}, "xmr_mm_u32_tc_bt_inj1_nc2"),
    ("limb_grouped_nc2", dict(kernel=K_MM_U32, nc=2, N=64, K=128, ro=RO), {}, "xmr_mm_u32_tc_grp_inj0_nc2"),
    ("limb_grouped_inj1_nc3", dict(kernel=K_MM_U32, nc=3, N=64, K=128, ro=RO, p=0.3), {}, "xmr_mm_u32_tc_bt_grp_inj1_nc3"),
    ("tiled_single_nc3", dict(kernel=K_MM_U32, nc=3, M=128, N=256, K=32), {"COAST_MM_PATH": "tiled"}, "xmr_mm_u32_tiled_bt_inj0_nc3"),
    ("tiled_batched_inj1_nc2", dict(kernel=K_MM_U32, nc=2, M=64, N=128, K=48, batch=4, p=0.3), {}, "xmr_mm_u32_tiled_bt_inj1_nc2"),
    ("tiled_grouped_inj1_nc1", dict(kernel=K_MM_U32, nc=1, N=128, K=16, ro=RO, p=0.3), {"COAST_MM_PATH": "tiled"},
     "xmr_mm_u32_tiled_bt_grp_inj1_nc1"),
    ("plain_single_nc3", dict(kernel=K_MM_U32, nc=3, M=9, N=9, K=9), {}, "xmr_mm_u32_bt_inj0_nc3"),
    ("plain_store_votes_nc3", dict(kernel=K_MM_U32, nc=3, M=128, N=128, K=128, flags=0x7), {}, "xmr_mm_u32_bt_inj0_nc3"),
    ("plain_batched_inj1_nc2", dict(kernel=K_MM_U32, nc=2, M=64, N=128, K=16, batch=2, p=0.3), {"COAST_MM_PATH": "naive"},
     "xmr_mm_u32_bt_inj1_nc2"),
    ("plain_grouped_inj1_nc3", dict(kernel=K_MM_U32, nc=3, N=9, K=7, ro=RO, p=0.3), {}, "xmr_mm_u32_bt_grp_inj1_nc3"),
    ("tf32_single_nc3", dict(kernel=K_GEMM_TF32, nc=3, M=512, N=512, K=128), {}, "xmr_gemm_tf32_nc3_inj0"),
    ("tf32_narrow_nc1", dict(kernel=K_GEMM_TF32, nc=1, M=512, N=384, K=64, p=0.3), {"COAST_GEMM_PAIR": "0"}, "xmr_gemm_tf32n_nc1_inj1"),
    ("tf32_wide_nc1", dict(kernel=K_GEMM_TF32, nc=1, M=384, N=512, K=64), {}, "xmr_gemm_tf32_nc1_inj0"),
    ("tf32_pair_nc1", dict(kernel=K_GEMM_TF32, nc=1, M=512, N=512, K=64), {}, "xmr_gemm_tf32p_nc1_inj0"),
    ("tf32_pair_nc2", dict(kernel=K_GEMM_TF32, nc=2, M=512, N=384, K=64, p=0.3), {}, "xmr_gemm_tf32p_nc2_inj1"),
    ("tf32_batched_pair_nc2", dict(kernel=K_GEMM_TF32, nc=2, M=256, N=128, K=96, batch=3), {}, "xmr_gemm_tf32p_nc2_inj0"),
    ("tf32_grouped_nc3", dict(kernel=K_GEMM_TF32, nc=3, N=256, K=64, ro=RO), {}, "xmr_gemm_tf32_grp_inj0_nc3"),
    ("tf32_grouped_nc1", dict(kernel=K_GEMM_TF32, nc=1, N=128, K=32, ro=RO, p=0.3), {}, "xmr_gemm_tf32n_grp_inj1_nc1"),
    ("bf16_single_nc3", dict(kernel=K_GEMM_BF16, nc=3, M=512, N=512, K=128), {}, "xmr_gemm_bf16_bt_inj0_nc3"),
    ("bf16_single_nc2", dict(kernel=K_GEMM_BF16, nc=2, M=512, N=512, K=64, p=0.3), {"COAST_GEMM_PAIR": "0"}, "xmr_gemm_bf16_bt_inj1_nc2"),
    ("bf16_narrow_nc1", dict(kernel=K_GEMM_BF16, nc=1, M=512, N=384, K=64, p=0.3), {"COAST_GEMM_PAIR": "0"}, "xmr_gemm_bf16n_bt_inj1_nc1"),
    ("bf16_wide_nc1", dict(kernel=K_GEMM_BF16, nc=1, M=384, N=512, K=64), {}, "xmr_gemm_bf16_bt_inj0_nc1"),
    ("bf16_pair_nc1", dict(kernel=K_GEMM_BF16, nc=1, M=512, N=512, K=64), {}, "xmr_gemm_bf16p_bt_inj0_nc1"),
    ("bf16_pair_nc3", dict(kernel=K_GEMM_BF16, nc=3, M=512, N=256, K=128, p=0.3), {"COAST_GEMM_PAIR": "1"}, "xmr_gemm_bf16p_bt_inj1_nc3"),
    ("bf16_batched_pair_nc2", dict(kernel=K_GEMM_BF16, nc=2, M=256, N=128, K=192, batch=3), {}, "xmr_gemm_bf16p_bt_inj0_nc2"),
    ("bf16_batched_nc3", dict(kernel=K_GEMM_BF16, nc=3, M=128, N=128, K=64, batch=300), {}, "xmr_gemm_bf16_bt_inj0_nc3"),
    ("bf16_grouped_nc2", dict(kernel=K_GEMM_BF16, nc=2, N=256, K=128, ro=RO), {}, "xmr_gemm_bf16_bt_grp_inj0_nc2"),
    ("bf16_grouped_nc1", dict(kernel=K_GEMM_BF16, nc=1, N=256, K=64, ro=RO, p=0.3), {}, "xmr_gemm_bf16n_bt_grp_inj1_nc1"),
]


@pytest.mark.parametrize("case", LAUNCHES, ids=[c[0] for c in LAUNCHES])
def test_the_bit_keeps_the_launch_and_reads_b_transposed_in_place(mock_dir, tmp_path, case):
    _, op, e, name = case
    op = dict(op, op="launch", unit_base=(1 << 32) - 5)
    (rb, evb), (rt_, evt) = [run(mock_dir, tmp_path, [dict(op, bt=bt)], env_extra=e) for bt in (False, True)]
    rb, rt_ = rb["ops"][0], rt_["ops"][0]
    assert rb["rc"] == 0 and rt_["rc"] == 0, (rb, rt_)
    lb, lt = work(evb), work(evt)
    kb, kt = lb[-1], lt[-1]
    assert kt["name"] == name
    assert (kt["grid"], kt["block"], kt["smem"]) == (kb["grid"], kb["block"], kb["smem"])
    ab, at = args_of(kb), args_of(kt)
    fields = ("n_units", "unit_base", "M", "N", "K", "mode", "flags", "n_sites", "plan_mode", "threshold", "n_tiles")
    assert [getattr(at, f) for f in fields] == [getattr(ab, f) for f in fields] and at.mode & (BT | MM_GROUPED | MM_BATCHED) == 0
    assert (at.inp, at.aux, at.out) == (rt_["in"], rt_["aux"], rt_["out"])        # B^T for the plain, tiled and recompute reads
    kernel, grouped = op["kernel"], "ro" in op
    batch = G if grouped else op.get("batch", 1)
    N, K = op["N"], op["K"]
    pre_b, pre_t = [x["name"] for x in lb[:-1]], [x["name"] for x in lt[:-1]]
    sb, st = scratch(evb, rb["sizes"]), scratch(evt, rt_["sizes"])
    if kernel == K_MM_U32 and "_tc_" in name:
        # the limb planes: A split as before, B^T split like A into the same [plane][batch N][K] planes; scratch as before
        assert pre_b == [("xmr_mm_grp_split_a" if grouped else "xmr_mm_split_a"), "xmr_mm_split_bt"] + (["xmr_mm_group_scan"] if grouped else [])
        assert pre_t == [pre_b[0], "xmr_mm_split_a"] + pre_b[2:]
        assert arg0_ptr(lt[1]) == rt_["aux"] and st == sb
        assert [m[1:] for m in maps(evt)] == [m[1:] for m in maps(evb)]
        assert maps(evt)[1][1:4] == (1, K, batch * N)
    elif kernel == K_MM_U32:                                       # tiled and plain: no pre-pass but the grouped scan
        assert pre_t == pre_b == (["xmr_mm_group_scan"] if grouped and "_tiled_" in name else [])
        assert st == sb and not maps(evt)
    else:
        es = 2 if kernel == K_GEMM_BF16 else 4
        pair = "tf32p_" in name or "bf16p_" in name
        # no transposing pre-pass and no B^T scratch: the scan and the group block alone for groups, nothing otherwise
        assert pre_t == (["xmr_mm_group_scan"] if grouped else [])
        assert st == ([GRP_BYTES(G)] if grouped else [])
        if kernel == K_GEMM_TF32:
            assert pre_b == [("xmr_gemm_bt")] + (["xmr_mm_group_scan"] if grouped else [])
            assert sb == [batch * K * N * 4 + (GRP_BYTES(G) if grouped else 0)]
        else:
            assert sb == st
        ma, mb = maps(evt)
        # A: as before (grouped: a 128-row placeholder on d_aux, rebased by the scan); B: the caller's B^T, (batch N) rows of K
        assert ma[1:] == maps(evb)[0][1:] and ma[0] == (rt_["aux"] if grouped else rt_["in"])
        assert mb == (rt_["aux"], es, K, batch * N, 128 // es, 64 if pair else 128)


REFUSALS = [
    ("crc16", dict(kernel=K_CRC16, M=0, N=0, K=0, n=64, unit_bytes=64)),
    ("sha256", dict(kernel=K_SHA256, M=0, N=0, K=0, n=64, unit_bytes=64)),
    ("aes128", dict(kernel=K_AES128, M=0, N=0, K=0, n=64)),
    ("qsort", dict(kernel=K_QSORT, M=0, N=0, K=0, n=64, unit_bytes=64)),
    ("chstone_sha", dict(kernel=K_CHSTONE_SHA, M=0, N=0, K=0, n=4, unit_bytes=64)),
    ("chstone_aes", dict(kernel=K_CHSTONE_AES, M=0, N=0, K=0, n=4)),
]


@pytest.mark.parametrize("call", ["launch", "run_host"])
@pytest.mark.parametrize("case", REFUSALS, ids=[c[0] for c in REFUSALS])
def test_the_bit_on_any_other_kernel_is_refused(mock_dir, tmp_path, case, call):
    _, op = case
    res, ev = run(mock_dir, tmp_path, [dict(op, op=call, bt=True, alloc=[4096, 4096, 4096])])
    r = res["ops"][0]
    assert r["rc"] == BAD_ARG and "COAST_MM_B_TRANSPOSED" in r["err"] and "MM_U32, GEMM_TF32 and GEMM_BF16 only" in r["err"], r
    assert not work(ev) and not [e for e in ev if e["op"] == "h2d"]


@pytest.mark.parametrize("form", ["batch", "groups"])
def test_bf16_b_rows_bound_moves_from_k_to_n(mock_dir, tmp_path, form):
    """2^31 bounds B's stacked tensor-map rows: batch K (G K) for BF16 reading B in place, batch N (G N) for B^T"""
    tiny = [16, 16, 16]
    if form == "batch":
        wide_n = dict(M=128, N=256, K=64, batch=1 << 23, alloc=tiny)   # batch N = 2^31, batch K = 2^29
        wide_k = dict(M=128, N=128, K=512, batch=1 << 22, alloc=tiny)  # the reverse: batch K = 2^31, batch N = 2^29
        needle = "batch*M and batch*%s must be below 2^31"
    else:
        wide_n = dict(N=4096, K=64, ro=[0, 128], M=1 << 19, alloc=tiny)   # G N = 2^31
        wide_k = dict(N=128, K=4096, ro=[0, 128], M=1 << 19, alloc=tiny)  # G K = 2^31
        needle = "G*%s must be below 2^31"
    for op, refused_with in ((wide_n, True), (wide_k, False)):
        for bt in (False, True):
            res, ev = run(mock_dir, tmp_path, [dict(op, op="launch", kernel=K_GEMM_BF16, nc=3, bt=bt)], driver_errors=True)
            r = res["ops"][0]
            refused = bt == refused_with
            if refused:
                assert r["rc"] == BAD_ARG and needle % ("N" if bt else "K") in r["err"], (op, bt, r)
            else:                                                  # past the bound, as far as the maps: the mock's buffers are too small
                assert "2^31" not in r["err"] and [e for e in ev if e["op"] == "tmap_at"], (op, bt, r)
                assert {"op": "error", "what": "tensor map covers memory outside a live allocation"} in ev
            assert not work(ev)


def test_bound_on_tf32_and_mm_u32_stays_on_n(mock_dir, tmp_path):
    for kernel in (K_GEMM_TF32, K_MM_U32):
        res, ev = run(mock_dir, tmp_path, [dict(op="launch", kernel=kernel, nc=3, M=128, N=256, K=64, batch=1 << 23, bt=True, alloc=[16, 16, 16])])
        r = res["ops"][0]
        assert r["rc"] == BAD_ARG and "batch*M and batch*N must be below 2^31" in r["err"] and not work(ev)


@pytest.mark.parametrize("kernel", [K_GEMM_TF32, K_GEMM_BF16])
def test_misaligned_b_transposed_is_refused(mock_dir, tmp_path, kernel):
    res, ev = run(mock_dir, tmp_path, [dict(op="launch", kernel=kernel, nc=3, M=128, N=128, K=64, bt=True, shift=[0, 4, 0])])
    r = res["ops"][0]
    assert r["rc"] == BAD_ARG and "16-byte aligned" in r["err"] and not work(ev)


def test_misaligned_b_transposed_takes_the_plain_mm_u32_kernel(mock_dir, tmp_path):
    """as without the bit: the tensor-core and tiled paths need 16-byte aligned buffers, the plain kernel takes any"""
    res, ev = run(mock_dir, tmp_path, [dict(op="launch", kernel=K_MM_U32, nc=2, M=128, N=128, K=128, bt=True, shift=[0, 4, 0])])
    assert res["ops"][0]["rc"] == 0 and [e["name"] for e in work(ev)] == ["xmr_mm_u32_bt_inj0_nc2"]


def spans(ev, op, base, size):
    return [(e["host"] - base, e["bytes"], e["stream"]) for e in ev if e["op"] == op and base <= e["host"] < base + size]


def copies(ev, r, sizes):
    return [spans(ev, op, r[k], s) for op, k, s in (("h2d", "host_in", sizes[0]), ("h2d", "host_aux", sizes[1]),
                                                      ("d2h", "host_out", sizes[2]), ("h2d", "host_rows", sizes[3]))]


HOST = [
    ("row_blocks_bf16", dict(kernel=K_GEMM_BF16, nc=3, M=1024, N=128, K=64), {}, "row-blocks"),
    ("row_blocks_tf32", dict(kernel=K_GEMM_TF32, nc=2, M=1024, N=128, K=64), {}, "row-blocks"),
    ("row_blocks_mm_u32", dict(kernel=K_MM_U32, nc=3, M=640, N=64, K=128), {}, "row-blocks"),
    ("products_bf16", dict(kernel=K_GEMM_BF16, nc=2, M=128, N=128, K=64, batch=5), {"COAST_HOST_CHUNK_BYTES": "150000"}, "staged"),
    ("products_tf32", dict(kernel=K_GEMM_TF32, nc=1, M=128, N=128, K=64, batch=5), {"COAST_HOST_CHUNK_BYTES": "200000"}, "staged"),
    ("products_mm_u32", dict(kernel=K_MM_U32, nc=3, M=64, N=128, K=32, batch=7), {"COAST_HOST_CHUNK_BYTES": "100000"}, "staged"),
    ("groups_bf16", dict(kernel=K_GEMM_BF16, nc=3, N=128, K=64, ro=[7, 100, 228, 228, 500, 501]), {"COAST_HOST_CHUNK_BYTES": "70000"}, "groups"),
    ("groups_tf32", dict(kernel=K_GEMM_TF32, nc=2, N=128, K=64, ro=[7, 100, 228, 228, 500, 501]), {"COAST_HOST_CHUNK_BYTES": "120000"}, "groups"),
    ("groups_mm_u32", dict(kernel=K_MM_U32, nc=1, N=64, K=128, ro=[7, 100, 228, 228, 500, 501]), {"COAST_HOST_CHUNK_BYTES": "120000"}, "groups"),
]


@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("case", HOST, ids=[c[0] for c in HOST])
def test_host_call_copies_the_bytes_of_the_b_layout(mock_dir, tmp_path, case, pinned):
    _, op, e, path = case
    recs = []
    for bt in (False, True):
        res, ev = run(mock_dir, tmp_path, [dict(op, op="run_host", bt=bt, pinned=pinned, unit_base=5)], env_extra=e)
        r = res["ops"][0]
        assert r["rc"] == 0 and r["path"] == path, r
        es = 2 if op["kernel"] == K_GEMM_BF16 else 4
        ro = op.get("ro")
        rows, b = (ro[-1], len(ro) - 1) if ro else (op.get("batch", 1) * op["M"], op.get("batch", 1))
        sizes = (es * rows * op["K"], es * b * op["K"] * op["N"], 4 * rows * op["N"], 8 * len(ro) if ro else 0)
        la = [x for x in work(ev) if x["name"] not in PREPASSES]
        recs.append((copies(ev, r, sizes), [(args_of(x).n_units, args_of(x).unit_base, args_of(x).M) for x in la],
                     [args_of(x).mode & BT for x in la]))
    assert recs[0][:2] == recs[1][:2] and len(recs[0][0][0]) > 1 and set(recs[1][2]) == {0}
