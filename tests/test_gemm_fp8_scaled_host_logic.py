"""Host logic of scaled GEMM_FP8 (COAST_MM_SCALE_TENSOR / COAST_MM_SCALE_ROWWISE) on a GPU-less box, against the mock driver
(tests/mock_cuda/mock_cuda_scaled.c: tests/mock_cuda/mock_cuda.c plus a record of the scale pointers of every xmr_scaled_*
launch) through tests/mock_cuda/mm_scaled_child.py.  Pinned here: the xmr_scaled_fp8* kernel each shape gets, and that everything else of the
launch -- the pre-pass, grid, block, shared memory, tensor maps, scratch and argument block -- is the unscaled launch's; that the
scale pointers are the last two parameters (after the maps, and for groups after ro and the group block) and reach the kernel
unchanged; the internal row-wise mode bit and no caller scale bit in the argument block; every refusal; the scale bytes the host
call copies per chunk for row blocks, whole products and groups, tensorwise and row-wise; that the 20 functions run the E4M3
wgmma; and that none keeps more stack than its unscaled twin.  That all 20 are reached is tests/test_mm_plan_sweep.py's."""
import os
import re
import subprocess

import pytest

import mock_run
from mock_run import BAD_ARG, K_CRC16, K_GEMM_BF16, K_GEMM_FP8, K_GEMM_TF32, ROOT, args_of, maps, res_usage, run, sass_by_function, spans
from coast_b200.runtime import MM_SCALE_ROWWISE, MM_SCALE_TENSOR

CHILD = "mm_scaled_child.py"
ROWWISE_BIT = 0x400                                       # XMR_MODE_SCALE_ROWWISE (coast_b200/csrc/xmr_args.h)
RO = [3, 3, 100, 101, 101, 500, 700]


@pytest.fixture(scope="session")
def mock_dir(tmp_path_factory, built_lib):
    d = tmp_path_factory.mktemp("mockcuda_scaled")
    subprocess.run(["gcc", "-O1", "-shared", "-fPIC", "-Wall", "-I/usr/local/cuda/include", "-o", str(d / "libcuda.so.1"),
                    os.path.join(ROOT, "tests", "mock_cuda", "mock_cuda_scaled.c")], check=True)
    return d


def work(ev):
    """the launches of mock_run.work, each xmr_scaled_* one with the "sa" and "sb" of the scales record that follows it"""
    launches = {id(e) for e in mock_run.work(ev)}
    out = []
    for i, e in enumerate(ev):
        if id(e) in launches:
            if e["name"].startswith("xmr_scaled_"):
                nxt = ev[i + 1]
                assert nxt["op"] == "scales" and nxt["name"] == e["name"], nxt
                e = dict(e, sa=nxt["sa"], sb=nxt["sb"])
            out.append(e)
    return out


def scaled_name(name):
    return name.replace("xmr_gemm_fp8", "xmr_scaled_fp8")


def launch_record(ev, r):
    """what a launch did, with every device address named by the caller's buffer or the scratch allocation it lies in"""
    mine = {r["in"], r["aux"], r["out"], r["sa"], r["sb"], r["rows"]}
    scratch = [e for e in ev if e["op"] == "alloc" and not e["host"] and e["ptr"] not in mine]
    names = {r["in"]: "in", r["aux"]: "aux", r["out"]: "out"}

    def where(p):
        for j, e in enumerate(scratch):
            if e["ptr"] <= p < e["ptr"] + e["bytes"]:
                return f"scratch{j}+{p - e['ptr']}"
        return names.get(p, p)
    la = work(ev)
    k = la[-1]
    a = args_of(k)
    return dict(names=[e["name"].replace("xmr_scaled_fp8", "xmr_gemm_fp8") for e in la],
                geometry=[(e["grid"], e["block"], e["smem"], e["stream"]) for e in la],
                maps=[(where(m[0]),) + m[1:] for m in maps(ev)], scratch=[e["bytes"] for e in scratch],
                args=(a.n_units, a.unit_base, a.M, a.N, a.K, a.mode & ~ROWWISE_BIT, a.flags, a.n_sites, a.plan_mode, a.threshold),
                where=(where(a.inp), where(a.out), where(a.aux))), k, a


def device_address(ev, copy):
    """the device address an h2d copy event wrote to"""
    return [e["ptr"] for e in ev if e["op"] == "alloc" and e["id"] == copy["alloc"]][-1] + copy["offset"]


# (id, nc, M, N, K, batch or None, environment, unscaled kernel)
LAUNCHES = [
    ("single_nc3", 3, 512, 512, 128, None, {}, "xmr_gemm_fp8_inj0_nc3"),
    ("narrow_nc1", 1, 512, 384, 128, None, {}, "xmr_gemm_fp8n_inj0_nc1"),
    ("wide_nc1", 1, 384, 512, 256, None, {}, "xmr_gemm_fp8_inj0_nc1"),
    ("pair_nc1", 1, 512, 512, 128, None, {}, "xmr_gemm_fp8p_inj0_nc1"),
    ("pair_nc2", 2, 512, 384, 128, None, {}, "xmr_gemm_fp8p_inj0_nc2"),
    ("pair_nc3", 3, 512, 512, 128, None, {"COAST_GEMM_PAIR": "1"}, "xmr_gemm_fp8p_inj0_nc3"),
    ("single_nc2", 2, 512, 512, 128, None, {"COAST_GEMM_PAIR": "0"}, "xmr_gemm_fp8_inj0_nc2"),
    ("batched_nc3", 3, 128, 128, 128, 300, {}, "xmr_gemm_fp8_inj0_nc3"),
    ("batched_pair_nc2", 2, 256, 128, 384, 3, {}, "xmr_gemm_fp8p_inj0_nc2"),
    ("batched_wide_nc1", 1, 128, 256, 128, 5, {}, "xmr_gemm_fp8_inj0_nc1"),
    ("grouped_nc3", 3, None, 128, 128, None, {}, "xmr_gemm_fp8_grp_inj0_nc3"),
    ("grouped_nc1", 1, None, 256, 256, None, {"COAST_GEMM_PAIR": "1"}, "xmr_gemm_fp8_grp_inj0_nc1"),
]


@pytest.mark.parametrize("scale", ["tensor", "row"])
@pytest.mark.parametrize("bt", [False, True], ids=["B", "Bt"])
@pytest.mark.parametrize("case", LAUNCHES, ids=[c[0] for c in LAUNCHES])
def test_scaled_launch_is_the_unscaled_launch_plus_two_pointers(mock_dir, tmp_path, case, bt, scale):
    _, nc, M, N, K, batch, env, name = case
    op = dict(op="launch", kernel=K_GEMM_FP8, nc=nc, N=N, K=K, unit_base=1 << 32, flags=3, bt=bt, p=0.25)
    op.update(dict(ro=RO) if M is None else dict(M=M))
    if batch:
        op["batch"] = batch
    recs = []
    for child, o in ((CHILD, op), (CHILD, dict(op, scale=scale))):
        res, ev, _ = run(mock_dir, tmp_path, [o], child=child, env_extra=env)
        r = res["ops"][0]
        assert r["rc"] == 0, r["err"]
        recs.append((r, ev) + launch_record(ev, r))
    (_, _, plain, k0, a0), (r, ev, scaled, k, a) = recs
    assert k0["name"] == name.replace("inj0", "inj1") and k["name"] == scaled_name(k0["name"])
    assert scaled == plain                                         # the same plan, everything but the kernel and its last two params
    assert (k["sa"], k["sb"]) == (r["sa"], r["sb"]) and "sa" not in k0
    assert a.mode == a0.mode | (ROWWISE_BIT if scale == "row" else 0)
    assert a.mode & (MM_SCALE_TENSOR | MM_SCALE_ROWWISE) == 0 and a0.mode & ROWWISE_BIT == 0


OK = dict(kernel=K_GEMM_FP8, M=128, N=128, K=128)
REFUSALS = [
    ("tensor_on_bf16", dict(OK, kernel=K_GEMM_BF16, scale="tensor"), "COAST_MM_SCALE_TENSOR: scaled products exist for GEMM_FP8 only (kernel 8)"),
    ("row_on_tf32", dict(OK, kernel=K_GEMM_TF32, scale="row"), "COAST_MM_SCALE_ROWWISE: scaled products exist for GEMM_FP8 only (kernel 4)"),
    ("row_on_crc16", dict(OK, kernel=K_CRC16, scale="row"), "scaled products exist for GEMM_FP8 only (kernel 0)"),
    ("both_bits", dict(OK, scale="row", mode=MM_SCALE_TENSOR | MM_SCALE_ROWWISE), "cannot be combined"),
    ("both_bits_on_bf16", dict(OK, kernel=K_GEMM_BF16, scale="row", mode=MM_SCALE_TENSOR | MM_SCALE_ROWWISE), "GEMM_FP8 only"),
    ("null_a", dict(OK, scale="tensor", scale_null=[True, False]), "COAST_MM_SCALE_TENSOR: d_scale_a and d_scale_b must point"),
    ("null_b", dict(OK, scale="row", scale_null=[False, True]), "COAST_MM_SCALE_ROWWISE: d_scale_a and d_scale_b must point"),
    ("null_b_grouped", dict(kernel=K_GEMM_FP8, N=128, K=128, ro=[0, 128], scale="row", scale_null=[False, True]), "d_scale_b"),
    ("misaligned_a", dict(OK, scale="tensor", scale_shift=[2, 0]), "COAST_MM_SCALE_TENSOR: d_scale_a must be 4-byte aligned"),
    ("misaligned_a_row", dict(OK, scale="row", scale_shift=[6, 0]), "COAST_MM_SCALE_ROWWISE: d_scale_a must be 4-byte aligned"),
    ("misaligned_b_row", dict(OK, scale="row", scale_shift=[4, 4]), "COAST_MM_SCALE_ROWWISE: d_scale_b must be 8-byte aligned"),
]


@pytest.mark.parametrize("case", REFUSALS, ids=[c[0] for c in REFUSALS])
def test_refusals_name_their_rule_and_launch_nothing(mock_dir, tmp_path, case):
    _, op, needle = case
    res, ev, _ = run(mock_dir, tmp_path, [dict(op, op="launch"), dict(op, op="run_host")], child=CHILD)
    for r in res["ops"]:
        assert r["rc"] == BAD_ARG and needle in r["err"], r
    assert not work(ev)


def test_tensorwise_takes_a_4_byte_aligned_b_scale(mock_dir, tmp_path):
    """one float of B is read as one float: only the row-wise pairs need 8 bytes"""
    res, ev, _ = run(mock_dir, tmp_path, [dict(OK, op="launch", scale="tensor", scale_shift=[4, 4])], child=CHILD)
    r = res["ops"][0]
    assert r["rc"] == 0 and (work(ev)[-1]["sa"], work(ev)[-1]["sb"]) == (r["sa"], r["sb"]) and r["sb"] % 8 == 4


# ------------------------------------------------------------------------------------------ the host call's scale bytes
@pytest.mark.parametrize("scale", ["tensor", "row"])
@pytest.mark.parametrize("pinned", [False, True])
def test_host_call_row_blocks(mock_dir, tmp_path, pinned, scale):
    M, N, K = 1024, 256, 128
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", kernel=K_GEMM_FP8, nc=3, M=M, N=N, K=K, pinned=pinned, unit_base=5, scale=scale)],
                     child=CHILD)
    r = res["ops"][0]
    assert r["rc"] == 0 and r["path"] == "row-blocks", r
    one = scale == "tensor"                                        # the scale buffers hold one float each
    ups_a = [u[:2] for u in spans(ev, "h2d", r["host_sa"], 4 if one else 4 * M)]
    ups_b = [u[:2] for u in spans(ev, "h2d", r["host_sb"], 4 if one else 4 * N)]
    if scale == "tensor":                                          # 8 bytes go up once
        assert ups_a == [(0, 4)] and ups_b == [(0, 4)]
    else:                                                          # B's column scales once with B; each block its rows' A scales
        assert ups_a == [(i * 128 * 4, 128 * 4) for i in range(8)] and ups_b == [(0, 4 * N)]
    la = [e for e in work(ev) if e["name"].startswith("xmr_scaled")]
    assert len(la) == 8 and len({e["sb"] for e in la}) == 1
    assert len({e["sa"] for e in la}) == (1 if scale == "tensor" else 3)          # three slots
    assert [u[:2] for u in spans(ev, "h2d", r["host_in"], M * K)] == [(i * 128 * K, 128 * K) for i in range(8)]


@pytest.mark.parametrize("scale", ["tensor", "row"])
@pytest.mark.parametrize("pinned", [False, True])
def test_host_call_whole_products(mock_dir, tmp_path, pinned, scale):
    M, N, K, batch = 128, 128, 256, 5
    ab, bb, cb = M * K, K * N, M * N * 4
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", kernel=K_GEMM_FP8, nc=2, M=M, N=N, K=K, batch=batch, pinned=pinned,
                                               scale=scale, bt=True)],
                     child=CHILD, env_extra={"COAST_HOST_CHUNK_BYTES": str(2 * (ab + bb + cb) + 100)})
    r = res["ops"][0]
    assert r["rc"] == 0, r
    chunks = [(0, 2), (2, 2), (4, 1)]                              # the unscaled call's chunks
    assert [u[:2] for u in spans(ev, "h2d", r["host_in"], batch * ab)] == [(f * ab, n * ab) for f, n in chunks]
    one = scale == "tensor"
    ups_a = [u[:2] for u in spans(ev, "h2d", r["host_sa"], 4 if one else 4 * batch * M)]
    ups_b = [u[:2] for u in spans(ev, "h2d", r["host_sb"], 4 if one else 4 * batch * N)]
    if scale == "tensor":
        assert ups_a == [(0, 4)] and ups_b == [(0, 4)]
    else:
        assert ups_a == [(4 * f * M, 4 * n * M) for f, n in chunks] and ups_b == [(4 * f * N, 4 * n * N) for f, n in chunks]
    la = work(ev)
    assert [e["name"] for e in la] == ["xmr_scaled_fp8_inj0_nc2"] * 3
    assert [args_of(e).n_units for e in la] == [n * M * N for _, n in chunks]


@pytest.mark.parametrize("scale", ["tensor", "row"])
@pytest.mark.parametrize("pinned", [False, True])
def test_host_call_groups(mock_dir, tmp_path, pinned, scale):
    N, K, ro, budget = 128, 128, [7, 100, 228, 228, 500, 501], 90000
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", kernel=K_GEMM_FP8, nc=3, N=N, K=K, ro=ro, unit_base=1000, pinned=pinned,
                                               scale=scale)],
                     child=CHILD, env_extra={"COAST_HOST_CHUNK_BYTES": str(budget)})
    r = res["ops"][0]
    assert r["rc"] == 0 and r["path"] == "groups", r
    chunks, f, G = [], 0, len(ro) - 1
    while f < G:                                                   # the unscaled schedule's rule
        e = f + 1
        while e < G and (ro[e + 1] - ro[f]) * (K + N * 4) + (e + 1 - f) * (K * N + 8) + 8 <= budget:
            e += 1
        chunks.append((f, e))
        f = e
    assert len(chunks) > 2
    one = scale == "tensor"
    ups_a = [u for u in spans(ev, "h2d", r["host_sa"], 4 if one else 4 * ro[-1])]
    ups_b = [u[:2] for u in spans(ev, "h2d", r["host_sb"], 4 if one else 4 * G * N)]
    la = [e for e in work(ev) if e["name"].startswith("xmr_scaled")]
    with_rows = [(f, e) for f, e in chunks if ro[e] > ro[f]]
    assert len(la) == len(with_rows)
    if scale == "tensor":
        assert [u[:2] for u in ups_a] == [(0, 4)] and ups_b == [(0, 4)]
        return
    # A scales [ro[first], ro[e]) biased like d_in: the kernel's pointer + ro[first] rows is where they landed
    assert [u[:2] for u in ups_a] == [(4 * ro[f], 4 * (ro[e] - ro[f])) for f, e in with_rows]
    assert ups_b == [(4 * f * N, 4 * (e - f) * N) for f, e in chunks]
    copies_a = [e for e in ev if e["op"] == "h2d" and r["host_sa"] <= e["host"] < r["host_sa"] + 4 * ro[-1]]
    for k, (f, e), c in zip(la, with_rows, copies_a):
        assert k["sa"] + 4 * ro[f] == device_address(ev, c) and k["sb"] % 8 == 0, (f, e)


# ------------------------------------------------------------------------------------------ every function's SASS and stack
def test_scaled_functions_run_the_e4m3_wgmma_and_round_to_nearest(built_lib):
    sass = sass_by_function()
    fns = sorted(f for f in sass if f.startswith("xmr_scaled_fp8"))
    assert len(fns) == 20
    for f in fns:
        assert re.search(r"QGMMA\.64x128x32\.F32\.E4M3\.E4M3", sass[f]), f
        assert "FMUL" in sass[f] and not re.search(r"FMUL\.(FTZ|RZ|RM|RP)", sass[f]), f


def test_no_scaled_function_keeps_more_stack_than_its_twin(built_lib):
    res = res_usage()
    fns = sorted(f for f in res if f.startswith("xmr_scaled_fp8"))
    assert len(fns) == 20
    for f in fns:
        twin = f.replace("xmr_scaled_fp8", "xmr_gemm_fp8")
        assert res[f]["STACK"] <= res[twin]["STACK"] and res[f]["LOCAL"] <= res[twin]["LOCAL"], (f, res[f], res[twin])
