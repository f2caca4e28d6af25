"""Host logic of COAST_K_GEMM_I8 on a GPU-less box, against the mock driver (tests/mock_cuda/mock_cuda.c) through
tests/mock_cuda/mm_child.py, whose A and B buffers hold 1-byte elements.  GEMM_I8 plans every launch as GEMM_FP8 does; pinned
here: over GEMM_FP8's plan space of tests/test_mm_plan_sweep.py (one product, a batch, groups, with and without B^T, NC 1-3 with
and without a plan, every COAST_GEMM_PAIR setting), every GEMM_I8 launch makes exactly the driver calls of its GEMM_FP8 twin --
grid, block, shared memory, UINT8 tensor maps, the byte-transposing pre-pass, scratch and argument block -- except for the kernel's
name, xmr_gemm_i8 for xmr_gemm_fp8; so do coast_run_host calls, pinned or not; scales, bfloat16 output and unassigned ids are
refused with their messages; every xmr_gemm_i8* function runs the s8 wgmma and keeps the register, stack and local budget of its
FP8 twin.  That all twenty xmr_gemm_i8* functions are reached is tests/test_mm_plan_sweep.py's."""
import re

import pytest

from mock_run import BAD_ARG, K_CRC16, K_GEMM_FP8, SMS, args_of, maps, mock_dir, res_usage, run, sass_by_function, work  # noqa: F401
from coast_b200.runtime import K_GEMM_I8, MM_OUT_BF16, MM_SCALE_ROWWISE, MM_SCALE_TENSOR
from test_gemm_out_bf16_host_logic import mode_of, normalised
from test_mm_plan_sweep import ENVS, RO, SHAPES

I8, FP8 = "xmr_gemm_i8", "xmr_gemm_fp8"


def twin(name):
    """the GEMM_FP8 kernel of an xmr_gemm_i8* name"""
    return FP8 + name[len(I8):] if name.startswith(I8) else name


def as_i8(ops):
    return [dict(op, kernel=K_GEMM_I8) for op in ops]


def renamed(ev):
    """the events of an I8 run with each xmr_gemm_i8* launch named as its FP8 twin"""
    return [dict(e, name=twin(e["name"])) if e["op"] == "launch" else e for e in ev]


def compared(ev):
    """normalised(ev), with the biased pointers of grouped host-call chunks (d_in and d_out of a chunk point ro[first] rows
    before its buffers, into no allocation) named by the next live allocation above them: a<id>-<distance>"""
    norm, live = normalised(ev), {}
    for raw, e in zip(ev, norm):
        if raw["op"] == "alloc":
            live[raw["id"]] = raw["ptr"]
        elif raw["op"] == "free":
            live.pop(raw["id"], None)
        elif e["op"] == "launch" and isinstance(e["args"], list):
            for i in (0, 1, 2):
                p = e["args"][i]
                if isinstance(p, int) and p:
                    above = [(b, k) for k, b in live.items() if b > p]
                    if above:
                        b, k = min(above)
                        e["args"][i] = f"a{k}-{b - p}"
    return norm


def sweep_ops():
    """tests/test_mm_plan_sweep.py's launches of GEMM_FP8"""
    single, grouped = SHAPES[K_GEMM_FP8]
    ops = []
    for bt in (False, True):
        for nc in (1, 2, 3):
            for p in (0, 0.3):
                base = dict(op="launch", kernel=K_GEMM_FP8, nc=nc, bt=bt, p=p, unit_base=(1 << 32) - 5, flags=3)
                for M, N, K in single:
                    ops += [dict(base, M=M, N=N, K=K), dict(base, M=M, N=N, K=K, batch=2)]
                ops += [dict(base, N=N, K=K, ro=RO) for N, K in grouped]
    return ops


@pytest.mark.parametrize("env", ENVS, ids=["default", "mm_tiled", "mm_naive", "pair0", "pair1"])
def test_every_launch_is_its_fp8_twin_but_for_the_name(mock_dir, tmp_path, env):
    ops = sweep_ops()
    res0, ev0, _ = run(mock_dir, tmp_path, ops, env_extra=env)
    res1, ev1, _ = run(mock_dir, tmp_path, as_i8(ops), env_extra=env)
    assert [r["err"] for r in res0["ops"] + res1["ops"] if r["rc"]] == []
    names0 = [e["name"] for e in work(ev0) if e["name"].startswith(FP8)]
    names1 = [e["name"] for e in work(ev1) if e["name"].startswith(I8)]
    assert len(names1) == len(ops) and [twin(n) for n in names1] == names0
    assert not [e for e in work(ev1) if e["name"].startswith(FP8)]
    assert compared(renamed(ev1)) == compared(ev0)


# (id, op): row blocks, one shot, whole products per chunk (B and B^T), groups per chunk
HOST_CALLS = [
    ("row_blocks", dict(M=1024, N=128, K=128), {}),
    ("one_shot", dict(M=384, N=256, K=128), {}),
    ("products", dict(M=128, N=128, K=256, batch=5), {"COAST_HOST_CHUNK_BYTES": str(2 * (128 * 256 * 2 + 128 * 128 * 4) + 100)}),
    ("products_bt", dict(M=128, N=128, K=256, batch=5, bt=True), {"COAST_HOST_CHUNK_BYTES": "120000"}),
    ("groups", dict(N=128, K=128, ro=[7, 100, 228, 228, 500, 501]), {"COAST_HOST_CHUNK_BYTES": "90000"}),
]


@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("case", HOST_CALLS, ids=[c[0] for c in HOST_CALLS])
def test_host_call_is_its_fp8_twin_but_for_the_name(mock_dir, tmp_path, case, pinned):
    _, shape, env = case
    op = dict(shape, op="run_host", kernel=K_GEMM_FP8, nc=3, pinned=pinned, unit_base=5, p=0.3, flags=3)
    res0, ev0, _ = run(mock_dir, tmp_path, [op], env_extra=env)
    res1, ev1, _ = run(mock_dir, tmp_path, as_i8([op]), env_extra=env)
    (r0,), (r1,) = res0["ops"], res1["ops"]
    assert r0["rc"] == 0 and r1["rc"] == 0 and r1["path"] == r0["path"], (r0, r1)
    assert len([e for e in work(ev1) if e["name"].startswith(I8)]) >= 1
    assert compared(renamed(ev1)) == compared(ev0)


# ------------------------------------------------------------------------------------------ refusals
OK = dict(kernel=K_GEMM_I8, nc=3, M=128, N=128, K=128)
REFUSALS = [
    ("scale_tensor", dict(OK, mode=MM_SCALE_TENSOR), "COAST_MM_SCALE_TENSOR: scaled products exist for GEMM_FP8 only (kernel 12)"),
    ("scale_rowwise", dict(OK, mode=MM_SCALE_ROWWISE), "COAST_MM_SCALE_ROWWISE: scaled products exist for GEMM_FP8 only (kernel 12)"),
    ("out_bf16", dict(OK, mode=MM_OUT_BF16), "COAST_MM_OUT_BF16: bfloat16 output exists for GEMM_BF16 and GEMM_FP8 only (kernel 12)"),
    ("out_bf16_grouped", dict(N=128, K=128, ro=[0, 128], kernel=K_GEMM_I8, mode=mode_of(dict(ro=1)) | MM_OUT_BF16),
     "COAST_MM_OUT_BF16: bfloat16 output exists for GEMM_BF16 and GEMM_FP8 only (kernel 12)"),
    ("k_64", dict(OK, K=64), "GEMM_I8 tiles are 128x128x128: M,N must be multiples of 128 and K of 128"),
    ("grouped_k_192", dict(N=128, K=192, ro=[0, 128], kernel=K_GEMM_I8), "GEMM_I8 grouped tiles are 128 x 128 x 128"),
    ("misaligned_aux", dict(OK, shift=[0, 1, 0]), "16-byte aligned"),
    ("batched_on_crc16", dict(OK, kernel=K_CRC16, batch=2),
     "COAST_MM_BATCHED: batched products exist for MM_U32, GEMM_TF32 and GEMM_BF16 only, plus GEMM_FP8 and GEMM_I8 (kernel 0)"),
    ("grouped_on_crc16", dict(N=128, K=128, ro=[0, 128], kernel=K_CRC16),
     "COAST_MM_GROUPED: grouped products exist for MM_U32, GEMM_TF32 and GEMM_BF16 only, plus GEMM_FP8 and GEMM_I8 (kernel 0)"),
    ("bt_on_crc16", dict(OK, kernel=K_CRC16, bt=True),
     "COAST_MM_B_TRANSPOSED: a transposed B exists for MM_U32, GEMM_TF32 and GEMM_BF16 only, plus GEMM_FP8 and GEMM_I8 (kernel 0)"),
    ("id_9", dict(OK, kernel=9), "unknown kernel id 9"),
    ("id_11", dict(OK, kernel=11), "unknown kernel id 11"),
    ("id_13", dict(OK, kernel=13), "unknown kernel id 13"),
]


@pytest.mark.parametrize("case", REFUSALS, ids=[c[0] for c in REFUSALS])
def test_refusals_name_their_rule_and_launch_nothing(mock_dir, tmp_path, case):
    _, op, needle = case
    code = BAD_ARG if "tiles" not in needle else None
    res, ev, _ = run(mock_dir, tmp_path, [dict(op, op="launch")])
    r = res["ops"][0]
    assert r["rc"] != 0 and needle in r["err"], r
    assert code is None or r["rc"] == code, r
    assert not work(ev)


@pytest.mark.parametrize("mode", [MM_SCALE_TENSOR, MM_SCALE_ROWWISE, MM_OUT_BF16])
def test_the_host_call_refuses_scales_and_bf16_output(mock_dir, tmp_path, mode):
    res, ev, _ = run(mock_dir, tmp_path, [dict(OK, op="run_host", mode=mode)])
    r = res["ops"][0]
    assert r["rc"] == BAD_ARG and "(kernel 12)" in r["err"], r
    assert not work(ev)


def test_store_vote_flags_warn_with_the_kernel_name(mock_dir, tmp_path):
    res, ev, err = run(mock_dir, tmp_path, [dict(OK, op="launch", flags=0x200)])
    assert res["ops"][0]["rc"] == 0 and "NOT honoured by the gemm_i8 kernel" in err
    assert [e["name"] for e in work(ev)] == ["xmr_gemm_bt_u8", "xmr_gemm_i8_inj0_nc3"]
    assert args_of(work(ev)[-1]).n_sites == 1


# ------------------------------------------------------------------------------------------ SASS and resources
def test_every_i8_function_runs_the_s8_wgmma(built_lib):
    sass = sass_by_function()
    fns = sorted(f for f in sass if f.startswith(I8))
    assert len(fns) == 20
    for f in fns:
        assert re.search(r"IGMMA\.64x128x32\.S8\.S8", sass[f]), f
        assert "QGMMA" not in sass[f] and "IGMMA" not in sass[twin(f)], f


def test_every_i8_function_keeps_the_budget_of_its_fp8_twin(built_lib):
    """168 registers, as every wgmma GEMM kernel (the s32 accumulators take the registers fp32 ones do), and no more stack or
    local memory than the FP8 kernel of the same variant, NC and injection"""
    res = res_usage()
    fns = sorted(f for f in res if f.startswith(I8))
    assert len(fns) == 20
    for f in fns:
        t = res[twin(f)]
        assert res[f]["REG"] == 168 and res[f]["STACK"] <= t["STACK"] and res[f]["LOCAL"] <= t["LOCAL"], (f, res[f], t)
