"""Host logic of COAST_K_GEMM_F16 and COAST_MM_OUT_F16 on a GPU-less box, against tests/mock_cuda/mock_cuda_f16.c (the mock
driver of tests/mock_cuda/mock_cuda.c plus FLOAT16 tensor maps and a record of every map's data type) through
tests/mock_cuda/mm_child.py, whose A and B buffers hold 2-byte elements for both kernels.  GEMM_F16 plans every launch as
GEMM_BF16 does; pinned here: over GEMM_BF16's plan space of tests/test_mm_plan_sweep.py (one product, a batch, groups, with and
without B^T, NC 1-3 with and without a plan, under every path switch), every GEMM_F16 launch makes exactly the driver calls of its
GEMM_BF16 twin -- grid, block, shared memory, tensor maps, scratch and argument block -- except for the kernel's name
(xmr_gemm_f16 for xmr_gemm_bf16) and the maps' data type (FLOAT16 for BFLOAT16); the same holds with COAST_MM_OUT_F16 against
COAST_MM_OUT_BF16 (xmr_h16_f16 for xmr_o16_bf16) and for host calls, pinned or not; all 80 functions are reached; the
refusals; the MM_OPS row that tests/test_abi.py does not parse; the f16 HGMMA and the f16 pack in SASS, and the register and
stack budget of every function against its BF16 twin."""
import os
import re
import subprocess

import pytest

from mock_run import (BAD_ARG, K_CRC16, K_GEMM_BF16, K_GEMM_FP8, K_GEMM_I8, K_GEMM_TF32, ROOT, args_of, cubin_functions,
                      res_usage, run, sass_by_function, work)
from coast_b200.runtime import K_GEMM_F16, MM_OUT_BF16, MM_OUT_F16, MM_SCALE_ROWWISE, MM_SCALE_TENSOR
from test_gemm_i8_host_logic import compared
from test_gemm_out_bf16_host_logic import mode_of
from test_mm_plan_sweep import ENVS, RO, SHAPES

DT_FLOAT16, DT_BFLOAT16 = 6, 9                            # CUtensorMapDataType
F16, BF16, H16, O16 = "xmr_gemm_f16", "xmr_gemm_bf16", "xmr_h16_f16", "xmr_o16_bf16"


@pytest.fixture(scope="session")
def mock_dir(tmp_path_factory, built_lib):
    d = tmp_path_factory.mktemp("mockcuda_f16")
    subprocess.run(["gcc", "-O1", "-shared", "-fPIC", "-Wall", "-I/usr/local/cuda/include", "-o", str(d / "libcuda.so.1"),
                    os.path.join(ROOT, "tests", "mock_cuda", "mock_cuda_f16.c")], check=True)
    return d


def twin(name):
    """the GEMM_BF16 kernel of a GEMM_F16 name: xmr_gemm_f16* -> xmr_gemm_bf16*, xmr_h16_f16* -> xmr_o16_bf16*"""
    for mine, theirs in ((F16, BF16), (H16, O16)):
        if name.startswith(mine):
            return theirs + name[len(mine):]
    return name


def as_f16(ops):
    """the ops as GEMM_F16, with COAST_MM_OUT_F16 where they have COAST_MM_OUT_BF16"""
    out = []
    for op in ops:
        op = dict(op, kernel=K_GEMM_F16)
        if op.get("mode", 0) & MM_OUT_BF16:
            op["mode"] = op["mode"] & ~MM_OUT_BF16 | MM_OUT_F16
        out.append(op)
    return out


def as_bf16_run(ev, dt):
    """the events of a GEMM_F16 run as its GEMM_BF16 twin would log them: every map has data type dt, which becomes BFLOAT16,
    and every GEMM_F16 launch is named as its twin"""
    out = []
    for e in ev:
        if e["op"] == "tmap_dt":
            assert e["dt"] == dt, e
            e = dict(e, dt=DT_BFLOAT16)
        elif e["op"] == "launch":
            e = dict(e, name=twin(e["name"]))
        out.append(e)
    return out


def sweep_ops(out16=False):
    """tests/test_mm_plan_sweep.py's launches of GEMM_BF16, with bfloat16 output if out16"""
    single, grouped = SHAPES[K_GEMM_BF16]
    ops = []
    for bt in (False, True):
        for nc in (1, 2, 3):
            for p in (0, 0.3):
                base = dict(op="launch", kernel=K_GEMM_BF16, nc=nc, bt=bt, p=p, unit_base=(1 << 32) - 5, flags=3)
                shapes = [dict(M=M, N=N, K=K) for M, N, K in single] + [dict(M=M, N=N, K=K, batch=2) for M, N, K in single]
                shapes += [dict(N=N, K=K, ro=RO) for N, K in grouped]
                for s in shapes:
                    op = dict(base, **s)
                    ops.append(dict(op, mode=mode_of(op) | MM_OUT_BF16) if out16 else op)
    return ops


def comparable(ev, biased):
    """compared(ev) of tests/test_gemm_i8_host_logic.py; with `biased` (grouped host calls), the d_in and d_out of the argument
    blocks are dropped: a chunk's point ro[first] rows before its slot buffers, wherever the host heap's layout puts that"""
    out = compared(ev)
    for e in out:
        if biased and e["op"] == "launch" and isinstance(e["args"], list):
            e["args"] = ["biased", "biased"] + e["args"][2:]
    return out


def check_twins(mock_dir, tmp_path, ops, env):
    """runs ops and their GEMM_F16 form; returns the GEMM_F16 kernel names launched"""
    res0, ev0, _ = run(mock_dir, tmp_path, ops, env_extra=env)
    res1, ev1, _ = run(mock_dir, tmp_path, as_f16(ops), env_extra=env)
    assert [r["err"] for r in res0["ops"] + res1["ops"] if r["rc"]] == []
    assert [r.get("path") for r in res1["ops"]] == [r.get("path") for r in res0["ops"]]
    names1 = [e["name"] for e in work(ev1) if e["name"].startswith((F16, H16))]
    assert [twin(n) for n in names1] == [e["name"] for e in work(ev0) if e["name"].startswith((BF16, O16))]
    assert not [e for e in work(ev1) if e["name"].startswith((BF16, O16))]
    assert [e["dt"] for e in ev0 if e["op"] == "tmap_dt"].count(DT_FLOAT16) == 0
    assert len([e for e in ev1 if e["op"] == "tmap_dt"]) == len([e for e in ev1 if e["op"] == "tmap"]) > 0
    biased = any(op["op"] == "run_host" and "ro" in op for op in ops)
    assert comparable(as_bf16_run(ev1, DT_FLOAT16), biased) == comparable(ev0, biased)
    return names1


@pytest.mark.parametrize("out16", [False, True], ids=["fp32_c", "f16_c"])
@pytest.mark.parametrize("env", ENVS, ids=["default", "mm_tiled", "mm_naive", "pair0", "pair1"])
def test_every_launch_is_its_bf16_twin_but_for_the_name_and_the_map_type(mock_dir, tmp_path, env, out16):
    ops = sweep_ops(out16)
    names = check_twins(mock_dir, tmp_path, ops, env)
    assert len(names) == len(ops) and all(n.startswith(H16 if out16 else F16) for n in names)


def test_all_80_functions_are_reached(mock_dir, tmp_path):
    launched = set()
    for env in ENVS:
        for out16 in (False, True):
            res, ev, _ = run(mock_dir, tmp_path, as_f16(sweep_ops(out16)), env_extra=env)
            assert [r["err"] for r in res["ops"] if r["rc"]] == []
            launched |= {e["name"] for e in work(ev)}
    have = {f for f in cubin_functions() if f.startswith((F16, H16))}
    assert len(have) == 80
    assert launched >= have and not {n for n in launched if n.startswith((F16, H16))} - have


# (id, op, env): row blocks, one shot, whole products per chunk (B and B^T), groups per chunk
HOST_CALLS = [
    ("row_blocks", dict(M=1024, N=256, K=128), {}),
    ("one_shot", dict(M=384, N=256, K=128), {}),
    ("products", dict(M=128, N=256, K=128, batch=5), {"COAST_HOST_CHUNK_BYTES": "300000"}),
    ("products_bt", dict(M=128, N=128, K=256, batch=5, bt=True), {"COAST_HOST_CHUNK_BYTES": "120000"}),
    ("groups", dict(N=128, K=128, ro=[7, 100, 228, 228, 500, 501]), {"COAST_HOST_CHUNK_BYTES": "60000"}),
]


@pytest.mark.parametrize("out16", [False, True], ids=["fp32_c", "f16_c"])
@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("case", HOST_CALLS, ids=[c[0] for c in HOST_CALLS])
def test_host_call_is_its_bf16_twin_but_for_the_name_and_the_map_type(mock_dir, tmp_path, case, pinned, out16):
    _, shape, env = case
    op = dict(shape, op="run_host", kernel=K_GEMM_BF16, nc=3, pinned=pinned, unit_base=5, p=0.3, flags=3)
    if out16:
        op["mode"] = mode_of(op) | MM_OUT_BF16
    names = check_twins(mock_dir, tmp_path, [op], env)
    assert names and all(n.startswith(H16 if out16 else F16) for n in names)


# ------------------------------------------------------------------------------------------ refusals
OK = dict(kernel=K_GEMM_F16, nc=3, M=128, N=128, K=128)
OUT_F16_ELSEWHERE = "COAST_MM_OUT_F16: float16 output exists for GEMM_F16 only (kernel {})"
REFUSALS = [
    *[(f"out_f16_on_{n}", dict(OK, kernel=k, K=256, mode=MM_OUT_F16), OUT_F16_ELSEWHERE.format(k))
      for n, k in (("bf16", K_GEMM_BF16), ("tf32", K_GEMM_TF32), ("fp8", K_GEMM_FP8), ("i8", K_GEMM_I8), ("mm_u32", 3))],
    ("out_f16_on_crc16", dict(OK, kernel=K_CRC16, M=0, N=0, K=0, n=64, unit_bytes=64, alloc=[1 << 16] * 3, mode=MM_OUT_F16),
     OUT_F16_ELSEWHERE.format(K_CRC16)),
    ("out_f16_with_out_bf16", dict(OK, mode=MM_OUT_F16 | MM_OUT_BF16),
     "COAST_MM_OUT_F16 and COAST_MM_OUT_BF16 cannot be combined: one C type per launch"),
    ("out_bf16", dict(OK, mode=MM_OUT_BF16),
     "COAST_MM_OUT_BF16: bfloat16 output exists for GEMM_BF16 and GEMM_FP8 only (kernel 14)"),
    ("out_bf16_grouped", dict(N=128, K=128, ro=[0, 128], kernel=K_GEMM_F16, mode=mode_of(dict(ro=1)) | MM_OUT_BF16),
     "COAST_MM_OUT_BF16: bfloat16 output exists for GEMM_BF16 and GEMM_FP8 only (kernel 14)"),
    ("scale_tensor", dict(OK, mode=MM_SCALE_TENSOR), "COAST_MM_SCALE_TENSOR: scaled products exist for GEMM_FP8 only (kernel 14)"),
    ("scale_rowwise", dict(OK, mode=MM_SCALE_ROWWISE | MM_OUT_F16),
     "COAST_MM_SCALE_ROWWISE: scaled products exist for GEMM_FP8 only (kernel 14)"),
    ("k_32", dict(OK, K=32), "GEMM_F16 tiles are 128x128x64: M,N must be multiples of 128 and K of 64 (got 128,128,32)"),
    ("n_64", dict(OK, N=64, mode=MM_OUT_F16), "GEMM_F16 tiles are 128x128x64: M,N must be multiples of 128 and K of 64"),
    ("grouped_k_96", dict(N=128, K=96, ro=[0, 128], kernel=K_GEMM_F16), "GEMM_F16 grouped tiles are 128 x 128 x 64"),
    ("misaligned_aux", dict(OK, shift=[0, 2, 0]), "16-byte aligned"),
    ("id_13", dict(OK, kernel=13), "kernel 13"),
    ("id_15", dict(OK, kernel=15), "kernel 15"),
]


@pytest.mark.parametrize("call", ["launch", "run_host"])
@pytest.mark.parametrize("case", REFUSALS, ids=[c[0] for c in REFUSALS])
def test_refusals_name_their_rule_and_launch_nothing(mock_dir, tmp_path, case, call):
    _, op, needle = case
    if call == "run_host" and "shift" in op:
        pytest.skip("the child misaligns device buffers only")
    res, ev, _ = run(mock_dir, tmp_path, [dict(op, op=call)])
    r = res["ops"][0]
    assert r["rc"] != 0 and (needle in r["err"] or needle.replace("kernel ", "unknown kernel id ") in r["err"]), r
    assert r["rc"] == BAD_ARG or "tiles" in needle or needle.startswith("kernel"), r
    assert not work(ev)


def test_store_vote_flags_warn_with_the_kernel_name(mock_dir, tmp_path):
    res, ev, err = run(mock_dir, tmp_path, [dict(OK, op="launch", flags=0x200)])
    assert res["ops"][0]["rc"] == 0 and "NOT honoured by the gemm_f16 kernel" in err
    assert [e["name"] for e in work(ev)] == ["xmr_gemm_f16_inj0_nc3"]
    a = args_of(work(ev)[-1])
    assert a.n_sites == 1 and a.mode & (MM_OUT_F16 | MM_OUT_BF16) == 0


def test_out_f16_bit_never_reaches_the_kernel(mock_dir, tmp_path):
    res, ev, _ = run(mock_dir, tmp_path, [dict(OK, op="launch", mode=MM_OUT_F16)])
    assert res["ops"][0]["rc"] == 0 and [e["name"] for e in work(ev)] == ["xmr_h16_f16_inj0_nc3"]
    assert args_of(work(ev)[-1]).mode & MM_OUT_F16 == 0


# ------------------------------------------------------------------------------------------ the MM_OPS row and the cubin
def test_the_f16_mm_ops_row_is_bf16s_with_the_float16_map_type():
    """tests/test_abi.py parses the positional MM_OPS rows; GEMM_F16's is written with designators, and checked here"""
    src = open(os.path.join(ROOT, "coast_b200", "csrc", "coast_rt.c")).read()
    row = re.search(r"\[COAST_K_GEMM_F16\]\s*=\s*\{([^}]*)\}", src[src.index("} MM_OPS["):]).group(1)
    fields = dict(re.findall(r"\.(\w+)\s*=\s*([^,]+?)\s*(?:,|$)", row.strip()))
    assert fields == {"ty": '"F16"', "prefix": '"gemm"', "stem": '"f16"', "bk": "XMR_GEMM_BF16_BK",
                      "dt": "CU_TENSOR_MAP_DATA_TYPE_FLOAT16", "b_in_place": "1", "bt_kernels": "1", "nc_first": "0",
                      "grp_variant": "1", "c16": '"h16"'}, fields
    bf16 = re.search(r'\[COAST_K_GEMM_BF16\]\s*=\s*\{\s*"BF16",\s*"gemm",\s*"bf16",\s*XMR_GEMM_BF16_BK,\s*'
                     r'CU_TENSOR_MAP_DATA_TYPE_BFLOAT16,\s*1,\s*1,\s*0,\s*1,\s*"o16"\s*\}', src)
    assert bf16, "GEMM_BF16's row, whose layout fields GEMM_F16 shares"


def test_the_f16_prefixes_start_functions_of_the_cubin(built_lib):
    have = cubin_functions()
    for prefix in (F16, H16):
        assert any(f.startswith(prefix) for f in have), prefix
    assert not any(f.startswith("xmr_o16_f16") or f.startswith("xmr_h16_bf16") for f in have)


def new_functions(table):
    fns = sorted(f for f in table if f.startswith((F16, H16)))
    assert len(fns) == 80
    return fns


def test_every_f16_function_runs_the_f16_hgmma_and_h16_functions_pack_f16(built_lib):
    sass = sass_by_function()
    for f in new_functions(sass):
        assert re.search(r"HGMMA\.64x128x16\.F32 ", sass[f]) and not re.search(r"HGMMA\S*BF16", sass[f]), f
        assert re.search(r"HGMMA\.64x128x16\.F32\.BF16 ", sass[twin(f)]), f
        if f.startswith(H16):
            assert re.search(r"F2FP\.F16\.F32\.PACK_AB", sass[f]) and not re.search(r"F2FP\.BF16", sass[f]), f
        else:
            assert not re.search(r"F2FP", sass[f]), f


def test_no_f16_function_keeps_more_registers_or_stack_than_its_bf16_twin(built_lib):
    res = res_usage()
    for f in new_functions(res):
        t = res[twin(f)]
        assert res[f]["REG"] <= t["REG"] and res[f]["STACK"] <= t["STACK"] and res[f]["LOCAL"] <= t["LOCAL"], (f, res[f], t)
