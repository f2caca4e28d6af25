"""Host logic of BF16 output (COAST_MM_OUT_BF16) on a GPU-less box, against the mock driver (tests/mock_cuda/mock_cuda.c)
through tests/mock_cuda/mm_child.py and mm_scaled_child.py.  Pinned here: over the plan space of tests/test_mm_plan_sweep.py
(GEMM_BF16 and GEMM_FP8), every launch with the bit makes exactly the driver calls of the same launch without it -- grid,
block, shared memory, tensor maps, pre-passes, scratch, copies and argument block -- except for the kernel's name, which is its
fp32 twin's with the xmr_o16_ prefix; the bit is refused on every other kernel and with a scale bit; a host call downloads
exactly 2 bytes per C element, with no gap and no overlap, for row blocks, products and groups; and every xmr_o16_* function
rounds with the F2FP.BF16 pack and keeps no more registers or stack than its twin.  That all 60 xmr_o16_* functions are reached
and none is missing is tests/test_mm_plan_sweep.py's."""
import ctypes as C
import re

import pytest

from mock_run import (BAD_ARG, UNSUPPORTED, K_AES128, K_CHSTONE_SHA, K_CRC16, K_GEMM_BF16, K_GEMM_FP8, K_GEMM_TF32, K_MM_U32,
                      K_QSORT, K_SHA256, MM_B_TRANSPOSED, MM_BATCHED, MM_GROUPED, UNIT_OFFSETS, XmrArgs, mock_dir, res_usage,  # noqa: F401
                      run, sass_by_function, spans, work)
from coast_b200.runtime import MM_OUT_BF16, MM_SCALE_ROWWISE, MM_SCALE_TENSOR
from test_mm_plan_sweep import ENVS, RO, SHAPES

O16 = "xmr_o16_"


def twin(name):
    """the fp32-output kernel of an xmr_o16_* name"""
    return "xmr_gemm_" + name[len(O16):] if name.startswith(O16) else name


def mode_of(op):
    """the mode mm_child.py gives an op, plus the scale bit of mm_scaled_child.py"""
    m = (MM_GROUPED if "ro" in op else MM_BATCHED if "batch" in op else 0) | (MM_B_TRANSPOSED if op.get("bt") else 0)
    return m | {"tensor": MM_SCALE_TENSOR, "row": MM_SCALE_ROWWISE}.get(op.get("scale"), 0)


def with_bit(ops):
    return [dict(op, mode=mode_of(op) | MM_OUT_BF16) for op in ops]


def normalised(ev):
    """the events with every device address named by the live allocation it lies in (a<id>+<offset>) and host addresses
    dropped, so that two child processes can be compared"""
    live = {}

    def name(p):
        for i, (base, size) in live.items():
            if base <= p < base + max(size, 1):
                return f"a{i}+{p - base}"
        return p
    out = []
    for e in ev:
        e = dict(e)
        if e["op"] == "alloc":
            live[e["id"]] = (e["ptr"], e["bytes"])
            e.pop("ptr")
        elif e["op"] == "free":
            live.pop(e["id"], None)
        elif e["op"] == "tmap":
            e["addr"] = name(e["addr"])
        elif e["op"] in ("h2d", "d2h"):
            e.pop("host")
        elif e["op"] == "launch":
            e["name"] = twin(e["name"])
            raw = bytes.fromhex(e.pop("arg0"))
            if len(raw) == 128:
                a = XmrArgs.from_buffer_copy(raw)
                e["args"] = [name(a.inp), name(a.out), name(a.aux), a.n_units, a.unit_base, name(a.counters), name(a.plan_table),
                             name(a.status), a.unit_bytes, a.flags, a.mode, a.M, a.N, a.K, a.plan_mode, a.seed_lo, a.seed_hi,
                             a.threshold, a.n_sites, a.n_tiles]
            else:
                e["args"] = name(int.from_bytes(raw, "little"))
        out.append(e)
    return out


def sweep_ops():
    """tests/test_mm_plan_sweep.py's launches of GEMM_BF16 and GEMM_FP8"""
    ops = []
    for kernel in (K_GEMM_BF16, K_GEMM_FP8):
        single, grouped = SHAPES[kernel]
        for bt in (False, True):
            for nc in (1, 2, 3):
                for p in (0, 0.3):
                    base = dict(op="launch", kernel=kernel, nc=nc, bt=bt, p=p, unit_base=(1 << 32) - 5)
                    for M, N, K in single:
                        ops += [dict(base, M=M, N=N, K=K), dict(base, M=M, N=N, K=K, batch=2)]
                    ops += [dict(base, N=N, K=K, ro=RO) for N, K in grouped]
    return ops


@pytest.mark.parametrize("env", ENVS, ids=["default", "mm_tiled", "mm_naive", "pair0", "pair1"])
def test_every_launch_is_its_fp32_twin_but_for_the_name(mock_dir, tmp_path, env):
    ops = sweep_ops()
    res0, ev0, _ = run(mock_dir, tmp_path, ops, env_extra=env)
    res1, ev1, _ = run(mock_dir, tmp_path, with_bit(ops), env_extra=env)
    assert [r["err"] for r in res0["ops"] + res1["ops"] if r["rc"]] == []
    names0 = [e["name"] for e in work(ev0) if e["name"].startswith(("xmr_gemm_bf16", "xmr_gemm_fp8"))]
    names1 = [e["name"] for e in work(ev1) if e["name"].startswith(O16)]
    assert len(names1) == len(ops) and [twin(n) for n in names1] == names0
    assert normalised(ev1) == normalised(ev0)


# ------------------------------------------------------------------------------------------ refusals
# (id, kernel, another mode bit): the matmul kernels also batched, the ragged kernels also ragged
REFUSED = [(f"{n}_{x}", k, b) for n, k, extras in (
    ("tf32", K_GEMM_TF32, ("plain", "batched")), ("mm_u32", K_MM_U32, ("plain", "batched")), ("crc16", K_CRC16, ("plain", "ragged")),
    ("sha256", K_SHA256, ("plain", "ragged")), ("qsort", K_QSORT, ("plain", "ragged")), ("aes128", K_AES128, ("plain",)),
    ("chstone_sha", K_CHSTONE_SHA, ("plain",))) for x, b in (("plain", 0), ("batched", MM_BATCHED), ("ragged", UNIT_OFFSETS)) if x in extras]


@pytest.mark.parametrize("case", REFUSED, ids=[c[0] for c in REFUSED])
def test_the_bit_is_refused_on_every_other_kernel(mock_dir, tmp_path, case):
    _, kernel, extra = case
    mm = kernel in (K_GEMM_TF32, K_MM_U32)
    op = dict(kernel=kernel, nc=3, mode=MM_OUT_BF16 | extra, alloc=[1 << 16, 1 << 16, 1 << 16])
    op.update(dict(M=128, N=128, K=128, batch=1) if mm else dict(M=0, N=0, K=0, n=64, unit_bytes=64))
    res, ev, _ = run(mock_dir, tmp_path, [dict(op, op="launch"), dict(op, op="run_host")])
    want = f"COAST_MM_OUT_BF16: bfloat16 output exists for GEMM_BF16 and GEMM_FP8 only (kernel {kernel})"
    for r in res["ops"]:
        assert r["rc"] == BAD_ARG and r["err"] == want, r
    assert not work(ev)


@pytest.mark.parametrize("scale", ["tensor", "row"])
def test_the_bit_with_a_scale_bit_is_not_built(mock_dir, tmp_path, scale):
    op = dict(kernel=K_GEMM_FP8, nc=3, M=128, N=128, K=128, scale=scale)
    op["mode"] = mode_of(op) | MM_OUT_BF16
    res, ev, _ = run(mock_dir, tmp_path, [dict(op, op="launch"), dict(op, op="run_host")], child="mm_scaled_child.py")
    for r in res["ops"]:
        assert r["rc"] == UNSUPPORTED and "scaled GEMM_FP8 has no bfloat16-output kernels" in r["err"], r
    assert not work(ev)


# ------------------------------------------------------------------------------------------ the host call's C bytes
def downloads(ev, r, size):
    return sorted(u[:2] for u in spans(ev, "d2h", r["host_out"], size))


def covers(d, total):
    """the downloads tile [0, total) with no gap and no overlap"""
    at = 0
    for off, n in d:
        assert off == at, (off, at)
        at += n
    assert at == total


HOST_CALLS = [
    ("row_blocks", K_GEMM_BF16, dict(M=1024, N=256, K=128), {}, "row-blocks"),
    ("one_shot", K_GEMM_FP8, dict(M=384, N=256, K=128), {}, "one-shot"),
    ("products", K_GEMM_BF16, dict(M=128, N=256, K=128, batch=5), {"COAST_HOST_CHUNK_BYTES": "300000"}, "staged"),
    ("groups", K_GEMM_FP8, dict(N=128, K=128, ro=[7, 100, 228, 228, 500, 501]), {"COAST_HOST_CHUNK_BYTES": "60000"}, "groups"),
    ("products_bt", K_GEMM_FP8, dict(M=128, N=128, K=256, batch=5, bt=True), {"COAST_HOST_CHUNK_BYTES": "120000"}, "staged"),
]


@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("case", HOST_CALLS, ids=[c[0] for c in HOST_CALLS])
def test_host_call_downloads_two_bytes_per_element(mock_dir, tmp_path, case, pinned):
    _, kernel, shape, env, path = case
    op = dict(shape, op="run_host", kernel=kernel, nc=3, pinned=pinned, unit_base=3)
    rows = shape["ro"][-1] - shape["ro"][0] if "ro" in shape else shape["M"] * shape.get("batch", 1)
    first = shape["ro"][0] if "ro" in shape else 0
    res, ev, _ = run(mock_dir, tmp_path, [dict(op, mode=mode_of(op) | MM_OUT_BF16), op], env_extra=env)
    (r1, r0) = res["ops"]
    assert r1["rc"] == 0 and r0["rc"] == 0 and r1["path"] == path, (r1, r0)
    n = rows * shape["N"]
    d1 = [(o - 2 * first * shape["N"], b) for o, b in downloads(ev, r1, 4 * (first + rows) * shape["N"] + 64)]
    d0 = [(o - 4 * first * shape["N"], b) for o, b in downloads(ev, r0, 4 * (first + rows) * shape["N"] + 64)]
    covers(d1, 2 * n)
    covers(d0, 4 * n)
    la = [e["name"] for e in work(ev) if e["name"].startswith(("xmr_o16_", "xmr_gemm_")) and "_inj" in e["name"]]
    assert la == [n for n in la[:len(d1)] if n.startswith(O16)] + [twin(la[0])] * len(d0)


# ------------------------------------------------------------------------------------------ SASS and resources
def test_every_o16_function_rounds_with_the_bf16_pack(built_lib):
    sass = sass_by_function()
    fns = sorted(f for f in sass if f.startswith(O16))
    assert len(fns) == 60
    for f in fns:
        assert re.search(r"F2FP\.BF16\.F32\.PACK_AB", sass[f]), f
        assert not re.search(r"F2FP\.BF16", sass[twin(f)]), f


def test_no_o16_function_keeps_more_registers_or_stack_than_its_twin(built_lib):
    res = res_usage()
    fns = sorted(f for f in res if f.startswith(O16))
    assert len(fns) == 60
    for f in fns:
        t = res[twin(f)]
        assert res[f]["REG"] <= t["REG"] and res[f]["STACK"] <= t["STACK"] and res[f]["LOCAL"] <= t["LOCAL"], (f, res[f], t)


def test_argument_block_is_unchanged():
    assert C.sizeof(XmrArgs) == 128
