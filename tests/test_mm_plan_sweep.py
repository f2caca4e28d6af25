"""The matmul plan space on a GPU-less box, against the mock driver (tests/mock_cuda/mock_cuda_bt.c), whose cuModuleGetFunction
finds only the function symbols of the loaded cubin.  Every matmul kernel (MM_U32, GEMM_TF32, GEMM_BF16) is launched as one
product, a batch and groups, with and without a transposed B, at NC 1-3 with and without a fault plan, on shapes that land on
each path and under each path switch.  The kernel names are put together at run time, so this is what shows that every name
the host code can reach exists in the cubin, and that every matmul function of the cubin is reachable.

SWEEP is shared with tools/mm_launch_trace.py, which runs it (with refusals and host calls added) against two builds and
compares their driver calls."""
import json
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K_MM_U32, K_GEMM_TF32, K_GEMM_BF16 = 3, 4, 8
MM_PREFIXES = ("xmr_mm_u32", "xmr_gemm_tf32", "xmr_gemm_bf16")
KNOBS = ("COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT", "COAST_HOST_CHUNK_BYTES",
         "COAST_HOST_PATH", "COAST_STRICT_FLAGS", "COAST_MM_PATH")
ENVS = [{}, {"COAST_MM_PATH": "tiled"}, {"COAST_MM_PATH": "naive"}, {"COAST_GEMM_PAIR": "0"}, {"COAST_GEMM_PAIR": "1"}]
RO = [3, 3, 100, 101, 101, 500, 700]

# per kernel: one-product shapes (M, N, K) and grouped shapes (N, K) that land on each path
SHAPES = {
    K_MM_U32: ([(128, 128, 128), (64, 128, 16), (9, 9, 9)],                 # limb tensor-core kernel, tiled, plain
               [(128, 128), (128, 16), (9, 7)]),
    K_GEMM_TF32: ([(512, 512, 64), (384, 512, 64), (512, 384, 64), (384, 384, 64)],   # pairs, wide, narrow, 128 x 128
                  [(256, 64), (128, 32)]),
    K_GEMM_BF16: ([(512, 512, 64), (384, 512, 64), (512, 384, 64), (384, 384, 64)],
                  [(256, 64), (128, 128)]),
}


def plan_ops():
    """the launches of the plan space, for every environment in ENVS"""
    ops = []
    for kernel, (single, grouped) in SHAPES.items():
        for bt in (False, True):
            for nc in (1, 2, 3):
                for p in (0, 0.3):
                    base = dict(op="launch", kernel=kernel, nc=nc, bt=bt, p=p, unit_base=(1 << 32) - 5)
                    for M, N, K in single:
                        ops.append(dict(base, M=M, N=N, K=K))
                        ops.append(dict(base, M=M, N=N, K=K, batch=2))
                    for N, K in grouped:                        # M is G here: a grouped op leaves it out
                        ops.append(dict(base, N=N, K=K, ro=RO))
    return ops


SWEEP = [(env, plan_ops()) for env in ENVS]


@pytest.fixture(scope="session")
def mock_dir(tmp_path_factory, built_lib):
    d = tmp_path_factory.mktemp("mockcuda_sweep")
    subprocess.run(["gcc", "-O1", "-shared", "-fPIC", "-Wall", "-I/usr/local/cuda/include", "-o", str(d / "libcuda.so.1"),
                    os.path.join(ROOT, "tests", "mock_cuda", "mock_cuda_bt.c")], check=True)
    return d


def run_child(mock_dir, root, log, ops, env_extra):
    """runs ops in one child process against root's library; returns (results, mock events)"""
    if os.path.exists(log):
        os.unlink(log)
    env = dict(os.environ, LD_LIBRARY_PATH=f"{mock_dir}:" + os.environ.get("LD_LIBRARY_PATH", ""), MOCK_CUDA_LOG=str(log))
    for k in KNOBS:
        env.pop(k, None)
    env.update(env_extra)
    res = subprocess.run([sys.executable, os.path.join(root, "tests", "mock_cuda", "mm_bt_child.py"), json.dumps({"ops": ops})],
                         capture_output=True, text=True, env=env, timeout=600)
    assert res.returncode == 0, res.stdout + res.stderr
    events = [json.loads(ln) for ln in open(log)] if os.path.exists(log) else []
    return json.loads(res.stdout.strip().splitlines()[-1])["ops"], events


def cubin_functions():
    elf = subprocess.run(["cuobjdump", "-elf", os.path.join(ROOT, "coast_b200", "csrc", "coast_kernels.cubin")],
                         capture_output=True, text=True).stdout
    return set(re.findall(r"\.text\.(xmr_\w+)", elf))


def test_every_matmul_kernel_of_the_cubin_is_reached_and_no_name_is_missing(mock_dir, tmp_path):
    launched = set()
    for env, ops in SWEEP:
        results, events = run_child(mock_dir, ROOT, tmp_path / "mock.log", ops, env)
        assert [r["err"] for r in results if r["rc"]] == []
        assert [e for e in events if e["op"] == "error"] == []
        assert events[-1] == {"op": "exit", "live_allocations": 0}
        launched |= {e["name"] for e in events if e["op"] == "launch" and e["name"].startswith(MM_PREFIXES)}
    have = {f for f in cubin_functions() if f.startswith(MM_PREFIXES)}
    assert len(have) == 126
    assert launched == have, (sorted(have - launched), sorted(launched - have))
