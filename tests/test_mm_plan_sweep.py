"""The matmul plan space on a GPU-less box, against the mock driver (tests/mock_cuda/mock_cuda.c), whose cuModuleGetFunction
finds only the function symbols of the loaded cubin.  Every matmul kernel (MM_U32, GEMM_TF32, GEMM_BF16, GEMM_FP8, GEMM_I8) is
launched as one product, a batch and groups, with and without a transposed B, at NC 1-3 with and without a fault plan, on shapes
that land on each path and under each path switch; GEMM_FP8 also with tensorwise and row-wise scales, and GEMM_BF16 and GEMM_FP8
with bfloat16 output.  The kernel names are put together at run time, so this is what shows that every name the host code can
reach exists in the cubin, and that every matmul function of the cubin is reachable.  Scaled launches run through
tests/mock_cuda/mm_scaled_child.py, which passes the scale pointers; the others through mm_child.py.

SWEEP is shared with tools/mm_launch_trace.py, which runs it (with refusals and host calls added) against two builds and
compares their driver calls."""
from mock_run import (K_GEMM_BF16, K_GEMM_FP8, K_GEMM_I8, K_GEMM_TF32, K_MM_U32, MM_B_TRANSPOSED, MM_BATCHED, MM_GROUPED,  # noqa: F401
                      MM_OUT_BF16, cubin_functions, mock_dir, run)  # (mock_dir is a fixture)

MM_PREFIXES = ("xmr_mm_u32", "xmr_gemm_tf32", "xmr_gemm_bf16", "xmr_gemm_fp8", "xmr_gemm_i8", "xmr_scaled_fp8", "xmr_o16_")
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
    K_GEMM_FP8: ([(512, 512, 128), (384, 512, 128), (512, 384, 128), (384, 384, 256)],      # K a multiple of 128
                 [(256, 128), (128, 256)]),
    K_GEMM_I8: ([(512, 512, 128), (384, 512, 128), (512, 384, 128), (384, 384, 256)],
                [(256, 128), (128, 256)]),
}
# per kernel: the epilogues besides the plain one -- scales (`scale` of mm_scaled_child.py) and bfloat16 output (a mode bit)
EPILOGUES = {K_GEMM_BF16: [dict(out_bf16=True)],
             K_GEMM_FP8: [dict(scale="tensor"), dict(scale="row"), dict(out_bf16=True)]}


def child_of(op):
    return "mm_scaled_child.py" if "scale" in op else "mm_child.py"


def with_mode(op):
    """an op with out_bf16 as the descriptor's mode: the mode bits the op implies plus COAST_MM_OUT_BF16"""
    if not op.pop("out_bf16", False):
        return op
    implied = (MM_BATCHED if "batch" in op else 0) | (MM_GROUPED if "ro" in op else 0) | (MM_B_TRANSPOSED if op.get("bt") else 0)
    return dict(op, mode=implied | MM_OUT_BF16)


def plan_ops():
    """the launches of the plan space, for every environment in ENVS"""
    ops = []
    for kernel, (single, grouped) in SHAPES.items():
        for epilogue in [{}] + EPILOGUES.get(kernel, []):
            for bt in (False, True):
                for nc in (1, 2, 3):
                    for p in (0, 0.3):
                        base = dict(op="launch", kernel=kernel, nc=nc, bt=bt, p=p, unit_base=(1 << 32) - 5, **epilogue)
                        for M, N, K in single:
                            ops.append(with_mode(dict(base, M=M, N=N, K=K)))
                            ops.append(with_mode(dict(base, M=M, N=N, K=K, batch=2)))
                        for N, K in grouped:                    # M is G here: a grouped op leaves it out
                            ops.append(with_mode(dict(base, N=N, K=K, ro=RO)))
    return ops


SWEEP = [(env, plan_ops()) for env in ENVS]


def test_every_matmul_kernel_of_the_cubin_is_reached_and_no_name_is_missing(mock_dir, tmp_path):
    launched = set()
    for env, ops in SWEEP:
        for child in ("mm_child.py", "mm_scaled_child.py"):
            res, events, _ = run(mock_dir, tmp_path, [op for op in ops if child_of(op) == child], child=child, env_extra=env)
            assert [r["err"] for r in res["ops"] if r["rc"]] == []          # a name missing from the cubin is a mock error
            launched |= {e["name"] for e in events if e["op"] == "launch" and e["name"].startswith(MM_PREFIXES)}
    have = {f for f in cubin_functions() if f.startswith(MM_PREFIXES)}
    assert len(have) == 246                                     # MM_U32's 66 and the 180 wgmma GEMM kernels
    assert launched == have, (sorted(have - launched), sorted(launched - have))
