"""Batched matmuls (COAST_MM_BATCHED) against one launch per product: one JSON line.

Cases (TMR, one stream, one process):
  tf32  : 64 products of 512 x 512 x 512, TF32 GEMM (integer-valued operands in [-8, 8]);
  limb  : 64 products of 512 x 512 x 512, exact u32 on the u8-limb tensor-core kernel (Philox operands);
  plain : 65,536 products of 9 x 9 x 9 (the reference's matrixMultiply size), exact u32 on the plain kernel.
For each: the time of one batched launch and of a loop of per-product launches (descriptors built beforehand, so the loop
pays the launches, not Python), both from CUDA events around `--steps` repetitions after `--warmup`; their ratio; the useful
and the issued rate (TF32 FLOP/s for the GEMM, multiply-adds/s for the exact kernels; issued = useful x 3 replicas); and
whether the two arms' outputs are identical.  The card name and its power limit are read in the same run.

    python tools/bench_batched_mm.py [--steps 5] [--warmup 1] [--cases tf32,limb,plain]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CASES = {"tf32": ("gemm_tf32", 512, 512, 512, 64), "limb": ("mm_u32", 512, 512, 512, 64), "plain": ("mm_u32", 9, 9, 9, 65536)}
NC = 3


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:                                         # a number we could not read is reported as missing
        return None


def timed(torch, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / 1e3 / steps


def run_case(rt, torch, cb, name, steps, warmup):
    kind, M, N, K, batch = CASES[name]
    kernel = cb.K_GEMM_TF32 if kind == "gemm_tf32" else cb.K_MM_U32
    if kernel == cb.K_GEMM_TF32:
        g = torch.Generator(device="cuda").manual_seed(1)
        A = torch.randint(-8, 9, (batch * M * K,), dtype=torch.float32, device="cuda", generator=g)
        B = torch.randint(-8, 9, (batch * K * N,), dtype=torch.float32, device="cuda", generator=g)
        out1, out2 = torch.zeros(batch * M * N, dtype=torch.float32, device="cuda"), torch.zeros(batch * M * N, dtype=torch.float32, device="cuda")
    else:
        A = torch.empty(batch * M * K, dtype=torch.int32, device="cuda")
        B = torch.empty(batch * K * N, dtype=torch.int32, device="cuda")
        rt.fill_philox(A, seed=1)
        rt.fill_philox(B, seed=2)
        out1, out2 = torch.zeros(batch * M * N, dtype=torch.int32, device="cuda"), torch.zeros(batch * M * N, dtype=torch.int32, device="cuda")
    mn = M * N
    one = rt.make_desc(kernel, NC, A, out1, batch * mn, mode=cb.MM_BATCHED, M=M, N=N, K=K, d_aux=B)
    singles = [rt.make_desc(kernel, NC, A[b * M * K:(b + 1) * M * K], out2[b * mn:(b + 1) * mn], mn, M=M, N=N, K=K,
                            d_aux=B[b * K * N:(b + 1) * K * N], unit_base=b * mn) for b in range(batch)]
    stream = rt.stream_handle()
    L = rt.L

    def batched():
        rc = L.coast_launch(C.byref(one), stream)
        assert rc == 0, L.coast_last_error()

    def loop():
        for d in singles:
            rc = L.coast_launch(C.byref(d), stream)
            assert rc == 0, L.coast_last_error()

    t_one = timed(torch, batched, steps, warmup)
    t_loop = timed(torch, loop, steps, warmup)
    rt.sync()
    useful = batch * M * N * K * (2 if kernel == cb.K_GEMM_TF32 else 1)        # FLOP (GEMM) or multiply-adds (exact)
    unit = "tflops" if kernel == cb.K_GEMM_TF32 else "gmacs"
    scale = 1e12 if kernel == cb.K_GEMM_TF32 else 1e9
    return {"case": name, "kernel": kind, "batch": batch, "M": M, "N": N, "K": K, "nc": NC,
            "batched_s": t_one, "loop_s": t_loop, "speedup": t_loop / t_one,
            f"useful_{unit}_batched": useful / t_one / scale, f"issued_{unit}_batched": NC * useful / t_one / scale,
            f"useful_{unit}_loop": useful / t_loop / scale, f"issued_{unit}_loop": NC * useful / t_loop / scale,
            "outputs_identical": bool(torch.equal(out1.view(torch.int32), out2.view(torch.int32)))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--cases", default="tf32,limb,plain")
    args = ap.parse_args()
    import torch
    import coast_b200 as cb
    for k in ("COAST_MM_PATH", "COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT"):
        os.environ.pop(k, None)
    rt = cb.Runtime(0)
    res = [run_case(rt, torch, cb, c, args.steps, args.warmup) for c in args.cases.split(",")]
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit(), "steps": args.steps,
                      "results": res}))


if __name__ == "__main__":
    main()
