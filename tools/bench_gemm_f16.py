"""GEMM_F16 beside GEMM_BF16, GEMM_TF32 on the upcast operands and unprotected torch.matmul in float16, in one process: one JSON
line.

For each square size (default 4096 and 8192), then the grouped case of tools/bench_grouped_mm.py (2^16 rows, N = K = 2048, 64
Zipf-routed experts), NC 1/2/3 and each C type -- fp32, and 16-bit (COAST_MM_OUT_F16 for GEMM_F16, COAST_MM_OUT_BF16 for
GEMM_BF16) -- the variants alternate round by round:
  * f16:  GEMM_F16 on float16 A and B (B read in place);
  * bf16: GEMM_BF16 on bfloat16 A and B of the same shape (B read in place);
  * tf32: GEMM_TF32 on the operands upcast to fp32, the exact protected route a float16 caller had before GEMM_F16: twice the
          operand bytes and the B transpose pre-pass, which is part of its time.  Its C is always fp32;
  * torch_f16: unprotected torch.matmul on the float16 tensors (float16 C; square sizes only).
`--rounds` rounds of `--steps` launches each, after `--warmup`, over `--buffers` rotating operand sets so that a launch does not
find the previous one's operands in L2.  Times come from CUDA events.  Per variant: seconds per launch (median of the rounds, and
their min and max) and useful TFLOP/s (2 M N K); per case, f16's time over bf16's and over tf32's.  The card name and its power
limit are read in the same run; no device setting is changed.

    python tools/bench_gemm_f16.py [--sizes 4096,8192] [--ncs 1,2,3] [--steps 10] [--rounds 5] [--warmup 2] [--buffers 3]
                                   [--grouped 65536,2048,2048,64]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_grouped_mm import power_limit, routed_rows, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="4096,8192")
    ap.add_argument("--ncs", default="1,2,3")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--buffers", type=int, default=3)
    ap.add_argument("--grouped", default="65536,2048,2048,64", help="rows,N,K,experts of the grouped case ('' skips it)")
    args = ap.parse_args()
    import torch
    import coast_b200 as cb
    if not torch.cuda.is_available():
        sys.exit("bench_gemm_f16: no GPU; nothing is measured on a CPU")
    for k in ("COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT"):
        os.environ.pop(k, None)
    rt = cb.Runtime(0)
    head = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit()}
    L, stream = rt.L, rt.stream_handle()
    kernel = {"f16": cb.K_GEMM_F16, "bf16": cb.K_GEMM_BF16, "tf32": cb.K_GEMM_TF32}
    out16 = {"f16": cb.MM_OUT_F16, "bf16": cb.MM_OUT_BF16, "tf32": 0}

    def operands(rows, K, n_b, N, seed):
        """integers in [-8, 8] (exact in every type): {type: (A, B)}, B as n_b stacked K x N matrices"""
        g = torch.Generator(device="cuda").manual_seed(seed)
        A = torch.randint(-8, 9, (rows, K), device="cuda", generator=g).float()
        B = torch.randint(-8, 9, (n_b * K, N), device="cuda", generator=g).float()
        return {"f16": (A.half(), B.half()), "bf16": (A.bfloat16(), B.bfloat16()), "tf32": (A, B)}

    def launcher(descs):
        state = {"i": 0}

        def go():
            d = descs[state["i"] % len(descs)]
            state["i"] += 1
            rc = L.coast_launch(C.byref(d), stream)
            assert rc == 0, L.coast_last_error()
        return go

    def measure(fns, flop):
        times = {k: [] for k in fns}
        for r in range(args.rounds):
            for k, fn in fns.items():
                times[k].append(timed(torch, fn, args.steps, args.warmup if r == 0 else 1))
        rt.sync()
        out = {k: {"s_per_launch": statistics.median(ts), "s_min": min(ts), "s_max": max(ts),
                   "useful_tflops": flop / statistics.median(ts) / 1e12} for k, ts in times.items()}
        out["f16_over_bf16"] = out["f16"]["s_per_launch"] / out["bf16"]["s_per_launch"]
        out["f16_over_tf32"] = out["f16"]["s_per_launch"] / out["tf32"]["s_per_launch"]
        return out

    def cases(sets, n_units, flop, info, vendor=None, mode=0, **kw):
        for nc in [int(x) for x in args.ncs.split(",")]:
            for c16 in (False, True):
                fns = {}
                for ty in kernel:
                    m = mode | (out16[ty] if c16 else 0)
                    esize = 2 if m & (cb.MM_OUT_F16 | cb.MM_OUT_BF16) else 4
                    outs = [torch.empty(n_units * esize, dtype=torch.uint8, device="cuda") for _ in sets]
                    fns[ty] = launcher([rt.make_desc(kernel[ty], nc, s[ty][0], o, n_units, d_aux=s[ty][1], flags=3, mode=m, **kw)
                                        for s, o in zip(sets, outs)])
                if vendor:
                    fns["torch_f16"] = vendor
                results.append({**info, "nc": nc, "c": "16-bit" if c16 else "fp32", **measure(fns, flop)})

    results = []
    for n in [int(x) for x in args.sizes.split(",") if x]:
        sets = [operands(n, n, 1, n, seed=10 * i + 1) for i in range(args.buffers)]
        state = {"i": 0}

        def vendor():
            A, B = sets[state["i"] % args.buffers]["f16"]
            state["i"] += 1
            torch.matmul(A, B)
        cases(sets, n * n, 2.0 * n ** 3, {"case": "square", "M": n, "N": n, "K": n}, vendor, M=n, N=n, K=n)
        del sets
        torch.cuda.empty_cache()
    if args.grouped:
        R, N, K, G = [int(x) for x in args.grouped.split(",")]
        rows = routed_rows(G, R)
        ro = [0]
        for x in rows:
            ro.append(ro[-1] + x)
        d_rows = torch.tensor(ro, dtype=torch.int64, device="cuda")
        sets = [operands(R, K, G, N, seed=10 * i + 2) for i in range(args.buffers)]
        cases(sets, R * N, 2.0 * R * N * K, {"case": "grouped", "rows": R, "N": N, "K": K, "experts": G, "max_rows": max(rows)},
              mode=cb.MM_GROUPED, M=G, N=N, K=K, d_rows=d_rows)
    print(json.dumps({**head, "steps": args.steps, "rounds": args.rounds, "buffers": args.buffers, "results": results}))


if __name__ == "__main__":
    main()
