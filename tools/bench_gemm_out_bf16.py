"""BF16 output (COAST_MM_OUT_BF16) beside fp32 output, in one process: one JSON line.

For each square size (default 4096 and 8192), then the grouped case of tools/bench_grouped_mm.py (2^16 rows, N = K = 2048, 64
Zipf-routed experts), for GEMM_BF16 (B read in place) and GEMM_FP8 (B^T read in place, COAST_MM_B_TRANSPOSED, so no pre-pass
hides or adds anything) and NC 1/2/3, the fp32-output and the bf16-output launch alternate round by round on the same operands.
Beside them, on the square sizes, unprotected torch.matmul in bfloat16 and torch._scaled_mm at scale 1 with bf16 output.
`--rounds` rounds of `--steps` launches each, after `--warmup`, over `--buffers` rotating operand sets so that a launch does not
find the previous one's operands in L2.  Times come from CUDA events.  Per case: seconds per launch (median of the rounds, and their min and max), useful TFLOP/s (2 M N K), and the bf16
launch's time over the fp32 one's.  The card name and its power limit are read in the same run; no device setting is changed.

    python tools/bench_gemm_out_bf16.py [--sizes 4096,8192] [--ncs 1,2,3] [--ops bf16,fp8] [--steps 10] [--rounds 5]
                                        [--warmup 2] [--buffers 3] [--grouped 65536,2048,2048,64]
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
    ap.add_argument("--ops", default="bf16,fp8")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--buffers", type=int, default=3)
    ap.add_argument("--grouped", default="65536,2048,2048,64", help="rows,N,K,experts of the grouped case ('' skips it)")
    args = ap.parse_args()
    import torch
    import coast_b200 as cb
    if not torch.cuda.is_available():
        sys.exit("bench_gemm_out_bf16: no GPU; nothing is measured on a CPU")
    for k in ("COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT"):
        os.environ.pop(k, None)
    rt = cb.Runtime(0)
    head = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit()}
    L, stream = rt.L, rt.stream_handle()
    ops = [x for x in args.ops.split(",") if x]
    one = torch.ones((), device="cuda")

    def operands(op, rows, K, n_b, N, seed):
        """integers in [-1, 1]: BF16 A and B (K x N per product) or E4M3 A and B^T (N x K per product)"""
        g = torch.Generator(device="cuda").manual_seed(seed)
        dt = torch.bfloat16 if op == "bf16" else torch.float8_e4m3fn
        A = torch.randint(-1, 2, (rows, K), device="cuda", generator=g).float().to(dt)
        B = torch.randint(-1, 2, (n_b * K, N) if op == "bf16" else (n_b * N, K), device="cuda", generator=g).float().to(dt)
        return A, B

    def launcher(descs):
        state = {"i": 0}

        def go():
            d = descs[state["i"] % len(descs)]
            state["i"] += 1
            rc = L.coast_launch(C.byref(d), stream)
            assert rc == 0, L.coast_last_error()
        return go

    def descs(op, sets, outs, nc, o16, n_units, mode=0, **kw):
        kernel = cb.K_GEMM_BF16 if op == "bf16" else cb.K_GEMM_FP8
        mode |= (0 if op == "bf16" else cb.MM_B_TRANSPOSED) | (cb.MM_OUT_BF16 if o16 else 0)
        return [rt.make_desc(kernel, nc, A, o, n_units, d_aux=B, flags=3, mode=mode, **kw) for (A, B), o in zip(sets, outs[o16])]

    def measure(fns, flop):
        times = {k: [] for k in fns}
        for r in range(args.rounds):
            for k, fn in fns.items():
                times[k].append(timed(torch, fn, args.steps, args.warmup if r == 0 else 1))
        rt.sync()
        out = {k: {"s_per_launch": statistics.median(ts), "s_min": min(ts), "s_max": max(ts),
                   "useful_tflops": flop / statistics.median(ts) / 1e12} for k, ts in times.items()}
        if "fp32_out" in out:
            out["bf16_out"]["over_fp32_out"] = out["bf16_out"]["s_per_launch"] / out["fp32_out"]["s_per_launch"]
        return out

    def outputs(n):
        return {False: [torch.empty(n, dtype=torch.float32, device="cuda") for _ in range(args.buffers)],
                True: [torch.empty(n, dtype=torch.bfloat16, device="cuda") for _ in range(args.buffers)]}

    results = []
    for n in [int(x) for x in args.sizes.split(",") if x]:
        outs = outputs(n * n)
        for op in ops:
            sets = [operands(op, n, n, 1, n, seed=10 * i + 1) for i in range(args.buffers)]
            state = {"i": 0}

            def vendor():
                A, B = sets[state["i"] % args.buffers]
                state["i"] += 1
                if op == "bf16":
                    torch.matmul(A, B)
                else:
                    torch._scaled_mm(A, B.t(), scale_a=one, scale_b=one, out_dtype=torch.bfloat16)
            for nc in [int(x) for x in args.ncs.split(",")]:
                fns = {name: launcher(descs(op, sets, outs, nc, o16, n * n, M=n, N=n, K=n))
                       for name, o16 in (("fp32_out", False), ("bf16_out", True))}
                fns["torch_bf16_out"] = vendor
                results.append({"case": "square", "op": op, "M": n, "N": n, "K": n, "nc": nc, **measure(fns, 2.0 * n ** 3)})
            del sets
        del outs
        torch.cuda.empty_cache()
    if args.grouped:
        R, N, K, G = [int(x) for x in args.grouped.split(",")]
        rows = routed_rows(G, R)
        ro = [0]
        for x in rows:
            ro.append(ro[-1] + x)
        d_rows = torch.tensor(ro, dtype=torch.int64, device="cuda")
        outs = outputs(R * N)
        for op in ops:
            sets = [operands(op, R, K, G, N, seed=10 * i + 2) for i in range(args.buffers)]
            for nc in [int(x) for x in args.ncs.split(",")]:
                fns = {name: launcher(descs(op, sets, outs, nc, o16, R * N, mode=cb.MM_GROUPED, M=G, N=N, K=K, d_rows=d_rows))
                       for name, o16 in (("fp32_out", False), ("bf16_out", True))}
                results.append({"case": "grouped", "op": op, "rows": R, "N": N, "K": K, "experts": G, "max_rows": max(rows), "nc": nc,
                                **measure(fns, 2.0 * R * N * K)})
            del sets
    print(json.dumps({**head, "steps": args.steps, "rounds": args.rounds, "buffers": args.buffers, "results": results}))


if __name__ == "__main__":
    main()
