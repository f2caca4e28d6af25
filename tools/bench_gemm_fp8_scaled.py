"""Scaled GEMM_FP8 (COAST_MM_SCALE_TENSOR / COAST_MM_SCALE_ROWWISE) beside unscaled GEMM_FP8, in one process: one JSON line.

For each square size (default 4096 and 8192), then the grouped case of tools/bench_grouped_mm.py (2^16 rows, N = K = 2048, 64
Zipf-routed experts), and NC 1/2/3, the launches alternate round by round: unscaled GEMM_FP8, tensorwise scaled, row-wise scaled,
all three reading the same B^T in place (COAST_MM_B_TRANSPOSED, so no pre-pass hides or adds anything), and unprotected
torch._scaled_mm with tensorwise scales and fp32 output (square sizes only).  `--rounds` rounds of `--steps` launches each, after
`--warmup`, over `--buffers` rotating operand sets so that a launch does not find the previous one's operands in L2.  Times come
from CUDA events.  Per case: seconds per launch (median of the rounds, and their min and max), useful TFLOP/s (2 M N K), and the
scaled launches' time over the unscaled one's.  The card name and its power limit are read in the same run; no device setting is
changed.

    python tools/bench_gemm_fp8_scaled.py [--sizes 4096,8192] [--ncs 1,2,3] [--steps 10] [--rounds 5] [--warmup 2] [--buffers 3]
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
        sys.exit("bench_gemm_fp8_scaled: no GPU; nothing is measured on a CPU")
    for k in ("COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT"):
        os.environ.pop(k, None)
    rt = cb.Runtime(0)
    head = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit()}
    L, stream = rt.L, rt.stream_handle()
    modes = {"unscaled": 0, "tensor": cb.MM_SCALE_TENSOR, "row": cb.MM_SCALE_ROWWISE}
    one = torch.ones((), device="cuda")

    def operands(rows, K, n_b, N, seed):
        """E4M3 integers in [-1, 1]; B^T (N x K per product); scales: one float each, and per row / per product column"""
        g = torch.Generator(device="cuda").manual_seed(seed)
        A = torch.randint(-1, 2, (rows, K), device="cuda", generator=g).float().to(torch.float8_e4m3fn)
        Bt = torch.randint(-1, 2, (n_b * N, K), device="cuda", generator=g).float().to(torch.float8_e4m3fn)
        sa = torch.rand(rows, device="cuda", generator=g) + 0.5
        sb = torch.rand(n_b * N, device="cuda", generator=g) + 0.5
        return A, Bt, sa, sb

    def launcher(descs):
        state = {"i": 0}

        def go():
            d = descs[state["i"] % len(descs)]
            state["i"] += 1
            rc = L.coast_launch(C.byref(d), stream)
            assert rc == 0, L.coast_last_error()
        return go

    def descs(sets, outs, nc, kind, n_units, mode=0, **kw):
        out = []
        for (A, Bt, sa, sb), o in zip(sets, outs):
            a, b = {"unscaled": (None, None), "tensor": (sa[:1], sb[:1]), "row": (sa, sb)}[kind]
            out.append(rt.make_desc(cb.K_GEMM_FP8, nc, A, o, n_units, d_aux=Bt, flags=3, mode=mode | cb.MM_B_TRANSPOSED | modes[kind],
                                    scale_a=a, scale_b=b, **kw))
        return out

    def measure(fns, flop):
        times = {k: [] for k in fns}
        for r in range(args.rounds):
            for k, fn in fns.items():
                times[k].append(timed(torch, fn, args.steps, args.warmup if r == 0 else 1))
        rt.sync()
        out = {k: {"s_per_launch": statistics.median(ts), "s_min": min(ts), "s_max": max(ts),
                   "useful_tflops": flop / statistics.median(ts) / 1e12} for k, ts in times.items()}
        for k in ("tensor", "row"):
            out[k]["over_unscaled"] = out[k]["s_per_launch"] / out["unscaled"]["s_per_launch"]
        return out

    results = []
    for n in [int(x) for x in args.sizes.split(",") if x]:
        sets = [operands(n, n, 1, n, seed=10 * i + 1) for i in range(args.buffers)]
        outs = [torch.empty(n * n, dtype=torch.float32, device="cuda") for _ in range(args.buffers)]
        state = {"i": 0}

        def vendor():
            A, Bt, _, _ = sets[state["i"] % args.buffers]
            state["i"] += 1
            torch._scaled_mm(A, Bt.t(), scale_a=one, scale_b=one, out_dtype=torch.float32, use_fast_accum=True)
        for nc in [int(x) for x in args.ncs.split(",")]:
            fns = {k: launcher(descs(sets, outs, nc, k, n * n, M=n, N=n, K=n)) for k in modes}
            fns["scaled_mm"] = vendor
            results.append({"case": "square", "M": n, "N": n, "K": n, "nc": nc, **measure(fns, 2.0 * n ** 3)})
        del sets, outs
        torch.cuda.empty_cache()
    if args.grouped:
        R, N, K, G = [int(x) for x in args.grouped.split(",")]
        rows = routed_rows(G, R)
        ro = [0]
        for x in rows:
            ro.append(ro[-1] + x)
        d_rows = torch.tensor(ro, dtype=torch.int64, device="cuda")
        sets = [operands(R, K, G, N, seed=10 * i + 2) for i in range(args.buffers)]
        outs = [torch.zeros(R * N, dtype=torch.float32, device="cuda") for _ in range(args.buffers)]
        for nc in [int(x) for x in args.ncs.split(",")]:
            fns = {k: launcher(descs(sets, outs, nc, k, R * N, mode=cb.MM_GROUPED, M=G, N=N, K=K, d_rows=d_rows)) for k in modes}
            results.append({"case": "grouped", "rows": R, "N": N, "K": K, "experts": G, "max_rows": max(rows), "nc": nc,
                            **measure(fns, 2.0 * R * N * K)})
    print(json.dumps({**head, "steps": args.steps, "rounds": args.rounds, "buffers": args.buffers, "results": results}))


if __name__ == "__main__":
    main()
