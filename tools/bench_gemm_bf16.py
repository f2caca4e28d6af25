"""GEMM_BF16 beside GEMM_TF32 on the same shapes, in one process: one JSON line.

For each square size (default 4096 and 8192) and NC 1/2/3 the two kernels are launched alternately (`--rounds` rounds of
`--steps` launches each, after `--warmup`), each over `--buffers` rotating operand sets so that a launch does not find the
previous one's operands in L2.  Times come from CUDA events and include everything a launch enqueues: for TF32 that is the
B transpose pre-pass, whose own time is reported beside it (CUDA events around that kernel alone are not available from outside
the library, so it is taken from torch.profiler in a run of its own); BF16 has no pre-pass.  Per case: seconds per launch (median
of the rounds, and their spread), useful TFLOP/s (2 M N K), issued TFLOP/s (NC times that: every replica's wgmma runs), and both
as a share of the data-sheet dense peak of the operand type (989 TFLOP/s BF16, 495 TFLOP/s TF32: NVIDIA's figures for an H100
SXM at 700 W, not rates reached here).  Then the grouped case (2^16 rows, N = K = 2048, 64 Zipf-routed experts) for both types.
The card name and its power limit are read in the same run; no device setting is changed.

    python tools/bench_gemm_bf16.py [--sizes 4096,8192] [--ncs 1,2,3] [--steps 10] [--rounds 3] [--warmup 2] [--buffers 3]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_grouped_mm import power_limit, routed_rows, timed  # noqa: E402

PEAK = {"bf16": 989e12, "tf32": 495e12}                     # data-sheet dense TFLOP/s, H100 SXM at 700 W


def operands(torch, kind, rows, K, n_b, N, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dt = torch.bfloat16 if kind == "bf16" else torch.float32
    A = torch.randint(-8, 9, (rows * K,), dtype=torch.int32, device="cuda", generator=g).to(dt)
    B = torch.randint(-8, 9, (n_b * K * N,), dtype=torch.int32, device="cuda", generator=g).to(dt)
    return A, B


def prepass_seconds(torch, fn, names=("xmr_gemm_bt", "xmr_mm_group_scan")):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    t = 0.0
    for e in prof.key_averages():
        if e.key in names:
            t += getattr(e, "device_time_total", None) or e.cuda_time_total
    return t / 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="4096,8192")
    ap.add_argument("--ncs", default="1,2,3")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--buffers", type=int, default=3)
    ap.add_argument("--grouped", default="65536,2048,2048,64", help="rows,N,K,experts of the grouped case ('' skips it)")
    args = ap.parse_args()
    import torch
    import coast_b200 as cb
    if not torch.cuda.is_available():
        sys.exit("bench_gemm_bf16: no GPU; nothing is measured on a CPU")
    for k in ("COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT"):
        os.environ.pop(k, None)
    rt = cb.Runtime(0)
    L, stream = rt.L, rt.stream_handle()
    kid = {"bf16": cb.K_GEMM_BF16, "tf32": cb.K_GEMM_TF32}

    def launcher(descs):
        state = {"i": 0}

        def go():
            d = descs[state["i"] % len(descs)]
            state["i"] += 1
            rc = L.coast_launch(C.byref(d), stream)
            assert rc == 0, L.coast_last_error()
        return go

    def measure(fns, flop, nc):
        """fns: {kind: launch}; alternating rounds"""
        times = {k: [] for k in fns}
        for r in range(args.rounds):
            for k, fn in fns.items():
                times[k].append(timed(torch, fn, args.steps, args.warmup if r == 0 else 1))
        rt.sync()
        out = {}
        for k, ts in times.items():
            t = statistics.median(ts)
            out[k] = {"s_per_launch": t, "s_min": min(ts), "s_max": max(ts), "useful_tflops": flop / t / 1e12,
                      "issued_tflops": nc * flop / t / 1e12, "useful_share_of_datasheet_peak": flop / t / PEAK[k],
                      "issued_share_of_datasheet_peak": nc * flop / t / PEAK[k]}
        return out

    results = []
    for n in [int(x) for x in args.sizes.split(",") if x]:
        sets = {k: [operands(torch, k, n, n, 1, n, seed=10 * i + 1) for i in range(args.buffers)] for k in kid}
        outs = [torch.empty(n * n, dtype=torch.float32, device="cuda") for _ in range(args.buffers)]
        for nc in [int(x) for x in args.ncs.split(",")]:
            fns = {k: launcher([rt.make_desc(kid[k], nc, A, o, n * n, M=n, N=n, K=n, d_aux=B, flags=3) for (A, B), o in zip(sets[k], outs)])
                   for k in kid}
            r = measure(fns, 2.0 * n ** 3, nc)
            r["tf32"]["prepass_s"] = prepass_seconds(torch, fns["tf32"])
            r["bf16"]["prepass_s"] = prepass_seconds(torch, fns["bf16"])
            results.append({"case": "square", "M": n, "N": n, "K": n, "nc": nc, **r,
                            "bf16_over_tf32_speed": r["tf32"]["s_per_launch"] / r["bf16"]["s_per_launch"]})
        del sets, outs
        torch.cuda.empty_cache()
    if args.grouped:
        R, N, K, G = [int(x) for x in args.grouped.split(",")]
        rows = routed_rows(G, R)
        ro = [0]
        for x in rows:
            ro.append(ro[-1] + x)
        d_rows = torch.tensor(ro, dtype=torch.int64, device="cuda")
        sets = {k: [operands(torch, k, R, K, G, N, seed=10 * i + 2) for i in range(args.buffers)] for k in kid}
        outs = [torch.zeros(R * N, dtype=torch.float32, device="cuda") for _ in range(args.buffers)]
        for nc in [int(x) for x in args.ncs.split(",")]:
            fns = {k: launcher([rt.make_desc(kid[k], nc, A, o, R * N, mode=cb.MM_GROUPED, M=G, N=N, K=K, d_aux=B, d_rows=d_rows, flags=3)
                                for (A, B), o in zip(sets[k], outs)]) for k in kid}
            r = measure(fns, 2.0 * R * N * K, nc)
            for k in kid:
                r[k]["prepass_s"] = prepass_seconds(torch, fns[k])
            results.append({"case": "grouped", "rows": R, "N": N, "K": K, "experts": G, "max_rows": max(rows), "nc": nc, **r,
                            "bf16_over_tf32_speed": r["tf32"]["s_per_launch"] / r["bf16"]["s_per_launch"]})
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit(), "steps": args.steps, "rounds": args.rounds,
                      "buffers": args.buffers, "datasheet_peak_tflops": {k: v / 1e12 for k, v in PEAK.items()}, "results": results}))


if __name__ == "__main__":
    main()
