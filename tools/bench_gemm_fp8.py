"""GEMM_FP8 beside GEMM_BF16 on the same shapes, in one process: one JSON line.

For each square size (default 4096 and 8192) and NC 1/2/3, three launches alternate: GEMM_FP8 with B (K x N, which the byte
pre-pass transposes), GEMM_FP8 with B^T (COAST_MM_B_TRANSPOSED, read in place) and GEMM_BF16 with B (`--rounds` rounds of
`--steps` launches each, after `--warmup`), each over `--buffers` rotating operand sets so that a launch does not find the
previous one's operands in L2.  Times come from CUDA events and include everything a launch enqueues; the pre-pass's own time
is taken from torch.profiler in a run of its own and reported as a share of the launch.  Per case: seconds per launch (median
of the rounds, and their spread), useful TFLOP/s (2 M N K), issued TFLOP/s (NC times that: every replica's wgmma runs), and both
as a share of the data-sheet dense peak of the operand type (1,979 TFLOP/s FP8, 989 TFLOP/s BF16: NVIDIA's figures for an H100
SXM at 700 W, not rates reached here).  The vendor reference is unprotected torch._scaled_mm (E4M3, scales 1.0, fp32 out, fast
accumulation) on the same operands, timed in the same rounds.  Then the grouped case (2^16 rows, N = K = 2048, 64 Zipf-routed
experts).  The card name and its power limit are read in the same run; no device setting is changed.

--numerics (instead of timing) measures what the FP8 path computes rather than how fast: the width of the tensor core's FP8
accumulator (one product of 2^16 and K - 1 products of 2^(16 - d) per row, against the exact sum), and, on uniform(-1, 1)
operands rounded to E4M3, max |C - C64| / sum_k |a_ik b_kj| for the protected kernel and for torch._scaled_mm with fast
accumulation on and off.

    python tools/bench_gemm_fp8.py [--sizes 4096,8192] [--ncs 1,2,3] [--steps 10] [--rounds 3] [--warmup 2] [--buffers 3]
    python tools/bench_gemm_fp8.py --numerics
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_grouped_mm import power_limit, routed_rows, timed  # noqa: E402

PEAK = {"fp8": 1979e12, "fp8_bt": 1979e12, "bf16": 989e12, "scaled_mm": 1979e12}   # data-sheet dense FLOP/s, H100 SXM at 700 W


def operands(torch, kind, rows, K, n_b, N, seed):
    """integer operands in [-1, 1]: the same values in either type; FP8 B is K x N, its B^T N x K per product"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randint(-1, 2, (rows, K), dtype=torch.int32, device="cuda", generator=g)
    B = torch.randint(-1, 2, (n_b, K, N), dtype=torch.int32, device="cuda", generator=g)
    if kind == "bf16":
        return A.to(torch.bfloat16), B.to(torch.bfloat16)
    A8 = A.to(torch.float32).to(torch.float8_e4m3fn)
    B8 = B.to(torch.float32).to(torch.float8_e4m3fn)
    return A8, (B8.transpose(1, 2).contiguous() if kind == "fp8_bt" else B8)


def prepass_seconds(torch, fn, names=("xmr_gemm_bt_u8", "xmr_mm_group_scan")):
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


def numerics(torch, rt, cb):
    """the accumulator width and the general-operand error ratios (see the module text)"""
    f8 = torch.float8_e4m3fn
    one = torch.ones((), device="cuda")

    def protected(A, Bt, nc=1):
        M, K = A.shape
        N = Bt.shape[0]
        out, _ = rt.run(cb.K_GEMM_FP8, nc, A.contiguous(), M * N, M=M, N=N, K=K, aux=Bt.contiguous(), mode=cb.MM_B_TRANSPOSED,
                        out=torch.empty(M * N, dtype=torch.float32, device="cuda"))
        return out.view(torch.float32).view(M, N).double()

    def scaled(A, Bt, fast):
        return torch._scaled_mm(A, Bt.t(), scale_a=one, scale_b=one, out_dtype=torch.float32, use_fast_accum=fast).double()

    width = []
    M = N = 128
    ea = 8 - (torch.arange(M, device="cuda") % 18).double()                # row i: a = 2^ea, ea = 8 .. -9
    eb = torch.where(torch.arange(N, device="cuda") % 2 == 0, 8.0, 0.0).double()   # even columns b = 2^8, odd b = 1
    small = torch.pow(2.0, ea[:, None] + eb[None, :])                      # the K - 1 small products of element (i, j)
    ratio = (16 - ea[:, None] - eb[None, :]).long()                        # log2 of 2^16 over a small product: 0 .. 25
    for K in (128, 1024, 4096):
        A = torch.empty(M, K, dtype=torch.float64, device="cuda")
        Bt = torch.empty(N, K, dtype=torch.float64, device="cuda")
        A[:, 0], Bt[:, 0] = 256.0, 256.0                                   # one product of 2^16 at k = 0
        A[:, 1:], Bt[:, 1:] = torch.pow(2.0, ea)[:, None], torch.pow(2.0, eb)[:, None]
        A8, Bt8 = A.float().to(f8), Bt.float().to(f8)
        exact = 65536.0 + (K - 1) * small
        row = {"K": K}
        for name, c in (("protected", protected(A8, Bt8)), ("scaled_mm_fast", scaled(A8, Bt8, True)), ("scaled_mm", scaled(A8, Bt8, False))):
            ok = c == exact
            arrived = (c - 65536.0) / small / (K - 1)                       # share of the small products' sum that arrived
            row[name] = {"exact_up_to_ratio_log2": max([r for r in range(26) if ok[ratio <= r].all()] or [-1]),
                         "arrived_share_by_ratio_log2": {r: float(arrived[ratio == r].min()) for r in range(26)}}
        width.append(row)
    bound = []
    for M, N, K in ((512, 768, 512), (1024, 1024, 2048), (256, 384, 8192)):
        g = torch.Generator(device="cuda").manual_seed(K)
        A = (torch.rand(M, K, device="cuda", generator=g) * 2 - 1).to(f8)
        Bt = (torch.rand(N, K, device="cuda", generator=g) * 2 - 1).to(f8)
        c64 = A.float().double() @ Bt.float().double().t()
        s = A.float().double().abs() @ Bt.float().double().abs().t()
        r = {"M": M, "N": N, "K": K}
        for name, c in (("protected", protected(A, Bt)), ("scaled_mm_fast", scaled(A, Bt, True)), ("scaled_mm", scaled(A, Bt, False))):
            r[name] = float(((c - c64).abs() / s).max())
        bound.append(r)
    return {"accumulator": width, "general_operand_ratio": bound}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="4096,8192")
    ap.add_argument("--ncs", default="1,2,3")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--buffers", type=int, default=3)
    ap.add_argument("--grouped", default="65536,2048,2048,64", help="rows,N,K,experts of the grouped case ('' skips it)")
    ap.add_argument("--numerics", action="store_true")
    args = ap.parse_args()
    import torch
    import coast_b200 as cb
    if not torch.cuda.is_available():
        sys.exit("bench_gemm_fp8: no GPU; nothing is measured on a CPU")
    for k in ("COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT"):
        os.environ.pop(k, None)
    rt = cb.Runtime(0)
    head = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit()}
    if args.numerics:
        print(json.dumps({**head, **numerics(torch, rt, cb)}))
        return
    L, stream = rt.L, rt.stream_handle()
    kid = {"fp8": cb.K_GEMM_FP8, "fp8_bt": cb.K_GEMM_FP8, "bf16": cb.K_GEMM_BF16}
    bt_mode = {"fp8": 0, "fp8_bt": cb.MM_B_TRANSPOSED, "bf16": 0}
    one = torch.ones((), device="cuda")

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
            m = 1 if k == "scaled_mm" else nc
            out[k] = {"s_per_launch": t, "s_min": min(ts), "s_max": max(ts), "useful_tflops": flop / t / 1e12,
                      "issued_tflops": m * flop / t / 1e12, "useful_share_of_datasheet_peak": flop / t / PEAK[k],
                      "issued_share_of_datasheet_peak": m * flop / t / PEAK[k]}
        return out

    results = []
    for n in [int(x) for x in args.sizes.split(",") if x]:
        sets = {k: [operands(torch, k, n, n, 1, n, seed=10 * i + 1) for i in range(args.buffers)] for k in kid}
        outs = [torch.empty(n * n, dtype=torch.float32, device="cuda") for _ in range(args.buffers)]
        state = {"i": 0}

        def vendor():
            A, Bt = sets["fp8_bt"][state["i"] % args.buffers]
            state["i"] += 1
            torch._scaled_mm(A, Bt[0].t(), scale_a=one, scale_b=one, out_dtype=torch.float32, use_fast_accum=True)
        for nc in [int(x) for x in args.ncs.split(",")]:
            fns = {k: launcher([rt.make_desc(kid[k], nc, A, o, n * n, M=n, N=n, K=n, d_aux=B, mode=bt_mode[k], flags=3)
                                for (A, B), o in zip(sets[k], outs)]) for k in kid}
            fns["scaled_mm"] = vendor
            r = measure(fns, 2.0 * n ** 3, nc)
            for k in ("fp8", "fp8_bt"):
                r[k]["prepass_share"] = prepass_seconds(torch, fns[k]) / r[k]["s_per_launch"]
            results.append({"case": "square", "M": n, "N": n, "K": n, "nc": nc, **r,
                            "fp8_over_bf16_speed": r["bf16"]["s_per_launch"] / r["fp8"]["s_per_launch"],
                            "fp8_bt_over_bf16_speed": r["bf16"]["s_per_launch"] / r["fp8_bt"]["s_per_launch"]})
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
            fns = {k: launcher([rt.make_desc(kid[k], nc, A, o, R * N, mode=cb.MM_GROUPED | bt_mode[k], M=G, N=N, K=K, d_aux=B,
                                             d_rows=d_rows, flags=3) for (A, B), o in zip(sets[k], outs)]) for k in kid}
            r = measure(fns, 2.0 * R * N * K, nc)
            for k in kid:
                r[k]["prepass_share"] = prepass_seconds(torch, fns[k]) / r[k]["s_per_launch"]
            results.append({"case": "grouped", "rows": R, "N": N, "K": K, "experts": G, "max_rows": max(rows), "nc": nc, **r,
                            "fp8_over_bf16_speed": r["bf16"]["s_per_launch"] / r["fp8"]["s_per_launch"],
                            "fp8_bt_over_bf16_speed": r["bf16"]["s_per_launch"] / r["fp8_bt"]["s_per_launch"]})
    print(json.dumps({**head, "steps": args.steps, "rounds": args.rounds, "buffers": args.buffers,
                      "datasheet_peak_tflops": {k: v / 1e12 for k, v in PEAK.items()}, "results": results}))


if __name__ == "__main__":
    main()
