"""GEMM_I8 beside GEMM_FP8, today's int8 route through MM_U32, and unprotected torch._int_mm, in one process: one JSON line.

For each square size (default 4096 and 8192), then the grouped case of tools/bench_grouped_mm.py (2^16 rows, N = K = 2048, 64
Zipf-routed experts), and NC 1/2/3, these alternate round by round:
  i8_bt    GEMM_I8, the caller's B^T read in place (COAST_MM_B_TRANSPOSED);
  i8_b     GEMM_I8, B through the byte-transposing pre-pass;
  fp8_bt, fp8_b  the same two for GEMM_FP8 on E4M3 operands of the same bytes' size;
  mm_u32   MM_U32 on the operands sign-extended to int32 (the protected int8 route before GEMM_I8: 4x the operand bytes);
  torch_int_mm  unprotected torch._int_mm (squares: A . (B^T)^T; grouped: one call per non-empty expert).
`--rounds` rounds of `--steps` launches each, after `--warmup`, over `--buffers` rotating operand sets so that a launch does not
find the previous one's operands in L2.  Times come from CUDA events.  Per case: seconds per launch (median of the rounds, and
their min and max), useful T multiply-adds x 2 per second (2 M N K / time, "useful_tops"), and each time over i8_bt's.  The card
name and its power limit are read in the same run; no device setting is changed.

    python tools/bench_gemm_i8.py [--sizes 4096,8192] [--ncs 1,2,3] [--steps 10] [--rounds 5] [--warmup 2] [--buffers 3]
                                  [--grouped 65536,2048,2048,64] [--skip mm_u32]
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
    ap.add_argument("--skip", default="", help="comma-separated kinds to leave out")
    args = ap.parse_args()
    import torch
    import coast_b200 as cb
    if not torch.cuda.is_available():
        sys.exit("bench_gemm_i8: no GPU; nothing is measured on a CPU")
    for k in ("COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT", "COAST_MM_PATH"):
        os.environ.pop(k, None)
    rt = cb.Runtime(0)
    head = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit()}
    L, stream = rt.L, rt.stream_handle()
    skip = {x for x in args.skip.split(",") if x}
    ncs = [int(x) for x in args.ncs.split(",")]

    def operand_set(rows, K, P, N, seed):
        """uniform int8 A (rows x K), B (P K x N) and B^T (P N x K); E4M3 A and B^T of integers in [-1, 1]"""
        g = torch.Generator(device="cuda").manual_seed(seed)
        A = torch.randint(-128, 128, (rows, K), device="cuda", generator=g, dtype=torch.int8)
        B = torch.randint(-128, 128, (P * K, N), device="cuda", generator=g, dtype=torch.int8)
        Bt = B.view(P, K, N).transpose(1, 2).contiguous().view(P * N, K)
        A8 = torch.randint(-1, 2, (rows, K), device="cuda", generator=g).float().to(torch.float8_e4m3fn)
        B8 = torch.randint(-1, 2, (P * K, N), device="cuda", generator=g).float().to(torch.float8_e4m3fn)
        B8t = B8.view(P, K, N).transpose(1, 2).contiguous().view(P * N, K)
        return dict(A=A, B=B, Bt=Bt, A8=A8, B8=B8, B8t=B8t)

    def launcher(descs):
        state = {"i": 0}

        def go():
            d = descs[state["i"] % len(descs)]
            state["i"] += 1
            rc = L.coast_launch(C.byref(d), stream)
            assert rc == 0, L.coast_last_error()
        return go

    def kinds(sets, outs, nc, n_units, mode=0, **kw):
        """the protected launches of one case, as functions that run one launch each"""
        fns = {}
        for name, kernel, a, b, bt in (("i8_bt", cb.K_GEMM_I8, "A", "Bt", True), ("i8_b", cb.K_GEMM_I8, "A", "B", False),
                                       ("fp8_bt", cb.K_GEMM_FP8, "A8", "B8t", True), ("fp8_b", cb.K_GEMM_FP8, "A8", "B8", False)):
            if name not in skip:
                m = mode | (cb.MM_B_TRANSPOSED if bt else 0)
                fns[name] = launcher([rt.make_desc(kernel, nc, s[a], o, n_units, d_aux=s[b], flags=3, mode=m, **kw)
                                      for s, o in zip(sets, outs)])
        if "mm_u32" not in skip:
            fns["mm_u32"] = launcher([rt.make_desc(cb.K_MM_U32, nc, s["A32"], o, n_units, d_aux=s["B32"], flags=3, mode=mode, **kw)
                                      for s, o in zip(sets, outs)])
        return fns

    def widen(sets):
        if "mm_u32" not in skip:
            for s in sets:
                s["A32"], s["B32"] = s["A"].to(torch.int32), s["B"].to(torch.int32)

    def measure(fns, flop):
        times = {k: [] for k in fns}
        for r in range(args.rounds):
            for k, fn in fns.items():
                times[k].append(timed(torch, fn, args.steps, args.warmup if r == 0 else 1))
        rt.sync()
        out = {k: {"s_per_launch": statistics.median(ts), "s_min": min(ts), "s_max": max(ts),
                   "useful_tops": flop / statistics.median(ts) / 1e12} for k, ts in times.items()}
        if "i8_bt" in out:
            for k in out:
                out[k]["over_i8_bt"] = out[k]["s_per_launch"] / out["i8_bt"]["s_per_launch"]
        return out

    def rotating(fn_of_set, sets):
        state = {"i": 0}

        def go():
            fn_of_set(sets[state["i"] % len(sets)])
            state["i"] += 1
        return go

    results = []
    for n in [int(x) for x in args.sizes.split(",") if x]:
        sets = [operand_set(n, n, 1, n, seed=10 * i + 1) for i in range(args.buffers)]
        widen(sets)
        outs = [torch.empty(n * n, dtype=torch.int32, device="cuda") for _ in range(args.buffers)]
        for nc in ncs:
            fns = kinds(sets, outs, nc, n * n, M=n, N=n, K=n)
            if "torch_int_mm" not in skip:
                fns["torch_int_mm"] = rotating(lambda s: torch._int_mm(s["A"], s["Bt"].t()), sets)
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
        sets = [operand_set(R, K, G, N, seed=10 * i + 2) for i in range(args.buffers)]
        widen(sets)
        outs = [torch.empty(R * N, dtype=torch.int32, device="cuda") for _ in range(args.buffers)]

        def experts(s):                                          # torch._int_mm needs more than 16 rows
            for g in range(G):
                if ro[g + 1] - ro[g] > 16:
                    torch._int_mm(s["A"][ro[g]:ro[g + 1]], s["Bt"][g * N:(g + 1) * N].t())
        for nc in ncs:
            fns = kinds(sets, outs, nc, R * N, mode=cb.MM_GROUPED, M=G, N=N, K=K, d_rows=d_rows)
            if "torch_int_mm" not in skip:
                fns["torch_int_mm"] = rotating(experts, sets)
            results.append({"case": "grouped", "rows": R, "N": N, "K": K, "experts": G, "max_rows": max(rows), "nc": nc,
                            **measure(fns, 2.0 * R * N * K)})
    print(json.dumps({**head, "steps": args.steps, "rounds": args.rounds, "buffers": args.buffers, "results": results}))


if __name__ == "__main__":
    main()
