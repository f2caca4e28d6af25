"""Matmuls on a transposed B (COAST_MM_B_TRANSPOSED) beside the B launch, in one process: one JSON line.

A caller holding linear-layer weights has W = B^T (N x K).  Three ways to compute x @ W.T are timed, alternating in each round:
  b       : the B launch on a B (K x N) that is already there;
  bt      : the launch with the bit on W itself;
  today   : what such a caller had to do before the bit: W.t().contiguous() (a torch copy) and then the B launch.
For GEMM_TF32 and GEMM_BF16 at each square size and NC, and for the grouped 64-expert Zipf workload of tools/bench_grouped_mm.py
for TF32, BF16 and the exact u32 limb kernel (MM_U32 on its tensor-core path).  Times come from CUDA events: the median of
`--rounds` rounds of `--steps` launches each after `--warmup`, with the rounds' spread (min, max).  The outputs of b and bt are
compared bit for bit on the same seeded operands.  The card name and its power limit are read in the same run; no device
setting is changed.

    python tools/bench_mm_bt.py [--sizes 4096,8192] [--ncs 1,2,3] [--steps 10] [--rounds 5] [--warmup 2]
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


def operands(torch, kind, rows, K, n_b, N, seed):
    """A (rows x K) and W = B^T (n_b x N x K), integer-valued in the kernel's element type"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "mm_u32":
        return (torch.randint(-2 ** 31, 2 ** 31 - 1, (rows, K), dtype=torch.int32, device="cuda", generator=g),
                torch.randint(-2 ** 31, 2 ** 31 - 1, (n_b, N, K), dtype=torch.int32, device="cuda", generator=g))
    dt = torch.bfloat16 if kind == "bf16" else torch.float32
    return (torch.randint(-8, 9, (rows, K), dtype=torch.int32, device="cuda", generator=g).to(dt),
            torch.randint(-8, 9, (n_b, N, K), dtype=torch.int32, device="cuda", generator=g).to(dt))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="4096,8192")
    ap.add_argument("--ncs", default="1,2,3")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--grouped", default="65536,2048,2048,64", help="rows,N,K,experts of the grouped case ('' skips it)")
    args = ap.parse_args()
    import torch
    import coast_b200 as cb
    if not torch.cuda.is_available():
        sys.exit("bench_mm_bt: no GPU; nothing is measured on a CPU")
    for k in ("COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT", "COAST_MM_PATH"):
        os.environ.pop(k, None)
    rt = cb.Runtime(0)
    L, stream = rt.L, rt.stream_handle()
    kid = {"tf32": cb.K_GEMM_TF32, "bf16": cb.K_GEMM_BF16, "mm_u32": cb.K_MM_U32}

    def launch(d):
        rc = L.coast_launch(C.byref(d), stream)
        assert rc == 0, L.coast_last_error()

    def measure(fns):
        times = {k: [] for k in fns}
        for r in range(args.rounds):
            for k, fn in fns.items():
                times[k].append(timed(torch, fn, args.steps, args.warmup if r == 0 else 1))
        rt.sync()
        return {k: {"s_per_launch": statistics.median(ts), "s_min": min(ts), "s_max": max(ts)} for k, ts in times.items()}

    def case(kind, nc, A, W, rows, N, K, mode=0, **kw):
        """b / bt / today on one operand set; the outputs of b and bt compared"""
        B = W.transpose(1, 2).contiguous()
        n = rows * N
        dt = torch.int32 if kind == "mm_u32" else torch.float32
        ob, ot, oc = (torch.zeros(n, dtype=dt, device="cuda") for _ in range(3))
        Wf = W.reshape(-1, K)
        db = rt.make_desc(kid[kind], nc, A, ob, n, mode=mode, N=N, K=K, d_aux=B, flags=3, **kw)
        dbt = rt.make_desc(kid[kind], nc, A, ot, n, mode=mode | cb.MM_B_TRANSPOSED, N=N, K=K, d_aux=Wf, flags=3, **kw)
        scratch = {}

        def today():
            Bc = W.transpose(1, 2).contiguous()                  # the caller's copy, then the B launch on it
            scratch["d"] = rt.make_desc(kid[kind], nc, A, oc, n, mode=mode, N=N, K=K, d_aux=Bc, flags=3, **kw)
            launch(scratch["d"])
        r = measure({"b": lambda: launch(db), "bt": lambda: launch(dbt), "today": today})
        r["outputs_equal"] = bool(torch.equal(ob, ot)) and bool(torch.equal(ob, oc))
        r["bt_over_b"] = r["bt"]["s_per_launch"] / r["b"]["s_per_launch"]
        r["today_over_bt"] = r["today"]["s_per_launch"] / r["bt"]["s_per_launch"]
        return r

    results = []
    for sz in [int(x) for x in args.sizes.split(",") if x]:
        for kind in ("tf32", "bf16"):
            A, W = operands(torch, kind, sz, sz, 1, sz, seed=sz)
            for nc in [int(x) for x in args.ncs.split(",")]:
                r = case(kind, nc, A, W, sz, sz, sz, M=sz)
                results.append({"case": "square", "kernel": kind, "M": sz, "N": sz, "K": sz, "nc": nc, **r})
            del A, W
            torch.cuda.empty_cache()
    if args.grouped:
        R, N, K, G = [int(x) for x in args.grouped.split(",")]
        rows = routed_rows(G, R)
        ro = [0]
        for x in rows:
            ro.append(ro[-1] + x)
        d_rows = torch.tensor(ro, dtype=torch.int64, device="cuda")
        for kind in ("tf32", "bf16", "mm_u32"):
            A, W = operands(torch, kind, R, K, G, N, seed=2)
            for nc in [int(x) for x in args.ncs.split(",")]:
                r = case(kind, nc, A, W, R, N, K, mode=cb.MM_GROUPED, M=G, d_rows=d_rows)
                results.append({"case": "grouped", "kernel": kind, "rows": R, "N": N, "K": K, "experts": G, "max_rows": max(rows),
                                "nc": nc, **r})
            del A, W
            torch.cuda.empty_cache()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit(), "steps": args.steps, "rounds": args.rounds,
                      "results": results}))


if __name__ == "__main__":
    main()
