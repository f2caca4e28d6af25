"""Grouped matmuls (COAST_MM_GROUPED) on a mixture-of-experts-like workload: one JSON line.

Workload: G experts share N and K; R routed rows are split over them by a skewed (Zipf, exponent 1.1) distribution, so a few
experts get most rows and some get none.  For the TF32 GEMM (integer-valued operands) and the exact u32 limb kernel, at NC 1/2/3:
  grouped : one grouped launch over the G products;
  padded  : one COAST_MM_BATCHED launch with every product padded to the largest row count (rounded up to 128 rows);
  loop    : G single launches, each product's rows padded to a multiple of 128 (TF32 and the limb kernel need that), empty
            products skipped (descriptors built beforehand, so the loop pays the launches, not Python).
Times come from CUDA events around `--steps` repetitions after `--warmup`.  Reported per case: the useful rate (2 R N K FLOP for
TF32, R N K multiply-adds for the exact kernel, per second), the padded and loop times as ratios to the grouped one, whether
the grouped outputs equal the loop's, and the share of the grouped launch's GPU time spent in its pre-passes (B transpose or
limb split, and the tile scan), from torch.profiler.  The card name and its power limit are read in the same run.

    python tools/bench_grouped_mm.py [--experts 64] [--rows 131072] [--n 4096] [--k 4096] [--steps 3] [--warmup 1]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PREPASSES = ("xmr_gemm_bt", "xmr_mm_grp_split_a", "xmr_mm_split_bt", "xmr_mm_group_scan")


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


def routed_rows(G, R, seed=1):
    import random
    rnd = random.Random(seed)
    w = [1.0 / (g + 1) ** 1.1 for g in range(G)]
    rnd.shuffle(w)
    rows = [int(R * x / sum(w)) for x in w]
    for g in range(G // 8):                                  # some experts get no tokens
        rows[rnd.randrange(G)] = 0
    rows[max(range(G), key=lambda g: rows[g])] += R - sum(rows)
    return rows


def prepass_share(torch, fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    pre = tot = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if not e.key.startswith("xmr_"):
            continue
        tot += t
        if e.key in PREPASSES:
            pre += t
    return pre / tot if tot else None


def run_case(rt, torch, cb, kind, nc, G, rows, N, K, steps, warmup):
    L, stream = rt.L, rt.stream_handle()
    kernel = cb.K_GEMM_TF32 if kind == "tf32" else cb.K_MM_U32
    R = sum(rows)
    ro = [0]
    for r in rows:
        ro.append(ro[-1] + r)
    pad = -(-max(rows) // 128) * 128
    dt = torch.float32 if kernel == cb.K_GEMM_TF32 else torch.int32
    if kernel == cb.K_GEMM_TF32:
        g = torch.Generator(device="cuda").manual_seed(1)
        A = torch.randint(-8, 9, (R * K,), dtype=dt, device="cuda", generator=g)
        B = torch.randint(-8, 9, (G * K * N,), dtype=dt, device="cuda", generator=g)
    else:
        A, B = torch.empty(R * K, dtype=dt, device="cuda"), torch.empty(G * K * N, dtype=dt, device="cuda")
        rt.fill_philox(A, seed=1)
        rt.fill_philox(B, seed=2)
    d_rows = torch.tensor(ro, dtype=torch.int64, device="cuda")
    C1 = torch.zeros(R * N, dtype=dt, device="cuda")
    grouped = rt.make_desc(kernel, nc, A, C1, R * N, mode=cb.MM_GROUPED, M=G, N=N, K=K, d_aux=B, d_rows=d_rows)

    def launch(d):
        rc = L.coast_launch(C.byref(d), stream)
        assert rc == 0, L.coast_last_error()

    t_grp = timed(torch, lambda: launch(grouped), steps, warmup)
    share = prepass_share(torch, lambda: launch(grouped))
    rt.sync()
    # loop of single launches on 128-row padded copies of each product's A (C rows past the product are scratch)
    Ap = torch.zeros(sum(-(-r // 128) * 128 for r in rows) * K, dtype=dt, device="cuda")
    Cp = torch.zeros(Ap.numel() // K * N, dtype=dt, device="cuda")
    singles, off = [], 0
    for gi, r in enumerate(rows):
        if r == 0:
            continue
        m = -(-r // 128) * 128
        Ap[off * K:(off + r) * K] = A[ro[gi] * K:ro[gi + 1] * K]
        singles.append(rt.make_desc(kernel, nc, Ap[off * K:(off + m) * K], Cp[off * N:(off + m) * N], m * N, M=m, N=N, K=K,
                                    d_aux=B[gi * K * N:(gi + 1) * K * N], unit_base=ro[gi] * N))
        off += m
    t_loop = timed(torch, lambda: [launch(d) for d in singles], steps, warmup)
    rt.sync()
    same, off = True, 0
    for gi, r in enumerate(rows):
        if r:
            same &= bool(torch.equal(Cp[off * N:(off + r) * N].view(torch.int32), C1[ro[gi] * N:ro[gi + 1] * N].view(torch.int32)))
            off += -(-r // 128) * 128
    del Ap, Cp
    torch.cuda.empty_cache()
    # padded batched launch: every product at the largest row count
    t_pad = None
    need = G * pad * (K + N) * 4 * (2 if kernel == cb.K_MM_U32 else 1)
    if torch.cuda.mem_get_info()[0] > need + (4 << 30):
        Apad = torch.zeros(G * pad * K, dtype=dt, device="cuda")
        Cpad = torch.zeros(G * pad * N, dtype=dt, device="cuda")
        batched = rt.make_desc(kernel, nc, Apad, Cpad, G * pad * N, mode=cb.MM_BATCHED, M=pad, N=N, K=K, d_aux=B)
        t_pad = timed(torch, lambda: launch(batched), steps, warmup)
        rt.sync()
        del Apad, Cpad
        torch.cuda.empty_cache()
    useful = R * N * K * (2 if kernel == cb.K_GEMM_TF32 else 1)
    unit, scale = ("tflops", 1e12) if kernel == cb.K_GEMM_TF32 else ("tmacs", 1e12)
    return {"kernel": kind, "nc": nc, "experts": G, "rows": R, "max_rows": max(rows), "empty_experts": rows.count(0), "N": N, "K": K,
            "grouped_s": t_grp, f"useful_{unit}": useful / t_grp / scale,
            "padded_batched_s": t_pad, "padded_over_grouped": t_pad / t_grp if t_pad else None,
            "loop_s": t_loop, "loop_over_grouped": t_loop / t_grp, "prepass_share": share, "outputs_equal_loop": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--experts", type=int, default=64)
    ap.add_argument("--rows", type=int, default=1 << 17)
    ap.add_argument("--n", type=int, default=4096)
    ap.add_argument("--k", type=int, default=4096)
    ap.add_argument("--kernels", default="tf32,limb")
    ap.add_argument("--ncs", default="1,2,3")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    import torch
    import coast_b200 as cb
    for k in ("COAST_MM_PATH", "COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT"):
        os.environ.pop(k, None)
    rt = cb.Runtime(0)
    rows = routed_rows(args.experts, args.rows)
    res = [run_case(rt, torch, cb, kind, int(nc), args.experts, rows, args.n, args.k, args.steps, args.warmup)
           for kind in args.kernels.split(",") for nc in args.ncs.split(",")]
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit(), "steps": args.steps,
                      "results": res}))


if __name__ == "__main__":
    main()
