"""Ragged SHA-256 / CRC16 / quicksort batches (COAST_UNIT_OFFSETS) against the uniform kernels: one JSON line.

Configs (TMR): SHA-256 on 2^20 messages of lengths uniform in [0, 4096); SHA-256 on 2^22 messages of a skewed lognormal mix
(median 256 B, capped at 64 KiB); CRC16 on 2^24 messages of lengths uniform in [0, 255]; quicksort (qsort_uniform, only when
asked for) on 2^20 int32 arrays of lengths uniform in [0, 1024] elements.  Data is Philox.  For each: input MB/s and
compressions/s (SHA), bytes/s (CRC) or elements/s (quicksort) over CUDA events around >= 20 launches after a warm-up, input
buffers rotated so no launch finds its input in L2; the ratio to a uniform launch (general path for SHA-256 and CRC16,
xmr_qsort for quicksort) with the same replica count and the same total work (units of the mean length); the pre-pass
kernels' share of the time from torch.profiler in a run of its own; and the warp efficiency of the schedule (sum of costs /
sum over warp-tiles of max cost x units), computed on the CPU from the lengths with and without the cost ordering.  For
quicksort that last number is an estimate from the lengths alone: the work of one array depends on its data, not only on
its length.  The card name and its power limit are read in the same run.

    python tools/bench_ragged.py [--steps 20] [--warmup 3] [--configs sha_uniform,sha_lognormal,crc_uniform,qsort_uniform]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def lengths(cfg, rng):
    if cfg == "sha_uniform":
        return rng.integers(0, 4096, 1 << 20), 4095
    if cfg == "sha_lognormal":
        return np.minimum(rng.lognormal(np.log(256.0), 1.0, 1 << 22).astype(np.int64), 1 << 16), 1 << 16
    if cfg == "qsort_uniform":                                # bytes of int32 arrays of 0..1024 elements
        return 4 * rng.integers(0, 1025, 1 << 20), 4096
    return rng.integers(0, 256, 1 << 24), 255


def cost(cfg, L):
    if cfg.startswith("qsort"):
        return L // 4                                         # elements: an estimate, the data decides the real work
    return (L + 8) // 64 + 1 if cfg.startswith("sha") else L


def warp_efficiency(c, upw):
    """sum of costs / sum over warp-tiles of (max cost x units per tile)"""
    n = len(c) // upw * upw
    tiles = c[:n].reshape(-1, upw)
    return float(tiles.sum() / (tiles.max(axis=1).sum() * upw))


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:                                         # a number we could not read is reported as missing
        return None


def timed(torch, launch, steps, warmup):
    for i in range(warmup):
        launch(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        launch(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--configs", default="sha_uniform,sha_lognormal,crc_uniform")
    args = ap.parse_args()
    import torch
    import coast_b200 as cb
    rt = cb.Runtime(0)
    rng = np.random.default_rng(2026)
    res = {"device": torch.cuda.get_device_name(0), "power_limit_w": power_limit(), "steps": max(args.steps, 20), "configs": {}}
    steps = res["steps"]
    for cfg in args.configs.split(","):
        kernel = cb.K_SHA256 if cfg.startswith("sha") else cb.K_QSORT if cfg.startswith("qsort") else cb.K_CRC16
        L, bound = lengths(cfg, rng)
        n = len(L)
        off_h = np.concatenate([[0], np.cumsum(L)]).astype(np.int64)
        total = int(off_h[-1])
        off = torch.from_numpy(off_h).cuda()
        bufs = []                                             # two input buffers, each far larger than L2, used in turn
        for s in range(2):
            b = torch.empty((total + 64) // 4 * 4, dtype=torch.uint8, device="cuda")
            rt.fill_philox(b, seed=s + 1)
            bufs.append(b)
        out = torch.empty(total + 64 if kernel == cb.K_QSORT else n * (32 if kernel == cb.K_SHA256 else 2), dtype=torch.uint8,
                          device="cuda")
        flags = cb.F_COUNT_ERRORS | cb.F_COUNT_SYNCS

        def ragged(i):
            rt.launch(rt.make_desc(kernel, 3, bufs[i % 2], out, n, flags=flags, mode=cb.UNIT_OFFSETS, unit_bytes=bound, d_aux=off))
        mean = max(int(round(total / n)), 1)
        if kernel == cb.K_QSORT:
            mean = max(int(round(total / n / 4)), 1) * 4          # whole elements
        if kernel == cb.K_SHA256 and mean == 64:
            mean = 65                                         # 64-byte messages take the TMA ring kernels, not the general path

        def uniform(i):
            rt.launch(rt.make_desc(kernel, 3, bufs[i % 2], out, min(n, total // mean), flags=flags, unit_bytes=mean))
        t_r = timed(torch, ragged, steps, args.warmup)
        t_u = timed(torch, uniform, steps, args.warmup)
        st = rt.sync()
        assert st.errors_corrected == 0 and st.injected == 0
        n_u = min(n, total // mean)
        c = cost(cfg, L)
        work_r = int(c.sum()) if kernel != cb.K_CRC16 else total
        work_u = n_u * ((mean + 8) // 64 + 1) if kernel == cb.K_SHA256 else n_u * mean // 4 if kernel == cb.K_QSORT else n_u * mean
        rate_r, rate_u = work_r / t_r, work_u / t_u
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for i in range(5):
                ragged(i)
            torch.cuda.synchronize()
        k = {e.key: e.device_time_total for e in prof.key_averages()}
        pre = sum(v for kk, v in k.items() if kk.startswith("xmr_ragged_"))
        upw = 32 // 3
        order = np.argsort(-c, kind="stable")
        res["configs"][cfg] = {
            "n": n, "input_bytes": total, "mean_len": total / n, "ms_ragged": t_r * 1e3, "ms_uniform": t_u * 1e3,
            "input_MBps": total / t_r / 1e6,
            {cb.K_SHA256: "compressions_per_s", cb.K_QSORT: "elements_per_s"}.get(kernel, "bytes_per_s"): rate_r,
            "uniform_rate": rate_u, "ratio_to_uniform": rate_r / rate_u,
            "prepass_share": pre / max(sum(k.values()), 1e-9),
            "warp_eff_unsorted": warp_efficiency(c, upw), "warp_eff_sorted": warp_efficiency(c[order], upw),
            **({"warp_eff_is_estimate_from_lengths": True} if kernel == cb.K_QSORT else {}),
        }
        del bufs, out, off
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
