"""Integer pipe rates on the GPU, and how close the SHA-256 TMR kernel runs to its ALU-pipe floor.

    python tools/sha_pipe_rates.py [--json OUT] [--skip-bench] [--skip-sha]

1. Builds a small standalone sm_90a cubin of instruction streams with the nvcc the project builds with, loads it
   through the driver API (cuModuleLoadData, as coast_rt.c does) and times each stream with clock64().  Every stream
   is 8 independent dependency chains per thread, 8 warps per sub-partition, so issue, not latency, bounds it.
   The loop body's SASS is read back: the report gives the opcodes that really ran, not the ones the source asked for.
   The viadd+shf mix decides which pipe VIADD issues on (viadd_pipe).
2. Runs `bench.py --workload sha256` and sets its roofline.kernel_ms (at the delivered SM clock) against the static
   ALU floor of xmr_sha256_b64_seg_nc3_inj0: ALU-pipe instructions in its SASS x warps / sub-partitions / measured
   ALU rate, with VIADD on the pipe measured for it; the floors with and without VIADD on the ALU pipe are reported
   beside it.  Above 1.25x the floor the ALU pipe is not what bounds the kernel.
3. Times the other SHA-256 kernels (interleaved 64-byte NC 1/2/3, general length) with CUDA events.

Rates are warp instructions per clock per SM sub-partition (4 per SM).  The card's name and power limit are read in
the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEG_KERNEL = "xmr_sha256_b64_seg_nc3_inj0"

# opcode -> pipe, for the opcodes the SHA-256 kernels issue in their rounds (the rest is counted as "other")
ALU_OPS = {"SHF", "LOP3", "IADD3", "PRMT", "ISETP", "LEA", "SEL", "MOV", "LOP", "SHL", "SHR", "IABS", "FLO", "POPC", "BREV"}
IMAD_OPS = {"IMAD", "HFMA2"}


def pipe_of(op: str) -> str:
    base = op.split(".")[0]
    if base in ALU_OPS:
        return "alu"
    if base in IMAD_OPS:
        return "imad"
    return "other"


def viadd_pipe(rates: dict) -> str:
    """'alu' or 'imad': the pipe VIADD issues on, from the measured viadd+shf mix.  Each pipe takes one warp instruction
    every 2 cycles; a VIADD + SHF stream reaches about 1 per cycle only if the two go to different pipes."""
    return "imad" if rates["viadd_shf_1_1"]["warp_inst_per_clk_per_smsp"]["all"] > 0.75 else "alu"


def pipe_of_measured(op: str, viadd: str) -> str:
    """pipe_of, with VIADD (which pipe_of leaves under "other") on the pipe the probe measured for it"""
    return viadd if op.split(".")[0] == "VIADD" else pipe_of(op)


# --- 1. the probe cubin ------------------------------------------------------------------------------------------------
# Each op updates chain x[i] from itself and its neighbour x[(i+1)&7] (so ptxas cannot fuse a chain into fewer
# instructions) and from values it cannot know (loaded from memory).  Multipliers come from the constant bank, as in
# the SHA-256 kernel, or from a register.
PROBE_OPS = {
    "shf_r_w":      ('asm("shf.r.wrap.b32 %0, %1, %2, 7;" : "=r"(X) : "r"(X), "r"(Y));', "SHF.R.W"),
    "shf_r_u32_hi": ('X = (X ^ 0u) >> (s & 31u); X ^= 0u;', "SHF.R.U32.HI"),
    "lop3":         ('asm("lop3.b32 %0, %1, %2, %3, 0x96;" : "=r"(X) : "r"(X), "r"(Y), "r"(v));', "LOP3"),
    "iadd3":        ('asm("add.u32 %0, %1, %2;\\n\\tadd.u32 %0, %0, %3;" : "=r"(X) : "r"(X), "r"(Y), "r"(v));', "IADD3"),
    "imad_reg":     ('asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(X) : "r"(X), "r"(mr), "r"(Y));', "IMAD"),
    "imad_const":   ('asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(X) : "r"(X), "r"(k_pow2[0]), "r"(Y));', "IMAD"),
    "imad_iadd":    ('X = X + Y;', "IMAD.IADD"),
    "imad_shl":     ('asm("mad.lo.u32 %0, %1, 32, %2;" : "=r"(X) : "r"(Y), "r"(X));', "IMAD.SHL"),
    "imad_hi":      ('asm("mad.hi.u32 %0, %1, %2, %3;" : "=r"(X) : "r"(X), "r"(k_pow2[22]), "r"(Y));', "IMAD.HI"),
    "imad_wide":    ('{ unsigned long long w; asm("mul.wide.u32 %0, %1, %2;" : "=l"(w) : "r"(X), "r"(mr)); '
                     'X = (uint32_t)w ^ (uint32_t)(w >> 32); }', "IMAD.WIDE"),
    "viadd":        ('X = X + Y + 0x1234567u;', "VIADD"),
}
# Ops that only run inside a mix: alone, ptxas folds a chain of them into one instruction per loop trip.  An immediate
# add is a VIADD only where ptxas chooses it: next to a shift it emits VIADD, next to an IMAD mostly IADD3 (the report
# prints the opcodes that ran).
MIX_OPS = {
    "viadd_imm":    ('X = X + 0x1234567u;', "VIADD"),
}
MIXES = {  # ALU form : IMAD form, in the ratio given (per chain, back to back)
    "shf+imad_const 1:1": (["shf_r_w", "imad_const"]),
    "shf+imad_hi 1:1":    (["shf_r_w", "imad_hi"]),
    "lop3+imad_const 1:1": (["lop3", "imad_const"]),
    "shf+imad_wide 1:1":  (["shf_r_w", "imad_wide"]),
    "shf+lop3+imad_const 2:1": (["shf_r_w", "lop3", "imad_const"]),
    "shf+lop3+imad_hi 2:1":    (["shf_r_w", "lop3", "imad_hi"]),
    # which pipe VIADD issues on: it co-issues with the one it does not share.  The shift is the variable-count
    # SHF.R.U32.HI because ptxas fuses a funnel shift and an immediate add into one LEA.HI.
    "viadd+shf 1:1":      (["shf_r_u32_hi", "viadd_imm"]),
    "viadd+imad 1:1":     (["imad_const", "viadd_imm"]),
}
UNROLL = 8          # ops per chain per loop trip (x 8 chains = 64 per form per trip)


def _kernel_src(name: str, forms: list[str]) -> str:
    body = []
    for _ in range(UNROLL):
        for i in range(8):
            for f in forms:
                body.append({**PROBE_OPS, **MIX_OPS}[f][0].replace("X", f"x{i}").replace("Y", f"x{(i + 1) & 7}"))
    return f"""
extern "C" __global__ void __launch_bounds__(256) probe_{name}(const uint32_t* in, uint32_t* out, long long* cyc, int iters) {{
    const uint32_t mr = in[0], s = in[1], v = in[2] + threadIdx.x;
    uint32_t x0 = v, x1 = v + 1, x2 = v + 2, x3 = v + 3, x4 = v + 4, x5 = v + 5, x6 = v + 6, x7 = v + 7;
    __syncthreads();
    const long long t0 = clock64();
#pragma unroll 1
    for (int it = 0; it < iters; ++it) {{
        {chr(10).join("        " + b for b in body)}
    }}
    __syncthreads();
    const long long t1 = clock64();
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
    out[blockIdx.x * blockDim.x + threadIdx.x] = x0 ^ x1 ^ x2 ^ x3 ^ x4 ^ x5 ^ x6 ^ x7;
}}
"""


def probe_source() -> tuple[str, dict[str, list[str]]]:
    kernels = {n: [n] for n in PROBE_OPS}
    kernels.update({re.sub(r"[^a-z0-9]+", "_", n): forms for n, forms in MIXES.items()})
    src = ["#include <stdint.h>",
           "__constant__ uint32_t k_pow2[32] = {" + ", ".join(f"{1 << k}u" for k in range(32)) + "};"]
    src += [_kernel_src(n, forms) for n, forms in kernels.items()]
    return "\n".join(src), kernels


def nvcc() -> str:
    home = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    for cand in (os.path.join(home, "bin", "nvcc"), shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    raise SystemExit("nvcc not found (set CUDA_HOME)")


def build_probe(tmp: str) -> tuple[str, dict[str, list[str]]]:
    src, kernels = probe_source()
    cu, cubin = os.path.join(tmp, "pipe_probe.cu"), os.path.join(tmp, "pipe_probe.cubin")
    open(cu, "w").write(src)
    subprocess.run([nvcc(), "-cubin", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-diag-suppress", "177", "-o", cubin, cu], check=True)
    return cubin, kernels


def sass_ops(cubin: str, fun: str) -> list[tuple[int, str, str]]:
    """(address, opcode with modifiers, whole line) of every instruction of one function"""
    txt = subprocess.run([os.path.join(os.path.dirname(nvcc()), "cuobjdump"), "-sass", "-fun", fun, cubin],
                         capture_output=True, text=True, check=True).stdout
    out = []
    for m in re.finditer(r"/\*([0-9a-f]{4,})\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)([^;]*);", txt):
        out.append((int(m.group(1), 16), m.group(2), m.group(0)))
    return out


def loop_body(ops):
    """the instructions between the target of the last backward branch and that branch"""
    for addr, op, line in reversed(ops):
        m = re.search(r"BRA\s+(?:`\(\.L_x_\d+\)|0x([0-9a-f]+))", line)
        if op.startswith("BRA") and m and m.group(1) and int(m.group(1), 16) < addr:
            tgt = int(m.group(1), 16)
            return [o for o in ops if tgt <= o[0] <= addr]
    raise RuntimeError("no backward branch in probe kernel")


def histogram(ops) -> dict[str, int]:
    h: dict[str, int] = {}
    for _, op, _ in ops:
        h[op] = h.get(op, 0) + 1
    return dict(sorted(h.items(), key=lambda kv: -kv[1]))


class Driver:
    def __init__(self, dev: int = 0):
        self.cu = C.CDLL("libcuda.so.1")
        self._ck(self.cu.cuInit(0), "cuInit")
        self.dev = C.c_int()
        self._ck(self.cu.cuDeviceGet(C.byref(self.dev), dev), "cuDeviceGet")
        self.ctx = C.c_void_p()
        self._ck(self.cu.cuDevicePrimaryCtxRetain(C.byref(self.ctx), self.dev), "cuDevicePrimaryCtxRetain")
        self._ck(self.cu.cuCtxSetCurrent(self.ctx), "cuCtxSetCurrent")

    @staticmethod
    def _ck(rc, what):
        if rc != 0:
            raise RuntimeError(f"{what} failed: CUresult {rc}")

    def attr(self, a: int) -> int:
        v = C.c_int()
        self._ck(self.cu.cuDeviceGetAttribute(C.byref(v), a, self.dev), "cuDeviceGetAttribute")
        return v.value

    def name(self) -> str:
        b = C.create_string_buffer(256)
        self._ck(self.cu.cuDeviceGetName(b, 256, self.dev), "cuDeviceGetName")
        return b.value.decode()

    def alloc(self, n: int) -> C.c_uint64:
        p = C.c_uint64()
        self._ck(self.cu.cuMemAlloc_v2(C.byref(p), C.c_size_t(n)), "cuMemAlloc")
        return p

    def h2d(self, dst, data: bytes):
        self._ck(self.cu.cuMemcpyHtoD_v2(dst, data, C.c_size_t(len(data))), "cuMemcpyHtoD")

    def d2h(self, src, n: int) -> bytes:
        b = C.create_string_buffer(n)
        self._ck(self.cu.cuMemcpyDtoH_v2(b, src, C.c_size_t(n)), "cuMemcpyDtoH")
        return b.raw

    def load(self, cubin: str):
        mod = C.c_void_p()
        self._ck(self.cu.cuModuleLoadData(C.byref(mod), open(cubin, "rb").read()), "cuModuleLoadData")
        return mod

    def fn(self, mod, name: str):
        f = C.c_void_p()
        self._ck(self.cu.cuModuleGetFunction(C.byref(f), mod, name.encode()), f"cuModuleGetFunction({name})")
        return f

    def launch(self, f, grid: int, block: int, args: list):
        ptrs = (C.c_void_p * len(args))(*[C.addressof(a) for a in args])
        self._ck(self.cu.cuLaunchKernel(f, grid, 1, 1, block, 1, 1, 0, None, ptrs, None), "cuLaunchKernel")
        self._ck(self.cu.cuCtxSynchronize(), "cuCtxSynchronize")


def card_info(drv: Driver) -> dict:
    info = {"name": drv.name(), "sms": drv.attr(16)}                 # CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"], info["sm_max_mhz"] = float(q[0]), float(q[1])
    except Exception as exc:  # the rates stand without it; say so
        info["power_limit_w"] = f"unread: {exc!r}"[:80]
    return info


def measure_rates(drv: Driver, cubin: str, kernels: dict[str, list[str]], iters: int = 4096) -> dict:
    mod = drv.load(cubin)
    sms = drv.attr(16)
    block = 256                                   # 8 warps = 2 per sub-partition per CTA
    grid = sms * 4                                # 4 CTAs per SM: 8 warps per sub-partition
    d_in, d_out, d_cyc = drv.alloc(16), drv.alloc(grid * block * 4), drv.alloc(grid * 8)
    drv.h2d(d_in, (0x9E3779B1).to_bytes(4, "little") + (3).to_bytes(4, "little") + (12345).to_bytes(4, "little") + bytes(4))
    res = {}
    for name, forms in kernels.items():
        f = drv.fn(mod, f"probe_{name}")
        body = loop_body(sass_ops(cubin, f"probe_{name}"))
        hist = histogram(body)
        args = [d_in, d_out, d_cyc, C.c_int(iters)]
        drv.launch(f, grid, block, args)          # warm-up
        drv.launch(f, grid, block, args)
        cyc = max(int.from_bytes(drv.d2h(d_cyc, grid * 8)[8 * i: 8 * i + 8], "little") for i in range(grid))
        warps_per_smsp = grid * block // 32 / (sms * 4)
        per_clk = lambda n: round(n * iters * warps_per_smsp / cyc, 4)
        pipes = {"alu": 0, "imad": 0, "other": 0}
        for op, n in hist.items():
            pipes[pipe_of(op)] += n
        res[name] = {"forms": forms, "loop_sass": hist,
                     "warp_inst_per_clk_per_smsp": {"all": per_clk(len(body)), **{p: per_clk(n) for p, n in pipes.items()}}}
        print(f"  {name:28s} all {per_clk(len(body)):.3f}  alu {per_clk(pipes['alu']):.3f}  imad {per_clk(pipes['imad']):.3f}"
              f"  | {', '.join(f'{k} {v}' for k, v in list(hist.items())[:4])}", flush=True)
    return res


# --- 2. the headline kernel against its ALU floor ----------------------------------------------------------------------
def kernel_pipe_counts(fun: str = SEG_KERNEL, viadd: str = "alu") -> dict:
    cubin = os.path.join(ROOT, "coast_b200", "csrc", "coast_kernels.cubin")
    hist = histogram(sass_ops(cubin, fun))
    pipes = {"alu": 0, "imad": 0, "other": 0}
    measured = dict(pipes)
    for op, n in hist.items():
        pipes[pipe_of(op)] += n
        measured[pipe_of_measured(op, viadd)] += n
    return {"function": fun, "pipes": pipes, "pipes_viadd_measured": measured, "viadd_pipe": viadd,
            "viadd": sum(n for op, n in hist.items() if op.split(".")[0] == "VIADD"), "top": dict(list(hist.items())[:12])}


def headline(alu_rate: float, sms: int, viadd: str) -> dict:
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--workload", "sha256", "--steps", "50", "--warmup", "10",
           "--no-cpu-baseline"]
    out = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
    if out.returncode != 0:
        raise RuntimeError(out.stdout[-2000:] + out.stderr[-2000:])
    line = json.loads([ln for ln in out.stdout.splitlines() if ln.startswith("{")][-1])
    k_ms, mhz = line["roofline"]["kernel_ms"], line["clocks"]["sm_mhz_in_timed_region"] or line["clocks"]["sm_mhz"]
    counts = kernel_pipe_counts(viadd=viadd)
    warps = (1 << 20) // 32 * 3
    floor_ms = lambda n_alu: n_alu * warps / (sms * 4) / alu_rate / (mhz * 1e3)
    without = floor_ms(counts["pipes"]["alu"])
    with_viadd = floor_ms(counts["pipes"]["alu"] + counts["viadd"])
    floor = floor_ms(counts["pipes_viadd_measured"]["alu"])
    return {"value_mbs": line["value"], "kernel_ms": k_ms, "sm_mhz_in_timed_region": mhz, "sass": counts,
            "alu_floor_ms_without_viadd": round(without, 5), "alu_floor_ms_with_viadd": round(with_viadd, 5),
            "alu_floor_ms": round(floor, 5), "kernel_over_alu_floor": round(k_ms / floor, 3),
            "gate": "ALU-bound" if k_ms <= 1.25 * floor else "not ALU-bound (above 1.25x the ALU floor)"}


# --- 3. the other SHA-256 kernels --------------------------------------------------------------------------------------
def other_sha_kernels(reps: int = 20) -> dict:
    sys.path.insert(0, ROOT)
    import torch
    import coast_b200 as cb
    rt = cb.Runtime(0)
    res = {}
    cases = [("b64_nc1", 1, 64, 0), ("b64_nc2", 2, 64, 0), ("b64_nc3_interleaved", 3, 64, cb.F_INTERLEAVE),
             ("gen4000_nc3", 3, 4000, cb.F_INTERLEAVE)]
    for name, nc, ub, fl in cases:
        n = (1 << 20) if ub == 64 else (1 << 15)
        d_in = torch.empty(n * ub, dtype=torch.uint8, device="cuda")
        rt.fill_philox(d_in, 11)
        d_out = torch.empty(n * 32, dtype=torch.uint8, device="cuda")
        desc = rt.make_desc(cb.K_SHA256, nc, d_in, d_out, n, unit_bytes=ub, flags=fl)
        for _ in range(3):
            rt.launch(desc)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            rt.launch(desc)
        b.record()
        b.synchronize()
        rt.sync()
        res[name] = {"units": n, "unit_bytes": ub, "kernel_ms": round(a.elapsed_time(b) / reps, 5)}
        print(f"  {name:22s} {res[name]['kernel_ms']:.4f} ms", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--json", help="write the full report here")
    ap.add_argument("--skip-bench", action="store_true", help="do not run bench.py for the ALU-floor gate")
    ap.add_argument("--skip-sha", action="store_true", help="do not time the other SHA-256 kernels")
    args = ap.parse_args()
    drv = Driver(0)
    card = card_info(drv)
    print("card:", card, flush=True)
    report = {"card": card}
    with tempfile.TemporaryDirectory() as tmp:
        cubin, kernels = build_probe(tmp)
        report["rates"] = measure_rates(drv, cubin, kernels)
    alu_rate = report["rates"]["shf_r_w"]["warp_inst_per_clk_per_smsp"]["alu"]
    report["viadd_pipe"] = viadd_pipe(report["rates"])
    print("VIADD issues on the", report["viadd_pipe"], "pipe", flush=True)
    if not args.skip_bench:
        report["headline"] = headline(alu_rate, card["sms"], report["viadd_pipe"])
        print("headline:", json.dumps(report["headline"]), flush=True)
    if not args.skip_sha:
        report["other_sha_kernels"] = other_sha_kernels()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
