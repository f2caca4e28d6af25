"""Child process of tests/test_mm_bt_host_logic.py: matmul launches and host calls of libcoast_rt.so against the mock driver
(tests/mock_cuda/mock_cuda_bt.c), with and without COAST_MM_B_TRANSPOSED.  Usage: python mm_bt_child.py <scenario-json>.
Each op gives `kernel`, M, N, K and either nothing (one product), `batch` (COAST_MM_BATCHED) or a row-offset table `ro`
(COAST_MM_GROUPED; M = G unless the op gives M); `bt` sets COAST_MM_B_TRANSPOSED.  A and B have the kernel's element size
(2 bytes for GEMM_BF16, else 4), C 4 bytes; `alloc` overrides the element counts [A, B, C], `shift` = [in, aux, out] byte
offsets misalign a buffer, `mode` and `n` override what the op implies.  Prints one JSON object."""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from coast_b200 import runtime as R  # noqa: E402  (structs + argtypes only; torch is never imported here)


def shape(op):
    """(mode, descriptor M, n_units, elements of A, B, C)"""
    N, K = op["N"], op["K"]
    bt = R.MM_B_TRANSPOSED if op.get("bt") else 0
    if "ro" in op:
        ro = op["ro"]
        G, rows = len(ro) - 1, ro[-1]
        return R.MM_GROUPED | bt, op.get("M", G), (ro[-1] - ro[0]) * N, max(rows, 1) * K, G * K * N, max(rows, 1) * N
    b = op.get("batch", 1)
    return (R.MM_BATCHED if "batch" in op else 0) | bt, op["M"], b * op["M"] * N, b * op["M"] * K, b * K * N, b * op["M"] * N


def main():
    sc = json.loads(sys.argv[1])
    L = R.load_library()
    L.coast_malloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t]
    L.coast_free.argtypes = [C.c_void_p]
    L.coast_memcpy_h2d.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.coast_host_alloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t]
    L.coast_host_free.argtypes = [C.c_void_p]
    res = {"init": L.coast_init(0)}
    assert res["init"] == 0, L.coast_last_error()
    out = []
    for op in sc["ops"]:
        mode, M, n, ea, eb, ec = shape(op)
        ea, eb, ec = op.get("alloc", [ea, eb, ec])
        kernel = op["kernel"]
        es = 2 if kernel == R.K_GEMM_BF16 else 4
        sizes = [es * ea + 64, es * eb + 64, 4 * ec + 64]
        shift = op.get("shift", [0, 0, 0])
        ro = op.get("ro")
        table = (C.c_uint64 * len(ro))(*ro) if ro else None
        d = R.LaunchDesc()
        d.kernel, d.num_clones, d.flags = kernel, op.get("nc", 3), op.get("flags", 0)
        d.mode, d.M, d.N, d.K = op.get("mode", mode), M, op["N"], op["K"]
        d.n_units, d.unit_base = op.get("n", n), op.get("unit_base", 0)
        if op.get("unit_bytes"):
            d.unit_bytes = op["unit_bytes"]
        plan = None
        if op.get("p"):                                         # a Bernoulli plan: the inj1 kernels
            plan = R._Plan(); plan.mode = R.PLAN_BERNOULLI; plan.seed_lo = 7; plan.threshold = int(op["p"] * 2 ** 32)
            d.plan = C.pointer(plan)
        if op["op"] == "launch":
            bufs = [C.c_void_p() for _ in sizes]
            for b, s in zip(bufs, sizes):
                assert L.coast_malloc(C.byref(b), s) == 0
            rows = C.c_void_p()
            if ro:
                assert L.coast_malloc(C.byref(rows), 8 * len(ro)) == 0
                assert L.coast_memcpy_h2d(rows, table, 8 * len(ro), None) == 0
                d.d_rows = rows.value
            d.d_in, d.d_aux, d.d_out = [b.value + s for b, s in zip(bufs, shift)]
            rc = L.coast_launch(C.byref(d), None)
            out.append({"rc": rc, "err": L.coast_last_error().decode() if rc else "", "in": d.d_in, "aux": d.d_aux, "out": d.d_out,
                        "rows": rows.value, "sizes": sizes + ([8 * len(ro)] if ro else [])})
            for b in bufs + ([rows] if ro else []):
                L.coast_free(b)
        else:                                                   # run_host: pageable or pinned host buffers
            pinned = op.get("pinned", False)
            if pinned:
                hs = [C.c_void_p() for _ in sizes]
                for h, s in zip(hs, sizes):
                    assert L.coast_host_alloc(C.byref(h), s) == 0
                ptrs = [h.value for h in hs]
            else:
                keep = [(C.c_uint8 * s)() for s in sizes]
                ptrs = [C.addressof(k) for k in keep]
            d.d_in, d.d_aux, d.d_out = ptrs
            if ro:
                d.d_rows = C.addressof(table)
            st = R._Stats()
            rc = L.coast_run_host_noabort(C.byref(d), C.byref(st))
            out.append({"rc": rc, "err": L.coast_last_error().decode() if rc else "", "host_in": ptrs[0], "host_aux": ptrs[1],
                        "host_out": ptrs[2], "host_rows": C.addressof(table) if ro else 0, "path": L.coast_last_host_path().decode()})
            if pinned:
                for h in hs:
                    L.coast_host_free(h)
    L.coast_shutdown()
    res["ops"] = out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
