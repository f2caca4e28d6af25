"""Child process of tests/test_grouped_mm_host_logic.py: grouped matmul (COAST_MM_GROUPED) launches and host calls of
libcoast_rt.so against the mock driver (tests/mock_cuda/mock_cuda.c).  Usage: python grouped_mm_child.py <scenario-json>.
Each op names a kernel, a replica count, N, K and a row-offset table `ro` (G + 1 entries; M = G unless the op gives M); buffers
hold ro[-1] rows of A and C and G matrices B (`alloc_rows` / `alloc_groups` override what they are sized for, so that a refusal
can be asked for without the memory).  Prints one JSON object."""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from coast_b200 import runtime as R  # noqa: E402  (structs + argtypes only; torch is never imported here)


def desc(op):
    ro = op["ro"]
    d = R.LaunchDesc()
    d.kernel, d.num_clones, d.flags = op.get("kernel", R.K_MM_U32), op.get("nc", 3), op.get("flags", 0)
    d.mode = op.get("mode", R.MM_GROUPED)
    d.M, d.N, d.K = op.get("M", len(ro) - 1), op["N"], op["K"]
    d.n_units = op["n"] if "n" in op else (ro[-1] - ro[0]) * op["N"]
    d.unit_base = op.get("unit_base", 0)
    return d


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
        ro, N, K = op["ro"], op["N"], op["K"]
        rows = op.get("alloc_rows", max(ro[-1], 1))
        groups = op.get("alloc_groups", max(len(ro) - 1, 1))
        sizes = [max(4 * rows * K, 16), max(4 * groups * K * N, 16), max(4 * rows * N, 16), 8 * len(ro)]
        plan = None
        if op.get("p"):
            plan = R._Plan(); plan.mode = 1; plan.seed_lo = 7; plan.threshold = int(op["p"] * 2 ** 32)
        table = (C.c_uint64 * len(ro))(*ro)
        if op["op"] == "launch":
            bufs = [C.c_void_p() for _ in sizes]
            for b, s in zip(bufs, sizes):
                assert L.coast_malloc(C.byref(b), s) == 0
            assert L.coast_memcpy_h2d(bufs[3], table, 8 * len(ro), None) == 0
            d = desc(op)
            d.d_in, d.d_aux, d.d_out = bufs[0].value, bufs[1].value, bufs[2].value
            d.d_rows = None if op.get("null_rows") else bufs[3].value + op.get("rows_shift", 0)
            if plan is not None:
                d.plan = C.pointer(plan)
            rc = L.coast_launch(C.byref(d), None)
            out.append({"rc": rc, "err": L.coast_last_error().decode() if rc else "", "in": bufs[0].value, "aux": bufs[1].value,
                        "out": bufs[2].value, "rows": bufs[3].value})
            for b in bufs:
                L.coast_free(b)
        else:                                                   # run_host: pageable or pinned host buffers
            pinned = op.get("pinned", False)
            if pinned:
                hs = [C.c_void_p() for _ in sizes[:3]]
                for h, s in zip(hs, sizes):
                    assert L.coast_host_alloc(C.byref(h), s) == 0
                ptrs = [h.value for h in hs]
            else:
                keep = [(C.c_uint8 * s)() for s in sizes[:3]]
                ptrs = [C.addressof(k) for k in keep]
            d = desc(op)
            d.d_in, d.d_aux, d.d_out = ptrs
            d.d_rows = None if op.get("null_rows") else C.addressof(table)
            if plan is not None:
                d.plan = C.pointer(plan)
            st = R._Stats()
            rc = L.coast_run_host_noabort(C.byref(d), C.byref(st))
            out.append({"rc": rc, "err": L.coast_last_error().decode() if rc else "", "host_in": ptrs[0], "host_aux": ptrs[1],
                        "host_out": ptrs[2], "host_rows": C.addressof(table), "path": L.coast_last_host_path().decode()})
            if pinned:
                for h in hs:
                    L.coast_host_free(h)
    L.coast_shutdown()
    res["ops"] = out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
