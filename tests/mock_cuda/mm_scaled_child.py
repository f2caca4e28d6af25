"""Child process of the scaled GEMM_FP8 host-logic tests: the launches and host calls of tests/mock_cuda/mm_child.py with the
scale pointers of COAST_MM_SCALE_TENSOR / COAST_MM_SCALE_ROWWISE.  Usage: python mm_scaled_child.py <scenario-json>.
An op is mm_child.py's plus `scale`: "tensor" (one float each), "row" (one per stacked row of A -- groups: ro[-1] -- and P*N
for B) or absent (no scale bit, no buffers).  `scale_shift` = [a, b] byte offsets misalign them, `scale_null` = [a, b] leaves
either null.  Prints one JSON object whose records add the scale pointers."""
import ctypes as C
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from mm_child import R, shape  # noqa: E402


def scale_counts(op):
    """floats of A's and B's scales the op implies"""
    if op.get("scale") == "tensor":
        return 1, 1
    N = op["N"]
    if "ro" in op:
        return max(op["ro"][-1], 1), (len(op["ro"]) - 1) * N
    b = op.get("batch", 1)
    return b * op["M"], b * N


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
        scaled = op.get("scale")
        mode |= {"tensor": R.MM_SCALE_TENSOR, "row": R.MM_SCALE_ROWWISE}.get(scaled, 0)
        kernel = op["kernel"]
        es = R.MM_ELEM_BYTES.get(kernel, 4)
        sizes = [es * ea + 64, es * eb + 64, 4 * ec + 64]
        fa, fb = scale_counts(op) if scaled else (0, 0)
        ssizes = [4 * fa + 64, 4 * fb + 64] if scaled else []
        shift = op.get("shift", [0, 0, 0])
        sshift = op.get("scale_shift", [0, 0])
        snull = op.get("scale_null", [False, False])
        ro = op.get("ro")
        table = (C.c_uint64 * len(ro))(*ro) if ro else None
        d = R.LaunchDesc()
        d.kernel, d.num_clones, d.flags = kernel, op.get("nc", 3), op.get("flags", 0)
        d.mode, d.M, d.N, d.K = op.get("mode", mode), M, op["N"], op["K"]
        d.n_units, d.unit_base = op.get("n", n), op.get("unit_base", 0)
        plan = None
        if op.get("p"):                                         # a Bernoulli plan: the inj1 kernels
            plan = R._Plan(); plan.mode = R.PLAN_BERNOULLI; plan.seed_lo = 7; plan.threshold = int(op["p"] * 2 ** 32)
            d.plan = C.pointer(plan)
        if op["op"] == "launch":
            bufs = [C.c_void_p() for _ in sizes + ssizes]
            for b, s in zip(bufs, sizes + ssizes):
                assert L.coast_malloc(C.byref(b), s) == 0
            rows = C.c_void_p()
            if ro:
                assert L.coast_malloc(C.byref(rows), 8 * len(ro)) == 0
                assert L.coast_memcpy_h2d(rows, table, 8 * len(ro), None) == 0
                d.d_rows = rows.value
            d.d_in, d.d_aux, d.d_out = [b.value + s for b, s in zip(bufs, shift)]
            if scaled:
                d.d_scale_a, d.d_scale_b = [None if z else b.value + s for b, s, z in zip(bufs[3:], sshift, snull)]
            rc = L.coast_launch(C.byref(d), None)
            out.append({"rc": rc, "err": L.coast_last_error().decode() if rc else "", "in": d.d_in, "aux": d.d_aux, "out": d.d_out,
                        "rows": rows.value, "sa": d.d_scale_a or 0, "sb": d.d_scale_b or 0})
            for b in bufs + ([rows] if ro else []):
                L.coast_free(b)
        else:                                                   # run_host: pageable or pinned host buffers
            pinned = op.get("pinned", False)
            allsz = sizes + ssizes
            if pinned:
                hs = [C.c_void_p() for _ in allsz]
                for h, s in zip(hs, allsz):
                    assert L.coast_host_alloc(C.byref(h), s) == 0
                ptrs = [h.value for h in hs]
            else:
                keep = [(C.c_uint8 * s)() for s in allsz]
                ptrs = [C.addressof(k) for k in keep]
            d.d_in, d.d_aux, d.d_out = ptrs[:3]
            if scaled:
                d.d_scale_a, d.d_scale_b = [None if z else h + s for h, s, z in zip(ptrs[3:], sshift, snull)]
            if ro:
                d.d_rows = C.addressof(table)
            st = R._Stats()
            rc = L.coast_run_host_noabort(C.byref(d), C.byref(st))
            out.append({"rc": rc, "err": L.coast_last_error().decode() if rc else "", "host_in": ptrs[0], "host_aux": ptrs[1],
                        "host_out": ptrs[2], "host_sa": ptrs[3] if scaled else 0, "host_sb": ptrs[4] if scaled else 0,
                        "host_rows": C.addressof(table) if ro else 0, "path": L.coast_last_host_path().decode()})
            if pinned:
                for h in hs:
                    L.coast_host_free(h)
    L.coast_shutdown()
    res["ops"] = out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
