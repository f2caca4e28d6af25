"""Child process of tests/test_ragged_qsort_host_logic.py: ragged quicksort (COAST_UNIT_OFFSETS with COAST_K_QSORT) launches
and host calls of libcoast_rt.so against the mock driver (tests/mock_cuda/mock_cuda.c).  A quicksort batch's output is the
size of its input (each array is sorted into the bytes it came from).  Usage: python ragged_qsort_child.py <scenario-json>.
Prints one JSON object."""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from coast_b200 import runtime as R  # noqa: E402  (structs + argtypes only; torch is never imported here)


def main():
    sc = json.loads(sys.argv[1])
    L = R.load_library()
    L.coast_malloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t]
    L.coast_free.argtypes = [C.c_void_p]
    L.coast_host_alloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t]
    L.coast_host_free.argtypes = [C.c_void_p]
    res = {"init": L.coast_init(0)}
    assert res["init"] == 0, L.coast_last_error()
    out = []
    for op in sc["ops"]:
        d = R.LaunchDesc()
        d.kernel, d.num_clones, d.flags = op.get("kernel", R.K_QSORT), op.get("nc", 3), op.get("flags", 0)
        d.mode = op.get("mode", R.UNIT_OFFSETS)
        offs = op.get("offsets")
        if offs is None:                                        # a long batch: element counts repeated, 4-byte offsets from `first`
            offs = [op["first"]]
            for e in op["elems"] * op["repeat"]:
                offs.append(offs[-1] + 4 * e)
        d.n_units, d.unit_base, d.unit_bytes = len(offs) - 1, op.get("unit_base", 0), op["unit_bytes"]
        total = max(offs) + 16
        if op.get("p"):
            plan = R._Plan(); plan.mode = 1; plan.seed_lo = 7; plan.threshold = int(op["p"] * 2 ** 32)
            d.plan = C.pointer(plan)
        if op["op"] == "launch":
            p_in, p_out, p_aux = C.c_void_p(), C.c_void_p(), C.c_void_p()
            assert L.coast_malloc(C.byref(p_in), total) == 0 and L.coast_malloc(C.byref(p_out), total) == 0
            assert L.coast_malloc(C.byref(p_aux), 8 * len(offs) + 16) == 0
            C.memmove(p_aux.value, (C.c_uint64 * len(offs))(*offs), 8 * len(offs))
            d.d_in, d.d_out = p_in.value + op.get("in_misalign", 0), p_out.value + op.get("out_misalign", 0)
            d.d_aux = p_aux.value
            rc = L.coast_launch(C.byref(d), None)
            out.append({"rc": rc, "err": L.coast_last_error().decode() if rc else "", "aux": p_aux.value, "in": p_in.value,
                        "out": p_out.value})
            for p in (p_in, p_out, p_aux):
                L.coast_free(p)
        else:                                                   # run_host: pageable or pinned host buffers
            pinned = op.get("pinned", False)
            if pinned:
                hi, ho = C.c_void_p(), C.c_void_p()
                assert L.coast_host_alloc(C.byref(hi), total) == 0 and L.coast_host_alloc(C.byref(ho), total) == 0
                h_in, h_out = hi.value, ho.value
            else:
                b_in, b_out = (C.c_uint32 * (total // 4 + 1))(), (C.c_uint32 * (total // 4 + 1))()
                h_in, h_out = C.addressof(b_in), C.addressof(b_out)
            aux = (C.c_uint64 * len(offs))(*offs)
            d.d_in, d.d_out, d.d_aux = h_in, h_out, C.addressof(aux)
            st = R._Stats()
            rc = L.coast_run_host_noabort(C.byref(d), C.byref(st))
            out.append({"rc": rc, "err": L.coast_last_error().decode() if rc else "", "host_in": h_in, "host_out": h_out,
                        "host_aux": C.addressof(aux), "path": L.coast_last_host_path().decode()})
            if pinned:
                L.coast_host_free(hi); L.coast_host_free(ho)
    L.coast_shutdown()
    res["ops"] = out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
