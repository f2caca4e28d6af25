"""Child process of tests/test_ragged_host_logic.py: ragged (COAST_UNIT_OFFSETS) launches and host calls of libcoast_rt.so
against the mock driver (tests/mock_cuda/mock_cuda.c).  Usage: python ragged_child.py <scenario-json>.  Prints one JSON object."""
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
        d.kernel, d.num_clones, d.flags = op.get("kernel", 1), op.get("nc", 3), op.get("flags", 0)
        d.mode = op.get("mode", R.UNIT_OFFSETS)
        offs = op["offsets"]
        n = op.get("n", len(offs) - 1)
        d.n_units, d.unit_base, d.unit_bytes = n, op.get("unit_base", 0), op["unit_bytes"]
        total = max(offs) + 16
        m = len(offs) - 1                                       # units the buffers hold (n may be set larger to test the bound)
        if op.get("p"):
            plan = R._Plan(); plan.mode = 1; plan.seed_lo = 7; plan.threshold = int(op["p"] * 2 ** 32)
            d.plan = C.pointer(plan)
        if op["op"] == "launch":
            p_in, p_out, p_aux = C.c_void_p(), C.c_void_p(), C.c_void_p()
            assert L.coast_malloc(C.byref(p_in), total) == 0 and L.coast_malloc(C.byref(p_out), m * 32 + 16) == 0
            assert L.coast_malloc(C.byref(p_aux), 8 * len(offs) + 16) == 0
            C.memmove(p_aux.value, (C.c_uint64 * len(offs))(*offs), 8 * len(offs))
            d.d_in, d.d_out = p_in.value, p_out.value
            d.d_aux = None if op.get("null_aux") else p_aux.value + op.get("aux_misalign", 0)
            rc = L.coast_launch(C.byref(d), None)
            out.append({"rc": rc, "err": L.coast_last_error().decode() if rc else "", "aux": p_aux.value, "in": p_in.value})
            for p in (p_in, p_out, p_aux):
                L.coast_free(p)
        else:                                                   # run_host: pageable or pinned host buffers
            pinned = op.get("pinned", False)
            ob = 32 if d.kernel == 1 else 2
            if pinned:
                hi, ho = C.c_void_p(), C.c_void_p()
                assert L.coast_host_alloc(C.byref(hi), total) == 0 and L.coast_host_alloc(C.byref(ho), m * ob + 16) == 0
                h_in, h_out = hi.value, ho.value
            else:
                b_in, b_out = (C.c_uint8 * total)(), (C.c_uint8 * (m * ob + 16))()
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
