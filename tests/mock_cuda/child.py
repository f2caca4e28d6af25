"""Child process of tests/test_host_logic.py: drives libcoast_rt.so against the mock driver (tests/mock_cuda/mock_cuda.c).
Usage: python child.py <scenario-json>.  Prints one JSON object."""
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
    pre = None
    if sc.get("before_init"):                               # compute calls before coast_init must fail loudly, not crash
        d0 = R.LaunchDesc(); d0.kernel = 1; d0.num_clones = 3; d0.n_units = 1; d0.unit_bytes = 64
        pre = {"launch": L.coast_launch(C.byref(d0), None), "err": L.coast_last_error().decode()}
    res = {"init": L.coast_init(0), "before_init": pre}
    if res["init"]:
        res["error"] = L.coast_last_error().decode()
        print(json.dumps(res))
        return

    def dmalloc(n):
        p = C.c_void_p()
        rc = L.coast_malloc(C.byref(p), n)
        assert rc == 0, L.coast_last_error()
        return p.value

    out = []
    for op in sc["ops"]:
        kind = op["op"]
        d = R.LaunchDesc()
        d.kernel, d.num_clones, d.flags, d.mode = op.get("kernel", 0), op.get("nc", 3), op.get("flags", 0), op.get("mode", 0)
        d.n_units, d.unit_base, d.unit_bytes = op.get("n", 0), op.get("unit_base", 0), op.get("unit_bytes", 0)
        d.M, d.N, d.K = op.get("M", 0), op.get("N", 0), op.get("K", 0)
        plan = None
        if op.get("p"):
            plan = R._Plan(); plan.mode = 1; plan.seed_lo = 7; plan.threshold = int(op["p"] * 2 ** 32)
            d.plan = C.pointer(plan)
        if kind == "launch":
            bufs = [dmalloc(max(op["in_bytes"], 16)), dmalloc(max(op["out_bytes"], 16))]
            d.d_in, d.d_out = bufs[0] + op.get("misalign", 0), bufs[1]
            if op.get("aux_bytes"):
                bufs.append(dmalloc(op["aux_bytes"]))
                d.d_aux = bufs[2]
            rc = L.coast_launch(C.byref(d), None)
            st = R._Stats()
            rc2 = L.coast_sync_noabort(None, C.byref(st)) if rc == 0 else 0
            for b in bufs:
                L.coast_free(b)
            out.append({"rc": rc, "sync_rc": rc2, "err": L.coast_last_error().decode() if rc else ""})
        elif kind == "run_host":
            h_in = (C.c_uint8 * max(op["in_bytes"], 1))()
            h_out = (C.c_uint8 * max(op["out_bytes"], 1))()
            for i in range(0, op["in_bytes"], 4099):
                h_in[i] = (i * 7 + 1) & 0xFF
            d.d_in, d.d_out = C.addressof(h_in), C.addressof(h_out)
            st = R._Stats()
            rc = L.coast_run_host_noabort(C.byref(d), C.byref(st))
            out.append({"rc": rc, "err": L.coast_last_error().decode() if rc else "", "host_in": C.addressof(h_in),
                        "host_out": C.addressof(h_out), "first_fault_unit": st.first_fault_unit})
        elif kind == "run_host_pinned":                     # pinned (mapped) host buffers: the zero-copy host call, or staged when forced
            L.coast_host_alloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t]
            L.coast_host_free.argtypes = [C.c_void_p]
            hi, ho, hs = C.c_void_p(), C.c_void_p(), C.c_void_p()
            assert L.coast_host_alloc(C.byref(hi), max(op["in_bytes"], 16)) == 0
            assert L.coast_host_alloc(C.byref(ho), max(op["out_bytes"], 16)) == 0
            d.d_in, d.d_out = hi.value, ho.value
            if op.get("status"):
                assert L.coast_host_alloc(C.byref(hs), op["n"]) == 0
                d.d_status = hs.value
            st = R._Stats()
            rc = L.coast_run_host_noabort(C.byref(d), C.byref(st))
            out.append({"rc": rc, "err": L.coast_last_error().decode() if rc else "", "host_in": hi.value, "host_out": ho.value,
                        "host_status": hs.value})
            for h in (hi, ho, hs):
                if h.value:
                    L.coast_host_free(h)
        elif kind == "run_host_status":                     # pageable buffers + a host d_status: staged per chunk
            h_in = (C.c_uint8 * op["in_bytes"])()
            h_out = (C.c_uint8 * op["out_bytes"])()
            h_st = (C.c_uint8 * op["n"])()
            d.d_in, d.d_out, d.d_status = C.addressof(h_in), C.addressof(h_out), C.addressof(h_st)
            st = R._Stats()
            rc = L.coast_run_host_noabort(C.byref(d), C.byref(st))
            out.append({"rc": rc, "err": L.coast_last_error().decode() if rc else "", "host_in": C.addressof(h_in),
                        "host_out": C.addressof(h_out), "host_status": C.addressof(h_st)})
        elif kind == "sha_ctx":                             # what sha256_hash leaves in the caller's scratch arrays
            L.coast_set_opt_passes(b"-TMR")
            L.coast_xmr_sha256_hash.argtypes = [C.c_void_p] * 4 + [C.c_uint32, C.c_void_p]
            recs = []
            for ln in op["lens"]:
                cd, bl, stt, dig = (C.c_uint8 * 64)(*([0xEE] * 64)), (C.c_uint32 * 2)(9, 9), (C.c_uint32 * 8)(*([7] * 8)), (C.c_uint8 * 32)()
                data = (C.c_uint8 * ln)(*[(i * 3 + 1) & 0xFF for i in range(ln)])
                L.coast_xmr_sha256_hash(cd, bl, stt, data, ln, dig)
                recs.append({"len": ln, "bitlen": list(bl), "state": list(stt), "data": list(cd), "digest": list(dig)})
            out.append({"recs": recs})
        elif kind == "two_threads":                         # single-caller guard: a second thread gets COAST_ERR_BUSY, never a race
            import threading
            seen = [set(), set()]
            def hammer(k):
                for _ in range(op.get("iters", 20000)):
                    seen[k].add(L.coast_stats_reset(None))
            ts = [threading.Thread(target=hammer, args=(k,)) for k in range(2)]
            [t.start() for t in ts]; [t.join() for t in ts]
            out.append({"codes": sorted(seen[0] | seen[1]), "after": L.coast_stats_reset(None)})
        elif kind == "run_host_aux":                        # AES with per-unit keys (+ write-back), or a matmul: three host buffers
            h_in = (C.c_uint8 * op["in_bytes"])()
            h_aux = (C.c_uint8 * op["aux_bytes"])()
            h_out = (C.c_uint8 * op["out_bytes"])()
            d.d_in, d.d_aux, d.d_out = C.addressof(h_in), C.addressof(h_aux), C.addressof(h_out)
            st = R._Stats()
            rc = L.coast_run_host_noabort(C.byref(d), C.byref(st))
            out.append({"rc": rc, "err": L.coast_last_error().decode() if rc else "", "host_in": C.addressof(h_in),
                        "host_aux": C.addressof(h_aux), "host_out": C.addressof(h_out)})
        elif kind == "entries":                             # the reference-facing entry points (what the make flow binds)
            L.coast_set_opt_passes(op.get("passes", "-TMR -countErrors").encode())
            msg = b"Automated TMR"
            crc = L.coast_xmr_crc16(msg, len(msg))
            L.coast_xmr_sha256_hash.argtypes = [C.c_void_p] * 4 + [C.c_uint32, C.c_void_p]
            cd, bl, stt, data, dig = (C.c_uint8 * 64)(), (C.c_uint32 * 2)(), (C.c_uint32 * 8)(), (C.c_uint8 * 10)(), (C.c_uint8 * 32)()
            L.coast_xmr_sha256_hash(cd, bl, stt, data, 10, dig)
            L.coast_xmr_sha256_hash(cd, bl, stt, data, 0, dig)          # empty message: still one padded block
            state, key = (C.c_uint8 * 16)(), (C.c_uint8 * 16)()
            L.coast_xmr_aes_enc_dec.argtypes = [C.c_void_p, C.c_void_p, C.c_ubyte]
            L.coast_xmr_aes_enc_dec(state, key, 0)
            L.coast_xmr_aes_enc_dec(state, key, 1)
            f, s2, r = (C.c_uint32 * 81)(), (C.c_uint32 * 81)(), (C.c_uint32 * 81)()
            L.coast_xmr_matrix_multiply_u32.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
            L.coast_xmr_matrix_multiply_u32(f, s2, r, 9)
            indata, in_i, dg = (C.c_uint8 * 16384)(), (C.c_int * 2)(8192, 8192), (C.c_uint32 * 5)()
            L.coast_xmr_chstone_sha_stream.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
            L.coast_xmr_chstone_sha_stream(indata, in_i, 2, 8192, dg)
            out.append({"rc": 0, "crc": crc, "tmr_error_cnt": C.c_uint32.in_dll(L, "TMR_ERROR_CNT").value})
        elif kind == "misc":
            r = {}
            r["reinit_same"] = L.coast_init(0)
            r["reinit_other"] = L.coast_init(1)
            buf = dmalloc(4096)
            r["fill0"] = L.coast_fill_philox(buf, 0, 0, 1, None)
            r["fill"] = L.coast_fill_philox(buf, 1024, 5, 1, None)
            r["snapshot"] = L.coast_stats_snapshot(None, buf)
            st = R._Stats()
            d.kernel, d.num_clones, d.n_units, d.unit_bytes = 1, 3, 0, 64
            h = (C.c_uint8 * 64)()
            d.d_in, d.d_out = C.addressof(h), C.addressof(h)
            r["run_host_empty"] = L.coast_run_host_noabort(C.byref(d), C.byref(st))
            r["stats"] = [st.errors_corrected, st.dwc_detected, st.syncs, st.injected, st.first_fault_unit]
            tp = R._Plan(); tp.mode = 2
            d.n_units = 4; d.plan = C.pointer(tp)
            r["run_host_table"] = L.coast_run_host_noabort(C.byref(d), C.byref(st)); r["run_host_table_err"] = L.coast_last_error().decode()
            d.d_in, d.d_out = buf, buf
            r["launch_table_without_table"] = L.coast_launch(C.byref(d), None); r["launch_table_err"] = L.coast_last_error().decode()
            L.coast_free(buf)
            out.append(r)
        elif kind == "sync_fold":                           # counters -> the reference's run-time symbols
            buf = dmalloc(1 << 16)
            d.kernel, d.num_clones, d.n_units, d.unit_bytes, d.flags = 1, op.get("nc", 3), 100, 64, 3
            d.d_in, d.d_out = buf, buf
            r = {"launch": L.coast_launch(C.byref(d), None)}
            st = R._Stats()
            r["sync"] = (L.coast_sync if op.get("abort") else L.coast_sync_noabort)(None, C.byref(st))
            r["stats"] = [st.errors_corrected, st.dwc_detected, st.syncs, st.injected, st.first_fault_unit]
            r["TMR_ERROR_CNT"] = C.c_uint32.in_dll(L, "TMR_ERROR_CNT").value
            r["SYNC_COUNT"] = C.c_uint64.in_dll(L, "__SYNC_COUNT").value
            st2 = R._Stats()
            L.coast_sync_noabort(None, C.byref(st2))        # counters were reset by the first sync
            r["second"] = [st2.errors_corrected, st2.dwc_detected, st2.syncs, st2.injected, st2.first_fault_unit]
            L.coast_free(buf)
            out.append(r)
        elif kind == "peer_counters":                       # multi-GPU fold over peer memory: a second block stands in for the owner's
            L.coast_counters_export.argtypes = [C.c_void_p]
            L.coast_counters_attach.argtypes = [C.c_void_p]
            own = C.create_string_buffer(64)
            r = {"export": L.coast_counters_export(own)}
            peer = dmalloc(40)                              # "the owner's block" (the mock's IPC handle is the pointer itself)
            C.memmove(peer, bytes(32) + b"\xff" * 8, 40)
            h = C.create_string_buffer(bytes(C.c_uint64(peer)) + bytes(56), 64)
            r["attach"] = L.coast_counters_attach(h); r["attach_err"] = L.coast_last_error().decode() if r["attach"] else ""
            r["attach_twice"] = L.coast_counters_attach(h) if r["attach"] == 0 else None
            buf = dmalloc(1 << 16)
            d.kernel, d.num_clones, d.n_units, d.unit_bytes, d.flags = 1, 3, 100, 64, 3
            d.d_in, d.d_out = buf, buf
            r["launch"] = L.coast_launch(C.byref(d), None)
            st = R._Stats()
            r["sync_attached"] = L.coast_sync_noabort(None, C.byref(st))
            r["stats_attached"] = [st.errors_corrected, st.dwc_detected, st.syncs, st.injected, st.first_fault_unit]
            r["peer_block"] = list((C.c_uint64 * 5).from_address(peer))
            r["peer_ptr"] = peer
            r["detach"] = L.coast_counters_detach()
            r["launch_local"] = L.coast_launch(C.byref(d), None)
            r["sync_local"] = L.coast_sync_noabort(None, C.byref(st))
            r["stats_local"] = [st.errors_corrected, st.dwc_detected, st.syncs, st.injected, st.first_fault_unit]
            r["peer_block_after"] = list((C.c_uint64 * 5).from_address(peer))
            L.coast_free(buf); L.coast_free(peer)
            out.append(r)
        elif kind == "shutdown":
            out.append({"rc": L.coast_shutdown()})
    L.coast_shutdown()                                      # a no-op after a "shutdown" op; the mock reports what is still live
    res["ops"] = out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
