"""What every host-logic test shares: libcoast_rt.so runs in a child process (tests/mock_cuda/*_child.py) against the mock
driver (tests/mock_cuda/mock_cuda.c, test infrastructure: it runs no workload, it records and bounds-checks driver calls),
and the test reads back the child's results and the driver calls, one JSON event per line.  Kernel ids, mode bits and error
codes are the runtime's own (coast_b200/runtime.py imports no torch at module level)."""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from coast_b200.runtime import (ERR_BAD_ARG as BAD_ARG, ERR_UNSUPPORTED as UNSUPPORTED, K_AES128, K_CHSTONE_AES,  # noqa: E402,F401
                                K_CHSTONE_SHA, K_CRC16, K_GEMM_BF16, K_GEMM_FP8, K_GEMM_TF32, K_MM_U32, K_QSORT, K_SHA256,
                                MM_B_TRANSPOSED, MM_BATCHED, MM_ELEM_BYTES, MM_GROUPED, UNIT_OFFSETS)

# every environment switch of libcoast_rt.so: a child starts with none of them, so only a test's env_extra sets one
KNOBS = ("COAST_DEVICE", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_PAIR", "COAST_GEMM_TAIL_SPLIT",
         "COAST_HOST_CHUNK_BYTES", "COAST_HOST_PATH", "COAST_MM_PATH", "COAST_NUMA_BIND", "COAST_OPT_PASSES", "COAST_QSORT_PATH",
         "COAST_REPORT_COUNTERS", "COAST_STRICT_FLAGS")
SMS = 132                                                # the mock device's multiprocessor count
GRP_BYTES = lambda G: 128 + 4 * (G + 1)                  # noqa: E731  (xmr_mm_grp_bytes)


class XmrArgs(C.Structure):                     # coast_b200/csrc/xmr_args.h
    _fields_ = [("inp", C.c_uint64), ("out", C.c_uint64), ("aux", C.c_uint64), ("n_units", C.c_uint64), ("unit_base", C.c_uint64),
                ("counters", C.c_uint64), ("plan_table", C.c_uint64), ("status", C.c_uint64),
                ("unit_bytes", C.c_uint32), ("flags", C.c_uint32), ("mode", C.c_uint32), ("M", C.c_uint32), ("N", C.c_uint32),
                ("K", C.c_uint32), ("plan_mode", C.c_uint32), ("seed_lo", C.c_uint32), ("seed_hi", C.c_uint32),
                ("threshold", C.c_uint32), ("n_sites", C.c_uint32), ("n_tiles", C.c_uint32), ("key", C.c_uint8 * 16)]


@pytest.fixture(scope="session")
def mock_dir(tmp_path_factory, built_lib):
    d = tmp_path_factory.mktemp("mockcuda")
    subprocess.run(["gcc", "-O1", "-shared", "-fPIC", "-Wall", "-I/usr/local/cuda/include", "-o", str(d / "libcuda.so.1"),
                    os.path.join(ROOT, "tests", "mock_cuda", "mock_cuda.c")], check=True)
    return d


def run(mock_dir, tmp_path, ops, child="mm_child.py", env_extra=None, driver_errors=False):
    """runs ops in one child process; returns (the child's JSON result, the mock's events, the child's stderr).  The driver
    must have refused nothing (unless driver_errors) and every allocation must be freed by exit."""
    log = tmp_path / "mock.log"
    if log.exists():
        log.unlink()                                        # one log per child run
    env = dict(os.environ, LD_LIBRARY_PATH=f"{mock_dir}:" + os.environ.get("LD_LIBRARY_PATH", ""), MOCK_CUDA_LOG=str(log))
    for k in KNOBS:
        env.pop(k, None)
    env.update(env_extra or {})
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "mock_cuda", child), json.dumps({"ops": ops})],
                         capture_output=True, text=True, env=env, timeout=600)
    assert res.returncode == 0, res.stdout + res.stderr
    events = [json.loads(ln) for ln in open(log)] if log.exists() else []
    if not driver_errors:
        assert not [e for e in events if e["op"] == "error"], [e for e in events if e["op"] == "error"]
    assert events[-1] == {"op": "exit", "live_allocations": 0}
    return json.loads(res.stdout.strip().splitlines()[-1]), events, res.stderr


def args_of(ev):
    """the 128-byte argument block of an xmr_* kernel launch"""
    assert C.sizeof(XmrArgs) == 128
    return XmrArgs.from_buffer_copy(bytes.fromhex(ev["arg0"]))


def arg0_ptr(ev):
    """the first kernel parameter of a helper launch (the mock logs its 8 bytes): a pointer"""
    return int.from_bytes(bytes.fromhex(ev["arg0"]), "little")


def work(ev):
    return [e for e in ev if e["op"] == "launch" and e["name"] != "xmr_counters_reset"]


def maps(ev):
    """(start, element bytes, dim0, dim1, box0, box1) of every tensor map, in encoding order"""
    return [(t["addr"], t["elem"], t["dim0"], t["dim1"], t["box0"], t["box1"]) for t in ev if t["op"] == "tmap"]


def scratch(ev, sizes):
    """bytes of every allocation after the caller's buffers (sizes, in order) and before the matmul kernel"""
    allocs = [(i, e["bytes"]) for i, e in enumerate(ev) if e["op"] == "alloc" and not e["host"]]
    for j in range(len(allocs) - len(sizes) + 1):
        if [b for _, b in allocs[j:j + len(sizes)]] == sizes:
            k = ev.index(work(ev)[-1])
            return [b for i, b in allocs[j + len(sizes):] if i < k]
    raise AssertionError("the caller's buffers are not in the log")


def spans(ev, op, base, size):
    """(host offset, bytes, stream, device offset) of every copy of kind op whose host side lies in [base, base + size)"""
    return [(e["host"] - base, e["bytes"], e["stream"], e["offset"]) for e in ev if e["op"] == op and base <= e["host"] < base + size]
