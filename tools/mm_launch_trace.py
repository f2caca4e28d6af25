"""Prints the driver calls of every matmul launch and host call in the plan sweep, one normalised line per mock-driver event,
so that two builds of libcoast_rt.so can be compared with diff:

    python tools/mm_launch_trace.py --root <checkout> > trace.txt

The sweep is tests/test_mm_plan_sweep.py's, plus refusals (zero dimensions, n_units off the shape, the 2^31 row bounds,
misaligned or null buffers and row offsets, too many groups, combined mode bits, store votes) and host calls (pageable and
pinned buffers, several chunks, COAST_HOST_PATH=one-shot).  It runs <checkout>/coast_b200/libcoast_rt.so against this tree's
mock driver (tests/mock_cuda/mock_cuda.c) through tests/mock_cuda/mm_child.py (scaled ops: mm_scaled_child.py), one op per init,
with a marker in the log between ops, CHUNK_OPS ops per child process.  Pointers are made
comparable across processes: an 8-byte word of an argument block, a tensor-map base or a copy's device side that points into
a live allocation becomes a<id>+<offset>, a host-call chunk's biased d_in / d_out an offset from the slot buffer it is copied
through, and a pageable host address an offset into the op's buffers.  After each op its rc, error text and coast_last_host_path()."""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(HERE, "tests"))
import test_mm_plan_sweep as S  # noqa: E402
from mock_run import (KNOBS, K_CRC16, K_GEMM_BF16, K_GEMM_FP8, K_GEMM_I8, K_GEMM_TF32, K_MM_U32, K_SHA256,  # noqa: E402
                      MM_B_TRANSPOSED as BT, MM_BATCHED as BATCHED, MM_GROUPED as GROUPED, UNIT_OFFSETS)

MM = (K_MM_U32, K_GEMM_TF32, K_GEMM_BF16, K_GEMM_FP8, K_GEMM_I8)
CHUNK_OPS = 128                  # ops per child process: the mock driver keeps at most 4096 allocation records per process


def edge_ops():
    """(environment, ops) of the refusals and the host calls"""
    tiny = [16, 16, 16]
    ops = []
    for k in MM:
        b = dict(op="launch", kernel=k, nc=3)
        ops += [dict(b, M=0, N=128, K=64), dict(b, M=128, N=0, K=64), dict(b, M=128, N=128, K=0),
                dict(b, M=128, N=128, K=64, n=100), dict(b, M=128, N=128, K=64, n=0),
                dict(b, M=128, N=128, K=64, batch=2, n=3 * 128 * 128 + 1), dict(b, M=0, N=128, K=64, batch=2),
                dict(b, N=0, K=64, ro=[0, 128]), dict(b, N=128, K=0, ro=[0, 128]), dict(b, N=128, K=64, ro=[0, 128], n=100),
                dict(b, M=128, N=256, K=64, batch=1 << 23, alloc=tiny), dict(b, M=128, N=128, K=512, batch=1 << 22, alloc=tiny),
                dict(b, M=1 << 24, N=128, K=64, batch=128, alloc=tiny),
                dict(b, N=4096, K=64, ro=[0, 128], M=1 << 19, alloc=tiny), dict(b, N=128, K=4096, ro=[0, 128], M=1 << 19, alloc=tiny),
                dict(b, N=128, K=64, ro=[0, 1 << 31], alloc=tiny), dict(b, N=128, K=64, ro=[0, 128], M=(1 << 20) + 1),
                dict(b, N=128, K=64, ro=[0, 128], M=0), dict(b, M=4, N=128, K=64, mode=GROUPED),
                dict(b, N=128, K=64, ro=[0, 128], rows_shift=4),
                dict(b, M=128, N=128, K=64, mode=BATCHED | GROUPED), dict(b, M=128, N=128, K=64, batch=1, mode=BATCHED | GROUPED),
                dict(b, N=128, K=64, ro=[0, 128], mode=GROUPED | UNIT_OFFSETS), dict(b, M=128, N=128, K=64, mode=UNIT_OFFSETS),
                dict(b, M=128, N=128, K=64, flags=0x7), dict(b, M=128, N=128, K=64, flags=0x7, batch=2),
                dict(b, N=128, K=64, ro=[0, 128], flags=0x7)]
        for shift in ([8, 0, 0], [0, 8, 0], [0, 0, 8], [4, 0, 0], [0, 4, 0]):
            ops += [dict(b, M=128, N=128, K=128, shift=shift), dict(b, M=128, N=128, K=128, batch=2, shift=shift),
                    dict(b, N=128, K=128, ro=[0, 100, 300], shift=shift)]
        ops += [dict(b, M=128, N=128, K=64, p=0.3, op="run_host", n=5)]
    for k in (K_CRC16, K_SHA256):                                   # a matmul bit on another kernel
        for mode in (BATCHED, GROUPED, BT, BATCHED | BT, GROUPED | BT, UNIT_OFFSETS | BATCHED, UNIT_OFFSETS | BT):
            for call in ("launch", "run_host"):
                ops.append(dict(op=call, kernel=k, nc=3, M=0, N=0, K=0, n=64, unit_bytes=64, mode=mode, alloc=[4096, 4096, 4096]))
    host = []
    for k in MM:
        for pinned in (False, True):
            for bt in (False, True):
                b = dict(op="run_host", kernel=k, nc=2, bt=bt, pinned=pinned, unit_base=5)
                host += [dict(b, M=1024, N=128, K=64), dict(b, M=640, N=128, K=128), dict(b, M=128, N=128, K=64),
                         dict(b, M=128, N=128, K=64, batch=5), dict(b, N=128, K=64, ro=[7, 100, 228, 228, 500, 501]),
                         dict(b, N=128, K=64, ro=[7, 7]), dict(b, M=128, N=128, K=64, p=0.3),
                         dict(b, M=128, N=128, K=64, batch=2, shift=[4, 0, 0])]
    strict = [dict(op="launch", kernel=k, nc=3, M=128, N=128, K=64, flags=0x7) for k in MM]
    return [({}, ops), ({"COAST_STRICT_FLAGS": "1"}, strict), ({}, host), ({"COAST_HOST_CHUNK_BYTES": "70000"}, host),
            ({"COAST_HOST_PATH": "one-shot"}, host)]


def child(root, ops, start):
    """runs each op as its own init .. shutdown of root's library, a marker line with its index (from start) in the mock's log
    before it"""
    sys.path.insert(0, os.path.join(HERE, "tests", "mock_cuda"))
    import mm_child
    import mm_scaled_child
    mm_child.R.lib_path = lambda: os.path.join(root, "coast_b200", "libcoast_rt.so")
    results = []
    for i, op in enumerate(ops):
        with open(os.environ["MOCK_CUDA_LOG"], "a") as f:
            f.write(json.dumps({"op": "begin", "index": start + i}) + "\n")
        sys.argv = ["mm_child.py", json.dumps({"ops": [op]})]
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            (mm_scaled_child if S.child_of(op) == "mm_scaled_child.py" else mm_child).main()
        results.append(json.loads(buf.getvalue().strip().splitlines()[-1])["ops"][0])
    print(json.dumps(results))


def normalise(events, results, start):
    live = {}                                                       # id -> (base, bytes)
    lines, op = [], -1

    def dev(w, near=None):
        if near in live:
            return f"a{near}{w - live[near][0]:+d}"
        for i, (base, n) in live.items():
            if base <= w < base + n:
                return f"a{i}+{w - base}"
        return hex(w)

    def slot_allocs(j):
        """the slot buffers of a host-call chunk's launch at events[j], which its biased d_in / d_out point below: the last upload
        from the op's input before it on that stream, and the first download into the op's output after it"""
        s = events[j]["stream"]
        up = next((e["alloc"] for e in reversed(events[:j]) if e["op"] == "h2d" and e["stream"] == s and
                   (buf_of(e["host"]) or (0, ""))[1] == "host_in"), None)
        down = next((e["alloc"] for e in events[j:] if e["op"] == "d2h" and e["stream"] == s and
                     (buf_of(e["host"]) or (0, ""))[1] == "host_out"), None)
        return up, down

    def buf_of(h):
        r = results[op]
        below = [(h - r[k], k) for k in ("host_in", "host_aux", "host_out", "host_rows") if r.get(k) and r[k] <= h]
        return min(below) if below else None

    def host(h):
        if not dev(h).startswith("0x"):                             # pinned: a host allocation of the driver
            return dev(h)
        b = buf_of(h)
        return f"{b[1]}+{b[0]}" if b else "?"

    for j, e in enumerate(events):
        kind = e["op"]
        if kind == "begin":
            if op >= 0:
                lines.append("result " + json.dumps({k: results[op].get(k) for k in ("rc", "err", "path")}))
            op = e["index"] - start
            lines.append(f"op {e['index']}")
        elif kind == "alloc":
            live[e["id"]] = (e["ptr"], e["bytes"])
            lines.append(f"alloc a{e['id']} {e['bytes']} host={e['host']}")
        elif kind == "free":
            live.pop(e["id"], None)
            lines.append(f"free a{e['id']}")
        elif kind == "launch":
            raw = bytes.fromhex(e["arg0"])
            near = slot_allocs(j) if len(raw) == 128 and e["stream"] else (None, None)      # host calls run on their own streams
            words = [dev(int.from_bytes(raw[i:i + 8], "little"), near[i // 8] if i < 16 else None) for i in range(0, len(raw), 8)]
            lines.append(f"launch {e['name']} grid={e['grid']} block={e['block']} smem={e['smem']} stream={e['stream']} " + " ".join(words))
        elif kind in ("h2d", "d2h"):
            lines.append(f"{kind} a{e['alloc']}+{e['offset']} {e['bytes']} {host(e['host'])} stream={e['stream']}")
        elif kind == "tmap":
            lines.append(json.dumps(dict(e, addr=dev(e["addr"])), sort_keys=True))
        else:
            lines.append(json.dumps(e, sort_keys=True))
    if op >= 0:
        lines.append("result " + json.dumps({k: results[op].get(k) for k in ("rc", "err", "path")}))
    return lines


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--root", required=True, help="checkout whose coast_b200/libcoast_rt.so is traced")
    ap.add_argument("--child", help=argparse.SUPPRESS)          # a JSON file: the first op's index and the ops
    a = ap.parse_args()
    if a.child:
        job = json.load(open(a.child))
        return child(a.root, job["ops"], job["start"])
    root = os.path.abspath(a.root)
    n_ops = n_events = 0
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.run(["gcc", "-O1", "-shared", "-fPIC", "-Wall", "-I/usr/local/cuda/include", "-o", os.path.join(tmp, "libcuda.so.1"),
                        os.path.join(HERE, "tests", "mock_cuda", "mock_cuda.c")], check=True)
        log, ops_file = os.path.join(tmp, "mock.log"), os.path.join(tmp, "ops.json")
        for env_extra, all_ops in S.SWEEP + edge_ops():
            print("env " + json.dumps(env_extra, sort_keys=True))
            env = dict(os.environ, LD_LIBRARY_PATH=f"{tmp}:" + os.environ.get("LD_LIBRARY_PATH", ""), MOCK_CUDA_LOG=log)
            for k in KNOBS:
                env.pop(k, None)
            env.update(env_extra)
            for start in range(0, len(all_ops), CHUNK_OPS):
                ops = all_ops[start:start + CHUNK_OPS]
                if os.path.exists(log):
                    os.unlink(log)
                with open(ops_file, "w") as f:
                    json.dump({"start": start, "ops": ops}, f)
                res = subprocess.run([sys.executable, os.path.abspath(__file__), "--root", root, "--child", ops_file],
                                     capture_output=True, text=True, env=env, timeout=3600)
                if res.returncode:
                    sys.exit(res.stdout + res.stderr)
                events = [json.loads(ln) for ln in open(log)]
                for ln in normalise(events, json.loads(res.stdout.strip().splitlines()[-1]), start):
                    print(ln)
                n_ops += len(ops)
                n_events += sum(e["op"] != "begin" for e in events)
    print(f"{n_ops} ops, {n_events} events", file=sys.stderr)


if __name__ == "__main__":
    main()
