"""The exact chunks of coast_run_host() on a GPU-less box, against the mock driver (tests/mock_cuda/mock_cuda.c).  The other
host-logic tests check that every byte is copied once; these pin the schedule itself: for every chunk, in order, each upload
and download (which caller buffer, offset, bytes, stream), the launch's n_units, unit_base and M, and the events of the matmul's
shared operand.  The expected lists are built here from the schedule rules:
  uniform units  chunks ramp 1, 2, 4 .. MiB (in input bytes) up to COAST_HOST_CHUNK_BYTES and shrink again towards the end
                 (each at most half of what remains); a unit larger than that is a chunk of its own;
  ragged units   a chunk is the longest unit range whose span (twice for quicksort) and per-unit bytes fit a budget that
                 ramps 1 MiB -> COAST_HOST_CHUNK_BYTES; a longer unit is a chunk of its own;
  matmul         B once on stream 1, then C in at most 8 blocks of 128-row groups (M % 128 == 0 and M >= 512), else one shot;
  batched        as many whole products as COAST_HOST_CHUNK_BYTES holds (at least one).
Chunk i runs on host stream i % 3.  The staging memory a call keeps may be smaller than these rules' slot sizes, never larger."""
import numpy as np
import pytest

from mock_run import K_AES128, K_GEMM_TF32, K_MM_U32, K_SHA256, args_of, mock_dir, run  # noqa: F401  (mock_dir is a fixture)

KEY_PER_UNIT, KEY_WRITEBACK = 2, 4
HS = (0x1001, 0x1002, 0x1003)          # the mock numbers streams 0x1000 + k in creation order: the host call's three come first
MIB = 1 << 20


def trace(ev, bufs, in_place=False):
    """the host call's work in order: copies of the caller's buffers, protected launches, the shared operand's events"""
    out = []
    for e in ev:
        if e["op"] in ("h2d", "d2h"):
            name = [k for k, (base, size) in bufs.items() if base <= e["host"] < base + max(size, 1)]
            if name:                                       # (the counters' download is no chunk's)
                out.append((e["op"], name[0], e["host"] - bufs[name[0]][0], e["bytes"], e["stream"]))
        elif e["op"] == "launch" and "_nc" in e["name"]:
            a = args_of(e)
            where = a.inp - bufs["in"][0] if in_place else None
            out.append(("launch", a.n_units, a.unit_base, a.M, e["stream"], where))
        elif e["op"] in ("event_record", "wait_event"):
            out.append((e["op"], e["stream"]))
    return out


def kept_allocations(ev):
    """bytes of the device memory the call keeps past its end: staging slots and the matmul's B (not the counters, the first
    allocation; not host memory; not launch scratch, released before the call's last stream synchronisation)"""
    end = max(i for i, e in enumerate(ev) if e["op"] == "stream_sync")
    freed = {e["id"] for e in ev[:end] if e["op"] == "free"}
    return sorted(e["bytes"] for e in ev[:end] if e["op"] == "alloc" and not e["host"] and e["id"] != 0 and e["id"] not in freed)


def assert_kept_within(ev, slot_sizes):
    got, bound = kept_allocations(ev), sorted(slot_sizes)
    assert len(got) == len(bound) and all(g <= b for g, b in zip(got, bound)), (got, bound)


# ---------------------------------------------------------------- uniform units
def uniform_chunks(n, ib, chunk_bytes=16 * MIB):
    ibs = ib or 1
    lo = max(MIB // ibs, 1)
    hi = max(chunk_bytes // ibs, lo)
    done, ramp, chunks = 0, lo, []
    while done < n:
        left = n - done
        k = min(ramp, hi)
        if k > left // 2 and left > 2 * lo:
            k = left // 2
        k = min(max(k, lo), left)
        ramp *= 2
        chunks.append((done, k))
        done += k
    return chunks, min(hi, n)


def uniform_expect(n, ib, ob, unit_base=0, ab=0, writeback=False, status=False, hybrid=False, chunk_bytes=16 * MIB):
    chunks, largest = uniform_chunks(n, ib, chunk_bytes)
    ops = []
    for i, (f, k) in enumerate(chunks):
        s = HS[i % 3]
        if ib and not hybrid:
            ops.append(("h2d", "in", f * ib, k * ib, s))
        if ab:
            ops.append(("h2d", "aux", f * ab, k * ab, s))
        ops.append(("launch", k, unit_base + f, 0, s, f * ib if hybrid else None))
        ops.append(("d2h", "out", f * ob, k * ob, s))
        if writeback:
            ops.append(("d2h", "aux", f * ab, k * ab, s))
        if status:
            ops.append(("d2h", "status", f, k, s))
    slot = [largest * ob] + ([] if hybrid else [max(largest * ib, 16)]) + ([largest * ab] if ab else []) + ([largest] if status else [])
    return ops, slot * min(3, len(chunks))


@pytest.mark.parametrize("chunk_bytes", [None, 3_000_000])
def test_sha256_ramps_up_and_down(mock_dir, tmp_path, chunk_bytes):
    n = MIB + 123
    env = {"COAST_HOST_CHUNK_BYTES": str(chunk_bytes)} if chunk_bytes else None
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", kernel=K_SHA256, nc=3, n=n, unit_bytes=64, in_bytes=64 * n,
                                               out_bytes=32 * n, unit_base=1000), dict(op="shutdown")], "child.py", env_extra=env)
    r = res["ops"][0]
    assert r["rc"] == 0, r
    ops, slots = uniform_expect(n, 64, 32, unit_base=1000, chunk_bytes=chunk_bytes or 16 * MIB)
    sizes = [o[1] for o in ops if o[0] == "launch"]
    assert sizes[:5] == ([16384, 32768, 65536, 131072, 262144] if not chunk_bytes else [16384, 32768, 46875, 46875, 46875])
    assert sizes[-1] < sizes[4] and sum(sizes) == n          # ... and down again
    assert trace(ev, {"in": (r["host_in"], 64 * n), "out": (r["host_out"], 32 * n)}) == ops
    assert_kept_within(ev, slots)


def test_aes_per_unit_keys_with_write_back(mock_dir, tmp_path):
    n = 200000
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host_aux", kernel=K_AES128, nc=2, n=n, mode=KEY_PER_UNIT | KEY_WRITEBACK,
                                               in_bytes=16 * n, aux_bytes=16 * n, out_bytes=16 * n, unit_base=7), dict(op="shutdown")], "child.py")
    r = res["ops"][0]
    assert r["rc"] == 0, r
    ops, slots = uniform_expect(n, 16, 16, unit_base=7, ab=16, writeback=True)
    assert trace(ev, {"in": (r["host_in"], 16 * n), "aux": (r["host_aux"], 16 * n), "out": (r["host_out"], 16 * n)}) == ops
    assert_kept_within(ev, slots)


def test_aes_status_bytes(mock_dir, tmp_path):
    n = 300001
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host_status", kernel=K_AES128, nc=2, n=n, in_bytes=16 * n, out_bytes=16 * n),
                                          dict(op="shutdown")], "child.py")
    r = res["ops"][0]
    assert r["rc"] == 0, r
    ops, slots = uniform_expect(n, 16, 16, status=True)
    assert trace(ev, {"in": (r["host_in"], 16 * n), "out": (r["host_out"], 16 * n), "status": (r["host_status"], n)}) == ops
    assert_kept_within(ev, slots)


def test_hybrid_sha256_reads_the_pinned_input_in_place(mock_dir, tmp_path):
    n = 300000
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host_pinned", kernel=K_SHA256, nc=3, n=n, unit_bytes=64, in_bytes=64 * n,
                                               out_bytes=32 * n, unit_base=77, status=True), dict(op="shutdown")], "child.py",
                     env_extra={"COAST_HOST_PATH": "hybrid"})
    r = res["ops"][0]
    assert r["rc"] == 0, r
    ops, slots = uniform_expect(n, 64, 32, unit_base=77, status=True, hybrid=True)
    bufs = {"in": (r["host_in"], 64 * n), "out": (r["host_out"], 32 * n), "status": (r["host_status"], n)}
    assert trace(ev, bufs, in_place=True) == ops
    assert_kept_within(ev, slots)


def test_empty_sha256_input(mock_dir, tmp_path):
    n = 3
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", kernel=K_SHA256, nc=3, n=n, unit_bytes=0, in_bytes=0, out_bytes=32 * n,
                                               unit_base=9), dict(op="shutdown")], "child.py")
    r = res["ops"][0]
    assert r["rc"] == 0, r
    ops, slots = uniform_expect(n, 0, 32, unit_base=9)
    assert ops == [("launch", 3, 9, 0, HS[0], None), ("d2h", "out", 0, 96, HS[0])]
    assert trace(ev, {"in": (r["host_in"], 1), "out": (r["host_out"], 32 * n)}) == ops
    assert_kept_within(ev, slots)                            # the input slot is still 16 bytes: the launch needs an address


# ---------------------------------------------------------------- ragged units
def ragged_expect(off, ob, qs, unit_base, chunk_bytes):
    n, per_unit, copies = len(off) - 1, ob + 8, 2 if qs else 1
    first, budget, ops, i = 0, min(MIB, chunk_bytes), [], 0
    max_span, max_cnt = 16, 1
    while first < n:
        e = first + 1
        while e < n and (off[e + 1] - off[first]) * copies + (e + 1 - first) * per_unit <= budget:
            e += 1
        s, cnt, span = HS[i % 3], e - first, off[e] - off[first]
        if span:
            ops.append(("h2d", "in", off[first], span, s))
        ops.append(("h2d", "aux", 8 * first, 8 * (cnt + 1), s))
        ops.append(("launch", cnt, unit_base + first, 0, s, None))
        if not qs:
            ops.append(("d2h", "out", first * ob, cnt * ob, s))
        elif span:
            ops.append(("d2h", "out", off[first], span, s))
        max_span, max_cnt = max(max_span, span), max(max_cnt, cnt)
        first, budget, i = e, min(2 * budget, chunk_bytes), i + 1
    return ops, [max_span, 8 * (max_cnt + 1), max_span if qs else max_cnt * ob] * min(3, i)


def test_ragged_sha256(mock_dir, tmp_path):
    rng = np.random.default_rng(11)
    lens = rng.integers(0, 3000, 400)
    lens[::37] = 0
    lens[100] = 50000                                        # longer than the chunk bytes: a chunk of its own
    off = [int(x) for x in 5 + np.concatenate([[0], np.cumsum(lens)])]
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", kernel=K_SHA256, offsets=off, unit_bytes=50000, unit_base=1000)], "ragged_child.py",
                      env_extra={"COAST_HOST_CHUNK_BYTES": "20000"})
    r = res["ops"][0]
    assert r["rc"] == 0 and r["path"] == "staged", r
    ops, slots = ragged_expect(off, 32, False, 1000, 20000)
    assert len([o for o in ops if o[0] == "launch"]) > 20
    bufs = {"in": (r["host_in"], off[-1] + 16), "aux": (r["host_aux"], 8 * len(off)), "out": (r["host_out"], 32 * len(lens) + 16)}
    assert trace(ev, bufs) == ops
    assert_kept_within(ev, slots)


def test_ragged_quicksort(mock_dir, tmp_path):
    rng = np.random.default_rng(12)
    elems = rng.integers(0, 1025, 200)
    elems[::17] = 0
    off = [int(x) for x in 12 + 4 * np.concatenate([[0], np.cumsum(elems)])]
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", offsets=off, unit_bytes=4096, unit_base=3)], "ragged_qsort_child.py",
                     env_extra={"COAST_HOST_CHUNK_BYTES": "30000"})
    r = res["ops"][0]
    assert r["rc"] == 0 and r["path"] == "staged", r
    ops, slots = ragged_expect(off, 0, True, 3, 30000)
    assert len([o for o in ops if o[0] == "launch"]) > 20
    bufs = {"in": (r["host_in"], off[-1] + 16), "aux": (r["host_aux"], 8 * len(off)), "out": (r["host_out"], off[-1] + 16)}
    assert trace(ev, bufs) == ops
    assert_kept_within(ev, slots)


# ---------------------------------------------------------------- matmuls
@pytest.mark.parametrize("kernel,M,N,K,blocks", [(K_GEMM_TF32, 1024, 256, 128, 8), (K_MM_U32, 128, 128, 128, 1)])
def test_matmul_row_blocks_share_one_upload_of_b(mock_dir, tmp_path, kernel, M, N, K, blocks):
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host_aux", kernel=kernel, nc=3, n=M * N, M=M, N=N, K=K, in_bytes=M * K * 4,
                                               aux_bytes=K * N * 4, out_bytes=M * N * 4, unit_base=5), dict(op="shutdown")], "child.py")
    r = res["ops"][0]
    assert r["rc"] == 0, r
    rows = M // blocks
    ops = []
    for i in range(blocks):
        s, r0 = HS[i % 3], i * rows
        ops.append(("h2d", "in", r0 * K * 4, rows * K * 4, s))
        if i == 0:                                           # B follows the first block of A, on stream 1
            ops += [("h2d", "aux", 0, K * N * 4, HS[1]), ("event_record", HS[1])]
        ops += [("wait_event", s), ("launch", rows * N, 5 + r0 * N, rows, s, None), ("d2h", "out", r0 * N * 4, rows * N * 4, s)]
    bufs = {"in": (r["host_in"], M * K * 4), "aux": (r["host_aux"], K * N * 4), "out": (r["host_out"], M * N * 4)}
    assert trace(ev, bufs) == ops
    assert_kept_within(ev, [K * N * 4] + [rows * K * 4, rows * N * 4] * min(3, blocks))


@pytest.mark.parametrize("kernel,M,N,K,batch,budget,per", [
    (K_MM_U32, 64, 64, 64, 10, 100000, 2),
    (K_GEMM_TF32, 128, 128, 32, 9, 200000, 2),
])
def test_batched_chunks_of_whole_products(mock_dir, tmp_path, kernel, M, N, K, batch, budget, per):
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", kernel=kernel, nc=3, M=M, N=N, K=K, batch=batch, unit_base=1000)],
                       env_extra={"COAST_HOST_CHUNK_BYTES": str(budget)})
    r = res["ops"][0]
    assert r["rc"] == 0 and r["path"] == "staged", r
    ab, bb, cb, mn = 4 * M * K, 4 * K * N, 4 * M * N, M * N
    assert per == max(budget // (ab + bb + cb), 1)
    ops = []
    for i, f in enumerate(range(0, batch, per)):
        s, cnt = HS[i % 3], min(per, batch - f)
        ops += [("h2d", "in", f * ab, cnt * ab, s), ("h2d", "aux", f * bb, cnt * bb, s), ("launch", cnt * mn, 1000 + f * mn, M, s, None),
                ("d2h", "out", f * cb, cnt * cb, s)]
    bufs = {"in": (r["host_in"], batch * ab), "aux": (r["host_aux"], batch * bb), "out": (r["host_out"], batch * cb)}
    assert trace(ev, bufs) == ops
    assert_kept_within(ev, [per * ab, per * bb, per * cb] * min(3, -(-batch // per)))
