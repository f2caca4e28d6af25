"""Host logic of ragged quicksort batches (COAST_UNIT_OFFSETS with COAST_K_QSORT) on a GPU-less box, against the mock driver
(tests/mock_cuda/mock_cuda.c): kernel selection after the cost-ordering pre-pass, one scratch allocation holding the pre-pass
part and the per-warp replica slots, loud failures for bad arguments, and the chunks of the ragged host call (each chunk
uploads and downloads the same byte span at the same offsets, with both d_in and d_out biased by its first offset)."""
import numpy as np
import pytest

from mock_run import BAD_ARG, K_QSORT, SMS, UNSUPPORTED, UNIT_OFFSETS, args_of, mock_dir, run  # noqa: F401
from test_host_logic import _declared_bounds

QSORT_THREADS = 128


def offsets(elems, first=12):
    return [int(x) for x in first + 4 * np.concatenate([[0], np.cumsum(elems)])]


def slots_offset(n):
    """xmr_ragged_slots: the ragged header, bucket counts and permutation, rounded up to 128 bytes"""
    return (64 + 4 * 1024 + 4 * n + 127) // 128 * 128


@pytest.mark.parametrize("n_copies,nc,p,want", [
    (50, 3, 0, "xmr_qsort_var_inj0_nc3"),
    (13000, 3, 0, "xmr_qsort_var_inj0_nc3"),               # more warp-tiles than one resident wave
    (50, 1, 0.5, "xmr_qsort_var_inj1_nc1"),
    (50, 2, 0.5, "xmr_qsort_var_inj1_nc2"),
])
def test_ragged_qsort_launch_runs_the_prepass_then_the_var_kernel_in_one_scratch(mock_dir, tmp_path, n_copies, nc, p, want):
    elems = [0, 5, 64, 200, 1, 33, 1024] * n_copies
    op = dict(op="launch", nc=nc, elems=[0, 5, 64, 200, 1, 33, 1024], repeat=n_copies, first=12, unit_bytes=4096,
              unit_base=1 << 32, flags=3)
    if p:
        op["p"] = p
    res, ev, _ = run(mock_dir, tmp_path, [op], "ragged_qsort_child.py")
    r = res["ops"][0]
    assert r["rc"] == 0, r["err"]
    launches = [e for e in ev if e["op"] == "launch" and e["name"] != "xmr_counters_reset"]
    assert [e["name"] for e in launches] == ["xmr_ragged_hist", "xmr_ragged_scan", "xmr_ragged_scatter", want]
    assert len({e["stream"] for e in launches}) == 1                                   # stream order
    n = len(elems)
    for pre in (launches[0], launches[2]):                                             # the pre-pass reads the caller's offsets
        assert int.from_bytes(bytes.fromhex(pre["arg0"]), "little") == r["aux"]
    assert launches[1]["grid"] == 1 and launches[1]["block"] == 1024
    k = launches[3]
    a = args_of(k)
    assert a.mode & UNIT_OFFSETS and a.unit_bytes == 4096 and a.n_units == n and a.unit_base == 1 << 32
    assert a.inp == r["in"] and a.out == r["out"]
    assert k["block"] == _declared_bounds()[want][0] == QSORT_THREADS
    upw = 32 // nc
    warps = -(-n // upw)
    assert k["grid"] == min(-(-warps // (QSORT_THREADS // 32)), SMS * 16)              # at most one resident wave
    if n_copies > 10000:
        assert k["grid"] == SMS * 16
    size = slots_offset(n) + k["grid"] * QSORT_THREADS * 4096
    scratch = [e for e in ev if e["op"] == "alloc" and e["bytes"] == size]
    allocs = [e for e in ev if e["op"] == "alloc"]
    assert len(scratch) == 1 and allocs[-1] == scratch[0]                              # the launch's one allocation
    assert {"op": "free", "id": scratch[0]["id"]} in ev[ev.index(k):]                  # released after the kernel


@pytest.mark.parametrize("case", ["bound_zero", "bound_odd", "bound_big", "in_misaligned", "out_misaligned"])
def test_bad_ragged_qsort_arguments_fail_loudly(mock_dir, tmp_path, case):
    op = dict(op="launch", offsets=offsets([3, 4, 5]), unit_bytes=64)
    op.update({"bound_zero": dict(unit_bytes=0), "bound_odd": dict(unit_bytes=62), "bound_big": dict(unit_bytes=4100),
               "in_misaligned": dict(in_misalign=2), "out_misaligned": dict(out_misalign=1)}[case])
    res, ev, _ = run(mock_dir, tmp_path, [op], "ragged_qsort_child.py")
    r = res["ops"][0]
    assert r["rc"] == BAD_ARG and "COAST_UNIT_OFFSETS" in r["err"], r
    assert not [e for e in ev if e["op"] == "launch" and e["name"] != "xmr_counters_reset"]


def test_the_bounds_themselves_are_accepted_and_aes_still_refused(mock_dir, tmp_path):
    res, _, _ = run(mock_dir, tmp_path, [dict(op="launch", offsets=offsets([1024, 0, 7]), unit_bytes=4096),
                                         dict(op="launch", offsets=offsets([1, 0, 1]), unit_bytes=4),
                                         dict(op="launch", kernel=2, offsets=offsets([4, 4]), unit_bytes=64)], "ragged_qsort_child.py")
    assert [r["rc"] for r in res["ops"]] == [0, 0, BAD_ARG]
    assert "COAST_UNIT_OFFSETS" in res["ops"][2]["err"]


def test_nested_scheduling_of_a_ragged_batch_is_unsupported(mock_dir, tmp_path):
    op = dict(op="launch", offsets=offsets([3, 4, 5]), unit_bytes=64)
    res, ev, _ = run(mock_dir, tmp_path, [op], "ragged_qsort_child.py", env_extra={"COAST_QSORT_PATH": "nested"})
    r = res["ops"][0]
    assert r["rc"] == UNSUPPORTED and "COAST_QSORT_PATH=nested" in r["err"], r
    assert not [e for e in ev if e["op"] == "launch" and "qsort" in e["name"]]


@pytest.mark.parametrize("offs", [[0, 12, 8, 20], [0, 12, 400, 404], [0, 12, 18, 24]])
def test_bad_host_offsets_fail_before_any_copy(mock_dir, tmp_path, offs):
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", offsets=offs, unit_bytes=64)], "ragged_qsort_child.py")
    r = res["ops"][0]
    assert r["rc"] == BAD_ARG and "COAST_UNIT_OFFSETS" in r["err"], r
    assert not [e for e in ev if e["op"] in ("h2d", "launch") and e.get("name", "") != "xmr_counters_reset"]


@pytest.mark.parametrize("pinned", [False, True])
def test_host_chunks_upload_and_download_the_same_spans_with_both_pointers_biased(mock_dir, tmp_path, pinned):
    rng = np.random.default_rng(3)
    elems = rng.integers(0, 1025, 300)
    elems[::37] = 0
    off = offsets(elems, first=20)
    n = len(elems)
    budget = 40000
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", offsets=off, unit_bytes=4096, pinned=pinned, unit_base=1000)], "ragged_qsort_child.py",
                     env_extra={"COAST_HOST_CHUNK_BYTES": str(budget)})
    r = res["ops"][0]
    assert r["rc"] == 0 and r["path"] == "staged", r
    h2d = [e for e in ev if e["op"] == "h2d" and r["host_in"] <= e["host"] < r["host_in"] + off[-1] + 16]
    d2h = [e for e in ev if e["op"] == "d2h" and r["host_out"] <= e["host"] < r["host_out"] + off[-1] + 16]
    ups = [(e["host"] - r["host_in"], e["bytes"]) for e in h2d]
    downs = [(e["host"] - r["host_out"], e["bytes"]) for e in d2h]
    assert ups == downs                                        # the same spans at the same offsets, in order
    pos = off[0]
    for o, b in ups:                                           # every byte once, in contiguous pieces
        assert o == pos, (o, pos)
        pos += b
    assert pos == off[-1]
    slices = [((e["host"] - r["host_aux"]) // 8, e["bytes"] // 8 - 1) for e in ev
              if e["op"] == "h2d" and r["host_aux"] <= e["host"] < r["host_aux"] + 8 * (n + 1)]
    launches = [e for e in ev if e["op"] == "launch" and e["name"].startswith("xmr_qsort_var")]
    assert len(launches) == len(slices) > 5
    first = 0
    for (f, cnt), le in zip(slices, launches):
        a = args_of(le)
        assert f == first and a.n_units == cnt and a.unit_base == 1000 + first
        span = off[f + cnt] - off[f]
        assert cnt == 1 or 2 * span + 8 * cnt <= budget         # the chunk budget counts the span in and out
        assert (a.inp + off[f]) % (1 << 64) % 512 == 0 and (a.out + off[f]) % (1 << 64) % 512 == 0   # slots minus off[first]
        first += cnt
    assert first == n


@pytest.mark.parametrize("path", ["zerocopy", "hybrid"])
def test_forced_zero_copy_or_hybrid_ragged_qsort_host_calls_are_unsupported(mock_dir, tmp_path, path):
    res, _, _ = run(mock_dir, tmp_path, [dict(op="run_host", offsets=offsets([3, 9, 0]), unit_bytes=64, pinned=True)], "ragged_qsort_child.py",
                   env_extra={"COAST_HOST_PATH": path})
    r = res["ops"][0]
    assert r["rc"] == UNSUPPORTED and "staged only" in r["err"]
