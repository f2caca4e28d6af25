"""Host logic of ragged batches (COAST_UNIT_OFFSETS) on a GPU-less box, against the mock driver (tests/mock_cuda/mock_cuda.c):
kernel selection and the stream-ordered cost-ordering pre-pass, the argument block, loud failures for bad arguments and bad
host offsets, and the chunk schedule of the ragged host call (every byte copied once, each offset slice uploaded unchanged
with the input pointer biased by its first offset, a long unit alone in its chunk, no zero-copy path)."""
import numpy as np
import pytest

from mock_run import BAD_ARG, K_AES128, K_CRC16, K_SHA256, UNSUPPORTED, UNIT_OFFSETS, args_of, mock_dir, run  # noqa: F401
from test_host_logic import _declared_bounds


def offsets(lens, first=3):
    return [int(x) for x in first + np.concatenate([[0], np.cumsum(lens)])]


@pytest.mark.parametrize("kernel,nc,p,want", [
    (K_SHA256, 3, 0, "xmr_sha256_var_inj0_nc3"),
    (K_SHA256, 1, 0.5, "xmr_sha256_var_inj1_nc1"),
    (K_CRC16, 2, 0.5, "xmr_crc16_var_inj1_nc2"),
])
def test_ragged_launch_runs_the_prepass_then_the_var_kernel_and_frees_its_scratch(mock_dir, tmp_path, kernel, nc, p, want):
    lens = [0, 5, 64, 200, 1, 33] * 50
    off = offsets(lens)
    op = dict(op="launch", kernel=kernel, nc=nc, offsets=off, unit_bytes=255, unit_base=1 << 32, flags=3)
    if p:
        op["p"] = p
    res, ev, _ = run(mock_dir, tmp_path, [op], "ragged_child.py")
    r = res["ops"][0]
    assert r["rc"] == 0, r["err"]
    launches = [e for e in ev if e["op"] == "launch" and e["name"] != "xmr_counters_reset"]
    assert [e["name"] for e in launches] == ["xmr_ragged_hist", "xmr_ragged_scan", "xmr_ragged_scatter", want]
    assert len({e["stream"] for e in launches}) == 1                                   # stream order
    assert launches[1]["grid"] == 1 and launches[1]["block"] == 1024
    assert int.from_bytes(bytes.fromhex(launches[0]["arg0"]), "little") == r["aux"]   # the pre-pass reads the caller's offsets
    a = args_of(launches[3])
    n = len(lens)
    assert a.mode & UNIT_OFFSETS and a.unit_bytes == 255 and a.n_units == n and a.unit_base == 1 << 32 and a.flags & 3 == 3
    assert a.inp == r["in"]
    assert launches[3]["block"] == _declared_bounds()[want][0] == 256 and launches[3]["grid"] <= 132 * 8   # its __launch_bounds__
    scratch = [e for e in ev if e["op"] == "alloc" and e["bytes"] == 64 + 4 * 1024 + 4 * n]
    assert len(scratch) == 1
    assert {"op": "free", "id": scratch[0]["id"]} in ev[ev.index(launches[3]):]       # released after the kernel


@pytest.mark.parametrize("case", ["aes", "crc_bound", "sha_bound", "null_aux", "misaligned_aux", "n_too_large"])
def test_bad_ragged_arguments_fail_loudly(mock_dir, tmp_path, case):
    op = dict(op="launch", kernel=K_SHA256, offsets=offsets([3, 4, 5]), unit_bytes=100)
    op.update({"aes": dict(kernel=K_AES128), "crc_bound": dict(kernel=K_CRC16, unit_bytes=256),
               "sha_bound": dict(unit_bytes=(1 << 28) + 1), "null_aux": dict(null_aux=True),
               "misaligned_aux": dict(aux_misalign=4), "n_too_large": dict(n=1 << 32)}[case])
    res, ev, _ = run(mock_dir, tmp_path, [op], "ragged_child.py")
    r = res["ops"][0]
    assert r["rc"] == BAD_ARG and "COAST_UNIT_OFFSETS" in r["err"], r
    assert not [e for e in ev if e["op"] == "launch" and "ragged" in e["name"]]


def test_the_bounds_themselves_are_accepted(mock_dir, tmp_path):
    res, _, _ = run(mock_dir, tmp_path, [dict(op="launch", kernel=K_CRC16, offsets=offsets([255, 0, 7]), unit_bytes=255),
                                         dict(op="launch", kernel=K_SHA256, offsets=offsets([9, 0]), unit_bytes=1 << 28)], "ragged_child.py")
    assert [r["rc"] for r in res["ops"]] == [0, 0]


@pytest.mark.parametrize("offs", [[0, 10, 5, 20], [0, 10, 400, 401]])
def test_bad_host_offsets_fail_before_any_copy(mock_dir, tmp_path, offs):
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", kernel=K_CRC16, offsets=offs, unit_bytes=255)], "ragged_child.py")
    r = res["ops"][0]
    assert r["rc"] == BAD_ARG and "offsets must not decrease" in r["err"]
    assert not [e for e in ev if e["op"] in ("h2d", "launch") and e.get("name", "") != "xmr_counters_reset"]


@pytest.mark.parametrize("pinned", [False, True])
def test_host_chunk_schedule_copies_every_byte_once_and_each_offset_slice_unchanged(mock_dir, tmp_path, pinned):
    rng = np.random.default_rng(3)
    lens = rng.integers(0, 3000, 400)
    lens[::37] = 0
    lens[100] = 50000                                          # longer than the chunk bytes: a chunk of its own
    off = offsets(lens, first=5)
    n = len(lens)
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", kernel=K_SHA256, offsets=off, unit_bytes=50000, pinned=pinned,
                                               unit_base=1000)], "ragged_child.py", env_extra={"COAST_HOST_CHUNK_BYTES": "20000"})
    r = res["ops"][0]
    assert r["rc"] == 0 and r["path"] == "staged", r
    h2d = [e for e in ev if e["op"] == "h2d"]
    ins = sorted((e["host"] - r["host_in"], e["bytes"]) for e in h2d if r["host_in"] <= e["host"] < r["host_in"] + off[-1] + 16)
    pos = off[0]
    for o, b in ins:                                           # the input, exactly once, in contiguous pieces
        assert o == pos, (o, pos)
        pos += b
    assert pos == off[-1]
    slices = [((e["host"] - r["host_aux"]) // 8, e["bytes"] // 8 - 1) for e in h2d
              if r["host_aux"] <= e["host"] < r["host_aux"] + 8 * (n + 1)]
    launches = [e for e in ev if e["op"] == "launch" and e["name"].startswith("xmr_sha256_var")]
    assert len(launches) == len(slices) > 5
    first = 0
    for (f, cnt), le in zip(slices, launches):                 # each chunk's offsets, unchanged, and its launch
        a = args_of(le)
        assert f == first and a.n_units == cnt and a.unit_base == 1000 + first
        span = off[f + cnt] - off[f]
        assert cnt == 1 or span + cnt * 40 <= 20000
        if f == 100:
            assert cnt == 1
        assert (a.inp + off[f]) % (1 << 64) % 512 == 0       # the staging slot (512-byte aligned) minus off[first]
        first += cnt
    assert first == n
    d2h = [e for e in ev if e["op"] == "d2h" and r["host_out"] <= e["host"] < r["host_out"] + 32 * n]
    assert sum(e["bytes"] for e in d2h) == 32 * n


@pytest.mark.parametrize("path", ["zerocopy", "hybrid"])
def test_forced_zero_copy_or_hybrid_ragged_host_calls_are_unsupported(mock_dir, tmp_path, path):
    res, ev, _ = run(mock_dir, tmp_path, [dict(op="run_host", kernel=K_CRC16, offsets=offsets([3, 9, 0]), unit_bytes=255, pinned=True)], "ragged_child.py",
                     env_extra={"COAST_HOST_PATH": path})
    r = res["ops"][0]
    assert r["rc"] == UNSUPPORTED and "staged only" in r["err"]
    res, _, _ = run(mock_dir, tmp_path, [dict(op="run_host", kernel=K_CRC16, offsets=offsets([3, 9, 0]), unit_bytes=255, pinned=True)], "ragged_child.py")
    assert res["ops"][0]["rc"] == 0 and res["ops"][0]["path"] == "staged"
