"""GPU (H100): ragged batches of SHA-256 and CRC16 (COAST_UNIT_OFFSETS) -- n messages end to end with n + 1 byte offsets.

A ragged launch must equal n single-unit launches (include/coast_rt.h): every output byte, every d_status byte, the summed
counters and the minimum first_fault_unit.  The reference is `ragged_run` of test_ragged_oracle (the oracle, one uniform run
per distinct length, pinned there against single-unit oracle runs), fed through `both()` of test_gpu_parity.  The launches
are sized from their own grid so that the warps pull several warp-tiles each from the cost-ordered schedule."""
import hashlib
import re

import numpy as np
import pytest

from test_gpu_parity import both, check_status
from test_gpu_stream_exact import GiB, _free, _room
from test_ragged_oracle import UNIT_OFFSETS, RaggedOracle, ragged_run

pytestmark = pytest.mark.gpu

REPS = 3                                   # warp-tiles per warp of the grid, at least


def ragged_grid(rt, capfd, kernel, nc, n, bound):
    """(kernel name, grid) of a ragged launch over n zero-length units, from its F_VERBOSE line"""
    import torch
    import coast_b200 as cb
    buf = torch.zeros(16, dtype=torch.uint8, device="cuda")
    off = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    capfd.readouterr()
    rt.run(kernel, nc, buf, n, mode=UNIT_OFFSETS, aux=off, unit_bytes=bound, flags=cb.F_VERBOSE)
    err = capfd.readouterr().err
    m = re.search(r"coast_rt: (\S+) grid=(\d+) block=(\d+) smem=\d+ units=%d\b" % n, err)
    assert m, err
    return m.group(1), int(m.group(2)), int(m.group(3))


def sized_n(rt, capfd, kernel, nc, bound):
    """n such that the grid's warps pull at least REPS warp-tiles each"""
    upw = 32 // nc
    probe = 64 * rt.sm_count() * 8 * upw
    _, grid, block = ragged_grid(rt, capfd, kernel, nc, probe, bound)
    assert grid * (block // 32) * upw < probe
    n = REPS * grid * (block // 32) * upw + 7
    name, grid_n, _ = ragged_grid(rt, capfd, kernel, nc, n, bound)
    assert grid_n == grid and "_var_" in name, (name, grid, grid_n)
    print(f"{name}: grid={grid} block={block} n={n}")
    return n


def lengths(kind, n, bound, rng):
    if kind == "random":
        L = rng.integers(0, bound + 1, n)
        L[:: 97] = 0
    elif kind == "equal":
        L = np.full(n, min(bound, 77))
    else:                                  # skewed: a few units at the bound, most tiny
        L = rng.integers(0, 9, n)
        L[rng.choice(n, max(n // 200, 3), replace=False)] = bound
    return L.astype(np.int64)


def packed(L, rng, lead=1):
    off = lead + np.concatenate([[0], np.cumsum(L)]).astype(np.int64)
    buf = rng.integers(0, 256, int(off[-1]) + 5, dtype=np.uint8)
    return buf, off


def status_written_twice(rt, kernel, nc, buf, n, kw, st):
    """d_status of the same launch over buffers poisoned 0x00 and 0xFF: equal (so every byte was written), zero on the units
    the plan does not hit, and under DWC nonzero exactly on the detected units"""
    import torch
    import coast_b200 as cb
    from test_gpu_parity import dev
    from test_gpu_stream_exact import plan_hits
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, **kw["plan_kw"]) if "plan_kw" in kw else \
        cb.FaultPlan(mode=cb.PLAN_TABLE, table=dev(rt, kw["table"])) if "table" in kw else None
    got = []
    for poison in (0x00, 0xFF):
        s = torch.full((n,), poison, dtype=torch.uint8, device="cuda")
        rt.run(kernel, nc, dev(rt, buf), n, flags=kw["flags"], mode=UNIT_OFFSETS, aux=dev(rt, kw["aux"]),
               unit_bytes=kw["unit_bytes"], unit_base=kw["unit_base"], plan=plan, status=s)
        got.append(s.cpu().numpy())
    assert np.array_equal(got[0], got[1]), f"{int((got[0] != got[1]).sum())} status bytes never written"
    if "plan_kw" in kw:
        thr = min(int(kw["plan_kw"]["p"] * 2 ** 32), 0xFFFFFFFF)
        hit = plan_hits(kw["plan_kw"]["seed"], thr, kw["unit_base"], n).numpy()
    elif "table" in kw:
        hit = (kw["table"] & np.uint32(0x80000000)) != 0
    else:
        hit = np.zeros(n, dtype=bool)
    assert not got[0][~hit].any()
    if nc == 2:
        assert int((got[0] != 0).sum()) == st["dwc_detected"]


RUNS = [  # plan, flags
    ("none", 0),
    ("bernoulli", 3),
    ("table", 3 | 0x100),
    ("bernoulli", 3 | 0x200),              # -storeDataSync: the in-loop votes
]


@pytest.mark.parametrize("kind", ["random", "equal", "skewed"])
@pytest.mark.parametrize("nc", [1, 2, 3])
@pytest.mark.parametrize("kname", ["sha", "crc"])
def test_ragged_exact_against_single_unit_semantics(rt, oracle, capfd, kname, nc, kind):
    import coast_b200 as cb
    kernel = cb.K_SHA256 if kname == "sha" else cb.K_CRC16
    bound = {"sha": 300 if kind != "skewed" else 4000, "crc": 255}[kname]
    n = sized_n(rt, capfd, kernel, nc, bound)
    rng = np.random.default_rng(nc * 31 + len(kind))
    L = lengths(kind, n, bound, rng)
    buf, off = packed(L, rng)
    ro = RaggedOracle(oracle)
    base = (1 << 32) - n // 2
    for plan, flags in RUNS:
        kw = dict(flags=flags, mode=UNIT_OFFSETS, unit_bytes=bound, aux=off, unit_base=base, status=True)
        if plan == "bernoulli":
            kw["plan_kw"] = dict(seed=0x5EED + nc, p=0.3)
        elif plan == "table":
            sites = 536 * ((L + 8) // 64 + 1) if kname == "sha" else 2 * L
            site = (rng.integers(0, 1 << 30, n) % np.maximum(sites + 2, 1)).astype(np.int64)
            ent = 0x80000000 | (rng.integers(0, 3, n) << 29) | (site << 5) | rng.integers(0, 32, n)
            kw["table"] = np.where(rng.random(n) < 0.3, ent, 0).astype(np.uint32)
        if flags & 0x200 and nc > 1:
            # with the in-loop votes a unit's disagreement count can be any byte value, the poison included: the status
            # check launches twice over differently poisoned buffers instead
            kw["status"] = False
            _, st = both(rt, ro, kernel, nc, buf, n, **kw)
            status_written_twice(rt, kernel, nc, buf, n, kw, st)
        else:
            _, st = both(rt, ro, kernel, nc, buf, n, **kw)
        if plan != "none":
            assert st["injected"] > 0
            if nc > 1:
                assert st["first_fault_unit"] != cb.NO_FAULT_UNIT


@pytest.mark.parametrize("L", [10, 64, 100, 4000])
@pytest.mark.parametrize("kname", ["sha", "crc"])
def test_equal_lengths_equal_the_uniform_launch(rt, kname, L):
    """an all-equal ragged batch gives the bytes and counters of the uniform launch (L = 64 is the TMA ring path there)"""
    import torch
    import coast_b200 as cb
    if kname == "crc" and L > 255:
        L = 255
    kernel = cb.K_SHA256 if kname == "sha" else cb.K_CRC16
    n = 20000 if L < 1000 else 3000
    d_in = torch.empty(n * L + 16, dtype=torch.uint8, device="cuda")
    rt.fill_philox(d_in, seed=L)
    off = torch.arange(n + 1, dtype=torch.int64, device="cuda") * L
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=77, p=0.2)
    for nc in (1, 2, 3):
        u_out, u_st = rt.run(kernel, nc, d_in, n, unit_bytes=L, flags=3, plan=plan, unit_base=1 << 32)
        r_out, r_st = rt.run(kernel, nc, d_in, n, unit_bytes=L, flags=3, plan=plan, unit_base=1 << 32, mode=UNIT_OFFSETS, aux=off)
        assert torch.equal(u_out, r_out) and u_st == r_st and r_st.injected > 0


@pytest.mark.parametrize("kname", ["sha", "crc"])
def test_shards_concatenate_to_one_launch_and_misaligned_d_in(rt, oracle, kname):
    """two shard launches (sliced offsets, unit_base = lo, the same d_in) equal one launch, counters included; d_in itself
    starts at an odd address"""
    import torch
    import coast_b200 as cb
    kernel = cb.K_SHA256 if kname == "sha" else cb.K_CRC16
    bound = 700 if kname == "sha" else 255
    rng = np.random.default_rng(11)
    n = 50001
    L = rng.integers(0, bound + 1, n)
    off_h = np.concatenate([[0], np.cumsum(L)]).astype(np.int64)
    raw = torch.empty((int(off_h[-1]) + 11) // 4 * 4, dtype=torch.uint8, device="cuda")
    rt.fill_philox(raw, seed=5)
    d_in = raw[3:]
    assert d_in.data_ptr() % 2 == 1
    off = torch.from_numpy(off_h).cuda()
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=123, p=0.25)
    kw = dict(unit_bytes=bound, flags=3, plan=plan, mode=UNIT_OFFSETS)
    one, st1 = rt.run(kernel, 3, d_in, n, aux=off, **kw)
    lo = 20011
    a, sa = rt.run(kernel, 3, d_in, lo, aux=off[: lo + 1], unit_base=0, **kw)
    b, sb = rt.run(kernel, 3, d_in, n - lo, aux=off[lo:], unit_base=lo, **kw)
    assert torch.equal(torch.cat([a, b]), one)
    assert st1.injected == sa.injected + sb.injected > 0
    assert st1.errors_corrected == sa.errors_corrected + sb.errors_corrected
    assert st1.syncs == sa.syncs + sb.syncs
    assert st1.first_fault_unit == min(sa.first_fault_unit, sb.first_fault_unit)
    # and they are the ragged reference's bytes
    ref, _ = ragged_run(oracle, kernel, 3, raw[3:].cpu().numpy(), off_h, n, unit_bytes=bound, flags=3,
                        plan=oracle.make_plan(oracle.PLAN_BERNOULLI, seed=123, p=0.25))
    assert one.cpu().numpy().tobytes() == ref.tobytes()
    del raw, d_in, one, a, b
    _free()


def test_bad_device_offsets_are_refused_before_the_launch(rt):
    import torch
    import coast_b200 as cb
    buf = torch.zeros(64, dtype=torch.uint8, device="cuda")
    for off in ([0, 10, 5], [0, 10, 300], [0, 10, 65]):
        with pytest.raises(cb.CoastError) as e:
            rt.run(cb.K_CRC16, 3, buf, 2, mode=UNIT_OFFSETS, aux=torch.tensor(off, device="cuda"), unit_bytes=255)
        assert e.value.code == cb.runtime.ERR_BAD_ARG
    with pytest.raises(cb.CoastError) as e:                        # the bit on another kernel: refused by the library
        rt.run(cb.K_AES128, 3, buf, 2, mode=UNIT_OFFSETS, aux=torch.tensor([0, 16, 32], device="cuda"))
    assert e.value.code == cb.runtime.ERR_BAD_ARG


@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("kname", ["sha", "crc"])
def test_host_call_many_chunks_equals_the_device_launch(rt, monkeypatch, kname, pinned):
    import torch
    import coast_b200 as cb
    kernel = cb.K_SHA256 if kname == "sha" else cb.K_CRC16
    bound = 3000 if kname == "sha" else 255
    rng = np.random.default_rng(21)
    n = 4001
    L = rng.integers(0, bound + 1, n)
    L[::50] = 0
    off_h = np.concatenate([[0], np.cumsum(L)]).astype(np.uint64) + 1
    h_in = torch.from_numpy(rng.integers(0, 256, int(off_h[-1]) + 3, dtype=np.uint8))
    ob = 32 if kname == "sha" else 2
    h_out = torch.zeros(n * ob, dtype=torch.uint8)
    if pinned:
        h_in, h_out = h_in.pin_memory(), h_out.pin_memory()
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=8, p=0.3)
    d_out, d_st = rt.run(kernel, 3, h_in.cuda(), n, mode=UNIT_OFFSETS, aux=torch.from_numpy(off_h.view(np.int64)).cuda(),
                         unit_bytes=bound, flags=3, plan=plan, unit_base=1 << 33)
    monkeypatch.setenv("COAST_HOST_CHUNK_BYTES", str(8192))
    h_st = rt.run_host(kernel, 3, h_in, h_out, n, mode=UNIT_OFFSETS, h_aux=off_h, unit_bytes=bound, flags=3, plan=plan,
                       unit_base=1 << 33)
    assert rt.last_host_path == "staged"
    assert torch.equal(h_out, d_out.cpu()) and h_st == d_st and d_st.injected > 0
    monkeypatch.setenv("COAST_HOST_PATH", "zerocopy")
    with pytest.raises(cb.CoastError) as e:
        rt.run_host(kernel, 3, h_in, h_out, n, mode=UNIT_OFFSETS, h_aux=off_h, unit_bytes=bound)
    assert e.value.code == cb.runtime.ERR_UNSUPPORTED


def test_sha256_tmr_ragged_batch_past_4gib(rt):
    """one ragged SHA-256 TMR batch of more than 4 GiB (64-bit offsets), every digest checked with hashlib, d_status and
    the counters against the plan"""
    import torch
    import coast_b200 as cb
    rng = np.random.default_rng(44)
    L = rng.integers(60000, 65537, 70000).astype(np.int64)
    L[::1000] = 0
    off_h = np.concatenate([[0], np.cumsum(L)]).astype(np.int64) + 5
    total = (int(off_h[-1]) + 11) // 4 * 4
    assert total > 4 * GiB
    n = len(L)
    _room(total + n * 40 + 2 * GiB)
    d_in = torch.empty(total, dtype=torch.uint8, device="cuda")
    rt.fill_philox(d_in, seed=4)
    off = torch.from_numpy(off_h).cuda()
    status = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    out = torch.full((n * 32,), 0xA5, dtype=torch.uint8, device="cuda")
    thr = 1 << 26
    _, st = rt.run(cb.K_SHA256, 3, d_in, n, mode=UNIT_OFFSETS, aux=off, unit_bytes=1 << 16, flags=3, out=out, status=status,
                   plan=cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=9, threshold=thr), unit_base=(1 << 32) - 100)
    from test_gpu_stream_exact import plan_hits
    hit = plan_hits(9, thr, (1 << 32) - 100, n).numpy()
    stat = status.cpu().numpy()
    check_status(stat, hit, 3, 3, st.as_dict())
    assert np.array_equal(stat != 0, hit)          # every flip reaches the digest
    digests = out.cpu().numpy().reshape(n, 32)
    del out, status
    step = 1 << 30
    host = np.empty(total, dtype=np.uint8)
    for s in range(0, total, step):
        host[s: s + step] = d_in[s: s + step].cpu().numpy()
    for u in range(n):
        assert digests[u].tobytes() == hashlib.sha256(host[off_h[u]: off_h[u + 1]]).digest(), u
    assert st.injected == int(hit.sum()) and st.errors_corrected == int(stat.astype(np.int64).sum())
    assert st.syncs == 32 * n
    del d_in, off, host
    _free()
