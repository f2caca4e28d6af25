"""GPU (H100): ragged quicksort batches (COAST_UNIT_OFFSETS with COAST_K_QSORT) -- n int32 arrays end to end with n + 1 byte
offsets, each sorted into the same bytes of d_out.

A ragged launch must equal n single-unit launches (include/coast_rt.h): every output byte (bytes outside the arrays keep
their poison), every d_status byte, the summed counters and the minimum first_fault_unit.  The reference is `ragged_qsort_run`
of test_ragged_qsort_oracle (one uniform oracle run per distinct length, pinned there against single-unit oracle runs and
numpy.sort).  The exact launches are sized from their own grid so that the warps pull several warp-tiles each from the
cost-ordered schedule."""
import os

import numpy as np
import pytest

from test_gpu_parity import dev
from test_gpu_ragged import sized_n
from test_gpu_stream_exact import GiB, _free, _room, plan_hits
from test_ragged_qsort_oracle import UNIT_OFFSETS, qsort_bounds, ragged_qsort_run

pytestmark = pytest.mark.gpu

POISON = 0xA5
BOUND = 4096
THREADS = max(os.cpu_count() or 1, 1)


def elem_counts(mix, n, rng):
    if mix == "random":                        # [0, 1024], zeros and full arrays included
        L = rng.integers(0, 1025, n)
        L[::97] = 0
        L[1::89] = 1024
    elif mix == "equal":
        L = np.full(n, 100)
    else:                                      # skewed: a few arrays at the bound, most tiny
        L = rng.integers(0, 9, n)
        L[rng.choice(n, max(n // 200, 3), replace=False)] = 1024
    return L.astype(np.int64)


def arrays(L, data, rng, lead=3, tail=2):
    """int32 arrays of L elements end to end after `lead` elements -> (bytes, int64 byte offsets)"""
    total = lead + int(L.sum()) + tail
    if data == "random":
        v = rng.integers(-(1 << 31), 1 << 31, total, dtype=np.int64).astype(np.int32)
    elif data == "equal":                      # all-equal values: every scan stops at once, every step swaps
        v = np.full(total, 7, dtype=np.int32)
    elif data == "sorted":
        v = np.arange(total, dtype=np.int32) - total // 2
    else:
        v = total // 2 - np.arange(total, dtype=np.int32)
    off = 4 * (lead + np.concatenate([[0], np.cumsum(L)])).astype(np.int64)
    return v.view(np.uint8), off


def table_plan(L, rng):
    """TABLE entries on 30 % of the units: compare-event sites (< 32 L), input-copy sites (>= 32 L), a few past the end"""
    n = len(L)
    site = rng.integers(0, 1 << 30, n) % np.maximum(33 * L + 2, 1)
    ent = 0x80000000 | (rng.integers(0, 3, n) << 29) | (site << 5) | rng.integers(0, 32, n)
    return np.where(rng.random(n) < 0.3, ent, 0).astype(np.uint32)


def launch(rt, nc, d_in, d_off, n, *, flags, plan, base, status_poison, out_bytes):
    import torch
    import coast_b200 as cb
    out = torch.full((out_bytes,), POISON, dtype=torch.uint8, device="cuda")
    status = torch.full((n,), status_poison, dtype=torch.uint8, device="cuda")
    gplan = None
    if plan is not None:
        gplan = cb.FaultPlan(mode=cb.PLAN_TABLE, table=dev(rt, plan)) if isinstance(plan, np.ndarray) else \
            cb.FaultPlan(mode=cb.PLAN_BERNOULLI, **plan)
    _, st = rt.run(cb.K_QSORT, nc, d_in, n, mode=UNIT_OFFSETS, aux=d_off, unit_bytes=BOUND, flags=flags, plan=gplan,
                   unit_base=base, out=out, status=status)
    return out.cpu().numpy(), status.cpu().numpy(), st.as_dict()


def exact(rt, oracle, nc, buf, off, n, L, *, flags, plan, base, ref=None):
    """one ragged launch against the reference, twice (d_status poisoned 0x00 and 0xFF): every output byte, all five
    counters, and d_status -- the same bytes both times, zero on units the plan does not hit and on empty arrays, under DWC
    nonzero exactly on the detected units, under TMR with -countErrors summing to the corrected errors"""
    import coast_b200 as cb
    d_in, d_off = dev(rt, buf), dev(rt, off)
    oplan = None
    if isinstance(plan, np.ndarray):
        oplan = oracle.make_plan(oracle.PLAN_TABLE, table=plan)
    elif plan is not None:
        oplan = oracle.make_plan(oracle.PLAN_BERNOULLI, **plan)
    if ref is None:
        ref = ragged_qsort_run(oracle, nc, buf, off, n, unit_bytes=BOUND, flags=flags, plan=oplan, unit_base=base,
                               out=np.full(len(buf), POISON, dtype=np.uint8), threads=THREADS)
    want, wst = ref
    got = [launch(rt, nc, d_in, d_off, n, flags=flags, plan=plan, base=base, status_poison=p, out_bytes=len(buf))
           for p in (0x00, 0xFF)]
    for out, _, st in got:
        if not np.array_equal(out, want):
            bad = np.flatnonzero(out != want)
            raise AssertionError(f"{len(bad)} output bytes differ, first at byte {bad[0]} (nc={nc} flags={flags:#x})")
        assert st == wst, (st, wst)
    s0, s1 = got[0][1], got[1][1]
    assert np.array_equal(s0, s1), f"{int((s0 != s1).sum())} status bytes never written"
    if isinstance(plan, np.ndarray):
        hit = (plan & np.uint32(0x80000000)) != 0
    elif plan is not None:
        hit = plan_hits(plan["seed"], min(int(plan["p"] * 2 ** 32), 0xFFFFFFFF), base, n).numpy()
    else:
        hit = np.zeros(n, dtype=bool)
    assert not s0[~hit | (L == 0)].any()
    if nc == 1:
        assert not s0.any()
    elif nc == 2:
        assert int((s0 != 0).sum()) == wst["dwc_detected"]
    elif flags & 1 and int(s0.max(initial=0)) < 255:
        assert int(s0.astype(np.int64).sum()) == wst["errors_corrected"]
    if plan is not None:
        assert wst["injected"] > 0
        if nc > 1:
            assert wst["first_fault_unit"] != cb.NO_FAULT_UNIT
    return ref


@pytest.mark.parametrize("data", ["random", "equal", "sorted", "reversed"])
@pytest.mark.parametrize("mix", ["random", "equal", "skewed"])
@pytest.mark.parametrize("nc", [1, 2, 3])
def test_ragged_qsort_exact_against_single_unit_semantics(rt, oracle, capfd, nc, mix, data):
    import coast_b200 as cb
    n = sized_n(rt, capfd, cb.K_QSORT, nc, BOUND)
    rng = np.random.default_rng(nc * 101 + len(mix) * 7 + len(data))
    L = elem_counts(mix, n, rng)
    buf, off = arrays(L, data, rng)
    base = (1 << 32) - n // 2
    plans = [None, dict(seed=0x5EED + nc, p=0.3), table_plan(L, rng)]
    for plan in plans:
        ref = None
        for flags in (3, 3 | cb.F_MAJORITY_VOTER):           # -countErrors -countSyncs, without and with the majority voter
            # the voter only decides between three disagreeing copies: without TMR or without faults the reference is the same
            same = nc < 3 or plan is None
            ref = exact(rt, oracle, nc, buf, off, n, L, flags=flags, plan=plan, base=base, ref=ref if same else None)


@pytest.mark.parametrize("L", [1, 17, 580, 1024])
def test_equal_lengths_equal_the_uniform_launch(rt, L):
    """an all-equal ragged batch gives the bytes and counters of the uniform xmr_qsort launch"""
    import torch
    import coast_b200 as cb
    n = 20000 if L < 1000 else 6000
    d_in = torch.empty(n * L, dtype=torch.int32, device="cuda")
    rt.fill_philox(d_in, seed=L)
    off = torch.arange(n + 1, dtype=torch.int64, device="cuda") * (4 * L)
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=77, p=0.2)
    for nc in (1, 2, 3):
        u_out, u_st = rt.run(cb.K_QSORT, nc, d_in, n, unit_bytes=4 * L, flags=3, plan=plan, unit_base=1 << 32)
        r_out, r_st = rt.run(cb.K_QSORT, nc, d_in, n, unit_bytes=BOUND, flags=3, plan=plan, unit_base=1 << 32,
                             mode=UNIT_OFFSETS, aux=off)
        assert torch.equal(u_out, r_out) and u_st == r_st and r_st.injected > 0
        if nc == 3:
            assert r_st.syncs > 0


def test_shards_equal_one_launch(rt, oracle):
    """two shard launches (off + lo, the same d_in and the same d_out, unit_base = lo) equal one launch, counters included,
    and the reference's bytes"""
    import torch
    import coast_b200 as cb
    rng = np.random.default_rng(11)
    n = 50001
    L = rng.integers(0, 1025, n)
    buf, off_h = arrays(L, "random", rng)
    d_in, off = dev(rt, buf), torch.from_numpy(off_h).cuda()
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=123, p=0.25)
    kw = dict(unit_bytes=BOUND, flags=3, plan=plan, mode=UNIT_OFFSETS)
    one = torch.full((len(buf),), POISON, dtype=torch.uint8, device="cuda")
    _, st1 = rt.run(cb.K_QSORT, 3, d_in, n, aux=off, out=one, **kw)
    two = torch.full((len(buf),), POISON, dtype=torch.uint8, device="cuda")
    lo = 20011
    _, sa = rt.run(cb.K_QSORT, 3, d_in, lo, aux=off[: lo + 1], unit_base=0, out=two, **kw)
    _, sb = rt.run(cb.K_QSORT, 3, d_in, n - lo, aux=off[lo:], unit_base=lo, out=two, **kw)
    assert torch.equal(one, two)
    assert st1.injected == sa.injected + sb.injected > 0
    assert st1.errors_corrected == sa.errors_corrected + sb.errors_corrected
    assert st1.syncs == sa.syncs + sb.syncs
    assert st1.first_fault_unit == min(sa.first_fault_unit, sb.first_fault_unit)
    ref, _ = ragged_qsort_run(oracle, 3, buf, off_h, n, unit_bytes=BOUND, flags=3, out=np.full(len(buf), POISON, np.uint8),
                              plan=oracle.make_plan(oracle.PLAN_BERNOULLI, seed=123, p=0.25), threads=THREADS)
    assert one.cpu().numpy().tobytes() == ref.tobytes()


def test_malformed_tables_are_clamped_and_rounded_on_the_device(rt, oracle):
    """offsets off the element grid, decreasing pairs and lengths above the bound, launched directly (Runtime.run refuses
    them): the kernel sorts the rounded, clamped ranges of the reference and stores nothing else"""
    import torch
    import coast_b200 as cb
    rng = np.random.default_rng(12)
    data = rng.integers(-999, 999, 1 << 16, dtype=np.int64).astype(np.int32).view(np.uint8)
    offs, pos = [], 6
    for u in range(3001):                          # offsets off the element grid; every 50th unit a spike: the unit before it
        if u % 50 == 25:                           # runs past the bound, the spike's own pair decreases
            offs.append(pos + 5000)
            pos += 600
        else:
            offs.append(pos + int(rng.integers(0, 4)))
            pos += int(rng.integers(4, 90))
    n = len(offs) - 1
    off_h = np.array(offs, dtype=np.int64)
    start, nbytes = qsort_bounds(off_h, n, 512)
    mask = np.zeros(len(data) + 4096, dtype=np.int64)
    for s, b in zip(start, nbytes):
        mask[s: s + b] += 1
    assert mask.max() == 1 and (nbytes == 512).any() and (off_h % 4 != 0).any()   # no two units overlap; the bound bites
    for nc in (1, 3):
        out = torch.full((len(data),), POISON, dtype=torch.uint8, device="cuda")
        d = rt.make_desc(cb.K_QSORT, nc, dev(rt, data), out, n, flags=3, mode=UNIT_OFFSETS, unit_bytes=512,
                         d_aux=torch.from_numpy(off_h).cuda())
        rt.launch(d)
        st = rt.sync()
        want, wst = ragged_qsort_run(oracle, nc, data, off_h, n, unit_bytes=512, flags=3,
                                     out=np.full(len(data), POISON, np.uint8), threads=THREADS)
        assert out.cpu().numpy().tobytes() == want.tobytes() and st.as_dict() == wst


@pytest.mark.parametrize("pinned", [False, True])
def test_host_call_many_chunks_equals_the_device_launch(rt, monkeypatch, pinned):
    import torch
    import coast_b200 as cb
    rng = np.random.default_rng(21)
    n = 4001
    L = rng.integers(0, 1025, n)
    L[::50] = 0
    buf, off_h = arrays(L, "random", rng)
    h_in = torch.from_numpy(buf.copy())
    h_out = torch.full((len(buf),), POISON, dtype=torch.uint8)
    if pinned:
        h_in, h_out = h_in.pin_memory(), h_out.pin_memory()
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=8, p=0.3)
    d_out = torch.full((len(buf),), POISON, dtype=torch.uint8, device="cuda")
    _, d_st = rt.run(cb.K_QSORT, 3, h_in.cuda(), n, mode=UNIT_OFFSETS, aux=torch.from_numpy(off_h).cuda(), unit_bytes=BOUND,
                     flags=3, plan=plan, unit_base=1 << 33, out=d_out)
    monkeypatch.setenv("COAST_HOST_CHUNK_BYTES", str(1 << 16))
    h_st = rt.run_host(cb.K_QSORT, 3, h_in, h_out, n, mode=UNIT_OFFSETS, h_aux=off_h.view(np.uint64), unit_bytes=BOUND,
                       flags=3, plan=plan, unit_base=1 << 33)
    assert rt.last_host_path == "staged"
    assert torch.equal(h_out, d_out.cpu()) and h_st == d_st and d_st.injected > 0
    monkeypatch.setenv("COAST_HOST_PATH", "zerocopy")
    with pytest.raises(cb.CoastError) as e:
        rt.run_host(cb.K_QSORT, 3, h_in, h_out, n, mode=UNIT_OFFSETS, h_aux=off_h.view(np.uint64), unit_bytes=BOUND)
    assert e.value.code == cb.runtime.ERR_UNSUPPORTED


def test_offsets_across_4gib(rt):
    """d_in and d_out larger than 4 GiB with off[0] just below 2^32: arrays straddle and lie beyond it; every element
    against a per-segment numpy sort, the bytes around the batch keep their poison"""
    import torch
    import coast_b200 as cb
    rng = np.random.default_rng(44)
    n = 3000
    L = rng.integers(0, 1025, n)
    off_h = ((1 << 32) - 4 * 1500) + 4 * np.concatenate([[0], np.cumsum(L)]).astype(np.int64)
    assert off_h[0] < 1 << 32 < off_h[-1] and ((off_h[:-1] < 1 << 32) & (off_h[1:] > 1 << 32)).any()
    total = int(off_h[-1]) + 4096
    _room(2 * total + GiB)
    d_in = torch.empty(total, dtype=torch.uint8, device="cuda")
    d_out = torch.full((total,), POISON, dtype=torch.uint8, device="cuda")
    lo, hi = int(off_h[0]), int(off_h[-1])
    rt.fill_philox(d_in[lo - 4096: hi + 4096], seed=4)
    _, st = rt.run(cb.K_QSORT, 3, d_in, n, mode=UNIT_OFFSETS, aux=torch.from_numpy(off_h).cuda(), unit_bytes=BOUND, flags=3,
                   out=d_out, plan=cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=9, p=0.3), unit_base=(1 << 32) - 100)
    src = d_in[lo: hi].cpu().numpy().view(np.int32)
    got = d_out[lo: hi].cpu().numpy().view(np.int32)
    assert (d_out[lo - 4096: lo].cpu().numpy() == POISON).all() and (d_out[hi: hi + 4096].cpu().numpy() == POISON).all()
    rel = (off_h - lo) // 4
    for u in range(n):                              # single faults are out-voted: every array is exactly sorted
        assert np.array_equal(got[rel[u]: rel[u + 1]], np.sort(src[rel[u]: rel[u + 1]])), u
    assert st.injected > 0 and st.errors_corrected > 0
    del d_in, d_out
    _free()


def test_bad_device_offsets_are_refused_before_the_launch(rt):
    import torch
    import coast_b200 as cb
    buf = torch.zeros(64, dtype=torch.uint8, device="cuda")
    for off, bound in (([0, 16, 8], 64), ([0, 16, 36], 16), ([0, 16, 68], 64), ([0, 16, 18], 64)):
        with pytest.raises(cb.CoastError) as e:                       # decreasing, above the bound, past inp, not whole elements
            rt.run(cb.K_QSORT, 3, buf, 2, mode=UNIT_OFFSETS, aux=torch.tensor(off, device="cuda"), unit_bytes=bound)
        assert e.value.code == cb.runtime.ERR_BAD_ARG, off
    with pytest.raises(cb.CoastError) as e:                           # a misaligned output
        rt.run(cb.K_QSORT, 3, buf, 2, mode=UNIT_OFFSETS, aux=torch.tensor([0, 16, 32], device="cuda"), unit_bytes=16,
               out=torch.zeros(72, dtype=torch.uint8, device="cuda")[2:66])
    assert e.value.code == cb.runtime.ERR_BAD_ARG
    out, st = rt.run(cb.K_QSORT, 3, buf, 2, mode=UNIT_OFFSETS, aux=torch.tensor([0, 16, 32], device="cuda"), unit_bytes=16)
    assert out.numel() == 64 and st.injected == 0                     # the default output mirrors inp
