"""Ragged quicksort batches (COAST_UNIT_OFFSETS with COAST_K_QSORT) on the CPU: the reference the GPU tests compare against.

A ragged quicksort launch is defined as n single-unit uniform launches (include/coast_rt.h): unit u sorts the int32 array
d_in[off[u] .. off[u+1]) with unit_bytes = its length and global index unit_base + u, and its sorted array lands in the same
bytes of d_out.  `ragged_qsort_run` computes that with one uniform oracle run per distinct length; the fault plan is handed
over as a per-unit TABLE decided against each unit's own 33 L sites.  A zero-length array (which the uniform path refuses)
has no sites, writes nothing, has d_status 0 and executes exactly one sync point, the `if (len < 2) return;` of
quicksort.c:122 -- what the oracle's orc_qsort_unit does at L = 0.  The kernel takes every offset rounded down to a multiple
of 4 and clamps every length to [0, unit_bytes] (a decreasing pair is empty); the reference does the same.  Here the reference
is pinned against real single-unit oracle runs and numpy.sort."""
import numpy as np
import pytest

from test_gpu_stream_exact import plan_draw
from test_ragged_oracle import NO_FAULT_UNIT, STAT_KEYS

UNIT_OFFSETS = 0x10000
F_COUNT_ERRORS, F_COUNT_SYNCS, F_MAJORITY = 0x1, 0x2, 0x100


def qsort_bounds(off, n, bound):
    """(first byte, byte length) of every unit as the kernel takes them: offsets rounded down to a multiple of 4, lengths
    clamped to [0, bound], a decreasing pair empty"""
    o = np.asarray(off)[: n + 1].astype(np.uint64) & ~np.uint64(3)
    hi, lo = o[1:], o[:-1]
    d = np.where(hi > lo, hi - lo, np.uint64(0))
    return lo.astype(np.int64), np.minimum(d, np.uint64(bound)).astype(np.int64)


def qsort_table(oracle, nc, elems, plan, unit_base):
    """the plan as one u32 entry per unit (0: no fault), each decided against the unit's own 33 L sites (width 32)"""
    n = len(elems)
    if plan is None or plan.mode == oracle.PLAN_NONE:
        return None
    if plan.mode == oracle.PLAN_TABLE:
        return np.asarray(plan._keep, dtype=np.uint32)[:n].copy()
    seed = int(plan.seed_lo) | (int(plan.seed_hi) << 32)
    x0, x1, x2, x3 = (t.numpy().astype(np.int64) for t in plan_draw(seed, unit_base, n))
    sites = 33 * elems
    hit = (x0 < int(plan.threshold)) & (sites > 0)
    site = x2 % np.maximum(sites, 1)
    ent = 0x80000000 | ((x1 % nc) << 29) | (site << 5) | (x3 % 32)
    return np.where(hit, ent, 0).astype(np.uint32)


def ragged_qsort_run(oracle, nc, inp, off, n, *, unit_bytes, flags=0, plan=None, unit_base=0, out=None, threads=1):
    """(output bytes, counters) of a ragged quicksort launch.  `out` is the output buffer before the launch (zeros the size
    of inp by default); only the units' bytes change."""
    inp = np.ascontiguousarray(inp).view(np.uint8).ravel()
    res = np.zeros(len(inp), dtype=np.uint8) if out is None else np.array(out, dtype=np.uint8).ravel().copy()
    start, nbytes = qsort_bounds(off, n, unit_bytes)
    elems = nbytes // 4
    table = qsort_table(oracle, nc, elems, plan, unit_base)
    st = {k: 0 for k in STAT_KEYS}
    st["first_fault_unit"] = NO_FAULT_UNIT
    order = np.argsort(elems, kind="stable")
    uniq, starts = np.unique(elems[order], return_index=True)
    bounds = list(starts) + [n]
    groups = [(order[bounds[g]:bounds[g + 1]], int(L)) for g, L in enumerate(uniq)]

    inp32 = inp[: len(inp) // 4 * 4].view(np.int32)   # units start on element boundaries: gather whole elements
    res32 = res[: len(res) // 4 * 4].view(np.int32)

    def one(group):                                   # one uniform oracle run over the units of one length
        idx, L = group
        pos = (start[idx] // 4)[:, None] + np.arange(L, dtype=np.int64)[None, :]
        gplan = oracle.make_plan(oracle.PLAN_TABLE, table=np.ascontiguousarray(table[idx])) if table is not None else None
        o, s = oracle.run(oracle.K_QSORT, nc, inp32[pos].ravel(), len(idx), flags=flags, unit_bytes=4 * L, plan=gplan,
                          unit_base=0)
        return pos, o, s

    for idx, L in groups:
        if L == 0 and nc == 3 and flags & F_COUNT_ERRORS and flags & F_COUNT_SYNCS:
            st["syncs"] += len(idx)                   # no sites, no stores, one `if (len < 2) return;`
    work = [g for g in groups if g[1]]
    if threads > 1:                                   # the oracle runs without the GIL: the groups in parallel
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(threads) as ex:
            results = list(ex.map(one, work))
    else:
        results = [one(g) for g in work]
    for (idx, L), (pos, o, s) in zip(work, results):
        res32[pos] = o.view(np.int32).reshape(len(idx), L)
        for k in STAT_KEYS[:4]:
            st[k] += s[k]
        if s["first_fault_unit"] != NO_FAULT_UNIT:
            st["first_fault_unit"] = min(st["first_fault_unit"], unit_base + int(idx[s["first_fault_unit"]]))
    return res, st


def packed_arrays(elems, rng, lead=2, tail=3, low=-(1 << 31), high=1 << 31):
    """int32 arrays of the given element counts end to end after `lead` junk elements -> (bytes, int64 byte offsets)"""
    total = lead + int(np.sum(elems)) + tail
    data = rng.integers(low, high, total, dtype=np.int64).astype(np.int32)
    off = 4 * (lead + np.concatenate([[0], np.cumsum(elems)])).astype(np.int64)
    return data.view(np.uint8), off


def single_unit_runs(oracle, nc, buf, off, n, *, unit_bytes, flags=0, plan_kw=None, table=None, unit_base=0):
    """the definition: one uniform single-unit oracle run per unit (zero-length units as defined above)"""
    start, nbytes = qsort_bounds(off, n, unit_bytes)
    res = np.zeros(len(buf), dtype=np.uint8)
    st = {k: 0 for k in STAT_KEYS}
    st["first_fault_unit"] = NO_FAULT_UNIT
    for u in range(n):
        B = int(nbytes[u])
        if B == 0:
            st["syncs"] += 1 if nc == 3 and flags & 3 == 3 else 0
            continue
        plan = None
        if table is not None:
            plan = oracle.make_plan(oracle.PLAN_TABLE, table=np.ascontiguousarray(table[u:u + 1]))
        elif plan_kw:
            plan = oracle.make_plan(oracle.PLAN_BERNOULLI, **plan_kw)
        o, s = oracle.run(oracle.K_QSORT, nc, buf[start[u]: start[u] + B], 1, flags=flags, unit_bytes=B, plan=plan,
                          unit_base=unit_base + u)
        res[start[u]: start[u] + B] = o
        for k in STAT_KEYS[:4]:
            st[k] += s[k]
        st["first_fault_unit"] = min(st["first_fault_unit"], s["first_fault_unit"])
    return res, st


CASES = [  # nc, flags
    (1, 3), (2, 3), (3, 3), (3, 3 | F_MAJORITY), (3, 0), (2, 0),
]


@pytest.mark.parametrize("plan", ["none", "bernoulli", "table"])
@pytest.mark.parametrize("case", CASES, ids=[f"nc{c[0]}-f{c[1]:x}" for c in CASES])
def test_ragged_qsort_reference_equals_single_unit_runs(oracle, case, plan):
    nc, flags = case
    rng = np.random.default_rng(nc * 13 + flags)
    n, bound = 60, 4 * 200
    elems = rng.integers(0, 201, n)
    elems[:6] = [0, 0, 200, 1, 2, 0]
    buf, off = packed_arrays(elems, rng, low=-50, high=50)          # duplicates: long scans and equal pivots
    base = (1 << 32) - 25                                            # global units cross 2^32
    plan_kw = table = oplan = None
    if plan == "bernoulli":
        plan_kw = dict(seed=41 + nc, p=0.3)
        oplan = oracle.make_plan(oracle.PLAN_BERNOULLI, **plan_kw)
    elif plan == "table":
        ents = []
        for u, L in enumerate(elems):
            L = int(L)
            if L == 0 or u % 5 == 4:
                ents.append(oracle.fault_entry(0, 3, 1) if L == 0 else 0)    # an entry on a unit without sites is ignored
            elif u % 2:
                ents.append(oracle.fault_entry(u % 3, int(rng.integers(0, 32 * L)), int(rng.integers(0, 32))))   # compare event
            else:
                ents.append(oracle.fault_entry(u % 3, 32 * L + int(rng.integers(0, L)), int(rng.integers(0, 32))))   # input copy
        table = np.array(ents, dtype=np.uint32)
        oplan = oracle.make_plan(oracle.PLAN_TABLE, table=table)
    want, wst = single_unit_runs(oracle, nc, buf, off, n, unit_bytes=bound, flags=flags, plan_kw=plan_kw, table=table,
                                 unit_base=base)
    got, gst = ragged_qsort_run(oracle, nc, buf, off, n, unit_bytes=bound, flags=flags, plan=oplan, unit_base=base)
    assert got.tobytes() == want.tobytes()
    assert gst == wst
    if plan == "none":
        assert gst["injected"] == 0
    else:
        assert gst["injected"] > 0
        if nc > 1:
            assert gst["first_fault_unit"] >= base and gst["first_fault_unit"] != NO_FAULT_UNIT
    if nc == 3 and flags & 3 == 3:                                   # every sync point counted, the zero-length units' included
        assert gst["syncs"] > 3 * n


def test_ragged_qsort_sorts_every_length_0_to_1024_like_numpy(oracle):
    rng = np.random.default_rng(7)
    elems = np.arange(1025)
    rng.shuffle(elems)
    buf, off = packed_arrays(elems, rng, low=-1000, high=1000)
    out, st = ragged_qsort_run(oracle, 3, buf, off, len(elems), unit_bytes=4096, flags=3, threads=4)
    assert out.tobytes() == ragged_qsort_run(oracle, 3, buf, off, len(elems), unit_bytes=4096, flags=3)[0].tobytes()
    a, o = buf.view(np.int32), out.view(np.int32)
    for u in range(len(elems)):
        s, e = off[u] // 4, off[u + 1] // 4
        assert np.array_equal(o[s:e], np.sort(a[s:e])), int(elems[u])
    assert not o[: off[0] // 4].any() and not o[off[-1] // 4:].any()   # nothing outside the units
    assert st["errors_corrected"] == 0 and st["injected"] == 0


def test_zero_length_arrays_have_one_sync_point_no_sites_and_no_stores(oracle):
    rng = np.random.default_rng(3)
    elems = np.array([0, 3, 0, 0, 5, 0])
    buf, off = packed_arrays(elems, rng)
    poison = np.full(len(buf), 0xA5, dtype=np.uint8)
    plan = oracle.make_plan(oracle.PLAN_BERNOULLI, seed=3, threshold=0xFFFFFFFF)
    out, st = ragged_qsort_run(oracle, 3, buf, off, len(elems), unit_bytes=64, flags=3, plan=plan, out=poison)
    assert st["injected"] == 2                                      # p = 1, but only the units with sites
    want3, s3 = oracle.run(oracle.K_QSORT, 3, buf[off[1]: off[2]], 1, unit_bytes=12, flags=3, plan=plan, unit_base=1)
    want5, s5 = oracle.run(oracle.K_QSORT, 3, buf[off[4]: off[5]], 1, unit_bytes=20, flags=3, plan=plan, unit_base=4)
    assert st["syncs"] == s3["syncs"] + s5["syncs"] + 4
    keep = np.ones(len(buf), dtype=bool)
    keep[off[1]: off[2]] = keep[off[4]: off[5]] = False
    assert (out[keep] == 0xA5).all()
    assert out[off[1]: off[2]].tobytes() == want3.tobytes() and out[off[4]: off[5]].tobytes() == want5.tobytes()


def test_offsets_round_down_to_elements_and_lengths_clamp():
    off = np.array([5, 16, 12, 12, 43, 4200 + 43, 4200 + 48], dtype=np.uint64)
    start, nbytes = qsort_bounds(off, 6, 64)
    assert start.tolist() == [4, 16, 12, 12, 40, 4240]
    assert nbytes.tolist() == [12, 0, 0, 28, 64, 8]                 # round down, decreasing, empty, rounded, above the bound


def test_clamped_and_rounded_tables_sort_exactly_those_elements(oracle):
    """a malformed table: offsets off the element grid, a decreasing pair, a length above the bound -- the reference sorts
    the rounded, clamped ranges and leaves every other byte alone (the same single-unit definition)"""
    rng = np.random.default_rng(9)
    data = rng.integers(-99, 99, 3000, dtype=np.int64).astype(np.int32).view(np.uint8)
    off = np.array([2906, 2947, 30, 30, 101, 2000, 2000 + 803, 2000 + 808], dtype=np.uint64)   # no two units overlap
    n, bound = 7, 400
    poison = np.full(len(data), 0xA5, dtype=np.uint8)
    out, st = ragged_qsort_run(oracle, 3, data, off, n, unit_bytes=bound, flags=3, out=poison)
    want, wst = single_unit_runs(oracle, 3, data, off, n, unit_bytes=bound, flags=3)
    start, nbytes = qsort_bounds(off, n, bound)
    assert nbytes.tolist() == [40, 0, 0, 72, 400, 400, 8] and start.tolist() == [2904, 2944, 28, 28, 100, 2000, 2800]
    mask = np.zeros(len(data), dtype=bool)
    for s, b in zip(start, nbytes):
        mask[s: s + b] = True
        assert np.array_equal(out[s: s + b].view(np.int32), np.sort(data[s: s + b].view(np.int32)))
    assert (out[~mask] == 0xA5).all() and out[mask].tobytes() == want[mask].tobytes() and st == wst
