"""Ragged batches (COAST_UNIT_OFFSETS) on the CPU: the reference the GPU tests compare against.

A ragged launch is defined as n single-unit launches: unit u with unit_bytes = its length, its own bytes and global index
unit_base + u (include/coast_rt.h).  `ragged_run` computes exactly that with the oracle, fast enough for launches of
several hundred thousand units: the units are grouped by length and each group is one uniform oracle run.  A group's units
are not consecutive, so the fault plan is handed over as a TABLE: each unit's Bernoulli decision is drawn for its global
index and taken modulo its own site count (a unit without sites is never hit).  Here that reference is pinned against real
single-unit oracle runs, hashlib and the CRC16 reference, at every length class of the padding."""
import hashlib

import numpy as np
import pytest

from test_gpu_stream_exact import crc16_ref, plan_draw

UNIT_OFFSETS = 0x10000
STAT_KEYS = ("errors_corrected", "dwc_detected", "syncs", "injected", "first_fault_unit")
NO_FAULT_UNIT = (1 << 64) - 1


def ragged_lengths(off, n, bound):
    """per-unit lengths as the kernels take them: off[u+1] - off[u] clamped to [0, bound]"""
    o = np.asarray(off)[: n + 1].astype(np.uint64)
    hi, lo = o[1:], o[:-1]
    d = np.where(hi > lo, hi - lo, np.uint64(0))
    return np.minimum(d, np.uint64(bound)).astype(np.int64)


def ragged_sites(oracle, kernel, lens):
    if kernel == oracle.K_SHA256:
        return 536 * ((lens + 8) // 64 + 1)
    assert kernel == oracle.K_CRC16
    return 2 * lens


def ragged_table(oracle, kernel, nc, lens, plan, unit_base):
    """the plan as one u32 entry per unit (0: no fault), each decided against the unit's own site count"""
    n = len(lens)
    if plan is None or plan.mode == oracle.PLAN_NONE:
        return None
    if plan.mode == oracle.PLAN_TABLE:
        return np.asarray(plan._keep, dtype=np.uint32)[:n].copy()
    seed = int(plan.seed_lo) | (int(plan.seed_hi) << 32)
    x0, x1, x2, x3 = (t.numpy().astype(np.int64) for t in plan_draw(seed, unit_base, n))
    sites = ragged_sites(oracle, kernel, lens)
    assert (sites < 1 << 24).all()
    hit = (x0 < int(plan.threshold)) & (sites > 0)
    site = x2 % np.maximum(sites, 1)
    width = np.where(site < lens, 16, 8) if kernel == oracle.K_CRC16 else np.full(n, 32)
    bit = x3 % width
    ent = 0x80000000 | ((x1 % nc) << 29) | (site << 5) | bit
    return np.where(hit, ent, 0).astype(np.uint32)


def ragged_run(oracle, kernel, nc, inp, off, n, *, unit_bytes, flags=0, plan=None, unit_base=0, threads=1):
    """(output bytes, counters) of a ragged launch, from one uniform oracle run per distinct length"""
    inp = np.ascontiguousarray(inp).view(np.uint8).ravel()
    o64 = np.asarray(off).astype(np.uint64)[: n + 1]
    lens = ragged_lengths(o64, n, unit_bytes)
    ob = oracle.out_bytes_per_unit(kernel)
    out = np.zeros((n, ob), dtype=np.uint8)
    table = ragged_table(oracle, kernel, nc, lens, plan, unit_base)
    st = {k: 0 for k in STAT_KEYS}
    st["first_fault_unit"] = NO_FAULT_UNIT
    order = np.argsort(lens, kind="stable")
    uniq, starts = np.unique(lens[order], return_index=True)
    bounds = list(starts) + [n]
    for g, L in enumerate(uniq):
        idx = order[bounds[g]:bounds[g + 1]]
        L = int(L)
        if L:
            pos = o64[idx].astype(np.int64)[:, None] + np.arange(L, dtype=np.int64)[None, :]
            data = inp[pos].ravel()
        else:
            data = np.zeros(16, dtype=np.uint8)
        gplan = oracle.make_plan(oracle.PLAN_TABLE, table=np.ascontiguousarray(table[idx])) if table is not None else None
        o, s = oracle.run(kernel, nc, data, len(idx), flags=flags, unit_bytes=L, plan=gplan, unit_base=0,
                          threads=threads if len(idx) >= 1 << 12 else 1)
        out[idx] = o.reshape(len(idx), ob)
        for k in STAT_KEYS[:4]:
            st[k] += s[k]
        if s["first_fault_unit"] != NO_FAULT_UNIT:
            st["first_fault_unit"] = min(st["first_fault_unit"], unit_base + int(idx[s["first_fault_unit"]]))
    return out.ravel(), st


class RaggedOracle:
    """pyoracle with the COAST_UNIT_OFFSETS mode (offsets in `aux`), for `both()` of test_gpu_parity"""

    def __init__(self, oracle):
        self._o = oracle

    def __getattr__(self, name):
        return getattr(self._o, name)

    def run(self, kernel, nc, inp, n, *, mode=0, aux=None, unit_bytes=0, flags=0, plan=None, unit_base=0, threads=1, **kw):
        if not mode & UNIT_OFFSETS:
            return self._o.run(kernel, nc, inp, n, mode=mode, aux=aux, unit_bytes=unit_bytes, flags=flags, plan=plan,
                               unit_base=unit_base, threads=threads, **kw)
        return ragged_run(self._o, kernel, nc, inp, aux, n, unit_bytes=unit_bytes, flags=flags, plan=plan,
                          unit_base=unit_base, threads=threads)


def pack(msgs, lead=1, tail=3):
    """messages end to end after `lead` junk bytes (so offsets are not multiples of 4) -> (bytes, int64 offsets)"""
    rng = np.random.default_rng(5)
    parts = [rng.integers(0, 256, lead, dtype=np.uint8)] + [np.frombuffer(bytes(m), dtype=np.uint8) for m in msgs]
    parts.append(rng.integers(0, 256, tail, dtype=np.uint8))
    off = lead + np.concatenate([[0], np.cumsum([len(m) for m in msgs])]).astype(np.int64)
    return np.concatenate(parts), off


def single_unit_runs(oracle, kernel, nc, buf, off, n, *, unit_bytes, flags=0, plan_kw=None, table=None, unit_base=0):
    """the definition: n uniform single-unit oracle runs; returns (outputs, summed counters, per-unit disagreement)"""
    lens = ragged_lengths(off, n, unit_bytes)
    ob = oracle.out_bytes_per_unit(kernel)
    out = np.zeros((n, ob), dtype=np.uint8)
    st = {k: 0 for k in STAT_KEYS}
    st["first_fault_unit"] = NO_FAULT_UNIT
    dis = np.zeros(n, dtype=bool)
    for u in range(n):
        L = int(lens[u])
        data = buf[int(off[u]): int(off[u]) + L] if L else np.zeros(1, dtype=np.uint8)
        plan = None
        if table is not None:
            plan = oracle.make_plan(oracle.PLAN_TABLE, table=np.ascontiguousarray(table[u:u + 1]))
        elif plan_kw:
            plan = oracle.make_plan(oracle.PLAN_BERNOULLI, **plan_kw)
        o, s = oracle.run(kernel, nc, data, 1, flags=flags, unit_bytes=L, plan=plan, unit_base=unit_base + u)
        out[u] = o
        for k in STAT_KEYS[:4]:
            st[k] += s[k]
        if s["first_fault_unit"] != NO_FAULT_UNIT:
            dis[u] = True
            st["first_fault_unit"] = min(st["first_fault_unit"], s["first_fault_unit"])
    return out.ravel(), st, dis


SHA_LENGTHS = list(range(201)) + [4000, 55, 56, 63, 64, 119, 120]


def test_ragged_sha256_digests_equal_hashlib_at_every_padding_class(oracle):
    rng = np.random.default_rng(1)
    msgs = [rng.integers(0, 256, L, dtype=np.uint8).tobytes() for L in SHA_LENGTHS]
    buf, off = pack(msgs)
    assert (off[:-1] % 4 != 0).any()
    out, st = ragged_run(oracle, oracle.K_SHA256, 3, buf, off, len(msgs), unit_bytes=4000)
    for i, m in enumerate(msgs):
        assert out[32 * i: 32 * i + 32].tobytes() == hashlib.sha256(m).digest(), SHA_LENGTHS[i]
    assert st["injected"] == 0 and st["first_fault_unit"] == NO_FAULT_UNIT


def test_ragged_crc16_equals_the_reference_and_the_shipped_message(oracle):
    rng = np.random.default_rng(2)
    msgs = [b"Automated TMR"] + [rng.integers(0, 256, L, dtype=np.uint8).tobytes() for L in [0, 1, 2, 3, 4, 5, 0, 63, 64, 65, 255, 0]]
    buf, off = pack(msgs, lead=3)
    out, _ = ragged_run(oracle, oracle.K_CRC16, 3, buf, off, len(msgs), unit_bytes=255)
    crcs = out.view(np.uint16)
    assert int(crcs[0]) == 0x5BA3
    import torch
    for i, m in enumerate(msgs):
        ref = int(crc16_ref(torch.frombuffer(bytearray(m) or bytearray(1), dtype=torch.uint8)[: len(m)].reshape(1, -1))[0])
        assert int(crcs[i]) == ref == (0xFFFF if not m else oracle.crc16(m)), i


def test_ragged_lengths_clamp_decreasing_pairs_and_long_units():
    off = np.array([10, 20, 15, 15, 400, 401], dtype=np.uint64)
    assert ragged_lengths(off, 5, 255).tolist() == [10, 0, 0, 255, 1]


CASES = [  # kernel name, nc, flags
    ("sha", 1, 3), ("sha", 2, 3), ("sha", 3, 3), ("sha", 3, 3 | 0x100), ("sha", 3, 3 | 0x200), ("sha", 2, 0x200),
    ("crc", 1, 3), ("crc", 2, 3), ("crc", 3, 3), ("crc", 3, 3 | 0x100), ("crc", 3, 3 | 0x200), ("crc", 2, 3 | 0x200),
]


@pytest.mark.parametrize("plan", ["bernoulli", "table"])
@pytest.mark.parametrize("case", CASES, ids=["-".join(map(str, c)) for c in CASES])
def test_ragged_reference_equals_single_unit_runs_under_faults(oracle, case, plan):
    name, nc, flags = case
    kernel = oracle.K_SHA256 if name == "sha" else oracle.K_CRC16
    bound = 300 if name == "sha" else 255
    rng = np.random.default_rng(nc * 7 + flags)
    n = 48
    lens = rng.integers(0, bound + 1, n)
    lens[:4] = [0, 0, bound, 1]
    buf, off = pack([rng.integers(0, 256, int(L), dtype=np.uint8).tobytes() for L in lens], lead=2)
    base = (1 << 32) - 20
    plan_kw = table = None
    if plan == "bernoulli":
        plan_kw = dict(seed=99 + nc, p=0.3)
        oplan = oracle.make_plan(oracle.PLAN_BERNOULLI, **plan_kw)
    else:
        sites = ragged_sites(oracle, kernel, lens)
        table = np.array([oracle.fault_entry(int(rng.integers(0, 4)), int(rng.integers(0, max(int(s), 1) + 3)), int(rng.integers(0, 32)))
                          if rng.random() < 0.6 else 0 for s in sites], dtype=np.uint32)
        oplan = oracle.make_plan(oracle.PLAN_TABLE, table=table)
    want, wst, dis = single_unit_runs(oracle, kernel, nc, buf, off, n, unit_bytes=bound, flags=flags, plan_kw=plan_kw,
                                      table=table, unit_base=base)
    got, gst = ragged_run(oracle, kernel, nc, buf, off, n, unit_bytes=bound, flags=flags, plan=oplan, unit_base=base)
    assert got.tobytes() == want.tobytes()
    assert gst == wst
    assert wst["injected"] > 0
    if nc > 1:
        assert dis.any() and wst["first_fault_unit"] == base + int(np.flatnonzero(dis)[0])


def test_zero_length_crc_units_are_never_injected(oracle):
    msgs = [b"", b"\x01", b"", b"", b"abc"]
    buf, off = pack(msgs)
    plan = oracle.make_plan(oracle.PLAN_BERNOULLI, seed=3, threshold=0xFFFFFFFF)
    out, st = ragged_run(oracle, oracle.K_CRC16, 3, buf, off, len(msgs), unit_bytes=255, flags=3, plan=plan)
    assert st["injected"] == 2                       # p = 1, but only the units with sites
    assert [int(x) for x in out.view(np.uint16)[[0, 2, 3]]] == [0xFFFF] * 3
    assert st["syncs"] == 5                          # one SoR-exit vote per unit
