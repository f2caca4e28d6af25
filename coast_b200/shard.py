"""Multi-GPU host logic: the protected workloads shard by independent units (SURVEY.md 8e).

One process per GPU; rank r owns the contiguous GLOBAL unit range shard_range(n, r, world) and
passes its start as ``unit_base`` so the Philox fault plan -- keyed by the global unit index --
is identical to the single-GPU run.  No data-path collective exists: the only exchange is the
reduction of the five counters (SUM for the four counts, MIN for first_fault_unit).
"""
from __future__ import annotations

NO_FAULT_UNIT = 0xFFFFFFFFFFFFFFFF
_I64_MAX = 0x7FFFFFFFFFFFFFFF


def shard_range(n_units: int, rank: int, world: int) -> tuple[int, int]:
    """Contiguous, balanced: the first (n % world) ranks get one extra unit."""
    if world < 1 or not (0 <= rank < world):
        raise ValueError("bad rank/world")
    base, rem = divmod(n_units, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_groups(row_offsets, rank: int, world: int) -> tuple[int, int]:
    """Whole products [g_lo, g_hi) of a grouped matmul (COAST_MM_GROUPED) for ``rank``, balanced by rows: rank r takes the
    products whose first row falls in its share [r R / world, (r + 1) R / world) of the R rows (a product with no rows goes
    with the next one's start).  ``row_offsets`` is the G + 1 offset table (any sequence of ints).  The shard's launch passes
    d_rows + g_lo, d_aux + g_lo K N, M = g_hi - g_lo, n_units = (ro[g_hi] - ro[g_lo]) N and unit_base + (ro[g_lo] - ro[0]) N."""
    if world < 1 or not (0 <= rank < world):
        raise ValueError("bad rank/world")
    ro = [int(x) for x in row_offsets]
    G, R = len(ro) - 1, ro[-1] - ro[0]
    if G < 1:
        raise ValueError("row_offsets needs G + 1 >= 2 entries")

    def cut(r):                          # first product whose first row lies at or past rank r's share
        if r <= 0:
            return 0
        if r >= world:
            return G
        t = ro[0] + (r * R) // world
        lo, hi = 0, G
        while lo < hi:
            mid = (lo + hi) // 2
            if ro[mid] < t:
                lo = mid + 1
            else:
                hi = mid
        return lo
    return cut(rank), cut(rank + 1)


def stats_to_tensor(stats: dict, torch, device="cpu"):
    f = stats["first_fault_unit"]
    return torch.tensor([stats["errors_corrected"], stats["dwc_detected"], stats["syncs"], stats["injected"],
                         _I64_MAX if f == NO_FAULT_UNIT else f], dtype=torch.int64, device=device)


def tensor_to_stats(t) -> dict:
    v = [int(x) for x in t.tolist()]
    return dict(errors_corrected=v[0], dwc_detected=v[1], syncs=v[2], injected=v[3],
                first_fault_unit=NO_FAULT_UNIT if v[4] == _I64_MAX else v[4])


def allreduce_stats(t, dist, group=None):
    """In place: SUM over the four counters, MIN over first_fault_unit (works for nccl and gloo)."""
    dist.all_reduce(t[:4], op=dist.ReduceOp.SUM, group=group)
    dist.all_reduce(t[4:], op=dist.ReduceOp.MIN, group=group)
    return t


def device_counters_to_stats_tensor(raw):
    """raw: int64 view of the 5 u64 device counters (coast_stats_snapshot); maps ~0 -> INT64_MAX for MIN."""
    out = raw.clone()
    out[4] = _I64_MAX if int(raw[4]) == -1 else raw[4]
    return out


def negotiate_peer_counter_block(dist, rank: int, torch, device, export_fn, probe_fn, log=None):
    """Agree, across all ranks, on folding the counters through rank 0's counter block over NVLink peer memory
    (include/coast_rt.h: coast_counters_export / coast_counters_attach).

    rank 0 calls ``export_fn() -> 64 bytes``; the handle is broadcast; every other rank calls ``probe_fn(handle)`` (attach + detach
    once).  Returns the handle if EVERY rank succeeded, else None on every rank -- a failure anywhere (no CUDA IPC, no peer access)
    makes all ranks fall back together, and no rank is ever left waiting in a collective.  Works for nccl and gloo."""
    h = torch.zeros(64, dtype=torch.uint8, device=device)
    ok = torch.ones(1, dtype=torch.int32, device=device)
    if rank == 0:
        try:
            h.copy_(torch.frombuffer(bytearray(export_fn()), dtype=torch.uint8))
        except Exception as exc:
            if log:
                log(f"counter block cannot be exported: {exc}")
            ok.zero_()
    dist.broadcast(h, src=0)
    dist.broadcast(ok, src=0)
    handle = bytes(h.cpu().numpy().tobytes())
    if rank != 0 and int(ok[0]) == 1:
        try:
            probe_fn(handle)
        except Exception as exc:
            if log:
                log(f"peer counter block unavailable on rank {rank}: {exc}")
            ok.zero_()
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    return handle if int(ok[0]) == 1 else None
