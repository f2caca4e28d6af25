"""CPU model of the grouped-matmul tile schedule (coast_b200/csrc/xmr_mm_grp.cuh): the one-CTA scan that writes tile_start[g],
the exclusive scan of ceil(M_g / TM), the binary search that maps a tile id to its product, tile_coords inside the product, the
persistent CTAs of the wgmma kernels (tile blockIdx.x, + grid, ...) and the grid bound the host launches, (R / TM + G) * column
tiles.  For random row tables -- empty products, one-row products, one product holding most rows -- and SM counts 1..132 it
checks that every C element of every product is computed exactly once, that no tile mixes two products, that rows past a
product are never stored, and that a malformed table (clamped offsets) stores only inside [ro[0], ro[0] + R) rows."""
import random

import pytest

SCAN_THREADS = 1024


def clamped(ro, g, R):
    o = ro[g]
    return 0 if o <= ro[0] else min(o - ro[0], R)


def rows_of(ro, g, R):
    s = clamped(ro, g, R)
    return s, max(s, clamped(ro, g + 1, R))


def scan(ro, G, R, TM, tiles_n):
    """xmr_mm_group_scan: each of 1024 threads sums its contiguous slice of products, a two-level exclusive scan, saturating"""
    cap = 0x7FFFFFFF // tiles_n
    per = -(-G // SCAN_THREADS)
    mine = []
    for t in range(SCAN_THREADS):
        g0, g1 = min(G, t * per), min(G, t * per + per)
        mine.append(min(sum(-(-(rows_of(ro, g, R)[1] - rows_of(ro, g, R)[0]) // TM) for g in range(g0, g1)), cap))
    ts, run = [0] * (G + 1), 0
    for t in range(SCAN_THREADS):
        g0, g1 = min(G, t * per), min(G, t * per + per)
        for g in range(g0, g1):
            ts[g] = min(run, cap)
            s, e = rows_of(ro, g, R)
            run += -(-(e - s) // TM)
    ts[G] = min(run, cap)
    return ts


def search(G, x, v):
    lo, hi = 0, G
    while hi - lo > 1:
        mid = (lo + hi) >> 1
        if v(mid) <= x:
            lo = mid
        else:
            hi = mid
    return lo


def tile_of(ro, R, ts, G, tiles_n, group_m, t):
    g = search(G, t // tiles_n, lambda x: ts[x])
    start, end = rows_of(ro, g, R)
    t0, tiles_m = ts[g], ts[g + 1] - ts[g]
    lt = t - t0 * tiles_n
    if tiles_m == 0 or lt >= tiles_m * tiles_n:
        return g, start, start, 0, 0
    per_group = group_m * tiles_n
    q, w = divmod(lt, per_group)
    rows = min(group_m, tiles_m - q * group_m)
    return g, start, end, q * group_m + w % rows, w // rows


def run_schedule(ro, N, TM, BN, group_m, sms):
    """every (product, row, column) the persistent kernel stores, with the tile that stored it"""
    G, R = len(ro) - 1, ro[-1] - ro[0]
    tiles_n = N // BN
    ts = scan(ro, G, R, TM, tiles_n)
    n_tiles = ts[G] * tiles_n
    grid = min(sms, (R // TM + G) * tiles_n)
    assert n_tiles <= (R // TM + G) * tiles_n                     # the host's bound holds every tile
    stores = {}
    for cta in range(grid):
        for t in range(cta, n_tiles, grid):
            g, start, end, tm, tn = tile_of(ro, R, ts, G, tiles_n, group_m, t)
            for r in range(start + tm * TM, start + tm * TM + TM):
                if r >= end:                                      # masked: the next product's row, or past R
                    continue
                for c in range(tn * BN, tn * BN + BN, BN // 4):  # a few columns per tile stand for all of them
                    stores.setdefault((r, c), []).append((g, t))
    return stores, ts


def tables(seed):
    rnd = random.Random(seed)
    out = [[0, 1], [0, 0, 5, 5], [7, 7, 7, 300], [0] + [1] * 40]
    for _ in range(12):
        G = rnd.choice([1, 2, 5, 17, 64, 200])
        w = [0 if rnd.random() < 0.3 else (1 if rnd.random() < 0.2 else rnd.randint(1, 400)) for _ in range(G)]
        if rnd.random() < 0.5:
            w[rnd.randrange(G)] = rnd.randint(1000, 3000)      # one huge product
        ro = [rnd.randint(0, 50)]
        for x in w:
            ro.append(ro[-1] + x)
        if ro[-1] > ro[0]:
            out.append(ro)
    return [ro for ro in out if ro[-1] > ro[0]]


@pytest.mark.parametrize("TM,BN,N,group_m", [(128, 128, 256, 16), (128, 32, 64, 16), (64, 128, 128, 1), (128, 128, 384, 3)])
@pytest.mark.parametrize("sms", [1, 7, 132])
def test_every_element_exactly_once_and_no_tile_mixes_products(TM, BN, N, group_m, sms):
    for ro in tables(TM + BN + sms):
        stores, ts = run_schedule(ro, N, TM, BN, group_m, sms)
        R = ro[-1] - ro[0]
        want = {(r, c) for r in range(R) for c in range(0, N, BN // 4)}
        assert set(stores) == want, ro                             # every element of every product ...
        assert all(len(v) == 1 for v in stores.values()), ro      # ... exactly once
        for (r, _), [(g, t)] in stores.items():
            assert ro[g] - ro[0] <= r < ro[g + 1] - ro[0]         # stored by its own product's tile
        by_tile = {}
        for (r, _), [(g, t)] in stores.items():
            by_tile.setdefault(t, set()).add(g)
        assert all(len(gs) == 1 for gs in by_tile.values())        # no tile mixes products
        assert ts == sorted(ts)                                    # a valid table scans to a non-decreasing tile_start


def test_empty_products_take_no_tiles():
    ro = [0, 0, 0, 130, 130, 131, 131]
    ts = scan(ro, 6, 131, 128, 1)
    assert ts == [0, 0, 0, 2, 2, 3, 3]


def test_scan_over_many_products_uses_every_thread_slice():
    ro = list(range(0, 3 * 5000 + 1, 3))                          # 5000 products of 3 rows: 5 per scan thread
    ts = scan(ro, 5000, 15000, 64, 2)
    assert ts == list(range(5001))


@pytest.mark.parametrize("ro", [[10, 50, 30, 90, 5000], [10, 5, 60, 200], [10, 10, 10]])
def test_a_malformed_table_stores_only_inside_the_rows(ro):
    """decreasing pairs and offsets past R: clamped, stores stay in [0, R) rows of the launch"""
    R = 120
    G = len(ro) - 1
    ts = scan(ro, G, R, 128, 1)
    for t in range(ts[G]):
        g, start, end, tm, tn = tile_of(ro, R, ts, G, 1, 16, t)
        assert 0 <= start <= end <= R
        assert all(r < R for r in range(start + tm * 128, min(end, start + tm * 128 + 128)))
