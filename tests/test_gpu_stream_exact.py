"""The streaming kernels (SHA-256, AES-128, CRC16, quicksort, CHStone sha and aes) past their first wave and past 4 GiB.

The ring kernels run persistent CTAs, at most one resident wave: each CTA loops over tiles (`tile += gridDim.x`), its ring
flips parity, AES refills its 3-stage ring and drains its deferred-fault queue, CRC walks pairs of tiles.  The grid-stride
kernels are capped at four waves.  Every multi-wave case here reads the grid from the launch itself (F_VERBOSE) and sizes
n so that each CTA runs several iterations, then compares every output byte, all five counters and d_status with the
oracle (`both`).

Past 4 GiB the oracle is too slow, so plain references of the same operations run on the device in chunks: SHA-256
(FIPS 180-4), AES-128 (FIPS-197), CRC16 (bit-serial, the polynomial of crc16.c) and the Philox fault-plan decision.  They
are written in torch on int64 lanes masked to 32 bits, run the same on the CPU and on the GPU, and are pinned here on the
CPU against hashlib, the NIST AES records, the shipped CRC and the oracle."""
import hashlib
import os
import re

import numpy as np
import pytest

from test_gpu_parity import both, msgs

M32 = 0xFFFFFFFF
GiB = 1 << 30


# ------------------------------------------------------------------------------------------ Philox plan decisions
def _mulhilo(a, c):
    """(hi, lo) 32-bit halves of the 64-bit product of the constant a and the u32 lanes c (int64 tensor)."""
    p_lo = a * (c & 0xFFFF)                     # < 2^48
    p_hi = a * (c >> 16)                        # < 2^48
    t = p_lo + ((p_hi & 0xFFFF) << 16)          # < 2^49
    return ((t >> 32) + (p_hi >> 16)) & M32, t & M32


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on int64 tensors of u32 values (the counter words may be tensors or ints, the key ints)."""
    import torch
    like = c0
    c1, c2, c3 = (x if isinstance(x, torch.Tensor) else torch.full_like(like, x) for x in (c1, c2, c3))
    for _ in range(10):
        hi0, lo0 = _mulhilo(0xD2511F53, c0)
        hi1, lo1 = _mulhilo(0xCD9E8D57, c2)
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + 0x9E3779B9) & M32, (k1 + 0xBB67AE85) & M32
    return c0, c1, c2, c3


def plan_draw(seed, unit_base, n, device="cpu", start=0):
    """The four Philox words of units unit_base + start .. unit_base + start + n - 1 of a Bernoulli plan."""
    import torch
    g = unit_base + start + torch.arange(n, dtype=torch.int64, device=device)
    return philox4x32_10(g & M32, g >> 32, 0, 0, seed & M32, (seed >> 32) & M32)


def plan_decisions(seed, threshold, unit_base, n, nc, n_sites, site_bits=lambda s: 32, device="cpu", start=0):
    """Per unit: hit, replica, site, bit of a Bernoulli plan, as the oracle's orc_fault_for_unit decides them."""
    x0, x1, x2, x3 = plan_draw(seed, unit_base, n, device, start)
    site = x2 % n_sites
    return x0 < threshold, x1 % nc, site, x3 % site_bits(site)


def plan_hits(seed, threshold, unit_base, n, device="cpu", chunk=1 << 24):
    import torch
    return torch.cat([plan_draw(seed, unit_base, min(chunk, n - s), device, s)[0] < threshold for s in range(0, n, chunk)]) \
        if n else torch.zeros(0, dtype=torch.bool, device=device)


# ------------------------------------------------------------------------------------------ SHA-256 (FIPS 180-4)
def _icbrt(x):
    lo, hi = 0, 1 << (x.bit_length() // 3 + 2)
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if mid ** 3 <= x else (lo, mid - 1)
    return lo


def _primes(k):
    ps, c = [], 2
    while len(ps) < k:
        if all(c % p for p in ps):
            ps.append(c)
        c += 1
    return ps


# the first 32 bits of the fractional parts of the square roots of the first 8 primes and the cube roots of the first 64
SHA_H0 = [__import__("math").isqrt(p << 64) & M32 for p in _primes(8)]
SHA_K = [_icbrt(p << 96) & M32 for p in _primes(64)]


def _rotr(x, k):
    return ((x >> k) | (x << (32 - k))) & M32


def sha256_ref(m):
    """SHA-256 digests of n messages of the same length: m is a (n, L) uint8 tensor, the result (n, 32) uint8."""
    import torch
    n, L = m.shape
    nb = (L + 8) // 64 + 1
    tail = torch.zeros(nb * 64 - L, dtype=torch.uint8)                 # 0x80, zeros, the bit length big-endian
    tail[0] = 0x80
    tail[-8:] = torch.tensor(list((8 * L).to_bytes(8, "big")), dtype=torch.uint8)
    blocks = torch.cat([m, tail.to(m.device).expand(n, -1)], dim=1).view(n, nb * 16, 4).to(torch.int64)
    words = (blocks[..., 0] << 24) | (blocks[..., 1] << 16) | (blocks[..., 2] << 8) | blocks[..., 3]
    del blocks
    h = [torch.full((n,), v, dtype=torch.int64, device=m.device) for v in SHA_H0]
    for b in range(nb):
        w = [words[:, 16 * b + t] for t in range(16)]
        a, bb, c, d, e, f, g, hh = h
        for t in range(64):
            if t >= 16:
                w15, w2 = w[(t - 15) % 16], w[(t - 2) % 16]
                s0 = _rotr(w15, 7) ^ _rotr(w15, 18) ^ (w15 >> 3)
                s1 = _rotr(w2, 17) ^ _rotr(w2, 19) ^ (w2 >> 10)
                w[t % 16] = (w[t % 16] + s0 + w[(t - 7) % 16] + s1) & M32
            t1 = hh + (_rotr(e, 6) ^ _rotr(e, 11) ^ _rotr(e, 25)) + ((e & f) ^ (~e & g & M32)) + SHA_K[t] + w[t % 16]
            t2 = (_rotr(a, 2) ^ _rotr(a, 13) ^ _rotr(a, 22)) + ((a & bb) ^ (a & c) ^ (bb & c))
            a, bb, c, d, e, f, g, hh = (t1 + t2) & M32, a, bb, c, (d + t1) & M32, e, f, g
        h = [(x + y) & M32 for x, y in zip(h, (a, bb, c, d, e, f, g, hh))]
    st = torch.stack(h, dim=1)
    return torch.stack([(st >> s) & 0xFF for s in (24, 16, 8, 0)], dim=2).reshape(n, 32).to(torch.uint8)


# ------------------------------------------------------------------------------------------ AES-128 (FIPS-197)
def _gf_mul(a, b):
    r = 0
    while b:
        if b & 1:
            r ^= a
        a = ((a << 1) ^ (0x11B if a & 0x80 else 0)) & 0xFF
        b >>= 1
    return r


def _sbox():
    inv = [0] + [next(y for y in range(1, 256) if _gf_mul(x, y) == 1) for x in range(1, 256)]
    rotl = lambda b, k: ((b << k) | (b >> (8 - k))) & 0xFF
    return [b ^ rotl(b, 1) ^ rotl(b, 2) ^ rotl(b, 3) ^ rotl(b, 4) ^ 0x63 for b in inv]


AES_SBOX = _sbox()
AES_INV_SBOX = [AES_SBOX.index(v) for v in range(256)]
# state byte i is row i % 4 of column i // 4; ShiftRows moves row r left by r columns
AES_SHIFT = [(i % 4) + 4 * ((i // 4 + i % 4) % 4) for i in range(16)]
AES_INV_SHIFT = [(i % 4) + 4 * ((i // 4 - i % 4) % 4) for i in range(16)]


def _xt(x):
    return ((x << 1) ^ ((x >> 7) * 0x1B)) & 0xFF


def _mix(s, inverse):
    import torch
    a = s.view(-1, 4, 4)                                                 # [unit][column][row]
    if inverse:                                                          # {0e, 0b, 0d, 09} = 8a ^ {4a ^ 2a, 2a ^ a, 4a ^ a, a}
        x2 = _xt(a); x4 = _xt(x2); x8 = _xt(x4)
        m14, m11, m13, m9 = x8 ^ x4 ^ x2, x8 ^ x2 ^ a, x8 ^ x4 ^ a, x8 ^ a
        out = m14 ^ torch.roll(m11, -1, 2) ^ torch.roll(m13, -2, 2) ^ torch.roll(m9, -3, 2)
    else:                                                                # {02, 03, 01, 01}
        a1 = torch.roll(a, -1, 2)
        out = _xt(a) ^ _xt(a1) ^ a1 ^ torch.roll(a, -2, 2) ^ torch.roll(a, -3, 2)
    return out.reshape(-1, 16)


def aes128_round_keys(key):
    """(n, 16) or (16,) uint8 keys -> (n, 11, 16) int64 round keys (FIPS-197 KeyExpansion)."""
    import torch
    k = key.to(torch.int64).reshape(-1, 16)
    sbox = torch.tensor(AES_SBOX, dtype=torch.int64, device=k.device)
    w = [k[:, 4 * i: 4 * i + 4] for i in range(4)]
    rcon = 1
    for i in range(4, 44):
        t = w[i - 1]
        if i % 4 == 0:
            t = sbox[torch.roll(t, -1, 1)]
            t = torch.cat([t[:, :1] ^ rcon, t[:, 1:]], dim=1)
            rcon = _xt(rcon)
        w.append(w[i - 4] ^ t)
    return torch.stack([torch.cat(w[4 * r: 4 * r + 4], dim=1) for r in range(11)], dim=1)


def aes128_ref(blocks, key, decrypt=False):
    """AES-128 of (n, 16) uint8 blocks under one (16,) key or one key per block ((n, 16)); the result is (n, 16) uint8."""
    import torch
    dv = blocks.device
    rk = aes128_round_keys(key.to(dv))
    rk = rk.expand(blocks.shape[0], -1, -1) if rk.shape[0] == 1 else rk
    sbox = torch.tensor(AES_INV_SBOX if decrypt else AES_SBOX, dtype=torch.int64, device=dv)
    perm = torch.tensor(AES_INV_SHIFT if decrypt else AES_SHIFT, dtype=torch.int64, device=dv)
    s = blocks.to(torch.int64)
    if not decrypt:
        s = s ^ rk[:, 0]
        for r in range(1, 11):
            s = sbox[s[:, perm]]
            if r < 10:
                s = _mix(s, False)
            s = s ^ rk[:, r]
    else:
        s = s ^ rk[:, 10]
        for r in range(9, -1, -1):
            s = sbox[s[:, perm]] ^ rk[:, r]
            if r > 0:
                s = _mix(s, True)
    return s.to(torch.uint8)


# ------------------------------------------------------------------------------------------ CRC16 (crc16.c)
def crc16_ref(m):
    """crc16.c's CRC of n messages of the same length, bit by bit: polynomial 0x1021, initial value 0xFFFF, no
    reflection, no final xor.  m is a (n, L) uint8 tensor; the result is (n,) int64."""
    import torch
    crc = torch.full((m.shape[0],), 0xFFFF, dtype=torch.int64, device=m.device)
    for i in range(m.shape[1]):
        crc = crc ^ (m[:, i].to(torch.int64) << 8)
        for _ in range(8):
            crc = ((crc << 1) ^ ((crc >> 15) * 0x1021)) & 0xFFFF
    return crc


# ------------------------------------------------------------------------------------------ the references, pinned (CPU)
def test_sha256_ref_matches_hashlib_at_every_length_and_the_oracle(oracle):
    import torch
    for L in range(131):
        m = msgs(oracle, 5, L, L + 1).reshape(5, L)
        got = sha256_ref(torch.from_numpy(m)).numpy()
        for u in range(5):
            assert got[u].tobytes() == hashlib.sha256(m[u].tobytes()).digest(), L
            if u == 0:
                assert got[u].tobytes() == oracle.sha256(m[u].tobytes())
    assert SHA_K[0] == 0x428A2F98 and SHA_K[63] == 0xC67178F2 and SHA_H0[0] == 0x6A09E667 and SHA_H0[7] == 0x5BE0CD19


def test_aes128_ref_matches_the_nist_records_and_the_oracle(oracle, golden):
    import torch
    rec = np.frombuffer(bytes.fromhex(golden["aes"]["records"]), dtype=np.uint8).reshape(568, 80)
    keys, keys2, cipher, plain, inp = (torch.from_numpy(np.ascontiguousarray(rec[:, 16 * i: 16 * i + 16])) for i in range(5))
    assert torch.equal(aes128_ref(inp, keys), cipher)
    assert torch.equal(aes128_ref(cipher, keys2, decrypt=True), plain)
    vt = rec[14 + 42 + 256:]                                       # ECBVarTxt128: all-zero key, one key for every block
    assert torch.equal(aes128_ref(torch.from_numpy(np.ascontiguousarray(vt[:, 64:80])), torch.zeros(16, dtype=torch.uint8)),
                       torch.from_numpy(np.ascontiguousarray(vt[:, 32:48])))
    b = msgs(oracle, 64, 16, 3).reshape(64, 16)
    k = msgs(oracle, 64, 16, 4).reshape(64, 16)
    enc = aes128_ref(torch.from_numpy(b), torch.from_numpy(k)).numpy()
    dec = aes128_ref(torch.from_numpy(b), torch.from_numpy(k), decrypt=True).numpy()
    one = aes128_ref(torch.from_numpy(b), torch.from_numpy(k[7])).numpy()
    for u in range(64):
        assert enc[u].tobytes() == oracle.aes128(b[u].tobytes(), k[u].tobytes(), 0)[0]
        assert dec[u].tobytes() == oracle.aes128(b[u].tobytes(), k[u].tobytes(), 1)[0]
        assert one[u].tobytes() == oracle.aes128(b[u].tobytes(), k[7].tobytes(), 0)[0]


def test_crc16_ref_matches_the_shipped_message_and_the_golden_messages(oracle, golden):
    import torch
    m = torch.tensor(list(bytes.fromhex(golden["crc16"]["shipped_msg"])), dtype=torch.uint8)
    assert int(crc16_ref(m.view(1, -1))[0]) == 0x5BA3 == golden["crc16"]["shipped_crc"]
    for mh, c in golden["crc16"]["random"]:
        assert int(crc16_ref(torch.tensor(list(bytes.fromhex(mh)), dtype=torch.uint8).view(1, -1))[0]) == c
    for L in (1, 13, 64, 255):
        mm = msgs(oracle, 9, L, L).reshape(9, L)
        got = crc16_ref(torch.from_numpy(mm)).tolist()
        assert got == [oracle.crc16(mm[u].tobytes()) for u in range(9)]


@pytest.mark.parametrize("kernel,nc,unit_bytes,base", [
    ("K_SHA256", 3, 64, 0), ("K_SHA256", 2, 100, (1 << 32) - 700), ("K_CRC16", 3, 64, (1 << 32) - 5),
    ("K_CRC16", 1, 13, 3 << 32), ("K_AES128", 2, 16, (1 << 32) - 1000), ("K_AES128", 3, 16, (1 << 40) + 17)])
def test_plan_decisions_match_the_oracle_across_2_to_the_32(oracle, kernel, nc, unit_bytes, base):
    k = getattr(oracle, kernel)
    n, seed, thr = 2000, 0x1234_5678_9ABC, int(0.3 * 2 ** 32)
    ns = oracle.fault_sites(k, unit_bytes)
    hit, rep, site, bit = plan_decisions(seed, thr, base, n, nc, ns, lambda s: _site_bits(oracle, k, unit_bytes, s))
    plan = oracle.make_plan(oracle.PLAN_BERNOULLI, seed=seed, threshold=thr)
    for u in range(n):
        want = oracle.fault_for_unit(plan, k, nc, unit_bytes, 0, base + u, u)
        got = (int(rep[u]), int(site[u]), int(bit[u])) if hit[u] else None
        assert got == want, (u, got, want)
    assert 400 < int(hit.sum()) < 800
    assert (plan_hits(seed, thr, base, n, chunk=300) == hit).all()


def _site_bits(oracle, kernel, unit_bytes, site):
    """bit width of the value at each fault site (orc_fault_site_bits)"""
    if kernel == oracle.K_CRC16:
        return 8 + 8 * (site < unit_bytes)
    return 8 if kernel in (oracle.K_AES128, oracle.K_CHSTONE_AES) else 32


# ------------------------------------------------------------------------------------------ multi-wave sizing
def _geom():
    """the plain #define values of coast_b200/csrc/xmr_geom.h (CTA sizes, warps, tile rows)"""
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "coast_b200", "csrc", "xmr_geom.h")
    with open(path) as f:
        src = f.read()
    return {k: int(v.rstrip("u"), 0) for k, v in re.findall(r"#define[ \t]+(XMR_\w+)[ \t]+((?:0x)?[0-9a-fA-F]+u?)[ \t]*$", src, re.M)}


def _upw(nc):
    return 32 // nc


def launch_grid(rt, capfd, kernel, nc, n, in_bytes, aux=False, **kw):
    """(kernel name, grid) of a launch over n zero units of in_bytes each, read from its F_VERBOSE line"""
    import torch
    import coast_b200 as cb
    buf = torch.zeros(max(n * in_bytes, 16), dtype=torch.uint8, device="cuda")
    kw["flags"] = kw.get("flags", 0) | cb.F_VERBOSE
    capfd.readouterr()
    out, _ = rt.run(kernel, nc, buf, n, aux=buf if aux else None, **kw)
    err = capfd.readouterr().err
    del buf, out
    torch.cuda.empty_cache()
    m = re.search(r"coast_rt: (\S+) grid=(\d+) block=\d+ smem=\d+ units=%d\b" % n, err)
    assert m, err
    return m.group(1), int(m.group(2))


def multi_wave_n(rt, capfd, kernel, nc, rows, reps, rem, in_bytes, **kw):
    """Size n from the launch.  `rows` is what one CTA takes per iteration of its loop.  A probe launch far past the grid
    cap gives the grid; n = reps x grid x rows + rem.  The launch at n must use the same grid, so each of its CTAs runs
    at least `reps` iterations, whatever CTA size or occupancy a later change brings.  Returns (n, grid, kernel name)."""
    probe = 64 * rt.sm_count() * rows
    _, grid = launch_grid(rt, capfd, kernel, nc, probe, in_bytes, **kw)
    assert grid * rows < probe, (grid, rows, probe)                   # the probe's grid was capped, not sized by the work
    n = reps * grid * rows + rem
    name, grid_n = launch_grid(rt, capfd, kernel, nc, n, in_bytes, **kw)
    assert grid_n == grid and n >= reps * grid_n * rows, (n, grid, grid_n, rows)
    print(f"{name}: grid={grid} rows/iteration={rows} n={n} iterations/CTA={-(-n // (grid * rows))}")
    return n, grid, name


def run_multi_wave(rt, oracle, kernel, nc, inp, n, seed, p=0.05, unit_base=(1 << 32) - 12345, **kw):
    """no plan and a Bernoulli plan, both with d_status, at a unit_base whose global units cross 2^32 inside the launch"""
    _, st0 = both(rt, oracle, kernel, nc, inp, n, unit_base=unit_base, status=True, **kw)
    assert st0["injected"] == 0 and st0["errors_corrected"] == st0["dwc_detected"] == 0
    _, st1 = both(rt, oracle, kernel, nc, inp, n, unit_base=unit_base, status=True, plan_kw=dict(seed=seed, p=p), **kw)
    assert st1["injected"] > 0
    return st1


# ------------------------------------------------------------------------------------------ SHA-256 multi-wave
SHA_CASES = [  # (id, nc, flags, unit_bytes, rows per CTA iteration, reps)
    ("seg_nc3", 3, 3, 64, 128, 6),
    ("seg_nc3_majority", 3, 3 | 0x100, 64, 128, 6),
    ("interleaved_nc3", 3, 3 | 0x8, 64, 8 * 10, 6),
    ("ring_nc1", 1, 3, 64, 8 * 32, 6),
    ("ring_nc2", 2, 3, 64, 8 * 16, 6),
    ("general_nc3", 3, 3, 100, 8 * 10, 3),
    ("general_nc2", 2, 3, 100, 8 * 16, 3),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", SHA_CASES, ids=[c[0] for c in SHA_CASES])
def test_sha256_multi_wave_every_digest_and_counter(rt, oracle, capfd, case):
    import coast_b200 as cb
    cid, nc, flags, ub, rows, reps = case
    g = _geom()
    assert rows == (g["XMR_SHA_SEG_TILE_ROWS"] if cid.startswith("seg") else g["XMR_WARPS"] * _upw(nc))
    n, grid, name = multi_wave_n(rt, capfd, cb.K_SHA256, nc, rows, reps, 37, ub, unit_bytes=ub, flags=flags)
    assert ("seg" in name) == cid.startswith("seg") and ("gen" in name) == (ub != 64), name
    m = msgs(oracle, n, ub, 5)
    st = run_multi_wave(rt, oracle, cb.K_SHA256, nc, m, n, seed=nc + ub, unit_bytes=ub, flags=flags)
    if nc == 3:
        assert st["syncs"] == 32 * n and st["errors_corrected"] >= st["injected"]


# ------------------------------------------------------------------------------------------ CRC16 multi-wave
@pytest.mark.gpu
@pytest.mark.parametrize("nc", [1, 2, 3])
def test_crc16_table_kernel_multi_wave(rt, oracle, capfd, nc):
    """the table kernel takes PAIRS of tiles per iteration: rows = 2 x tile rows"""
    import coast_b200 as cb
    tile = (768 if nc == 1 else 1024) // 32 * _upw(nc)
    assert tile == {1: 768, 2: 512, 3: 320}[nc]
    n, grid, name = multi_wave_n(rt, capfd, cb.K_CRC16, nc, 2 * tile, 6, tile + 11, 64, unit_bytes=64)
    assert name.startswith("xmr_crc16_b64"), name
    m = msgs(oracle, n, 64, 7)
    st = run_multi_wave(rt, oracle, cb.K_CRC16, nc, m, n, seed=40 + nc, unit_bytes=64, flags=3)
    if nc == 3:
        assert st["errors_corrected"] == st["injected"]


@pytest.mark.gpu
@pytest.mark.parametrize("nc", [2, 3])
def test_crc16_general_path_multi_wave(rt, oracle, capfd, nc):
    import coast_b200 as cb
    n, grid, name = multi_wave_n(rt, capfd, cb.K_CRC16, nc, 8 * _upw(nc), 3, 5, 13, unit_bytes=13)
    assert name.startswith("xmr_crc16_gen"), name
    run_multi_wave(rt, oracle, cb.K_CRC16, nc, msgs(oracle, n, 13, 8), n, seed=50 + nc, unit_bytes=13, flags=3)


# ------------------------------------------------------------------------------------------ AES multi-wave
AES_MODES = {"enc": 0, "dec": 1, "enck": 2, "deck": 3}


@pytest.mark.gpu
@pytest.mark.parametrize("residue", [0, 4, 3])               # n % 16: row pack shift 4, 2, 0
@pytest.mark.parametrize("nc", [1, 2, 3])
@pytest.mark.parametrize("mode", list(AES_MODES))
def test_aes_multi_wave_every_block_and_counter(rt, oracle, capfd, mode, nc, residue):
    import coast_b200 as cb
    tile = 16 * _upw(nc) * (2 if nc == 1 else 4)
    assert tile == {1: 1024, 2: 1024, 3: 640}[nc]
    md = AES_MODES[mode]
    n, grid, name = multi_wave_n(rt, capfd, cb.K_AES128, nc, tile, 6, 16 * 37 + residue, 16, aux=md & 2 != 0, mode=md,
                                 key=bytes(16))
    assert name.startswith(f"xmr_aes128_{mode}_nc{nc}"), name
    blocks = msgs(oracle, n, 16, 11 + residue)
    keys = msgs(oracle, n, 16, 12) if md & 2 else None
    run_multi_wave(rt, oracle, cb.K_AES128, nc, blocks, n, seed=60 + nc + residue, p=0.02, mode=md, flags=3,
                   key=bytes(range(3, 19)), aux=keys)


# ------------------------------------------------------------------------------------------ the AES deferred-fault queue
AES_QCAP = 96


def simulate_aes_queue(hit_mid, n, grid, nc):
    """Each warp's count of queued units (one-key kernels): tiles go to CTAs as tile % grid, row (warp*J + j)*UPW + u of a
    tile to warp `warp`; after each tile the warp drains in the loop when q_count > AES_QCAP - J*UPW.  Returns
    (in-loop drains, the largest q_count any warp reached)."""
    J, upw = (2 if nc == 1 else 4), _upw(nc)
    trows = 16 * J * upw
    n_tiles = (n + trows - 1) // trows
    mid = np.zeros(n_tiles * trows, dtype=np.int64)
    mid[:n] = hit_mid
    per_warp = mid.reshape(n_tiles, 16, J * upw).sum(axis=2)            # [tile][warp]: row (warp*J + j)*UPW + u
    iters = (n_tiles + grid - 1) // grid
    per_warp = np.concatenate([per_warp, np.zeros((iters * grid - n_tiles, 16), dtype=np.int64)])
    per_warp = per_warp.reshape(iters, grid, 16)                         # tile = it * grid + cta
    q = np.zeros((grid, 16), dtype=np.int64)
    drains, qmax = 0, 0
    for it in range(iters):
        q += per_warp[it]
        qmax = max(qmax, int(q.max()))
        fire = q > AES_QCAP - J * upw
        drains += int(fire.sum())
        q[fire] = 0
    return drains, qmax


def fill_queue_table(n, grid, nc):
    """A TABLE plan that brings every warp's queue to exactly AES_QCAP entries: mid-round flips (site >= 16) on the first
    c rows of each warp in each tile, with c cycling so that q_count sits exactly at the drain threshold
    AES_QCAP - J*UPW after one tile and a full tile follows."""
    J, upw = (2 if nc == 1 else 4), _upw(nc)
    ju = J * upw
    thr = AES_QCAP - ju
    k = -(-thr // ju)
    counts = np.array([thr - ju * (k - 1)] + [ju] * k)
    loc = np.arange(n, dtype=np.int64)
    tile, idx = loc // (16 * ju), loc % ju                              # row (warp*J + j)*UPW + u: idx = j*UPW + u
    on = idx < counts[(tile // grid) % len(counts)]
    e = 0x80000000 | ((loc % nc) << 29) | ((16 + loc % 160) << 5) | (loc % 8)
    return np.where(on, e, 0).astype(np.uint32), on


@pytest.mark.gpu
@pytest.mark.parametrize("plan", ["p0.25", "all", "fill"])
@pytest.mark.parametrize("nc", [1, 2, 3])
@pytest.mark.parametrize("dec", [0, 1])
def test_aes_deferred_queue_drains_inside_the_tile_loop(rt, oracle, capfd, dec, nc, plan):
    """The one-key kernels defer units with a mid-round flip to a queue of AES_QCAP entries per warp and drain it inside
    the tile loop when the next tile might not fit.  The drains are simulated from the plan, the tile -> CTA map and the
    row -> warp map; the run must then equal the oracle on every block and counter."""
    import coast_b200 as cb
    tile = 16 * _upw(nc) * (2 if nc == 1 else 4)
    n, grid, name = multi_wave_n(rt, capfd, cb.K_AES128, nc, tile, 6, 0, 16, mode=dec, key=bytes(16))
    kw = {}
    if plan == "fill":
        kw["table"], mid = fill_queue_table(n, grid, nc)
        hits = int(mid.sum())
    else:
        kw["plan_kw"] = dict(seed=70 + nc, p=0.25) if plan == "p0.25" else dict(seed=80 + nc, threshold=0xFFFFFFFF)
        thr = kw["plan_kw"].get("threshold", int(0.25 * 2 ** 32))
        hit, _, site, _ = plan_decisions(kw["plan_kw"]["seed"], thr, 999, n, nc, 176)
        mid, hits = (hit & (site >= 16)).numpy(), int(hit.sum())
    drains, qmax = simulate_aes_queue(mid, n, grid, nc)
    print(f"{name} {plan}: grid={grid} n={n} in-loop drains={drains} largest q_count={qmax}")
    assert drains >= grid and AES_QCAP - (2 if nc == 1 else 4) * _upw(nc) < qmax <= AES_QCAP
    if plan == "fill":
        assert qmax == AES_QCAP
    blocks = msgs(oracle, n, 16, 13)
    _, st = both(rt, oracle, cb.K_AES128, nc, blocks, n, key=bytes(range(16)), mode=dec, flags=3, unit_base=999,
                 status=True, **kw)
    assert st["injected"] == hits
    if nc == 2:
        assert st["dwc_detected"] == st["injected"]                    # every state flip reaches the output


# ------------------------------------------------------------------------------------------ quicksort, CHStone
@pytest.mark.gpu
@pytest.mark.parametrize("path", ["fsm", "nested"])
@pytest.mark.parametrize("nc", [2, 3])
def test_quicksort_multi_wave(rt, oracle, capfd, monkeypatch, path, nc):
    import coast_b200 as cb
    if path == "nested":
        monkeypatch.setenv("COAST_QSORT_PATH", "nested")
    else:
        monkeypatch.delenv("COAST_QSORT_PATH", raising=False)
    L = 48
    n, grid, name = multi_wave_n(rt, capfd, cb.K_QSORT, nc, _geom()["XMR_QSORT_THREADS"] // 32 * _upw(nc), 3, 3, 4 * L, unit_bytes=4 * L)
    assert name.startswith("xmr_qsortn" if path == "nested" else "xmr_qsort_"), name
    a = oracle.fill_philox(n * L, 0, 90 + nc).view(np.int32)
    g, _ = both(rt, oracle, cb.K_QSORT, nc, a, n, unit_bytes=4 * L, flags=3, unit_base=(1 << 32) - 77, status=True)
    assert (g.view(np.int32).reshape(n, L) == np.sort(a.reshape(n, L), axis=1)).all()
    both(rt, oracle, cb.K_QSORT, nc, a, n, unit_bytes=4 * L, flags=3, unit_base=(1 << 32) - 77, status=True,
         plan_kw=dict(seed=nc, p=0.05))


@pytest.mark.gpu
@pytest.mark.parametrize("nc", [1, 3])
def test_chstone_sha_multi_wave(rt, oracle, capfd, nc):
    import coast_b200 as cb
    n, grid, name = multi_wave_n(rt, capfd, cb.K_CHSTONE_SHA, nc, _geom()["XMR_WARPS"] * _upw(nc), 3, 9, 128, unit_bytes=128)
    run_multi_wave(rt, oracle, cb.K_CHSTONE_SHA, nc, msgs(oracle, n, 128, 14), n, seed=nc, unit_bytes=128, flags=3)


@pytest.mark.gpu
@pytest.mark.parametrize("dec", [0, 1])
@pytest.mark.parametrize("nc", [2, 3])
def test_chstone_aes_multi_wave(rt, oracle, capfd, nc, dec):
    """CHStone aes: one byte per int, 64-byte units; per-unit keys"""
    import torch
    import coast_b200 as cb
    rows = _geom()["XMR_AES_WARPS"] * _upw(nc)
    n, grid, name = multi_wave_n(rt, capfd, cb.K_CHSTONE_AES, nc, rows, 3, 7, 64, aux=True, mode=dec | 2)
    assert name.startswith(f"xmr_chaes_{'dec' if dec else 'enc'}_nc{nc}"), name
    blocks = (msgs(oracle, n, 64, 15).view(np.uint32) & 0xFF).view(np.uint8)          # one byte per int
    keys = (msgs(oracle, n, 64, 16).view(np.uint32) & 0xFF).view(np.uint8)
    run_multi_wave(rt, oracle, cb.K_CHSTONE_AES, nc, blocks, n, seed=nc + 4 * dec, mode=dec | 2, aux=keys, flags=3)


# ------------------------------------------------------------------------------------------ past 4 GiB, on the device
def _room(nbytes):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"needs {nbytes} bytes of free device memory, {free} free")


def _free(*_):
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _chunks(n, c):
    return ((s, min(c, n - s)) for s in range(0, n, c))


@pytest.mark.gpu
def test_sha256_segmented_tmr_2p29_past_4gib(rt):
    """bench.py's sha256_2p29: 2^29 x 64-byte messages, 32 GiB in, 16 GiB out, TMR, a Bernoulli plan whose global units
    cross 2^32 inside the launch, and d_status.  Every digest equals the reference, and every flip reaches the digest
    (the rounds and the feed-forward are bijections in the state), so d_status is nonzero exactly on the hit units."""
    import torch
    import coast_b200 as cb
    n = 1 << 29
    base = (1 << 32) - (1 << 28)
    thr = 1 << 22                                                      # p = 2^-10
    _room(n * (64 + 32 + 1) + 6 * GiB)
    d_in = torch.empty(n * 64, dtype=torch.uint8, device="cuda")
    rt.fill_philox(d_in, seed=29)
    out = torch.full((n * 32,), 0xA5, dtype=torch.uint8, device="cuda")
    status = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    _, st = rt.run(cb.K_SHA256, 3, d_in, n, unit_bytes=64, flags=3, out=out, status=status, unit_base=base,
                   plan=cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=0x2929, threshold=thr))
    hits, first, s_sum = 0, None, 0
    for s, c in _chunks(n, 1 << 22):
        hit = plan_draw(0x2929, base, c, "cuda", s)[0] < thr
        ref = sha256_ref(d_in[64 * s: 64 * (s + c)].view(c, 64))
        bad = (out[32 * s: 32 * (s + c)].view(c, 32) != ref).any(dim=1)
        assert not bad.any(), f"{int(bad.sum())} wrong digests in units {s}..{s + c}, first at {s + int(bad.nonzero()[0])}"
        stc = status[s: s + c]
        assert torch.equal(stc != 0, hit), f"status != hit set in units {s}..{s + c}"
        hits += int(hit.sum())
        s_sum += int(stc.to(torch.int64).sum())
        if first is None and hit.any():
            first = base + s + int(hit.nonzero()[0])
    assert st.injected == hits and abs(hits - n / 1024) < 6 * (n / 1024) ** 0.5
    assert st.errors_corrected == s_sum and st.dwc_detected == 0
    assert st.first_fault_unit == first and first < 1 << 32
    assert st.syncs == 32 * n
    del d_in, out, status
    _free()


@pytest.mark.gpu
def test_sha256_general_path_past_4gib(rt):
    import torch
    import coast_b200 as cb
    n, L = (1 << 26) + 5, 100
    _room(n * (L + 32) + 4 * GiB)
    d_in = torch.empty((n * L + 3) // 4 * 4, dtype=torch.uint8, device="cuda")
    rt.fill_philox(d_in, seed=26)
    out = torch.full((n * 32,), 0xA5, dtype=torch.uint8, device="cuda")
    _, st = rt.run(cb.K_SHA256, 3, d_in, n, unit_bytes=L, flags=3, out=out)
    for s, c in _chunks(n, 1 << 22):
        ref = sha256_ref(d_in[L * s: L * (s + c)].view(c, L))
        assert torch.equal(out[32 * s: 32 * (s + c)].view(c, 32), ref), f"units {s}..{s + c}"
    assert st.as_dict() == dict(errors_corrected=0, dwc_detected=0, syncs=32 * n, injected=0, first_fault_unit=cb.NO_FAULT_UNIT)
    del d_in, out
    _free()


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["table", "general"])
def test_crc16_past_4gib(rt, path):
    """the table kernel on 64-byte units and the general path on 13-byte units, TMR with a Bernoulli plan: every CRC
    equals the reference, and every flip shows (one u16 vote per unit; CRC steps are invertible)"""
    import torch
    import coast_b200 as cb
    n, L = ((1 << 26) + (1 << 20) + 7, 64) if path == "table" else ((1 << 28) + (1 << 26), 13)
    base, thr = (1 << 32) - n // 2, 1 << 20
    _room(n * (L + 3) + 4 * GiB)
    d_in = torch.empty((n * L + 3) // 4 * 4, dtype=torch.uint8, device="cuda")
    rt.fill_philox(d_in, seed=L)
    out = torch.full((n * 2,), 0xA5, dtype=torch.uint8, device="cuda")
    status = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    _, st = rt.run(cb.K_CRC16, 3, d_in, n, unit_bytes=L, flags=3, out=out, status=status, unit_base=base,
                   plan=cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=16, threshold=thr))
    o16 = out.view(torch.int16)
    hits = 0
    for s, c in _chunks(n, 1 << 24):
        ref = crc16_ref(d_in[L * s: L * (s + c)].view(c, L))
        assert torch.equal(o16[s: s + c].to(torch.int64) & 0xFFFF, ref), f"units {s}..{s + c}"
        hit = plan_draw(16, base, c, "cuda", s)[0] < thr
        assert torch.equal(status[s: s + c] != 0, hit) and int(status[s: s + c].max()) <= 1
        hits += int(hit.sum())
    assert st.injected == st.errors_corrected == hits > 0 and st.syncs == n and st.dwc_detected == 0
    del d_in, out, status, o16
    _free()


@pytest.mark.gpu
@pytest.mark.parametrize("perkey", [False, True])
def test_aes_past_4gib(rt, capfd, perkey):
    """enc (one key) and enck (a key per block, its own d_aux addressing), DWC, n % 16 == 8 (row pack 2).  With a plan:
    every flip is detected, and the output is replica 0's, so it equals the reference except where replica 0 was hit."""
    import torch
    import coast_b200 as cb
    n = (1 << 28) + (1 << 20) + 8
    base, thr = (1 << 32) - n // 3, 1 << 20
    _room(n * (16 * (3 if perkey else 2) + 1) + 4 * GiB)
    d_in = torch.empty(n * 16, dtype=torch.uint8, device="cuda")
    rt.fill_philox(d_in, seed=128)
    keys = None
    if perkey:
        keys = torch.empty(n * 16, dtype=torch.uint8, device="cuda")
        rt.fill_philox(keys, seed=129)
    key = bytes(range(100, 116))
    out = torch.full((n * 16,), 0xA5, dtype=torch.uint8, device="cuda")
    status = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
    capfd.readouterr()
    _, st = rt.run(cb.K_AES128, 2, d_in, n, key=key, aux=keys, mode=cb.AES_KEY_PER_UNIT if perkey else 0, out=out,
                   status=status, unit_base=base, flags=cb.F_VERBOSE, plan=cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=5, threshold=thr))
    assert f"xmr_aes128_{'enck' if perkey else 'enc'}_nc2_inj1 " in capfd.readouterr().err
    hits = 0
    kt = torch.tensor(list(key), dtype=torch.uint8, device="cuda")
    for s, c in _chunks(n, 1 << 20):
        ref = aes128_ref(d_in[16 * s: 16 * (s + c)].view(c, 16), keys[16 * s: 16 * (s + c)].view(c, 16) if perkey else kt)
        hit, rep, _, _ = plan_decisions(5, thr, base, c, 2, 176, device="cuda", start=s)
        wrong = (out[16 * s: 16 * (s + c)].view(c, 16) != ref).any(dim=1)
        assert torch.equal(wrong, hit & (rep == 0)), f"units {s}..{s + c}"
        assert torch.equal(status[s: s + c] != 0, hit)
        hits += int(hit.sum())
    assert st.injected == st.dwc_detected == hits > 0 and st.errors_corrected == 0
    del d_in, keys, out, status
    _free()
