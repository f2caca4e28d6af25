"""GPU (H100): seeded differential fuzzing of the whole C ABI against the oracle -- random kernel, clone count, size,
flag combination, fault-plan kind (none / Bernoulli / explicit table with deliberately invalid entries), unit_base.
Every case must agree bit for bit in output AND counters."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _case(rng, oracle):
    k = int(rng.integers(0, 5))
    nc = int(rng.integers(1, 4))
    flags = int(rng.choice([0, 1, 3, 3 | 0x100, 3 | 0x8, 3 | 0x10, 0x20 & 0]))
    kw = {}
    if k == 0:      # crc16
        L = int(rng.choice([1, 2, 13, 63, 64, 65, 255]))
        n = int(rng.integers(1, 700))
        kernel, inp, kw = oracle.K_CRC16, rng.integers(0, 256, n * L, dtype=np.uint8), dict(unit_bytes=L)
    elif k == 1:    # sha256
        L = int(rng.choice([0, 1, 55, 56, 64, 64, 64, 100, 128, 300]))
        n = int(rng.integers(1, 900))
        kernel, inp, kw = oracle.K_SHA256, rng.integers(0, 256, max(n * L, 4), dtype=np.uint8), dict(unit_bytes=L)
    elif k == 2:    # aes
        n = int(rng.integers(1, 3000))
        mode = int(rng.choice([0, 0, 1, 2, 3]))
        kernel, inp = oracle.K_AES128, rng.integers(0, 256, n * 16, dtype=np.uint8)
        kw = dict(mode=mode, key=bytes(rng.integers(0, 256, 16, dtype=np.uint8)))
        if mode & 2:
            kw["aux"] = rng.integers(0, 256, n * 16, dtype=np.uint8)
    elif k == 3:    # exact matmul: every path (naive / tiled / tensor-core limbs)
        M, N, K = [(9, 9, 9), (33, 17, 40), (64, 128, 48), (128, 64, 128), (128, 128, 256), (256, 192, 128)][int(rng.integers(0, 6))]
        n = M * N
        kernel, inp = oracle.K_MM_U32, rng.integers(0, 2 ** 32, M * K, dtype=np.uint64).astype(np.uint32)
        kw = dict(M=M, N=N, K=K, aux=rng.integers(0, 2 ** 32, K * N, dtype=np.uint64).astype(np.uint32))
    else:           # quicksort
        L = int(rng.choice([1, 2, 3, 16, 100, 580]))
        n = int(rng.integers(1, 120))
        vals = rng.integers(-2 ** 31, 2 ** 31, n * L, dtype=np.int64).astype(np.int32)
        if rng.random() < 0.3:
            vals = (vals & 3).astype(np.int32)              # heavy duplicates
        kernel, inp, kw = oracle.K_QSORT, vals, dict(unit_bytes=4 * L)
    plan_kind = int(rng.integers(0, 3))
    plan_kw, table = None, None
    if plan_kind == 1:
        plan_kw = dict(seed=int(rng.integers(0, 2 ** 40)), threshold=int(rng.integers(1, 2 ** 32)))
    elif plan_kind == 2:
        ns = oracle.fault_sites(kernel, kw.get("unit_bytes", 0), kw.get("K", 0))
        table = np.zeros(n, dtype=np.uint32)
        for u in rng.choice(n, size=min(n, 1 + n // 3), replace=False):
            site = int(rng.integers(0, ns + 3)) if ns else 0          # sometimes out of range -> must be ignored identically
            table[u] = oracle.fault_entry(int(rng.integers(0, 4)) & 3, site, int(rng.integers(0, 32)))
            if rng.random() < 0.1:
                table[u] &= 0x7FFFFFFF                                  # valid bit cleared
    unit_base = int(rng.choice([0, 0, 12345, 2 ** 33 + 7]))
    return kernel, nc, inp, n, flags, kw, plan_kw, table, unit_base


@pytest.mark.parametrize("chunk", range(8))
def test_differential_fuzz(rt, oracle, chunk):
    from test_gpu_parity import both
    rng = np.random.default_rng(1000 + chunk)
    for _ in range(25):
        kernel, nc, inp, n, flags, kw, plan_kw, table, unit_base = _case(rng, oracle)
        both(rt, oracle, kernel, nc, inp, n, flags=flags, plan_kw=plan_kw, table=table, unit_base=unit_base, **kw)
