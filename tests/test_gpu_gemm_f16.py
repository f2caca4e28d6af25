"""GPU (H100): COAST_K_GEMM_F16 (float16 A and B, fp32 accumulators, wgmma m64n128k16 f16, GEMM_BF16's layout) and its FP16
output (COAST_MM_OUT_F16, the xmr_h16_* kernels).

Exact wherever arithmetic allows it: integer operands in [-16, 16] with K 256 < 2^24 make every partial sum an exact fp32
integer, so outputs equal the CPU reference (tests/gemm_f16_ref.py) bit for bit in any summation order.  Pinned here:
  * every variant (narrow, wide, pair, single CTA) at NC 1-3, with no plan, Bernoulli plans and TABLE plans, both voters, B and
    B^T, against the reference, counters and d_status included; batches, and groups with Zipf routing and empty experts;
    multi-wave shapes; a shard; the host call;
  * FP16 output: the reference bit for bit on integer operands, and the fp32 launch's C converted by torch on N(0, 1) operands
    with and without plans (but for the documented sign-of-zero corner), and on sums that overflow to infinity;
  * unprotected torch.matmul on half tensors and GEMM_TF32 on the upcast operands, bit for bit on integer data; a float64
    product within an fp32-accumulation bound on random data; and the same bits from every variant, NC and B layout;
  * what the H100 does with subnormal operands, and the NaN pattern of the f16 conversion."""
import numpy as np
import pytest

import gemm_f16_ref as ref
from mm_gpu import STAT_KEYS, add_stats, both, cpu, dev, env, gpu, no_stats, transposed
from test_gpu_gemm_bf16_fp8 import zipf_offsets
from coast_b200.runtime import (F_MAJORITY_VOTER, F_VERBOSE, K_GEMM_F16, K_GEMM_TF32, MM_B_TRANSPOSED as MM_BT, MM_BATCHED,
                                MM_GROUPED, MM_OUT_F16)

pytestmark = pytest.mark.gpu

POISON16 = 0x7E5A                                  # a NaN; every NaN the conversion writes is ref.NAN_F16
RO = [3, 3, 100, 101, 101, 500, 700, 828]          # from row 3: empty products, a one-row product, a 128-row product


class F16:
    """the operand record tests/mm_gpu.py's gpu(), cpu() and both() take"""
    name, kernel = "f16", K_GEMM_F16
    ref, bits, value = ref, staticmethod(ref.bits), staticmethod(ref.value)

    @staticmethod
    def tensor(x):
        import torch
        return torch.from_numpy(np.ascontiguousarray(x).view(np.int16)).view(torch.float16)

    @staticmethod
    def int_operands(M, N, K, seed, amax=16):
        return ref.int_operands(np.random.default_rng(seed), M, N, K, amax)

    @staticmethod
    def normal_operands(M, N, K, seed):
        """N(0, 1) rounded to float16 by torch"""
        import torch
        g = torch.Generator().manual_seed(seed)

        def one(r, c):
            return torch.randn(r, c, generator=g).to(torch.float16).view(torch.int16).numpy().view(np.uint16).copy()
        return one(M, K), one(K, N)


def launch(rt, nc, A, B, *, h16=False, flags=3, plan=None, table=None, unit_base=0, mode=0, M=None, n=None, rows=None, bt=False,
           status=None):
    """A: (rows x K), B: (P K x N) float16 patterns -> (C as uint16 f16 patterns (h16) or uint32 fp32 patterns; stats dict)"""
    import torch
    import coast_b200 as cb
    if not h16:
        return gpu(rt, F16, nc, A, B, flags=flags, plan=plan, table=table, unit_base=unit_base, status=status, mode=mode, M=M, n=n,
                   rows=rows, bt=bt)
    K, N = A.shape[1], B.shape[1]
    if table is not None:
        plan = cb.FaultPlan(mode=cb.PLAN_TABLE, table=torch.from_numpy(table.view(np.int32).copy()).cuda())
    out = torch.full((A.shape[0] * N,), POISON16, dtype=torch.int16, device="cuda").view(torch.float16)
    aux = dev(F16, transposed(B, K)) if bt else dev(F16, B)
    _, st = rt.run(K_GEMM_F16, nc, dev(F16, A), A.shape[0] * N if n is None else n, M=A.shape[0] if M is None else M, N=N, K=K,
                   aux=aux, flags=flags, plan=plan, unit_base=unit_base, status=status,
                   mode=mode | MM_OUT_F16 | (MM_BT if bt else 0), rows=rows, out=out)
    return out.cpu().view(torch.int16).numpy().view(np.uint16), st.as_dict()


def exact(A, B):
    return F16.value(A).astype(np.float64) @ F16.value(B).astype(np.float64)


# (id, environment, NC, M, N, the kernel the launcher must pick)
VARIANTS = [
    ("narrow_nc1", {}, 1, 256, 384, "xmr_gemm_f16n_inj0_nc1"),
    ("wide_nc1", {"COAST_GEMM_PAIR": "0"}, 1, 256, 256, "xmr_gemm_f16_inj0_nc1"),
    ("pair_nc1", {}, 1, 256, 256, "xmr_gemm_f16p_inj0_nc1"),
    ("pair_nc2", {}, 2, 256, 128, "xmr_gemm_f16p_inj0_nc2"),
    ("single_nc2", {"COAST_GEMM_PAIR": "0"}, 2, 256, 128, "xmr_gemm_f16_inj0_nc2"),
    ("single_nc3", {}, 3, 256, 128, "xmr_gemm_f16_inj0_nc3"),
    ("pair_nc3", {"COAST_GEMM_PAIR": "1"}, 3, 256, 256, "xmr_gemm_f16p_inj0_nc3"),
]


def table_plan(oracle, n, seed):
    rng = np.random.default_rng(seed)
    tab = np.zeros(n, dtype=np.uint32)
    for u in rng.choice(n, size=300, replace=False):
        site = 0 if rng.random() < 0.8 else 1                      # site 1 does not exist: ignored
        tab[u] = oracle.fault_entry(int(rng.integers(0, 4)), site, int(rng.integers(0, 32)))   # replica >= NC: ignored
    return tab


@pytest.mark.parametrize("K", [64, 448, 1088])                     # one k-block; one ring wrap; many wraps
@pytest.mark.parametrize("variant", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_integer_operands_bit_exact_with_the_oracle(rt, oracle, variant, K, monkeypatch, capfd):
    import torch
    _, e, nc, M, N, kname = variant
    env(monkeypatch, **e)
    A, B = F16.int_operands(M, N, K, seed=K + 10 * nc)
    n = M * N
    capfd.readouterr()
    gpu(rt, F16, nc, A, B, flags=F_VERBOSE)
    assert f"{kname} " in capfd.readouterr().err
    g, st = both(rt, oracle, F16, nc, A, B)
    assert (g.view(np.float32).reshape(M, N).astype(np.float64) == exact(A, B)).all()
    assert st["errors_corrected"] == st["dwc_detected"] == 0 and st["syncs"] == (n if nc == 3 else 0)
    for bt in (False, True):
        _, st = both(rt, oracle, F16, nc, A, B, plan_kw=dict(seed=K, p=0.3), bt=bt)
        assert st["injected"] > n // 5
    both(rt, oracle, F16, nc, A, B, flags=3 | F_MAJORITY_VOTER, plan_kw=dict(seed=K + 1, p=0.3), bt=True)
    base = 2 ** 32 - n // 2                                        # the global units cross 2^32
    tab = table_plan(oracle, n, K + nc)
    for bt in (False, True):
        status = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
        g, gs = gpu(rt, F16, nc, A, B, table=tab, unit_base=base, status=status, bt=bt)
        o, os_ = cpu(oracle, F16, nc, A, B, table=tab, unit_base=base)
        assert (g == o).all() and {k: gs[k] for k in STAT_KEYS} == {k: os_[k] for k in STAT_KEYS} and gs["injected"] > 0
        s = status.cpu().numpy()
        assert set(np.unique(s)) <= {0, 1}
        assert int(s.sum()) == (gs["errors_corrected"] if nc == 3 else gs["dwc_detected"] if nc == 2 else 0)


@pytest.mark.parametrize("bt", [False, True], ids=["B", "Bt"])
@pytest.mark.parametrize("nc", [1, 2, 3])
def test_batches_and_zipf_groups_equal_the_reference_per_product(rt, oracle, monkeypatch, nc, bt):
    """a batch of 3 and 16 Zipf-routed experts (some empty) from row 3, each product against the reference with the plan's
    global units; rows outside the group table keep the poison"""
    import torch
    env(monkeypatch)
    N, K = 256, 192
    plan_kw = dict(seed=11 + nc, p=0.2)
    import coast_b200 as cb
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, **plan_kw)
    # batch: 3 products of 256 rows
    A, B = F16.int_operands(3 * 256, N, 3 * K, seed=nc)
    A = np.ascontiguousarray(A[:, :K])
    g, gs = gpu(rt, F16, nc, A, B, plan=plan, unit_base=7, mode=MM_BATCHED, M=256, bt=bt)
    tot = no_stats()
    for p in range(3):
        o, os_ = cpu(oracle, F16, nc, A[p * 256:(p + 1) * 256], B[p * K:(p + 1) * K], plan_kw=plan_kw, unit_base=7 + p * 256 * N)
        assert (g[p * 256 * N:(p + 1) * 256 * N] == o).all(), p
        add_stats(tot, os_)
    assert {k: gs[k] for k in STAT_KEYS} == tot and gs["injected"] > 0
    # groups
    ro = zipf_offsets(16, 1500, start=3, seed=nc)
    G = len(ro) - 1
    A, B = F16.int_operands(ro[-1], N, G * K, seed=10 + nc)
    A = np.ascontiguousarray(A[:, :K])
    rows = torch.tensor(ro, dtype=torch.int64, device="cuda")
    g, gs = gpu(rt, F16, nc, A, B, plan=plan, unit_base=9, mode=MM_GROUPED, M=G, n=(ro[-1] - ro[0]) * N, rows=rows, bt=bt)
    assert (g[:ro[0] * N] == 0x7FC00000).all()                    # the poison of mm_gpu.gpu: NaN
    tot = no_stats()
    for p in range(G):
        if ro[p + 1] == ro[p]:
            continue
        o, os_ = cpu(oracle, F16, nc, A[ro[p]:ro[p + 1]], B[p * K:(p + 1) * K], plan_kw=plan_kw, unit_base=9 + (ro[p] - ro[0]) * N)
        assert (g[ro[p] * N:ro[p + 1] * N] == o).all(), p
        add_stats(tot, os_)
    assert {k: gs[k] for k in STAT_KEYS} == tot


@pytest.mark.parametrize("M,N,K", [(2048, 2048, 256), (1408, 1792, 512)])
def test_multi_wave_every_variant_equals_fp64(rt, monkeypatch, M, N, K):
    A, B = F16.int_operands(M, N, K, seed=M)
    want = exact(A, B)
    for e in ({}, {"COAST_GEMM_PAIR": "0"}, {"COAST_GEMM_TAIL_SPLIT": "0"}):
        env(monkeypatch, **e)
        for nc in (1, 2, 3):
            g, st = gpu(rt, F16, nc, A, B, bt=nc == 2)
            assert (g.view(np.float32).reshape(M, N).astype(np.float64) == want).all(), (e, nc)
            assert st["errors_corrected"] == st["dwc_detected"] == 0


def test_shard_and_host_call(rt, oracle, monkeypatch):
    """two row shards of one product equal the whole launch; the host call in row blocks and in Zipf groups equals the device
    launch, fp32 and f16 C"""
    import torch
    import coast_b200 as cb
    env(monkeypatch, COAST_HOST_CHUNK_BYTES="400000")
    N, K = 256, 256
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, seed=3, p=0.2)
    A, B = F16.int_operands(1024, N, K, seed=1)
    full, fs = gpu(rt, F16, 3, A, B, plan=plan, unit_base=10)
    tot = no_stats()
    parts = []
    for lo in (0, 512):
        g, st = gpu(rt, F16, 3, A[lo:lo + 512], B, plan=plan, unit_base=10 + lo * N)
        parts.append(g)
        add_stats(tot, st)
    assert (np.concatenate(parts) == full).all() and {k: fs[k] for k in STAT_KEYS} == tot
    for h16 in (False, True):
        dev_out, ds = launch(rt, 3, A, B, h16=h16, plan=plan)
        h_out = np.zeros(1024 * N, dtype=np.uint16 if h16 else np.uint32)
        st = rt.run_host(K_GEMM_F16, 3, F16.tensor(A), h_out, 1024 * N, M=1024, N=N, K=K, h_aux=F16.tensor(B), flags=3, plan=plan,
                         mode=MM_OUT_F16 if h16 else 0)
        assert np.array_equal(h_out, dev_out) and st.as_dict() == ds and rt.last_host_path == "row-blocks"
    ro = zipf_offsets(10, 700, start=3, seed=9)
    G = len(ro) - 1
    A, B = F16.int_operands(ro[-1], N, G * K, seed=2)
    A = np.ascontiguousarray(A[:, :K])
    rows = torch.tensor(ro, dtype=torch.int64, device="cuda")
    for h16 in (False, True):
        dev_out, ds = launch(rt, 3, A, B, h16=h16, M=G, n=(ro[-1] - ro[0]) * N, mode=MM_GROUPED, rows=rows)
        h_out = np.zeros(ro[-1] * N, dtype=np.uint16 if h16 else np.uint32)
        st = rt.run_host(K_GEMM_F16, 3, F16.tensor(A), h_out, (ro[-1] - ro[0]) * N, M=G, N=N, K=K, h_aux=F16.tensor(B), flags=3,
                         mode=MM_GROUPED | (MM_OUT_F16 if h16 else 0), h_rows=np.array(ro, dtype=np.uint64))
        assert np.array_equal(h_out[ro[0] * N:], dev_out[ro[0] * N:]) and st.syncs == ds["syncs"]
        assert rt.last_host_path == "groups"


# ------------------------------------------------------------------------------------------ FP16 output
@pytest.mark.parametrize("voter", [0, F_MAJORITY_VOTER], ids=["select", "majority"])
@pytest.mark.parametrize("variant", VARIANTS, ids=[v[0] for v in VARIANTS])
def test_f16_output_bit_exact_with_the_reference(rt, oracle, monkeypatch, variant, voter):
    """integer operands with sums up to 2^16 (more than float16's 11 significant bits: roundings and ties happen)"""
    import coast_b200 as cb
    _, e, nc, M, N, kname = variant
    env(monkeypatch, **e)
    A, B = F16.int_operands(M, N, 256, seed=nc + 3)
    for bt in (False, True):
        for plan_kw, base in ((None, 0), (dict(seed=3 + nc, p=0.3), 2 ** 32 - M * N // 2)):
            plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, **plan_kw) if plan_kw else None
            g, gs = launch(rt, nc, A, B, h16=True, flags=3 | voter, plan=plan, unit_base=base, bt=bt)
            pl = oracle.make_plan(oracle.PLAN_BERNOULLI, **plan_kw) if plan_kw else None
            o, os_, _ = ref.run_f16(oracle, nc, A, B, flags=3 | voter, plan=pl, unit_base=base)
            assert np.array_equal(g, o), (bt, np.flatnonzero(g != o)[:8], g[g != o][:4], o[g != o][:4])
            assert {k: gs[k] for k in STAT_KEYS} == {k: os_[k] for k in STAT_KEYS}


def torch_f16(c32):
    """fp32 bit patterns -> float16 patterns, converted by torch on the device"""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(c32).view(np.float32)).cuda()
    return t.to(torch.float16).view(torch.int16).cpu().numpy().view(np.uint16)


LAYOUTS = [("single", None), ("batched", 3), ("grouped", RO)]


@pytest.mark.parametrize("voter", [0, F_MAJORITY_VOTER], ids=["select", "majority"])
@pytest.mark.parametrize("bt", [False, True], ids=["B", "Bt"])
@pytest.mark.parametrize("layout", LAYOUTS, ids=[c[0] for c in LAYOUTS])
def test_f16_output_is_the_fp32_output_converted_by_torch(rt, oracle, monkeypatch, layout, bt, voter):
    """N(0, 1) operands: for the same plan, the f16 C is the fp32 C converted, but where the select voter meets a sign flip on
    replica 0 of a nonzero value that rounds to zero (DESIGN.md §3.15): there it is the zero of the other sign"""
    import torch
    import coast_b200 as cb
    env(monkeypatch)
    name, extra = layout
    N, K = 256, 512
    kw = {}
    if name == "single":
        A, B = F16.normal_operands(512, N, K, 1)
    elif name == "batched":
        A, B = F16.normal_operands(extra * 256, N, K * extra, 2)
        A = np.ascontiguousarray(A[:, :K])
        kw = dict(M=256, mode=MM_BATCHED)
    else:
        G = len(extra) - 1
        A, B = F16.normal_operands(extra[-1], N, K * G, 3)
        A = np.ascontiguousarray(A[:, :K])
        kw = dict(M=G, mode=MM_GROUPED, n=(extra[-1] - extra[0]) * N, rows=torch.tensor(extra, dtype=torch.int64, device="cuda"))
    first = extra[0] if name == "grouped" else 0
    n = (A.shape[0] - first) * N
    clean, _ = launch(rt, 1, A, B, bt=bt, **kw)
    for nc in (1, 2, 3):
        for plan_kw, base in ((None, 0), (dict(seed=4 + nc, p=0.3), 2 ** 32 - 1000)):
            plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, **plan_kw) if plan_kw else None
            g32, s32 = launch(rt, nc, A, B, flags=3 | voter, plan=plan, unit_base=base, bt=bt, **kw)
            g16, s16 = launch(rt, nc, A, B, h16=True, flags=3 | voter, plan=plan, unit_base=base, bt=bt, **kw)
            want = torch_f16(g32[first * N:])
            if plan_kw and nc == 3 and not voter:
                pl = oracle.make_plan(oracle.PLAN_BERNOULLI, **plan_kw)
                c = clean[first * N:]
                for u, r, bit in ref.sref.faults(oracle, pl, nc, K, n, base):
                    if r == 0 and bit == 31 and c[u] & 0x7FFFFFFF and ref.rne(c[u:u + 1])[0] & 0x7FFF == 0:
                        want[u] ^= 0x8000
            assert np.array_equal(g16[first * N:], want), np.flatnonzero(g16[first * N:] != want)[:8]
            assert (g16[:first * N] == POISON16).all()
            assert s16["injected"] == s32["injected"] and s16["syncs"] == s32["syncs"]
            if nc > 1:
                key = "errors_corrected" if nc == 3 else "dwc_detected"
                assert s16[key] <= s32[key]


def test_f16_output_overflows_to_infinity(rt, oracle, monkeypatch):
    """row i of A is 2048 + 16 i in column 0 (exact float16), B[0, j] = +-(16 + j / 64) rounded: the products pass 65504 and
    65520 along each row, with both signs, and the device agrees with the reference on where infinity starts"""
    env(monkeypatch)
    M, N, K = 128, 256, 64
    A, B = np.zeros((M, K), np.uint16), np.zeros((K, N), np.uint16)
    A[:, 0] = F16.bits(2048 + 16 * np.arange(M, dtype=np.float32))
    col = np.array(16 + np.arange(N) / 64, dtype=np.float32).astype(np.float16).astype(np.float32)
    B[0, :] = F16.bits(np.where(np.arange(N) % 2, -col, col))
    for nc in (1, 3):
        g, _ = launch(rt, nc, A, B, h16=True)
        o, _, _ = ref.run_f16(oracle, nc, A, B)
        assert np.array_equal(g, o)
        assert (g == 0x7C00).sum() > 1000 and (g == 0xFC00).sum() > 1000


def test_nan_pattern_of_the_conversion_and_nan_votes(rt, oracle, monkeypatch):
    """inf x 0 and inf - inf make NaN accumulators of either sign; the device writes one f16 NaN pattern, the reference's, and
    every NaN element disagrees with itself under DWC and TMR"""
    env(monkeypatch)
    M, N, K = 128, 128, 64
    A, B = F16.int_operands(M, N, K, seed=5)
    A[3, 0], A[4, 1], A[4, 2] = 0x7C00, 0x7C00, 0xFC00              # +inf; +inf and -inf in one row
    B[0, 5] = 0                                                    # +inf x 0 in C[3, 5]
    B[1, :] = B[2, :] = F16.bits(np.float32(1.0))                  # inf - inf along row 4
    for nc in (1, 2, 3):
        g, gs = launch(rt, nc, A, B, h16=True)
        nan = (g & 0x7FFF) > 0x7C00
        assert nan.reshape(M, N)[4].all() and nan.reshape(M, N)[3, 5]
        assert set(np.unique(g[nan]).tolist()) == {ref.NAN_F16}, sorted(hex(x) for x in np.unique(g[nan]))
        o, os_, _ = ref.run_f16(oracle, nc, A, B)
        assert np.array_equal(g, o) and {k: gs[k] for k in STAT_KEYS} == {k: os_[k] for k in STAT_KEYS}
        g32, s32 = launch(rt, nc, A, B)
        assert s32["errors_corrected" if nc == 3 else "dwc_detected"] == (int(nan.sum()) if nc > 1 else 0)


# ------------------------------------------------------------------------------------------ against torch and the TF32 route
def test_equals_torch_matmul_on_half_tensors_and_gemm_tf32_on_the_upcast_operands(rt, monkeypatch):
    import torch
    env(monkeypatch)
    saved = torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction
    torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = False
    try:
        for M, N, K in ((512, 512, 1024), (384, 384, 512)):
            A, B = F16.int_operands(M, N, K, seed=M)
            want16 = torch.matmul(dev(F16, A), dev(F16, B)).view(torch.int16).cpu().numpy().view(np.uint16).ravel()
            fa, fb = dev(F16, A).float(), dev(F16, B).float()
            tf32, _ = rt.run(K_GEMM_TF32, 1, fa, M * N, M=M, N=N, K=K, aux=fb)
            want32 = tf32.cpu().numpy().view(np.uint32)
            for nc in (1, 3):
                for bt in (False, True):
                    g16, _ = launch(rt, nc, A, B, h16=True, bt=bt)
                    g32, _ = launch(rt, nc, A, B, bt=bt)
                    assert np.array_equal(g16, want16) and np.array_equal(g32, want32), (nc, bt)
    finally:
        torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = saved


RUNS = [({"COAST_GEMM_PAIR": p}, nc) for nc in (1, 2, 3) for p in ("0", "1")] + [({"COAST_GEMM_TAIL_SPLIT": "0"}, 1)]


@pytest.mark.parametrize("M,N,K", [(512, 768, 320), (256, 384, 64), (384, 256, 2048)])
def test_random_operands_every_variant_same_bits_and_within_fp32_bound(rt, monkeypatch, M, N, K):
    """N(0, 1) operands: every variant, replica count and B layout gives the same bits, within GEMM_TF32's bound 2e-6 K of the
    float64 product (the products are exact; only the fp32 sums round)"""
    A, B = F16.normal_operands(M, N, K, seed=K)
    want = exact(A, B)
    first = None
    for e, nc in RUNS:
        env(monkeypatch, **e)
        for bt in (False, True):
            g, st = launch(rt, nc, A, B, bt=bt)
            assert st["errors_corrected"] == st["dwc_detected"] == 0
            if first is None:
                first = g
                err = np.abs(g.view(np.float32).reshape(M, N).astype(np.float64) - want)
                assert (err <= 2e-6 * K * np.maximum(1.0, np.abs(want) / 8)).all(), err.max()
            assert (g == first).all(), (e, nc, bt)


def test_subnormal_operands_are_exact(rt, oracle, monkeypatch):
    """float16 subnormals (k 2^-24, 0 < |k| < 1024) times integers: every product and partial sum is exact in fp32, and the H100's
    f16 wgmma keeps them -- C equals the float64 product and the reference, no operand flushed to zero"""
    env(monkeypatch)
    M, N, K = 256, 256, 128
    rng = np.random.default_rng(4)
    A = F16.bits(rng.integers(-1023, 1024, (M, K)).astype(np.float32) * np.float32(2.0 ** -24))
    _, B = F16.int_operands(M, N, K, seed=4, amax=4)
    assert (((A & 0x7C00) == 0) & ((A & 0x3FF) != 0)).mean() > 0.99
    for nc in (1, 3):
        g, st = both(rt, oracle, F16, nc, A, B)
        assert (g.view(np.float32).reshape(M, N).astype(np.float64) == exact(A, B)).all()
        assert (g != 0).mean() > 0.99
