"""The two wgmma matmul kernels pinned bit for bit (CPU reference tests + H100 tests).

TF32 GEMM (xmr_gemm_tf32.cuh).  With integer-valued operands |x| <= amax and amax^2 * K < 2^24, every product and every
partial sum is an integer below 2^24, so fp32 adds them exactly in any order.  The tensor-core result, the oracle
(orc_gemm_tf32_elem sums in double) and an fp64 matmul then agree BIT FOR BIT, and the exact harness of test_gpu_parity
(`both`: output bytes and all five counters, with and without faults) covers the GEMM like the integer kernels.  Only the
uniform-operand tests of test_gpu_gemm.py keep a tolerance.

Exact u32 matmul on u8 limbs (xmr_mm_tc.cuh).  The s32 limb accumulators pass 2^31 for K > 8256 at worst-case limbs and
must wrap.  Every element is checked against mm_u32_ref, an exact mod-2^32 matmul on 16-bit limbs in float64.

Every exact check here compares every element of the output."""
import numpy as np
import pytest

from mm_gpu import POISON, STAT_KEYS, env as _gemm_env
from test_gpu_parity import both, dev, host


# ------------------------------------------------------------------------------------------ references (CPU)
def int_operands(M, N, K, seed, amax=8):
    """integer-valued fp32 A (M x K) and B (K x N), uniform in [-amax, amax], from Philox words.  |C| <= amax^2 * K < 2^24:
    every partial sum is exact in fp32, whatever the order of the additions."""
    assert amax * amax * K < 2 ** 24, (amax, K)
    from oracle import pyoracle as po
    w = po.fill_philox(M * K + K * N, 0, seed).astype(np.int64) % (2 * amax + 1) - amax
    return w[: M * K].astype(np.float32).reshape(M, K), w[M * K:].astype(np.float32).reshape(K, N)


def junk_low_bits(x, seed):
    """x with random bits 0..11 in every fp32 word and bit 12 clear: truncation to TF32 (bits 0..12 dropped) and rounding
    to nearest at bit 13 both give back x's TF32 value, so the result cannot depend on which one the tensor core does"""
    from oracle import pyoracle as po
    junk = po.fill_philox(x.size, 0, seed).reshape(x.shape) & np.uint32(0xFFF)
    return ((x.view(np.uint32) & np.uint32(0xFFFFE000)) | junk).view(np.float32)


def tf32_trunc(x):
    return (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def tf32_rne(x):
    u = x.view(np.uint32).astype(np.uint64)
    u = (u + 0xFFF + ((u >> 13) & 1)) & 0xFFFFE000
    return u.astype(np.uint32).view(np.float32)


def mm_u32_ref(A, B):
    """Exact C = A . B mod 2^32 of u32 matrices: numpy uint32, or torch int32 holding the u32 bits (any device).
    With 16-bit limbs, C = A0.B0 + ((A0.B1 + A1.B0) mod 2^16) << 16 (mod 2^32).  Each limb product sum is below
    2^32 * K < 2^53, so the three float64 matmuls are exact for K < 2^21.  Returns int64 values in [0, 2^32)."""
    K = A.shape[1]
    assert B.shape[0] == K and K < 2 ** 21
    if isinstance(A, np.ndarray):
        wide, f64, i64 = (lambda x: x.astype(np.int64) & 0xFFFFFFFF), (lambda x: x.astype(np.float64)), (lambda x: x.astype(np.int64))
    else:
        import torch
        wide, f64, i64 = (lambda x: x.to(torch.int64) & 0xFFFFFFFF), (lambda x: x.to(torch.float64)), (lambda x: x.to(torch.int64))
    a, b = wide(A), wide(B)
    a0, a1, b0, b1 = f64(a & 0xFFFF), f64(a >> 16), f64(b & 0xFFFF), f64(b >> 16)
    lo = i64(a0 @ b0)
    mid = i64(a0 @ b1) + i64(a1 @ b0)
    return (lo + ((mid & 0xFFFF) << 16)) & 0xFFFFFFFF


def test_int_operands_are_exact_small_integers(oracle):
    A, B = int_operands(64, 48, 16384, seed=3)
    for X in (A, B):
        assert (X == np.round(X)).all() and np.abs(X).max() == 8 and (X == 0).any()
        assert (tf32_trunc(X).view(np.uint32) == X.view(np.uint32)).all()        # exact in TF32 as well
    with pytest.raises(AssertionError):
        int_operands(8, 8, 16384, seed=3, amax=32)                               # 2^10 * 2^14: sums would reach 2^24


def test_junk_low_bits_keeps_the_tf32_value_under_truncation_and_rounding(oracle):
    A, _ = int_operands(128, 8, 512, seed=5)
    J = junk_low_bits(A, seed=6)
    u, ju = A.view(np.uint32), J.view(np.uint32)
    assert not (ju & np.uint32(0x1000)).any()                                    # bit 12 clear
    assert (ju & np.uint32(0xFFFFE000) == u).all() and (ju != u).mean() > 0.99   # only bits 0..11 differ, nearly everywhere
    assert (tf32_trunc(J).view(np.uint32) == u).all()
    assert (tf32_rne(J).view(np.uint32) == u).all()
    # the rounding model is not vacuous: with bit 12 set as well, rounding to nearest moves the value, truncation does not
    J2 = (ju | np.uint32(0x1FFF)).view(np.float32)
    assert (tf32_trunc(J2).view(np.uint32) == u).all() and (tf32_rne(J2).view(np.uint32)[u != 0] != u[u != 0]).all()


@pytest.mark.parametrize("M,N,K", [(9, 9, 9), (17, 33, 5), (3, 130, 257), (64, 48, 130)])
def test_mm_u32_ref_matches_the_oracle(oracle, M, N, K):
    import torch
    A = oracle.fill_philox(M * K, 0, 4 + K)
    B = oracle.fill_philox(K * N, 0, 44 + K)
    A[:7] = 0xFFFFFFFF
    B[-5:] = 0xFFFFFFFF
    o, _ = oracle.run(oracle.K_MM_U32, 1, A, M * N, M=M, N=N, K=K, aux=B)
    want = o.view(np.uint32).reshape(M, N).astype(np.int64)
    assert (mm_u32_ref(A.reshape(M, K), B.reshape(K, N)) == want).all()
    got_t = mm_u32_ref(torch.from_numpy(A.view(np.int32).reshape(M, K)), torch.from_numpy(B.view(np.int32).reshape(K, N)))
    assert (got_t.numpy() == want).all()


@pytest.mark.parametrize("K", [1, 5, 8320, 16640, 32768, 2 ** 20 + 3])
def test_mm_u32_ref_all_ones_closed_form(K):
    """(2^32 - 1)^2 == 1 (mod 2^32), so the all-0xFFFFFFFF product is K mod 2^32 in every element"""
    A = np.full((2, K), 0xFFFFFFFF, dtype=np.uint32)
    B = np.full((K, 3), 0xFFFFFFFF, dtype=np.uint32)
    assert (mm_u32_ref(A, B) == K % 2 ** 32).all()


# ------------------------------------------------------------------------------------------ TF32 GEMM == oracle, bit for bit
# (id, COAST_GEMM_PAIR, NC, M, N, the kernel the launcher must pick)
GEMM_VARIANTS = [
    ("tf32n_nc1", None, 1, 256, 384, "xmr_gemm_tf32n_nc1"),       # N % 256 != 0: 128 x 128 tiles
    ("wide_nc1", "0", 1, 256, 256, "xmr_gemm_tf32_nc1"),          # 128 x 256 tiles
    ("pair_nc1", None, 1, 256, 256, "xmr_gemm_tf32p_nc1"),
    ("pair_nc2", None, 2, 256, 128, "xmr_gemm_tf32p_nc2"),
    ("single_nc2", "0", 2, 256, 128, "xmr_gemm_tf32_nc2"),
    ("single_nc3", None, 3, 256, 128, "xmr_gemm_tf32_nc3"),
    ("pair_nc3", "1", 3, 256, 256, "xmr_gemm_tf32p_nc3"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("K", [32, 192, 224, 1056])      # one k-block; one 6-stage ring exactly; one wrap; many wraps
@pytest.mark.parametrize("variant", GEMM_VARIANTS, ids=[v[0] for v in GEMM_VARIANTS])
def test_gemm_tf32_integer_operands_bit_exact_with_the_oracle(rt, oracle, variant, K, monkeypatch, capfd):
    import coast_b200 as cb
    _, pair, nc, M, N, kname = variant
    _gemm_env(monkeypatch, **({"COAST_GEMM_PAIR": pair} if pair else {}))
    A, B = int_operands(M, N, K, seed=K + 10 * nc)
    n = M * N
    capfd.readouterr()
    rt.run(cb.K_GEMM_TF32, nc, dev(rt, A), n, M=M, N=N, K=K, aux=dev(rt, B), flags=cb.F_VERBOSE)
    assert f"{kname}_inj0 " in capfd.readouterr().err
    mm = dict(M=M, N=N, K=K, aux=B)
    g, st = both(rt, oracle, oracle.K_GEMM_TF32, nc, A, n, flags=3, **mm)
    assert (g.view(np.float32).reshape(M, N).astype(np.float64) == A.astype(np.float64) @ B.astype(np.float64)).all()
    assert st["errors_corrected"] == st["dwc_detected"] == 0 and st["syncs"] == (n if nc == 3 else 0)
    both(rt, oracle, oracle.K_GEMM_TF32, nc, A, n, flags=0, **mm)
    _, st = both(rt, oracle, oracle.K_GEMM_TF32, nc, A, n, flags=3, plan_kw=dict(seed=K, p=0.1), **mm)
    assert st["injected"] > n // 20
    both(rt, oracle, oracle.K_GEMM_TF32, nc, A, n, flags=3 | cb.F_MAJORITY_VOTER, plan_kw=dict(seed=K + 1, p=0.3), **mm)
    both(rt, oracle, oracle.K_GEMM_TF32, nc, A, n, flags=1, plan_kw=dict(seed=K + 2, threshold=1 << 30), unit_base=2 ** 33 + 7, **mm)
    rng = np.random.default_rng(K + nc)
    tab = np.zeros(n, dtype=np.uint32)
    for u in rng.choice(n, size=300, replace=False):
        site = 0 if rng.random() < 0.8 else 1                      # site 1 does not exist: ignored
        tab[u] = oracle.fault_entry(int(rng.integers(0, 4)), site, int(rng.integers(0, 32)))   # replica 3 / >= NC: ignored
        if rng.random() < 0.1:
            tab[u] &= 0x7FFFFFFF                                   # valid bit clear: ignored
    _, st = both(rt, oracle, oracle.K_GEMM_TF32, nc, A, n, flags=3, table=tab, unit_base=12345, **mm)
    assert st["injected"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("nc", [1, 3])
def test_gemm_tf32_reads_only_the_tf32_bits_of_each_operand(rt, oracle, nc):
    """junk in bits 0..11 of every operand word changes nothing: the output equals the clean integer operands' bit for bit"""
    import coast_b200 as cb
    M, N, K = 256, 384, 224
    A, B = int_operands(M, N, K, seed=31)
    clean, _ = oracle.run(oracle.K_GEMM_TF32, 1, A, M * N, M=M, N=N, K=K, aux=B)
    out, st = rt.run(cb.K_GEMM_TF32, nc, dev(rt, junk_low_bits(A, 5)), M * N, M=M, N=N, K=K, aux=dev(rt, junk_low_bits(B, 6)), flags=3)
    assert host(out).tobytes() == clean.tobytes()
    assert st.errors_corrected == 0


# every kernel variant and every schedule knob at multi-wave sizes: (environment, NC, desc mode)
TF32_RUNS = [({"COAST_GEMM_PAIR": p}, nc, 0) for nc in (1, 2, 3) for p in ("0", "1")] + [
    ({"COAST_GEMM_TAIL_SPLIT": "0"}, 1, 0),
    ({"COAST_GEMM_TAIL_SPLIT": "0", "COAST_GEMM_PAIR": "0"}, 1, 0),
] + [({"COAST_GEMM_GROUP_M": g}, nc, 0) for g in ("1", "3", "16", "255") for nc in (1, 3)] + [
    ({"COAST_GEMM_L2_HINTS": "0"}, 1, 0),
    ({"COAST_GEMM_L2_HINTS": "0"}, 3, 0),
    ({}, 1, 5),                                                   # desc mode: group of 5 tile-rows
    ({"COAST_GEMM_PAIR": "0"}, 1, 7),
    ({}, 2, 5),
    ({}, 3, 7),
]


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", [(4096, 4096, 4096), (2560, 2048, 256), (2432, 2048, 256)])
def test_gemm_tf32_multi_wave_every_variant_and_knob_equals_fp64(rt, M, N, K, monkeypatch):
    """CTAs run several tiles each (the ring phase carries from tile to tile); 2560 / 2432 rows leave a short last round that
    the unprotected kernels split into half tiles.  Every run is bit-identical, and equal to the fp64 matmul on every element."""
    import torch
    import coast_b200 as cb
    A, B = int_operands(M, N, K, seed=7)
    dA, dB = dev(rt, A), dev(rt, B)
    ref = dA.to(torch.float64) @ dB.to(torch.float64)
    first = None
    for env, nc, mode in TF32_RUNS:
        _gemm_env(monkeypatch, **env)
        out = torch.full((M * N,), float("nan"), dtype=torch.float32, device="cuda")      # poison: every element must be written
        _, st = rt.run(cb.K_GEMM_TF32, nc, dA, M * N, M=M, N=N, K=K, aux=dB, flags=3, mode=mode, out=out)
        assert st.errors_corrected == 0 and st.dwc_detected == 0, (env, nc, mode)
        assert torch.equal(out.view(M, N).to(torch.float64), ref), (env, nc, mode)
        if first is None:
            first = out.view(torch.int32).clone()
        assert torch.equal(out.view(torch.int32), first), (env, nc, mode)


# ------------------------------------------------------------------------------------------ fp32 voter edges (DESIGN 3.5)
@pytest.mark.gpu
def test_gemm_vote_is_ordered_equal_on_signed_zeros(rt, oracle):
    """A zero row of A against B >= 0 gives a +0.0 row of C.  A flip of bit 31 of one replica's accumulator there makes
    -0.0, which equals +0.0 under `fcmp oeq`: the voter counts none of them and stores r0's value (-0.0 exactly where
    replica 0 was flipped).  A flip of bit 0 there makes a denormal, which does not compare equal: counted."""
    import coast_b200 as cb
    M, N, K = 256, 256, 64
    A, B = int_operands(M, N, K, seed=3)
    B = np.abs(B)
    z = 77
    A[z] = 0
    n = M * N
    tab = np.zeros(n, dtype=np.uint32)
    signs = [(z * N + 7 * c, c % 3) for c in range(30)]
    for u, r in signs:
        tab[u] = oracle.fault_entry(r, 0, 31)
    denormals = [(z * N + 250, 1), (z * N + 251, 0), (z * N + 252, 2)]
    for u, r in denormals:
        tab[u] = oracle.fault_entry(r, 0, 0)
    for nc in (2, 3):
        for flags in (3, 3 | cb.F_MAJORITY_VOTER) if nc == 3 else (3,):
            g, st = both(rt, oracle, oracle.K_GEMM_TF32, nc, A, n, M=M, N=N, K=K, aux=B, flags=flags, table=tab)
            row = g.view(np.uint32).reshape(M, N)[z]
            counted = [u for u, r in denormals if r < nc]
            assert st["injected"] == sum(r < nc for _, r in signs + denormals)
            assert (st["errors_corrected"] if nc == 3 else st["dwc_detected"]) == len(counted)
            assert st["first_fault_unit"] == min(counted)
            for u, r in signs:
                want = 0x80000000 if r == 0 and not flags & cb.F_MAJORITY_VOTER else 0
                assert row[u - z * N] == want, (nc, flags, u, r)
            assert row[251] == (1 if nc == 2 else 0)               # DWC stores r0's denormal; TMR votes r2's +0


@pytest.mark.gpu
@pytest.mark.parametrize("nc", [1, 2, 3])
def test_gemm_nan_row_disagrees_in_every_element(rt, oracle, nc):
    """a quiet NaN (0x7FC00000 survives TF32 truncation) in one row of A makes that C row NaN in every replica; NaN != NaN
    under `fcmp oeq`, so TMR -countErrors counts N disagreements and DWC N detections, as the oracle does.  The NaN payload the
    tensor core produces is not pinned: NaN positions must match, all other bits must be equal."""
    import coast_b200 as cb
    M, N, K = 256, 128, 96
    A, B = int_operands(M, N, K, seed=19)
    z = 130
    A[z, 9] = np.uint32(0x7FC00000).view(np.float32)
    o_out, o_st = oracle.run(oracle.K_GEMM_TF32, nc, A, M * N, M=M, N=N, K=K, aux=B, flags=3)
    g_out, g_st = rt.run(cb.K_GEMM_TF32, nc, dev(rt, A), M * N, M=M, N=N, K=K, aux=dev(rt, B), flags=3)
    g, o = host(g_out).view(np.float32).reshape(M, N), o_out.view(np.float32).reshape(M, N)
    nan = np.isnan(o)
    assert nan[z].all() and nan.sum() == N
    assert (np.isnan(g) == nan).all()
    assert (g.view(np.uint32)[~nan] == o.view(np.uint32)[~nan]).all()
    gd = g_st.as_dict()
    assert {k: gd[k] for k in STAT_KEYS} == {k: o_st[k] for k in STAT_KEYS}
    if nc > 1:
        assert (gd["errors_corrected"] if nc == 3 else gd["dwc_detected"]) == N and gd["first_fault_unit"] == z * N


# ------------------------------------------------------------------------------------------ per-unit status of device launches
@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["gemm", "mm"])
def test_matmul_device_launch_writes_the_per_unit_status(rt, oracle, kernel):
    """d_status[u] is 1 exactly at the units where the planned flip makes the replicas disagree, 0 elsewhere and everywhere
    under NC = 1; its sum is errors_corrected (TMR -countErrors) or dwc_detected (DWC)"""
    import torch
    import coast_b200 as cb
    rng = np.random.default_rng(8)
    if kernel == "gemm":
        kid, (M, N, K) = cb.K_GEMM_TF32, (256, 128, 64)
        A, B = int_operands(M, N, K, seed=23)
        A[5] = 0                                                   # a +0.0 row: bit-31 flips there do not disagree
        n_sites = 1
    else:
        kid, (M, N, K) = cb.K_MM_U32, (128, 128, 256)               # the tensor-core limb kernel
        A, B = oracle.fill_philox(M * K, 0, 4), oracle.fill_philox(K * N, 0, 44)
        n_sites = K
    n = M * N
    clean, _ = oracle.run(oracle.K_GEMM_TF32 if kernel == "gemm" else oracle.K_MM_U32, 1, A, n, M=M, N=N, K=K, aux=B)
    clean = clean.view(np.uint32)
    tab = np.zeros(n, dtype=np.uint32)
    picks = list(rng.choice(n, size=400, replace=False)) + [5 * N + c for c in range(0, N, 9)]
    ent = {}
    for u in picks:
        r, s, b = int(rng.integers(0, 4)), int(rng.integers(0, n_sites + 1)), int(rng.integers(0, 32))
        if u // N == 5 and kernel == "gemm":
            s, b = 0, 31
        tab[u] = oracle.fault_entry(r, s, b)
        ent[int(u)] = (r, s, b)
    table = torch.from_numpy(tab.view(np.int32).copy()).cuda()
    for nc in (1, 2, 3):
        want = np.zeros(n, dtype=np.uint8)
        for u, (r, s, b) in ent.items():
            if r < nc and s < n_sites:
                v = clean[u : u + 1]
                flipped = v ^ np.uint32(1 << b)
                want[u] = 1 if kernel == "mm" else int(flipped.view(np.float32)[0] != v.view(np.float32)[0])
        status = torch.full((n,), 0xEE, dtype=torch.uint8, device="cuda")
        _, st = rt.run(kid, nc, dev(rt, A), n, M=M, N=N, K=K, aux=dev(rt, B), flags=1,
                       plan=cb.FaultPlan(mode=cb.PLAN_TABLE, table=table), status=status)
        s = status.cpu().numpy()
        if nc == 1:
            assert not s.any()
        else:
            assert (s == want).all(), (nc, np.flatnonzero(s != want)[:10])
            assert 0 < int(s.sum()) == (st.errors_corrected if nc == 3 else st.dwc_detected)
            if kernel == "gemm":
                assert st.injected > int(s.sum())                  # the sign flips of +0.0 were injected and not counted


# ------------------------------------------------------------------------------------------ limb kernel: s32 accumulators wrap
def _limb_operands(M, N, K, kind, seed):
    from oracle import pyoracle as po
    if kind == "ones":
        return np.full(M * K, 0xFFFFFFFF, dtype=np.uint32), np.full(K * N, 0xFFFFFFFF, dtype=np.uint32)
    w = po.fill_philox(M * K + K * N, 0, seed) | np.uint32(0xC0C0C0C0)     # every limb >= 192
    return w[: M * K].copy(), w[M * K:].copy()


@pytest.mark.gpu
@pytest.mark.parametrize("K", [8320, 16640, 32768])      # S3 = 4*255^2*K passes 2^31 (K > 8256) and 2^32 (K > 16512)
@pytest.mark.parametrize("kind", ["ones", "high_limbs"])
def test_mm_limb_accumulators_wrap_past_2_31(rt, K, kind, monkeypatch):
    import torch
    import coast_b200 as cb
    for nc in (1, 2, 3):
        M, N = (128, 64) if nc == 1 else (128, 128)
        A, B = _limb_operands(M, N, K, kind, seed=K + nc)
        dA, dB = dev(rt, A), dev(rt, B)
        if kind == "ones":
            want = torch.full((M, N), K, dtype=torch.int64, device="cuda")
        else:
            want = mm_u32_ref(dA.view(M, K), dB.view(K, N))
        for path in ("tc", "tiled") if N % 128 == 0 else ("tc",):
            monkeypatch.setenv("COAST_MM_PATH", path)
            out = torch.full((M * N,), POISON, dtype=torch.int32, device="cuda")
            _, st = rt.run(cb.K_MM_U32, nc, dA, M * N, M=M, N=N, K=K, aux=dB, flags=3, out=out)
            assert torch.equal(out.view(M, N).to(torch.int64) & 0xFFFFFFFF, want), (nc, path)
            assert st.errors_corrected == 0 and st.dwc_detected == 0


@pytest.mark.gpu
@pytest.mark.parametrize("nc", [2, 3])
def test_mm_limb_faults_at_late_k_steps_past_2_31(rt, oracle, nc, monkeypatch):
    """faults after k-step 8192 of K = 16640: the epilogue re-sums `part` over more than 8192 k-steps, and every S_d of
    every replica has wrapped; outputs and counters equal the oracle's"""
    monkeypatch.delenv("COAST_MM_PATH", raising=False)
    M, N, K = 128, 64, 16640
    n = M * N
    A, B = _limb_operands(M, N, K, "high_limbs", seed=5)
    rng = np.random.default_rng(nc)
    tab = np.zeros(n, dtype=np.uint32)
    reps = rng.integers(0, 3, size=200)
    for u, r in zip(rng.choice(n, size=200, replace=False), reps):
        tab[u] = oracle.fault_entry(int(r), int(rng.integers(8192, K)), int(rng.integers(0, 32)))
    _, st = both(rt, oracle, oracle.K_MM_U32, nc, A, n, M=M, N=N, K=K, aux=B, flags=3, table=tab)
    assert st["injected"] == int((reps < nc).sum()) == (st["errors_corrected"] if nc == 3 else st["dwc_detected"])
    plan_kw = dict(seed=40 + nc, p=0.03)
    oplan = oracle.make_plan(oracle.PLAN_BERNOULLI, **plan_kw)
    late = [f for f in (oracle.fault_for_unit(oplan, oracle.K_MM_U32, nc, 0, K, u) for u in range(n)) if f and f[1] >= 8192]
    assert len(late) > 50
    both(rt, oracle, oracle.K_MM_U32, nc, A, n, M=M, N=N, K=K, aux=B, flags=3, plan_kw=plan_kw)


# ------------------------------------------------------------------------------------------ limb kernel: multi-wave grids
@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", [(1152, 1024, 384), (4096, 4096, 4096)])
def test_mm_limb_kernel_multi_wave_every_element(rt, M, N, K, monkeypatch):
    """1152 x 1024 x 384: 288 tiles at NC = 3 on 132 SMs and an odd number of k-blocks on the 2-stage ring; 4096^3: BASELINE
    size.  Every element of every replica count equals mm_u32_ref, for the tensor-core kernel and the CUDA-core tiled kernel."""
    import torch
    import coast_b200 as cb
    A = torch.empty(M * K, dtype=torch.int32, device="cuda")
    B = torch.empty(K * N, dtype=torch.int32, device="cuda")
    rt.fill_philox(A, seed=K + 1)
    rt.fill_philox(B, seed=K + 2)
    want = mm_u32_ref(A.view(M, K), B.view(K, N))
    for path, nc in [(p, nc) for p in ("tc", "tiled") for nc in (1, 2, 3)]:
        monkeypatch.setenv("COAST_MM_PATH", path)
        out = torch.full((M * N,), POISON, dtype=torch.int32, device="cuda")
        _, st = rt.run(cb.K_MM_U32, nc, A, M * N, M=M, N=N, K=K, aux=B, flags=3, out=out)
        assert torch.equal(out.view(M, N).to(torch.int64) & 0xFFFFFFFF, want), (path, nc)
        assert st.errors_corrected == 0 and st.dwc_detected == 0
