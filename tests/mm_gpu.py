"""What the GPU matmul tests share: the environment switches they clear, the counters they compare, the output poison, and
one record per GEMM operand type (BF16, FP8) with its device encoding, operand builders and CPU reference, so that one test
body runs either type.  numpy has neither type: operands are their bit patterns on the host (uint16, uint8)."""
import numpy as np

import gemm_bf16_ref
import gemm_fp8_ref
from coast_b200.runtime import K_GEMM_BF16, K_GEMM_FP8, MM_B_TRANSPOSED

# every switch of the matmul plans and of the host call: a test starts with none of them set
KNOBS = ("COAST_GEMM_PAIR", "COAST_GEMM_GROUP_M", "COAST_GEMM_L2_HINTS", "COAST_GEMM_TAIL_SPLIT", "COAST_MM_PATH",
         "COAST_HOST_CHUNK_BYTES", "COAST_HOST_PATH")
STAT_KEYS = ("errors_corrected", "dwc_detected", "syncs", "injected", "first_fault_unit")
POISON = 0x7FC00BAD                      # initial content of matmul output buffers, a NaN no kernel writes: a skipped element fails


def env(monkeypatch, **kv):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in kv.items():
        monkeypatch.setenv(k, v)


def no_stats():
    return dict(errors_corrected=0, dwc_detected=0, syncs=0, injected=0, first_fault_unit=2 ** 64 - 1)


def add_stats(tot, s):
    """adds the counters of one launch (a stats dict) to tot, as one launch over both would count them"""
    for k in STAT_KEYS[:4]:
        tot[k] += s[k]
    tot["first_fault_unit"] = min(tot["first_fault_unit"], s["first_fault_unit"])
    return tot


def transposed(B, K):
    """the products' B (P K x N, stacked) as their B^T (P N x K, stacked)"""
    N = B.shape[1]
    return np.ascontiguousarray(B.reshape(-1, K, N).transpose(0, 2, 1).reshape(-1, K))


class Bf16:
    name, kernel, nan, neg_zero = "bf16", K_GEMM_BF16, 0x7FC0, 0x8000
    ref, bits, value = gemm_bf16_ref, staticmethod(gemm_bf16_ref.bits), staticmethod(gemm_bf16_ref.value)

    @staticmethod
    def tensor(x):
        """bit patterns as a host tensor the runtime takes"""
        import torch
        return torch.from_numpy(np.ascontiguousarray(x).view(np.int16)).view(torch.bfloat16)

    @staticmethod
    def int_operands(M, N, K, seed, amax=8):
        """integers in [-amax, amax] with K amax^2 < 2^24: every partial sum is an exact fp32 integer"""
        rng = np.random.default_rng(seed)
        assert amax <= 256 and amax * amax * K < 2 ** 24
        A = rng.integers(-amax, amax + 1, size=(M, K)).astype(np.float32)
        B = rng.integers(-amax, amax + 1, size=(K, N)).astype(np.float32)
        return gemm_bf16_ref.bits(A), gemm_bf16_ref.bits(B)

    @staticmethod
    def uniform_operands(M, N, K, seed):
        """uniform(-1, 1) rounded to bfloat16 by torch (round to nearest even)"""
        import torch
        g = torch.Generator().manual_seed(seed)

        def one(r, c):
            return (torch.rand(r, c, generator=g) * 2 - 1).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16).copy()
        return one(M, K), one(K, N)

    @classmethod
    def stacked_operands(cls, rows, N, K, P, seed):
        """rows x K of A and P stacked K x N matrices B, integer-valued"""
        A, B = cls.int_operands(rows, N, P * K, seed)
        return A[:, :K].copy(), B

    @staticmethod
    def bound(A, B):
        """|C - C64| allowed per element on general operands: the products are exact, the fp32 sum is the tensor core's; the
        absolute bound 2e-6 K that GEMM_TF32 is held to"""
        return 2e-6 * A.shape[1]


class Fp8:
    name, kernel, nan, neg_zero = "fp8", K_GEMM_FP8, 0x7F, 0x80
    ref, bits, value = gemm_fp8_ref, staticmethod(gemm_fp8_ref.bits), staticmethod(gemm_fp8_ref.value)

    @staticmethod
    def tensor(x):
        """bit patterns as a host tensor the runtime takes"""
        import torch
        return torch.from_numpy(np.ascontiguousarray(x)).view(torch.float8_e4m3fn)

    @staticmethod
    def int_operands(M, N, K, seed, amax=1):
        return gemm_fp8_ref.int_operands(np.random.default_rng(seed), M, N, K, amax)

    @staticmethod
    def uniform_operands(M, N, K, seed):
        """uniform(-1, 1) rounded to E4M3 by torch (round to nearest even)"""
        import torch
        g = torch.Generator().manual_seed(seed)

        def one(r, c):
            return (torch.rand(r, c, generator=g) * 2 - 1).to(torch.float8_e4m3fn).view(torch.uint8).numpy().copy()
        return one(M, K), one(K, N)

    @staticmethod
    def stacked_operands(rows, N, K, P, seed):
        """rows x K of A and P stacked K x N matrices B, integers in [-1, 1]: each product stays in the exact domain"""
        rng = np.random.default_rng(seed)
        A, _ = gemm_fp8_ref.int_operands(rng, rows, N, K, 1)
        return A, np.concatenate([gemm_fp8_ref.int_operands(rng, 1, N, K, 1)[1] for _ in range(P)])

    @staticmethod
    def bound(A, B):
        """|C - C64| allowed per element on general operands: 2^-10 sum_k |a_ik b_kj|.  Measured at most 3.7e-4 (2^-11.4) of
        it on uniform(-1, 1) operands on an H100 up to K = 8192 (DESIGN.md §6): the bound leaves a factor of 2.6"""
        return 2.0 ** -10 * (np.abs(gemm_fp8_ref.value(A)).astype(np.float64) @ np.abs(gemm_fp8_ref.value(B)).astype(np.float64))


def dev(t, x):
    return t.tensor(x).cuda()


def gpu(rt, t, nc, A, B, *, flags=3, plan=None, table=None, unit_base=0, status=None, mode=0, M=None, n=None, rows=None, out=None,
        bt=False):
    """A: (rows x K), B: (P K x N) bit patterns of t -> (C bits as uint32, flat; stats dict); bt: launch with B^T"""
    import torch
    import coast_b200 as cb
    K, N = A.shape[1], B.shape[1]
    M = A.shape[0] if M is None else M
    n = A.shape[0] * N if n is None else n
    if table is not None:
        plan = cb.FaultPlan(mode=cb.PLAN_TABLE, table=torch.from_numpy(table.view(np.int32).copy()).cuda())
    if out is None:
        out = torch.full((A.shape[0] * N,), float("nan"), dtype=torch.float32, device="cuda")    # poison: every element is written
    aux = dev(t, transposed(B, K)) if bt else dev(t, B)
    _, st = rt.run(t.kernel, nc, dev(t, A), n, M=M, N=N, K=K, aux=aux, flags=flags, plan=plan, unit_base=unit_base,
                   status=status, mode=mode | (MM_B_TRANSPOSED if bt else 0), rows=rows, out=out)
    return out.cpu().numpy().view(np.uint32), st.as_dict()


def cpu(oracle, t, nc, A, B, *, flags=3, plan_kw=None, table=None, unit_base=0):
    plan = None
    if table is not None:
        plan = oracle.make_plan(oracle.PLAN_TABLE, table=table)
    elif plan_kw:
        plan = oracle.make_plan(oracle.PLAN_BERNOULLI, **plan_kw)
    return t.ref.run(oracle, nc, A, B, flags=flags, plan=plan, unit_base=unit_base, threads=8)


def both(rt, oracle, t, nc, A, B, *, flags=3, plan_kw=None, table=None, unit_base=0, bt=False):
    import coast_b200 as cb
    plan = cb.FaultPlan(mode=cb.PLAN_BERNOULLI, **plan_kw) if plan_kw else None
    g, gs = gpu(rt, t, nc, A, B, flags=flags, plan=plan, table=table, unit_base=unit_base, bt=bt)
    o, os_ = cpu(oracle, t, nc, A, B, flags=flags, plan_kw=plan_kw, table=table, unit_base=unit_base)
    assert (g == o).all(), (t.name, nc, flags, np.flatnonzero(g != o)[:8])
    assert {k: gs[k] for k in STAT_KEYS} == {k: os_[k] for k in STAT_KEYS}
    return g, gs
