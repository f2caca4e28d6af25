"""ctypes mirror of include/coast_rt.h.

Error behaviour mirrors the C ABI: every call that fails raises :class:`CoastError` carrying
``coast_last_error()``.  There is no CPU fallback anywhere in this module -- without the CUDA
driver ``Runtime()`` raises (COAST_ERR_NO_DRIVER), loudly.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass

HERE = os.path.dirname(os.path.abspath(__file__))

K_CRC16, K_SHA256, K_AES128, K_MM_U32, K_GEMM_TF32, K_QSORT, K_CHSTONE_SHA, K_CHSTONE_AES, K_GEMM_BF16 = range(9)
K_GEMM_FP8 = 10                              # FP8 E4M3 operands, fp32 out; id 9 is unassigned
K_GEMM_I8 = 12                               # int8 operands, int32 out, exact mod 2^32, integer vote; id 11 is unassigned
K_GEMM_F16 = 14                              # float16 operands, fp32 out (MM_OUT_F16: float16); GEMM_BF16's layout; id 13 is unassigned
F_COUNT_ERRORS, F_COUNT_SYNCS, F_NO_MEM_REPLICATION = 0x1, 0x2, 0x4
F_INTERLEAVE, F_SEGMENT, F_VERBOSE, F_MAJORITY_VOTER = 0x8, 0x10, 0x20, 0x100
F_STORE_DATA_SYNC, F_NO_STORE_DATA_SYNC, F_NO_LOAD_SYNC, F_NO_STORE_ADDR_SYNC = 0x200, 0x400, 0x800, 0x1000
PLAN_NONE, PLAN_BERNOULLI, PLAN_TABLE = 0, 1, 2
AES_DECRYPT, AES_KEY_PER_UNIT, AES_KEY_WRITEBACK = 1, 2, 4
UNIT_OFFSETS = COAST_UNIT_OFFSETS = 0x10000  # ragged CRC16 / SHA256 / QSORT batches: aux = n_units + 1 u64 byte offsets into inp
MM_BATCHED = COAST_MM_BATCHED = 0x20000      # batched MM_U32 / GEMM_TF32 / GEMM_BF16 / GEMM_FP8 / GEMM_I8 / GEMM_F16: n_units = batch*M*N, inp / aux / out hold batch A / B / C
MM_GROUPED = COAST_MM_GROUPED = 0x40000      # grouped MM_U32 / GEMM_TF32 / GEMM_BF16 / GEMM_FP8 / GEMM_I8 / GEMM_F16: M = G products, rows = G + 1 u64 row offsets, n_units = R*N
MM_B_TRANSPOSED = COAST_MM_B_TRANSPOSED = 0x80000  # MM_U32 / GEMM_TF32 / GEMM_BF16 / GEMM_FP8 / GEMM_I8 / GEMM_F16: aux holds B^T, N x K per product (nn.Linear.weight)
MM_SCALE_TENSOR = COAST_MM_SCALE_TENSOR = 0x100000    # GEMM_FP8: one fp32 scale of A and one of B, applied by every replica before the vote
MM_SCALE_ROWWISE = COAST_MM_SCALE_ROWWISE = 0x200000  # GEMM_FP8: one fp32 scale per row of the stacked A and per column of each product's B
MM_OUT_BF16 = COAST_MM_OUT_BF16 = 0x400000            # GEMM_BF16 / GEMM_FP8: C is bfloat16, every replica rounds before the vote
MM_OUT_F16 = COAST_MM_OUT_F16 = 0x800000              # GEMM_F16: C is float16, every replica rounds before the vote
NO_FAULT_UNIT = 0xFFFFFFFFFFFFFFFF
ERR_NO_DRIVER, ERR_NOT_INIT, ERR_BAD_ARG, ERR_UNSUPPORTED, ERR_BUSY = -100001, -100002, -100003, -100004, -100005

OUT_BYTES = {K_CRC16: 2, K_SHA256: 32, K_AES128: 16, K_MM_U32: 4, K_GEMM_TF32: 4, K_CHSTONE_SHA: 20, K_CHSTONE_AES: 64, K_GEMM_BF16: 4,
             K_GEMM_FP8: 4, K_GEMM_I8: 4, K_GEMM_F16: 4}
MM_ELEM_BYTES = {K_GEMM_BF16: 2, K_GEMM_FP8: 1, K_GEMM_I8: 1, K_GEMM_F16: 2}   # bytes per A and B element of the matmuls; 4 for MM_U32 and GEMM_TF32


def out_bytes(kernel: int, unit_bytes: int = 0, mode: int = 0) -> int:
    """bytes of output per unit; with MM_OUT_BF16, GEMM_BF16 and GEMM_FP8 write 2-byte bfloat16 C elements, and with
    MM_OUT_F16 GEMM_F16 writes 2-byte float16 ones"""
    if mode & MM_OUT_BF16 and kernel in (K_GEMM_BF16, K_GEMM_FP8) or mode & MM_OUT_F16 and kernel == K_GEMM_F16:
        return 2
    return unit_bytes if kernel == K_QSORT else OUT_BYTES[kernel]


class CoastError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"coast_rt error {code}: {msg}")
        self.code = code


class _Plan(C.Structure):
    _fields_ = [("mode", C.c_uint32), ("seed_lo", C.c_uint32), ("seed_hi", C.c_uint32), ("threshold", C.c_uint32),
                ("d_table", C.c_void_p)]


class LaunchDesc(C.Structure):
    _fields_ = [("kernel", C.c_uint32), ("num_clones", C.c_uint32), ("flags", C.c_uint32), ("mode", C.c_uint32),
                ("n_units", C.c_uint64), ("unit_base", C.c_uint64),
                ("unit_bytes", C.c_uint32), ("M", C.c_uint32), ("N", C.c_uint32), ("K", C.c_uint32),
                ("d_in", C.c_void_p), ("d_out", C.c_void_p), ("d_aux", C.c_void_p),
                ("key", C.c_uint8 * 16), ("plan", C.POINTER(_Plan)), ("d_status", C.c_void_p), ("d_rows", C.c_void_p),
                ("d_scale_a", C.c_void_p), ("d_scale_b", C.c_void_p)]


class _Stats(C.Structure):
    _fields_ = [("errors_corrected", C.c_uint64), ("dwc_detected", C.c_uint64), ("syncs", C.c_uint64),
                ("injected", C.c_uint64), ("first_fault_unit", C.c_uint64)]


@dataclass
class Stats:
    errors_corrected: int = 0
    dwc_detected: int = 0
    syncs: int = 0
    injected: int = 0
    first_fault_unit: int = NO_FAULT_UNIT

    def as_dict(self):
        return dict(errors_corrected=self.errors_corrected, dwc_detected=self.dwc_detected, syncs=self.syncs,
                    injected=self.injected, first_fault_unit=self.first_fault_unit)


@dataclass
class FaultPlan:
    """On-device single-bit-flip plan (include/coast_rt.h, "Fault plan")."""
    mode: int = PLAN_NONE
    seed: int = 0
    p: float = 0.0
    threshold: int | None = None
    table: object = None  # torch.uint32/int32 CUDA tensor, one entry per local unit (PLAN_TABLE)

    def to_c(self) -> _Plan:
        pl = _Plan()
        pl.mode = self.mode
        pl.seed_lo = self.seed & 0xFFFFFFFF
        pl.seed_hi = (self.seed >> 32) & 0xFFFFFFFF
        thr = self.threshold if self.threshold is not None else min(int(self.p * 2 ** 32), 0xFFFFFFFF)
        pl.threshold = thr
        pl.d_table = self.table.data_ptr() if self.table is not None else None
        return pl


def fault_entry(replica: int, site: int, bit: int) -> int:
    return 0x80000000 | ((replica & 3) << 29) | ((site & 0xFFFFFF) << 5) | (bit & 31)


def lib_path() -> str:
    return os.path.join(HERE, "libcoast_rt.so")


_LIB = None

EXPORTS = [
    "coast_init", "coast_numa_node", "coast_shutdown", "coast_last_error", "coast_version", "coast_parse_opt_passes", "coast_flags_honoured", "coast_launch",
    "coast_sync", "coast_sync_noabort", "coast_stats_snapshot", "coast_stats_reset", "coast_counters_export", "coast_counters_attach",
    "coast_counters_detach", "coast_sm_count", "coast_clock_probe", "coast_fault_sites",
    "coast_fault_site_bits", "coast_out_bytes_per_unit", "coast_out_bytes", "coast_votes_per_unit", "coast_malloc", "coast_free",
    "coast_memcpy_h2d", "coast_memcpy_d2h", "coast_memset", "coast_host_alloc", "coast_host_free",
    "coast_stream_create", "coast_stream_destroy", "coast_stream_sync", "coast_fill_philox", "coast_run_host",
    "coast_run_host_noabort", "coast_last_host_path",
    "coast_set_opt_passes", "coast_xmr_crc16", "coast_xmr_sha256_hash", "coast_xmr_aes_enc_dec",
    "coast_xmr_matrix_multiply_u32", "coast_xmr_chstone_sha_stream", "coast_xmr_chstone_aes", "TMR_ERROR_CNT", "__SYNC_COUNT", "FAULT_DETECTED_DWC",
]


def load_library():
    """dlopen the in-tree libcoast_rt.so; raises if it has not been built (no silent fallback)."""
    global _LIB
    if _LIB is None:
        path = lib_path()
        if not os.path.exists(path):
            raise CoastError(ERR_NOT_INIT, f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                                           "(or make -C coast_b200/csrc); there is no CPU fallback")
        L = C.CDLL(path)
        L.coast_last_error.restype = C.c_char_p
        L.coast_version.restype = C.c_char_p
        L.coast_last_host_path.restype = C.c_char_p
        L.coast_init.argtypes = [C.c_int]
        L.coast_parse_opt_passes.argtypes = [C.c_char_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        L.coast_set_opt_passes.argtypes = [C.c_char_p]
        L.coast_flags_honoured.argtypes = [C.c_uint32] * 3
        L.coast_flags_honoured.restype = C.c_uint32
        L.coast_launch.argtypes = [C.POINTER(LaunchDesc), C.c_void_p]
        L.coast_run_host.argtypes = [C.POINTER(LaunchDesc), C.POINTER(_Stats)]
        L.coast_run_host_noabort.argtypes = [C.POINTER(LaunchDesc), C.POINTER(_Stats)]
        L.coast_sync.argtypes = [C.c_void_p, C.POINTER(_Stats)]
        L.coast_sync_noabort.argtypes = [C.c_void_p, C.POINTER(_Stats)]
        L.coast_stats_snapshot.argtypes = [C.c_void_p, C.c_void_p]
        L.coast_stats_reset.argtypes = [C.c_void_p]
        L.coast_counters_export.argtypes = [C.c_void_p]
        L.coast_clock_probe.argtypes = [C.c_void_p, C.c_void_p]
        L.coast_counters_attach.argtypes = [C.c_void_p]
        L.coast_fault_sites.argtypes = [C.c_uint32] * 3
        L.coast_fault_sites.restype = C.c_uint32
        L.coast_fault_site_bits.argtypes = [C.c_uint32] * 4
        L.coast_fault_site_bits.restype = C.c_uint32
        L.coast_out_bytes_per_unit.argtypes = [C.c_uint32]
        L.coast_out_bytes_per_unit.restype = C.c_uint32
        L.coast_votes_per_unit.argtypes = [C.c_uint32]
        L.coast_votes_per_unit.restype = C.c_uint32
        L.coast_fill_philox.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint32, C.c_void_p]
        L.coast_xmr_crc16.argtypes = [C.c_char_p, C.c_ubyte]
        L.coast_xmr_crc16.restype = C.c_ushort
        _LIB = L
    return _LIB


def parse_opt_passes(opt_passes: str) -> tuple[int, int]:
    """OPT_PASSES string of a reference test Makefile -> (num_clones, flags)."""
    L = load_library()
    nc, fl = C.c_uint32(), C.c_uint32()
    rc = L.coast_parse_opt_passes(opt_passes.encode(), C.byref(nc), C.byref(fl))
    if rc:
        raise CoastError(rc, L.coast_last_error().decode())
    return nc.value, fl.value


class Runtime:
    """One process <-> one GPU.  Device memory and streams come from torch (plumbing)."""

    def __init__(self, device: int = 0):
        self.L = load_library()
        self.device = device
        self._check(self.L.coast_init(device))
        import torch  # after coast_init so a missing driver is reported by OUR library, loudly
        self.torch = torch
        torch.cuda.set_device(device)

    def _check(self, rc: int):
        if rc != 0:
            raise CoastError(rc, self.L.coast_last_error().decode())

    # -- low level -------------------------------------------------------------------------
    def stream_handle(self, stream=None) -> int:
        s = stream if stream is not None else self.torch.cuda.current_stream()
        return s.cuda_stream

    def make_desc(self, kernel, num_clones, d_in, d_out, n_units, *, flags=0, mode=0, unit_bytes=0, M=0, N=0, K=0,
                  d_aux=None, key: bytes | None = None, plan: FaultPlan | None = None, unit_base=0, d_status=None, d_rows=None,
                  scale_a=None, scale_b=None):
        d = LaunchDesc()
        d.kernel, d.num_clones, d.flags, d.mode = kernel, num_clones, flags, mode
        d.n_units, d.unit_base, d.unit_bytes = n_units, unit_base, unit_bytes
        d.M, d.N, d.K = M, N, K
        d.d_in = d_in.data_ptr() if hasattr(d_in, "data_ptr") else d_in
        d.d_out = d_out.data_ptr() if hasattr(d_out, "data_ptr") else d_out
        if d_aux is not None:
            d.d_aux = d_aux.data_ptr() if hasattr(d_aux, "data_ptr") else d_aux
        if key is not None:
            d.key = (C.c_uint8 * 16)(*key)
        if d_status is not None:
            d.d_status = d_status.data_ptr() if hasattr(d_status, "data_ptr") else d_status
        if d_rows is not None:
            d.d_rows = d_rows.data_ptr() if hasattr(d_rows, "data_ptr") else d_rows
        if scale_a is not None:
            d.d_scale_a = scale_a.data_ptr() if hasattr(scale_a, "data_ptr") else scale_a
        if scale_b is not None:
            d.d_scale_b = scale_b.data_ptr() if hasattr(scale_b, "data_ptr") else scale_b
        keep = None
        if plan is not None and plan.mode != PLAN_NONE:
            keep = plan.to_c()
            d.plan = C.pointer(keep)
        d._keep = (keep, d_in, d_out, d_aux, d_rows, scale_a, scale_b)
        return d

    def launch(self, desc: LaunchDesc, stream=None):
        self._check(self.L.coast_launch(C.byref(desc), self.stream_handle(stream)))

    def sync(self, stream=None, abort_on_dwc: bool = False) -> Stats:
        st = _Stats()
        fn = self.L.coast_sync if abort_on_dwc else self.L.coast_sync_noabort
        self._check(fn(self.stream_handle(stream), C.byref(st)))
        return Stats(st.errors_corrected, st.dwc_detected, st.syncs, st.injected, st.first_fault_unit)

    def stats_snapshot(self, d_out, stream=None):
        self._check(self.L.coast_stats_snapshot(self.stream_handle(stream), d_out.data_ptr()))

    def sm_count(self) -> int:
        return int(self.L.coast_sm_count())

    def clock_probe(self, d_out, stream=None):
        """d_out: int64 CUDA tensor of 2 * sm_count() elements -> {clock64, globaltimer ns} per SM"""
        self._check(self.L.coast_clock_probe(C.c_void_p(d_out.data_ptr()), self.stream_handle(stream)))

    # multi-GPU fold of the counters over NVLink peer memory (include/coast_rt.h: coast_counters_export / _attach / _detach)
    def counters_export(self) -> bytes:
        buf = C.create_string_buffer(64)
        self._check(self.L.coast_counters_export(buf))
        return buf.raw

    def counters_attach(self, handle: bytes):
        assert len(handle) == 64
        self._check(self.L.coast_counters_attach(C.create_string_buffer(handle, 64)))

    def counters_detach(self):
        self._check(self.L.coast_counters_detach())

    def stats_reset(self, stream=None):
        self._check(self.L.coast_stats_reset(self.stream_handle(stream)))

    def fill_philox(self, dst, seed: int, word_base: int = 0, stream=None):
        """dst: any CUDA tensor whose byte size is a multiple of 4."""
        nbytes = dst.numel() * dst.element_size()
        assert nbytes % 4 == 0
        self._check(self.L.coast_fill_philox(dst.data_ptr(), nbytes // 4, word_base, seed, self.stream_handle(stream)))

    def fault_sites(self, kernel, unit_bytes=0, K=0) -> int:
        return int(self.L.coast_fault_sites(kernel, unit_bytes, K))

    def fault_site_bits(self, kernel, unit_bytes, K, site) -> int:
        return int(self.L.coast_fault_site_bits(kernel, unit_bytes, K, site))

    @property
    def numa_node(self) -> int:
        return int(self.L.coast_numa_node())

    @property
    def last_host_path(self) -> str:
        return self.L.coast_last_host_path().decode()

    @property
    def tmr_error_cnt(self) -> int:
        return C.c_uint32.in_dll(self.L, "TMR_ERROR_CNT").value

    @property
    def sync_count(self) -> int:
        return C.c_uint64.in_dll(self.L, "__SYNC_COUNT").value

    # -- convenience: device tensors in, device tensor + Stats out ----------------------------
    def run(self, kernel, num_clones, inp, n_units, *, flags=0, mode=0, unit_bytes=0, M=0, N=0, K=0, aux=None,
            key: bytes | None = None, plan: FaultPlan | None = None, unit_base=0, out=None, stream=None, status=None, rows=None,
            scale_a=None, scale_b=None):
        """rows: with MM_GROUPED, the CUDA int64/uint64 tensor of M + 1 row offsets (M = the product count).
        K_GEMM_BF16: inp and aux are torch.bfloat16 tensors (or their uint16 / int16 views); the result is fp32 like K_GEMM_TF32's.
        K_GEMM_FP8: inp and aux are torch.float8_e4m3fn tensors (or their uint8 views); the result is fp32.  With MM_SCALE_TENSOR
        scale_a and scale_b are one-element float32 CUDA tensors; with MM_SCALE_ROWWISE scale_a holds one per stacked row of A and
        scale_b one per column of each product's B.  With MM_OUT_BF16 (K_GEMM_BF16, K_GEMM_FP8) the result is bfloat16 bytes, two
        per element: view it as torch.bfloat16.
        K_GEMM_I8: inp and aux are torch.int8 tensors (or their uint8 views); the result is int32, 4 bytes per element: view it as
        torch.int32.  It takes no scales and no MM_OUT_BF16.
        K_GEMM_F16: inp and aux are torch.float16 tensors (or their int16 / uint16 views); the result is fp32, or with MM_OUT_F16
        float16 bytes, two per element: view it as torch.float16.  It takes no scales and no MM_OUT_BF16 (the library refuses them)."""
        torch = self.torch
        self._check_i8(kernel, mode, scale_a, scale_b)
        if mode & MM_GROUPED:
            self._check_rows(rows, M, N, n_units, inp, K, out, MM_ELEM_BYTES.get(kernel, 4), out_bytes(kernel, unit_bytes, mode))
        if mode & (MM_SCALE_TENSOR | MM_SCALE_ROWWISE):
            self._check_scales(scale_a, scale_b, mode, M, N, n_units, rows)
        ragged_qsort = bool(mode & UNIT_OFFSETS) and kernel == K_QSORT
        if out is None and ragged_qsort:       # the arrays are sorted into the bytes they came from: out mirrors inp
            out = torch.zeros(inp.numel() * inp.element_size(), dtype=torch.uint8, device=f"cuda:{self.device}")
        if mode & UNIT_OFFSETS:
            self._check_offsets(inp, aux, n_units, unit_bytes, kernel=kernel, out=out)
        if out is None and mode & MM_GROUPED:   # C rows at ro[g]: out covers rows [0, ro[G]), like inp
            R_end = int(rows[: M + 1].view(torch.int64)[-1])
            out = torch.empty(R_end * N * out_bytes(kernel, unit_bytes, mode), dtype=torch.uint8, device=f"cuda:{self.device}")
        if out is None:
            out = torch.empty(n_units * out_bytes(kernel, unit_bytes, mode), dtype=torch.uint8, device=f"cuda:{self.device}")
        d = self.make_desc(kernel, num_clones, inp, out, n_units, flags=flags, mode=mode, unit_bytes=unit_bytes,
                           M=M, N=N, K=K, d_aux=aux, key=key, plan=plan, unit_base=unit_base, d_status=status, d_rows=rows,
                           scale_a=scale_a, scale_b=scale_b)
        self.launch(d, stream)
        return out, self.sync(stream)

    @staticmethod
    def _check_i8(kernel, mode, scale_a, scale_b):
        """K_GEMM_I8 computes the exact int32 product only: scales and bfloat16 output belong to GEMM_FP8 (and GEMM_BF16)"""
        if kernel == K_GEMM_I8 and (mode & (MM_SCALE_TENSOR | MM_SCALE_ROWWISE | MM_OUT_BF16) or scale_a is not None
                                    or scale_b is not None):
            raise CoastError(ERR_BAD_ARG, "K_GEMM_I8: no scales and no MM_OUT_BF16; its C is the exact int32 product")

    def _check_rows(self, rows, G, N, n_units, inp, K, out, esize=4, out_esize=4):
        """A grouped launch's device row offsets (int64 or uint64 tensor, G + 1 entries): they never decrease and span exactly
        n_units / N rows, which lie within inp (K elements of esize bytes per row) and out (N elements of out_esize bytes per row).  The kernels only clamp; this catches a bad table
        before it runs."""
        torch = self.torch
        if rows is None or not hasattr(rows, "data_ptr") or rows.dtype not in (torch.int64, torch.uint64) or not rows.is_cuda:
            raise CoastError(ERR_BAD_ARG, "MM_GROUPED: rows must be a CUDA int64/uint64 tensor of M + 1 row offsets")
        if G < 1 or rows.numel() < G + 1 or not rows.is_contiguous():
            raise CoastError(ERR_BAD_ARG, f"MM_GROUPED: rows holds {rows.numel()} offsets, a contiguous M + 1 = {G + 1} are needed")
        if N < 1 or n_units % N:
            raise CoastError(ERR_BAD_ARG, f"MM_GROUPED: n_units ({n_units}) must be a multiple of N ({N})")
        ro = rows[: G + 1].view(torch.int64)
        R = n_units // N
        in_rows = inp.numel() * inp.element_size() // (esize * K) if K else 0
        out_rows = out.numel() * out.element_size() // (out_esize * N) if out is not None else None
        bad = torch.stack([(ro < 0).any(), (ro[1:] < ro[:-1]).any(), ro[-1] - ro[0] != R, ro[-1] > in_rows]).tolist()
        if any(bad) or (out_rows is not None and int(ro[-1]) > out_rows):
            raise CoastError(ERR_BAD_ARG, f"MM_GROUPED: row offsets must not decrease, must span n_units / N = {R} rows and end "
                                          "within inp and out")

    def _check_scales(self, scale_a, scale_b, mode, M, N, n_units, rows):
        """A scaled launch's scales: contiguous float32 CUDA tensors, one element each (MM_SCALE_TENSOR), or (MM_SCALE_ROWWISE) one
        per stacked row of A -- M, batch*M, or for groups at least ro[G] since row r of inp uses scale_a[r] -- and one per column
        of each product's B, P*N.  The library reads what the shape says; this catches a short vector before it runs."""
        torch = self.torch
        for name, s in (("scale_a", scale_a), ("scale_b", scale_b)):
            if s is None or not hasattr(s, "data_ptr") or s.dtype != torch.float32 or not s.is_cuda or not s.is_contiguous():
                raise CoastError(ERR_BAD_ARG, f"MM_SCALE: {name} must be a contiguous float32 CUDA tensor")
        if not mode & MM_SCALE_ROWWISE:
            if scale_a.numel() != 1 or scale_b.numel() != 1:
                raise CoastError(ERR_BAD_ARG, "MM_SCALE_TENSOR: scale_a and scale_b hold one float each")
            return
        if N < 1 or n_units % N:
            raise CoastError(ERR_BAD_ARG, f"MM_SCALE_ROWWISE: n_units ({n_units}) must be a multiple of N ({N})")
        if mode & MM_GROUPED:
            P, need_a = M, int(rows[: M + 1].view(torch.int64)[-1])
            ok_a = scale_a.numel() >= need_a
        else:
            P = n_units // (M * N) if M else 0
            need_a = n_units // N
            ok_a = scale_a.numel() == need_a
        if not ok_a or scale_b.numel() != P * N:
            raise CoastError(ERR_BAD_ARG, f"MM_SCALE_ROWWISE: scale_a holds {scale_a.numel()} floats and scale_b {scale_b.numel()}; "
                                          f"one per row of A ({'at least ' if mode & MM_GROUPED else ''}{need_a}) and one per "
                                          f"column of each B ({P * N}) are needed")

    def _check_offsets(self, inp, aux, n_units, unit_bytes, *, kernel=None, out=None):
        """A ragged batch's device offsets (int64 or uint64 tensor, n_units + 1 entries): they never decrease, no length
        exceeds unit_bytes and the last one lies within inp.  The kernels only clamp; this catches a bad table before it runs.
        QSORT (int32 arrays sorted into the same bytes of out): every offset is a multiple of 4, inp and out are 4-byte
        aligned and the last offset lies within out too."""
        torch = self.torch
        if aux is None or not hasattr(aux, "data_ptr") or aux.dtype not in (torch.int64, torch.uint64) or not aux.is_cuda:
            raise CoastError(ERR_BAD_ARG, "UNIT_OFFSETS: aux must be a CUDA int64/uint64 tensor of n_units + 1 byte offsets")
        if aux.numel() < n_units + 1 or not aux.is_contiguous():
            raise CoastError(ERR_BAD_ARG, f"UNIT_OFFSETS: aux holds {aux.numel()} offsets, a contiguous n_units + 1 = {n_units + 1} are needed")
        off = aux[: n_units + 1].view(torch.int64)
        lens = off[1:] - off[:-1]
        nbytes = inp.numel() * inp.element_size()
        bad = torch.stack([(off < 0).any(), (lens < 0).any(), (lens > unit_bytes).any(), off[-1] > nbytes]).tolist()
        if any(bad):
            raise CoastError(ERR_BAD_ARG, "UNIT_OFFSETS: offsets must not decrease, no length may exceed unit_bytes "
                                          f"({unit_bytes}) and the last offset must lie within inp ({nbytes} bytes)")
        if kernel == K_QSORT:
            if inp.data_ptr() % 4 or (out is not None and out.data_ptr() % 4):
                raise CoastError(ERR_BAD_ARG, "UNIT_OFFSETS: QSORT's inp and out must be 4-byte aligned")
            obytes = out.numel() * out.element_size() if out is not None else nbytes
            if bool(((off & 3) != 0).any()) or int(off[-1]) > obytes:
                raise CoastError(ERR_BAD_ARG, "UNIT_OFFSETS: QSORT offsets must be multiples of 4 (whole int32 elements) and the "
                                              f"last one must lie within out ({obytes} bytes)")

    # -- the reference-facing host call: HOST buffers, H2D + kernel + D2H inside ---------------
    def run_host(self, kernel, num_clones, h_in, h_out, n_units, *, flags=0, mode=0, unit_bytes=0, M=0, N=0, K=0,
                 h_aux=None, key: bytes | None = None, plan: FaultPlan | None = None, unit_base=0,
                 abort_on_dwc: bool = False, h_rows=None, scale_a=None, scale_b=None) -> Stats:
        """h_in/h_out/h_aux: CPU torch tensors or numpy arrays (pinned memory makes the copies async); scale_a / scale_b: the
        host float32 scales of a MM_SCALE_TENSOR or MM_SCALE_ROWWISE call.  With MM_OUT_BF16, h_out receives bfloat16 bytes, two
        per element.  K_GEMM_I8: int8 operands, h_out receives int32 elements; no scales and no MM_OUT_BF16.  K_GEMM_F16: float16
        operands (or their 16-bit integer views); with MM_OUT_F16, h_out receives float16 bytes, two per element."""
        self._check_i8(kernel, mode, scale_a, scale_b)

        def ptr(x):
            if x is None:
                return None
            return x.data_ptr() if hasattr(x, "data_ptr") else x.ctypes.data
        d = self.make_desc(kernel, num_clones, ptr(h_in), ptr(h_out), n_units, flags=flags, mode=mode,
                           unit_bytes=unit_bytes, M=M, N=N, K=K, d_aux=ptr(h_aux), key=key, plan=plan,
                           unit_base=unit_base, d_rows=ptr(h_rows), scale_a=ptr(scale_a), scale_b=ptr(scale_b))
        d._keep2 = (h_in, h_out, h_aux, h_rows, scale_a, scale_b)
        st = _Stats()
        fn = self.L.coast_run_host if abort_on_dwc else self.L.coast_run_host_noabort
        self._check(fn(C.byref(d), C.byref(st)))
        return Stats(st.errors_corrected, st.dwc_detected, st.syncs, st.injected, st.first_fault_unit)
