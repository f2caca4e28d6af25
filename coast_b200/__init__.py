"""coast_b200 -- H100-native redundant execution (TMR/DWC) behind the COAST annotation surface.

The product is the C-ABI library ``libcoast_rt.so`` (include/coast_rt.h): hand-written sm_90a
kernels in which every live value of a protected region is computed by 2 (DWC) or 3 (TMR)
replicas on adjacent lanes and voted at the sphere-of-replication exit.  This package is the
thin Python host mirror used by the tests and bench.py; PyTorch supplies device memory,
streams and ``torch.distributed`` -- plumbing only.
"""
from .runtime import (  # noqa: F401
    AES_DECRYPT, AES_KEY_PER_UNIT, AES_KEY_WRITEBACK, F_COUNT_ERRORS, F_COUNT_SYNCS, F_INTERLEAVE, F_MAJORITY_VOTER,
    F_NO_MEM_REPLICATION, F_SEGMENT, F_VERBOSE, K_AES128, K_CHSTONE_AES, K_CHSTONE_SHA, K_CRC16, K_GEMM_BF16, K_GEMM_F16, K_GEMM_FP8, K_GEMM_I8, K_GEMM_TF32, K_MM_U32, K_QSORT, K_SHA256,
    F_NO_LOAD_SYNC, F_NO_STORE_ADDR_SYNC, F_NO_STORE_DATA_SYNC, F_STORE_DATA_SYNC,
    NO_FAULT_UNIT, UNIT_OFFSETS, MM_BATCHED, MM_GROUPED, MM_B_TRANSPOSED, MM_OUT_BF16, MM_OUT_F16, MM_SCALE_ROWWISE, MM_SCALE_TENSOR, PLAN_BERNOULLI, PLAN_NONE, PLAN_TABLE, CoastError, FaultPlan, LaunchDesc, Runtime, Stats,
    fault_entry, lib_path, load_library, parse_opt_passes,
)
from .build import build_library  # noqa: F401

__all__ = ["Runtime", "FaultPlan", "Stats", "CoastError", "build_library", "load_library", "parse_opt_passes"]
