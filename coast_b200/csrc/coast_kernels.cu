// coast_kernels.cu -- the sm_90a device module of libcoast_rt.so.
// Built to a cubin (nvcc -cubin -gencode arch=compute_90a,code=sm_90a -lineinfo), embedded into the
// host library as a byte array and loaded with cuModuleLoadData; every kernel is extern "C" so the
// runtime can look it up by name.
#include "xmr_common.cuh"
#include "xmr_util.cuh"
#include "xmr_sha256.cuh"
#include "xmr_aes128.cuh"
#include "xmr_crc16.cuh"
#include "xmr_mm.cuh"
#include "xmr_mm_tiled.cuh"
#include "xmr_gemm_tf32.cuh"
#include "xmr_mm_tc.cuh"
#include "xmr_qsort.cuh"
#include "xmr_chstone_sha.cuh"
#include "xmr_ragged.cuh"
