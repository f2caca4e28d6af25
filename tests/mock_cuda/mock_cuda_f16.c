/*
 * mock_cuda_f16.c -- the mock libcuda.so.1 of tests/mock_cuda/mock_cuda.c, plus FLOAT16 tensor maps and one record of every
 * map's data type.
 *
 * TEST INFRASTRUCTURE ONLY (tests/test_gemm_f16_host_logic.py builds it).  Every call behaves and is logged exactly as in
 * mock_cuda.c, which takes no FLOAT16 map.  A FLOAT16 map is checked as a BFLOAT16 one (the same 2-byte element rules), and
 * every map that is encoded is followed by one more line,
 *   {"op":"tmap_dt","dt":<CUtensorMapDataType>}
 * so a test can pin the data type GEMM_F16's maps carry and compare everything else with a GEMM_BF16 launch.
 */
#define cuTensorMapEncodeTiled mock_cuda_encode_logged
#include "mock_cuda.c"
#undef cuTensorMapEncodeTiled

CUresult cuTensorMapEncodeTiled(CUtensorMap* map, CUtensorMapDataType dt, cuuint32_t rank, void* addr, const cuuint64_t* gdim,
                                const cuuint64_t* gstr, const cuuint32_t* box, const cuuint32_t* estr, CUtensorMapInterleave il,
                                CUtensorMapSwizzle swz, CUtensorMapL2promotion l2, CUtensorMapFloatOOBfill oob) {
    const CUtensorMapDataType checked = dt == CU_TENSOR_MAP_DATA_TYPE_FLOAT16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : dt;
    CUresult r = mock_cuda_encode_logged(map, checked, rank, addr, gdim, gstr, box, estr, il, swz, l2, oob);
    if (r == CUDA_SUCCESS) LOG("{\"op\":\"tmap_dt\",\"dt\":%d}", (int)dt);
    return r;
}
