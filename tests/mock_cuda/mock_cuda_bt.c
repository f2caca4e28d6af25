/*
 * mock_cuda_bt.c -- mock_cuda.c with bfloat16 tensor maps (as mock_cuda_bf16.c) that also logs where each map starts.
 *
 * TEST INFRASTRUCTURE ONLY (tests/test_mm_bt_host_logic.py builds it into a temp dir as libcuda.so.1).  A transposed-B launch
 * differs from a B launch in the buffer B's map describes (the caller's d_aux instead of scratch), which the "tmap" lines do
 * not show; so every map is first logged as {"op":"tmap_at","addr":...}.  Then it is handled as mock_cuda_bf16.c handles it: a
 * bfloat16 map is logged as "tmap16" and handed on as the same bytes in 4-byte elements, every other map passes through, so
 * each check of mock_cuda.c applies.
 */
#include <cuda.h>
#define cuTensorMapEncodeTiled mock_encode_tiled_base
#include "mock_cuda.c"
#undef cuTensorMapEncodeTiled

CUresult cuTensorMapEncodeTiled(CUtensorMap* map, CUtensorMapDataType dt, cuuint32_t rank, void* addr, const cuuint64_t* gdim,
                                const cuuint64_t* gstr, const cuuint32_t* box, const cuuint32_t* estr, CUtensorMapInterleave il,
                                CUtensorMapSwizzle swz, CUtensorMapL2promotion l2, CUtensorMapFloatOOBfill oob) {
    LOG("{\"op\":\"tmap_at\",\"addr\":%llu}", (unsigned long long)(uintptr_t)addr);
    if (dt != CU_TENSOR_MAP_DATA_TYPE_BFLOAT16) return mock_encode_tiled_base(map, dt, rank, addr, gdim, gstr, box, estr, il, swz, l2, oob);
    if (rank < 1 || rank > 5) return bad("tensor map rank");
    if (gdim[0] % 2u || box[0] % 2u) return bad("bfloat16 tensor map: odd inner extent or box");
    cuuint64_t d[5];
    cuuint32_t b[5];
    size_t box_bytes = 2;
    for (cuuint32_t i = 0; i < rank; ++i) { d[i] = gdim[i]; b[i] = box[i]; box_bytes *= box[i]; }
    d[0] /= 2u; b[0] /= 2u;
    LOG("{\"op\":\"tmap16\",\"rank\":%u,\"elem\":2,\"dim0\":%llu,\"dim1\":%llu,\"box0\":%u,\"box1\":%u,\"box_bytes\":%zu,\"swizzle\":%d}", rank,
        (unsigned long long)gdim[0], (unsigned long long)(rank > 1 ? gdim[1] : 1), box[0], rank > 1 ? box[1] : 1, box_bytes, (int)swz);
    return mock_encode_tiled_base(map, CU_TENSOR_MAP_DATA_TYPE_UINT32, rank, addr, d, gstr, b, estr, il, swz, l2, oob);
}
