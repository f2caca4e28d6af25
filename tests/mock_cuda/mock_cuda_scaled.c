/*
 * mock_cuda_scaled.c -- the mock libcuda.so.1 of tests/mock_cuda/mock_cuda.c, plus one record per scaled GEMM_FP8 launch.
 *
 * TEST INFRASTRUCTURE ONLY (tests/test_gemm_fp8_scaled_host_logic.py builds it).  Every call behaves and is logged exactly as
 * in mock_cuda.c; a launch of an xmr_scaled_* function is followed by one more line,
 *   {"op":"scales","name":...,"sa":<d_scale_a>,"sb":<d_scale_b>}
 * with the two kernel parameters after the tensor maps (grouped kernels: after ro and the group block), so a test can pin the
 * parameter order and the pointers the kernel receives.
 */
#define cuLaunchKernel mock_cuda_launch_logged
#include "mock_cuda.c"
#undef cuLaunchKernel

CUresult cuLaunchKernel(CUfunction f, unsigned gx, unsigned gy, unsigned gz, unsigned bx, unsigned by, unsigned bz,
                        unsigned smem, CUstream s, void** params, void** extra) {
    CUresult r = mock_cuda_launch_logged(f, gx, gy, gz, bx, by, bz, smem, s, params, extra);
    const mock_fn* fn = (const mock_fn*)f;
    if (r == CUDA_SUCCESS && !strncmp(fn->name, "xmr_scaled_", 11)) {
        const int at = strstr(fn->name, "_grp_") ? 5 : 3;
        LOG("{\"op\":\"scales\",\"name\":\"%s\",\"sa\":%llu,\"sb\":%llu}", fn->name, (unsigned long long)*(const uintptr_t*)params[at],
            (unsigned long long)*(const uintptr_t*)params[at + 1]);
    }
    return r;
}
